// TEST INFRASTRUCTURE: compiles the signature half of the user-handler drain (include/b9gpu_handler.cuh: the call's
// sources, CPython's binding, phase A and B around a handler with B9H_SIGNATURE) and the example handlers that declare
// one (examples/handlers/handlers.cuh) for the host, so that tests/test_user_signature_on_host.py can compare them with
// their Python twins run through the oracle's loops on a CPU. `Probe` exercises every parameter kind.
#include <stdint.h>
#include <string.h>
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __restrict__
#define __constant__ static const
static inline float __uint_as_float(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline uint32_t __float_as_uint(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline float __fadd_rn(float a, float b) { volatile float z = a + b; return z; }     // IEEE binary32, round to nearest even
#include "../../examples/handlers/handlers.cuh"

// def probe(a, /, b, c=<unset>, *rest, d, e=<unset>): "|".join(tag(v) for v in (a, b, c, d, e, *rest))
// tag: "-" for an optional parameter left unset, a str's own text, else the name of the value's type
struct Probe {
    B9H_SIGNATURE(B9H_POS_ONLY("a"), B9H_POS_OR_KW("b"), B9H_POS_OR_KW_OPT("c"), B9H_VAR_POS("rest"), B9H_KW_ONLY("d"),
                  B9H_KW_ONLY_OPT("e"));
    template <class Out> static void tag(const b9h::Arg& v, Out& out) {
        static const char* const names[] = {"", "int", "float", "bool", "NoneType", "list", "dict"};
        const int k = v.kind();
        if (k == b9h::STR) b9_examples::put_str(v, out);
        else b9_examples::put_ascii(names[k], out);
    }
    template <class Out> static int call(const b9h::Call& c, Out& out) {
        out.str_begin();
        const int order[] = {0, 1, 2, 4, 5};
        for (int j = 0; j < 5; ++j) {
            if (j) out.cp('|');
            if (c.has(order[j])) tag(c[order[j]], out);
            else out.cp('-');
        }
        b9h::Items it = c.rest();
        b9h::Arg x;
        while (it.next(x)) { out.cp('|'); tag(x, out); }
        out.str_end();
        return 0;
    }
};

template <class H, int R>
static uint64_t batch(const uint8_t* blob, const uint64_t* off, const uint8_t* flags, const uint8_t* ids, uint32_t n,
                      uint8_t* status, uint8_t* has, int64_t* value, uint8_t* out, uint64_t* out_off) {
    uint64_t total = 0;
    for (uint32_t i = 0; i < n; ++i) {
        const uint8_t* p = blob + off[i];
        const uint32_t len = (uint32_t)(off[i + 1] - off[i]);
        b9h::rec_t<H> rec;
        b9h::task_phase_a<H, R>(p, len, flags[i], ids + 16 * i, rec);
        status[i] = rec.status; has[i] = rec.has; value[i] = rec.status == b9::ST_ERROR ? rec.value : 0;
        const uint32_t olen = rec.has ? rec.out_len : 0u;
        if (!out) { out_off[i] = total; total += olen; continue; }
        if (olen && !b9h::task_phase_b<H, R>(p, rec, out + out_off[i])) { status[i] = 255; has[i] = 0; }   // (two passes disagree)
        total += olen;
    }
    if (!out) out_off[n] = total;
    return total;
}

// As b9_uh_batch (user_handler_shim.cpp), for handler 0 greet, 1 join, 2 field_sum, 3 Probe.
extern "C" uint64_t b9_us_batch(const uint8_t* blob, const uint64_t* off, const uint8_t* flags, const uint8_t* ids, uint32_t n,
                                int handler, int rendering, uint8_t* status, uint8_t* has, int64_t* value, uint8_t* out, uint64_t* out_off) {
#define B9_US_CASE(k, H) \
    case k: return rendering ? batch<H, b9h::ENDPOINT>(blob, off, flags, ids, n, status, has, value, out, out_off) \
                             : batch<H, b9h::TASK_QUEUE>(blob, off, flags, ids, n, status, has, value, out, out_off);
    switch (handler) {
    B9_US_CASE(0, b9_examples::Greet)
    B9_US_CASE(1, b9_examples::Join)
    B9_US_CASE(2, b9_examples::FieldSum)
    default: break;
    }
    return rendering ? batch<Probe, b9h::ENDPOINT>(blob, off, flags, ids, n, status, has, value, out, out_off)
                     : batch<Probe, b9h::TASK_QUEUE>(blob, off, flags, ids, n, status, has, value, out, out_off);
#undef B9_US_CASE
}
