// TEST INFRASTRUCTURE: compiles the generic half of the user-handler drain (include/b9gpu_handler.cuh: the parse a
// rendering accepts, phase A with the counting sink, phase B with the writing sink) and the example handlers
// (examples/handlers/handlers.cuh) for the host, so that they can be compared with their Python twins run through the
// oracle's loops on a CPU (tests/test_user_handler_on_host.py).
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

template <class H, int R>
static uint64_t batch(const uint8_t* blob, const uint64_t* off, const uint8_t* flags, const uint8_t* ids, uint32_t n,
                      uint8_t* status, uint8_t* has, int64_t* value, uint8_t* out, uint64_t* out_off) {
    uint64_t total = 0;
    for (uint32_t i = 0; i < n; ++i) {
        const uint8_t* p = blob + off[i];
        const uint32_t len = (uint32_t)(off[i + 1] - off[i]);
        b9h::UserRec rec;
        b9h::user_phase_a<H, R>(p, b9h::user_parse<R>(p, len, flags[i], ids + 16 * i), rec);
        status[i] = rec.status; has[i] = rec.has; value[i] = rec.status == b9::ST_ERROR ? rec.value : 0;
        const uint32_t olen = rec.has ? rec.out_len : 0u;
        if (!out) { out_off[i] = total; total += olen; continue; }
        if (olen && !b9h::user_phase_b<H, R>(p, rec, out + out_off[i])) { status[i] = 255; has[i] = 0; }   // (two passes disagree)
        total += olen;
    }
    if (!out) out_off[n] = total;
    return total;
}

// n tasks blob[off[i] .. off[i+1]) with slot flags flags[i] and 16-byte ids, under example handler `handler`
// (0 echo_str, 1 crc32_str, 2 word_count, 3 prod) and `rendering` (0 task-queue, 1 endpoint), as the kernel treats one
// task. out == nullptr: fills status[i], has[i], value[i] (an ERROR's B9_EXC_* bit) and out_off (n + 1 entries: the record
// sizes as offsets) and returns the total. Otherwise writes record i at out[out_off[i] .. out_off[i+1]).
extern "C" uint64_t b9_uh_batch(const uint8_t* blob, const uint64_t* off, const uint8_t* flags, const uint8_t* ids, uint32_t n,
                                int handler, int rendering, uint8_t* status, uint8_t* has, int64_t* value, uint8_t* out, uint64_t* out_off) {
#define B9_UH_CASE(k, H) \
    case k: return rendering ? batch<H, b9h::ENDPOINT>(blob, off, flags, ids, n, status, has, value, out, out_off) \
                             : batch<H, b9h::TASK_QUEUE>(blob, off, flags, ids, n, status, has, value, out, out_off);
    switch (handler) {
    B9_UH_CASE(0, b9_examples::EchoStr)
    B9_UH_CASE(1, b9_examples::Crc32Str)
    B9_UH_CASE(2, b9_examples::WordCount)
    default: break;
    }
    return rendering ? batch<b9_examples::Prod, b9h::ENDPOINT>(blob, off, flags, ids, n, status, has, value, out, out_off)
                     : batch<b9_examples::Prod, b9h::TASK_QUEUE>(blob, off, flags, ids, n, status, has, value, out, out_off);
#undef B9_UH_CASE
}
