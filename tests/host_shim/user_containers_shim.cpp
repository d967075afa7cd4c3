// TEST INFRASTRUCTURE: compiles the container calls of the user-handler sinks (include/b9gpu_handler.cuh) with the
// example handlers that return lists and dicts (examples/handlers/handlers.cuh) and the container script handler
// (tests/handlers/containers.cuh) for the host, so that tests/test_user_containers_on_host.py can compare them with their
// Python twins on a CPU. As contract_shim.cpp, phase B writes each record into a buffer of its counted length followed
// by guard bytes: a writing pass that wrote past the reservation shows.
#include <stdint.h>
#include <string.h>
#include <vector>
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
#include "../handlers/containers.cuh"

constexpr uint32_t GUARD = 64;
constexpr uint8_t GUARD_BYTE = 0xA5;

template <class H, int R>
static uint64_t batch(const uint8_t* blob, const uint64_t* off, const uint8_t* flags, const uint8_t* ids, uint32_t n,
                      uint8_t* status, uint8_t* has, int64_t* value, uint8_t* guard_ok, uint8_t* out, uint64_t* out_off) {
    uint64_t total = 0;
    std::vector<uint8_t> buf;
    for (uint32_t i = 0; i < n; ++i) {
        const uint8_t* p = blob + off[i];
        const uint32_t len = (uint32_t)(off[i + 1] - off[i]);
        b9h::rec_t<H> rec;
        b9h::task_phase_a<H, R>(p, len, flags[i], ids + 16 * i, rec);
        status[i] = rec.status; has[i] = rec.has; value[i] = rec.status == b9::ST_ERROR ? rec.value : 0; guard_ok[i] = 1;
        const uint32_t olen = rec.has ? rec.out_len : 0u;
        if (!out) { out_off[i] = total; total += olen; continue; }
        if (olen) {
            buf.assign(olen + GUARD, GUARD_BYTE);
            const bool ok = b9h::task_phase_b<H, R>(p, rec, buf.data());
            for (uint32_t k = olen; k < olen + GUARD; ++k) if (buf[k] != GUARD_BYTE) guard_ok[i] = 0;
            if (ok) memcpy(out + out_off[i], buf.data(), olen);
            else { status[i] = b9::ST_UNSUPPORTED; has[i] = 0; }        // as user_drain: the two passes disagreed
        }
        total += olen;
    }
    if (!out) out_off[n] = total;
    return total;
}

// As b9_ct_batch (contract_shim.cpp), for handler 0 tokens, 1 grid, 2 describe, 3 pick, 4 cscript. A record whose two
// passes disagreed is UNSUPPORTED without result bytes, as the kernel stores it.
extern "C" uint64_t b9_uc_batch(const uint8_t* blob, const uint64_t* off, const uint8_t* flags, const uint8_t* ids, uint32_t n,
                                int handler, int rendering, uint8_t* status, uint8_t* has, int64_t* value, uint8_t* guard_ok,
                                uint8_t* out, uint64_t* out_off) {
#define B9_UC_CASE(k, H) \
    case k: return rendering ? batch<H, b9h::ENDPOINT>(blob, off, flags, ids, n, status, has, value, guard_ok, out, out_off) \
                             : batch<H, b9h::TASK_QUEUE>(blob, off, flags, ids, n, status, has, value, guard_ok, out, out_off);
    switch (handler) {
    B9_UC_CASE(0, b9_examples::Tokens)
    B9_UC_CASE(1, b9_examples::Grid)
    B9_UC_CASE(2, b9_examples::Describe)
    B9_UC_CASE(3, b9_examples::Pick)
    B9_UC_CASE(4, b9_containers::CScript)
    default: return 0;
    }
#undef B9_UC_CASE
}
