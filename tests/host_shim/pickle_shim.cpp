// TEST INFRASTRUCTURE: compiles the function path's pickle codec (pickle_device.cuh: the decoder, the runner's call
// rules, the four handlers and the result encoder) for the host, so that it can be compared with cloudpickle and the
// oracle's runner loop on a CPU (tests/test_pickle_on_host.py).
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
#include "../../beta9_b200/csrc/pickle_device.cuh"

// n blobs blob[off[i] .. off[i+1]) under `handler` (0 identity, 1 crc32, 2 vadd_f32, 3 json_sum). out == nullptr: fills
// status[i] and out_off (n + 1 entries: the result sizes as offsets) and returns the total. Otherwise writes result i at
// out[out_off[i] .. out_off[i+1]).
extern "C" uint64_t b9_pk_batch(const uint8_t* blob, const uint64_t* off, uint32_t n, int handler, uint8_t* status, uint8_t* out,
                                uint64_t* out_off) {
    static uint32_t table[256];
    for (uint32_t i = 0; i < 256; ++i) table[i] = b9::crc_table_entry(i);
    std::vector<uint8_t> mem(sizeof(b9::PkScratch));
    b9::PkScratch& S = *reinterpret_cast<b9::PkScratch*>(mem.data());
    uint64_t total = 0;
    for (uint32_t i = 0; i < n; ++i) {
        const uint8_t* p = blob + off[i];
        const b9::PkPlan pl = b9::pk_prepare(p, (uint32_t)(off[i + 1] - off[i]), handler, S, table);
        status[i] = pl.status;
        if (!out) { out_off[i] = total; total += pl.out_len; continue; }
        if (pl.out_len) b9::pk_write(p, S, pl, out + out_off[i]);
        total += pl.out_len;
    }
    if (!out) out_off[n] = total;
    return total;
}
