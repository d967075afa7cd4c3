// TEST INFRASTRUCTURE: compiles the endpoint drain's sequential half (endpoint_device.cuh: the response rules and
// rendering, over the HTTP-body parser and the four handlers) for the host, so that it can be compared with the oracle's
// endpoint request (oracle/pyoracle/endpoint.py) on a CPU (tests/test_endpoint_on_host.py).
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
#include "../../beta9_b200/csrc/endpoint_device.cuh"

// n bodies blob[off[i] .. off[i+1]) with slot flags flags[i], under `handler` (0 identity, 1 crc32, 2 vadd_f32,
// 3 json_sum), as the kernel treats one task. out == nullptr: fills status[i], has[i] and out_off (n + 1 entries: the
// record sizes as offsets) and returns the total. Otherwise writes record i at out[out_off[i] .. out_off[i+1]).
extern "C" uint64_t b9_ep_batch(const uint8_t* blob, const uint64_t* off, const uint8_t* flags, uint32_t n, int handler,
                                uint8_t* status, uint8_t* has, uint8_t* out, uint64_t* out_off) {
    static uint32_t table[256];
    for (uint32_t i = 0; i < 256; ++i) table[i] = b9::crc_table_entry(i);
    uint64_t total = 0;
    for (uint32_t i = 0; i < n; ++i) {
        const uint8_t* p = blob + off[i];
        const uint32_t len = (uint32_t)(off[i + 1] - off[i]);
        b9::TaskRec rec; memset(&rec, 0, sizeof rec);
        rec.status = b9::ST_UNSUPPORTED;
        if (b9::endpoint_accepts(flags[i])) b9::endpoint_phase_a(handler, p, b9::parse_payload(p, len, true), rec, table);
        status[i] = rec.status; has[i] = rec.has;
        const uint32_t olen = rec.has ? rec.out_len : 0u;
        if (!out) { out_off[i] = total; total += olen; continue; }
        if (olen) {
            if (rec.mode == b9::EM_COPY) memcpy(out + out_off[i], p + rec.src_off, rec.src_len);
            else b9::endpoint_emit(p, rec, out + out_off[i]);
        }
        total += olen;
    }
    if (!out) out_off[n] = total;
    return total;
}
