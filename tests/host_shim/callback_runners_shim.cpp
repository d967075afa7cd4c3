// TEST INFRASTRUCTURE: compiles the runners' callback writers (callback_runners.cuh: the endpoint record's T(E), the
// function result's json.dumps over the pickle pass's value graph, the callback_url rule) for the host, so that
// tests/test_callback_runners_on_host.py can compare them with json.dumps and the oracle on a CPU.
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
#include "../../beta9_b200/csrc/callback_runners.cuh"

extern "C" {

// T(E) into out (out == nullptr: its length only)
uint64_t b9_cbr_endpoint(const uint8_t* e, uint32_t n, uint8_t* out) { return b9::cbr_endpoint_body(e, n, out); }

// One pickled task under `handler`, as the function runner's callback pass settles it. Returns -1 when the pass does not
// complete the task (status != ST_OK: the record's own kind is HOST), else the CBR_* kind (0 POST, 1 UNSENDABLE, 2 HOST).
// For POST: D in out[0, *d_len) (cap bytes of room) and the callback_url's bytes at out[*d_len, + *u_len).
int b9_cbr_function(const uint8_t* blob, uint32_t len, int handler, uint8_t* out, uint32_t cap, uint32_t* d_len, uint32_t* u_len) {
    static uint32_t table[256];
    for (uint32_t i = 0; i < 256; ++i) table[i] = b9::crc_table_entry(i);
    std::vector<uint8_t> mem(sizeof(b9::PkScratch));
    b9::PkScratch& S = *reinterpret_cast<b9::PkScratch*>(mem.data());
    *d_len = 0; *u_len = 0;
    const b9::PkPlan pl = b9::pk_prepare(blob, len, handler, S, table);
    if (pl.status != b9::ST_OK) return -1;
    std::vector<uint8_t> rec(pl.out_len);
    b9::pk_write(blob, S, pl, rec.data());                        // (as the pass does before the callback: it reuses the stack)
    const int root = b9::pk_decode(blob, len, S);
    const int u = b9::cbr_callback_url(blob, S, root);
    if (u == -2) return b9::CBR_HOST;
    b9::CbrW w; w.o = nullptr; w.n = 0;
    const uint8_t k = b9::cbr_kind(b9::cbr_result(w, blob, S, pl));
    if (k != b9::CBR_POST) return k;
    uint32_t us = 0, un = 0;
    if (u >= 0) b9::pk_data(blob, S.node[u].x, &us, &un);
    if ((uint64_t)w.n + un > cap) return -2;
    *d_len = w.n;
    w.o = out; w.n = 0;
    b9::cbr_result(w, blob, S, pl);
    memcpy(out + *d_len, blob + us, un);
    *u_len = un;
    return k;
}

}
