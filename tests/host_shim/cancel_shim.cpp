// TEST INFRASTRUCTURE: compiles b9_cancel's key order, host sort / de-duplication and fence search (cancel.cuh) for the
// host, so that tests/test_cancel_on_host.py can check them against Python's byte order and set membership on a CPU.
#include <stdint.h>
#include <string.h>
#define __device__
#define __host__
#define __forceinline__ inline
#include "../../beta9_b200/csrc/cancel.cuh"

// the key of one 16-byte id: out[0] = hi, out[1] = lo
extern "C" void b9_cx_key(const uint8_t* id, uint64_t* out) {
    const b9::CancelKey k = b9::cancel_key_of(id);
    out[0] = k.hi; out[1] = k.lo;
}

// sorts and de-duplicates n ids: keys_out [n][2] (hi, lo) of the unique keys, which[n]; returns the unique count
extern "C" uint32_t b9_cx_sort_unique(const uint8_t* ids, uint32_t n, uint64_t* keys_out, uint32_t* which) {
    std::vector<b9::CancelKey> keys; std::vector<uint32_t> w;
    b9::cancel_sort_unique(ids, n, keys, w);
    for (size_t j = 0; j < keys.size(); ++j) { keys_out[2 * j] = keys[j].hi; keys_out[2 * j + 1] = keys[j].lo; }
    memcpy(which, w.data(), (size_t)n * 4);
    return (uint32_t)keys.size();
}

// sorts the n request ids as b9_cancel does, builds the fence as cancel_kernel does, and looks up m query ids:
// at[i] = index of query i among the unique sorted keys, or -1. Returns the fence stride.
extern "C" uint32_t b9_cx_find(const uint8_t* ids, uint32_t n, const uint8_t* queries, uint32_t m, int64_t* at) {
    std::vector<b9::CancelKey> keys; std::vector<uint32_t> w;
    b9::cancel_sort_unique(ids, n, keys, w);
    const uint32_t nk = (uint32_t)keys.size(), stride = b9::cancel_fence_stride(nk), nf = (nk + stride - 1u) / stride;
    std::vector<b9::CancelKey> fence(nf);
    for (uint32_t j = 0; j < nf; ++j) fence[j] = keys[(size_t)j * stride];
    for (uint32_t i = 0; i < m; ++i) {
        uint32_t q[4];
        memcpy(q, queries + (size_t)i * 16, 16);                  // the words a uint4 load of the slot's id gives
        at[i] = b9::cancel_find(fence.data(), nf, keys.data(), nk, stride, b9::cancel_key(q[0], q[1], q[2], q[3]));
    }
    return stride;
}
