// b9_cancel: marks pending tasks cancelled by id — what StopTasks (pkg/api/v1/task.go:333-398) does to a task's state,
// after which TaskQueuePop skips it (pkg/abstractions/taskqueue/taskqueue.go:238-270). Plain C++ behind CUDA qualifiers:
// tests/host_shim/cancel_shim.cpp builds the key order, the host sort and the fence search with g++.
//
// The requested ids are sorted and de-duplicated on the host; one device thread per ring slot looks its id up in them.
// Key order is the one decision both sides share: the 16 id bytes read as two big-endian u64 (hi = bytes 0..7), so that
// key order is memcmp order. cancel_key() builds a key from the four little-endian 32-bit words a uint4 load of the id
// gives (bytes 4i..4i+3 in word i), on the host from memcpy'd words, on the device from the slot's uint4.
#pragma once
#include <stdint.h>
#include <string.h>
#include <algorithm>
#include <vector>

namespace b9 {

constexpr uint32_t CANCEL_MARKED  = 0x01u;   // == B9_CANCEL_MARKED (include/b9gpu.h)
constexpr uint32_t CANCEL_ALREADY = 0x02u;   // == B9_CANCEL_ALREADY
constexpr uint32_t CANCEL_CLAIMED = 0x04u;   // == B9_CANCEL_CLAIMED
constexpr uint32_t CANCEL_FENCE_MAX = 2048;  // keys of the shared-memory fence: 32 KiB per CTA at most

struct alignas(16) CancelKey { uint64_t hi, lo; };

__host__ __device__ __forceinline__ uint32_t cancel_bswap32(uint32_t v) {
    return (v >> 24) | ((v >> 8) & 0xFF00u) | ((v << 8) & 0xFF0000u) | (v << 24);
}
__host__ __device__ __forceinline__ CancelKey cancel_key(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3) {
    CancelKey k;
    k.hi = ((uint64_t)cancel_bswap32(w0) << 32) | cancel_bswap32(w1);
    k.lo = ((uint64_t)cancel_bswap32(w2) << 32) | cancel_bswap32(w3);
    return k;
}
__host__ __device__ __forceinline__ bool cancel_key_less(const CancelKey& a, const CancelKey& b) {
    return a.hi < b.hi || (a.hi == b.hi && a.lo < b.lo);
}
__host__ __device__ __forceinline__ bool cancel_key_eq(const CancelKey& a, const CancelKey& b) { return a.hi == b.hi && a.lo == b.lo; }

// every `stride`-th key goes into the fence; the smallest power of two that keeps the fence within CANCEL_FENCE_MAX
__host__ __device__ __forceinline__ uint32_t cancel_fence_stride(uint32_t n_keys) {
    uint32_t s = 1;
    while ((n_keys + s - 1u) / s > CANCEL_FENCE_MAX) s <<= 1;
    return s;
}

// Index of `k` in the sorted, unique keys[0, n), or -1. fence[j] = keys[j * stride] for j < ceil(n / stride): the fence
// narrows the search to one stride of keys (log2(n_fence) steps on the fence, log2(stride) on keys[]).
__host__ __device__ __forceinline__ int64_t cancel_find(const CancelKey* fence, uint32_t n_fence, const CancelKey* keys, uint32_t n,
                                                        uint32_t stride, const CancelKey& k) {
    uint32_t lo = 0, hi = n_fence;                       // first fence key > k
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (cancel_key_less(k, fence[mid])) hi = mid; else lo = mid + 1u;
    }
    if (lo == 0) return -1;
    const uint32_t base = (lo - 1u) * stride;
    if (cancel_key_eq(fence[lo - 1u], k)) return (int64_t)base;
    uint32_t a = base + 1u;                               // first key >= k in (base, end)
    const uint32_t end = (n - base > stride) ? base + stride : n;
    uint32_t b = end;
    while (a < b) {
        const uint32_t mid = (a + b) >> 1;
        if (cancel_key_less(keys[mid], k)) a = mid + 1u; else b = mid;
    }
    return (a < end && cancel_key_eq(keys[a], k)) ? (int64_t)a : -1;
}

// host side: the key of 16 raw id bytes
inline CancelKey cancel_key_of(const uint8_t* id) {
    uint32_t w[4];
    memcpy(w, id, 16);
    return cancel_key(w[0], w[1], w[2], w[3]);
}

// keys := the n ids sorted and de-duplicated; which[i] := index in keys of the caller's id i
inline void cancel_sort_unique(const uint8_t* ids, uint32_t n, std::vector<CancelKey>& keys, std::vector<uint32_t>& which) {
    struct Item { CancelKey k; uint32_t i; };
    std::vector<Item> items(n);
    for (uint32_t i = 0; i < n; ++i) items[i] = Item{cancel_key_of(ids + (size_t)i * 16), i};
    std::sort(items.begin(), items.end(), [](const Item& a, const Item& b) { return cancel_key_less(a.k, b.k); });
    keys.clear(); keys.reserve(n);
    which.assign(n, 0);
    for (uint32_t j = 0; j < n; ++j) {
        if (keys.empty() || !cancel_key_eq(keys.back(), items[j].k)) keys.push_back(items[j].k);
        which[items[j].i] = (uint32_t)keys.size() - 1u;
    }
}

#ifdef __CUDACC__
// One thread per slot of the pending window [first_task, first_task + n) (mod slot_mask + 1), grid-stride. Its first
// n_claimed slots are a drain's claimed window: looked up only, reported CLAIMED. Every other hit that is not cancelled yet
// gets B9_TF_CANCELLED in its header word (the write expire_kernel makes); `count` += slots marked.
// Dynamic shared memory: n_fence keys.
__global__ void __launch_bounds__(256) cancel_kernel(uint64_t* __restrict__ hdr, const uint4* __restrict__ ids, uint32_t slot_mask,
                                                     uint64_t first_task, uint32_t n_claimed, uint32_t n,
                                                     const CancelKey* __restrict__ keys, uint32_t n_keys, uint32_t stride, uint32_t n_fence,
                                                     uint32_t* __restrict__ outcome, unsigned long long* __restrict__ count) {
    extern __shared__ CancelKey fence[];
    for (uint32_t j = threadIdx.x; j < n_fence; j += blockDim.x) fence[j] = keys[(size_t)j * stride];
    __syncthreads();
    for (uint32_t base = blockIdx.x * blockDim.x; base < n; base += gridDim.x * blockDim.x) {   // (block-uniform: whole warps ballot)
        const uint32_t i = base + threadIdx.x;
        bool marked = false;
        if (i < n) {
            const uint32_t slot = (uint32_t)((first_task + i) & slot_mask);
            const uint4 w = ids[slot];
            const int64_t at = cancel_find(fence, n_fence, keys, n_keys, stride, cancel_key(w.x, w.y, w.z, w.w));
            if (at >= 0) {
                if (i < n_claimed) {
                    atomicOr(outcome + at, CANCEL_CLAIMED);
                } else {
                    const uint64_t h = hdr[slot];
                    if ((h >> 32) & 1u) {
                        atomicOr(outcome + at, CANCEL_ALREADY);
                    } else {
                        hdr[slot] = h | (1ull << 32);
                        atomicOr(outcome + at, CANCEL_MARKED);
                        marked = true;
                    }
                }
            }
        }
        const uint32_t m = __ballot_sync(0xffffffffu, marked);
        if ((threadIdx.x & 31u) == 0u && m) atomicAdd(count, (unsigned long long)__popc(m));
    }
}
#endif

}  // namespace b9
