// callback_sign_kernel (b9_set_callback_policy): the callback kind and signature of every record of a task-queue drain,
// run on the drain stream after drain3_kernel (and the pickle pass), compiled as a translation unit of its own.
//
// Why not in b9gpu.cu: NVVM decides inlining for a whole module, and the SHA-256 round constants are a new __constant__
// array, so this kernel in b9gpu.cu's module could change how the drain kernels compile (wire_full.cu measured that). The
// device headers are included inside an anonymous namespace, as function_drain.cu does. The host half of the signing
// (the key's midstates, the drain's tail and the digest of {"data": {}}) is the same header's code, called from here.
#include <stdint.h>
#include <string.h>
#include <algorithm>
#include <cuda_runtime.h>

#pragma nv_diag_suppress 177     // (the headers' functions this kernel does not use: "declared but never referenced")
namespace {
#define B9_CALLBACK_KWARGS 1
#include "drain_kernel.cuh"
#include "callback_sign.cuh"
}

// the key's ipad / opad midstates, computed once per b9_set_callback_policy
void callback_midstates(const uint8_t* key, uint32_t key_len, uint32_t mid[16]) { b9::cb_midstates(key, key_len, mid); }

// b9gpu.cu's b9::DrainArgs comes from the same header as this file's copy; args_size guards that. `args` is the drain
// launch's argument block with tile_tasks as launch_drain3 chose it. keyed = 0: kinds only, every digest zero.
cudaError_t launch_callback_sign(const void* args, size_t args_size, const uint32_t mid[16], int keyed, int64_t ts,
                                 uint8_t* kind, uint8_t* digest, int sm_count, cudaStream_t s) {
    if (args_size != sizeof(b9::DrainArgs)) return cudaErrorInvalidValue;
    const b9::DrainArgs& a = *static_cast<const b9::DrainArgs*>(args);
    if (a.n_tasks == 0) return cudaSuccess;
    b9::CbSign sg;
    b9::cb_sign_init(sg, mid, ts);
    uint32_t e[8];
    b9::cb_sign_record(sg, reinterpret_cast<const uint8_t*>("{}"), 2, e);          // {"data": {}}
    uint8_t eb[32];
    for (int i = 0; i < 8; ++i) { eb[4 * i] = (uint8_t)(e[i] >> 24); eb[4 * i + 1] = (uint8_t)(e[i] >> 16); eb[4 * i + 2] = (uint8_t)(e[i] >> 8); eb[4 * i + 3] = (uint8_t)e[i]; }
    uint4 e0, e1;
    memcpy(&e0, eb, 16); memcpy(&e1, eb + 16, 16);
    int per_sm = 0;
    cudaError_t err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, b9::callback_sign_kernel, 128, 0);
    if (err != cudaSuccess) return err;
    const uint32_t grid = (uint32_t)std::min<uint64_t>((a.n_tasks + 127u) / 128u, (uint64_t)std::max(per_sm, 1) * (uint64_t)sm_count);
    b9::callback_sign_kernel<<<grid, 128, 0, s>>>(a, sg, keyed ? 1u : 0u, e0, e1, kind, reinterpret_cast<uint4*>(digest));
    return cudaGetLastError();
}
