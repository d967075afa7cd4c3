// wire_encode_kernel<true> (b9_wire_encode_full), compiled as a translation unit of its own.
//
// Why not in b9gpu.cu: NVVM decides inlining for a whole module, so a new kernel that calls the parser and the JSON helpers
// changes how the drain kernels compile. In b9gpu.cu's module this kernel raised drain3_kernel<0>'s (identity) stack
// frame from 880 to 896 bytes with 8 bytes of new spill stores, and json_sum's spills from 140 / 88 to 180 / 112 bytes.
// Here it has a module to itself, and b9gpu.cu's device code is what it was.
//
// The device headers are included inside an anonymous namespace: their kernels and out-of-line __device__ functions get
// host-side definitions in every translation unit that includes them, which would clash with b9gpu.cu's at link time.
// This file's copies are private to it.
#include <stdint.h>
#include <cuda_runtime.h>

#pragma nv_diag_suppress 177     // (the headers' functions this kernel does not use: "declared but never referenced")
namespace {
#include "wire_encode.cuh"
}

// b9gpu.cu's b9::WireArgs / b9::WireEnv come from the same header as this file's copies, so their layouts are the same;
// args_size guards that.
cudaError_t launch_wire_encode_full(const void* args, size_t args_size, const void* env, uint32_t grid, cudaStream_t s) {
    if (args_size != sizeof(b9::WireArgs)) return cudaErrorInvalidValue;
    b9::wire_encode_kernel<true><<<grid, 128, 0, s>>>(*static_cast<const b9::WireArgs*>(args), static_cast<const b9::WireEnv*>(env));
    return cudaGetLastError();
}
