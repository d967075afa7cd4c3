// pickle_pass_kernel (B9_DRAIN_PICKLE_FULL): the function path for every handler and plain Python values, run on the
// drain stream right after drain3_kernel, compiled as a translation unit of its own.
//
// Why not in b9gpu.cu: NVVM decides inlining for a whole module, so a new kernel that calls the JSON and sum helpers
// would change how the drain kernels compile (wire_full.cu measured that). The device headers are included inside an
// anonymous namespace, as wire_full.cu does: their out-of-line __device__ functions get host-side definitions in every
// translation unit that includes them, which would clash with b9gpu.cu's at link time.
//
// The pass visits the window's slots whose flags are exactly B9_TF_PICKLE (not cancelled, no HTTP_BODY, no TASK_MSG) and
// rewrites the records drain3_kernel left UNSUPPORTED; identity's one-str template stays the fast path. A slot's record
// index is the one drain3_kernel gave it. One warp per task, its lane 0 doing the sequential work against a PkScratch in
// the block's shared memory (28,744 bytes, plus the 1 KiB the SM reserves per block and crc32's 1 KiB table: seven
// blocks, i.e. seven tasks in flight, per SM). The pass is latency-bound: one thread of each resident warp works, about
// 900 on a 132-SM H100; scratch in global memory or a warp-cooperative decoder would keep more tasks in flight. Output
// bytes come from the same control block's cursor, one reserve_bytes per task (drain_kernel.cuh).
#include <stdint.h>
#include <algorithm>
#include <cuda_runtime.h>

#pragma nv_diag_suppress 177     // (the headers' functions this kernel does not use: "declared but never referenced")
namespace {
#include "drain_kernel.cuh"
#include "pickle_device.cuh"
}
static_assert(sizeof(b9::PkScratch) == 28744, "the scratch size and the occupancy above are stated for 28,744 bytes");

namespace {

template <int H>
__global__ void __launch_bounds__(32) pickle_pass_kernel(b9::DrainArgs a) {
    extern __shared__ __align__(16) uint8_t pk_smem[];
    __shared__ uint32_t s_crc[256];
    b9::PkScratch& S = *reinterpret_cast<b9::PkScratch*>(pk_smem);
    const int lane = threadIdx.x;
    if (H == 1) for (int i = lane; i < 256; i += 32) s_crc[i] = b9::crc_table_entry((uint32_t)i);
    __syncwarp();
    if (lane != 0) return;
    for (uint32_t i = blockIdx.x; i < a.n_tasks; i += gridDim.x) {
        const uint64_t h = a.hdr[(uint32_t)((a.first_task + i) & a.slot_mask)];
        if (b9::hdr_flags(h) != b9::B9_TF_PICKLE_BIT) continue;
        uint32_t j = i;                                            // the record index drain3_kernel gave the slot
        if (a.count_mode) {
            const uint32_t tile = i / a.tile_tasks;
            j = b9::tile_ready_before(a, tile, a.tile_tasks);
            for (uint32_t q = tile * a.tile_tasks; q < i; ++q) j += (b9::hdr_flags(a.hdr[(uint32_t)((a.first_task + q) & a.slot_mask)]) & 1u) ? 0u : 1u;
        }
        if (a.out.status[j] != b9::ST_UNSUPPORTED) continue;       // drain3_kernel settled it
        const uint8_t* p = a.payload + a.off[(uint32_t)((a.first_task + i) & a.slot_mask)];
        const b9::PkPlan pl = b9::pk_prepare(p, b9::hdr_len(h), H, S, s_crc);
        if (pl.status == b9::ST_UNSUPPORTED) continue;
        const b9::Reservation r = b9::reserve_bytes(a.out, (pl.out_len + 15u) & ~15u);
        if (r.fits && pl.out_len) b9::pk_write(p, S, pl, a.out.payload + r.base);
        b9::store_record(a.out, j, r.fits, r.base, pl.out_len, pl.status, pl.out_len ? 1 : 0);
    }
}

template <int H>
cudaError_t launch(const b9::DrainArgs& a, int sm_count, cudaStream_t s) {
    int per_sm = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, pickle_pass_kernel<H>, 32, sizeof(b9::PkScratch));
    if (e != cudaSuccess) return e;
    const uint32_t grid = (uint32_t)std::min<uint64_t>(a.n_tasks, (uint64_t)std::max(per_sm, 1) * (uint64_t)sm_count);
    pickle_pass_kernel<H><<<grid, 32, sizeof(b9::PkScratch), s>>>(a);
    return cudaGetLastError();
}

}  // namespace

// b9gpu.cu's b9::DrainArgs comes from the same header as this file's copy, so their layouts are the same; args_size
// guards that. `args` is the drain launch's argument block with tile_tasks as launch_drain3 chose it.
cudaError_t launch_pickle_pass(const void* args, size_t args_size, int handler, int sm_count, cudaStream_t s) {
    if (args_size != sizeof(b9::DrainArgs)) return cudaErrorInvalidValue;
    const b9::DrainArgs& a = *static_cast<const b9::DrainArgs*>(args);
    if (a.n_tasks == 0) return cudaSuccess;
    switch (handler) {
    case 0: return launch<0>(a, sm_count, s);
    case 1: return launch<1>(a, sm_count, s);
    case 2: return launch<2>(a, sm_count, s);
    default: return launch<3>(a, sm_count, s);
    }
}
