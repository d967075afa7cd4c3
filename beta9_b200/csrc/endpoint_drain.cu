// endpoint_drain_kernel (b9_endpoint_drain_launch): answers HTTP request bodies with the endpoint runner's response bytes
// (endpoint_device.cuh), compiled as a translation unit of its own.
//
// Why not in b9gpu.cu: NVVM decides inlining for a whole module, so a new kernel that calls the JSON and sum helpers
// would change how the drain kernels compile (wire_full.cu measured that). The device headers are included inside an
// anonymous namespace, as function_drain.cu does: their out-of-line __device__ functions get host-side definitions in
// every translation unit that includes them, which would clash with b9gpu.cu's at link time.
//
// Shape: persistent warps take warp-tiles of EP_TILE consecutive slots from the control block's ticket, one task per
// lane. Each lane reads its slot, parses its body (parse_payload, http = true) and runs phase A; a ballot over the
// non-cancelled lanes gives the record indices (count mode: plus the ready tasks before the tile, from
// tile_count_kernel run with EP_TILE), one warp scan of the record lengths and one warp_reserve_bytes per tile
// (drain_kernel.cuh, rounded up to 16 bytes as it says) place the bytes. Records that are the argument's token verbatim (identity's
// common string) are copied by the whole warp, one record after the other; every other record is written by its lane.
//
// The control ring (drain_kernel.cuh, D3_CTL_RING): this kernel zeroes the next launch's entry itself, as drain3_kernel
// does, so that back-to-back launches of either kind need no memset between them. It is never launched as a programmatic
// dependent and the host does not launch the next drain as its dependent, so at its start the previous launch has
// completed and nothing reads that entry any more.
#include <stdint.h>
#include <algorithm>
#include <cuda_runtime.h>

#pragma nv_diag_suppress 177     // (the headers' functions this kernel does not use: "declared but never referenced")
namespace {
#include "drain_kernel.cuh"
#include "endpoint_device.cuh"
}

namespace {

constexpr uint32_t EP_TILE = 32;       // slots per warp-tile: one per lane
constexpr int EP_WARPS = 4;            // warps per CTA

template <int H>
__global__ void __launch_bounds__(EP_WARPS * 32) endpoint_drain_kernel(b9::DrainArgs a) {
    __shared__ uint32_t s_crc[256];
    if (H == 1) {
        for (int i = threadIdx.x; i < 256; i += blockDim.x) s_crc[i] = b9::crc_table_entry((uint32_t)i);
        __syncthreads();
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *a.ctl_next = b9::DrainCtl{};
    const int lane = threadIdx.x & 31;
    for (;;) {
        unsigned long long tile = 0;
        if (lane == 0) tile = atomicAdd(&a.out.ctl->ticket, 1ull);
        tile = __shfl_sync(0xffffffffu, tile, 0);
        if (tile >= a.n_tiles) break;
        const uint32_t i = (uint32_t)tile * EP_TILE + (uint32_t)lane;
        const bool in = i < a.n_tasks;
        const uint32_t slot = (uint32_t)((a.first_task + i) & a.slot_mask);
        const uint64_t h = in ? __ldg(a.hdr + slot) : 0ull;
        const bool live = in && !(b9::hdr_flags(h) & 1u);
        b9::TaskRec rec;
        rec.status = b9::ST_UNSUPPORTED; rec.has = 0; rec.mode = b9::EM_NONE; rec.ready = 1;
        rec.out_len = 0; rec.src_off = 0; rec.src_len = 0; rec.value = 0;
        const uint8_t* p = a.payload;
        if (live) {
            p = a.payload + __ldg(a.off + slot);
            if (b9::endpoint_accepts(b9::hdr_flags(h)))
                b9::endpoint_phase_a(H, p, b9::parse_payload(p, b9::hdr_len(h), true), rec, H == 1 ? s_crc : nullptr);
        }

        // ---- record index (ballot), bytes (scan) and ONE cursor add per warp-tile
        const uint32_t live_mask = __ballot_sync(0xffffffffu, live);
        const uint32_t base_cnt = a.count_mode ? b9::tile_ready_before(a, tile, EP_TILE) : (uint32_t)tile * EP_TILE;
        if (lane == 0 && tile == a.n_tiles - 1) a.out.ctl->total_cnt = base_cnt + __popc(live_mask);
        const uint32_t j = base_cnt + __popc(live_mask & ((1u << lane) - 1u));
        const uint32_t my = rec.has ? rec.out_len : 0u;
        const uint32_t incl = b9::warp_incl_scan(my, lane);
        const uint32_t tb = __shfl_sync(0xffffffffu, incl, 31);
        const b9::Reservation r = b9::warp_reserve_bytes(a.out, (tb + 15u) & ~15u, lane);
        const unsigned long long ob = r.base + (incl - my);
        if (live) {
            b9::store_record_id(a.out, j, a.ids + slot);
            b9::store_record(a.out, j, r.fits, ob, my, rec.status, rec.has);
        }
        if (!r.fits) continue;
        const bool copy = rec.has && rec.mode == b9::EM_COPY;
        if (rec.has && !copy) b9::endpoint_emit(p, rec, a.out.payload + ob);
        uint32_t cm = __ballot_sync(0xffffffffu, copy);
        const unsigned long long src = (unsigned long long)(uintptr_t)(p + rec.src_off);
        while (cm) {                                                       // the verbatim records, the whole warp on each
            const int q = __ffs(cm) - 1;
            cm &= cm - 1u;
            const uint8_t* s = (const uint8_t*)(uintptr_t)__shfl_sync(0xffffffffu, src, q);
            const unsigned long long d = __shfl_sync(0xffffffffu, ob, q);
            const uint32_t n = __shfl_sync(0xffffffffu, rec.src_len, q);
            b9::warp_copy(a.out.payload + d, s, n, lane);
        }
    }
}

template <int H>
cudaError_t launch(const b9::DrainArgs& a, int sm_count, cudaStream_t s) {
    int per_sm = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, endpoint_drain_kernel<H>, EP_WARPS * 32, 0);
    if (e != cudaSuccess) return e;
    const uint64_t ctas_needed = ((uint64_t)a.n_tiles + EP_WARPS - 1) / EP_WARPS;
    const uint32_t grid = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(ctas_needed, (uint64_t)std::max(per_sm, 1) * (uint64_t)sm_count));
    endpoint_drain_kernel<H><<<grid, EP_WARPS * 32, 0, s>>>(a);
    return cudaGetLastError();
}

}  // namespace

// b9gpu.cu's b9::DrainArgs comes from the same header as this file's copy, so their layouts are the same; args_size
// guards that. `args` is the drain launch's argument block; its tile_tasks must be EP_TILE (the count-mode prefixes are
// per tile of that size) and n_tiles the window's tiles of it.
cudaError_t launch_endpoint_drain(const void* args, size_t args_size, int handler, int sm_count, cudaStream_t s) {
    if (args_size != sizeof(b9::DrainArgs)) return cudaErrorInvalidValue;
    const b9::DrainArgs& a = *static_cast<const b9::DrainArgs*>(args);
    if (a.tile_tasks != EP_TILE || a.n_tiles != (a.n_tasks + EP_TILE - 1) / EP_TILE) return cudaErrorInvalidValue;
    switch (handler) {
    case 0: return launch<0>(a, sm_count, s);
    case 1: return launch<1>(a, sm_count, s);
    case 2: return launch<2>(a, sm_count, s);
    default: return launch<3>(a, sm_count, s);
    }
}
