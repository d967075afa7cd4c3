// user_drain<H, R>: the drain kernel body for a user-written handler (include/b9gpu_handler.cuh, b9_handler_load).
// Included only by b9gpu_handler.cuh: B9_HANDLER instantiates it in the user's translation unit, which is compiled to
// an sm_90a cubin of its own and loaded at run time; libb9gpu.so holds none of it.
//
// The shape and the record rules are endpoint_drain_kernel's (endpoint_drain.cu): persistent warps of UD_WARPS-warp CTAs
// take warp-tiles of UD_TILE consecutive slots from the control block's ticket, one task per lane. Each lane parses its
// task (b9h::user_parse) and runs phase A (the handler with a counting sink); a ballot over the non-cancelled lanes gives
// the record indices (count mode: plus the ready tasks before the tile, from tile_count_kernel run with UD_TILE), one
// warp scan of the record lengths and one warp_reserve_bytes per tile, rounded up to 16 bytes as that kernel does, place
// the bytes; each lane then writes its own record (phase B: a string result calls the handler again with a writing sink).
// Under a retry policy (task-queue rendering) a status goes through retry_settle, which writes task_of for RETRY records.
//
// The control ring (drain_kernel.cuh, D3_CTL_RING): the kernel zeroes the next launch's entry, as the other drain kernels
// do. It is never launched as a programmatic dependent and the host does not launch the next drain as its dependent, so
// at its start the previous launch has completed and nothing reads that entry any more.
#pragma once
#include "drain_kernel.cuh"

namespace b9 {

constexpr uint32_t UD_TILE = 32;       // slots per warp-tile: one per lane (b9gpu.cu launches with tile_tasks = 32)
constexpr int UD_WARPS = 4;            // warps per CTA

template <class H, int R>
__device__ __forceinline__ void user_drain(const DrainArgs& a) {
    if (blockIdx.x == 0 && threadIdx.x == 0) *a.ctl_next = DrainCtl{};
    const int lane = threadIdx.x & 31;
    for (;;) {
        unsigned long long tile = 0;
        if (lane == 0) tile = atomicAdd(&a.out.ctl->ticket, 1ull);
        tile = __shfl_sync(0xffffffffu, tile, 0);
        if (tile >= a.n_tiles) break;
        const uint32_t i = (uint32_t)tile * UD_TILE + (uint32_t)lane;
        const bool in = i < a.n_tasks;
        const uint32_t slot = (uint32_t)((a.first_task + i) & a.slot_mask);
        const uint64_t h = in ? __ldg(a.hdr + slot) : 0ull;
        const bool live = in && !(hdr_flags(h) & 1u);
        b9h::UserRec rec;
        rec.status = ST_UNSUPPORTED; rec.has = 0; rec.vk = b9h::VK_UNSET; rec.out_len = 0; rec.src_off = 0; rec.src_len = 0; rec.value = 0;
        const uint8_t* p = a.payload;
        if (live) {
            p = a.payload + __ldg(a.off + slot);
            uint8_t idb[16];
            const uint32_t flags = hdr_flags(h);
            if (flags & B9_TF_TASK_MSG_BIT) {
                const uint4 id = __ldg(a.ids + slot);
                const uint32_t w[4] = {id.x, id.y, id.z, id.w};
                for (int b = 0; b < 16; ++b) idb[b] = (uint8_t)(w[b >> 2] >> (8 * (b & 3)));
            }
            b9h::user_phase_a<H, R>(p, b9h::user_parse<R>(p, hdr_len(h), flags, idb), rec);
        }

        // ---- record index (ballot), bytes (scan) and ONE cursor add per warp-tile
        const uint32_t live_mask = __ballot_sync(0xffffffffu, live);
        const uint32_t base_cnt = a.count_mode ? tile_ready_before(a, tile, UD_TILE) : (uint32_t)tile * UD_TILE;
        if (lane == 0 && tile == a.n_tiles - 1) a.out.ctl->total_cnt = base_cnt + __popc(live_mask);
        const uint32_t j = base_cnt + __popc(live_mask & ((1u << lane) - 1u));
        const uint32_t my = rec.has ? rec.out_len : 0u;
        const uint32_t incl = warp_incl_scan(my, lane);
        const uint32_t tb = __shfl_sync(0xffffffffu, incl, 31);
        const Reservation r = warp_reserve_bytes(a.out, (tb + 15u) & ~15u, lane);
        const unsigned long long ob = r.base + (incl - my);
        if (!live) continue;
        uint8_t status = rec.status;
        if (R == b9h::TASK_QUEUE && a.retry_mask) status = retry_settle(a, j, i, status, rec.value);
        store_record_id(a.out, j, a.ids + slot);
        store_record(a.out, j, r.fits, ob, my, status, rec.has);
        if (r.fits && rec.has && !b9h::user_phase_b<H, R>(p, rec, a.out.payload + ob))
            store_record(a.out, j, true, 0, 0, (uint8_t)ST_UNSUPPORTED, 0);    // the handler's two passes disagreed
    }
}

}  // namespace b9
