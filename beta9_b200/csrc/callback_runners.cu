// The function and endpoint runners' callbacks on the device (b9_set_callback_runners), compiled as a translation unit of
// its own for the reason callback_sign.cu, function_drain.cu and endpoint_drain.cu are: NVVM decides inlining for a whole
// module, and these kernels call the pickle, float and signing helpers the drain kernels also use.
//
// function_callback_kernel<H> runs in place of pickle_pass_kernel<H> (function_drain.cu) when a B9_DRAIN_PICKLE_FULL
// launch is made under a callback policy with B9_CB_RUNNER_FUNCTION, behind callback_sign_kernel (which wrote every
// record's kind and digest, B9_CB_HOST for the pickle slots). It does the pass's work, with the same shape and the same
// record bytes, and then, for every B9_TF_PICKLE slot (identity's one-str template settled in drain3_kernel included),
// settles the callback: the kind, D (callback_runners.cuh) and the task's own URL, reserved from the control block's
// cursor behind the record, and the signature of {"data": D}. Every other record's request is its result bytes R.
//
// endpoint_callback_kernel runs behind endpoint_drain_kernel under a policy with B9_CB_RUNNER_ENDPOINT: one thread per
// window task measures T(E) of its record, one warp scan and one warp_reserve_bytes place the warp's D bytes, and each
// thread writes and signs its D.
#include <stdint.h>
#include <string.h>
#include <algorithm>
#include <cuda_runtime.h>

#pragma nv_diag_suppress 177     // (the headers' functions these kernels do not use: "declared but never referenced")
namespace {
#define B9_CALLBACK_NO_SIGN_KERNEL 1
#include "drain_kernel.cuh"
#include "callback_sign.cuh"
#include "callback_runners.cuh"
}

namespace {

// the request arrays of b9_drain_fetch_callback_requests, record order
struct CbOut {
    uint8_t* kind; uint4* digest;
    uint64_t* body_off; uint32_t* body_len;
    uint64_t* url_off; uint32_t* url_len;
};

__device__ __forceinline__ void store_digest(const CbOut& o, uint32_t j, const uint32_t* d) {
    uint4 d0 = make_uint4(0, 0, 0, 0), d1 = d0;
    if (d) {                                                       // raw digest bytes in order, as callback_sign_kernel stores them
        d0 = make_uint4(__byte_perm(d[0], 0, 0x0123), __byte_perm(d[1], 0, 0x0123), __byte_perm(d[2], 0, 0x0123), __byte_perm(d[3], 0, 0x0123));
        d1 = make_uint4(__byte_perm(d[4], 0, 0x0123), __byte_perm(d[5], 0, 0x0123), __byte_perm(d[6], 0, 0x0123), __byte_perm(d[7], 0, 0x0123));
    }
    o.digest[2 * (size_t)j] = d0; o.digest[2 * (size_t)j + 1] = d1;
}

// record index of window task t (not cancelled), as callback_sign_kernel finds it
__device__ __forceinline__ uint32_t record_of(const b9::DrainArgs& a, uint32_t t) {
    if (!a.count_mode) return t;
    const uint32_t tile = t / a.tile_tasks;
    uint32_t j = b9::tile_ready_before(a, tile, a.tile_tasks);
    for (uint32_t q = tile * a.tile_tasks; q < t; ++q) j += (b9::hdr_flags(a.hdr[(uint32_t)((a.first_task + q) & a.slot_mask)]) & 1u) ? 0u : 1u;
    return j;
}

template <int H>
__global__ void __launch_bounds__(32) function_callback_kernel(b9::DrainArgs a, b9::CbSign sg, uint32_t keyed, CbOut co) {
    extern __shared__ __align__(16) uint8_t pk_smem[];
    __shared__ uint32_t s_crc[256];
    b9::PkScratch& S = *reinterpret_cast<b9::PkScratch*>(pk_smem);
    const int lane = threadIdx.x;
    if (H == 1) for (int i = lane; i < 256; i += 32) s_crc[i] = b9::crc_table_entry((uint32_t)i);
    __syncwarp();
    if (lane != 0) return;
    for (uint32_t i = blockIdx.x; i < a.n_tasks; i += gridDim.x) {
        const uint32_t slot = (uint32_t)((a.first_task + i) & a.slot_mask);
        const uint64_t h = a.hdr[slot];
        const uint32_t flags = b9::hdr_flags(h);
        if (a.count_mode && (flags & 1u)) continue;                // cancelled: no record
        const uint32_t j = record_of(a, i);
        if (flags != b9::B9_TF_PICKLE_BIT) {                       // callback_sign_kernel's record: the request is R
            co.body_off[j] = a.out.off[j]; co.body_len[j] = a.out.has[j] ? a.out.len[j] : 0u;
            co.url_off[j] = 0; co.url_len[j] = 0;
            continue;
        }
        const uint8_t* p = a.payload + a.off[slot];
        const uint32_t len = b9::hdr_len(h);
        const b9::PkPlan pl = b9::pk_prepare(p, len, H, S, s_crc);
        uint8_t st = a.out.status[j];
        if (st == b9::ST_UNSUPPORTED && pl.status != b9::ST_UNSUPPORTED) {   // the pickle pass's record
            const b9::Reservation r = b9::reserve_bytes(a.out, (pl.out_len + 15u) & ~15u);
            if (r.fits && pl.out_len) b9::pk_write(p, S, pl, a.out.payload + r.base);
            b9::store_record(a.out, j, r.fits, r.base, pl.out_len, pl.status, pl.out_len ? 1 : 0);
            st = pl.status;
        }
        uint8_t kind = b9::CB_HOST;
        uint64_t d_off = 0, u_off = 0; uint32_t d_len = 0, u_len = 0;
        uint32_t dg[8]; bool signed_ = false;
        if (st == b9::ST_OK && pl.status == b9::ST_OK) {
            // pk_write used the decoder's stack as its memo table: decoding again finds the same graph and the root
            const int root = b9::pk_decode(p, len, S);
            const int u = b9::cbr_callback_url(p, S, root);
            b9::CbrW w; w.o = nullptr; w.n = 0;
            const uint8_t k = u == -2 ? b9::CBR_HOST : b9::cbr_kind(b9::cbr_result(w, p, S, pl));
            if (k == b9::CBR_UNSENDABLE) kind = b9::CB_UNSENDABLE;
            else if (k == b9::CBR_POST) {
                uint32_t us = 0;
                if (u >= 0) b9::pk_data(p, S.node[u].x, &us, &u_len);
                d_len = w.n;
                const b9::Reservation r = b9::reserve_bytes(a.out, (d_len + u_len + 15u) & ~15u);
                if (r.fits) {
                    kind = b9::CB_POST;
                    d_off = r.base; u_off = u_len ? r.base + d_len : 0;
                    w.o = a.out.payload + d_off; w.n = 0;
                    b9::cbr_result(w, p, S, pl);
                    for (uint32_t q = 0; q < u_len; ++q) a.out.payload[u_off + q] = p[us + q];
                    if (keyed) { b9::cb_sign_record(sg, a.out.payload + d_off, d_len, dg); signed_ = true; }
                } else { d_len = 0; u_len = 0; }                   // (B9_ENOSPC: the fetch refuses this launch)
            }
        }
        co.kind[j] = kind;
        store_digest(co, j, signed_ ? dg : nullptr);
        co.body_off[j] = d_off; co.body_len[j] = d_len;
        co.url_off[j] = u_off; co.url_len[j] = u_len;
    }
}

constexpr uint32_t EP_CB_THREADS = 128;

__global__ void __launch_bounds__(EP_CB_THREADS) endpoint_callback_kernel(b9::DrainArgs a, b9::CbSign sg, uint32_t keyed, CbOut co) {
    const int lane = threadIdx.x & 31;
    if (__shfl_sync(0xffffffffu, a.out.ctl->overflow, 0)) return;  // B9_ENOSPC: no records to sign (the whole warp leaves)
    const uint32_t t = blockIdx.x * EP_CB_THREADS + threadIdx.x;
    const bool in = t < a.n_tasks;
    const uint32_t flags = in ? b9::hdr_flags(a.hdr[(uint32_t)((a.first_task + t) & a.slot_mask)]) : 0u;
    const bool live = in && !(a.count_mode && (flags & 1u));
    const uint32_t j = live ? record_of(a, t) : 0u;
    const uint8_t st = live ? a.out.status[j] : (uint8_t)b9::ST_UNSUPPORTED;
    const bool ok = live && st == b9::ST_OK && a.out.has[j];
    const uint8_t* e = ok ? a.out.payload + a.out.off[j] : nullptr;
    const uint64_t m = ok ? b9::cbr_endpoint_body(e, a.out.len[j], nullptr) : 0ull;
    const bool post = ok && m <= b9::CBR_MAX_BODY;                 // (the warp's D bytes stay within 32 bits)
    const uint32_t my = post ? (uint32_t)m : 0u;
    const uint32_t incl = b9::warp_incl_scan(my, lane);
    const uint32_t tb = __shfl_sync(0xffffffffu, incl, 31);
    const b9::Reservation r = b9::warp_reserve_bytes(a.out, (tb + 15u) & ~15u, lane);
    if (!live) return;
    const unsigned long long ob = r.base + (incl - my);
    uint8_t kind = st == b9::ST_OK ? (post ? b9::CB_POST : b9::CB_HOST) : st == b9::ST_REJECTED ? b9::CB_NONE : b9::CB_HOST;
    uint32_t dg[8]; bool signed_ = false;
    if (kind == b9::CB_POST && !r.fits) kind = b9::CB_HOST;        // (B9_ENOSPC: the fetch refuses this launch)
    if (kind == b9::CB_POST) {
        b9::cbr_endpoint_body(e, a.out.len[j], a.out.payload + ob);
        if (keyed) { b9::cb_sign_record(sg, a.out.payload + ob, my, dg); signed_ = true; }
    }
    co.kind[j] = kind;
    store_digest(co, j, signed_ ? dg : nullptr);
    co.body_off[j] = kind == b9::CB_POST ? ob : 0; co.body_len[j] = kind == b9::CB_POST ? my : 0u;
    co.url_off[j] = 0; co.url_len[j] = 0;
}

template <int H>
cudaError_t launch_function(const b9::DrainArgs& a, const b9::CbSign& sg, uint32_t keyed, const CbOut& co, int sm_count, cudaStream_t s) {
    int per_sm = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, function_callback_kernel<H>, 32, sizeof(b9::PkScratch));
    if (e != cudaSuccess) return e;
    const uint32_t grid = (uint32_t)std::min<uint64_t>(a.n_tasks, (uint64_t)std::max(per_sm, 1) * (uint64_t)sm_count);
    function_callback_kernel<H><<<grid, 32, sizeof(b9::PkScratch), s>>>(a, sg, keyed, co);
    return cudaGetLastError();
}

}  // namespace

// b9gpu.cu's b9::DrainArgs comes from the same header as this file's copy; args_size guards that. `args` is the drain
// launch's argument block (tile_tasks as the drain kernel used it). mid: the key's midstates; keyed = 0: no digests.
// out: kind, digest, body_off, body_len, url_off, url_len (device arrays of max_drain_tasks records).
cudaError_t launch_callback_runner(int endpoint, const void* args, size_t args_size, int handler, const uint32_t mid[16], int keyed,
                                   int64_t ts, void* const out[6], int sm_count, cudaStream_t s) {
    if (args_size != sizeof(b9::DrainArgs)) return cudaErrorInvalidValue;
    const b9::DrainArgs& a = *static_cast<const b9::DrainArgs*>(args);
    if (a.n_tasks == 0) return cudaSuccess;
    b9::CbSign sg;
    b9::cb_sign_init(sg, mid, ts);
    CbOut co;
    co.kind = (uint8_t*)out[0]; co.digest = (uint4*)out[1];
    co.body_off = (uint64_t*)out[2]; co.body_len = (uint32_t*)out[3];
    co.url_off = (uint64_t*)out[4]; co.url_len = (uint32_t*)out[5];
    const uint32_t k = keyed ? 1u : 0u;
    if (endpoint) {
        const uint32_t grid = (uint32_t)((a.n_tasks + EP_CB_THREADS - 1) / EP_CB_THREADS);
        endpoint_callback_kernel<<<grid, EP_CB_THREADS, 0, s>>>(a, sg, k, co);
        return cudaGetLastError();
    }
    switch (handler) {
    case 0: return launch_function<0>(a, sg, k, co, sm_count, s);
    case 1: return launch_function<1>(a, sg, k, co, sm_count, s);
    case 2: return launch_function<2>(a, sg, k, co, sm_count, s);
    default: return launch_function<3>(a, sg, k, co, sm_count, s);
    }
}
