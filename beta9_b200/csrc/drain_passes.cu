// The passes that run on the drain stream after the drain kernel, compiled as a translation unit of their own:
//   - function_pass_kernel<H, false> (B9_DRAIN_PICKLE_FULL): the function path for every handler and plain Python values,
//     right after drain3_kernel;
//   - callback_sign_kernel (b9_set_callback_policy): the callback kind and signature of every record of a task-queue drain,
//     behind the records' last writer;
//   - function_pass_kernel<H, true> (b9_set_callback_runners, B9_CB_RUNNER_FUNCTION): the same function pass, behind
//     callback_sign_kernel, which also settles the pickle slots' callbacks;
//   - endpoint_callback_kernel (B9_CB_RUNNER_ENDPOINT): the endpoint runner's callbacks, behind endpoint_drain_kernel.
//
// Why not in b9gpu.cu: NVVM decides inlining for a whole module, so a new kernel that calls the JSON, pickle and sum
// helpers would change how the drain kernels compile (wire_full.cu measured that), and the SHA-256 round constants are a
// __constant__ array of their own. The device headers are included inside an anonymous namespace, as wire_full.cu does:
// their out-of-line __device__ functions get host-side definitions in every translation unit that includes them, which
// would clash with b9gpu.cu's at link time. The host half of the signing (the key's midstates, the drain's tail and the
// digest of {"data": {}}) is callback_sign.cuh's code, called from here.
//
// Every launcher takes the drain launch's DrainArgs as `args`, with tile_tasks as the drain kernel used it: the passes find
// a window task's record with window_record. b9gpu.cu's b9::DrainArgs comes from the same header as this file's copy, so
// their layouts are the same; args_size guards that.
#include <stdint.h>
#include <algorithm>
#include <cuda_runtime.h>

#pragma nv_diag_suppress 177     // (the headers' functions these kernels do not use: "declared but never referenced")
namespace {
#include "drain_kernel.cuh"
#include "callback_sign.cuh"
#include "callback_runners.cuh"
}
static_assert(sizeof(b9::PkScratch) == 28744, "the scratch size and the occupancy below are stated for 28,744 bytes");

// What a runner's callback pass takes besides the drain's DrainArgs; b9gpu.cu declares the same struct. mid: the key's
// midstates, keyed = 0: no digests, ts: the drain's timestamp; out: the request arrays of b9_drain_fetch_callback_requests
// (kind, digest, body_off, body_len, url_off, url_len; device arrays of max_drain_tasks records).
struct CallbackPassArgs { const uint32_t* mid; int keyed; int64_t ts; void* out[6]; };

namespace {

// the request arrays, record order
struct CbOut {
    uint8_t* kind; uint4* digest;
    uint64_t* body_off; uint32_t* body_len;
    uint64_t* url_off; uint32_t* url_len;
};

// record j's digest: the raw HMAC bytes in order (the big-endian words d byte-swapped into the little-endian stores), or
// zeros for d == nullptr
__device__ __forceinline__ void store_digest(uint4* digest, uint32_t j, const uint32_t* d) {
    uint4 d0 = make_uint4(0, 0, 0, 0), d1 = d0;
    if (d) {
        d0 = make_uint4(__byte_perm(d[0], 0, 0x0123), __byte_perm(d[1], 0, 0x0123), __byte_perm(d[2], 0, 0x0123), __byte_perm(d[3], 0, 0x0123));
        d1 = make_uint4(__byte_perm(d[4], 0, 0x0123), __byte_perm(d[5], 0, 0x0123), __byte_perm(d[6], 0, 0x0123), __byte_perm(d[7], 0, 0x0123));
    }
    digest[2 * (size_t)j] = d0; digest[2 * (size_t)j + 1] = d1;
}

// the digest of {"data": {}}: the same for every record of a drain that posts it, computed once on the host
struct EmptyDigest { uint32_t w[8]; };

// The sign pass. Thread per window task. kind[j] is the record's b9_callback_kind; its digest the raw HMAC for a
// B9_CB_POST under a key, otherwise zero.
__global__ void __launch_bounds__(128) callback_sign_kernel(b9::DrainArgs a, b9::CbSign sg, uint32_t keyed, EmptyDigest empty,
                                                            uint8_t* __restrict__ kind, uint4* __restrict__ digest) {
    if (a.out.ctl->overflow) return;                               // B9_ENOSPC: no records to sign
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < a.n_tasks; t += gridDim.x * blockDim.x) {
        const uint32_t slot = (uint32_t)((a.first_task + t) & a.slot_mask);
        const uint64_t h = a.hdr[slot];
        const uint32_t flags = b9::hdr_flags(h);
        if (a.count_mode && (flags & 1u)) continue;                // cancelled: no record
        const uint32_t j = b9::window_record(a, t);
        const uint8_t st = a.out.status[j];
        uint8_t k;
        bool sign_r = false;
        if (flags & b9::B9_TF_PICKLE_BIT) k = b9::CB_HOST;
        else if (st == b9::ST_UNSUPPORTED) k = b9::CB_HOST;
        else if (st == b9::ST_OK) {
            if (!a.out.has[j]) k = b9::CB_POST;
            else if (b9::cb_nonfinite(a.out.payload + a.out.off[j], a.out.len[j])) k = b9::CB_UNSENDABLE;
            else { k = b9::CB_POST; sign_r = true; }
        } else if (st == b9::ST_ERROR) {
            const int mode = (flags & b9::B9_TF_TASK_MSG_BIT) ? 2 : (flags & b9::B9_TF_HTTP_BODY_BIT) ? 1 : 0;
            k = b9::cb_kwargs_have_callback_url(a.payload + a.off[slot], b9::hdr_len(h), mode) ? b9::CB_HOST : b9::CB_POST;
        } else k = b9::CB_NONE;                                    // REJECTED, RETRY, RETRY_LIMIT
        kind[j] = k;
        if (keyed && k == b9::CB_POST) {
            uint32_t dg[8];
            if (sign_r) b9::cb_sign_record(sg, a.out.payload + a.out.off[j], a.out.len[j], dg);
            else for (int i = 0; i < 8; ++i) dg[i] = empty.w[i];
            store_digest(digest, j, dg);
        } else store_digest(digest, j, nullptr);
    }
}

// The function pass: one warp per task, its lane 0 doing the sequential work against a PkScratch in the block's shared
// memory (28,744 bytes, plus the 1 KiB the SM reserves per block and crc32's 1 KiB table: seven blocks, i.e. seven tasks in
// flight, per SM). It is latency-bound: one thread of each resident warp works, about 900 on a 132-SM H100; scratch in
// global memory or a warp-cooperative decoder would keep more tasks in flight. Output bytes come from the same control
// block's cursor, one reserve_bytes per record (drain_kernel.cuh).
//
// CALLBACKS = false: the slots whose flags are exactly B9_TF_PICKLE (not cancelled, no HTTP_BODY, no TASK_MSG); it
// rewrites the records drain3_kernel left UNSUPPORTED, and identity's one-str template stays the fast path.
// CALLBACKS = true: every record, behind callback_sign_kernel (which wrote every record's kind and digest, B9_CB_HOST for
// the pickle slots). It writes the same records as CALLBACKS = false, and then, for every B9_TF_PICKLE slot (identity's
// one-str template settled in drain3_kernel included), settles the callback: the kind, D (callback_runners.cuh) and the
// task's own URL, reserved from the cursor behind the record, and the signature of {"data": D}. Every other record's
// request is its result bytes R.
template <int H, bool CALLBACKS>
__global__ void __launch_bounds__(32) function_pass_kernel(b9::DrainArgs a, b9::CbSign sg, uint32_t keyed, CbOut co) {
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
        if constexpr (CALLBACKS) {
            if (a.count_mode && (flags & 1u)) continue;            // cancelled: no record
        } else if (flags != b9::B9_TF_PICKLE_BIT) continue;
        const uint32_t j = b9::window_record(a, i);
        if (CALLBACKS && flags != b9::B9_TF_PICKLE_BIT) {          // callback_sign_kernel's record: the request is R
            co.body_off[j] = a.out.off[j]; co.body_len[j] = a.out.has[j] ? a.out.len[j] : 0u;
            co.url_off[j] = 0; co.url_len[j] = 0;
            continue;
        }
        uint8_t st = a.out.status[j];
        if (!CALLBACKS && st != b9::ST_UNSUPPORTED) continue;      // drain3_kernel settled it: nothing to decode
        const uint8_t* p = a.payload + a.off[slot];
        const uint32_t len = b9::hdr_len(h);
        const b9::PkPlan pl = b9::pk_prepare(p, len, H, S, s_crc);
        if (st == b9::ST_UNSUPPORTED && pl.status != b9::ST_UNSUPPORTED) {
            const b9::Reservation r = b9::reserve_bytes(a.out, (pl.out_len + 15u) & ~15u);
            if (r.fits && pl.out_len) b9::pk_write(p, S, pl, a.out.payload + r.base);
            b9::store_record(a.out, j, r.fits, r.base, pl.out_len, pl.status, pl.out_len ? 1 : 0);
            st = pl.status;
        }
        if constexpr (CALLBACKS) {
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
                    } else { d_len = 0; u_len = 0; }               // (B9_ENOSPC: the fetch refuses this launch)
                }
            }
            co.kind[j] = kind;
            store_digest(co.digest, j, signed_ ? dg : nullptr);
            co.body_off[j] = d_off; co.body_len[j] = d_len;
            co.url_off[j] = u_off; co.url_len[j] = u_len;
        }
    }
}

// The endpoint runner's callbacks: one thread per window task measures T(E) of its record, one warp scan and one
// warp_reserve_bytes place the warp's D bytes, and each thread writes and signs its D.
constexpr uint32_t EP_CB_THREADS = 128;

__global__ void __launch_bounds__(EP_CB_THREADS) endpoint_callback_kernel(b9::DrainArgs a, b9::CbSign sg, uint32_t keyed, CbOut co) {
    const int lane = threadIdx.x & 31;
    if (__shfl_sync(0xffffffffu, a.out.ctl->overflow, 0)) return;  // B9_ENOSPC: no records to sign (the whole warp leaves)
    const uint32_t t = blockIdx.x * EP_CB_THREADS + threadIdx.x;
    const bool in = t < a.n_tasks;
    const uint32_t flags = in ? b9::hdr_flags(a.hdr[(uint32_t)((a.first_task + t) & a.slot_mask)]) : 0u;
    const bool live = in && !(a.count_mode && (flags & 1u));
    const uint32_t j = live ? b9::window_record(a, t) : 0u;
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
    store_digest(co.digest, j, signed_ ? dg : nullptr);
    co.body_off[j] = kind == b9::CB_POST ? ob : 0; co.body_len[j] = kind == b9::CB_POST ? my : 0u;
    co.url_off[j] = 0; co.url_len[j] = 0;
}

// blocks of `threads` threads and `smem` dynamic shared bytes that fit on the GPU at once, at most `want`
template <class K>
cudaError_t resident_grid(K kernel, int threads, size_t smem, uint64_t want, int sm_count, uint32_t* grid) {
    int per_sm = 0;
    const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem);
    *grid = (uint32_t)std::min<uint64_t>(want, (uint64_t)std::max(per_sm, 1) * (uint64_t)sm_count);
    return e;
}

template <int H, bool CALLBACKS>
cudaError_t launch_function(const b9::DrainArgs& a, const b9::CbSign& sg, uint32_t keyed, const CbOut& co, int sm_count, cudaStream_t s) {
    uint32_t grid = 0;
    const cudaError_t e = resident_grid(function_pass_kernel<H, CALLBACKS>, 32, sizeof(b9::PkScratch), a.n_tasks, sm_count, &grid);
    if (e != cudaSuccess) return e;
    function_pass_kernel<H, CALLBACKS><<<grid, 32, sizeof(b9::PkScratch), s>>>(a, sg, keyed, co);
    return cudaGetLastError();
}

template <bool CALLBACKS>
cudaError_t launch_function(int handler, const b9::DrainArgs& a, const b9::CbSign& sg, uint32_t keyed, const CbOut& co, int sm_count, cudaStream_t s) {
    switch (handler) {
    case 0: return launch_function<0, CALLBACKS>(a, sg, keyed, co, sm_count, s);
    case 1: return launch_function<1, CALLBACKS>(a, sg, keyed, co, sm_count, s);
    case 2: return launch_function<2, CALLBACKS>(a, sg, keyed, co, sm_count, s);
    default: return launch_function<3, CALLBACKS>(a, sg, keyed, co, sm_count, s);
    }
}

void callback_setup(const CallbackPassArgs& cb, b9::CbSign& sg, CbOut& co) {
    b9::cb_sign_init(sg, cb.mid, cb.ts);
    co.kind = (uint8_t*)cb.out[0]; co.digest = (uint4*)cb.out[1];
    co.body_off = (uint64_t*)cb.out[2]; co.body_len = (uint32_t*)cb.out[3];
    co.url_off = (uint64_t*)cb.out[4]; co.url_len = (uint32_t*)cb.out[5];
}

}  // namespace

// the key's ipad / opad midstates, computed once per b9_set_callback_policy
void callback_midstates(const uint8_t* key, uint32_t key_len, uint32_t mid[16]) { b9::cb_midstates(key, key_len, mid); }

// keyed = 0: kinds only, every digest zero
cudaError_t launch_callback_sign(const void* args, size_t args_size, const uint32_t mid[16], int keyed, int64_t ts,
                                 uint8_t* kind, uint8_t* digest, int sm_count, cudaStream_t s) {
    if (args_size != sizeof(b9::DrainArgs)) return cudaErrorInvalidValue;
    const b9::DrainArgs& a = *static_cast<const b9::DrainArgs*>(args);
    if (a.n_tasks == 0) return cudaSuccess;
    b9::CbSign sg;
    b9::cb_sign_init(sg, mid, ts);
    EmptyDigest empty;
    b9::cb_sign_record(sg, reinterpret_cast<const uint8_t*>("{}"), 2, empty.w);    // {"data": {}}
    uint32_t grid = 0;
    const cudaError_t e = resident_grid(callback_sign_kernel, 128, 0, (a.n_tasks + 127u) / 128u, sm_count, &grid);
    if (e != cudaSuccess) return e;
    callback_sign_kernel<<<grid, 128, 0, s>>>(a, sg, keyed ? 1u : 0u, empty, kind, reinterpret_cast<uint4*>(digest));
    return cudaGetLastError();
}

// cb == nullptr: the pickle pass; otherwise the function runner's pass, behind launch_callback_sign
cudaError_t launch_function_pass(const void* args, size_t args_size, int handler, const CallbackPassArgs* cb, int sm_count, cudaStream_t s) {
    if (args_size != sizeof(b9::DrainArgs)) return cudaErrorInvalidValue;
    const b9::DrainArgs& a = *static_cast<const b9::DrainArgs*>(args);
    if (a.n_tasks == 0) return cudaSuccess;
    b9::CbSign sg{};
    CbOut co{};
    if (!cb) return launch_function<false>(handler, a, sg, 0, co, sm_count, s);
    callback_setup(*cb, sg, co);
    return launch_function<true>(handler, a, sg, cb->keyed ? 1u : 0u, co, sm_count, s);
}

// the endpoint runner's pass, behind endpoint_drain_kernel
cudaError_t launch_endpoint_callbacks(const void* args, size_t args_size, const CallbackPassArgs& cb, cudaStream_t s) {
    if (args_size != sizeof(b9::DrainArgs)) return cudaErrorInvalidValue;
    const b9::DrainArgs& a = *static_cast<const b9::DrainArgs*>(args);
    if (a.n_tasks == 0) return cudaSuccess;
    b9::CbSign sg;
    CbOut co;
    callback_setup(cb, sg, co);
    const uint32_t grid = (uint32_t)((a.n_tasks + EP_CB_THREADS - 1) / EP_CB_THREADS);
    endpoint_callback_kernel<<<grid, EP_CB_THREADS, 0, s>>>(a, sg, cb.keyed ? 1u : 0u, co);
    return cudaGetLastError();
}
