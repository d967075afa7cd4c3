// libb9gpu.so — host side of the C ABI declared in include/b9gpu.h.
//
// One b9_ctx = one GPU: the pending-task ring lives in HBM (payload bytes + SoA slot arrays),
// pushes DMA the caller's batch straight into it, drains run one persistent kernel over a FIFO
// window of the ring and DMA the dense result records back. The semantic model of the ring is
// the reference's FIFO Redis list (pkg/abstractions/taskqueue/client.go:29-96: RPUSH at the tail,
// LPOP at the head) with `RingBuffer`-style fixed capacity (pkg/abstractions/common/ring_buffer.go).
#include <cuda_runtime.h>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <chrono>
#include <deque>
#include <atomic>
#include <condition_variable>
#include <functional>
#include <memory>
#include <mutex>
#include <thread>
#include <new>
#include <string>
#include <vector>

#include "../../include/b9gpu.h"
#include "cancel.cuh"
#include "drain_kernel.cuh"
#include "drain2.cuh"
#include "rebalance_plan.h"
#include "ring_place.h"
#include "sink.h"
#include "submit_buffer.h"
#include "wire_encode.cuh"

#include <dlfcn.h>

// wire_encode_kernel<true> for b9_wire_encode_full, launched from its own translation unit (wire_full.cu says why);
// args: a WireArgs, env: the device copy of the WireEnv
cudaError_t launch_wire_encode_full(const void* args, size_t args_size, const void* env, uint32_t grid, cudaStream_t s);
// the passes that run after the drain kernel, from drain_passes.cu; args: the drain's DrainArgs (tile_tasks as the drain
// kernel used it). The callback sign pass (b9_set_callback_policy): mid: the key's midstates (callback_midstates), keyed = 0:
// kinds only.
void callback_midstates(const uint8_t* key, uint32_t key_len, uint32_t mid[16]);
cudaError_t launch_callback_sign(const void* args, size_t args_size, const uint32_t mid[16], int keyed, int64_t ts,
                                 uint8_t* kind, uint8_t* digest, int sm_count, cudaStream_t s);
// The runners' callback passes (b9_set_callback_runners); drain_passes.cu defines the same struct. out: kind, digest,
// body_off, body_len, url_off, url_len.
struct CallbackPassArgs { const uint32_t* mid; int keyed; int64_t ts; void* out[6]; };
// the function pass for B9_DRAIN_PICKLE_FULL: cb == nullptr, the pickle pass; otherwise the function runner's callback
// pass, which does the pickle pass's work behind the sign pass
cudaError_t launch_function_pass(const void* args, size_t args_size, int handler, const CallbackPassArgs* cb, int sm_count, cudaStream_t s);
// the endpoint runner's callback pass, behind endpoint_drain_kernel
cudaError_t launch_endpoint_callbacks(const void* args, size_t args_size, const CallbackPassArgs& cb, cudaStream_t s);
// endpoint_drain_kernel for b9_endpoint_drain_launch, from endpoint_drain.cu; args: the drain's DrainArgs, with tile_tasks
// = ENDPOINT_TILE_TASKS and n_tiles set for it
cudaError_t launch_endpoint_drain(const void* args, size_t args_size, int handler, int sm_count, cudaStream_t s);
constexpr uint32_t ENDPOINT_TILE_TASKS = 32;   // endpoint_drain.cu's EP_TILE (the launcher refuses any other)
constexpr int USER_DRAIN_WARPS = 4;            // user_drain.cuh's UD_WARPS (its tiles are ENDPOINT_TILE_TASKS slots too)

using namespace b9;

namespace {

thread_local std::string g_last_error;   // per calling thread, as the header promises

int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
    g_last_error = buf;
    return code;
}

#define CU(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) \
    return fail(B9_EIO, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); } while (0)

uint64_t pow2_ceil(uint64_t v) { uint64_t p = 1; while (p < v) p <<= 1; return p; }
void nccl_comm_destroy(void* comm);   // defined with the NCCL loader below

// Owning holders of the context's CUDA resources: what they hold is released when they are destroyed (b9_ctx_destroy sets
// the device first) or reset. They convert to the raw handle, so the code that uses them reads as with a plain one.
template <class H, cudaError_t (*Release)(H)> struct Owned {
    H v{};
    Owned() = default;
    Owned(const Owned&) = delete;
    Owned& operator=(const Owned&) = delete;
    ~Owned() { reset(); }
    void reset() { if (v) Release(v); v = H{}; }
    operator H() const { return v; }
    H operator->() const { return v; }
};
template <class T> cudaError_t free_device(T* p) { return cudaFree(p); }
template <class T> cudaError_t free_pinned(T* p) { return cudaFreeHost(p); }
template <class T> using DevPtr = Owned<T*, free_device<T>>;       // cudaMalloc
template <class T> using PinnedPtr = Owned<T*, free_pinned<T>>;    // cudaHostAlloc
using Event = Owned<cudaEvent_t, cudaEventDestroy>;
using Stream = Owned<cudaStream_t, cudaStreamDestroy>;

// Device (or page-locked) memory allocated on first use and grow-only: grow(need) keeps the buffer while it holds `need`
// bytes, else replaces it with need + headroom bytes, or with nothing when that fails (the sticky error is cleared).
// ensure() is grow() with a failure reported through fail(): B9_ENOMEM when the memory is short, else B9_EIO, with `what`
// as the message.
template <class T, bool Pinned = false> struct GrowBuf {
    Owned<T*, Pinned ? free_pinned<T> : free_device<T>> p; uint64_t cap = 0;
    operator T*() const { return p; }
    cudaError_t grow(uint64_t need, uint64_t headroom = 0) {
        if (need <= cap) return cudaSuccess;
        p.reset(); cap = 0;
        const cudaError_t e = Pinned ? cudaHostAlloc(&p.v, need + headroom, cudaHostAllocDefault) : cudaMalloc(&p.v, need + headroom);
        if (e != cudaSuccess) { p.v = nullptr; cudaGetLastError(); return e; }
        cap = need + headroom;
        return cudaSuccess;
    }
    int ensure(uint64_t need, const char* what, uint64_t headroom = 0) {
        const cudaError_t e = grow(need, headroom);
        if (e == cudaSuccess) return B9_OK;
        return fail(e == cudaErrorMemoryAllocation ? B9_ENOMEM : B9_EIO, "%s: %llu bytes: %s", what, (unsigned long long)(need + headroom),
                    cudaGetErrorString(e));
    }
};

struct Segment {             // one push = one contiguous byte range of the payload ring
    uint64_t first_task;     // logical index of its first task
    uint32_t n;
    uint64_t phys_start, bytes;
    cudaEvent_t ready;           // recorded on the ingest stream once the batch is fully on the device
    uint32_t max_len;            // longest task of the batch (0 = not known: tasks that arrived in a rebalance)
    uint32_t n_pickle;           // tasks of the batch carrying B9_TF_PICKLE (all of them when not known: a rebalance)
    bool drain_waited = false;   // a drain launch has made the drain stream wait for `ready` (stream order covers later launches)
};

constexpr uint64_t RING_SLACK = 256;   // readable bytes past the ring end (vector loads may over-read)
constexpr uint64_t SEG_ALIGN  = B9_SEG_ALIGN;

// A few persistent threads for the host-side pack (b9_batch_push_v): the calling thread is worker 0.
struct PackPool {
    std::vector<std::thread> th;
    std::mutex m; std::condition_variable cv, cv_done;
    std::function<void(int)> job;
    int nthreads = 1, generation = 0, pending = 0; bool stop = false;
    explicit PackPool(int n) : nthreads(n < 1 ? 1 : n) {
        for (int i = 1; i < nthreads; ++i) th.emplace_back([this, i] {
            int seen = 0;
            for (;;) {
                std::function<void(int)> f;
                { std::unique_lock<std::mutex> lk(m); cv.wait(lk, [&] { return stop || generation != seen; }); if (stop) return; seen = generation; f = job; }
                f(i);
                { std::lock_guard<std::mutex> lk(m); if (--pending == 0) cv_done.notify_one(); }
            }
        });
    }
    void run(const std::function<void(int)>& f) {
        { std::lock_guard<std::mutex> lk(m); job = f; pending = nthreads - 1; ++generation; }
        cv.notify_all();
        f(0);
        std::unique_lock<std::mutex> lk(m); cv_done.wait(lk, [&] { return pending == 0; });
    }
    ~PackPool() { { std::lock_guard<std::mutex> lk(m); stop = true; } cv.notify_all(); for (auto& t : th) t.join(); }
};

// page-locked staging of one packed batch (b9_batch_push_v): two of them alternate, so that batch k+1 is gathered
// while batch k is still on the wire
struct PackArena {
    GrowBuf<uint8_t, true> payload, ids; GrowBuf<uint64_t, true> offsets;
    Event free_ev; bool in_flight = false;
};

// results waiting on the device for b9_drain_fetch; dropping them is `res = WaitingResults{}`
struct WaitingResults {
    bool have = false, peek = false;
    bool retry = false;                        // they come from a drain launched under a retry policy
    bool cb = false, cb_keyed = false; int64_t cb_ts = 0;   // ... with a callback pass: its keying and Unix seconds
    bool cb_requests = false;                  // ... and a runner's callback pass wrote the request arrays (else they are R)
    uint32_t n = 0, popped = 0; uint64_t bytes = 0, in_bytes = 0; float kernel_ms = 0.f;
    bool ids_in_ring = false; uint64_t head = 0;   // record j's id is the ring id of task head + j (DrainOut::ids_compacted == 0)
    bool async = false;                        // the last launch returned before its kernels finished: finalize on fetch / sync
    uint32_t async_n = 0; uint64_t async_in_bytes = 0;
};

// A handler image loaded with b9_handler_load: its two B9_HANDLER entry points (b9gpu_handler.cuh) and their residency
struct UserHandler {
    cudaLibrary_t lib = nullptr;
    cudaKernel_t tq = nullptr, ep = nullptr;   // the task-queue and the endpoint drain
    int per_sm_tq = 1, per_sm_ep = 1;          // resident CTAs per SM
};

}  // namespace

struct b9_ctx {
    int device = 0;
    int sm_count = 0;
    uint32_t stage_bytes_override = 0; // B9_STAGE_BYTES: force the v2 stage-buffer size
    Stream stream;                             // drain kernels + D2H
    Stream stream_in;                          // H2D + ingest kernel (so that pushes overlap drains: PCIe is full duplex)
    std::vector<cudaEvent_t> event_pool;       // idle segment events (take_event / put_event)
    Event ev_a, ev_b, ev_c, ev_d;              // drain stream (under out_mu)
    Event ev_pa, ev_pb;                        // ingest stream (under in_mu)
    // Three locks, always taken in this order: in_mu (push submission: H2D + ingest kernel are enqueued in FIFO order),
    // out_mu (drain-side submission and the waiting-results state: launch, fetch, expire, cancel, wire records, rebalance), mu
    // (ring bookkeeping + stats; held for pointer arithmetic only, never across a CUDA synchronisation). Producers
    // therefore never wait for a drain's kernels or its D2H copy, and the drainer never waits for a push's DMA
    // (Dispatcher.Register's goroutine-safety contract, pkg/task/dispatch.go:71-73).
    std::mutex in_mu, out_mu, mu;
    std::mutex pack_mu; std::unique_ptr<PackPool> pack_pool; PackArena pack[2]; int pack_next = 0;
    // micro-batching of single-task submissions (b9_submit / b9_flush): two page-locked arenas, lock-free appends
    std::mutex sb_mu; std::unique_ptr<SubmitBuffer> sb; Event sb_free[2]; bool sb_in_flight[2] = {false, false};
    int sb_unpushed = -1; uint32_t sb_unpushed_n = 0;   // an arena whose push was refused (ring full): pushed again by the next flush
    std::atomic<uint64_t> running{0};           // tasks a drain has claimed (launched, not peeking) and not yet committed by a fetch

    // ---- pending ring (device)
    uint64_t ring_bytes = 0; uint32_t ring_tasks = 0, slot_mask = 0, max_task_bytes = 0;
    DevPtr<uint8_t>  d_payload;
    DevPtr<uint64_t> d_off; DevPtr<uint64_t> d_hdr; DevPtr<uint4> d_ids;
    DevPtr<int64_t>  d_ts;  DevPtr<int64_t> d_exp;
    // push staging (device): raw offsets + optional metadata of the batch being ingested
    DevPtr<uint64_t> d_in_off; DevPtr<int64_t> d_in_ts; DevPtr<int64_t> d_in_exp;
    DevPtr<uint8_t>  d_in_retries; DevPtr<uint8_t> d_in_flags;
    // the retry policy (b9_set_retry_policy; set under out_mu) and the re-push's device buffers (allocated with the first policy)
    uint32_t retry_mask = 0, max_retries = 0;
    GrowBuf<uint32_t> d_task_of;               // [max_drain_tasks] DrainArgs::task_of
    GrowBuf<uint32_t> d_retry_rec;             // [max_drain_tasks] the RETRY records of a fetch, in record order
    GrowBuf<uint4> d_retry_ids;                // [max_drain_tasks] their ids
    GrowBuf<uint8_t> d_retry_bytes;            // their payload bytes
    GrowBuf<void> d_retry_scan;                // cub scan scratch
    // the callback policy (b9_set_callback_policy; set under out_mu) and the sign pass's outputs (allocated with the first policy)
    bool cb_enabled = false, cb_keyed = false; uint32_t cb_mid[16] = {};
    GrowBuf<uint8_t> d_cb_kind;                // [max_drain_tasks] b9_callback_kind per record
    GrowBuf<uint8_t> d_cb_digest;              // [max_drain_tasks * 32] raw HMAC-SHA256 per record
    // the runners whose callbacks are settled on the device too (b9_set_callback_runners; set under out_mu) and their
    // passes' request arrays (allocated with the first runner): D and the task's own URL per record, in d_out_payload
    uint32_t cb_runners = 0;
    GrowBuf<uint64_t> d_cb_body_off, d_cb_url_off;   // [max_drain_tasks]
    GrowBuf<uint32_t> d_cb_body_len, d_cb_url_len;   // [max_drain_tasks]
    // ring bookkeeping (host)
    uint64_t head_task = 0, tail_task = 0;     // logical, monotonically increasing
    uint64_t write_pos = 0;                    // physical byte position of the next segment
    uint64_t pending_bytes = 0;
    std::deque<Segment> segs;

    // ---- drain staging (device)
    uint32_t max_drain_tasks = 0; uint64_t max_result_bytes = 0;
    DevPtr<uint8_t> d_out_payload; DevPtr<uint64_t> d_out_off; DevPtr<uint4> d_out_ids;
    DevPtr<uint8_t> d_out_status; DevPtr<uint8_t> d_out_has; DevPtr<uint32_t> d_out_len;
    DevPtr<SlowItem> d_slow;                    // identity: work list of deferred tasks (kernel tail)
    uint32_t drain_epoch = 0;                   // tag of the current launch's work-list items
    DevPtr<WireEnv> d_wire_env;
    DevPtr<uint32_t> d_crc_shift;               // crc32: zero-byte shift tables
    uint64_t cancelled_pending = 0;            // pending tasks carrying B9_TF_CANCELLED (pushed so, expired, or b9_cancel)
    GrowBuf<CancelKey> d_cancel_keys; GrowBuf<uint32_t> d_cancel_out;   // b9_cancel: sorted ids + outcome words
    DevPtr<DrainCtl> d_ctl; DevPtr<uint64_t> d_tile_state;   // d_ctl: D3_CTL_RING control blocks (drain_kernel.cuh)
    bool ctl_dirty = false;                    // the next drain's control block may be non-zero: zero the ring before it
    uint32_t ctl_last = 0;                     // control block of the last drain launch (read by finish_launch)
    bool last_op_drain = false;                // the drain stream's last operation is a drain3_kernel: the next may overlap it
    // launches since the last completion are timed as one span: ev_burst before the first one's kernel, ev_b right after
    // the last one's (recorded before anything else is enqueued on the drain stream, see end_drain_span)
    bool burst_open = false; Event ev_burst;
    PinnedPtr<DrainCtl> h_ctl;
    GrowBuf<uint8_t> d_xchg_send, d_xchg_recv; // b9_rebalance staging
    DevPtr<uint64_t> d_prefix; DevPtr<unsigned long long> d_scan_sums;   // b9_rebalance: byte prefix of the pending tasks, on the device
    DevPtr<uint64_t> d_rtab; PinnedPtr<uint64_t> h_rtab; size_t rtab_words = 0;   // b9_rebalance: all-gather tables + cut points (device / pinned), allocated once
    DevPtr<unsigned long long> d_count; PinnedPtr<unsigned long long> h_count;
    WaitingResults res;
    uint64_t res_gen = 0;                      // bumped whenever the waiting results change (launch, fetch commit)
    bool expired_since_launch = false, recount_cancelled = false;   // (b9_expire between a launch and its fetch: recount, see b9_drain_fetch)

    // ---- multi-GPU (NCCL, loaded with dlopen: the library has no link-time dependency on it)
    void* nccl_comm = nullptr; int comm_rank = 0, comm_world = 1;

    b9_stats stats{};

    // handler images of b9_handler_load (under out_mu): id B9_H_USER_BASE + k is users[k]
    std::vector<UserHandler> users;

    // what the members do not release themselves: the segment events, the submission arenas' page-locked memory
    // (submit_buffer.h builds without CUDA) and the handler images
    ~b9_ctx() {
        for (const UserHandler& u : users) cudaLibraryUnload(u.lib);
        for (const Segment& sg : segs) cudaEventDestroy(sg.ready);
        for (cudaEvent_t e : event_pool) cudaEventDestroy(e);
        if (sb) for (SubmitArena& A : sb->arena) {
            if (A.payload) cudaFreeHost(A.payload);
            if (A.offsets) cudaFreeHost(A.offsets);
            if (A.ids) cudaFreeHost(A.ids);
            if (A.flags) cudaFreeHost(A.flags);
        }
    }
};

namespace {

// A `ready` event for a new segment: an idle one of the pool, else a new one. Caller holds c->mu.
cudaError_t take_event(b9_ctx* c, cudaEvent_t* out) {
    if (c->event_pool.empty()) return cudaEventCreateWithFlags(out, cudaEventDisableTiming);
    *out = c->event_pool.back();
    c->event_pool.pop_back();
    return cudaSuccess;
}

// Gives a segment's `ready` event back to the pool. Caller holds c->mu.
void put_event(b9_ctx* c, cudaEvent_t e) { c->event_pool.push_back(e); }

// Appends a batch of n tasks at the tail as a new segment: ring bytes [start, start + bytes), its slots written by the work
// `ready` was recorded behind. max_len: its longest task (0: not known); n_pickle: its tasks carrying B9_TF_PICKLE. The next
// segment goes behind it, at most at `end` (the end of the free range it was placed in: the re-push fills ranges exactly,
// b9_ring_free_ranges). Caller holds c->mu.
void append_segment(b9_ctx* c, uint32_t n, uint64_t start, uint64_t bytes, uint32_t max_len, uint32_t n_pickle, cudaEvent_t ready,
                    uint64_t end = UINT64_MAX) {
    c->segs.push_back(Segment{c->tail_task, n, start, bytes, ready, max_len, n_pickle});
    c->write_pos = std::min<uint64_t>(start + b9_seg_span(bytes), end);
    c->tail_task += n;
    c->pending_bytes += bytes;
}

// Frees the segments the head has moved past. Caller holds c->mu.
void free_segments(b9_ctx* c) {
    while (!c->segs.empty() && c->segs.front().first_task + c->segs.front().n <= c->head_task) {
        put_event(c, c->segs.front().ready);
        c->segs.pop_front();
    }
    if (c->segs.empty()) c->write_pos = 0;
}

// Makes stream s wait until every pending task is on the device (each live segment's `ready`). Caller holds c->mu.
int wait_pending(const b9_ctx* c, cudaStream_t s) {
    for (const Segment& sg : c->segs) CU(cudaStreamWaitEvent(s, sg.ready, 0));
    return B9_OK;
}

// Copies the ids of the n tasks from `first_task` on between their ring slots and the linear buffer `buf` (16 bytes per id),
// in two pieces when the slots wrap the ring. to_ring: buf -> slots, else slots -> buf; kind as for cudaMemcpyAsync.
cudaError_t copy_slot_ids(const b9_ctx* c, uint64_t first_task, size_t n, const void* buf, bool to_ring, cudaMemcpyKind kind, cudaStream_t s) {
    const uint32_t slot0 = (uint32_t)(first_task & c->slot_mask);
    const size_t first = std::min<size_t>(n, (size_t)c->ring_tasks - slot0);
    auto copy = [&](uint4* slots, const uint8_t* lin, size_t k) {
        return to_ring ? cudaMemcpyAsync(slots, lin, k * 16, kind, s) : cudaMemcpyAsync((void*)lin, slots, k * 16, kind, s);
    };
    const cudaError_t e = copy(c->d_ids + slot0, (const uint8_t*)buf, first);
    if (e != cudaSuccess || first == n) return e;
    return copy(c->d_ids, (const uint8_t*)buf + first * 16, n - first);
}

// Closes the timed span of the drain launches enqueued so far (ev_b right behind the last drain kernel), before anything
// else goes on the drain stream. Caller holds c->out_mu.
void end_drain_span(b9_ctx* c) {
    if (!c->last_op_drain) return;
    c->last_op_drain = false;
    cudaSetDevice(c->device);
    cudaEventRecord(c->ev_b, c->stream);
}

// c->out_mu for every drain-stream user except b9_drain_launch: whatever it enqueues comes after the open span's end
struct OutLock {
    std::lock_guard<std::mutex> lk;
    explicit OutLock(b9_ctx* c) : lk(c->out_mu) { end_drain_span(c); }
};

// Physical payload offset of logical task `idx` of segment `sg` (idx == first_task + n gives the segment's
// end). Only partial-segment operations need it (a drain that stops inside a batch, the rebalance), so
// the host keeps no per-task index: the slot ring on the device is the index. Synchronous, 8 bytes.
int task_phys_off(b9_ctx* c, const Segment& sg, uint64_t idx, uint64_t* out) {
    if (idx == sg.first_task) { *out = sg.phys_start; return B9_OK; }
    if (idx == sg.first_task + sg.n) { *out = sg.phys_start + sg.bytes; return B9_OK; }
    c->last_op_drain = false;
    CU(cudaStreamWaitEvent(c->stream, sg.ready, 0));
    CU(cudaMemcpyAsync(&c->h_ctl->total, c->d_off + (uint32_t)(idx & c->slot_mask), sizeof(uint64_t), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    *out = c->h_ctl->total;
    return B9_OK;
}

// where can a segment of `bytes` go? returns false when the ring cannot take it now (ring_place.h)
bool place_segment(b9_ctx* c, uint64_t bytes, uint64_t* start) {
    uint64_t live = 0;
    for (const Segment& sg : c->segs) live += sg.bytes;
    return b9_ring_place(c->ring_bytes, !c->segs.empty(), c->segs.empty() ? 0 : c->segs.front().phys_start, c->write_pos, live, bytes, start) != 0;
}

// the context's result staging, with `ctl` as the control block whose byte cursor places the records' bytes. compacted:
// the launch leaves no record for cancelled slots (count mode), so its records' ids are written to d_out_ids; otherwise
// they stay in the ring and b9_drain_fetch copies them from there
DrainOut drain_out(const b9_ctx* c, DrainCtl* ctl, bool compacted) {
    DrainOut o;
    o.payload = c->d_out_payload; o.cap = c->max_result_bytes; o.off = c->d_out_off; o.len = c->d_out_len;
    o.ids = c->d_out_ids; o.status = c->d_out_status; o.has = c->d_out_has; o.ctl = ctl;
    o.ids_compacted = compacted ? 1u : 0u;
    return o;
}

// count mode (cancelled slots in the window): the ready-count prefix per warp-tile of `tile_tasks` slots that gives every
// record its index (tile_count_kernel + tile_scan_kernel, read by tile_ready_before)
cudaError_t launch_tile_counts(const DrainArgs& a, uint32_t tile_tasks, cudaStream_t s) {
    const uint32_t blocks = (a.n_tasks + TC_SLOTS - 1u) / TC_SLOTS;
    tile_count_kernel<<<blocks, TC_SLOTS, 0, s>>>(a.hdr, a.slot_mask, a.first_task, a.n_tasks, tile_tasks, (uint32_t*)a.tile_base, (uint32_t*)a.block_base);
    tile_scan_kernel<<<1, 1024, 0, s>>>((uint32_t*)a.block_base, blocks);
    return cudaGetLastError();
}

// every warp owns a slice of dynamic shared memory = control block + one stage buffer.
template <int H> uint32_t drain3_warp_stride(uint32_t in_cap) {
    const size_t ctl = (sizeof(D3Warp<D3Cfg<H>::T>) + 127u) & ~(size_t)127u;
    return (uint32_t)(ctl + (((size_t)in_cap + 64u + 127u) & ~(size_t)127u));
}
// overlap: the drain stream's last operation is a drain3_kernel and the window has no cancelled slot (so no count kernels
// run first): the kernel is launched as that one's programmatic dependent — its CTAs become resident as the previous
// grid's leave, and it waits for that grid's completion (griddepcontrol.wait) before it touches anything a drain writes
// *tt_out: the launch's tasks per warp-tile (a count-mode record index depends on it)
template <int H> cudaError_t launch_drain3(DrainArgs a, uint64_t avg_task_bytes, uint32_t max_task_len, uint32_t cap_override, int sm_count, bool overlap, cudaStream_t s, int* grid_out,
                                           uint32_t* tt_out) {
    constexpr int T = D3Cfg<H>::T;
    uint32_t in_cap = 0, stride = 0; size_t smem = 0; int per_sm = 0;
    void (*const kernel)(DrainArgs, uint32_t, uint32_t) = a.retry_mask ? drain3_kernel<H, true> : drain3_kernel<H, false>;
    // stage buffer per warp sized for the window's average warp-tile: tt tasks x 1.1 + 768 B, within [1 KiB, 48 KiB].
    // Tiles that do not fit are processed straight from global memory (same code, generic loads).
    // (crc32's configuration has long-tailed sizes - zipf strings - and gets a third of a tile of headroom: more would
    // cost resident warps, and its byte loop lives on those - 16 CTAs per SM fit with this, see D3Cfg::MIN_BLOCKS)
    auto size_for = [&](uint32_t tt) -> cudaError_t {
        const uint64_t want = (H == B9_H_CRC32) ? avg_task_bytes * tt * 27 / 20 + 768 : avg_task_bytes * tt * 11 / 10 + 768;
        in_cap = (uint32_t)std::min<uint64_t>(48u << 10, std::max<uint64_t>(1u << 10, want));
        // no tile of the window is longer than tt of its longest tasks (+ the alignment of its first byte): with uniform task
        // sizes (configs[3]: every task 372 bytes) the headroom above buys nothing and costs a resident CTA per SM
        if (H != B9_H_CRC32 && max_task_len) in_cap = (uint32_t)std::min<uint64_t>(in_cap, std::max<uint64_t>(1u << 10, (uint64_t)max_task_len * tt + 32u));
        in_cap = (in_cap + 127u) & ~127u;
        if (cap_override) in_cap = cap_override;
        stride = drain3_warp_stride<H>(in_cap);
        smem = (size_t)stride * D3_WARPS;
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, D3_WARPS * 32, smem);
        if (e != cudaSuccess) return e;
        if (per_sm < 1) per_sm = 1;
        return cudaSuccess;
    };
    uint32_t tt = (uint32_t)T;
    cudaError_t e = size_for(tt);
    if (e != cudaSuccess) return e;
    // json_sum works on a document with the whole warp: a window of about one 8-document tile per resident warp ends in a
    // ragged last round (configs[4]: 25 k documents per GPU over a few thousand resident warps); tiles of 4 balance it,
    // while larger windows (100 k documents) measured faster with 8
    if (H == B9_H_JSON_SUM && (uint64_t)(a.n_tasks + T - 1) / T < 3ull * (uint64_t)per_sm * (uint64_t)sm_count * D3_WARPS) {
        tt = 4u;
        e = size_for(tt);
        if (e != cudaSuccess) return e;
    }
    a.tile_tasks = tt;
    *tt_out = tt;
    a.n_tiles = (a.n_tasks + tt - 1) / tt;
    const uint32_t ctas_needed = (a.n_tiles + D3_WARPS - 1) / D3_WARPS;
    const int grid = (int)std::min<uint32_t>(ctas_needed, (uint32_t)(per_sm * sm_count));
    *grid_out = grid;
    // identity with nothing cancelled in the window has a uniform tile cost (its expensive tasks are deferred):
    // all but the last round of a worker's tiles are assigned statically, which measured faster; the same
    // switch made vadd_f32 slower, so it stays on pure work stealing like crc32 / json_sum.
    if (a.count_mode) {
        e = launch_tile_counts(a, tt, s);
        if (e != cudaSuccess) return e;
    }
    if (H == B9_H_IDENTITY) {
        // dyn: how many of a worker's last rounds come from the ticket counter. One is enough when every
        // tile costs the same; with 1 % of escape-dense strings a tile that holds one takes ~25 % longer (the warp checks its
        // escapes), a worker's static share can hold a dozen of them, and one round of slack does not absorb that: 3 rounds
        // measured faster than 1 on the mix and the same on clean input
        constexpr uint64_t dyn = 3;
        const uint64_t rounds = a.n_tiles / ((uint64_t)grid * D3_WARPS);
        a.static_rounds = rounds > dyn ? (uint32_t)(rounds - dyn) : 0u;
    }
    a.static_rounds = std::max(a.static_rounds, 1u);                       // every worker's first tile is static (drain3_kernel)
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid); cfg.blockDim = dim3(D3_WARPS * 32); cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = (overlap && !a.count_mode) ? 1 : 0;
    e = cudaLaunchKernelEx(&cfg, kernel, a, in_cap, stride);
    if (e != cudaSuccess) return e;
    return cudaGetLastError();
}

// Turns a pushed batch's relative offsets into ring slots (off, hdr, cold metadata).
__global__ void ingest_kernel(const uint64_t* __restrict__ rel_off, uint32_t n, uint64_t seg_start, uint64_t first_task, uint32_t slot_mask,
                              const int64_t* __restrict__ ts, const int64_t* __restrict__ exp, const uint8_t* __restrict__ retries,
                              const uint8_t* __restrict__ flags, uint64_t* __restrict__ off, uint64_t* __restrict__ hdr,
                              int64_t* __restrict__ ring_ts, int64_t* __restrict__ ring_exp) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t slot = (uint32_t)((first_task + i) & slot_mask);
    uint64_t o0 = rel_off[0], o = rel_off[i], o1 = rel_off[i + 1];
    off[slot] = seg_start + (o - o0);
    hdr[slot] = hdr_pack((uint32_t)(o1 - o), flags ? flags[i] : 0, retries ? retries[i] : 0);
    ring_ts[slot] = ts ? ts[i] : 0;
    ring_exp[slot] = exp ? exp[i] : 0;
}

// Marks expired pending tasks as cancelled (Dispatcher.monitor's unclaimed branch, dispatch.go:173-230).
__global__ void expire_kernel(uint64_t* __restrict__ hdr, const int64_t* __restrict__ expires, uint32_t slot_mask,
                              uint64_t first_task, uint32_t n, int64_t now_ns, unsigned long long* __restrict__ count) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t slot = (uint32_t)((first_task + i) & slot_mask);
    int64_t e = expires[slot];
    uint64_t h = hdr[slot];
    if (e != 0 && e <= now_ns && !(hdr_flags(h) & 1u)) {
        hdr[slot] = h | (1ull << 32);
        atomicAdd(count, 1ull);
    }
}

__global__ void count_cancelled_kernel(const uint64_t* __restrict__ hdr, uint32_t slot_mask, uint64_t first_task, uint32_t n, unsigned long long* __restrict__ count) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool hit = i < n && (hdr_flags(hdr[(uint32_t)((first_task + i) & slot_mask)]) & 1u);
    const uint32_t m = __ballot_sync(0xffffffffu, hit);
    if ((threadIdx.x & 31u) == 0u && m) atomicAdd(count, (unsigned long long)__popc(m));
}

// *out := the cancelled slots among tasks [head, head + depth), counted on stream s, which already waits for them. One kernel
// when depth > 0 (the caller counts it); synchronises s. Caller holds c->out_mu (d_count and h_count are the drain side's).
int count_cancelled(b9_ctx* c, uint64_t head, uint64_t depth, cudaStream_t s, uint64_t* out) {
    CU(cudaMemsetAsync(c->d_count, 0, sizeof(unsigned long long), s));
    if (depth) { count_cancelled_kernel<<<(uint32_t)((depth + 255) / 256), 256, 0, s>>>(c->d_hdr, c->slot_mask, head, (uint32_t)depth, c->d_count); CU(cudaGetLastError()); }
    CU(cudaMemcpyAsync(c->h_count, c->d_count, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    *out = *c->h_count;
    return B9_OK;
}

// cancelled_pending := the cancelled slots among the pending tasks, counted on the device. Caller holds c->out_mu (not c->mu).
int recount_cancelled_locked_out(b9_ctx* c) {
    uint64_t head = 0, depth = 0, count = 0;
    cudaStream_t s = c->stream;
    {
        std::lock_guard<std::mutex> lk(c->mu);
        head = c->head_task; depth = c->tail_task - c->head_task;
        if (const int rc = wait_pending(c, s)) return rc;
    }
    { const int rc = count_cancelled(c, head, depth, s, &count); if (rc) return rc; }
    std::lock_guard<std::mutex> lk(c->mu);
    // tasks pushed (with B9_TF_CANCELLED) after the snapshot are in cancelled_pending already but not in the count: keep them
    const uint64_t depth_now = c->tail_task - c->head_task;
    if (depth_now == depth) c->cancelled_pending = count;
    else c->cancelled_pending = std::max<uint64_t>(c->cancelled_pending, count);   // (an over-count only costs the count pre-pass)
    c->recount_cancelled = false;
    if (depth) c->stats.kernel_launches++;
    return B9_OK;
}

// Commits the pop of the fetched window (the head moves past it, its fully consumed segments are freed). Caller holds c->mu.
void commit_pop(b9_ctx* c) {
    c->head_task += c->res.popped; c->pending_bytes -= c->res.in_bytes; c->stats.tasks_drained += c->res.popped;
    c->cancelled_pending -= std::min<uint64_t>(c->cancelled_pending, (uint64_t)(c->res.popped - c->res.n));
    c->recount_cancelled = c->expired_since_launch;              // an expire ran between this drain's launch and its commit: its
                                                                  // count included tasks of the window that are gone now
    free_segments(c);
}

// The re-push's device half, for retried task k = the window task (task_of) of record rec[k]. retry_len_kernel, one thread
// per task: rel[k + 1] = its length (a scan then makes rel the exclusive byte prefix). retry_gather_kernel, one warp per
// task: its bytes are copied out of the claimed window into the scratch `bytes` at rel[k], with the slot words
// ingest_kernel writes for a push: retries + 1, the commit's timestamp, the same expiry, flags and id. The flags are the
// ones the task was pushed with: a task pushed cancelled leaves no record, so a CANCELLED bit here was set by a
// b9_expire sweep of the claimed window, and it is cleared. The reference's monitor expires only unclaimed tasks
// (dispatch.go:173-230) and RetryTask re-queues the task as it was; the kept expiry cancels it at the next b9_expire.
__global__ void retry_len_kernel(const uint32_t* __restrict__ rec, uint32_t n, const uint32_t* __restrict__ task_of, const uint64_t* __restrict__ hdr,
                                 uint64_t head, uint32_t slot_mask, uint64_t* __restrict__ rel) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k == 0) rel[0] = 0;
    if (k < n) rel[k + 1] = hdr_len(hdr[(uint32_t)((head + task_of[rec[k]]) & slot_mask)]);
}
__global__ void retry_gather_kernel(const uint32_t* __restrict__ rec, uint32_t n, const uint32_t* __restrict__ task_of, uint64_t head, uint32_t slot_mask,
                                    const uint8_t* __restrict__ payload, const uint64_t* __restrict__ off, const uint64_t* __restrict__ hdr,
                                    const uint4* __restrict__ ids, const int64_t* __restrict__ exp, const uint64_t* __restrict__ rel, int64_t now_unix,
                                    uint8_t* __restrict__ bytes, int64_t* __restrict__ o_ts, int64_t* __restrict__ o_exp, uint8_t* __restrict__ o_retries,
                                    uint8_t* __restrict__ o_flags, uint4* __restrict__ o_ids) {
    const uint32_t k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
    if (k >= n) return;
    const uint32_t slot = (uint32_t)((head + task_of[rec[k]]) & slot_mask);
    const uint64_t h = hdr[slot];
    warp_copy(bytes + rel[k], payload + off[slot], hdr_len(h), (int)lane);
    if (lane == 0) {
        o_ts[k] = now_unix; o_exp[k] = exp[slot]; o_retries[k] = (uint8_t)(hdr_retries(h) + 1u); o_flags[k] = (uint8_t)(hdr_flags(h) & ~B9_TF_CANCELLED); o_ids[k] = ids[slot];
    }
}

// b9_drain_fetch's commit when records are RETRY: the pop and the re-push of those tasks at the tail (Dispatcher.RetryTask's
// RPUSH, pkg/task/dispatch.go:232-285). Caller holds c->in_mu (the re-push is a push) and c->out_mu, and the records are
// fetched. Everything runs on the ingest stream, behind earlier pushes and ahead of later ones: the tasks are gathered out
// of the claimed window into scratch, then the space is placed in the same critical section that commits the pop (a
// producer cannot take the released space in between), then the bytes and slot words go to the new segment. When the
// ring has no room for it, nothing is committed: B9_ENOSPC. d2h_bytes: what the fetch read back, for the stats.
int commit_with_repush(b9_ctx* c, const std::vector<uint32_t>& retry_rec, float d2h_ms, uint64_t d2h_bytes) {
    const uint32_t k = (uint32_t)retry_rec.size();
    cudaStream_t s = c->stream_in;
    const uint64_t head = c->res.head;
    // (the retried bytes are at most the window's)
    { const int rc = c->d_retry_bytes.ensure(c->res.in_bytes + RING_SLACK, "b9_drain_fetch: re-push scratch"); if (rc) return rc; }
    size_t scan_bytes = 0;
    CU(cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, c->d_in_off + 1, c->d_in_off + 1, (int)k, s));
    { const int rc = c->d_retry_scan.ensure(scan_bytes, "b9_drain_fetch: re-push scan scratch"); if (rc) return rc; }
    const int64_t now = (int64_t)std::chrono::duration_cast<std::chrono::seconds>(std::chrono::system_clock::now().time_since_epoch()).count();
    CU(cudaMemcpyAsync(c->d_retry_rec, retry_rec.data(), (size_t)k * 4, cudaMemcpyHostToDevice, s));
    retry_len_kernel<<<(k + 255) / 256, 256, 0, s>>>(c->d_retry_rec, k, c->d_task_of, c->d_hdr, head, c->slot_mask, c->d_in_off);
    CU(cudaGetLastError());
    CU(cub::DeviceScan::InclusiveSum(c->d_retry_scan, scan_bytes, c->d_in_off + 1, c->d_in_off + 1, (int)k, s));
    retry_gather_kernel<<<(uint32_t)(((uint64_t)k * 32 + 255) / 256), 256, 0, s>>>(c->d_retry_rec, k, c->d_task_of, head, c->slot_mask, c->d_payload,
        c->d_off, c->d_hdr, c->d_ids, c->d_exp, c->d_in_off, now, c->d_retry_bytes, c->d_in_ts, c->d_in_exp, c->d_in_retries, c->d_in_flags, c->d_retry_ids);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(&c->h_ctl->total, c->d_in_off + k, sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    const uint64_t bytes = c->h_ctl->total;
    // Where the tasks go once the pop has released the window. The push segments the window consumes whole are free then;
    // a segment it ends inside is trimmed to start at the first task behind the window (its offset is read back here), so
    // that the window's bytes are free wherever they lie. The ring's free ranges then hold the retried bytes, which are at
    // most the window's: they are placed in range order as one segment, or two when the freed bytes straddle the ring's end.
    const uint64_t new_head = c->head_task + c->res.popped;               // (only drain-side calls move the head: out_mu is held)
    Segment part{}; bool partial = false;
    {
        std::lock_guard<std::mutex> lk(c->mu);
        for (const Segment& sg : c->segs)
            if (sg.first_task < new_head && new_head < sg.first_task + sg.n) { part = sg; partial = true; break; }
    }
    uint64_t cut = 0;
    if (partial) { const int rc = task_phys_off(c, part, new_head, &cut); if (rc) return rc; }
    uint64_t reg[2][2]; int n_reg = 0; uint64_t wp = 0;
    {
        std::lock_guard<std::mutex> lk(c->mu);
        bool have = false; uint64_t oldest = 0, live = 0;
        for (const Segment& sg : c->segs) {
            if (sg.first_task + sg.n <= new_head) continue;
            const uint64_t st = (partial && sg.first_task == part.first_task) ? cut : sg.phys_start;
            if (!have) { have = true; oldest = st; }
            live += sg.bytes - (st - sg.phys_start);
        }
        wp = have ? c->write_pos : 0;
        n_reg = b9_ring_free_ranges(c->ring_bytes, have, oldest, wp, live, reg);
    }
    // the plan: task range [i0, i1) at `at`, one entry per free range used (producers and drain-side calls are excluded
    // until the commit below, so the ranges stay free)
    struct Piece { uint32_t i0, i1; uint64_t at, end, lo, hi; };   // [lo, hi): its bytes in the scratch
    Piece plan[2]; int n_plan = 0;
    if (bytes == 0) plan[n_plan++] = Piece{0, k, wp, wp, 0, 0};                 // (empty HTTP bodies: no bytes to place)
    else if (n_reg && bytes <= reg[0][1] - reg[0][0]) plan[n_plan++] = Piece{0, k, reg[0][0], reg[0][1], 0, bytes};
    else if (n_reg == 2) {                                                 // split at a task boundary: the byte prefix is needed
        std::vector<uint64_t> rel((size_t)k + 1);
        CU(cudaMemcpyAsync(rel.data(), c->d_in_off, ((size_t)k + 1) * 8, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        uint32_t i = 0;
        for (int r = 0; r < 2 && i < k; ++r) {
            const uint64_t room = reg[r][1] - reg[r][0];
            const uint32_t e = (uint32_t)(std::upper_bound(rel.begin() + i, rel.end(), rel[i] + room) - rel.begin()) - 1u;
            if (e > i) { plan[n_plan++] = Piece{i, e, reg[r][0], reg[r][1], rel[i], rel[e]}; i = e; }
        }
        if (i < k) n_plan = 0;
    }
    // (never taken: the retried tasks are at most the window's slots and bytes, and the pop frees both)
    const bool slots_ok = (uint64_t)k <= (uint64_t)c->ring_tasks - (c->tail_task - new_head);
    if (!slots_ok || n_plan == 0)
        return fail(B9_ENOSPC, "b9_drain_fetch: the %u retried tasks (%llu bytes) find no room in the ring behind the pending ones; "
                    "nothing is committed", k, (unsigned long long)bytes);
    cudaEvent_t ready[2] = {nullptr, nullptr};
    {
        std::lock_guard<std::mutex> lk(c->mu);
        for (int q = 0; q < n_plan; ++q) CU(take_event(c, &ready[q]));
    }
    std::lock_guard<std::mutex> lk(c->mu);
    c->stats.last_drain_d2h_ms = d2h_ms;
    c->stats.bytes_d2h += d2h_bytes;
    commit_pop(c);
    if (partial)
        for (Segment& sg : c->segs)
            if (sg.first_task == part.first_task) {
                sg.bytes -= cut - sg.phys_start; sg.n -= (uint32_t)(new_head - sg.first_task);
                sg.first_task = new_head; sg.phys_start = cut;
                break;
            }
    const uint64_t tail = c->tail_task;
    // (enqueue only: nothing here waits for the device)
    CU(copy_slot_ids(c, tail, k, c->d_retry_ids, true, cudaMemcpyDeviceToDevice, s));
    for (int q = 0; q < n_plan; ++q) {
        const Piece& pc = plan[q];
        const uint32_t n = pc.i1 - pc.i0;
        if (pc.hi > pc.lo) CU(cudaMemcpyAsync(c->d_payload + pc.at, c->d_retry_bytes + pc.lo, pc.hi - pc.lo, cudaMemcpyDeviceToDevice, s));
        ingest_kernel<<<(n + 255) / 256, 256, 0, s>>>(c->d_in_off + pc.i0, n, pc.at, tail + pc.i0, c->slot_mask, c->d_in_ts + pc.i0,
                                                      c->d_in_exp + pc.i0, c->d_in_retries + pc.i0, c->d_in_flags + pc.i0,
                                                      c->d_off, c->d_hdr, c->d_ts, c->d_exp);
        CU(cudaGetLastError());
        CU(cudaEventRecord(ready[q], s));
        append_segment(c, n, pc.at, pc.hi - pc.lo, 0u, 0u, ready[q], pc.end);   // (no B9_TF_PICKLE task gets a RETRY record)
    }
    c->stats.kernel_launches += 3 + (uint64_t)n_plan;                      // (length, the scan, gather, ingest per segment)
    return B9_OK;
}

}  // namespace

extern "C" {

uint32_t b9_abi_version(void) { return B9_ABI_VERSION; }

int b9_set_retry_policy(b9_ctx* c, uint32_t exc_mask, uint32_t max_retries) {
    if (!c) return fail(B9_EINVAL, "b9_set_retry_policy: ctx is NULL");
    if (exc_mask & ~B9_EXC_ALL) return fail(B9_EINVAL, "b9_set_retry_policy: exception bits 0x%x are not B9_EXC_*", exc_mask & ~B9_EXC_ALL);
    if (max_retries > 255) return fail(B9_EINVAL, "b9_set_retry_policy: max_retries %u: a task's retries are one byte (b9_push_meta.retries)", max_retries);
    OutLock out_lk(c);
    if (exc_mask) {
        CU(cudaSetDevice(c->device));
        const uint64_t md = c->max_drain_tasks;
        int rc = c->d_task_of.ensure(md * sizeof(uint32_t), "b9_set_retry_policy: task_of");
        if (rc == B9_OK) rc = c->d_retry_rec.ensure(md * sizeof(uint32_t), "b9_set_retry_policy: retry records");
        if (rc == B9_OK) rc = c->d_retry_ids.ensure(md * sizeof(uint4), "b9_set_retry_policy: retry ids");
        if (rc) return rc;
    }
    c->retry_mask = exc_mask;
    c->max_retries = max_retries;
    return B9_OK;
}

int b9_set_callback_policy(b9_ctx* c, int enabled, const uint8_t* signing_key, uint32_t key_len) {
    if (!c) return fail(B9_EINVAL, "b9_set_callback_policy: ctx is NULL");
    if (enabled && key_len && !signing_key) return fail(B9_EINVAL, "b9_set_callback_policy: NULL signing_key with key_len %u", key_len);
    OutLock out_lk(c);
    if (enabled) {
        CU(cudaSetDevice(c->device));
        const uint64_t md = c->max_drain_tasks;
        int rc = c->d_cb_kind.ensure(md, "b9_set_callback_policy: callback kinds");
        if (rc == B9_OK) rc = c->d_cb_digest.ensure(md * 32, "b9_set_callback_policy: digests");
        if (rc) return rc;
    }
    c->cb_enabled = enabled != 0;
    c->cb_keyed = c->cb_enabled && key_len != 0;
    if (c->cb_keyed) callback_midstates(signing_key, key_len, c->cb_mid);
    else memset(c->cb_mid, 0, sizeof c->cb_mid);
    return B9_OK;
}

int b9_set_callback_runners(b9_ctx* c, uint32_t runners) {
    if (!c) return fail(B9_EINVAL, "b9_set_callback_runners: ctx is NULL");
    if (runners & ~(uint32_t)(B9_CB_RUNNER_FUNCTION | B9_CB_RUNNER_ENDPOINT)) return fail(B9_EINVAL, "b9_set_callback_runners: unknown bits 0x%x", runners);
    OutLock out_lk(c);
    if (runners) {
        CU(cudaSetDevice(c->device));
        const uint64_t md = c->max_drain_tasks;
        int rc = c->d_cb_body_off.ensure(md * sizeof(uint64_t), "b9_set_callback_runners: body offsets");   // (ensure takes bytes)
        if (rc == B9_OK) rc = c->d_cb_body_len.ensure(md * sizeof(uint32_t), "b9_set_callback_runners: body lengths");
        if (rc == B9_OK) rc = c->d_cb_url_off.ensure(md * sizeof(uint64_t), "b9_set_callback_runners: URL offsets");
        if (rc == B9_OK) rc = c->d_cb_url_len.ensure(md * sizeof(uint32_t), "b9_set_callback_runners: URL lengths");
        if (rc) return rc;
    }
    c->cb_runners = runners;
    return B9_OK;
}

int b9_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

const char* b9_last_error(const b9_ctx*) { return g_last_error.c_str(); }

static const char* const HANDLER_NAMES[B9_H_COUNT_] = {"identity", "crc32", "vadd_f32", "json_sum"};
const char* b9_handler_name(int h) { return (h >= 0 && h < B9_H_COUNT_) ? HANDLER_NAMES[h] : nullptr; }
int b9_handler_id(const char* name) {
    if (!name) return B9_EINVAL;
    if (!strcmp(name, "echo")) return B9_H_IDENTITY;
    for (int h = 0; h < B9_H_COUNT_; ++h) if (!strcmp(name, HANDLER_NAMES[h])) return h;
    return B9_ENOSYS;
}

// The length an image's own header gives it, checked against `size`: an ELF64 cubin whose header tables and sections lie
// within `size`, or a fatbin whose header and payload do. 0: neither, or truncated. (cudaLibraryLoadData takes no size:
// it reads what the header says, so the header is checked first.)
static uint64_t image_bytes(const uint8_t* b, uint64_t size) {
    if (size >= 64 && memcmp(b, "\x7f" "ELF", 4) == 0 && b[4] == 2) {                       // ELFCLASS64
        uint64_t phoff, shoff; uint16_t phentsize, phnum, shentsize, shnum;
        memcpy(&phoff, b + 0x20, 8); memcpy(&shoff, b + 0x28, 8);
        memcpy(&phentsize, b + 0x36, 2); memcpy(&phnum, b + 0x38, 2); memcpy(&shentsize, b + 0x3A, 2); memcpy(&shnum, b + 0x3C, 2);
        if (phoff > size || (uint64_t)phentsize * phnum > size - phoff) return 0;
        if (shoff > size || shentsize < 64 || (uint64_t)shentsize * shnum > size - shoff) return 0;
        uint64_t end = std::max<uint64_t>(phoff + (uint64_t)phentsize * phnum, shoff + (uint64_t)shentsize * shnum);
        for (uint32_t k = 0; k < shnum; ++k) {
            const uint8_t* sh = b + shoff + (uint64_t)k * shentsize;
            uint32_t type; uint64_t off, sz;
            memcpy(&type, sh + 4, 4); memcpy(&off, sh + 0x18, 8); memcpy(&sz, sh + 0x20, 8);
            if (type == 8) continue;                                                          // SHT_NOBITS
            if (off > size || sz > size - off) return 0;
            end = std::max<uint64_t>(end, off + sz);
        }
        return end;
    }
    uint32_t magic = 0;
    if (size >= 16) memcpy(&magic, b, 4);
    if (magic == 0xBA55ED50u) {                                                               // fatbin: magic, version, header size, payload size
        uint16_t hs; uint64_t fs;
        memcpy(&hs, b + 6, 2); memcpy(&fs, b + 8, 8);
        if (hs < 16 || fs > size || hs > size - fs) return 0;
        return hs + fs;
    }
    return 0;
}

int b9_handler_load(b9_ctx* c, const void* image, uint64_t size, const char* name, int32_t* handler_out) {
    if (!c || !image || !name || !handler_out) return fail(B9_EINVAL, "b9_handler_load: NULL argument");
    const size_t nl = strlen(name);
    bool ident = nl > 0 && nl <= 200 && !(name[0] >= '0' && name[0] <= '9');
    for (size_t k = 0; k < nl && ident; ++k) ident = name[k] == '_' || (name[k] >= '0' && name[k] <= '9') || ((name[k] | 0x20) >= 'a' && (name[k] | 0x20) <= 'z');
    if (!ident) return fail(B9_EINVAL, "b9_handler_load: \"%.64s\" is not a B9_HANDLER name (a C identifier)", name);
    if (!image_bytes((const uint8_t*)image, size))
        return fail(B9_EINVAL, "b9_handler_load: the image is not an ELF cubin or a fatbin that fits in %llu bytes", (unsigned long long)size);
    OutLock out_lk(c);
    CU(cudaSetDevice(c->device));
    UserHandler u;
    cudaError_t e = cudaLibraryLoadData(&u.lib, image, nullptr, nullptr, 0, nullptr, nullptr, 0);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(B9_EINVAL, "b9_handler_load: the image does not load on device %d: %s", c->device, cudaGetErrorString(e));
    }
    char tq[256], ep[256];
    snprintf(tq, sizeof tq, "b9h_v%d_tq_%s", B9_HANDLER_ABI_VERSION, name);
    snprintf(ep, sizeof ep, "b9h_v%d_ep_%s", B9_HANDLER_ABI_VERSION, name);
    e = cudaLibraryGetKernel(&u.tq, u.lib, tq);
    if (e == cudaSuccess) e = cudaLibraryGetKernel(&u.ep, u.lib, ep);
    if (e != cudaSuccess) {
        cudaGetLastError();
        cudaLibraryUnload(u.lib);
        return fail(B9_EINVAL, "b9_handler_load: the image has no entry %s / %s: it holds no B9_HANDLER(%s, ...), or it was built "
                               "against another handler ABI version than this library's %d (B9_HANDLER_ABI_VERSION)", tq, ep, name, B9_HANDLER_ABI_VERSION);
    }
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&u.per_sm_tq, (const void*)u.tq, USER_DRAIN_WARPS * 32, 0);
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&u.per_sm_ep, (const void*)u.ep, USER_DRAIN_WARPS * 32, 0);
    if (e != cudaSuccess) {
        cudaGetLastError();
        cudaLibraryUnload(u.lib);
        return fail(B9_EINVAL, "b9_handler_load: %s: %s", tq, cudaGetErrorString(e));
    }
    u.per_sm_tq = std::max(u.per_sm_tq, 1); u.per_sm_ep = std::max(u.per_sm_ep, 1);
    c->users.push_back(u);
    *handler_out = B9_H_USER_BASE + (int32_t)(c->users.size() - 1);
    return B9_OK;
}

int b9_ctx_create(const b9_opts* opts, b9_ctx** out) {
    if (!out) return fail(B9_EINVAL, "b9_ctx_create: out is NULL");
    *out = nullptr;
    b9_opts o{};
    if (opts) memcpy(&o, opts, std::min<size_t>(sizeof o, opts->struct_size ? opts->struct_size : sizeof o));
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return fail(B9_ENODEV, "b9_ctx_create: no CUDA device is visible; libb9gpu has no CPU path");
    }
    if (o.device < 0 || o.device >= ndev) return fail(B9_EINVAL, "b9_ctx_create: device %d of %d", o.device, ndev);
    b9_ctx* c = new (std::nothrow) b9_ctx();
    if (!c) return fail(B9_ENOMEM, "b9_ctx_create: host allocation failed");
    c->device = o.device;
    c->ring_bytes = pow2_ceil(o.ring_bytes ? o.ring_bytes : (1ull << 30));
    c->ring_tasks = (uint32_t)pow2_ceil(o.ring_tasks ? o.ring_tasks : (4u << 20));
    c->slot_mask = c->ring_tasks - 1;
    c->max_drain_tasks = o.max_drain_tasks ? o.max_drain_tasks : (2u << 20);
    if (c->max_drain_tasks >= (1u << 24)) c->max_drain_tasks = (1u << 24) - 1;
    if (c->max_drain_tasks > c->ring_tasks) c->max_drain_tasks = c->ring_tasks;
    c->max_result_bytes = o.max_result_bytes ? o.max_result_bytes : (1ull << 30);
    if (c->max_result_bytes >= (1ull << 38)) c->max_result_bytes = (1ull << 38) - 1;
    c->max_task_bytes = o.max_task_bytes ? std::min<uint32_t>(o.max_task_bytes, (1u << 30) - 1u) : (1u << 20);   // (two bits of a 32-bit length word carry flags)

#define CUC(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { \
    int rc_ = fail(e_ == cudaErrorMemoryAllocation ? B9_ENOMEM : B9_EIO, "%s failed: %s", #call, cudaGetErrorString(e_)); \
    b9_ctx_destroy(c); return rc_; } } while (0)
    CUC(cudaSetDevice(c->device));
    cudaDeviceProp prop{};
    CUC(cudaGetDeviceProperties(&prop, c->device));
    c->sm_count = prop.multiProcessorCount;
    CUC(cudaStreamCreateWithFlags(&c->stream.v, cudaStreamNonBlocking));
    CUC(cudaStreamCreateWithFlags(&c->stream_in.v, cudaStreamNonBlocking));
    CUC(cudaEventCreate(&c->ev_burst.v));
    CUC(cudaEventCreate(&c->ev_a.v)); CUC(cudaEventCreate(&c->ev_b.v)); CUC(cudaEventCreate(&c->ev_c.v)); CUC(cudaEventCreate(&c->ev_d.v));
    CUC(cudaEventCreate(&c->ev_pa.v)); CUC(cudaEventCreate(&c->ev_pb.v));
    const uint32_t rt = c->ring_tasks, md = c->max_drain_tasks;
    CUC(cudaMalloc(&c->d_payload.v, c->ring_bytes + RING_SLACK));
    CUC(cudaMemset(c->d_payload + c->ring_bytes, 0, RING_SLACK));
    CUC(cudaMalloc(&c->d_off.v, rt * sizeof(uint64_t)));
    CUC(cudaMalloc(&c->d_hdr.v, rt * sizeof(uint64_t)));
    CUC(cudaMalloc(&c->d_ids.v, rt * sizeof(uint4)));
    CUC(cudaMalloc(&c->d_ts.v, rt * sizeof(int64_t)));
    CUC(cudaMalloc(&c->d_exp.v, rt * sizeof(int64_t)));
    CUC(cudaMalloc(&c->d_in_off.v, ((size_t)rt + 1) * sizeof(uint64_t)));
    CUC(cudaMalloc(&c->d_in_ts.v, rt * sizeof(int64_t)));
    CUC(cudaMalloc(&c->d_in_exp.v, rt * sizeof(int64_t)));
    CUC(cudaMalloc(&c->d_in_retries.v, rt));
    CUC(cudaMalloc(&c->d_in_flags.v, rt));
    CUC(cudaMalloc(&c->d_out_payload.v, c->max_result_bytes + RING_SLACK));
    CUC(cudaMalloc(&c->d_out_off.v, ((size_t)md + 1) * sizeof(uint64_t)));
    CUC(cudaMalloc(&c->d_out_ids.v, (size_t)md * sizeof(uint4)));
    CUC(cudaMalloc(&c->d_out_status.v, md));
    CUC(cudaMalloc(&c->d_out_has.v, md));
    CUC(cudaMalloc(&c->d_out_len.v, (size_t)md * sizeof(uint32_t)));
    CUC(cudaMalloc(&c->d_slow.v, (size_t)md * sizeof(SlowItem)));
    CUC(cudaMemset(c->d_slow, 0, (size_t)md * sizeof(SlowItem)));
    CUC(cudaMalloc(&c->d_wire_env.v, sizeof(WireEnv)));
    {
        // Z_k = advance the reflected CRC-32 register over 2^k zero bytes, as 4 byte-indexed tables per k
        std::vector<uint32_t> tabs((size_t)CRC_SHIFT_LEVELS * 1024);
        uint32_t step[256];
        for (uint32_t i = 0; i < 256; ++i) { uint32_t v = i; for (int b = 0; b < 8; ++b) v = (v & 1u) ? (0xEDB88320u ^ (v >> 1)) : (v >> 1); step[i] = v; }
        auto apply = [&](const uint32_t* t, uint32_t v) { return t[v & 255] ^ t[256 + ((v >> 8) & 255)] ^ t[512 + ((v >> 16) & 255)] ^ t[768 + (v >> 24)]; };
        for (uint32_t j = 0; j < 4; ++j) for (uint32_t b = 0; b < 256; ++b) { uint32_t v = b << (8 * j); tabs[j * 256 + b] = step[v & 255] ^ (v >> 8); }   // k = 0: one zero byte
        for (int k = 1; k < CRC_SHIFT_LEVELS; ++k) {
            const uint32_t* prev = tabs.data() + (size_t)(k - 1) * 1024; uint32_t* cur = tabs.data() + (size_t)k * 1024;
            for (uint32_t j = 0; j < 4; ++j) for (uint32_t b = 0; b < 256; ++b) cur[j * 256 + b] = apply(prev, apply(prev, b << (8 * j)));
        }
        CUC(cudaMalloc(&c->d_crc_shift.v, tabs.size() * sizeof(uint32_t)));
        CUC(cudaMemcpy(c->d_crc_shift, tabs.data(), tabs.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    }
    CUC(cudaMalloc(&c->d_ctl.v, D3_CTL_RING * sizeof(DrainCtl)));
    CUC(cudaMemset(c->d_ctl, 0, D3_CTL_RING * sizeof(DrainCtl)));
    CUC(cudaMalloc(&c->d_tile_state.v, ((size_t)md / D2_THREADS + 2) * sizeof(uint64_t)));
    CUC(cudaMalloc(&c->d_count.v, sizeof(unsigned long long)));
    CUC(cudaHostAlloc(&c->h_ctl.v, sizeof(DrainCtl), cudaHostAllocDefault));
    CUC(cudaHostAlloc(&c->h_count.v, sizeof(unsigned long long), cudaHostAllocDefault));
    c->stats.sm_count = (uint32_t)c->sm_count;
    if (const char* v = getenv("B9_STAGE_BYTES")) c->stage_bytes_override = ((uint32_t)atoi(v) + 1023u) & ~1023u;
#undef CUC
    *out = c;
    return B9_OK;
}

void b9_ctx_destroy(b9_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    if (c->stream_in) cudaStreamSynchronize(c->stream_in);
    if (c->nccl_comm) nccl_comm_destroy(c->nccl_comm);
    delete c;                                   // (its members release the device memory, pinned memory, events and streams)
}

void* b9_host_alloc(b9_ctx* c, uint64_t bytes) {
    if (!c) { fail(B9_EINVAL, "b9_host_alloc: ctx is NULL"); return nullptr; }
    void* p = nullptr;
    cudaSetDevice(c->device);
    cudaError_t e = cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault);
    if (e != cudaSuccess) { fail(B9_ENOMEM, "cudaHostAlloc(%llu) failed: %s", (unsigned long long)bytes, cudaGetErrorString(e)); return nullptr; }
    return p;
}

void b9_host_free(b9_ctx* c, void* p) {
    if (!p) return;
    if (c) cudaSetDevice(c->device);
    cudaFreeHost(p);
}

// One push. Reservation and commit of the ring space are two short critical sections under c->mu; the DMA and the
// ingest kernel are enqueued between them under c->in_mu only, so a drain can run (and be synchronised) meanwhile.
// The batch becomes visible to drains (tail_task) only at the commit, after its `ready` event has been recorded.
// `after`: optional event recorded once the copies are enqueued (b9_batch_push_v's arena reuse).
static int push_impl(b9_ctx* c, const uint8_t* task_ids, const uint8_t* payload, const uint64_t* offsets, uint32_t n, const b9_push_meta* meta, bool wait,
                     cudaEvent_t after = nullptr) {
    if (!c) return fail(B9_EINVAL, "b9_batch_push: ctx is NULL");
    if (n == 0) return B9_OK;
    if (!task_ids || !payload || !offsets) return fail(B9_EINVAL, "b9_batch_push: NULL buffer");
    if (offsets[n] < offsets[0]) return fail(B9_EINVAL, "b9_batch_push: offsets not monotonic");
    const uint64_t bytes = offsets[n] - offsets[0];
    std::lock_guard<std::mutex> in_lk(c->in_mu);
    CU(cudaSetDevice(c->device));
    uint64_t start = 0, tail = 0;
    cudaEvent_t ready = nullptr;
    {
        std::lock_guard<std::mutex> lk(c->mu);
        free_segments(c);
        if ((uint64_t)n > (uint64_t)c->ring_tasks - (c->tail_task - c->head_task))
            return fail(B9_ENOSPC, "b9_batch_push: %u tasks do not fit (%llu of %u slots pending)", n,
                        (unsigned long long)(c->tail_task - c->head_task), c->ring_tasks);
        if (!place_segment(c, bytes, &start))
            return fail(B9_ENOSPC, "b9_batch_push: %llu payload bytes do not fit the ring (%llu pending of %llu)",
                        (unsigned long long)bytes, (unsigned long long)c->pending_bytes, (unsigned long long)c->ring_bytes);
        CU(take_event(c, &ready));
        tail = c->tail_task;
    }
    cudaStream_t s = c->stream_in;
    CU(cudaEventRecord(c->ev_pa, s));
    // the payload DMA goes first (into ring space that stays free until this push is committed), so that
    // the O(n) host-side validation of the index below runs while the bytes are already on the wire
    if (bytes) CU(cudaMemcpyAsync(c->d_payload + start, payload + offsets[0], bytes, cudaMemcpyHostToDevice, s));
    uint64_t n_cancelled = 0;
    uint32_t seg_max_len = 0, n_pickle = 0;
    {
        const uint32_t maxb = c->max_task_bytes;
        uint64_t bad = ~0ull, big = ~0ull, prev = offsets[0], longest = 0;
        for (uint32_t i = 0; i < n; ++i) {
            const uint64_t cur = offsets[i + 1];
            if (cur < prev) { if (bad == ~0ull) bad = i; }
            else { if (cur - prev > maxb && big == ~0ull) big = i; longest = std::max(longest, cur - prev); }
            prev = cur;
        }
        seg_max_len = (uint32_t)std::min<uint64_t>(longest, maxb);
        if (bad != ~0ull || big != ~0ull) {
            { std::lock_guard<std::mutex> lk(c->mu); put_event(c, ready); }
            cudaStreamSynchronize(s);            // the stray DMA must not outlive the caller's buffer
            if (bad != ~0ull) return fail(B9_EINVAL, "b9_batch_push: offsets not monotonic at task %llu", (unsigned long long)bad);
            return fail(B9_E2BIG, "b9_batch_push: task %llu is %llu bytes, max_task_bytes is %u", (unsigned long long)big,
                        (unsigned long long)(offsets[big + 1] - offsets[big]), maxb);
        }
        if (meta && meta->flags) for (uint32_t i = 0; i < n; ++i) {
            n_cancelled += (meta->flags[i] & B9_TF_CANCELLED) ? 1 : 0;
            n_pickle += (meta->flags[i] & B9_TF_PICKLE) ? 1 : 0;
        }
    }
    CU(cudaMemcpyAsync(c->d_in_off, offsets, ((size_t)n + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
    CU(copy_slot_ids(c, tail, n, task_ids, true, cudaMemcpyHostToDevice, s));   // (ids go straight into their ring slots)
    const int64_t* ts = nullptr; const int64_t* ex = nullptr; const uint8_t* rt = nullptr; const uint8_t* fl = nullptr;
    uint64_t meta_bytes = 0;
    if (meta) {
        if (meta->timestamp_unix)  { CU(cudaMemcpyAsync(c->d_in_ts, meta->timestamp_unix, (size_t)n * 8, cudaMemcpyHostToDevice, s)); ts = c->d_in_ts; meta_bytes += (uint64_t)n * 8; }
        if (meta->expires_unix_ns) { CU(cudaMemcpyAsync(c->d_in_exp, meta->expires_unix_ns, (size_t)n * 8, cudaMemcpyHostToDevice, s)); ex = c->d_in_exp; meta_bytes += (uint64_t)n * 8; }
        if (meta->retries)         { CU(cudaMemcpyAsync(c->d_in_retries, meta->retries, n, cudaMemcpyHostToDevice, s)); rt = c->d_in_retries; meta_bytes += n; }
        if (meta->flags)           { CU(cudaMemcpyAsync(c->d_in_flags, meta->flags, n, cudaMemcpyHostToDevice, s)); fl = c->d_in_flags; meta_bytes += n; }
    }
    CU(cudaEventRecord(c->ev_pb, s));
    if (after) CU(cudaEventRecord(after, s));
    ingest_kernel<<<(n + 255) / 256, 256, 0, s>>>(c->d_in_off, n, start, tail, c->slot_mask, ts, ex, rt, fl,
                                                  c->d_off, c->d_hdr, c->d_ts, c->d_exp);
    CU(cudaGetLastError());
    CU(cudaEventRecord(ready, s));
    {
        std::lock_guard<std::mutex> lk(c->mu);
        append_segment(c, n, start, bytes, seg_max_len, n_pickle, ready);   // (tail_task == tail: in_mu is held)
        c->cancelled_pending += n_cancelled;
        c->stats.kernel_launches++;
        c->stats.tasks_pushed += n;
        c->stats.bytes_h2d += bytes + ((uint64_t)n + 1) * 8 + (uint64_t)n * 16 + meta_bytes;
    }
    if (wait) {
        CU(cudaStreamSynchronize(s));            // the caller may reuse its buffers as soon as we return
        float ms = 0; cudaEventElapsedTime(&ms, c->ev_pa, c->ev_pb);
        std::lock_guard<std::mutex> lk(c->mu); c->stats.last_push_h2d_ms = ms;
    }
    return B9_OK;
}

int b9_batch_push(b9_ctx* c, const uint8_t* task_ids, const uint8_t* payload, const uint64_t* offsets, uint32_t n, const b9_push_meta* meta) {
    return push_impl(c, task_ids, payload, offsets, n, meta, true);
}

int b9_batch_push_async(b9_ctx* c, const uint8_t* task_ids, const uint8_t* payload, const uint64_t* offsets, uint32_t n, const b9_push_meta* meta) {
    return push_impl(c, task_ids, payload, offsets, n, meta, false);
}

// The pack step of the north star ("packs the whole pending batch into pinned host buffers"): n payloads scattered over
// the caller's (pageable) memory — Go's [][]byte — are gathered by a few threads into one of two page-locked arenas of
// the context, the n + 1 offsets are built on the way, and the arena is pushed asynchronously. Everything the call
// needs has been copied when it returns (cgo pointer rules); the arena is reused two pushes later, after its DMA.
int b9_batch_push_v(b9_ctx* c, const uint8_t* task_ids, const uint8_t* const* payloads, const uint32_t* lengths, uint32_t n, const b9_push_meta* meta) {
    if (!c) return fail(B9_EINVAL, "b9_batch_push_v: ctx is NULL");
    if (n == 0) return B9_OK;
    if (!task_ids || !payloads || !lengths) return fail(B9_EINVAL, "b9_batch_push_v: NULL buffer");
    std::lock_guard<std::mutex> pk(c->pack_mu);
    CU(cudaSetDevice(c->device));
    if (!c->pack_pool) {
        int nt = (int)std::min<unsigned>(16u, std::max(1u, std::thread::hardware_concurrency()));
        if (const char* e = getenv("B9_PACK_THREADS")) nt = std::max(1, atoi(e));
        c->pack_pool.reset(new (std::nothrow) PackPool(nt));
        if (!c->pack_pool) return fail(B9_ENOMEM, "b9_batch_push_v: thread pool");
    }
    const int T = c->pack_pool->nthreads;
    // pass 1: bytes per thread range (ranges of equal task count)
    std::vector<uint64_t> part((size_t)T + 1, 0);
    auto lo_of = [&](int t) { return (uint32_t)((uint64_t)n * (uint64_t)t / (uint64_t)T); };
    c->pack_pool->run([&](int t) {
        uint64_t sum = 0; const uint32_t lo = lo_of(t), hi = lo_of(t + 1);
        for (uint32_t i = lo; i < hi; ++i) sum += lengths[i];
        part[(size_t)t + 1] = sum;
    });
    for (int t = 0; t < T; ++t) part[(size_t)t + 1] += part[(size_t)t];
    const uint64_t total = part[(size_t)T];
    PackArena& A = c->pack[c->pack_next];
    c->pack_next ^= 1;
    if (A.in_flight) { CU(cudaEventSynchronize(A.free_ev)); A.in_flight = false; }   // its previous batch is on the device
    if (!A.free_ev) CU(cudaEventCreateWithFlags(&A.free_ev.v, cudaEventDisableTiming));
    // (room for a quarter more bytes, and a quarter + 16 more tasks)
    { const int rc = A.payload.ensure(total + 64, "b9_batch_push_v: page-locked payload", (total + 64) / 4); if (rc) return rc; }
    { const int rc = A.offsets.ensure(((uint64_t)n + 1) * 8, "b9_batch_push_v: page-locked offsets", ((uint64_t)n / 4 + 16) * 8); if (rc) return rc; }
    { const int rc = A.ids.ensure((uint64_t)n * 16, "b9_batch_push_v: page-locked ids", ((uint64_t)n / 4 + 16) * 16); if (rc) return rc; }
    // pass 2: gather
    c->pack_pool->run([&](int t) {
        const uint32_t lo = lo_of(t), hi = lo_of(t + 1);
        uint64_t o = part[(size_t)t];
        // the payloads sit anywhere in pageable memory: without a hint every task starts with a TLB miss and a chain of
        // cache misses the copy then waits for; the first lines of the task PF ahead are requested while this one is copied
        constexpr uint32_t PF = 8;
        for (uint32_t i = lo; i < hi; ++i) {
            if (i + PF < hi) {
                const uint8_t* q = payloads[i + PF];
                const uint32_t ql = lengths[i + PF];
                for (uint32_t b = 0; b < ql && b < 512u; b += 64u) __builtin_prefetch(q + b, 0, 0);
            }
            A.offsets[i] = o;
            const uint32_t l = lengths[i];
            if (l) memcpy(A.payload + o, payloads[i], l);
            o += l;
        }
        memcpy(A.ids + (size_t)lo * 16, task_ids + (size_t)lo * 16, (size_t)(hi - lo) * 16);
    });
    A.offsets[n] = total;
    const int rc = push_impl(c, A.ids, A.payload, A.offsets, n, meta, /*wait=*/false, A.free_ev);
    if (rc == B9_OK) A.in_flight = true;
    return rc;
}

// ---- single-task submissions from many threads, batched under the hood (submit_buffer.h) ------------------------------
static int sb_ensure(b9_ctx* c) {
    std::lock_guard<std::mutex> lk(c->sb_mu);
    if (c->sb) return B9_OK;
    CU(cudaSetDevice(c->device));
    uint64_t bytes = 64ull << 20; uint32_t tasks = 256u << 10;
    if (const char* e = getenv("B9_SUBMIT_BYTES")) bytes = (uint64_t)std::max<long long>(4096, atoll(e));
    if (const char* e = getenv("B9_SUBMIT_TASKS")) tasks = (uint32_t)std::max<long long>(16, atoll(e));
    tasks = std::min<uint32_t>(tasks, c->ring_tasks);
    bytes = std::min<uint64_t>(bytes, c->ring_bytes / 2);
    SubmitBuffer* sb = new (std::nothrow) SubmitBuffer();
    if (!sb) return fail(B9_ENOMEM, "b9_submit: buffer");
    for (int k = 0; k < 2; ++k) {
        SubmitArena& A = sb->arena[k];
        if (cudaHostAlloc(&A.payload, bytes, cudaHostAllocDefault) != cudaSuccess || cudaHostAlloc(&A.offsets, ((size_t)tasks + 1) * 8, cudaHostAllocDefault) != cudaSuccess ||
            cudaHostAlloc(&A.ids, (size_t)tasks * 16, cudaHostAllocDefault) != cudaSuccess || cudaHostAlloc(&A.flags, tasks, cudaHostAllocDefault) != cudaSuccess) {
            cudaGetLastError();
            return fail(B9_ENOMEM, "b9_submit: %llu bytes of page-locked memory per arena", (unsigned long long)bytes);
        }
        A.cap_bytes = bytes; A.cap_tasks = tasks;
        CU(cudaEventCreateWithFlags(&c->sb_free[k].v, cudaEventDisableTiming));
    }
    c->sb.reset(sb);
    return B9_OK;
}

static int sb_push(b9_ctx* c, int k, uint32_t n) {
    SubmitArena& A = c->sb->arena[k];
    b9_push_meta meta{}; meta.flags = A.any_flags.load(std::memory_order_relaxed) ? A.flags : nullptr;
    const int rc = push_impl(c, A.ids, A.payload, A.offsets, n, meta.flags ? &meta : nullptr, /*wait=*/false, c->sb_free[k]);
    if (rc == B9_OK) { c->sb_in_flight[k] = true; c->sb_unpushed = -1; }
    else { c->sb_unpushed = k; c->sb_unpushed_n = n; }                       // nothing is lost: the next flush pushes it again
    return rc;
}

int64_t b9_flush(b9_ctx* c) {
    if (!c) return fail(B9_EINVAL, "b9_flush: ctx is NULL");
    if (!c->sb) return 0;
    SubmitBuffer* sb = c->sb.get();
    std::lock_guard<std::mutex> lk(sb->flush_mu);
    CU(cudaSetDevice(c->device));
    int64_t pushed = 0;
    if (c->sb_unpushed >= 0) {                                               // an earlier batch the ring refused
        const uint32_t n = c->sb_unpushed_n;
        const int rc = sb_push(c, c->sb_unpushed, n);
        if (rc) return rc;
        pushed += n;
    }
    const int cur = sb->active.load(std::memory_order_acquire), other = cur ^ 1;
    if (sb->buffered() == 0) return pushed;
    // the other arena takes the submissions from now on: its previous batch must be on the device
    if (c->sb_in_flight[other]) { CU(cudaEventSynchronize(c->sb_free[other])); c->sb_in_flight[other] = false; }
    SubmitBuffer::reset(sb->arena[other]);
    uint32_t n = 0; uint64_t bytes = 0;
    sb->seal(&n, &bytes);
    if (n == 0) return pushed;
    const int rc = sb_push(c, cur, n);
    if (rc) return rc;
    return pushed + n;
}

int b9_submit(b9_ctx* c, const uint8_t* task_id, const uint8_t* payload, uint32_t length, uint8_t flags) {
    if (!c || !task_id || (!payload && length)) return fail(B9_EINVAL, "b9_submit: NULL argument");
    if (length > c->max_task_bytes) return fail(B9_E2BIG, "b9_submit: task is %u bytes, max_task_bytes is %u", length, c->max_task_bytes);
    if (!c->sb) { const int rc = sb_ensure(c); if (rc) return rc; }
    for (int attempt = 0; attempt < 64; ++attempt) {
        const int r = c->sb->submit(task_id, payload, length, flags);
        if (r == SUBMIT_OK) return B9_OK;
        if (r == SUBMIT_TOO_BIG) return fail(B9_E2BIG, "b9_submit: task is %u bytes, the submission arena holds %llu", length, (unsigned long long)c->sb->arena[0].cap_bytes);
        const int64_t f = b9_flush(c);                                       // the arena is full: hand it to the device, go on in the other one
        if (f < 0) return (int)f;
    }
    return fail(B9_ENOSPC, "b9_submit: the submission arenas stay full");
}

uint64_t b9_buffered(b9_ctx* c) {
    if (!c || !c->sb) return 0;
    return (uint64_t)c->sb->buffered() + (c->sb_unpushed >= 0 ? c->sb_unpushed_n : 0u);
}

uint64_t b9_depth(b9_ctx* c) {
    if (!c) return 0;
    std::lock_guard<std::mutex> lk(c->mu);
    return c->tail_task - c->head_task;
}

uint64_t b9_depth_bytes(b9_ctx* c) {
    if (!c) return 0;
    std::lock_guard<std::mutex> lk(c->mu);
    return c->pending_bytes;
}

uint64_t b9_running(b9_ctx* c) { return c ? c->running.load(std::memory_order_relaxed) : 0; }

int64_t b9_expire(b9_ctx* c, int64_t now_unix_ns) {
    if (!c) return fail(B9_EINVAL, "b9_expire: ctx is NULL");
    OutLock out_lk(c);
    CU(cudaSetDevice(c->device));
    uint64_t head = 0, depth = 0;
    {
        std::lock_guard<std::mutex> lk(c->mu);
        head = c->head_task; depth = c->tail_task - c->head_task;
        if (!depth) return 0;
        if (const int rc = wait_pending(c, c->stream)) return rc;
    }
    CU(cudaMemsetAsync(c->d_count, 0, sizeof(unsigned long long), c->stream));
    expire_kernel<<<(uint32_t)((depth + 255) / 256), 256, 0, c->stream>>>(c->d_hdr, c->d_exp, c->slot_mask, head, (uint32_t)depth, now_unix_ns, c->d_count);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(c->h_count, c->d_count, sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    std::lock_guard<std::mutex> lk(c->mu);
    c->stats.kernel_launches++;
    c->cancelled_pending += *c->h_count;
    c->expired_since_launch = true;
    return (int64_t)*c->h_count;
}

// StopTasks (pkg/api/v1/task.go:333-398) for the pending tasks of this ctx: cancel_kernel (cancel.cuh) over the ring.
// The claimed window of an outstanding drain is looked up but never written, so b9_drain_fetch's
// `cancelled_pending -= popped - records` stays exact without a recount.
int64_t b9_cancel(b9_ctx* c, const uint8_t* task_ids, uint32_t n, uint8_t* outcome) {
    if (!c) return fail(B9_EINVAL, "b9_cancel: ctx is NULL");
    if (n && !task_ids) return fail(B9_EINVAL, "b9_cancel: task_ids is NULL");
    if (n > (1u << 20)) return fail(B9_E2BIG, "b9_cancel: %u ids in one call, at most 2^20", n);
    if (outcome && n) memset(outcome, 0, n);
    if (n == 0) return 0;
    // sorted outside the locks: producers and drains do not wait for it
    std::vector<CancelKey> keys; std::vector<uint32_t> which;
    try { cancel_sort_unique(task_ids, n, keys, which); } catch (const std::bad_alloc&) { return fail(B9_ENOMEM, "b9_cancel: host allocation failed"); }
    const uint32_t n_keys = (uint32_t)keys.size();
    OutLock out_lk(c);
    CU(cudaSetDevice(c->device));
    cudaStream_t s = c->stream;
    uint64_t head = 0, depth = 0;
    {
        std::lock_guard<std::mutex> lk(c->mu);
        head = c->head_task; depth = c->tail_task - c->head_task;
        if (!depth) return 0;
        if (const int rc = wait_pending(c, s)) return rc;
    }
    const uint32_t claimed = (uint32_t)std::min<uint64_t>(c->running.load(std::memory_order_relaxed), depth);   // (set and cleared under out_mu)
    { const int rc = c->d_cancel_keys.ensure((uint64_t)n_keys * sizeof(CancelKey), "b9_cancel: keys"); if (rc) return rc; }
    { const int rc = c->d_cancel_out.ensure((uint64_t)n_keys * sizeof(uint32_t), "b9_cancel: outcome words"); if (rc) return rc; }
    CU(cudaMemcpyAsync(c->d_cancel_keys, keys.data(), (size_t)n_keys * sizeof(CancelKey), cudaMemcpyHostToDevice, s));
    CU(cudaMemsetAsync(c->d_cancel_out, 0, (size_t)n_keys * sizeof(uint32_t), s));
    CU(cudaMemsetAsync(c->d_count, 0, sizeof(unsigned long long), s));
    const uint32_t stride = cancel_fence_stride(n_keys), n_fence = (n_keys + stride - 1u) / stride;
    const uint32_t grid = (uint32_t)std::min<uint64_t>((depth + 255) / 256, (uint64_t)c->sm_count * 8u);
    cancel_kernel<<<grid, 256, (size_t)n_fence * sizeof(CancelKey), s>>>(c->d_hdr, c->d_ids, c->slot_mask, head, claimed, (uint32_t)depth,
                                                                         c->d_cancel_keys, n_keys, stride, n_fence, c->d_cancel_out, c->d_count);
    CU(cudaGetLastError());
    std::vector<uint32_t> words(n_keys);
    CU(cudaMemcpyAsync(words.data(), c->d_cancel_out, (size_t)n_keys * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    CU(cudaMemcpyAsync(c->h_count, c->d_count, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    const uint64_t marked = *c->h_count;
    {
        std::lock_guard<std::mutex> lk(c->mu);
        c->stats.kernel_launches++;
        c->cancelled_pending += marked;
    }
    if (outcome) for (uint32_t i = 0; i < n; ++i) outcome[i] = (uint8_t)words[which[i]];
    return (int64_t)marked;
}

// Waits for the last launch and publishes its outcome (records, bytes, overflow) to the ctx. Caller holds c->out_mu (not c->mu).
static int finish_launch(b9_ctx* c) {
    if (!c->res.async) return B9_OK;
    c->res.async = false;
    end_drain_span(c);
    CU(cudaMemcpyAsync(c->h_ctl, c->d_ctl + c->ctl_last, sizeof(DrainCtl), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    // one launch: the time around its kernels; a burst of B9_DRAIN_ASYNC launches: from the first one's start to the last one's end
    float ms = 0; cudaEventElapsedTime(&ms, c->ev_burst, c->ev_b);
    c->burst_open = false;
    c->res.kernel_ms = ms;
    if (c->h_ctl->overflow) {
        c->running.store(0, std::memory_order_relaxed);
        return fail(B9_ENOSPC, "b9_drain_launch: results exceed max_result_bytes (%llu); drain fewer tasks or enlarge the staging",
                    (unsigned long long)c->max_result_bytes);
    }
    c->res.bytes = c->h_ctl->bytes; c->res.n = c->h_ctl->total_cnt;
    c->res.popped = c->res.async_n;
    c->res.in_bytes = c->res.async_in_bytes;
    c->res.have = true;
    std::lock_guard<std::mutex> lk(c->mu);
    c->stats.last_drain_kernel_ms = ms;
    c->stats.last_drain_in_bytes = c->res.async_in_bytes;
    c->stats.last_drain_out_bytes = c->res.bytes;
    return B9_OK;
}

// What b9_drain_launch and b9_endpoint_drain_launch share: the window snapshot, the segment waits, the epoch and the
// control ring, the count-mode prefixes, the stats and the finish. endpoint: answer with endpoint_drain_kernel (the
// endpoint runner's responses) instead of drain3_kernel (the task-queue runner's results).
static int64_t drain_launch_common(b9_ctx* c, int handler, uint32_t max_tasks, int peek, bool endpoint) {
    std::lock_guard<std::mutex> out_lk(c->out_mu);
    // a user handler (b9_handler_load): an id this context returned, and not with the function path's pass
    const UserHandler* user = nullptr;
    if (handler >= B9_H_USER_BASE) {
        if ((size_t)(handler - B9_H_USER_BASE) >= c->users.size())
            return fail(B9_ENOSYS, "%s: unknown handler %d (not loaded into this context)", endpoint ? "b9_endpoint_drain_launch" : "b9_drain_launch", handler);
        if (peek & B9_DRAIN_PICKLE_FULL) return fail(B9_EINVAL, "b9_drain_launch: B9_DRAIN_PICKLE_FULL does not apply to a user handler (%d)", handler);
        user = &c->users[handler - B9_H_USER_BASE];
    }
    CU(cudaSetDevice(c->device));
    // results of an earlier launch that were never fetched are dropped; their tasks are still
    // pending (a pop is committed by a successful fetch, never by a launch). (An open burst of async launches stays open.)
    c->res = WaitingResults{};
    c->running.store(0, std::memory_order_relaxed);
    c->res_gen++;
    c->res.peek = (peek & B9_DRAIN_PEEK) != 0;
    // the callback pass signs with the host clock's Unix seconds, read once per launch (SignPayload's time.Now().Unix())
    c->res.cb = c->cb_enabled && (!endpoint || (c->cb_runners & B9_CB_RUNNER_ENDPOINT)); c->res.cb_keyed = c->res.cb && c->cb_keyed;
    c->res.cb_ts = c->res.cb_keyed ? (int64_t)std::chrono::duration_cast<std::chrono::seconds>(std::chrono::system_clock::now().time_since_epoch()).count() : 0;
    cudaStream_t s = c->stream;
    // the window: a snapshot of the ring's head under the bookkeeping lock. Only drain-side calls (all under out_mu)
    // move the head or free segments, so the snapshot stays valid while the launch is prepared without c->mu.
    struct Piece { Segment sg; uint64_t a, b; bool wait; };
    std::vector<Piece> pieces;
    uint64_t head = 0; uint32_t n = 0; uint32_t count_mode = 0;
    bool win_pickle = false;                                                // a B9_TF_PICKLE task may be in the window
    {
        std::lock_guard<std::mutex> lk(c->mu);
        head = c->head_task;
        const uint64_t depth = c->tail_task - c->head_task;
        n = (uint32_t)std::min<uint64_t>(std::min<uint64_t>(depth, max_tasks), c->max_drain_tasks);
        count_mode = c->cancelled_pending ? 1u : 0u;
        c->expired_since_launch = false;
        const uint64_t lo = head, hi = head + n;
        for (Segment& sg : c->segs) {
            const uint64_t a = std::max<uint64_t>(lo, sg.first_task), b = std::min<uint64_t>(hi, sg.first_task + sg.n);
            if (a < b) { pieces.push_back(Piece{sg, a, b, !sg.drain_waited}); sg.drain_waited = true; win_pickle |= sg.n_pickle != 0; }
        }
    }
    if (n == 0) { c->res.have = true; return 0; }
    uint64_t in_bytes = 0;                                                  // payload bytes of the window
    uint32_t win_max_len = 0; bool max_known = true;                        // its longest task, when every batch in it told
    for (const Piece& pc : pieces) { if (pc.sg.max_len) win_max_len = std::max(win_max_len, pc.sg.max_len); else max_known = false; }
    if (!max_known) win_max_len = 0;
    for (const Piece& pc : pieces) {
        if (pc.wait) {                                                      // this batch's H2D + ingest must have landed
            c->last_op_drain = false;                                       // (once per segment: stream order covers later drains)
            CU(cudaStreamWaitEvent(s, pc.sg.ready, 0));
        }
        uint64_t o0 = 0, o1 = 0;
        int rc = task_phys_off(c, pc.sg, pc.a, &o0); if (rc) return rc;
        rc = task_phys_off(c, pc.sg, pc.b, &o1); if (rc) return rc;
        in_bytes += o1 - o0;
    }
    DrainArgs a{};
    a.payload = c->d_payload; a.off = c->d_off; a.hdr = c->d_hdr; a.ids = c->d_ids; a.slot_mask = c->slot_mask;
    a.first_task = head; a.n_tasks = n; a.n_tiles = 0;                     // (set per handler by launch_drain3)
    a.tile_base = (const uint32_t*)c->d_tile_state.v; a.block_base = (const uint32_t*)c->d_tile_state.v + ((size_t)c->max_drain_tasks / D2_THREADS + 2);
    a.count_mode = count_mode;
    a.slow = c->d_slow; a.crc_shift_tabs = c->d_crc_shift;
    a.static_rounds = 0;
    a.retry_mask = endpoint ? 0u : c->retry_mask; a.max_retries = c->max_retries; a.task_of = c->d_task_of;
    c->res.retry = a.retry_mask != 0;
    c->drain_epoch = (c->drain_epoch + 1u) & 0xFFFFFFu;
    if (c->drain_epoch == 0u) {                                             // the 24-bit tag wrapped: forget old tags
        c->drain_epoch = 1u; c->ctl_dirty = true;                           // (and the control ring's order)
        c->last_op_drain = false;
        CU(cudaMemsetAsync(c->d_slow, 0, (size_t)c->max_drain_tasks * sizeof(SlowItem), s));
    }
    a.epoch = c->drain_epoch;
    // the control block: the previous drain kernel zeroed this one (drain_kernel.cuh, D3_CTL_RING), unless something
    // else ran since that the host cannot see through (a failed launch, the wire encoder, the epoch's wrap)
    c->ctl_last = a.epoch % D3_CTL_RING;
    a.out = drain_out(c, c->d_ctl + c->ctl_last, count_mode != 0); a.ctl_next = c->d_ctl + (a.epoch + 1u) % D3_CTL_RING;
    if (c->ctl_dirty) {
        c->last_op_drain = false;
        CU(cudaMemsetAsync(c->d_ctl, 0, D3_CTL_RING * sizeof(DrainCtl), s));
        c->ctl_dirty = false;
    }
    int grid = 0;
    if (!c->burst_open) { c->last_op_drain = false; CU(cudaEventRecord(c->ev_burst, s)); }
    // within a burst nothing is enqueued between one launch's kernel and the next one's: the span's end event is recorded
    // by whatever comes next (end_drain_span), the control block is read back by finish_launch
    const bool overlap = c->last_op_drain;
    c->last_op_drain = false;
    // a launch that failed leaves the control block and the stream's order unknown to the host
    auto launch_failed = [c](const char* what, cudaError_t e) {
        c->last_op_drain = false; c->ctl_dirty = true;
        return fail(B9_EIO, "%s launch failed: %s", what, cudaGetErrorString(e));
    };
    cudaError_t le;
    uint32_t tt = 0;
    if (endpoint || user) {
        // the endpoint drain and a user handler's drains (user_drain.cuh, either rendering) have one shape: 32-slot tiles,
        // one task per lane. Never a programmatic dependent, and the next drain3_kernel is not launched as its dependent
        // either: the timed span ends right behind it (end_drain_span below), which leaves last_op_drain false. The kernel
        // zeroes the next control block itself, as drain3_kernel does (endpoint_drain.cu).
        a.tile_tasks = ENDPOINT_TILE_TASKS;
        a.n_tiles = (n + ENDPOINT_TILE_TASKS - 1) / ENDPOINT_TILE_TASKS;
        tt = ENDPOINT_TILE_TASKS;                                           // (the callback sign pass's record indices)
        le = a.count_mode ? launch_tile_counts(a, ENDPOINT_TILE_TASKS, s) : cudaSuccess;
        if (le == cudaSuccess && !user) le = launch_endpoint_drain(&a, sizeof a, handler, c->sm_count, s);
        else if (le == cudaSuccess) {
            const uint64_t ctas_needed = ((uint64_t)a.n_tiles + USER_DRAIN_WARPS - 1) / USER_DRAIN_WARPS;
            const uint64_t resident = (uint64_t)(endpoint ? user->per_sm_ep : user->per_sm_tq) * (uint64_t)c->sm_count;
            const uint32_t ctas = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(ctas_needed, resident));
            void* args[] = {&a};
            le = cudaLaunchKernel((const void*)(endpoint ? user->ep : user->tq), dim3(ctas), dim3(USER_DRAIN_WARPS * 32), args, 0, s);
        }
        if (le != cudaSuccess) return launch_failed(user ? "user handler drain kernel" : "endpoint drain kernel", le);
        c->last_op_drain = true;
        c->burst_open = true;
        if (!c->res.cb) end_drain_span(c);                                  // (with the runner's callback pass: behind that)
    } else switch (handler) {
    case B9_H_IDENTITY: le = launch_drain3<0>(a, in_bytes / n, win_max_len, c->stage_bytes_override, c->sm_count, overlap, s, &grid, &tt); break;
    case B9_H_CRC32:    le = launch_drain3<1>(a, in_bytes / n, win_max_len, c->stage_bytes_override, c->sm_count, overlap, s, &grid, &tt); break;
    case B9_H_VADD_F32: le = launch_drain3<2>(a, in_bytes / n, win_max_len, c->stage_bytes_override, c->sm_count, overlap, s, &grid, &tt); break;
    default:            le = launch_drain3<3>(a, in_bytes / n, win_max_len, c->stage_bytes_override, c->sm_count, overlap, s, &grid, &tt); break;
    }
    if (!endpoint && !user) {
        if (le != cudaSuccess) return launch_failed("drain kernel", le);
        c->last_op_drain = true;
        c->burst_open = true;
    }
    // the function path beyond identity's one-str template: a pass over the window's pickle tasks that rewrites the records
    // drain3_kernel left UNSUPPORTED. The next drain kernel waits for it in full (no programmatic dependent launch), and
    // the timed span ends behind it.
    const bool pickle_pass = !endpoint && (peek & B9_DRAIN_PICKLE_FULL) && win_pickle;
    // the function runner's callbacks (b9_set_callback_runners): its pass does the pickle pass's work and runs behind the
    // sign pass, whose B9_CB_HOST it overwrites for the pickle slots
    const bool function_runner = pickle_pass && c->res.cb && (c->cb_runners & B9_CB_RUNNER_FUNCTION);
    const CallbackPassArgs cb = {c->cb_mid, c->res.cb_keyed ? 1 : 0, c->res.cb_ts,
                                 {c->d_cb_kind, c->d_cb_digest, c->d_cb_body_off, c->d_cb_body_len, c->d_cb_url_off, c->d_cb_url_len}};
    if (pickle_pass && !function_runner) {
        a.tile_tasks = tt;
        le = launch_function_pass(&a, sizeof a, handler, nullptr, c->sm_count, s);
        if (le != cudaSuccess) return launch_failed("pickle pass", le);
    }
    // under a callback policy: every record's callback kind and signature (drain_passes.cu), behind the records' last
    // writer (drain3_kernel or the pickle pass). Like the pickle pass it is never a programmatic dependent, the next drain
    // kernel waits for it in full, and the timed span ends behind it. It reads this launch's control block and count
    // prefixes, which nothing rewrites before the next launch. The runners' passes follow the same rules.
    if (c->res.cb && endpoint) {
        le = launch_endpoint_callbacks(&a, sizeof a, cb, s);
        if (le != cudaSuccess) return launch_failed("endpoint callback pass", le);
        c->res.cb_requests = true;
    } else if (c->res.cb) {
        a.tile_tasks = tt;
        le = launch_callback_sign(&a, sizeof a, c->cb_mid, cb.keyed, c->res.cb_ts, c->d_cb_kind, c->d_cb_digest, c->sm_count, s);
        if (le != cudaSuccess) return launch_failed("callback sign pass", le);
        if (function_runner) {
            le = launch_function_pass(&a, sizeof a, handler, &cb, c->sm_count, s);
            if (le != cudaSuccess) return launch_failed("function callback pass", le);
            c->res.cb_requests = true;
        }
    }
    if (pickle_pass || c->res.cb) end_drain_span(c);
    {
        std::lock_guard<std::mutex> lk(c->mu);
        c->stats.kernel_launches += (a.count_mode ? 3 : 1) + (pickle_pass ? 1 : 0) + (c->res.cb ? 1 : 0);   // (+ tile_count_kernel and tile_scan_kernel)
        c->stats.last_drain_tiles = (n + 127) / 128;                       // (reported in units of 128 tasks)
        c->stats.drains++;
    }
    c->res.async = true; c->res.async_n = n; c->res.async_in_bytes = in_bytes;
    c->res.ids_in_ring = !a.out.ids_compacted; c->res.head = head;        // (a burst of async launches: the last one's records wait)
    if (!c->res.peek) c->running.store(n, std::memory_order_relaxed);
    if (peek & B9_DRAIN_ASYNC) return (int64_t)n;   // records = n minus the cancelled slots: known after b9_sync / b9_drain_fetch
    int rc = finish_launch(c);
    return rc ? rc : (int64_t)c->res.n;
}

int64_t b9_drain_launch(b9_ctx* c, int handler, uint32_t max_tasks, int peek) {
    if (!c) return fail(B9_EINVAL, "b9_drain_launch: ctx is NULL");
    if (handler < 0 || (handler >= B9_H_COUNT_ && handler < B9_H_USER_BASE)) return fail(B9_ENOSYS, "b9_drain_launch: unknown handler %d", handler);
    return drain_launch_common(c, handler, max_tasks, peek, false);
}

int64_t b9_endpoint_drain_launch(b9_ctx* c, int handler, uint32_t max_tasks, int flags) {
    if (!c) return fail(B9_EINVAL, "b9_endpoint_drain_launch: ctx is NULL");
    if (handler < 0 || (handler >= B9_H_COUNT_ && handler < B9_H_USER_BASE)) return fail(B9_ENOSYS, "b9_endpoint_drain_launch: unknown handler %d", handler);
    if (flags & ~(B9_DRAIN_PEEK | B9_DRAIN_ASYNC)) return fail(B9_EINVAL, "b9_endpoint_drain_launch: unknown flag bits 0x%x", flags);
    return drain_launch_common(c, handler, max_tasks, flags, true);
}

// b9_drain_fetch, and with cb (b9_drain_fetch_callbacks) the launch's callback kinds and digests in the same read-back;
// with rq too (b9_drain_fetch_callback_requests) each record's D and URL
static int64_t drain_fetch(b9_ctx* c, b9_results* out, b9_callbacks* cb, b9_callback_requests* rq = nullptr) {
    std::unique_lock<std::mutex> in_lk(c->in_mu, std::defer_lock);
    std::unique_lock<std::mutex> out_lk(c->out_mu);
    end_drain_span(c);
    CU(cudaSetDevice(c->device));
    { int rc = finish_launch(c); if (rc) return rc; }
    if (!c->res.have) return fail(B9_EINVAL, "b9_drain_fetch: no drain results are waiting");
    if (cb && !c->res.cb) return fail(B9_EINVAL, "b9_drain_fetch_callbacks: the waiting results come from a launch without a callback pass");
    // a runner's pass signed each callback's D, which is not the record: only the fetch that returns D may hand them out
    if (cb && !rq && c->res.cb_requests)
        return fail(B9_EINVAL, "b9_drain_fetch_callbacks: the waiting results come from a launch with a runner's callback pass; "
                               "their signed bodies come with b9_drain_fetch_callback_requests");
    out->n_results = c->res.n; out->n_popped = c->res.popped; out->n_bytes = c->res.bytes; out->need_bytes = c->res.bytes;
    out->task_duration = 0.f;
    if (cb) cb->timestamp = c->res.cb_ts;
    if (c->res.n > out->cap_tasks || c->res.bytes > out->cap_bytes || (cb && c->res.n > cb->cap_tasks) || (rq && c->res.n > rq->cap_tasks))
        return fail(B9_ENOSPC, "b9_drain_fetch: need %u records / %llu bytes, caller gave %u / %llu (callbacks: %u, requests: %u)", c->res.n,
                    (unsigned long long)c->res.bytes, out->cap_tasks, (unsigned long long)out->cap_bytes, cb ? cb->cap_tasks : 0u,
                    rq ? rq->cap_tasks : 0u);
    cudaStream_t s = c->stream;
    const size_t n = c->res.n;
    CU(cudaEventRecord(c->ev_c, s));
    if (n) {
        if (!out->task_ids || !out->status || !out->has_result || !out->offsets || !out->lengths) return fail(B9_EINVAL, "b9_drain_fetch: NULL result array");
        CU(cudaMemcpyAsync(out->lengths, c->d_out_len, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        if (c->res.ids_in_ring) CU(copy_slot_ids(c, c->res.head, n, out->task_ids, false, cudaMemcpyDeviceToHost, s));   // (the window's slots)
        else CU(cudaMemcpyAsync(out->task_ids, c->d_out_ids, n * 16, cudaMemcpyDeviceToHost, s));
        CU(cudaMemcpyAsync(out->status, c->d_out_status, n, cudaMemcpyDeviceToHost, s));
        CU(cudaMemcpyAsync(out->has_result, c->d_out_has, n, cudaMemcpyDeviceToHost, s));
        CU(cudaMemcpyAsync(out->offsets, c->d_out_off, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
        if (c->res.bytes) {
            if (!out->payload) return fail(B9_EINVAL, "b9_drain_fetch: NULL payload buffer");
            CU(cudaMemcpyAsync(out->payload, c->d_out_payload, c->res.bytes, cudaMemcpyDeviceToHost, s));
        }
        if (cb) {
            if (!cb->kind || !cb->digest) return fail(B9_EINVAL, "b9_drain_fetch_callbacks: NULL callback array");
            CU(cudaMemcpyAsync(cb->kind, c->d_cb_kind, n, cudaMemcpyDeviceToHost, s));
            if (c->res.cb_keyed) CU(cudaMemcpyAsync(cb->digest, c->d_cb_digest, n * 32, cudaMemcpyDeviceToHost, s));
            else memset(cb->digest, 0, n * 32);                          // (without a key no digest is written)
        }
        if (rq) {
            if (!rq->body_offsets || !rq->body_lengths || !rq->url_offsets || !rq->url_lengths) return fail(B9_EINVAL, "b9_drain_fetch_callback_requests: NULL request array");
            if (c->res.cb_requests) {
                CU(cudaMemcpyAsync(rq->body_offsets, c->d_cb_body_off, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
                CU(cudaMemcpyAsync(rq->body_lengths, c->d_cb_body_len, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
                CU(cudaMemcpyAsync(rq->url_offsets, c->d_cb_url_off, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
                CU(cudaMemcpyAsync(rq->url_lengths, c->d_cb_url_len, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
            }
        }
    }
    CU(cudaEventRecord(c->ev_d, s));
    CU(cudaStreamSynchronize(s));
    // a launch without a runner's pass (task-queue records only): every record's D is its own R, or {} without result bytes
    if (rq && n && !c->res.cb_requests)
        for (size_t j = 0; j < n; ++j) {
            rq->body_offsets[j] = out->offsets[j]; rq->body_lengths[j] = out->has_result[j] ? out->lengths[j] : 0u;
            rq->url_offsets[j] = 0; rq->url_lengths[j] = 0;
        }
    float ms = 0; cudaEventElapsedTime(&ms, c->ev_c, c->ev_d);
    // the window's RETRY records (only a drain under a retry policy writes them), in record order: pushed again below
    std::vector<uint32_t> retry_rec;
    if (!c->res.peek && c->res.retry)
        for (size_t j = 0; j < n; ++j) if (out->status[j] == B9_ST_RETRY) retry_rec.push_back((uint32_t)j);
    // TaskQueueCompleteRequest.task_duration (taskqueue.proto:50): the runner reports the seconds it spent on a task; a
    // drain spends kernel + read-back time on res.popped tasks at once, so every task of the batch is charged its share
    if (c->res.popped) out->task_duration = (c->res.kernel_ms + ms) * 1e-3f / (float)c->res.popped;
    // the records, and with cb the kinds and (under a key) the digests
    const uint64_t d2h_bytes = c->res.bytes + n * (16 + 1 + 1 + 8 + 4) + (cb ? n * (1 + (c->res.cb_keyed ? 32 : 0)) : 0) +
                               (rq && c->res.cb_requests ? n * (8 + 4 + 8 + 4) : 0);
    if (!retry_rec.empty()) {
        // the re-push is a push: it takes the producers' lock, so that concurrent pushes land wholly before or after it. The
        // lock order is in_mu before out_mu: when a producer holds in_mu, out_mu is let go while the fetch waits for it, and
        // the commit goes ahead only if no other drain-side call has touched these results meanwhile
        if (!in_lk.try_lock()) {
            const uint64_t gen = c->res_gen;
            out_lk.unlock();
            in_lk.lock();
            out_lk.lock();
            end_drain_span(c);
            if (c->res_gen != gen || !c->res.have)
                return fail(B9_EINVAL, "b9_drain_fetch: another drain-side call replaced or committed these results meanwhile");
        }
        const int rc = commit_with_repush(c, retry_rec, ms, d2h_bytes);
        if (rc) return rc;
    } else {
        std::lock_guard<std::mutex> lk(c->mu);
        c->stats.last_drain_d2h_ms = ms;
        c->stats.bytes_d2h += d2h_bytes;
        if (!c->res.peek) commit_pop(c);
    }
    if (!c->res.peek && c->recount_cancelled) { int rc = recount_cancelled_locked_out(c); if (rc) return rc; }
    c->res = WaitingResults{};
    c->running.store(0, std::memory_order_relaxed);
    c->burst_open = false; c->res_gen++;
    return (int64_t)n;
}

int64_t b9_drain_fetch(b9_ctx* c, b9_results* out) {
    if (!c || !out) return fail(B9_EINVAL, "b9_drain_fetch: NULL argument");
    return drain_fetch(c, out, nullptr);
}

int64_t b9_drain_fetch_callbacks(b9_ctx* c, b9_results* out, b9_callbacks* cb) {
    if (!c || !out || !cb) return fail(B9_EINVAL, "b9_drain_fetch_callbacks: NULL argument");
    return drain_fetch(c, out, cb);
}

int64_t b9_drain_fetch_callback_requests(b9_ctx* c, b9_results* out, b9_callbacks* cb, b9_callback_requests* rq) {
    if (!c || !out || !cb || !rq) return fail(B9_EINVAL, "b9_drain_fetch_callback_requests: NULL argument");
    return drain_fetch(c, out, cb, rq);
}

int64_t b9_drain(b9_ctx* c, int handler, uint32_t max_tasks, b9_results* out) {
    if (!c || !out) return fail(B9_EINVAL, "b9_drain: NULL argument");
    if (out->cap_tasks < max_tasks) max_tasks = out->cap_tasks;
    int64_t r = b9_drain_launch(c, handler, max_tasks, /*peek=*/0);
    if (r < 0) return r;
    return b9_drain_fetch(c, out);   // on B9_ENOSPC nothing is consumed and the records stay fetchable
}

// =========================================================================== wire records
static size_t host_go_quote(const char* s, uint8_t* o, size_t cap) {
    // encode.go appendString for an (assumed valid UTF-8) host string; HTML-safe
    size_t n = 0;
    auto put = [&](uint8_t c) { if (n < cap) o[n] = c; ++n; };
    static const char HX[] = "0123456789abcdef";
    put('"');
    for (const unsigned char* p = (const unsigned char*)s; *p; ++p) {
        unsigned char c = *p;
        switch (c) {
        case '"': put('\\'); put('"'); break;
        case '\\': put('\\'); put('\\'); break;
        case '\b': put('\\'); put('b'); break;
        case '\f': put('\\'); put('f'); break;
        case '\n': put('\\'); put('n'); break;
        case '\r': put('\\'); put('r'); break;
        case '\t': put('\\'); put('t'); break;
        default:
            if (c < 0x20 || c == '<' || c == '>' || c == '&') { put('\\'); put('u'); put('0'); put('0'); put(HX[c >> 4]); put(HX[c & 15]); }
            else if (c == 0xE2 && p[1] == 0x80 && (p[2] == 0xA8 || p[2] == 0xA9)) { put('\\'); put('u'); put('2'); put('0'); put('2'); put(p[2] == 0xA8 ? '8' : '9'); p += 2; }
            else put(c);
        }
    }
    put('"');
    return n;
}

// b9_wire_encode (full = false) and b9_wire_encode_full: the same call around wire_encode_kernel<full>
static int64_t wire_encode(b9_ctx* c, const b9_wire_env* env, uint32_t max_tasks, bool full) {
    const char* const fn = full ? "b9_wire_encode_full" : "b9_wire_encode";
    if (!c || !env || !env->workspace_name || !env->stub_id) return fail(B9_EINVAL, "%s: NULL argument", fn);
    OutLock out_lk(c);
    CU(cudaSetDevice(c->device));
    c->res = WaitingResults{};
    c->running.store(0, std::memory_order_relaxed);
    c->burst_open = false; c->res_gen++;
    c->res.peek = true;
    uint64_t head = 0; uint32_t n = 0;
    cudaStream_t s = c->stream;
    {
        std::lock_guard<std::mutex> lk(c->mu);
        head = c->head_task;
        const uint64_t depth = c->tail_task - c->head_task;
        n = (uint32_t)std::min<uint64_t>(std::min<uint64_t>(depth, max_tasks), c->max_drain_tasks);
        if (const int rc = wait_pending(c, s)) return rc;
    }
    if (n == 0) { c->res.have = true; return 0; }
    WireEnv we; memset(&we, 0, sizeof we);
    {
        uint8_t* o = we.mid; size_t k = 0; const size_t cap = sizeof we.mid;
        auto lit = [&](const char* t) { for (; *t; ++t) { if (k < cap) o[k] = (uint8_t)*t; ++k; } };
        lit("\",\"workspace_name\":"); k += host_go_quote(env->workspace_name, o + std::min(k, cap), cap - std::min(k, cap));
        lit(",\"stub_id\":");          k += host_go_quote(env->stub_id, o + std::min(k, cap), cap - std::min(k, cap));
        lit(",\"executor\":");         k += host_go_quote(env->executor ? env->executor : "taskqueue", o + std::min(k, cap), cap - std::min(k, cap));
        lit(",\"args\":");
        if (k > cap) return fail(B9_E2BIG, "%s: workspace/stub names too long", fn);
        we.mid_len = (uint32_t)k;
    }
    we.max_retries = env->max_retries; we.timeout = env->timeout; we.ttl = env->ttl;
    CU(cudaMemcpyAsync(c->d_wire_env, &we, sizeof we, cudaMemcpyHostToDevice, s));
    CU(cudaMemsetAsync(c->d_ctl, 0, sizeof(DrainCtl), s));                  // (the control ring's first entry: the next drain zeroes the ring)
    c->ctl_dirty = true;
    WireArgs a{};
    a.payload = c->d_payload; a.off = c->d_off; a.hdr = c->d_hdr; a.ids = c->d_ids; a.ts = c->d_ts; a.exp = c->d_exp;
    a.slot_mask = c->slot_mask; a.first_task = head; a.n_tasks = n;
    a.out = drain_out(c, c->d_ctl, false);                                  // (a record for every task of the window)
    c->res.ids_in_ring = !a.out.ids_compacted; c->res.head = head;
    CU(cudaEventRecord(c->ev_a, s));
    if (full) CU(launch_wire_encode_full(&a, sizeof a, c->d_wire_env, (n + 127) / 128, s));
    else wire_encode_kernel<false><<<(n + 127) / 128, 128, 0, s>>>(a, c->d_wire_env);
    CU(cudaGetLastError());
    CU(cudaEventRecord(c->ev_b, s));
    CU(cudaMemcpyAsync(c->h_ctl, c->d_ctl, sizeof(DrainCtl), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));     // (the stack copy of `we` is consumed by now as well)
    if (c->h_ctl->overflow) return fail(B9_ENOSPC, "%s: records exceed max_result_bytes (%llu)", fn, (unsigned long long)c->max_result_bytes);
    c->res.bytes = c->h_ctl->bytes; c->res.n = n; c->res.popped = 0; c->res.have = true;
    float ms = 0; cudaEventElapsedTime(&ms, c->ev_a, c->ev_b); c->res.kernel_ms = ms;
    std::lock_guard<std::mutex> lk(c->mu);
    c->stats.kernel_launches++;
    c->stats.last_drain_out_bytes = c->res.bytes;
    c->stats.last_drain_kernel_ms = ms;
    return (int64_t)n;
}

int64_t b9_wire_encode(b9_ctx* c, const b9_wire_env* env, uint32_t max_tasks) { return wire_encode(c, env, max_tasks, false); }
int64_t b9_wire_encode_full(b9_ctx* c, const b9_wire_env* env, uint32_t max_tasks) { return wire_encode(c, env, max_tasks, true); }

// =========================================================================== multi-GPU: NCCL rebalance
}  // extern "C" (reopened below)

namespace {

struct NcclApi {
    void* lib = nullptr;
    int (*GetUniqueId)(void*) = nullptr;
    int (*CommInitRank)(void**, int, /*ncclUniqueId by value*/ struct B9NcclId, int) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
    int (*Send)(const void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    int (*Recv)(void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};
struct B9NcclId { char internal[128]; };
constexpr int NCCL_U8 = 1, NCCL_U64 = 5;        // ncclUint8, ncclUint64 (nccl.h ncclDataType_t)

NcclApi g_nccl;
std::mutex g_nccl_mu;

int load_nccl() {
    std::lock_guard<std::mutex> lk(g_nccl_mu);
    if (g_nccl.lib) return B9_OK;
    const char* path = getenv("B9_NCCL_LIB");
    void* h = dlopen(path ? path : "libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h && !path) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return fail(B9_EIO, "cannot load NCCL (%s); set B9_NCCL_LIB", dlerror());
#define SYM(field, name) *(void**)(&g_nccl.field) = dlsym(h, name); if (!g_nccl.field) return fail(B9_EIO, "NCCL symbol %s missing", name)
    SYM(GetUniqueId, "ncclGetUniqueId"); SYM(CommInitRank, "ncclCommInitRank"); SYM(CommDestroy, "ncclCommDestroy");
    SYM(AllGather, "ncclAllGather"); SYM(Send, "ncclSend"); SYM(Recv, "ncclRecv");
    SYM(GroupStart, "ncclGroupStart"); SYM(GroupEnd, "ncclGroupEnd"); SYM(GetErrorString, "ncclGetErrorString");
#undef SYM
    g_nccl.lib = h;
    return B9_OK;
}
void nccl_comm_destroy(void* comm) { if (comm && g_nccl.CommDestroy) g_nccl.CommDestroy(comm); }
#define NC(call) do { int r_ = (call); if (r_ != 0) return fail(B9_EIO, "%s failed: %s", #call, g_nccl.GetErrorString(r_)); } while (0)

// ---- rebalance, device side ---------------------------------------------------------------------------------------
// byte prefix of the pending tasks (prefix[0] = 0, prefix[i + 1] = bytes of tasks 0..i), from the slot ring's length words:
// three small kernels (block sums, scan of the block sums, write-out) — only the W cut points ever cross PCIe
constexpr uint32_t SCAN_BLOCK = 1024;        // tasks per block (256 threads x 4)
__global__ void __launch_bounds__(256) scan_block_sums_kernel(const uint64_t* __restrict__ hdr, uint32_t slot_mask, uint64_t first_task, uint32_t n,
                                                             unsigned long long* __restrict__ block_sum) {
    __shared__ unsigned long long s_w[8];
    const uint32_t base = blockIdx.x * SCAN_BLOCK + threadIdx.x * 4u;
    unsigned long long v = 0;
    #pragma unroll
    for (uint32_t k = 0; k < 4; ++k) if (base + k < n) v += hdr_len(hdr[(uint32_t)((first_task + base + k) & slot_mask)]);
    #pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    if ((threadIdx.x & 31u) == 0u) s_w[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) { unsigned long long t = 0; for (int w = 0; w < 8; ++w) t += s_w[w]; block_sum[blockIdx.x] = t; }
}
__global__ void __launch_bounds__(1024) scan_of_sums_kernel(unsigned long long* __restrict__ block_sum, uint32_t blocks) {   // in place, exclusive
    __shared__ unsigned long long s_w[32];
    const uint32_t per = (blocks + 1023u) / 1024u, lo = min(blocks, threadIdx.x * per), hi = min(blocks, lo + per);
    unsigned long long sum = 0;
    for (uint32_t i = lo; i < hi; ++i) sum += block_sum[i];
    unsigned long long inc = sum;
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    #pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const unsigned long long t = __shfl_up_sync(0xffffffffu, inc, d); if ((int)lane >= d) inc += t; }
    if (lane == 31) s_w[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        unsigned long long x = s_w[lane], y = x;
        #pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const unsigned long long t = __shfl_up_sync(0xffffffffu, y, d); if ((int)lane >= d) y += t; }
        s_w[lane] = y - x;
    }
    __syncthreads();
    unsigned long long run = s_w[warp] + inc - sum;
    for (uint32_t i = lo; i < hi; ++i) { const unsigned long long t = block_sum[i]; block_sum[i] = run; run += t; }
}
__global__ void __launch_bounds__(256) scan_write_kernel(const uint64_t* __restrict__ hdr, uint32_t slot_mask, uint64_t first_task, uint32_t n,
                                                        const unsigned long long* __restrict__ block_base, uint64_t* __restrict__ prefix) {
    __shared__ unsigned long long s_w[8];
    const uint32_t base = blockIdx.x * SCAN_BLOCK + threadIdx.x * 4u;
    unsigned long long l[4]; unsigned long long v = 0;
    #pragma unroll
    for (uint32_t k = 0; k < 4; ++k) { l[k] = (base + k < n) ? hdr_len(hdr[(uint32_t)((first_task + base + k) & slot_mask)]) : 0ull; v += l[k]; }
    unsigned long long inc = v;
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    #pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const unsigned long long t = __shfl_up_sync(0xffffffffu, inc, d); if ((int)lane >= d) inc += t; }
    if (lane == 31) s_w[warp] = inc;
    __syncthreads();
    unsigned long long before = block_base[blockIdx.x];
    for (uint32_t w = 0; w < warp; ++w) before += s_w[w];
    unsigned long long run = before + inc - v;
    if (blockIdx.x == 0 && threadIdx.x == 0) prefix[0] = 0;
    #pragma unroll
    for (uint32_t k = 0; k < 4; ++k) { run += l[k]; if (base + k < n) prefix[base + k + 1] = run; }
}

// What one rank learns in the planning phase, written by the cut kernel and read back in ONE copy.
struct RebalanceCuts {
    uint64_t lo[16], hi[16];             // my FIFO range for every destination rank
    uint64_t bytes[16];                  // payload bytes of that range
    uint64_t phys[16];                   // physical ring offset of its first task
    uint64_t contiguous[16];             // 1: the range is one contiguous byte range of the ring (send it from there)
    uint64_t keep_end_phys;              // physical offset of the first task that leaves to a HIGHER rank (= end of what I keep)
    uint64_t ok;                         // the plan succeeded
};
constexpr int REBALANCE_MAX_WORLD = 16;

// ONE thread: the same plan function the host exports (rebalance_plan.h) over the device-resident prefix, plus the physical
// facts the host needs to post the sends. tab = all-gathered (count, bytes, cancelled, 0) per rank; row_out = my row of the
// send matrix (tasks, bytes per destination), all-gathered next.
__global__ void rebalance_cut_kernel(const uint64_t* __restrict__ tab, uint32_t world, uint32_t rank, const uint64_t* __restrict__ prefix, uint64_t n,
                                     const uint64_t* __restrict__ off, const uint64_t* __restrict__ hdr, uint32_t slot_mask, uint64_t first_task,
                                     RebalanceCuts* __restrict__ cuts, uint64_t* __restrict__ row_out) {
    if (blockIdx.x || threadIdx.x) return;
    uint64_t counts[REBALANCE_MAX_WORLD], bytes[REBALANCE_MAX_WORLD];
    for (uint32_t r = 0; r < world; ++r) { counts[r] = tab[4 * r]; bytes[r] = tab[4 * r + 1]; }
    RebalanceCuts c;
    c.ok = b9_plan_ranges(world, rank, counts, bytes, prefix, n, c.lo, c.hi) == 0 ? 1ull : 0ull;
    for (uint32_t d = 0; d < world; ++d) {
        if (!c.ok) { c.lo[d] = c.hi[d] = 0; }
        const uint64_t lo = c.lo[d], hi = c.hi[d];
        c.bytes[d] = prefix[hi] - prefix[lo];
        c.phys[d] = 0; c.contiguous[d] = 1;
        if (hi > lo) {
            const uint32_t s0 = (uint32_t)((first_task + lo) & slot_mask), s1 = (uint32_t)((first_task + hi - 1) & slot_mask);
            c.phys[d] = off[s0];
            c.contiguous[d] = (off[s1] + hdr_len(hdr[s1]) - off[s0] == c.bytes[d] && off[s1] >= off[s0]) ? 1ull : 0ull;
        }
        row_out[2 * d] = hi - lo; row_out[2 * d + 1] = c.bytes[d];
    }
    const uint64_t keep_hi = c.hi[rank];
    c.keep_end_phys = keep_hi < n ? off[(uint32_t)((first_task + keep_hi) & slot_mask)] : 0;
    *cuts = c;
}

// slot words of the tasks that leave (ids, lengths as relative offsets, flags, retries, timestamps, expiries) into one
// meta message; with `out_payload` also their bytes (only for ranges that are not contiguous in the ring)
__global__ void gather_tasks_kernel(const uint8_t* __restrict__ payload, const uint64_t* __restrict__ off, const uint64_t* __restrict__ hdr,
                                    const uint4* __restrict__ ids, const int64_t* __restrict__ ts, const int64_t* __restrict__ exp,
                                    uint32_t slot_mask, uint64_t first_task, uint32_t n, const uint64_t* __restrict__ prefix /* device prefix, at the range's first task */,
                                    uint8_t* __restrict__ out_payload, uint64_t* __restrict__ o_rel, int64_t* __restrict__ o_ts, int64_t* __restrict__ o_exp,
                                    uint4* __restrict__ o_ids, uint8_t* __restrict__ o_flags, uint8_t* __restrict__ o_retries) {
    if (out_payload) {                                   // one warp per task
        const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
        if (w >= n) return;
        const uint32_t slot = (uint32_t)((first_task + w) & slot_mask);
        const uint64_t h = hdr[slot];
        const uint32_t len = hdr_len(h);
        const uint8_t* src = payload + off[slot];
        uint8_t* dst = out_payload + (prefix[w] - prefix[0]);
        for (uint32_t i = lane; i < len; i += 32) dst[i] = src[i];
        if (lane == 0) { o_rel[w] = prefix[w]; if (w + 1 == n) o_rel[n] = prefix[n]; o_ts[w] = ts[slot]; o_exp[w] = exp[slot]; o_ids[w] = ids[slot]; o_flags[w] = (uint8_t)hdr_flags(h); o_retries[w] = (uint8_t)(h >> 40); }
    } else {                                             // slot words only: one thread per task
        const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
        if (w >= n) return;
        const uint32_t slot = (uint32_t)((first_task + w) & slot_mask);
        const uint64_t h = hdr[slot];
        o_rel[w] = prefix[w]; if (w + 1 == n) o_rel[n] = prefix[n];
        o_ts[w] = ts[slot]; o_exp[w] = exp[slot]; o_ids[w] = ids[slot]; o_flags[w] = (uint8_t)hdr_flags(h); o_retries[w] = (uint8_t)(h >> 40);
    }
}

// layout of one peer's meta message for n tasks (every section 16-byte aligned)
struct MetaLayout { size_t rel, ts, exp, ids, flags, retries, total; };
MetaLayout meta_layout(uint64_t n) {
    auto al = [](size_t v) { return (v + 15) & ~(size_t)15; };
    MetaLayout m; size_t o = 0;
    m.rel = o; o = al(o + (n + 1) * 8);
    m.ts = o; o = al(o + n * 8);
    m.exp = o; o = al(o + n * 8);
    m.ids = o; o = al(o + n * 16);
    m.flags = o; o = al(o + n);
    m.retries = o; o = al(o + n);
    m.total = o; return m;
}

// drop k tasks from the tail of the ring (they were handed to another rank); cut_phys = physical offset of the first dropped
// task. Caller holds c->mu.
void drop_back(b9_ctx* c, uint64_t k, uint64_t cut_phys) {
    while (k && !c->segs.empty()) {
        Segment& sg = c->segs.back();
        if (sg.n <= k) {
            k -= sg.n; c->tail_task -= sg.n; c->pending_bytes -= sg.bytes; c->write_pos = sg.phys_start;
            put_event(c, sg.ready); c->segs.pop_back();
        } else {
            const uint32_t keep = sg.n - (uint32_t)k;
            const uint64_t nb = cut_phys - sg.phys_start;               // (the cut lies inside this segment)
            c->pending_bytes -= sg.bytes - nb; c->tail_task -= k;
            sg.n = keep; sg.bytes = nb;
            c->write_pos = sg.phys_start + b9_seg_span(nb);
            k = 0;
        }
    }
    if (c->segs.empty()) c->write_pos = 0;
}

}  // namespace

extern "C" {

int b9_rebalance_plan(uint32_t world, uint32_t rank, const uint64_t* counts, const uint64_t* bytes, const uint64_t* prefix, uint64_t n,
                      uint64_t* send_lo, uint64_t* send_hi) {
    if (!counts || !bytes || !prefix || !send_lo || !send_hi) return fail(B9_EINVAL, "b9_rebalance_plan: NULL argument");
    if (b9_plan_ranges(world, rank, counts, bytes, prefix, n, send_lo, send_hi)) return fail(B9_EINVAL, "b9_rebalance_plan: table inconsistent with prefix");
    return B9_OK;
}

int b9_comm_unique_id(uint8_t* out128) {
    if (!out128) return fail(B9_EINVAL, "b9_comm_unique_id: NULL");
    int rc = load_nccl(); if (rc) return rc;
    B9NcclId id; memset(&id, 0, sizeof id);
    NC(g_nccl.GetUniqueId(&id));
    memcpy(out128, id.internal, 128);
    return B9_OK;
}

int b9_comm_init(b9_ctx* c, const uint8_t* id128, int rank, int world) {
    if (!c || !id128 || world < 1 || rank < 0 || rank >= world) return fail(B9_EINVAL, "b9_comm_init: bad argument");
    if (world > REBALANCE_MAX_WORLD) return fail(B9_EINVAL, "b9_comm_init: world %d > %d", world, REBALANCE_MAX_WORLD);
    int rc = load_nccl(); if (rc) return rc;
    std::lock_guard<std::mutex> in_lk(c->in_mu);
    OutLock out_lk(c);
    CU(cudaSetDevice(c->device));
    B9NcclId id; memcpy(id.internal, id128, 128);
    if (c->nccl_comm) { nccl_comm_destroy(c->nccl_comm); c->nccl_comm = nullptr; }   // re-init: the old communicator is not leaked
    void* comm = nullptr;
    NC(g_nccl.CommInitRank(&comm, world, id, rank));
    c->nccl_comm = comm; c->comm_rank = rank; c->comm_world = world;
    if (world > 1) {
        // everything the planning phase of b9_rebalance touches is allocated here, once: the byte prefix of a full slot ring,
        // the block sums of its scan, the all-gather tables and the page-locked block the cut points come back in
        if (!c->d_prefix) {
            CU(cudaMalloc(&c->d_prefix.v, ((size_t)c->ring_tasks + 2) * sizeof(uint64_t)));
            CU(cudaMalloc(&c->d_scan_sums.v, ((size_t)c->ring_tasks / SCAN_BLOCK + 2) * sizeof(unsigned long long)));
        }
        if (!c->d_rtab) {
            c->rtab_words = 4 * (size_t)REBALANCE_MAX_WORLD * 2 + 2 * (size_t)REBALANCE_MAX_WORLD * (REBALANCE_MAX_WORLD + 1) + (size_t)REBALANCE_MAX_WORLD + sizeof(RebalanceCuts) / 8 + 16;
            CU(cudaMalloc(&c->d_rtab.v, c->rtab_words * sizeof(uint64_t)));
            CU(cudaHostAlloc(&c->h_rtab.v, c->rtab_words * sizeof(uint64_t), cudaHostAllocDefault));
        }
        // ... and a first size for the two arenas the slot words (and non-contiguous payload ranges) are staged in (a failure
        // here is not an error: b9_rebalance grows them to what it needs)
        const uint64_t first = std::max<uint64_t>((uint64_t)c->ring_tasks * 48 / 2, 16ull << 20);
        (void)c->d_xchg_send.grow(first);
        (void)c->d_xchg_recv.grow(first);
    }
    // NCCL sets its point-to-point channels up lazily, on the first send/recv of every pair and of every
    // channel a message is spread over (seconds on an 8-GPU box): do that here, once, with an all-to-all
    // large enough to touch all of them (B9_COMM_WARMUP_BYTES per peer, default 4 MiB), plus the
    // all-gather b9_rebalance opens with, so that the first real exchange finds everything connected
    if (world > 1) {
        size_t per = 4u << 20;
        if (const char* e = getenv("B9_COMM_WARMUP_BYTES")) per = (size_t)std::max<long long>(16, atoll(e));
        DevPtr<uint8_t> d;
        CU(cudaMalloc(&d.v, (size_t)world * per * 2));
        CU(cudaMemsetAsync(d, 0, (size_t)world * per * 2, c->stream));
        NC(g_nccl.AllGather(d, d + per, 16, NCCL_U64, comm, c->stream));      // (world * 128 bytes <= per)
        NC(g_nccl.GroupStart());
        for (int p = 0; p < world; ++p) {
            if (p == rank) continue;
            NC(g_nccl.Send(d + (size_t)p * per * 2, per, NCCL_U8, p, comm, c->stream));
            NC(g_nccl.Recv(d + (size_t)p * per * 2 + per, per, NCCL_U8, p, comm, c->stream));
        }
        NC(g_nccl.GroupEnd());
        CU(cudaStreamSynchronize(c->stream));
    }
    return B9_OK;
}

// Collective: every rank of the communicator must call it. Moves pending tasks between the ranks' rings so that every
// rank holds ~1/W of the pending payload BYTES (SURVEY.md §8e). Nothing per-task crosses PCIe:
//   1. device: byte prefix of my pending tasks from the slot ring's length words (three small scan kernels);
//   2. all-gather of (count, bytes, cancelled) per rank — on the device;
//   3. device: ONE thread runs the byte-quantile plan (rebalance_plan.h, the function the CPU tests run) against the
//      prefix and writes my cut points, the physical ring offsets at the cuts and my row of the send matrix;
//   4. all-gather of the matrix rows; ONE copy brings table + cuts + matrix to the host (first synchronise);
//   5. every rank decides whether what arrives fits its ring — slot count AND contiguous byte placement, with what leaves
//      still in place — and the ranks vote (all-gather of one flag, second synchronise): if any rank cannot take its
//      share, ALL return B9_ENOSPC with their rings untouched;
//   6. the exchange, one grouped ncclSend/ncclRecv: payload ranges that are contiguous in the ring (a batch pushed in one
//      piece is) leave straight from the ring, arriving payload lands straight in the ring space placed in 5; only the
//      slot words (41 B per task) are staged through the two arenas;
//   7. bookkeeping: what left is dropped from both ends, what arrived is appended source by source (ingest_kernel).
int b9_rebalance(b9_ctx* c, b9_rebalance_info* info) {
    if (!c) return fail(B9_EINVAL, "b9_rebalance: ctx is NULL");
    if (!c->nccl_comm) return fail(B9_EINVAL, "b9_rebalance: b9_comm_init was not called");
    std::lock_guard<std::mutex> in_lk(c->in_mu);       // the exchange rewrites both ends of the ring: no push, no drain meanwhile
    OutLock out_lk(c);
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    const int W = c->comm_world, R = c->comm_rank;
    cudaStream_t s = c->stream;
    static const bool trace = getenv("B9_REBALANCE_TRACE") != nullptr;       // phase wall times on stderr
    auto t_last = std::chrono::steady_clock::now();
    auto phase = [&](const char* what) {
        if (!trace) return;
        cudaStreamSynchronize(s);
        const auto now = std::chrono::steady_clock::now();
        fprintf(stderr, "[b9_rebalance rank %d] %-28s %8.3f ms\n", R, what, std::chrono::duration<double, std::milli>(now - t_last).count());
        t_last = now;
    };
    if (W == 1) {
        if (info) { memset(info, 0, sizeof *info); info->world = 1; info->tasks_before = info->tasks_after = c->tail_task - c->head_task; info->bytes_before = info->bytes_after = c->pending_bytes; }
        return B9_OK;
    }
    if (const int rc = wait_pending(c, s)) return rc;
    c->res = WaitingResults{};
    c->running.store(0, std::memory_order_relaxed);
    c->burst_open = false;
    free_segments(c);
    const uint64_t n = c->tail_task - c->head_task;
    const uint64_t my_bytes = c->pending_bytes;
    // ---- layout of the device / pinned table (64-bit words)
    uint64_t* const d_me = c->d_rtab;                                   // [4] count, bytes, cancelled, 0
    uint64_t* const d_tab = d_me + 4;                                   // [4 W] all-gathered
    uint64_t* const d_row = d_tab + 4 * REBALANCE_MAX_WORLD;            // [2 W] my matrix row
    uint64_t* const d_mat = d_row + 2 * REBALANCE_MAX_WORLD;            // [2 W W]
    uint64_t* const d_vote = d_mat + 2 * REBALANCE_MAX_WORLD * REBALANCE_MAX_WORLD;   // [1 + W]
    RebalanceCuts* const d_cuts = (RebalanceCuts*)(d_vote + 1 + REBALANCE_MAX_WORLD);
    uint64_t* const h = c->h_rtab;
    const size_t off_tab = 4, off_row = off_tab + 4 * REBALANCE_MAX_WORLD, off_mat = off_row + 2 * REBALANCE_MAX_WORLD,
                 off_vote = off_mat + 2 * REBALANCE_MAX_WORLD * REBALANCE_MAX_WORLD, off_cuts = off_vote + 1 + REBALANCE_MAX_WORLD;
    // ---- 1. byte prefix on the device
    const uint32_t blocks = (uint32_t)((n + SCAN_BLOCK - 1) / SCAN_BLOCK);
    if (n) {
        scan_block_sums_kernel<<<blocks, 256, 0, s>>>(c->d_hdr, c->slot_mask, c->head_task, (uint32_t)n, c->d_scan_sums);
        scan_of_sums_kernel<<<1, 1024, 0, s>>>(c->d_scan_sums, blocks);
        scan_write_kernel<<<blocks, 256, 0, s>>>(c->d_hdr, c->slot_mask, c->head_task, (uint32_t)n, c->d_scan_sums, c->d_prefix);
        CU(cudaGetLastError());
        c->stats.kernel_launches += 3;
    } else CU(cudaMemsetAsync(c->d_prefix, 0, sizeof(uint64_t), s));
    // ---- 2. all-gather (count, bytes, cancelled)
    h[0] = n; h[1] = my_bytes; h[2] = c->cancelled_pending; h[3] = 0;
    CU(cudaMemcpyAsync(d_me, h, 4 * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
    NC(g_nccl.AllGather(d_me, d_tab, 4, NCCL_U64, c->nccl_comm, s));
    // ---- 3. cuts, 4. matrix
    rebalance_cut_kernel<<<1, 32, 0, s>>>(d_tab, (uint32_t)W, (uint32_t)R, c->d_prefix, n, c->d_off, c->d_hdr, c->slot_mask, c->head_task, d_cuts, d_row);
    CU(cudaGetLastError());
    c->stats.kernel_launches++;
    NC(g_nccl.AllGather(d_row, d_mat, (size_t)2 * W, NCCL_U64, c->nccl_comm, s));
    CU(cudaMemcpyAsync(h + off_tab, d_tab, (c->rtab_words - off_tab) * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    phase("prefix + plan + matrix");
    const RebalanceCuts& cuts = *(const RebalanceCuts*)(h + off_cuts);
    const uint64_t* tab = h + off_tab;
    const uint64_t* mat = h + off_mat;
    auto M_tasks = [&](int src, int dst) { return mat[((size_t)src * W + dst) * 2]; };
    auto M_bytes = [&](int src, int dst) { return mat[((size_t)src * W + dst) * 2 + 1]; };
    if (!cuts.ok) return fail(B9_EIO, "b9_rebalance: ring bookkeeping inconsistent with the slot ring (%llu tasks, %llu bytes)", (unsigned long long)n, (unsigned long long)my_bytes);
    bool any_cancelled = false;
    for (int r = 0; r < W; ++r) any_cancelled |= tab[4 * r + 2] != 0;
    // ---- 5. does what arrives fit? (placement with everything that leaves still in place: a receive never lands on bytes a send reads)
    uint64_t sent_tasks = 0, sent_bytes = 0, recv_tasks = 0, recv_bytes = 0;
    for (int d = 0; d < W; ++d) if (d != R) { sent_tasks += cuts.hi[d] - cuts.lo[d]; sent_bytes += cuts.bytes[d]; recv_tasks += M_tasks(d, R); recv_bytes += M_bytes(d, R); }
    std::vector<uint64_t> r_start(W, 0);
    bool fits = n - sent_tasks + recv_tasks <= c->ring_tasks;
    {
        // a dry run of the appends on a copy of the placement state
        uint64_t wp = c->write_pos, live = 0; bool have = !c->segs.empty();
        const uint64_t oldest = have ? c->segs.front().phys_start : 0;
        for (const Segment& sg : c->segs) live += sg.bytes;
        for (int src = 0; src < W && fits; ++src) {
            if (src == R || !M_tasks(src, R)) continue;
            const uint64_t pb = M_bytes(src, R);
            uint64_t st = 0;
            if (!b9_ring_place(c->ring_bytes, have, have ? oldest : 0, wp, live, pb, &st)) { fits = false; break; }
            r_start[src] = st;
            have = true;                                               // (an empty ring's first arrival is placed at 0 and becomes the oldest segment: oldest = 0)
            wp = st + b9_seg_span(pb); live += pb;
        }
    }
    h[0] = fits ? 1 : 0;
    CU(cudaMemcpyAsync(d_vote, h, sizeof(uint64_t), cudaMemcpyHostToDevice, s));
    NC(g_nccl.AllGather(d_vote, d_vote + 1, 1, NCCL_U64, c->nccl_comm, s));
    CU(cudaMemcpyAsync(h + off_vote, d_vote, (size_t)(1 + W) * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    for (int r = 0; r < W; ++r)
        if (!h[off_vote + 1 + r])
            return fail(B9_ENOSPC, "b9_rebalance: rank %d cannot take its share (%llu tasks / %llu bytes arrive here); no rank changed its ring",
                        r, (unsigned long long)recv_tasks, (unsigned long long)recv_bytes);
    phase("feasibility vote");
    // ---- 6. stage the slot words of what leaves (and the payload of ranges that are not one piece of the ring)
    auto al = [](uint64_t x) { return (x + 255ull) & ~255ull; };
    uint64_t need_s = 0, need_r = 0;
    for (int d = 0; d < W; ++d) {
        if (d == R) continue;
        const uint64_t k = cuts.hi[d] - cuts.lo[d];
        if (k) need_s += al(meta_layout(k).total) + (cuts.contiguous[d] ? 0 : al(cuts.bytes[d] + 16));
        const uint64_t rk = M_tasks(d, R);
        if (rk) need_r += al(meta_layout(rk).total);
    }
    { const int rc = c->d_xchg_send.ensure(need_s, "b9_rebalance: send staging", need_s / 4); if (rc) return rc; }
    { const int rc = c->d_xchg_recv.ensure(need_r, "b9_rebalance: receive staging", need_r / 4); if (rc) return rc; }
    std::vector<uint8_t*> s_meta(W, nullptr), r_meta(W, nullptr);
    std::vector<const uint8_t*> s_pay(W, nullptr);
    uint64_t so = 0, ro = 0;
    for (int d = 0; d < W; ++d) {
        if (d == R) continue;
        const uint64_t k = cuts.hi[d] - cuts.lo[d];
        if (k) {
            const MetaLayout ml = meta_layout(k);
            s_meta[d] = c->d_xchg_send + so; so += al(ml.total);
            uint8_t* staged = nullptr;
            if (!cuts.contiguous[d]) { staged = c->d_xchg_send + so; so += al(cuts.bytes[d] + 16); }
            s_pay[d] = staged ? staged : c->d_payload + cuts.phys[d];
            const uint32_t threads = staged ? (uint32_t)k * 32u : (uint32_t)k;
            gather_tasks_kernel<<<(threads + 255) / 256, 256, 0, s>>>(c->d_payload, c->d_off, c->d_hdr, c->d_ids, c->d_ts, c->d_exp, c->slot_mask,
                                                                       c->head_task + cuts.lo[d], (uint32_t)k, c->d_prefix + cuts.lo[d], staged,
                                                                       (uint64_t*)(s_meta[d] + ml.rel), (int64_t*)(s_meta[d] + ml.ts), (int64_t*)(s_meta[d] + ml.exp),
                                                                       (uint4*)(s_meta[d] + ml.ids), s_meta[d] + ml.flags, s_meta[d] + ml.retries);
            CU(cudaGetLastError());
            c->stats.kernel_launches++;
        }
        const uint64_t rk = M_tasks(d, R);
        if (rk) { r_meta[d] = c->d_xchg_recv + ro; ro += al(meta_layout(rk).total); }
    }
    // ---- the exchange: one grouped send/recv; arriving payload goes straight to its place in the ring
    NC(g_nccl.GroupStart());
    for (int d = 0; d < W; ++d) {
        if (d == R) continue;
        const uint64_t k = cuts.hi[d] - cuts.lo[d];
        if (k) {
            NC(g_nccl.Send(s_meta[d], meta_layout(k).total, NCCL_U8, d, c->nccl_comm, s));
            if (cuts.bytes[d]) NC(g_nccl.Send(s_pay[d], cuts.bytes[d], NCCL_U8, d, c->nccl_comm, s));
        }
        const uint64_t rk = M_tasks(d, R);
        if (rk) {
            NC(g_nccl.Recv(r_meta[d], meta_layout(rk).total, NCCL_U8, d, c->nccl_comm, s));
            if (M_bytes(d, R)) NC(g_nccl.Recv(c->d_payload + r_start[d], M_bytes(d, R), NCCL_U8, d, c->nccl_comm, s));
        }
    }
    NC(g_nccl.GroupEnd());
    phase("pack slot words + exchange");
    // ---- 7. what left: a prefix of my FIFO went to lower ranks, a suffix to higher ranks
    {
        const uint64_t front = cuts.lo[R], back = n - cuts.hi[R];
        uint64_t front_bytes = 0;
        for (int d = 0; d < R; ++d) front_bytes += cuts.bytes[d];
        if (back) drop_back(c, back, cuts.keep_end_phys);
        if (front) { c->pending_bytes -= front_bytes; c->head_task += front; free_segments(c); }
    }
    // what arrived is appended, source by source, as new segments at the places chosen in 5
    for (int src = 0; src < W; ++src) {
        const uint64_t rk = (src == R) ? 0 : M_tasks(src, R);
        if (!rk) continue;
        const MetaLayout ml = meta_layout(rk);
        const uint64_t pb = M_bytes(src, R);
        const uint64_t start = r_start[src];
        CU(copy_slot_ids(c, c->tail_task, rk, r_meta[src] + ml.ids, true, cudaMemcpyDeviceToDevice, s));
        ingest_kernel<<<(uint32_t)((rk + 255) / 256), 256, 0, s>>>((const uint64_t*)(r_meta[src] + ml.rel), (uint32_t)rk, start, c->tail_task, c->slot_mask,
                                                                  (const int64_t*)(r_meta[src] + ml.ts), (const int64_t*)(r_meta[src] + ml.exp),
                                                                  r_meta[src] + ml.retries, r_meta[src] + ml.flags, c->d_off, c->d_hdr, c->d_ts, c->d_exp);
        CU(cudaGetLastError());
        c->stats.kernel_launches++;
        cudaEvent_t ready;
        CU(take_event(c, &ready));
        CU(cudaEventRecord(ready, s));
        append_segment(c, (uint32_t)rk, start, pb, 0u, (uint32_t)rk, ready);   // (max_len and the pickle tasks not known)
    }
    // ---- cancelled tasks may have moved either way: recount over the new window (only if some rank held any)
    if (any_cancelled) {
        const uint64_t depth = c->tail_task - c->head_task;
        uint64_t count = 0;
        { const int rc = count_cancelled(c, c->head_task, depth, s, &count); if (rc) return rc; }
        if (depth) c->stats.kernel_launches++;
        c->cancelled_pending = count;
    } else {
        CU(cudaStreamSynchronize(s));         // the caller's next call may be on any stream; the exchange is complete when we return
        c->cancelled_pending = 0;
    }
    phase("drop + append + recount");
    if (info) {
        info->world = (uint32_t)W; info->rank = (uint32_t)R;
        info->tasks_before = n; info->bytes_before = my_bytes;
        info->tasks_sent = sent_tasks; info->bytes_sent = sent_bytes; info->tasks_received = recv_tasks; info->bytes_received = recv_bytes;
        info->tasks_after = c->tail_task - c->head_task; info->bytes_after = c->pending_bytes;
    }
    return B9_OK;
}

// =========================================================================== result sink (SURVEY.md §8(f) row 1)
uint64_t b9_sink_object_bytes(uint32_t n_records, uint64_t blob_bytes) { return b9sink::layout(n_records, blob_bytes).total; }

int64_t b9_sink_pack(const b9_results* r, uint8_t* obj, uint64_t cap) {
    if (!r || !obj) return fail(B9_EINVAL, "b9_sink_pack: NULL argument");
    const uint32_t n = r->n_results;
    const b9sink::Layout L = b9sink::layout(n, r->n_bytes);
    if (cap < L.total) return fail(B9_ENOSPC, "b9_sink_pack: object needs %llu bytes, caller gave %llu", (unsigned long long)L.total, (unsigned long long)cap);
    memset(obj, 0, L.blob);                                               // header + index, padding included: the object is deterministic
    b9sink::write_header(obj, n, r->n_bytes, r->task_duration, r->n_popped);
    if (n) {
        memcpy(obj + L.ids, r->task_ids, (size_t)n * 16); memcpy(obj + L.offsets, r->offsets, (size_t)n * 8);
        memcpy(obj + L.lengths, r->lengths, (size_t)n * 4); memcpy(obj + L.status, r->status, n); memcpy(obj + L.has, r->has_result, n);
    }
    if (r->n_bytes) memcpy(obj + L.blob, r->payload, r->n_bytes);
    return (int64_t)L.total;
}

// b9_drain_fetch with the records landing as ONE sink object in the caller's buffer: the device-to-host copies write the
// object's sections directly (pass page-locked memory for full PCIe bandwidth), the header is written last.
int64_t b9_drain_fetch_object(b9_ctx* c, uint8_t* obj, uint64_t cap, uint64_t* object_bytes) {
    if (!c || !obj) return fail(B9_EINVAL, "b9_drain_fetch_object: NULL argument");
    uint32_t n = 0; uint64_t bytes = 0;
    {
        OutLock out_lk(c);
        CU(cudaSetDevice(c->device));
        { int rc = finish_launch(c); if (rc) return rc; }
        if (!c->res.have) return fail(B9_EINVAL, "b9_drain_fetch_object: no drain results are waiting");
        n = c->res.n; bytes = c->res.bytes;
    }
    const b9sink::Layout L = b9sink::layout(n, bytes);
    if (object_bytes) *object_bytes = L.total;
    if (cap < L.total) return fail(B9_ENOSPC, "b9_drain_fetch_object: object needs %llu bytes, caller gave %llu", (unsigned long long)L.total, (unsigned long long)cap);
    memset(obj, 0, sizeof(b9sink::Header));
    b9_results r; memset(&r, 0, sizeof r);
    r.task_ids = obj + L.ids; r.offsets = (uint64_t*)(obj + L.offsets); r.lengths = (uint32_t*)(obj + L.lengths);
    r.status = obj + L.status; r.has_result = obj + L.has; r.payload = obj + L.blob;
    r.cap_tasks = n ? n : 1; r.cap_bytes = bytes ? bytes : 1;
    const int64_t got = b9_drain_fetch(c, &r);
    if (got < 0) return got;
    // the gaps between the sections (alignment) are part of the object: make them deterministic
    auto zero_gap = [&](uint64_t from, uint64_t to) { if (to > from) memset(obj + from, 0, to - from); };
    zero_gap(L.ids + (uint64_t)n * 16, L.offsets); zero_gap(L.offsets + (uint64_t)n * 8, L.lengths); zero_gap(L.lengths + (uint64_t)n * 4, L.status);
    zero_gap(L.status + n, L.has); zero_gap(L.has + n, L.blob);
    b9sink::write_header(obj, n, bytes, r.task_duration, r.n_popped);
    return got;
}

int b9_sink_get(const uint8_t* obj, uint64_t size, uint32_t index, b9_sink_record* rec) {
    const b9sink::Header* h = b9sink::check(obj, size);
    if (!h || !rec) return fail(B9_EINVAL, "b9_sink_get: not a sink object");
    if (index >= h->n_records) return fail(B9_EINVAL, "b9_sink_get: record %u of %u", index, h->n_records);
    const uint64_t off = ((const uint64_t*)(obj + h->off_offsets))[index];
    const uint32_t len = ((const uint32_t*)(obj + h->off_lengths))[index];
    if (off + len > h->blob_bytes) return fail(B9_EINVAL, "b9_sink_get: record %u points outside the blob", index);
    rec->task_id = obj + h->off_ids + (uint64_t)index * 16;
    rec->status = obj[h->off_status + index]; rec->has_result = obj[h->off_has + index];
    rec->data = obj + h->off_blob + off; rec->length = len; rec->index = index;
    return B9_OK;
}

int b9_sink_find(const uint8_t* obj, uint64_t size, const uint8_t* task_id, b9_sink_record* rec) {
    const b9sink::Header* h = b9sink::check(obj, size);
    if (!h || !task_id || !rec) return fail(B9_EINVAL, "b9_sink_find: not a sink object");
    const uint8_t* ids = obj + h->off_ids;
    for (uint32_t i = 0; i < h->n_records; ++i)
        if (memcmp(ids + (uint64_t)i * 16, task_id, 16) == 0) return b9_sink_get(obj, size, i, rec);
    return B9_ENOENT;
}

int64_t b9_sink_result_json(const uint8_t* data, uint64_t length, uint8_t* out, uint64_t cap) {
    if (length == 0) return 0;                                             // `if len(result) > 0`: the field stays unset
    if (!data || !out) return fail(B9_EINVAL, "b9_sink_result_json: NULL argument");
    uint64_t vs = 0, ve = 0;
    if (b9sink::raw_message(data, length, &vs, &ve)) {
        if (ve - vs > cap) return fail(B9_ENOSPC, "b9_sink_result_json: %llu bytes needed", (unsigned long long)(ve - vs));
        memcpy(out, data + vs, ve - vs);
        return (int64_t)(ve - vs);
    }
    const uint64_t need = 11 + b9sink::base64_len(length) + 2;             // {"base64":"..."}
    if (need > cap) return fail(B9_ENOSPC, "b9_sink_result_json: %llu bytes needed", (unsigned long long)need);
    memcpy(out, "{\"base64\":\"", 11);
    b9sink::base64_std(data, length, out + 11);
    memcpy(out + 11 + b9sink::base64_len(length), "\"}", 2);
    return (int64_t)need;
}

int b9_stats_get(b9_ctx* c, b9_stats* out) {
    if (!c || !out) return fail(B9_EINVAL, "b9_stats_get: NULL argument");
    std::lock_guard<std::mutex> lk(c->mu);
    *out = c->stats;
    return B9_OK;
}

int b9_sync(b9_ctx* c) {
    if (!c) return fail(B9_EINVAL, "b9_sync: ctx is NULL");
    CU(cudaSetDevice(c->device));
    { OutLock span_lk(c); }                    // the open span ends behind the last drain kernel, not after this wait
    CU(cudaStreamSynchronize(c->stream_in));
    CU(cudaStreamSynchronize(c->stream));
    OutLock out_lk(c);
    return finish_launch(c);
}

int b9_task_queue_scale(int64_t queue_length, int64_t tasks_per_container, int64_t max_containers, int64_t max_replicas, int* valid) {
    if (valid) *valid = 1;
    if (queue_length == 0) return 0;
    if (queue_length == -1 || tasks_per_container <= 0) { if (valid) *valid = 0; return 0; }
    int64_t desired = queue_length / tasks_per_container + (queue_length % tasks_per_container > 0 ? 1 : 0);
    return (int)std::min<int64_t>(std::min<int64_t>(max_containers, max_replicas), desired);
}

}  // extern "C"
