// Shared definitions of the drain: ring slot words, the control block, the result records every drain kernel writes
// (DrainOut and its helpers), the argument block and the SDK's canonical frame. The drain itself is drain2.cuh.
// Reference behaviour realised per task:
//     pop + decode   pkg/abstractions/taskqueue/client.go:43-96, taskqueue.go:213-214
//     loads + call   sdk/src/beta9/runner/taskqueue.py:196-201,349-361
//     result         sdk/src/beta9/runner/taskqueue.py:378, runner/common.py:484-489
#pragma once
#include <stdint.h>
#include "json_device.cuh"
#include "handlers_device.cuh"
#include "handler_seq.cuh"

namespace b9 {

// ring header word: len:32 | flags:8 | retries:8 | reserved:16
__host__ __device__ __forceinline__ uint64_t hdr_pack(uint32_t len, uint8_t flags, uint8_t retries) {
    return (uint64_t)len | ((uint64_t)flags << 32) | ((uint64_t)retries << 40);
}
__host__ __device__ __forceinline__ uint32_t hdr_len(uint64_t h) { return (uint32_t)h; }
__host__ __device__ __forceinline__ uint32_t hdr_flags(uint64_t h) { return (uint32_t)(h >> 32) & 0xFFu; }
__host__ __device__ __forceinline__ uint32_t hdr_retries(uint64_t h) { return (uint32_t)(h >> 40) & 0xFFu; }
constexpr uint32_t B9_TF_HTTP_BODY_BIT = 0x02u;      // == B9_TF_HTTP_BODY (include/b9gpu.h)
constexpr uint32_t B9_TF_PICKLE_BIT    = 0x04u;      // == B9_TF_PICKLE
constexpr uint32_t B9_TF_TASK_MSG_BIT  = 0x08u;      // == B9_TF_TASK_MSG

struct DrainCtl {
    unsigned long long ticket;      // next tile to hand out
    unsigned long long total;       // scratch word for 8-byte read-backs (task_phys_off)
    unsigned long long bytes;       // result-byte cursor (one atomicAdd per tile); final value = total bytes
    unsigned int overflow;          // result staging too small
    unsigned int total_cnt;         // result records of the whole window
    unsigned int n_slow;            // identity: tasks deferred to the tail of the kernel (non-canonical escapes, foreign framing), reserved so far
    unsigned int slow_head;         // identity: next deferred task to take
    unsigned int workers_done;      // identity: workers that are through with their tiles (everything they defer is published before)
};

// Control blocks of the drain: a ring, so that no memset has to run between two back-to-back drain kernels. Launch e uses
// entry e % D3_CTL_RING and, after its grid-dependency wait (launch e - 1 has completed), zeroes entry (e + 1) % D3_CTL_RING
// for launch e + 1. Two entries suffice: the entry launch e zeroes is the one launch e - 1 used, and nothing reads that one
// any more — launch e - 1 is complete, launch e + 1 touches its own entry only after its own wait (launch e has completed,
// zeroing included), and the host reads an entry only for the launch it finishes, which is then the last one enqueued.
constexpr uint32_t D3_CTL_RING = 2;

// A task the identity main loop could not settle. Published without a lock: w1 first, then (after a fence) w0, whose upper
// 24 bits carry the launch's epoch — a consumer that claimed the slot polls w0 until the epoch is this launch's.
struct SlowItem {
    unsigned long long w0;          // payload ring offset (40 bits) | epoch << 40
    unsigned long long w1;          // len (30 bits) | bit 30 = HTTP body, bit 31 = the SDK's canonical frame is present | record index (24 bits) << 32 | bit 56 = cloudpickle-framed
                                    // | bit 57 = a TaskMessage record (B9_TF_TASK_MSG)
};

// The result records of a drain (or a wire encoding): record j is its id, status[j], has[j] and the bytes
// payload[off[j], off[j] + len[j]). Every kernel that writes records places their bytes with reserve_bytes /
// warp_reserve_bytes and writes the rest with store_record and store_record_id.
// Where record j's id lives: when the launch compacts its records (a drain in count mode: cancelled slots leave no
// record), in ids[j]; otherwise record j is the window's task j, and its id stays in that task's ring slot, which nothing
// writes before the results are fetched (a pop is committed by the fetch): the fetch copies it from there, and no
// kernel spends 16 bytes of reads and 16 of writes per record on copying it.
struct DrainOut {
    uint8_t*  payload; uint64_t cap;
    uint64_t* off;                  // [n_tasks + 1]  start of each record's bytes
    uint32_t* len;                  // [n_tasks]      length of each record's bytes
    uint4*    ids;                  // [n_tasks]      written only when ids_compacted
    uint8_t*  status;               // [n_tasks]
    uint8_t*  has;                  // [n_tasks]
    DrainCtl* ctl;                  // the byte cursor and the overflow flag; for a drain, this launch's entry of the control ring
    uint32_t  ids_compacted;        // 1: record j's id is ids[j]; 0: it is the ring id of the window's task j
};

// Result bytes are placed by an atomicAdd on ctl->bytes. A reservation that ends past `cap` sets ctl->overflow (the host
// then reports B9_ENOSPC and consumes nothing); the records it was for get offset 0 and their bytes are not written.
// The caller chooses the byte count. drain3_kernel's identity tiles round it up to 16 bytes, because d3_copy_tile writes
// a tile's range with aligned 16-byte stores. slow_task and the pickle pass, which take bytes from the same cursor, round
// as well so that an identity drain's cursor stays aligned, and the endpoint kernel rounds as identity's tiles do. The
// other handlers' tiles and the wire encoder reserve exact byte counts: no d3_copy_tile shares their cursor.
struct Reservation { unsigned long long base; bool fits; };

// one thread reserves `bytes`
__device__ __forceinline__ Reservation reserve_bytes(const DrainOut& o, uint32_t bytes) {
    Reservation r; r.base = 0;
    if (bytes) r.base = atomicAdd(&o.ctl->bytes, (unsigned long long)bytes);
    r.fits = r.base + bytes <= o.cap;
    if (!r.fits) o.ctl->overflow = 1u;
    return r;
}
// the whole warp, `bytes` the same on every lane: lane 0 reserves, every lane gets the reservation
__device__ __forceinline__ Reservation warp_reserve_bytes(const DrainOut& o, uint32_t bytes, int lane) {
    Reservation r; r.base = 0;
    if (lane == 0 && bytes) r.base = atomicAdd(&o.ctl->bytes, (unsigned long long)bytes);
    r.base = __shfl_sync(0xffffffffu, r.base, 0);
    r.fits = r.base + bytes <= o.cap;
    if (!r.fits && lane == 0) o.ctl->overflow = 1u;
    return r;
}
// record j except its id; its bytes are at `off` when their reservation fits
__device__ __forceinline__ void store_record(const DrainOut& o, uint32_t j, bool fits, unsigned long long off, uint32_t len, uint8_t status, uint8_t has) {
    o.off[j] = fits ? off : 0; o.len[j] = len; o.status[j] = status; o.has[j] = has;
}
// record j's id, whose ring slot is `ring_id`: copied to ids[j] only when the launch compacts its records (the id
// is not even loaded otherwise)
__device__ __forceinline__ void store_record_id(const DrainOut& o, uint32_t j, const uint4* ring_id) {
    if (o.ids_compacted) o.ids[j] = __ldg(ring_id);
}

__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v, int lane) {
    #pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, v, d); if (lane >= d) v += t; }
    return v;
}
__device__ __forceinline__ uint32_t warp_excl_scan(uint32_t v, int lane) { return warp_incl_scan(v, lane) - v; }

struct DrainArgs {
    // ring (inputs)
    const uint8_t*  payload;        // ring bytes
    const uint64_t* off;            // [ring_tasks] physical byte offset of each task's payload
    const uint64_t* hdr;            // [ring_tasks]
    const uint4*    ids;            // [ring_tasks] raw UUID
    uint32_t slot_mask;             // ring_tasks - 1
    uint64_t first_task;            // logical index of the window's first task
    uint32_t n_tasks;
    uint32_t n_tiles;
    DrainOut out;                   // out.ctl: this launch's entry of the control ring, ctl[epoch % D3_CTL_RING]
    DrainCtl* ctl_next;             // the next launch's entry: zeroed by this launch once the previous one has completed
    const uint32_t* tile_base;     // count_mode: [n_tiles] ready tasks before each warp-tile inside its 256-slot block (tile_count_kernel)
    const uint32_t* block_base;     // count_mode: [n / 256 + 1] ready tasks before each 256-slot block (tile_scan_kernel); last = window total
    uint32_t count_mode;            // 0 = no pending task is cancelled (record index = task index), 1 = record index from tile_base
    SlowItem* slow;                 // identity: [n_tasks] work list of deferred tasks
    uint32_t epoch;                 // identity: this launch's tag in SlowItem.w0 (1 .. 2^24 - 1)
    const uint32_t* crc_shift_tabs; // crc32: [levels][4][256] "advance the CRC register over 2^k zero bytes" tables
    uint32_t static_rounds;         // a worker's first static_rounds tiles are worker + q * workers, the rest come from the ticket counter
    uint32_t tile_tasks;            // json_sum: tasks per warp-tile of THIS launch (4 or 8: small windows balance better on finer tiles); others: fixed
    // the context's retry policy (b9_set_retry_policy): an ERROR whose class is in retry_mask is RETRY / RETRY_LIMIT
    uint32_t retry_mask;            // B9_EXC_* bits; 0 = no policy: every answer as without one
    uint32_t max_retries;
    uint32_t* task_of;              // [n_tasks] with a policy: the window task of record j, written for RETRY records (b9_drain_fetch
                                    // re-pushes them) and, by identity's main loop, for every task it defers to the kernel's tail
                                    // (drain3_kernel<H, true>: the launch with a policy; <H, false> is the drain without one)
};

// The user-handler ABI (b9_handler_load, include/b9gpu_handler.cuh): a handler image's entry points receive this
// DrainArgs (with its DrainOut and DrainCtl) by value, and their names carry this version, so that an image built against
// another layout has no entry this library looks up. Bump the version with any change to those structs: the assert below
// fails until the size it names is updated together with it.
#define B9_HANDLER_ABI_VERSION 1
static_assert(B9_HANDLER_ABI_VERSION == 1 && sizeof(DrainArgs) == 208 && sizeof(DrainOut) == 72 && sizeof(DrainCtl) == 48,
              "DrainArgs / DrainOut / DrainCtl changed: bump B9_HANDLER_ABI_VERSION and the sizes here");

// The status record j (of window task t) is written with: an ERROR whose exception class the retry policy names becomes
// RETRY while the task's retries are below max_retries, else RETRY_LIMIT (Dispatcher.RetryTask's test,
// pkg/task/dispatch.go:232-285). `value` is rec.value: an ERROR's exception class. t == ~0u: task_of[j] holds the task.
__device__ __forceinline__ uint8_t retry_settle(const DrainArgs& a, uint32_t j, uint32_t t, uint8_t status, long long value) {
    if (status != ST_ERROR || !((uint32_t)value & a.retry_mask)) return status;
    if (t == ~0u) t = a.task_of[j];
    const uint32_t retries = hdr_retries(__ldg(a.hdr + (uint32_t)((a.first_task + t) & a.slot_mask)));
    if (retries >= a.max_retries) return (uint8_t)ST_RETRY_LIMIT;
    a.task_of[j] = t;
    return (uint8_t)ST_RETRY;
}

// where record j's id is, once store_record_id has run for it (DrainOut::ids_compacted)
__device__ __forceinline__ const uint4* record_id(const DrainArgs& a, uint32_t j) {
    return a.out.ids_compacted ? a.out.ids + j : a.ids + (uint32_t)((a.first_task + j) & a.slot_mask);
}

constexpr uint32_t TC_SLOTS = 256;             // slots per tile_count_kernel block (8 warps x 32)
// count_mode: ready tasks before warp-tile `tile` (of T slots) — the record index of its first ready task
__device__ __forceinline__ uint32_t tile_ready_before(const DrainArgs& a, unsigned long long tile, uint32_t T) {
    return __ldg(a.tile_base + tile) + __ldg(a.block_base + (uint32_t)((tile * T) / TC_SLOTS));
}
// the record index of window task t, which is not cancelled, for the passes that run after the drain kernel: t in a dense
// window; in count mode the ready tasks before its warp-tile plus the ready slots before it in the tile (a.tile_tasks as
// the drain kernel used it)
__device__ __forceinline__ uint32_t window_record(const DrainArgs& a, uint32_t t) {
    if (!a.count_mode) return t;
    const uint32_t tile = t / a.tile_tasks;
    uint32_t j = tile_ready_before(a, tile, a.tile_tasks);
    for (uint32_t q = tile * a.tile_tasks; q < t; ++q) j += (hdr_flags(a.hdr[(uint32_t)((a.first_task + q) & a.slot_mask)]) & 1u) ? 0u : 1u;
    return j;
}

// warp-cooperative byte copy global -> global (arbitrary alignment on both sides).
// 16-byte stores on the destination, 4-byte loads + funnel shift on the source.
__device__ inline void warp_copy(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, uint32_t n, int lane) {
    uint32_t head = (uint32_t)((16u - ((uintptr_t)dst & 15u)) & 15u);
    if (head > n) head = n;
    if (lane < (int)head) dst[lane] = src[lane];
    dst += head; src += head; n -= head;
    uint32_t nvec = n >> 4;
    if (nvec) {
        uint32_t sh = (uint32_t)((uintptr_t)src & 3u);
        const uint32_t* sw = (const uint32_t*)(src - sh);
        uint4* dv = (uint4*)dst;
        uint32_t bits = sh * 8;
        for (uint32_t v = lane; v < nvec; v += 32) {
            const uint32_t* s4 = sw + 4 * v;
            uint32_t w0 = s4[0], w1 = s4[1], w2 = s4[2], w3 = s4[3];   // plain loads: the source may be shared memory
            uint4 o;
            if (sh) {
                uint32_t w4 = s4[4];           // may read up to 3 bytes past the payload: the ring / stage buffer has slack
                o.x = __funnelshift_r(w0, w1, bits); o.y = __funnelshift_r(w1, w2, bits);
                o.z = __funnelshift_r(w2, w3, bits); o.w = __funnelshift_r(w3, w4, bits);
            } else { o.x = w0; o.y = w1; o.z = w2; o.w = w3; }
            dv[v] = o;
        }
    }
    uint32_t done = nvec << 4, tail = n - done;
    if (lane < (int)tail) dst[done + lane] = src[done + lane];
}

// ---- the SDK's canonical frame around one string argument ------------------------------------
// json.dumps({"args": (s,), "kwargs": {}})  ->  {"args": ["<body>"], "kwargs": {}}
__device__ __constant__ uint8_t FRAME_PRE[11] = {'{', '"', 'a', 'r', 'g', 's', '"', ':', ' ', '[', '"'};
__device__ __constant__ uint8_t FRAME_SUF[17] = {'"', ']', ',', ' ', '"', 'k', 'w', 'a', 'r', 'g', 's', '"', ':', ' ', '{', '}', '}'};
constexpr uint32_t FRAME_PRE_LEN = 11, FRAME_SUF_LEN = 17;

}  // namespace b9
