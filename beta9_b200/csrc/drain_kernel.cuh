// Shared definitions of the drain: ring slot words, the control block, the argument block, the SDK's
// canonical frame, and the two small ring kernels (expire, ingest). The drain itself is drain2.cuh.
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

// A task the identity main loop could not settle. Published without a lock: w1 first, then (after a fence) w0, whose upper
// 24 bits carry the launch's epoch — a consumer that claimed the slot polls w0 until the epoch is this launch's.
struct SlowItem {
    unsigned long long w0;          // payload ring offset (40 bits) | epoch << 40
    unsigned long long w1;          // len (30 bits) | bit 30 = HTTP body, bit 31 = the SDK's canonical frame is present | record index (24 bits) << 32 | bit 56 = cloudpickle-framed
                                    // | bit 57 = a TaskMessage record (B9_TF_TASK_MSG)
};

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
    // outputs
    uint8_t*  out_payload; uint64_t out_cap;
    uint64_t* out_off;              // [n_tasks + 1]  start of each record's bytes
    uint32_t* out_len;              // [n_tasks]      length of each record's bytes
    uint4*    out_ids;              // [n_tasks]
    uint8_t*  out_status;           // [n_tasks]
    uint8_t*  out_has;              // [n_tasks]
    // control
    DrainCtl* ctl;
    const uint32_t* tile_base;      // count_mode: [n_tiles] ready tasks before each warp-tile inside its 256-slot block (tile_count_kernel)
    const uint32_t* block_base;     // count_mode: [n / 256 + 1] ready tasks before each 256-slot block (tile_scan_kernel); last = window total
    int handler;
    uint32_t count_mode;            // 0 = no pending task is cancelled (record index = task index), 1 = record index from tile_base
    SlowItem* slow;                 // identity: [n_tasks] work list of deferred tasks
    uint32_t epoch;                 // identity: this launch's tag in SlowItem.w0 (1 .. 2^24 - 1)
    const uint32_t* crc_shift_tabs; // crc32: [levels][4][256] "advance the CRC register over 2^k zero bytes" tables
    uint32_t static_rounds;         // a worker's first static_rounds tiles are worker + q * workers, the rest come from the ticket counter
    uint32_t tile_tasks;            // json_sum: tasks per warp-tile of THIS launch (4 or 8: small windows balance better on finer tiles); others: fixed
};

__device__ __forceinline__ uint64_t ld_volatile_u64(const uint64_t* p) { return *(const volatile uint64_t*)p; }
__device__ __forceinline__ void st_volatile_u64(uint64_t* p, uint64_t v) { *(volatile uint64_t*)p = v; }

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

}  // namespace b9
