/*
 * b9gpu — C ABI of the GPU-native task fan-out path (libb9gpu.so, H100 / sm_90a).
 *
 * This is the drop-in boundary for ONE hot path of beam-cloud/beta9: the per-request task
 * dispatch loop (push a task through the queue, pop it in a runner, deserialise, call the
 * handler, serialise the result). The reference has no FFI for this path; the seams it does have
 * are in-process Go interfaces, and each entry point below names the reference interface it
 * replaces (paths relative to the reference repo). INTEGRATION.md shows the cgo and ctypes stubs
 * that bind them.
 *
 * Conventions
 *   - plain C, no exceptions across the boundary; `int` returns: 0 = ok, negative = -errno style
 *     code below; `b9_last_error()` gives text for the CALLING THREAD's last failure (thread-local,
 *     whatever ctx is passed; a cgo caller must stay on its OS thread between the failing call and
 *     this one: runtime.LockOSThread, INTEGRATION.md §1).
 *   - a `b9_ctx` owns all device and pinned memory of one GPU; callers own the buffers they pass.
 *     Every call copies what it needs before returning (cgo pointer rules), so Go may free or
 *     reuse its slices immediately. Buffers obtained from `b9_host_alloc` are page-locked: pass
 *     those for full PCIe bandwidth (pageable memory works, more slowly).
 *   - thread safety: all functions may be called concurrently from many OS threads (goroutine
 *     backed or not). Producers and the drainer of one ctx run CONCURRENTLY: pushes serialise among
 *     themselves (FIFO order is the order in which they are enqueued), drain-side calls (launch,
 *     fetch, expire, wire records) serialise among themselves, and neither side waits for the
 *     other's DMA or kernels. b9_rebalance excludes both for its duration.
 *   - a batch is packed SoA: `task_ids` n x 16 raw UUID bytes, `payload` one blob, `offsets`
 *     n+1 byte offsets into it. A task's payload is the exact `TaskQueuePutRequest.payload`
 *     bytes (pkg/abstractions/taskqueue/taskqueue.proto:20-23), i.e. what the SDK's
 *     `json.dumps({"args": args, "kwargs": kwargs})` produced
 *     (sdk/src/beta9/abstractions/taskqueue.py:284-287).
 */
#ifndef B9GPU_H
#define B9GPU_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B9_ABI_VERSION 2u   /* 2: b9_results.task_duration, b9_batch_push_v, b9_running */

/* ---- error codes ------------------------------------------------------------------------ */
#define B9_OK          0
#define B9_EINVAL    (-22)   /* bad argument                                                    */
#define B9_ENOMEM    (-12)   /* host or device allocation failed                                */
#define B9_ENOSPC    (-28)   /* pending ring full / caller's result buffers too small           */
#define B9_E2BIG      (-7)   /* one task or one batch exceeds a configured maximum              */
#define B9_EIO        (-5)   /* CUDA / NCCL runtime error (text in b9_last_error)               */
#define B9_ENODEV    (-19)   /* no usable CUDA device                                           */
#define B9_ENOSYS    (-38)   /* handler id unknown                                              */
#define B9_ENOENT     (-2)   /* b9_sink_find: no record of that task in the object              */

/* ---- GPU "kernel handlers": the user-function slot (sdk/src/beta9/runner/common.py:297-305)
 *      for which a device implementation exists. Semantics are those of the Python functions in
 *      oracle/pyoracle/handlers.py invoked as `handler(*args, **kwargs)`. ------------------- */
enum b9_handler {
    B9_H_IDENTITY = 0,  /* def identity(s, /): return s              (configs[0] echo, configs[1])
                         * any JSON argument: strings, numbers (float64, Python's int/float reading of
                         * Go's text), non-empty lists and objects (Go's sorted, de-duplicated keys)     */
    B9_H_CRC32    = 1,  /* def crc32(s, /): return zlib.crc32(s.encode())                (configs[2]) */
    B9_H_VADD_F32 = 2,  /* base64(fp32 a||b) -> base64(a+b)                               (configs[3]) */
    B9_H_JSON_SUM = 3,  /* def json_sum(obj, /): return sum(obj["values"])                (configs[4])
                         * ints exactly in a C long, floats with CPython 3.12's compensated sum       */
    B9_H_COUNT_
};

/* ---- per-task status, reported in b9_results.status ---------------------------------------
 * COMPLETE/ERROR/RETRY are the runner's TaskStatus values (sdk/src/beta9/type.py TaskStatus,
 * set at sdk/src/beta9/runner/taskqueue.py:344-361). REJECTED means the reference would have
 * answered TaskQueuePutResponse{Ok:false} and never created the task
 * (pkg/abstractions/taskqueue/taskqueue.go:213-218): the batch interface validates on the device,
 * at drain time. UNSUPPORTED means the payload is valid but outside what the device handler
 * implements: the host must route that task through the reference's own CPU loop. The device
 * never guesses. For identity and json_sum that is: a number literal of more than 19 significant
 * digits whose rounding the fast parser cannot settle, nesting deeper than 16 (identity) / 64
 * levels, an object of more than 64 members (identity), and a json_sum whose Python value needs
 * an int outside the C long range. */
enum b9_status {
    B9_ST_COMPLETE    = 0,
    B9_ST_ERROR       = 1,
    B9_ST_RETRY       = 2,
    B9_ST_REJECTED    = 3,
    B9_ST_UNSUPPORTED = 4
};

/* ---- per-task flags (b9_push_meta.flags / ring header) ------------------------------------ */
#define B9_TF_CANCELLED 0x01u  /* task already completed/cancelled/expired: TaskQueuePop skips it
                                  (taskqueue.go:261-265); the drain compacts it away           */

#define B9_TF_HTTP_BODY 0x02u  /* the payload is an HTTP request body of the task-queue endpoint
                                  (pkg/abstractions/taskqueue/http.go:38-78), not the SDK's put payload:
                                  args / kwargs follow SerializeHttpPayload (pkg/task/serialize.go:16-101) —
                                  a MAP decode: exact keys, "args" only if a list, "kwargs" only if an object,
                                  otherwise the body's remaining keys are the keyword arguments; an empty body
                                  is an empty payload; B9_ST_REJECTED = HTTP 400 "invalid request payload".
                                  (Query-string arguments are the host's to merge before the push.)            */

#define B9_TF_PICKLE    0x04u  /* the payload is the argument blob of the FUNCTION path: cloudpickle.dumps({"args": args,
                                  "kwargs": kwargs}) as `.map()` / `.remote()` send it (sdk/src/beta9/abstractions/function.py:
                                  198-205), which the gateway hands to the runner untouched when it starts 80 05 95
                                  (pkg/abstractions/function/task.go:84,104-108); the result bytes are cloudpickle.dumps(result)
                                  (sdk/src/beta9/runner/function.py:236-283). The device settles ONE shape bit-exactly — a single
                                  `str` argument (< 64 KiB of UTF-8), no keyword arguments, handler identity — and reports every
                                  other pickle B9_ST_UNSUPPORTED for the host's CPU loop.                                      */

#define B9_TF_TASK_MSG  0x08u  /* the payload is a TaskMessage record as TaskQueuePop returns it (pkg/abstractions/taskqueue/taskqueue.go:
                                  238-309): the JSON TaskMessage.Encode writes (pkg/types/task.go:79-90) — a popped record, or the one
                                  Dispatcher.RetryTask re-encodes (pkg/task/dispatch.go:232-285). The drain runs the runner's half of the
                                  loop on it: json.loads, the handler, serialize_result (sdk/src/beta9/runner/taskqueue.py:196-201,349-378).
                                  Results and statuses go into b9_results like any other task's; the record id is the slot's id from the
                                  push, which must be the record's "task_id". B9_ST_REJECTED never comes out of this path (the task exists).
                                  The device answers a record only where CPython's reading of it equals its reading of Go's re-encoding
                                  (DESIGN.md §4 "Queue records"): the whole record UTF-8, strict JSON, "task_id" / "args" / "kwargs" once
                                  each and exact, args a list or null, kwargs an object or null; inside them no lone or encoded surrogate,
                                  every number exactly Go's float text, object keys sorted and unique. Every record TaskMessage.Encode
                                  writes is inside; anything else is B9_ST_UNSUPPORTED, and so is TASK_MSG together with HTTP_BODY or
                                  PICKLE. b9_wire_encode reports a TASK_MSG task UNSUPPORTED. The host fills b9_push_meta's timestamp /
                                  expires / retries from the record it decoded; the device does not read them from the bytes.        */

typedef struct b9_ctx b9_ctx;

typedef struct b9_opts {
    uint32_t struct_size;        /* sizeof(b9_opts), for forward compatibility                  */
    int32_t  device;             /* CUDA device ordinal                                         */
    uint64_t ring_bytes;         /* payload ring capacity in bytes (rounded up to 2^k); 0 = 1 GiB */
    uint32_t ring_tasks;         /* task-slot ring capacity (rounded up to 2^k);       0 = 4 Mi  */
    uint32_t max_drain_tasks;    /* most tasks one drain may take (< 2^24);            0 = 2 Mi  */
    uint64_t max_result_bytes;   /* device result staging per drain;                   0 = 1 GiB */
    uint32_t max_task_bytes;     /* largest single payload accepted;                   0 = 1 MiB */
    uint32_t flags;              /* reserved, 0                                                  */
} b9_opts;

/* optional per-task metadata for a push; NULL pointers mean "all zero" */
typedef struct b9_push_meta {
    const int64_t *timestamp_unix;   /* TaskMessage.Timestamp      (pkg/types/task.go:64)       */
    const int64_t *expires_unix_ns;  /* TaskMessage.Policy.Expires (pkg/types/task.go:121)      */
    const uint8_t *retries;          /* TaskMessage.Retries        (pkg/types/task.go:63)       */
    const uint8_t *flags;            /* B9_TF_*                                                  */
} b9_push_meta;

/* caller-owned result buffers for one drain */
typedef struct b9_results {
    uint8_t  *task_ids;     /* [cap_tasks*16] raw UUID of every task that produced a record      */
    uint8_t  *status;       /* [cap_tasks]    enum b9_status                                     */
    uint8_t  *has_result;   /* [cap_tasks]    0: runner sends no result bytes (falsy result or
                                              error, runner/taskqueue.py:378), 1: bytes present  */
    uint64_t *offsets;      /* [cap_tasks]    result i = payload[offsets[i] .. offsets[i]+lengths[i]) */
    uint32_t *lengths;      /* [cap_tasks]                                                       */
    uint8_t  *payload;      /* [cap_bytes]    TaskQueueCompleteRequest.result bytes
                                              (taskqueue.proto:47-56). Records are FIFO-ordered, their
                                              bytes are laid out in tile-completion order, each tile's
                                              range rounded up to 16 bytes: always go through offsets */
    uint32_t  cap_tasks;
    uint64_t  cap_bytes;
    /* filled by the library */
    uint32_t  n_results;    /* records written                                                   */
    uint32_t  n_popped;     /* tasks removed from the queue (n_results + compacted-away ones)    */
    uint64_t  n_bytes;      /* bytes of payload in use (records + the <= 15 bytes of padding a tile's
                               range is rounded up by): what a copy of the blob has to carry     */
    uint64_t  need_bytes;   /* on B9_ENOSPC: payload capacity that would have sufficed           */
    float     task_duration;/* seconds charged to EVERY task of this drain: (kernel + read-back time) / n_popped.
                               Feeds TaskQueueCompleteRequest.task_duration (taskqueue.proto:50), which the gateway
                               RPUSHes (taskqueue.go:352) and taskQueueAutoscalerSampleFunc averages
                               (taskqueue/autoscaler.go:18-51)                                    */
    uint32_t  reserved_;
} b9_results;

typedef struct b9_stats {
    uint64_t tasks_pushed, tasks_drained, bytes_h2d, bytes_d2h;
    uint64_t kernel_launches;        /* kernels launched by this library since ctx creation      */
    uint64_t drains;
    float    last_push_h2d_ms;       /* CUDA-event time of the last push's H2D copies            */
    float    last_drain_kernel_ms;   /* CUDA-event time around the last drain's kernel(s); after a burst of
                                        B9_DRAIN_ASYNC launches: from the first one's start to the last one's end */
    float    last_drain_d2h_ms;      /* CUDA-event time of the last drain's D2H copies           */
    uint32_t last_drain_tiles;
    uint32_t sm_count;
    uint64_t last_drain_in_bytes;    /* payload bytes of the tasks the last drain consumed       */
    uint64_t last_drain_out_bytes;   /* result bytes the last drain produced                     */
} b9_stats;

/* ---- lifecycle ----------------------------------------------------------------------------- */
uint32_t    b9_abi_version(void);
int         b9_device_count(void);
int         b9_ctx_create(const b9_opts *opts, b9_ctx **out);
void        b9_ctx_destroy(b9_ctx *ctx);
const char *b9_last_error(const b9_ctx *ctx);         /* ctx may be NULL for create failures     */
const char *b9_handler_name(int handler);             /* "identity", "crc32", ...; NULL if unknown */
int         b9_handler_id(const char *name);          /* inverse; B9_ENOSYS if unknown           */

/* page-locked host memory for callers (so that push/drain DMA straight from/to their buffers) */
void       *b9_host_alloc(b9_ctx *ctx, uint64_t bytes);
void        b9_host_free(b9_ctx *ctx, void *p);

/* ---- producer side ---------------------------------------------------------------------------
 * b9_batch_push replaces, for n tasks at once, `taskQueueClient.Push` = Encode + RPUSH
 * (pkg/abstractions/taskqueue/client.go:29-41) as reached from `RedisTaskQueue.put`
 * (pkg/abstractions/taskqueue/taskqueue.go:176-208) -> `Dispatcher.SendAndExecute`
 * (pkg/task/dispatch.go:75-118) -> `TaskQueueTask.Execute` (taskqueue/task.go:16-47).
 * Tasks are appended in order (FIFO, like RPUSH). Returns B9_ENOSPC when the ring cannot take the
 * whole batch (nothing is appended), B9_E2BIG when a task exceeds max_task_bytes. */
int      b9_batch_push(b9_ctx *ctx, const uint8_t *task_ids, const uint8_t *payload,
                       const uint64_t *offsets, uint32_t n, const b9_push_meta *meta);

/* Same, but returns as soon as the copies are enqueued on the context's ingest stream: the caller's
 * buffers MUST be page-locked (b9_host_alloc) and stay untouched until b9_sync() or until a drain has
 * returned the batch's results. Lets the next batch stream in while the previous one is drained and
 * read back (PCIe is full duplex). */
int      b9_batch_push_async(b9_ctx *ctx, const uint8_t *task_ids, const uint8_t *payload,
                             const uint64_t *offsets, uint32_t n, const b9_push_meta *meta);

/* The pack step: the n payloads sit anywhere in the caller's (pageable) memory — Go's `[][]byte`, one slice per
 * TaskQueuePutRequest.payload — and are gathered by a few library threads (B9_PACK_THREADS, default min(16, cores))
 * into one of two page-locked arenas owned by the context, together with the n + 1 offsets; the arena is then pushed
 * like b9_batch_push_async. Everything is copied when the call returns (cgo pointer rules: `payloads[i]` may point into
 * Go memory only if the array of pointers itself is C memory — INTEGRATION.md §1 shows the binding); while batch k is on
 * the wire, batch k+1 is gathered into the other arena. */
int      b9_batch_push_v(b9_ctx *ctx, const uint8_t *task_ids, const uint8_t *const *payloads,
                         const uint32_t *lengths, uint32_t n, const b9_push_meta *meta);

/* ONE task per call, from any number of threads — the reference's own call pattern: `RedisTaskQueue.put` per gRPC / HTTP
 * request goroutine (pkg/abstractions/taskqueue/taskqueue.go:176-226), the endpoint's `RequestBuffer.ForwardRequest`
 * per request (pkg/abstractions/endpoint/buffer.go:139-168, a mutex-guarded RingBuffer drained one element at a time,
 * buffer.go:170-195). b9_submit appends the payload straight into a page-locked arena of the context (a lock-free
 * reservation + memcpy; the bytes are copied when it returns) and b9_flush hands everything submitted since the last flush
 * to the device as ONE batch, in submission order; while that batch is on the wire, submissions go on into a second arena.
 * A full arena flushes itself. b9_flush returns the number of tasks it pushed (a batch the ring refused — B9_ENOSPC — is
 * kept and pushed again by the next flush). b9_buffered: tasks submitted and not yet pushed (admission: b9_depth +
 * b9_buffered against max_pending_tasks). B9_SUBMIT_BYTES / B9_SUBMIT_TASKS size the arenas (64 MiB / 256 Ki). */
int      b9_submit(b9_ctx *ctx, const uint8_t *task_id, const uint8_t *payload, uint32_t length, uint8_t flags);
int64_t  b9_flush(b9_ctx *ctx);
uint64_t b9_buffered(b9_ctx *ctx);

/* Pending tasks = what `TaskRepository.TasksInFlight` / `taskQueueClient.QueueLength` report for
 * this queue (pkg/repository/task_redis.go:112-119, taskqueue/client.go:99-106); feeds
 * `taskQueueAutoscalerSampleFunc` (taskqueue/autoscaler.go:18-51) unchanged. */
uint64_t b9_depth(b9_ctx *ctx);
uint64_t b9_depth_bytes(b9_ctx *ctx);

/* Tasks a drain has claimed and not yet handed back: the window of the last b9_drain_launch (without B9_DRAIN_PEEK) until
 * its b9_drain_fetch commits the pop. What `TaskRepository.TasksClaimed` (pkg/repository/task_redis.go:58) /
 * `taskQueueClient.TasksRunning` (taskqueue/client.go:109) count for this queue: the first thing
 * `taskQueueAutoscalerSampleFunc` reads (taskqueue/autoscaler.go:19). Lock-free. b9_depth() still includes these tasks. */
uint64_t b9_running(b9_ctx *ctx);

/* Marks every pending task whose expires_unix_ns is non-zero and <= now as cancelled — the
 * unclaimed-task branch of `Dispatcher.monitor` (pkg/task/dispatch.go:173-230). Returns count. */
int64_t  b9_expire(b9_ctx *ctx, int64_t now_unix_ns);

/* ---- consumer side ---------------------------------------------------------------------------
 * b9_drain replaces, for up to max_tasks pending tasks in FIFO order, the whole
 *   TaskQueuePop (taskqueue.go:228-310, client.go:43-96)
 *   -> runner json.loads + handler + serialize_result
 *      (sdk/src/beta9/runner/taskqueue.py:185-204,317-404; runner/common.py:297-305,484-489)
 *   -> TaskQueueComplete's result hand-off (taskqueue.go:312-404)
 * round trip: one persistent kernel deserialises, runs `handler`, and serialises every ready
 * task, then the records are copied to `out`. Returns the number of result records (>= 0) or a
 * negative error. On B9_ENOSPC (caller buffers too small) nothing is consumed, the records stay
 * on the device and `b9_drain_fetch` can collect them with larger buffers. */
int64_t  b9_drain(b9_ctx *ctx, int handler, uint32_t max_tasks, b9_results *out);

/* Two-step form: run the kernel only (results stay in device staging), then fetch. `flags`:
 * B9_DRAIN_PEEK leaves the tasks in the queue, so the same resident batch can be drained again (the
 * benchmark's device-resident timing, retry-on-device-failure). B9_DRAIN_ASYNC returns as soon as
 * the kernels are enqueued, with the number of tasks in the window; the record count, byte count and
 * a result-staging overflow (B9_ENOSPC) are reported by the next b9_drain_fetch or b9_sync. A host that
 * pipelines drains (launch k+1 while it post-processes k) keeps the GPU busy back to back this way. */
#define B9_DRAIN_PEEK  1
#define B9_DRAIN_ASYNC 2
int64_t  b9_drain_launch(b9_ctx *ctx, int handler, uint32_t max_tasks, int flags);
int64_t  b9_drain_fetch(b9_ctx *ctx, b9_results *out);

/* ---- queue wire records ------------------------------------------------------------------------
 * b9_wire_encode materialises, for the first max_tasks pending tasks (they stay pending), the bytes
 * `TaskMessage.Encode` produces (pkg/types/task.go:55-65,79-90) — what client.Push RPUSHes
 * (taskqueue/client.go:29-41) and Dispatcher.Send stores as task state (pkg/task/dispatch.go:105-112):
 * the durable record the Go host keeps in Redis. Fetch them with b9_drain_fetch (record i = pending
 * task i; status 0 = bytes present, 3 = the payload is invalid JSON (no task would exist), 4 = outside
 * the device encoder's domain: non-integer numbers, unsorted / duplicate map keys). Per-task
 * timestamp / expires / retries come from b9_push_meta. */
typedef struct b9_wire_env {
    const char *workspace_name;   /* TaskMessage.WorkspaceName                                     */
    const char *stub_id;          /* TaskMessage.StubId                                            */
    const char *executor;         /* TaskMessage.Executor; NULL = "taskqueue" (types.ExecutorTaskQueue) */
    uint32_t    max_retries;      /* TaskPolicy.MaxRetries (pkg/types/task.go:118-123)             */
    int32_t     timeout;          /* TaskPolicy.Timeout                                            */
    uint32_t    ttl;              /* TaskPolicy.TTL                                                */
} b9_wire_env;
int64_t  b9_wire_encode(b9_ctx *ctx, const b9_wire_env *env, uint32_t max_tasks);

/* ---- multi-GPU: one ctx (= one process, one GPU) per rank of a box -------------------------------
 * The pending ring is sharded over the ranks; tasks are independent units (SURVEY.md §8e), so the
 * drain needs no collective. When ingest landed unevenly, b9_rebalance moves pending tasks so that
 * every rank holds ~1/world of the pending payload BYTES: an all-gather of (count, bytes), the same
 * byte-quantile plan on every rank (b9_rebalance_plan, also callable on its own), an all-gather of
 * the send matrix, then one grouped ncclSend/ncclRecv all-to-all of slot words + payload over
 * NVLink. NCCL is loaded with dlopen (B9_NCCL_LIB or libnccl.so.2). The unique id is created on one
 * rank and handed to the others by the host (the gateway, or torch.distributed in bench.py). */
typedef struct b9_rebalance_info {
    uint32_t world, rank;
    uint64_t tasks_before, bytes_before;
    uint64_t tasks_sent, bytes_sent, tasks_received, bytes_received;
    uint64_t tasks_after, bytes_after;
} b9_rebalance_info;

int      b9_comm_unique_id(uint8_t *out128);
int      b9_comm_init(b9_ctx *ctx, const uint8_t *id128, int rank, int world);
int      b9_rebalance(b9_ctx *ctx, b9_rebalance_info *info);   /* collective over the communicator */
/* prefix[i] = payload bytes of the caller's pending tasks 0..i-1; fills the local FIFO range
 * [send_lo[d], send_hi[d]) destined for every rank d. Pure host arithmetic. */
int      b9_rebalance_plan(uint32_t world, uint32_t rank, const uint64_t *counts, const uint64_t *bytes,
                           const uint64_t *prefix, uint64_t n, uint64_t *send_lo, uint64_t *send_hi);

/* ---- result sink: one packed object per drain -------------------------------------------------------
 * The reference stores every result with its own object-store PUT — `Dispatcher.StoreTaskResult`
 * (pkg/task/dispatch.go:120-144), key "task/<id>/result" (dispatch.go:18-20), called from TaskQueueComplete when
 * `in.Result != nil` (pkg/abstractions/taskqueue/taskqueue.go:394-399) — and the REST read-back applies
 * `addResultToTask` (pkg/api/v1/task.go:295-325). Batched: the records of a drain form ONE self-describing object
 * (128-byte header, SoA index: ids, offsets, lengths, status, has_result; then the result blob), uploaded once; the
 * gateway keeps (object, record index) with the task. b9_drain_fetch_object is b9_drain_fetch with the device-to-host
 * copies writing that object directly into `obj` (no per-task host work; *object_bytes = its size, also on B9_ENOSPC);
 * b9_sink_pack builds the same object from records fetched the ordinary way. b9_sink_get / b9_sink_find give record i /
 * the record of a task id (linear in the number of records) with pointers INTO the object; a record with has_result == 0
 * is a task for which the reference uploads nothing. b9_sink_result_json is addResultToTask's rule for the bytes of one
 * stored result: 0 = the field stays unset (empty object), else the number of bytes written to `out`: the JSON value
 * itself when the bytes are valid JSON (json.Unmarshal into a json.RawMessage: syntax check only, white space around
 * the value dropped), otherwise {"base64":"<std base64>"}. The sink functions are pure host code (no GPU needed). */
typedef struct b9_sink_record {
    const uint8_t *task_id;      /* 16 raw UUID bytes                                                     */
    const uint8_t *data;         /* TaskQueueCompleteRequest.result bytes (meaningful when has_result)    */
    uint32_t       length, index;
    uint8_t        status, has_result;
} b9_sink_record;
uint64_t b9_sink_object_bytes(uint32_t n_records, uint64_t blob_bytes);
int64_t  b9_sink_pack(const b9_results *results, uint8_t *obj, uint64_t cap);
int64_t  b9_drain_fetch_object(b9_ctx *ctx, uint8_t *obj, uint64_t cap, uint64_t *object_bytes);
int      b9_sink_get(const uint8_t *obj, uint64_t size, uint32_t index, b9_sink_record *rec);
int      b9_sink_find(const uint8_t *obj, uint64_t size, const uint8_t *task_id, b9_sink_record *rec);
int64_t  b9_sink_result_json(const uint8_t *data, uint64_t length, uint8_t *out, uint64_t cap);

int      b9_stats_get(b9_ctx *ctx, b9_stats *out);
int      b9_sync(b9_ctx *ctx);

/* ---- host-side helpers kept bit-compatible with the reference --------------------------------
 * `taskQueueScaleFunc` (pkg/abstractions/taskqueue/autoscaler.go:53-79): desired containers for a
 * queue depth; *valid = 0 when the sample is invalid (queue_length == -1). */
int      b9_task_queue_scale(int64_t queue_length, int64_t tasks_per_container,
                             int64_t max_containers, int64_t max_replicas, int *valid);

#ifdef __cplusplus
}
#endif
#endif /* B9GPU_H */
