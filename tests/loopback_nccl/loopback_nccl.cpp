// A loopback stand-in for the nine NCCL calls libb9gpu.so makes (ncclGetUniqueId, ncclCommInitRank, ncclCommDestroy,
// ncclAllGather, ncclSend, ncclRecv, ncclGroupStart, ncclGroupEnd, ncclGetErrorString), for W communicator ranks that
// live in ONE process on ONE device, one host thread per rank. Real NCCL refuses two ranks on one GPU; loaded through
// B9_NCCL_LIB, this library lets all of b9_rebalance -- scan, cut, gather, vote, exchange, ingest -- run on one GPU.
//
// Stream order. Every call blocks its host thread until its data has moved:
//   - it first synchronises the caller's stream, so what it sends is final;
//   - it publishes its buffers to the communicator's rendezvous (one mutex, one condition variable);
//   - it copies what this rank receives from the peers' buffers, device to device on its own stream, and synchronises it;
//   - it returns only once every peer has finished reading this rank's send buffers.
// So work the caller enqueues after the call sees the data, and a sender never reuses a buffer early.
//
// An AllGather is a round all W ranks join. Send / Recv are queued between GroupStart and GroupEnd and matched at
// GroupEnd by (source, destination, order of posting) -- a group only waits for the peers it exchanges with, as in NCCL.
// Errors come back as ncclResult_t codes that ncclGetErrorString explains: a byte-count or datatype mismatch between a
// matched Send and Recv, two ranks calling different collectives, or a wait longer than the timeout (60 s, or
// LB_NCCL_TIMEOUT_S) -- which is how an unmatched operation shows. Nothing aborts and nothing waits forever; a
// communicator that timed out fails every later call at once.
//
// The CUDA driver API is reached through dlopen("libcuda.so.1") with the few prototypes declared below: no CUDA
// header and no runtime library. Plain C++: g++ -O2 -std=c++17 -shared -fPIC -o libloopback_nccl.so loopback_nccl.cpp
//
// Not part of NCCL's API, and never called by libb9gpu.so: lb_log_count / lb_log_get read a per-rank log of every
// call -- the operation, the peer, the byte count, and for an AllGather of at most 64 uint64 words the words this rank
// contributed.
#include <dlfcn.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

#include <chrono>
#include <condition_variable>
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

namespace {

// ---- CUDA driver API, declared by hand
typedef int CUresult;
typedef void* CUcontext;
typedef void* CUstream;
typedef unsigned long long CUdeviceptr;

struct Driver {
    bool tried = false, ok = false;
    CUresult (*StreamSynchronize)(CUstream) = nullptr;
    CUresult (*MemcpyDtoDAsync)(CUdeviceptr, CUdeviceptr, size_t, CUstream) = nullptr;
    CUresult (*MemcpyDtoH)(void*, CUdeviceptr, size_t) = nullptr;
    CUresult (*CtxGetCurrent)(CUcontext*) = nullptr;
    CUresult (*CtxSetCurrent)(CUcontext) = nullptr;
};
Driver g_cu;

// ncclResult_t (nccl.h)
enum { kSuccess = 0, kUnhandledCudaError = 1, kSystemError = 2, kInternalError = 3, kInvalidArgument = 4, kInvalidUsage = 5, kRemoteError = 6 };
// operations in the log
enum { kOpInit = 1, kOpAllGather = 2, kOpSend = 3, kOpRecv = 4 };
constexpr size_t kLogWords = 64;

thread_local std::string t_error;
int err(int code, const std::string& what) { t_error = "loopback nccl: " + what; return code; }

std::chrono::seconds timeout() {
    static const long s = [] { const char* e = getenv("LB_NCCL_TIMEOUT_S"); const long v = e ? atol(e) : 0; return v > 0 ? v : 60L; }();
    return std::chrono::seconds(s);
}

size_t type_size(int dt) {
    switch (dt) {
        case 0: case 1: return 1;                 // ncclInt8, ncclUint8
        case 6: case 9: return 2;                 // ncclFloat16, ncclBfloat16
        case 2: case 3: case 7: return 4;         // ncclInt32, ncclUint32, ncclFloat32
        case 4: case 5: case 8: return 8;         // ncclInt64, ncclUint64, ncclFloat64
        default: return 0;
    }
}

// one posted Send, owned by the sender's GroupEnd until a receiver has read it
struct SendSlot {
    const void* src; size_t bytes; int dtype;
    bool done = false; int code = kSuccess; std::string why;
};

struct Shared {
    int world = 0;
    std::vector<bool> joined;
    int n_joined = 0, n_alive = 0;
    bool broken = false; std::string broken_why;
    // AllGather rounds (all ranks)
    std::vector<const void*> ag_src;
    std::vector<size_t> ag_bytes; std::vector<int> ag_dtype;
    int ag_posted = 0, ag_copied = 0;
    uint64_t ag_posted_gen = 0, ag_copied_gen = 0;
    // point-to-point: chan[s * world + d] = the Sends s posted to d and no receiver has taken yet, in posting order
    std::vector<std::deque<SendSlot*>> chan;
};

struct Comm { uint64_t key; int rank; int world; std::shared_ptr<Shared> sh; CUcontext ctx; };

struct LogEntry { int op; int peer; uint64_t bytes; std::vector<uint64_t> words; };

std::mutex g_mu;
std::condition_variable g_cv;
std::map<uint64_t, std::shared_ptr<Shared>> g_comms;       // unique-id key -> rendezvous of the ranks that joined it
std::map<int, std::vector<LogEntry>> g_log;                 // rank -> every call it made, in order
uint64_t g_next_id = 1;

struct PostedOp { bool send; const void* src; void* dst; size_t bytes; int dtype; int peer; };
struct Group { int depth = 0; Comm* comm = nullptr; CUstream stream = nullptr; std::vector<PostedOp> ops; std::string bad; };
thread_local Group t_group;

int load_driver() {
    std::lock_guard<std::mutex> lk(g_mu);
    if (!g_cu.tried) {
        g_cu.tried = true;
        if (void* h = dlopen("libcuda.so.1", RTLD_NOW | RTLD_LOCAL)) {
            *(void**)&g_cu.StreamSynchronize = dlsym(h, "cuStreamSynchronize");
            *(void**)&g_cu.MemcpyDtoDAsync = dlsym(h, "cuMemcpyDtoDAsync_v2");
            *(void**)&g_cu.MemcpyDtoH = dlsym(h, "cuMemcpyDtoH_v2");
            *(void**)&g_cu.CtxGetCurrent = dlsym(h, "cuCtxGetCurrent");
            *(void**)&g_cu.CtxSetCurrent = dlsym(h, "cuCtxSetCurrent");
            g_cu.ok = g_cu.StreamSynchronize && g_cu.MemcpyDtoDAsync && g_cu.MemcpyDtoH && g_cu.CtxGetCurrent && g_cu.CtxSetCurrent;
        }
    }
    return g_cu.ok ? kSuccess : err(kSystemError, "cannot load libcuda.so.1 or one of its entry points");
}

void log_call(int rank, int op, int peer, uint64_t bytes, std::vector<uint64_t> words = {}) {
    std::lock_guard<std::mutex> lk(g_mu);
    g_log[rank].push_back(LogEntry{op, peer, bytes, std::move(words)});
}

// the calling thread works in the communicator's context (a thread that has not touched CUDA gets the one the
// communicator was created under)
int enter(const Comm* c, CUstream stream) {
    if (int rc = load_driver()) return rc;
    CUcontext cur = nullptr;
    if (g_cu.CtxGetCurrent(&cur)) return err(kUnhandledCudaError, "cuCtxGetCurrent failed");
    if (!cur && c->ctx && g_cu.CtxSetCurrent(c->ctx)) return err(kUnhandledCudaError, "cuCtxSetCurrent failed");
    if (g_cu.StreamSynchronize(stream)) return err(kUnhandledCudaError, "cuStreamSynchronize of the caller's stream failed");
    return kSuccess;
}

// waits on g_cv (g_mu held through lk) until pred(); false on timeout or when the communicator broke meanwhile
template <class Pred>
bool wait_until(std::unique_lock<std::mutex>& lk, Shared& sh, Pred pred) {
    const auto deadline = std::chrono::steady_clock::now() + timeout();
    while (!pred()) {
        if (sh.broken) return false;
        if (g_cv.wait_until(lk, deadline) == std::cv_status::timeout && !pred()) return false;
    }
    return true;
}

int broke(Shared& sh, const std::string& why) {             // g_mu held
    if (!sh.broken) { sh.broken = true; sh.broken_why = why; }
    g_cv.notify_all();
    return err(sh.broken_why == why ? kInternalError : kRemoteError, sh.broken_why);
}

std::string dstr(size_t bytes, int dtype) { return std::to_string(bytes) + " bytes of datatype " + std::to_string(dtype); }

int all_gather(Comm* c, const void* src, void* dst, size_t bytes, int dtype, CUstream stream) {
    Shared& sh = *c->sh;
    const int W = c->world, R = c->rank;
    std::unique_lock<std::mutex> lk(g_mu);
    if (sh.broken) return err(kRemoteError, "communicator broken earlier: " + sh.broken_why);
    sh.ag_src[R] = src; sh.ag_bytes[R] = bytes; sh.ag_dtype[R] = dtype;
    const uint64_t gen = sh.ag_posted_gen;
    if (++sh.ag_posted == W) { sh.ag_posted = 0; ++sh.ag_posted_gen; g_cv.notify_all(); }
    else if (!wait_until(lk, sh, [&] { return sh.ag_posted_gen != gen; }))
        return broke(sh, "rank " + std::to_string(R) + " waited " + std::to_string(timeout().count()) + " s for its peers to join an AllGather");
    // every rank sees the same published round and reaches the same verdict
    std::string why;
    for (int p = 0; p < W && why.empty(); ++p)
        if (sh.ag_bytes[p] != bytes || sh.ag_dtype[p] != dtype)
            why = "AllGather of " + dstr(sh.ag_bytes[p], sh.ag_dtype[p]) + " on rank " + std::to_string(p) + " against " + dstr(bytes, dtype) + " on rank " + std::to_string(R);
    std::vector<const void*> srcs(sh.ag_src);
    lk.unlock();
    int rc = kSuccess;
    if (why.empty()) {
        for (int p = 0; p < W && rc == kSuccess; ++p) {
            void* to = (uint8_t*)dst + (size_t)p * bytes;
            if (bytes && to != srcs[p] && g_cu.MemcpyDtoDAsync((CUdeviceptr)to, (CUdeviceptr)srcs[p], bytes, stream)) rc = err(kUnhandledCudaError, "cuMemcpyDtoDAsync failed");
        }
        if (rc == kSuccess && g_cu.StreamSynchronize(stream)) rc = err(kUnhandledCudaError, "cuStreamSynchronize after the copies failed");
    }
    lk.lock();
    const uint64_t cgen = sh.ag_copied_gen;
    if (++sh.ag_copied == W) { sh.ag_copied = 0; ++sh.ag_copied_gen; g_cv.notify_all(); }
    else if (!wait_until(lk, sh, [&] { return sh.ag_copied_gen != cgen; }))
        return broke(sh, "rank " + std::to_string(R) + " waited " + std::to_string(timeout().count()) + " s for its peers to finish an AllGather");
    if (!why.empty()) return err(kInvalidUsage, why);
    return rc;
}

int group_end(Comm* c, const std::vector<PostedOp>& ops, CUstream stream) {
    Shared& sh = *c->sh;
    const int W = c->world, R = c->rank;
    std::vector<std::unique_ptr<SendSlot>> mine;
    std::unique_lock<std::mutex> lk(g_mu);
    if (sh.broken) return err(kRemoteError, "communicator broken earlier: " + sh.broken_why);
    for (const PostedOp& o : ops)
        if (o.send) {
            mine.emplace_back(new SendSlot{o.src, o.bytes, o.dtype, false, kSuccess, {}});
            sh.chan[(size_t)R * W + o.peer].push_back(mine.back().get());
        }
    g_cv.notify_all();
    // match my receives in posting order, per source, against the sends in theirs
    std::vector<SendSlot*> taken;
    int rc = kSuccess; std::string why;
    for (const PostedOp& o : ops) {
        if (o.send) continue;
        std::deque<SendSlot*>& q = sh.chan[(size_t)o.peer * W + R];
        if (!wait_until(lk, sh, [&] { return !q.empty(); })) {
            for (SendSlot* t : taken) { t->done = true; t->code = kRemoteError; t->why = "the receiver timed out"; }
            return broke(sh, "rank " + std::to_string(R) + ": a Recv of " + dstr(o.bytes, o.dtype) + " from rank " + std::to_string(o.peer) +
                             " found no matching Send within " + std::to_string(timeout().count()) + " s");
        }
        SendSlot* s = q.front(); q.pop_front();
        taken.push_back(s);
        if (rc != kSuccess) continue;
        if (s->bytes != o.bytes || s->dtype != o.dtype) {
            why = "Send of " + dstr(s->bytes, s->dtype) + " from rank " + std::to_string(o.peer) + " matched with a Recv of " + dstr(o.bytes, o.dtype) +
                  " on rank " + std::to_string(R);
            rc = kInvalidUsage;
        } else if (o.bytes && g_cu.MemcpyDtoDAsync((CUdeviceptr)o.dst, (CUdeviceptr)s->src, o.bytes, stream)) {
            why = "cuMemcpyDtoDAsync failed"; rc = kUnhandledCudaError;
        }
    }
    lk.unlock();
    if (rc == kSuccess && g_cu.StreamSynchronize(stream)) { why = "cuStreamSynchronize after the copies failed"; rc = kUnhandledCudaError; }
    lk.lock();
    for (SendSlot* t : taken) { t->done = true; t->code = rc; t->why = why; }
    g_cv.notify_all();
    // my send buffers are free once every receiver has read them
    for (auto& s : mine) {
        if (!wait_until(lk, sh, [&] { return s->done; })) {
            // withdraw what nobody took, so that no peer reads this buffer after we return
            for (auto& m : mine)
                if (!m->done) for (auto& q : sh.chan) for (auto it = q.begin(); it != q.end(); ++it) if (*it == m.get()) { q.erase(it); break; }
            return broke(sh, "rank " + std::to_string(R) + ": a Send of " + dstr(s->bytes, s->dtype) + " found no matching Recv within " +
                             std::to_string(timeout().count()) + " s");
        }
        if (rc == kSuccess && s->code != kSuccess) { rc = s->code; why = s->why; }
    }
    if (rc != kSuccess) return err(rc, why);
    return kSuccess;
}

}  // namespace

extern "C" {

struct ncclUniqueId { char internal[128]; };
typedef int ncclResult_t;
typedef void* ncclComm_t;

ncclResult_t ncclGetUniqueId(ncclUniqueId* id) {
    if (!id) return err(kInvalidArgument, "ncclGetUniqueId: NULL");
    memset(id, 0, sizeof *id);
    uint64_t key;
    { std::lock_guard<std::mutex> lk(g_mu); key = ((uint64_t)getpid() << 32) | g_next_id++; }
    memcpy(id->internal, "b9lb", 4);
    memcpy(id->internal + 8, &key, 8);
    return kSuccess;
}

ncclResult_t ncclCommInitRank(ncclComm_t* comm, int nranks, ncclUniqueId id, int rank) {
    if (!comm || nranks < 1 || rank < 0 || rank >= nranks) return err(kInvalidArgument, "ncclCommInitRank: bad argument");
    if (memcmp(id.internal, "b9lb", 4) != 0) return err(kInvalidArgument, "ncclCommInitRank: not an id ncclGetUniqueId of this library made");
    if (int rc = load_driver()) return rc;
    uint64_t key; memcpy(&key, id.internal + 8, 8);
    CUcontext ctx = nullptr;
    if (g_cu.CtxGetCurrent(&ctx)) return err(kUnhandledCudaError, "cuCtxGetCurrent failed");
    std::unique_lock<std::mutex> lk(g_mu);
    std::shared_ptr<Shared>& slot = g_comms[key];
    if (!slot) {
        slot = std::make_shared<Shared>();
        slot->world = nranks; slot->joined.assign(nranks, false);
        slot->ag_src.assign(nranks, nullptr); slot->ag_bytes.assign(nranks, 0); slot->ag_dtype.assign(nranks, 0);
        slot->chan.resize((size_t)nranks * nranks);
    }
    std::shared_ptr<Shared> sh = slot;
    if (sh->world != nranks) return err(kInvalidUsage, "ncclCommInitRank: world " + std::to_string(nranks) + " against " + std::to_string(sh->world) + " of the other ranks");
    if (sh->joined[rank]) return err(kInvalidUsage, "ncclCommInitRank: rank " + std::to_string(rank) + " joined twice");
    sh->joined[rank] = true; ++sh->n_joined; ++sh->n_alive;
    g_log[rank].push_back(LogEntry{kOpInit, -1, (uint64_t)nranks, {}});
    g_cv.notify_all();
    if (!wait_until(lk, *sh, [&] { return sh->n_joined == sh->world; })) {
        sh->joined[rank] = false; --sh->n_joined; --sh->n_alive;
        if (!sh->n_alive && g_comms[key] == sh) g_comms.erase(key);
        return err(kInternalError, "ncclCommInitRank: rank " + std::to_string(rank) + " waited " + std::to_string(timeout().count()) + " s for the other ranks");
    }
    *comm = new Comm{key, rank, nranks, sh, ctx};
    return kSuccess;
}

ncclResult_t ncclCommDestroy(ncclComm_t comm) {
    if (!comm) return kSuccess;
    Comm* c = (Comm*)comm;
    {
        std::lock_guard<std::mutex> lk(g_mu);
        if (--c->sh->n_alive == 0) {
            auto it = g_comms.find(c->key);
            if (it != g_comms.end() && it->second == c->sh) g_comms.erase(it);
        }
    }
    delete c;
    return kSuccess;
}

ncclResult_t ncclAllGather(const void* sendbuff, void* recvbuff, size_t count, int datatype, ncclComm_t comm, CUstream stream) {
    if (!comm) return err(kInvalidArgument, "ncclAllGather: NULL communicator");
    if (t_group.depth) return err(kInvalidUsage, "ncclAllGather inside a group: the loopback does not support it");
    const size_t ts = type_size(datatype);
    if (!ts) return err(kInvalidArgument, "ncclAllGather: unknown datatype " + std::to_string(datatype));
    Comm* c = (Comm*)comm;
    if (int rc = enter(c, stream)) return rc;
    const size_t bytes = count * ts;
    std::vector<uint64_t> words;
    if (bytes && bytes % 8 == 0 && bytes / 8 <= kLogWords) {
        words.resize(bytes / 8);
        if (g_cu.MemcpyDtoH(words.data(), (CUdeviceptr)sendbuff, bytes)) return err(kUnhandledCudaError, "cuMemcpyDtoH of the logged words failed");
    }
    log_call(c->rank, kOpAllGather, -1, bytes, std::move(words));
    return all_gather(c, sendbuff, recvbuff, bytes, datatype, stream);
}

ncclResult_t ncclGroupStart() { ++t_group.depth; return kSuccess; }

ncclResult_t ncclGroupEnd() {
    if (t_group.depth == 0) return err(kInvalidUsage, "ncclGroupEnd without ncclGroupStart");
    if (--t_group.depth) return kSuccess;
    Group g;
    std::swap(g, t_group);
    if (!g.bad.empty()) return err(kInvalidUsage, g.bad);
    if (!g.comm) return kSuccess;                             // an empty group
    if (int rc = enter(g.comm, g.stream)) return rc;
    return group_end(g.comm, g.ops, g.stream);
}

static ncclResult_t post(bool send, const void* src, void* dst, size_t count, int datatype, int peer, ncclComm_t comm, CUstream stream) {
    const char* name = send ? "ncclSend" : "ncclRecv";
    if (!comm) return err(kInvalidArgument, std::string(name) + ": NULL communicator");
    Comm* c = (Comm*)comm;
    const size_t ts = type_size(datatype);
    if (!ts) return err(kInvalidArgument, std::string(name) + ": unknown datatype " + std::to_string(datatype));
    if (peer < 0 || peer >= c->world || peer == c->rank) return err(kInvalidArgument, std::string(name) + ": peer " + std::to_string(peer) + " is not another rank");
    log_call(c->rank, send ? kOpSend : kOpRecv, peer, count * ts);
    const PostedOp op{send, src, dst, count * ts, datatype, peer};
    if (!t_group.depth) {                                     // outside a group: a group of one
        if (int rc = enter(c, stream)) return rc;
        return group_end(c, {op}, stream);
    }
    if (t_group.comm && t_group.comm != c) t_group.bad = "one group spans two communicators";
    if (t_group.comm && t_group.stream != stream) t_group.bad = "one group spans two streams";
    t_group.comm = c; t_group.stream = stream;
    t_group.ops.push_back(op);
    return kSuccess;
}

ncclResult_t ncclSend(const void* sendbuff, size_t count, int datatype, int peer, ncclComm_t comm, CUstream stream) {
    return post(true, sendbuff, nullptr, count, datatype, peer, comm, stream);
}

ncclResult_t ncclRecv(void* recvbuff, size_t count, int datatype, int peer, ncclComm_t comm, CUstream stream) {
    return post(false, nullptr, recvbuff, count, datatype, peer, comm, stream);
}

const char* ncclGetErrorString(ncclResult_t code) {
    if (!t_error.empty()) return t_error.c_str();
    switch (code) {
        case kSuccess: return "no error";
        case kInvalidArgument: return "invalid argument";
        case kInvalidUsage: return "invalid usage";
        default: return "loopback nccl error";
    }
}

// ---- the log (not NCCL API)
long lb_log_count(int rank) {
    std::lock_guard<std::mutex> lk(g_mu);
    auto it = g_log.find(rank);
    return it == g_log.end() ? 0 : (long)it->second.size();
}

// entry `index` of rank's log: its operation (1 init, 2 AllGather, 3 Send, 4 Recv), peer (-1: none), byte count and up
// to max_words logged words; returns how many words it has (copied: min(that, max_words)), or -1 if there is no such entry
int lb_log_get(int rank, long index, int* op, int* peer, uint64_t* bytes, uint64_t* words, int max_words) {
    std::lock_guard<std::mutex> lk(g_mu);
    auto it = g_log.find(rank);
    if (it == g_log.end() || index < 0 || (size_t)index >= it->second.size()) return -1;
    const LogEntry& e = it->second[(size_t)index];
    if (op) *op = e.op;
    if (peer) *peer = e.peer;
    if (bytes) *bytes = e.bytes;
    if (words) for (size_t k = 0; k < e.words.size() && (int)k < max_words; ++k) words[k] = e.words[k];
    return (int)e.words.size();
}

}  // extern "C"
