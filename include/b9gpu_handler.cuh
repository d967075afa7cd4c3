// b9gpu_handler.cuh — the device-side companion of b9gpu.h: write a drain handler of your own, compile it to an sm_90a
// cubin, and load it into a context with b9_handler_load.
//
// A handler is a struct with one function template. It receives args[0] of the call as the Python runner receives it
// (b9h::Arg) and writes one result value into a sink (Out):
//
//     #include "b9gpu_handler.cuh"
//     struct WordCount {                       // twin: def word_count(s, /): return len(s.split())
//         template <class Out> __device__ static int call(const b9h::Arg& s, Out& out) {
//             if (s.kind() != b9h::STR) return B9_EXC_ATTRIBUTE_ERROR;
//             ...                              // walk s.chars(), count runs of non-space code points
//             out.integer(n);
//             return 0;
//         }
//     };
//     B9_HANDLER(word_count, WordCount)       // the entry points b9_handler_load looks up
//
// call's return value: 0 = the handler returned (COMPLETE, with the value it wrote); one B9_EXC_* bit = it raised that
// class (ERROR, and b9_set_retry_policy applies to it as to a built-in handler's); B9H_DECLINE = the device does not
// answer this task (UNSUPPORTED: the host runs it on its CPU loop). Anything else is UNSUPPORTED too.
//
// The call rule is the built-in handlers': a positional-only one-parameter function. A call with anything but exactly one
// positional argument and no keyword arguments is ERROR / TypeError before `call` runs.
//
// `call` runs twice for a string result: once with a counting sink (status, length, falsiness), then, once the warp has
// reserved the record's bytes, with a writing sink. It must therefore be deterministic: a second pass that writes another
// number of bytes than the first counted makes the record UNSUPPORTED, and the writing sink never writes past the
// record's reservation. A number, bool or None result is written from the value the first pass stored.
//
// The result is rendered as the runner would:
//   b9_drain_launch            serialize_result(result) if result else None: json.dumps with its defaults (ensure_ascii,
//                              NaN / Infinity written); a falsy result (None, False, 0, 0.0, -0.0, "") is COMPLETE
//                              without result bytes
//   b9_endpoint_drain_launch   JSONResponse(result).body: compact, ensure_ascii=False, every result has a body; a
//                              non-finite float is UNSUPPORTED (allow_nan=False raises)
// A string holding a surrogate or a code point above U+10FFFF is UNSUPPORTED in both.
//
// This header is plain C++ behind CUDA qualifiers up to the kernel, which only nvcc sees: a host test can compile a
// handler and both sinks with g++ (tests/host_shim/user_handler_shim.cpp). Compile handlers with
// beta9_b200.build.compile_handlers, or by hand:
//     nvcc -cubin -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -I<repo>/include -o my.cubin my_handlers.cu
#pragma once
#include <stdint.h>
#include "b9gpu.h"
#include "../beta9_b200/csrc/json_device.cuh"
#include "../beta9_b200/csrc/f64_device.cuh"
#include "../beta9_b200/csrc/handler_seq.cuh"
#include "../beta9_b200/csrc/endpoint_device.cuh"
#include "../beta9_b200/csrc/task_msg.cuh"

#define B9H_DECLINE (-1)

namespace b9h {

enum Kind { STR = 0, INT, FLOAT, BOOL, NONE, LIST, DICT };
enum Rendering { TASK_QUEUE = 0, ENDPOINT = 1 };

__device__ __forceinline__ double mul_rn(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}

// The code points of a string argument as Go decoded them (invalid UTF-8 and lone surrogates are U+FFFD), or, for a
// TaskMessage record, as json.loads read them.
struct Chars {
    const uint8_t* p; uint32_t i, end;
    __device__ bool next(uint32_t& cp) { if (i >= end) return false; cp = b9::next_cp(p, i, end); return true; }
};

class Arg;
struct Items;

// A read-only view of one JSON value p[s, e) (validated) as the runner's json.loads made it. `unsure` is set when the
// handler asked something the device cannot answer exactly (the int / float type of a number whose float64 f64_parse
// cannot settle, an int outside int64): whatever the handler then returns, the record is UNSUPPORTED.
class Arg {
public:
    __device__ Arg() : p_(nullptr), s_(0), e_(0), unsure_(nullptr) {}
    __device__ Arg(const uint8_t* p, uint32_t s, uint32_t e, bool* unsure) : p_(p), s_(s), e_(e), unsure_(unsure) {}

    __device__ int kind() const {
        switch (p_[s_]) {
        case '"': return STR;
        case 't': case 'f': return BOOL;
        case 'n': return NONE;
        case '[': return LIST;
        case '{': return DICT;
        default: { long long i; double f; bool range = false; return num(&i, &f, &range) == FLOAT ? FLOAT : INT; }
        }
    }
    // STR: its code points
    __device__ Chars chars() const { Chars c; c.p = p_; c.i = s_ + 1; c.end = e_ - 1; return c; }
    // INT (in *i) or FLOAT (in *f) for a number token -- Go's text decides: digits only (an integral value below 1e21,
    // or zero) is a Python int -- and for a bool its int value; B9H_DECLINE for an int outside int64, a literal
    // f64_parse cannot settle, or any other kind
    __device__ int number(long long* i, double* f) const {
        bool range = false;
        const int k = num(i, f, &range);
        if (range) *unsure_ = true;
        return k;
    }
    __device__ Items items() const;
    // "", [], {}
    __device__ bool empty() const {
        const uint8_t c = p_[s_];
        if (c == '"') return e_ - s_ == 2;
        if (c == '[' || c == '{') return b9::only_ws(p_, s_ + 1, e_ - 1);
        return false;
    }

private:
    // number() without the range rule: *range = an int outside int64 (its kind is still INT)
    __device__ int num(long long* i, double* f, bool* range) const;
    const uint8_t* p_; uint32_t s_, e_; bool* unsure_;
};

// A list's elements, in order
struct Items {
    const uint8_t* p; uint32_t i, e; bool* unsure;
    __device__ bool next(Arg& x) {
        while (b9::is_ws(p[i])) ++i;
        if (p[i] == ']') return false;
        if (p[i] == ',') { ++i; while (b9::is_ws(p[i])) ++i; }
        uint32_t f = 0;
        const uint32_t vs = i;
        i = (uint32_t)b9::skip_value(p, i, e, f);
        x = Arg(p, vs, i, unsure);
        return true;
    }
};

__device__ inline Items Arg::items() const { Items it; it.p = p_; it.i = s_ + 1; it.e = e_; it.unsure = unsure_; return it; }

__device__ inline int Arg::num(long long* i, double* f, bool* range) const {
    const uint8_t d = p_[s_];
    if (d == 't' || d == 'f') { *i = d == 't' ? 1 : 0; return INT; }
    if (d != '-' && !b9::is_digit(d)) return B9H_DECLINE;
    uint32_t fl = 0; bool simple = false;
    b9::scan_number(p_, s_, e_, fl, &simple);
    if (simple) {                                    // <= 15 digits: exact in a float64, Go writes them back
        const bool neg = d == '-'; long long v = 0;
        for (uint32_t k = s_ + (neg ? 1 : 0); k < e_; ++k) v = v * 10 + (p_[k] - '0');
        *i = neg ? -v : v;
        return INT;
    }
    unsigned long long b = 0;
    if (!b9::f64_parse(p_, s_, e_, &b)) { *unsure_ = true; return B9H_DECLINE; }
    if (!b9::go_text_is_int(b)) { *f = b9::f64_from_bits(b); return FLOAT; }
    // the int is the value of Go's text: the shortest digits padded with zeros
    const b9::F64Dec dd = b9::f64_shortest(b);
    unsigned long long m = dd.f;
    const unsigned long long lim = dd.neg ? 9223372036854775808ull : 9223372036854775807ull;
    for (int z = dd.n; z < dd.dp && m <= lim; ++z) m = (m > lim / 10u) ? lim + 1u : m * 10u;
    if (dd.cls == 1) { *i = 0; return INT; }
    if (m > lim) { *range = true; return B9H_DECLINE; }
    *i = dd.neg ? (long long)(0ull - m) : (long long)m;
    return INT;
}

// ---- the sinks ------------------------------------------------------------------------------------------------------
// What the first pass learns about the one value the handler writes
enum ValueKind : uint8_t { VK_UNSET = 0, VK_NONE, VK_BOOL, VK_INT, VK_FLOAT, VK_STR, VK_BAD };

template <int R> __device__ __forceinline__ uint32_t str_cp_len(uint32_t cp) { return R == ENDPOINT ? b9::ep_emit_len(cp) : b9::py_escaped_len(cp); }
template <int R> __device__ __forceinline__ uint32_t str_cp_write(uint32_t cp, uint8_t* o) { return R == ENDPOINT ? b9::ep_emit(cp, o) : b9::py_emit(cp, o); }
__device__ __forceinline__ bool cp_ok(uint32_t cp) { return cp <= 0x10FFFFu && (cp - 0xD800u) >= 0x800u; }

// Pass 1: counts the string's bytes and keeps a number's value. vk = VK_BAD for anything the renderings cannot write:
// a second value, a string left open, a surrogate or a code point past U+10FFFF.
template <int R> struct CountSink {
    uint8_t vk = VK_UNSET; bool open = false;
    uint32_t n = 0, cps = 0;
    long long v = 0;                 // VK_BOOL / VK_INT; VK_FLOAT: the double's bits
    __device__ bool start(uint8_t k) { if (vk != VK_UNSET || open) { vk = VK_BAD; open = false; return false; } vk = k; return true; }
    __device__ void none() { start(VK_NONE); }
    __device__ void boolean(bool b) { if (start(VK_BOOL)) v = b ? 1 : 0; }
    __device__ void integer(long long x) { if (start(VK_INT)) v = x; }
    __device__ void real(double d) { if (start(VK_FLOAT)) v = (long long)b9::f64_to_bits(d); }
    __device__ void str_begin() { if (start(VK_STR)) { open = true; n = 2; cps = 0; } }
    __device__ void cp(uint32_t c) {
        if (!open) { vk = VK_BAD; return; }
        if (!cp_ok(c)) { vk = VK_BAD; open = false; return; }
        n += str_cp_len<R>(c); ++cps;
    }
    __device__ void str_end() { if (!open) vk = VK_BAD; open = false; }
};

// Pass 2 of a string result: writes at most `cap` bytes at o
template <int R> struct WriteSink {
    uint8_t* o; uint32_t cap, n = 0; bool ok = true, open = false, done = false;
    __device__ WriteSink(uint8_t* out, uint32_t c) : o(out), cap(c) {}
    __device__ void bad() { ok = false; }
    __device__ void none() { bad(); }
    __device__ void boolean(bool) { bad(); }
    __device__ void integer(long long) { bad(); }
    __device__ void real(double) { bad(); }
    __device__ void str_begin() { if (done || open || cap < 2) { bad(); return; } o[0] = '"'; n = 1; open = true; }
    __device__ void cp(uint32_t c) {
        if (!ok || !open || !cp_ok(c)) { bad(); return; }
        if (n + str_cp_len<R>(c) + 1 > cap) { bad(); return; }       // (+1: the closing quote)
        n += str_cp_write<R>(c, o + n);
    }
    __device__ void str_end() { if (!ok || !open) { bad(); return; } o[n++] = '"'; open = false; done = true; }
};

// ---- phase A and B around a handler ---------------------------------------------------------------------------------
struct UserRec {
    uint32_t src_off, src_len;   // args[0]'s token: pass 2 of a string result calls the handler on it again
    uint32_t out_len;
    uint8_t status, has, vk;
    long long value;             // ERROR: the exception class (one B9_EXC_* bit); else the number pass 1 stored
};

// The tasks a rendering answers, parsed: task-queue: an SDK payload (flags 0), an HTTP body (B9_TF_HTTP_BODY) or a
// TaskMessage record of the slot's id (B9_TF_TASK_MSG); endpoint: exactly B9_TF_HTTP_BODY (endpoint_accepts). Anything
// else (B9_TF_PICKLE, combinations) is UNSUPPORTED. `id`: the slot's 16 raw id bytes (read only for a record).
template <int R> __device__ inline b9::Parsed user_parse(const uint8_t* p, uint32_t n, uint32_t flags, const uint8_t* id) {
    b9::Parsed pr;
    if (R == ENDPOINT ? b9::endpoint_accepts(flags) : (flags == 0 || flags == B9_TF_HTTP_BODY)) return b9::parse_payload(p, n, flags != 0);
    if (R == TASK_QUEUE && flags == B9_TF_TASK_MSG) return b9::parse_task_msg(p, n, id);
    pr.status = b9::ST_UNSUPPORTED; pr.nargs = 0; pr.a0_off = pr.a0_len = 0;
    return pr;
}

// record length of a number / bool / None result (o == nullptr), or its bytes
template <int R> __device__ inline uint32_t scalar_write(uint8_t vk, long long v, uint8_t* o) {
    switch (vk) {
    case VK_NONE: if (o) { o[0] = 'n'; o[1] = 'u'; o[2] = 'l'; o[3] = 'l'; } return 4;
    case VK_BOOL:
        if (v) { if (o) { o[0] = 't'; o[1] = 'r'; o[2] = 'u'; o[3] = 'e'; } return 4; }
        if (o) { o[0] = 'f'; o[1] = 'a'; o[2] = 'l'; o[3] = 's'; o[4] = 'e'; } return 5;
    case VK_INT: {
        const unsigned long long mag = v < 0 ? 0ull - (unsigned long long)v : (unsigned long long)v;
        const uint32_t l = b9::dec_len_u64(mag);
        if (o) { if (v < 0) *o++ = '-'; b9::write_dec(o, mag, l); }
        return l + (v < 0 ? 1u : 0u);
    }
    default: return b9::py_json_float((unsigned long long)v, o);     // VK_FLOAT
    }
}

// Phase A: status, has and the record's length; `pr` is user_parse's
template <class H, int R> __device__ inline void user_phase_a(const uint8_t* p, const b9::Parsed& pr, UserRec& rec) {
    rec.src_off = 0; rec.src_len = 0; rec.out_len = 0; rec.has = 0; rec.vk = VK_UNSET; rec.value = 0;
    if (pr.status != b9::ST_OK) { rec.status = pr.status; return; }
    if (pr.nargs != 1 || pr.kwargs_nonempty) { rec.status = b9::ST_ERROR; rec.value = B9_EXC_TYPE_ERROR; return; }
    bool unsure = false;
    const Arg arg(p, pr.a0_off, pr.a0_off + pr.a0_len, &unsure);
    CountSink<R> out;
    const int ret = H::call(arg, out);
    rec.status = b9::ST_UNSUPPORTED;
    if (unsure) return;
    if (ret != 0) {
        if (ret > 0 && ret <= (int)B9_EXC_ALL && !(ret & (ret - 1))) { rec.status = b9::ST_ERROR; rec.value = ret; }
        return;
    }
    if (out.vk == VK_UNSET || out.vk == VK_BAD || out.open) return;
    if (out.vk == VK_FLOAT && R == ENDPOINT && (((unsigned long long)out.v >> 52) & 0x7FFull) == 0x7FFull) return;   // allow_nan=False
    rec.status = b9::ST_OK;
    rec.vk = out.vk; rec.value = out.v;
    if (R == TASK_QUEUE) {                                        // `serialize_result(result) if result else None`
        const bool falsy = out.vk == VK_NONE || ((out.vk == VK_BOOL || out.vk == VK_INT) && out.v == 0) ||
                           (out.vk == VK_FLOAT && ((unsigned long long)out.v << 1) == 0) || (out.vk == VK_STR && out.cps == 0);
        if (falsy) return;
    }
    rec.has = 1;
    rec.src_off = pr.a0_off; rec.src_len = pr.a0_len;
    rec.out_len = out.vk == VK_STR ? out.n : scalar_write<R>(out.vk, out.v, nullptr);
}

// Phase B: writes the record's rec.out_len bytes at o. false: the handler's second pass did not write what its first
// counted (the bytes at o are then not a record, and the caller makes it UNSUPPORTED).
template <class H, int R> __device__ inline bool user_phase_b(const uint8_t* p, const UserRec& rec, uint8_t* o) {
    if (rec.vk != VK_STR) { scalar_write<R>(rec.vk, rec.value, o); return true; }
    bool unsure = false;
    const Arg arg(p, rec.src_off, rec.src_off + rec.src_len, &unsure);
    WriteSink<R> out(o, rec.out_len);
    const int ret = H::call(arg, out);
    return ret == 0 && !unsure && out.ok && out.done && out.n == rec.out_len;
}

}  // namespace b9h

#ifdef __CUDACC__
#include "../beta9_b200/csrc/user_drain.cuh"
#define B9H_ENTRY_(v, kind, name) b9h_v##v##_##kind##_##name
#define B9H_ENTRY(v, kind, name) B9H_ENTRY_(v, kind, name)
// The two entry points of handler struct H under `name` (an identifier): the task-queue drain and the endpoint drain.
// Their names carry B9_HANDLER_ABI_VERSION (drain_kernel.cuh): b9_handler_load finds no entry in an image built against
// another version.
#define B9_HANDLER(name, H)                                                                                                   \
    extern "C" __global__ void __launch_bounds__(b9::UD_WARPS * 32) B9H_ENTRY(B9_HANDLER_ABI_VERSION, tq, name)(b9::DrainArgs a) { \
        b9::user_drain<H, b9h::TASK_QUEUE>(a);                                                                                 \
    }                                                                                                                         \
    extern "C" __global__ void __launch_bounds__(b9::UD_WARPS * 32) B9H_ENTRY(B9_HANDLER_ABI_VERSION, ep, name)(b9::DrainArgs a) { \
        b9::user_drain<H, b9h::ENDPOINT>(a);                                                                                   \
    }
#else
#define B9_HANDLER(name, H)
#endif
