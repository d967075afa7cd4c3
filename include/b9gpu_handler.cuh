// b9gpu_handler.cuh — the device-side companion of b9gpu.h: write a drain handler of your own, compile it to an sm_90a
// cubin, and load it into a context with b9_handler_load.
//
// A handler is a struct with one function template. It receives args[0] of the call as the Python runner receives it
// (b9h::Arg), or the whole call bound to a declared signature (b9h::Call, below), and writes one result value into a
// sink (Out):
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
// A handler may instead declare its Python signature; `call` then receives the bound call:
//
//     struct Greet {                           // twin: def greet(name, greeting="Hello", *, punct="!"): ...
//         B9H_SIGNATURE(B9H_POS_OR_KW("name"), B9H_POS_OR_KW_OPT("greeting"), B9H_KW_ONLY_OPT("punct"));
//         template <class Out> __device__ static int call(const b9h::Call& c, Out& out);   // c[i], c.has(i), c.rest()
//     };
//
// Parameters (at most 8, in `def` order) are B9H_POS_ONLY, B9H_POS_OR_KW, B9H_VAR_POS (*args: c.rest() iterates the
// surplus positionals) and B9H_KW_ONLY, each required or _OPT. An optional parameter not passed reads as absent
// (c.has(i) == false) and the handler applies its default. Names are ASCII identifiers; `context` (the runner's
// FunctionContext) is refused; static_asserts check both, and Python's parameter order. The call is bound as CPython binds
// handler(*args, **kwargs): every failure (too many positionals, a missing required parameter, an unexpected keyword, a
// positional-only name passed as a keyword, multiple values for one parameter) is ERROR / TypeError before `call` runs.
// The arguments are the runner's: an SDK payload's args / kwargs as Go's struct decode kept them (kwargs objects that
// Go would merge are UNSUPPORTED); an HTTP body's as SerializeHttpPayload makes them (a last "args" list is the
// positionals, a last "kwargs" object alone is the kwargs, else the body's other top-level keys are); a record's own.
// Keywords match by decoded code points, the last of duplicate keys deciding. Arg::get reads a dict by key the same way.
//
// The sink takes one value: none(), boolean(b), integer(i), real(d), a string (str_begin(), cp(c) per code point,
// str_end()), an argument passed through (value(a): the bytes the built-in identity handler writes for it), or a
// container. A list (list_begin() ... list_end()) holds any number of values; a dict (dict_begin() ... dict_end())
// alternates a key, always a string, and its value:
//
//     out.dict_begin();                        // twin: return {"type": "str", "value": x}
//     out.str_begin(); put("type"); out.str_end();  out.str_begin(); put("str"); out.str_end();
//     out.str_begin(); put("value"); out.str_end(); out.value(x);
//     out.dict_end();
//
// Containers nest at most 16 deep and a dict holds at most 64 members, with no two keys equal (Python would keep one).
// Past those limits the record is UNSUPPORTED, as it is for a close that matches no open container, a non-string key,
// a dict closed after its key, a container call inside an open string, a result left open, and a value(a) whose
// argument identity declines (nesting past 16, more than 64 members, a number f64_parse cannot settle).
//
// `call` runs twice for a string, container or value() result: once with a counting sink (status, length, falsiness),
// then, once the warp has reserved the record's bytes, with a writing sink. It must therefore be deterministic: a second
// pass that writes another number of bytes than the first counted makes the record UNSUPPORTED, and the writing sink
// never writes past the record's reservation. A number, bool or None result is written from the value the first pass
// stored.
//
// The result is rendered as the runner would:
//   b9_drain_launch            serialize_result(result) if result else None: json.dumps with its defaults (ensure_ascii,
//                              ", " and ": ", NaN / Infinity written, dict keys in the order written); a falsy result
//                              (None, False, 0, 0.0, -0.0, "", [], {}, or a value() identity drops) is COMPLETE
//                              without result bytes
//   b9_endpoint_drain_launch   JSONResponse(result).body: compact, ensure_ascii=False, every result has a body; a
//                              non-finite float at any depth is UNSUPPORTED (allow_nan=False raises)
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
__device__ __forceinline__ double add_rn(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
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
template <int R> struct CountSink;
template <int R> struct WriteSink;

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
    // DICT: the value of `key` as the runner's dict holds it (of duplicate keys the last one; keys compared by their
    // decoded code points); false when the dict has no such key, or this is not a dict. `key` is a STR Arg (any other
    // kind matches nothing) or a NUL-terminated UTF-8 string.
    __device__ bool get(const Arg& key, Arg& out) const;
    __device__ bool get(const char* key, Arg& out) const;
    // "", [], {}
    __device__ bool empty() const {
        const uint8_t c = p_[s_];
        if (c == '"') return e_ - s_ == 2;
        if (c == '[' || c == '{') return b9::only_ws(p_, s_ + 1, e_ - 1);
        return false;
    }

private:
    friend class Call;
    template <int> friend struct CountSink;
    template <int> friend struct WriteSink;
    // number() without the range rule: *range = an int outside int64 (its kind is still INT)
    __device__ int num(long long* i, double* f, bool* range) const;
    // the sinks' value(a): identity's bytes for the token in rendering R (o == nullptr: their count), -1 where
    // py_value_json / ep_value_json decline
    template <int R> __device__ int64_t json(uint8_t* o) const {
        return R == ENDPOINT ? b9::ep_value_json(p_, s_, e_, o) : b9::py_value_json(p_, s_, e_, o);
    }
    // Python's truth value of the token: what the built-in identity handler drops as falsy
    __device__ bool truthy() const {
        switch (p_[s_]) {
        case '"': return e_ - s_ > 2;
        case 't': return true;
        case 'n': case 'f': return false;
        case '[': case '{': return !empty();
        default: { unsigned long long b = 0; b9::f64_parse(p_, s_, e_, &b); return (b << 1) != 0; }
        }
    }
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

// The members of a validated object whose body starts at i (just past its '{') and which ends before e, in text order:
// key body [ks, ke) (between the quotes, still escaped), value [vs, ve). An internal helper of Arg::get and Call::bind,
// not part of the handler contract: it walks the text, duplicates included, while the runner's dict holds Go's sorted,
// de-duplicated keys; a handler reads a dict through Arg::get.
struct Members {
    const uint8_t* p; uint32_t i, e;
    __device__ bool next(uint32_t& ks, uint32_t& ke, uint32_t& vs, uint32_t& ve) {
        while (b9::is_ws(p[i])) ++i;
        if (p[i] == '}') return false;
        if (p[i] == ',') { ++i; while (b9::is_ws(p[i])) ++i; }
        uint32_t f = 0;
        ks = i + 1;
        i = (uint32_t)b9::scan_string(p, i, e, f);
        ke = i - 1;
        while (b9::is_ws(p[i]) || p[i] == ':') ++i;
        vs = i;
        i = (uint32_t)b9::skip_value(p, i, e, f);
        ve = i;
        return true;
    }
};

// Does the decoded key body p[ks, ke) equal the UTF-8 bytes s[0, n)? Each decoded code point is encoded back to UTF-8
// and compared, so a name or a C-string key is never decoded itself.
__device__ inline bool key_eq(const uint8_t* p, uint32_t ks, uint32_t ke, const uint8_t* s, uint32_t n) {
    uint32_t j = 0;
    while (ks < ke) {
        const uint32_t cp = b9::next_cp(p, ks, ke);
        const uint32_t l = cp < 0x80 ? 1u : cp < 0x800 ? 2u : cp < 0x10000 ? 3u : 4u;
        if (j + l > n) return false;
        if (l == 1) { if (s[j] != cp) return false; }
        else {
            const uint8_t lead = l == 2 ? 0xC0 : l == 3 ? 0xE0 : 0xF0;
            if (s[j] != (uint8_t)(lead | (cp >> (6 * (l - 1))))) return false;
            for (uint32_t k = 1; k < l; ++k) if (s[j + k] != (uint8_t)(0x80 | ((cp >> (6 * (l - 1 - k))) & 0x3F))) return false;
        }
        j += l;
    }
    return j == n;
}

// ... or the decoded string body q[qs, qe)
__device__ inline bool key_eq(const uint8_t* p, uint32_t ks, uint32_t ke, const uint8_t* q, uint32_t qs, uint32_t qe) {
    while (ks < ke && qs < qe) if (b9::next_cp(p, ks, ke) != b9::next_cp(q, qs, qe)) return false;
    return ks >= ke && qs >= qe;
}

__host__ __device__ constexpr uint32_t cstr_len(const char* s) { uint32_t n = 0; while (s[n]) ++n; return n; }

__device__ inline bool Arg::get(const Arg& key, Arg& out) const {
    if (p_[s_] != '{' || key.p_[key.s_] != '"') return false;
    Members m{p_, s_ + 1, e_};
    uint32_t ks, ke, vs, ve;
    bool found = false;
    while (m.next(ks, ke, vs, ve))
        if (key_eq(p_, ks, ke, key.p_, key.s_ + 1, key.e_ - 1)) { out = Arg(p_, vs, ve, unsure_); found = true; }
    return found;
}

__device__ inline bool Arg::get(const char* key, Arg& out) const {
    if (p_[s_] != '{') return false;
    const uint32_t n = cstr_len(key);
    Members m{p_, s_ + 1, e_};
    uint32_t ks, ke, vs, ve;
    bool found = false;
    while (m.next(ks, ke, vs, ve))
        if (key_eq(p_, ks, ke, (const uint8_t*)key, n)) { out = Arg(p_, vs, ve, unsure_); found = true; }
    return found;
}

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
// What the first pass learns about the one value the handler writes: VK_LIST / VK_DICT, a container it built;
// VK_VALUE, an argument it passed through with value()
enum ValueKind : uint8_t { VK_UNSET = 0, VK_NONE, VK_BOOL, VK_INT, VK_FLOAT, VK_STR, VK_BAD, VK_LIST, VK_DICT, VK_VALUE };

template <int R> __device__ __forceinline__ uint32_t str_cp_len(uint32_t cp) { return R == ENDPOINT ? b9::ep_emit_len(cp) : b9::py_escaped_len(cp); }
template <int R> __device__ __forceinline__ uint32_t str_cp_write(uint32_t cp, uint8_t* o) { return R == ENDPOINT ? b9::ep_emit(cp, o) : b9::py_emit(cp, o); }
__device__ __forceinline__ bool cp_ok(uint32_t cp) { return cp <= 0x10FFFFu && (cp - 0xD800u) >= 0x800u; }
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

__device__ __forceinline__ bool nonfinite(long long bits) { return (((unsigned long long)bits >> 52) & 0x7FFull) == 0x7FFull; }
// the separators of a rendering: json.dumps's ", " and ": ", JSONResponse's "," and ":"
template <int R> __host__ __device__ constexpr uint32_t sep_len() { return R == ENDPOINT ? 1u : 2u; }

// Containers (list_begin ... list_end, dict_begin ... dict_end) nest at most PY_VALUE_MAX_DEPTH deep. Both sinks keep
// one bit per open container, bit d for depth d: `dict` (a dict, else a list), `started` (an item or member written:
// the next one needs a separator) and `keyed` (a dict whose key is written and whose value is due). A dict's members
// alternate a str key (str_begin / cp / str_end) and a value; key_open: the open string is a key.

// Pass 1: counts the result's bytes and keeps a number's value. vk = VK_BAD for anything the renderings cannot write:
// a second value, a string or container left open, a surrogate or a code point past U+10FFFF, a close that matches no
// open container, a key that is not a string, a dict closed after a key, a 17th open container, a value() its
// rendering declines, a non-finite float inside a container of the endpoint rendering.
template <int R> struct CountSink {
    uint8_t vk = VK_UNSET; bool open = false;
    uint32_t n = 0, cps = 0;
    long long v = 0;                 // VK_BOOL / VK_INT; VK_FLOAT: the double's bits
    int depth = 0; uint32_t dict = 0, started = 0, keyed = 0; bool key_open = false;
    bool truthy = false;             // VK_LIST / VK_DICT / VK_VALUE: the result is not empty (falsy)
    __device__ bool start(uint8_t k) { if (vk != VK_UNSET || open) { vk = VK_BAD; open = false; return false; } vk = k; return true; }
    // a value or key begins inside the innermost container; false when that breaks a rule (vk is then VK_BAD)
    __device__ bool item(bool str) {
        if (vk == VK_BAD) return false;
        const uint32_t bit = 1u << (depth - 1);
        if (open || ((dict & bit) && !(keyed & bit) && !str)) { vk = VK_BAD; open = false; return false; }
        if (keyed & bit) { keyed &= ~bit; n += sep_len<R>(); return true; }
        if (started & bit) n += sep_len<R>();
        started |= bit;
        key_open = (dict & bit) != 0;
        return true;
    }
    __device__ void scalar(uint8_t k, long long x) {
        if (!item(false)) return;
        if (R == ENDPOINT && k == VK_FLOAT && nonfinite(x)) { vk = VK_BAD; return; }      // allow_nan=False
        n += scalar_write<R>(k, x, nullptr);
    }
    __device__ void none() { if (depth) scalar(VK_NONE, 0); else start(VK_NONE); }
    __device__ void boolean(bool b) { if (depth) scalar(VK_BOOL, b ? 1 : 0); else if (start(VK_BOOL)) v = b ? 1 : 0; }
    __device__ void integer(long long x) { if (depth) scalar(VK_INT, x); else if (start(VK_INT)) v = x; }
    __device__ void real(double d) {
        if (depth) scalar(VK_FLOAT, (long long)b9::f64_to_bits(d));
        else if (start(VK_FLOAT)) v = (long long)b9::f64_to_bits(d);
    }
    __device__ void str_begin() {
        if (depth) { if (item(true)) { open = true; n += 2; } return; }
        if (start(VK_STR)) { open = true; n = 2; cps = 0; }
    }
    __device__ void cp(uint32_t c) {
        if (!open) { vk = VK_BAD; return; }
        if (!cp_ok(c)) { vk = VK_BAD; open = false; return; }
        n += str_cp_len<R>(c); ++cps;
    }
    __device__ void str_end() {
        if (!open) vk = VK_BAD;
        else if (key_open) { keyed |= 1u << (depth - 1); key_open = false; }
        open = false;
    }
    __device__ void begin(uint8_t k) {
        if (depth) { if (!item(false)) return; }
        else if (!start(k)) return;
        if (depth == b9::PY_VALUE_MAX_DEPTH) { vk = VK_BAD; return; }
        const uint32_t bit = 1u << depth;
        dict = k == VK_DICT ? dict | bit : dict & ~bit; started &= ~bit; keyed &= ~bit;
        ++depth; ++n;
    }
    __device__ void end(uint8_t k) {
        if (vk == VK_BAD) return;
        const uint32_t bit = depth ? 1u << (depth - 1) : 0u;
        if (open || !depth || ((dict & bit) != 0) != (k == VK_DICT) || (keyed & bit)) { vk = VK_BAD; open = false; return; }
        --depth; ++n;
        if (!depth) truthy = (started & 1u) != 0;
    }
    __device__ void list_begin() { begin(VK_LIST); }
    __device__ void list_end() { end(VK_LIST); }
    __device__ void dict_begin() { begin(VK_DICT); }
    __device__ void dict_end() { end(VK_DICT); }
    __device__ void value(const Arg& a) {
        if (depth) { if (!item(false)) return; }
        else if (!start(VK_VALUE)) return;
        const int64_t l = a.json<R>(nullptr);
        if (l < 0) { vk = VK_BAD; return; }
        n += (uint32_t)l;
        if (!depth) truthy = a.truthy();
    }
};

// Pass 2 of a string, container or value() result: writes at most `cap` bytes at o. A number, bool or None is written
// only inside a container (at the top level, from the value pass 1 stored). dict_end checks the member keys it has
// just written: more than PY_VALUE_MAX_MEMBERS, or two equal ones (the writers are canonical: equal bytes are equal
// code points), fail the pass.
template <int R> struct WriteSink {
    uint8_t* o; uint32_t cap, n = 0; bool ok = true, open = false, done = false;
    int depth = 0; uint32_t dict = 0, started = 0, keyed = 0; bool key_open = false;
    uint32_t at[b9::PY_VALUE_MAX_DEPTH];     // where each open container's bracket is
    __device__ WriteSink(uint8_t* out, uint32_t c) : o(out), cap(c) {}
    __device__ void bad() { ok = false; }
    __device__ bool room(uint32_t l) { if (n + l > cap) { bad(); return false; } return true; }
    __device__ bool item(bool str) {
        const uint32_t bit = 1u << (depth - 1);
        if (!ok || open || ((dict & bit) && !(keyed & bit) && !str)) { bad(); return false; }
        if ((keyed & bit) || (started & bit)) {
            if (!room(sep_len<R>())) return false;
            o[n] = (keyed & bit) ? ':' : ',';
            if (R == TASK_QUEUE) o[n + 1] = ' ';
            n += sep_len<R>();
            if (keyed & bit) { keyed &= ~bit; return true; }
        }
        started |= bit;
        key_open = (dict & bit) != 0;
        return true;
    }
    __device__ void scalar(uint8_t k, long long x) {
        if (!depth) { bad(); return; }
        if (!item(false)) return;
        if (R == ENDPOINT && k == VK_FLOAT && nonfinite(x)) { bad(); return; }
        if (room(scalar_write<R>(k, x, nullptr))) n += scalar_write<R>(k, x, o + n);
    }
    __device__ void none() { scalar(VK_NONE, 0); }
    __device__ void boolean(bool b) { scalar(VK_BOOL, b ? 1 : 0); }
    __device__ void integer(long long x) { scalar(VK_INT, x); }
    __device__ void real(double d) { scalar(VK_FLOAT, (long long)b9::f64_to_bits(d)); }
    __device__ void str_begin() {
        if (depth) { if (item(true) && room(2)) { o[n++] = '"'; open = true; } return; }     // (2: the closing quote)
        if (done || open || cap < 2) { bad(); return; } o[0] = '"'; n = 1; open = true;
    }
    __device__ void cp(uint32_t c) {
        if (!ok || !open || !cp_ok(c)) { bad(); return; }
        if (n + str_cp_len<R>(c) + 1 > cap) { bad(); return; }       // (+1: the closing quote)
        n += str_cp_write<R>(c, o + n);
    }
    __device__ void str_end() {
        if (!ok || !open) { bad(); return; }
        o[n++] = '"'; open = false;
        if (!depth) done = true;
        else if (key_open) { keyed |= 1u << (depth - 1); key_open = false; }
    }
    __device__ void begin(bool is_dict) {
        if (depth) { if (!item(false)) return; }
        else if (done || open) { bad(); return; }
        if (depth == b9::PY_VALUE_MAX_DEPTH || !room(1)) { bad(); return; }
        const uint32_t bit = 1u << depth;
        dict = is_dict ? dict | bit : dict & ~bit; started &= ~bit; keyed &= ~bit;
        at[depth++] = n;
        o[n++] = is_dict ? '{' : '[';
    }
    __device__ void end(bool is_dict) {
        const uint32_t bit = depth ? 1u << (depth - 1) : 0u;
        if (!ok || open || !depth || ((dict & bit) != 0) != is_dict || (keyed & bit)) { bad(); return; }
        if (is_dict && !keys_ok(at[depth - 1] + 1)) { bad(); return; }
        if (!room(1)) return;
        o[n++] = is_dict ? '}' : ']';
        if (!--depth) done = true;
    }
    __device__ void list_begin() { begin(false); }
    __device__ void list_end() { end(false); }
    __device__ void dict_begin() { begin(true); }
    __device__ void dict_end() { end(true); }
    __device__ void value(const Arg& a) {
        if (depth) { if (!item(false)) return; }
        else if (done || open) { bad(); return; }
        const int64_t l = a.json<R>(nullptr);
        if (l < 0 || !room((uint32_t)l)) { bad(); return; }
        n += (uint32_t)a.json<R>(o + n);
        if (!depth) done = true;
    }

    // the bytes this sink wrote: one string o[i] == '"' ... (past its closing quote), one value (to the ',' or the end e
    // that follows it), the next member key of a dict body (i: its start or the end of a value; [ks, ke): between the
    // quotes; false at e)
    __device__ uint32_t skip_str(uint32_t i, uint32_t e) const {
        for (++i; i < e && o[i] != '"'; ++i) if (o[i] == '\\') ++i;
        return i + 1;
    }
    __device__ uint32_t skip_value(uint32_t i, uint32_t e) const {
        int d = 0;
        while (i < e) {
            const uint8_t c = o[i];
            if (c == '"') { i = skip_str(i, e); continue; }
            if (c == '[' || c == '{') ++d;
            else if (c == ']' || c == '}') --d;
            else if (c == ',' && d == 0) return i;
            ++i;
        }
        return i;
    }
    __device__ bool next_key(uint32_t& i, uint32_t e, uint32_t& ks, uint32_t& ke) const {
        while (i < e && (o[i] == ',' || o[i] == ' ')) ++i;
        if (i >= e) return false;
        ks = i + 1;
        i = skip_str(i, e);
        ke = i - 1;
        i = skip_value(i + sep_len<R>(), e);
        return true;
    }
    // the members of the dict body o[s, n): at most PY_VALUE_MAX_MEMBERS, no two keys equal
    __device__ bool keys_ok(uint32_t s) const {
        uint32_t i = s, ks, ke, members = 0;
        while (next_key(i, n, ks, ke)) {
            if (++members > b9::PY_VALUE_MAX_MEMBERS) return false;
            uint32_t j = s, js, je;
            while (next_key(j, ks - 1, js, je)) {
                if (je - js != ke - ks) continue;
                uint32_t k = 0;
                while (k < ke - ks && o[js + k] == o[ks + k]) ++k;
                if (k == ke - ks) return false;
            }
        }
        return true;
    }
};

// ---- phase A and B around a handler ---------------------------------------------------------------------------------
struct UserRec {
    uint32_t src_off, src_len;   // args[0]'s token: pass 2 of a string or container result calls the handler on it again
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

// What `call` returned (ret), whether it asked something the device cannot answer (unsure) and what it wrote (out) as
// the record's status, has and length: the rules of user_phase_a below, for a handler with a signature (user_phase_a
// keeps its own copy so that the one-Arg entries compile to the same code as before signatures existed).
template <int R> __device__ inline bool phase_a_settle(int ret, bool unsure, const CountSink<R>& out, UserRec& rec) {
    rec.status = b9::ST_UNSUPPORTED;
    if (unsure) return false;
    if (ret != 0) {
        if (ret > 0 && ret <= (int)B9_EXC_ALL && !(ret & (ret - 1))) { rec.status = b9::ST_ERROR; rec.value = ret; }
        return false;
    }
    if (out.vk == VK_UNSET || out.vk == VK_BAD || out.open || out.depth) return false;
    if (out.vk == VK_FLOAT && R == ENDPOINT && (((unsigned long long)out.v >> 52) & 0x7FFull) == 0x7FFull) return false;   // allow_nan=False
    rec.status = b9::ST_OK;
    rec.vk = out.vk; rec.value = out.v;
    if (R == TASK_QUEUE) {                                        // `serialize_result(result) if result else None`
        const bool falsy = out.vk == VK_NONE || ((out.vk == VK_BOOL || out.vk == VK_INT) && out.v == 0) ||
                           (out.vk == VK_FLOAT && ((unsigned long long)out.v << 1) == 0) || (out.vk == VK_STR && out.cps == 0) ||
                           (out.vk >= VK_LIST && !out.truthy);
        if (falsy) return false;
    }
    rec.has = 1;
    rec.out_len = out.vk >= VK_STR ? out.n : scalar_write<R>(out.vk, out.v, nullptr);
    return true;
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
    if (out.vk == VK_UNSET || out.vk == VK_BAD || out.open || out.depth) return;
    if (out.vk == VK_FLOAT && R == ENDPOINT && (((unsigned long long)out.v >> 52) & 0x7FFull) == 0x7FFull) return;   // allow_nan=False
    rec.status = b9::ST_OK;
    rec.vk = out.vk; rec.value = out.v;
    if (R == TASK_QUEUE) {                                        // `serialize_result(result) if result else None`
        const bool falsy = out.vk == VK_NONE || ((out.vk == VK_BOOL || out.vk == VK_INT) && out.v == 0) ||
                           (out.vk == VK_FLOAT && ((unsigned long long)out.v << 1) == 0) || (out.vk == VK_STR && out.cps == 0) ||
                           (out.vk >= VK_LIST && !out.truthy);
        if (falsy) return;
    }
    rec.has = 1;
    rec.src_off = pr.a0_off; rec.src_len = pr.a0_len;
    rec.out_len = out.vk >= VK_STR ? out.n : scalar_write<R>(out.vk, out.v, nullptr);
}

// Phase B: writes the record's rec.out_len bytes at o. false: the handler's second pass did not write what its first
// counted (the bytes at o are then not a record, and the caller makes it UNSUPPORTED).
template <class H, int R> __device__ inline bool user_phase_b(const uint8_t* p, const UserRec& rec, uint8_t* o) {
    if (rec.vk < VK_STR) { scalar_write<R>(rec.vk, rec.value, o); return true; }
    bool unsure = false;
    const Arg arg(p, rec.src_off, rec.src_off + rec.src_len, &unsure);
    WriteSink<R> out(o, rec.out_len);
    const int ret = H::call(arg, out);
    return ret == 0 && !unsure && out.ok && out.done && out.n == rec.out_len;
}

// ---- declared signatures ------------------------------------------------------------------------------------------
// A handler that declares its Python signature with B9H_SIGNATURE receives the bound call (b9h::Call) instead of one Arg.
enum ParamKind : uint8_t { P_POS_ONLY = 0, P_POS_OR_KW, P_VAR_POS, P_KW_ONLY };
constexpr int MAX_PARAMS = 8;

struct Param {
    uint8_t kind; bool opt; const char* name;
    __host__ __device__ constexpr Param() : kind(P_POS_ONLY), opt(false), name("") {}
    __host__ __device__ constexpr Param(uint8_t k, bool o, const char* s) : kind(k), opt(o), name(s) {}
};
struct Sig {
    int n; Param p[MAX_PARAMS];
};
template <class... Ps> __host__ __device__ constexpr Sig make_sig(Ps... ps) {
    const Param a[] = {ps...};
    Sig s{};
    s.n = (int)sizeof...(ps);
    for (int k = 0; k < s.n && k < MAX_PARAMS; ++k) s.p[k] = a[k];
    return s;
}

// the compile-time checks B9H_SIGNATURE makes (each a static_assert of its own, so that the message names the rule)
__host__ __device__ constexpr bool sig_names_ok(const Sig& s) {          // ASCII identifiers
    for (int k = 0; k < s.n && k < MAX_PARAMS; ++k) {
        const char* c = s.p[k].name;
        if (!((c[0] >= 'A' && c[0] <= 'Z') || (c[0] >= 'a' && c[0] <= 'z') || c[0] == '_')) return false;
        for (int j = 1; c[j]; ++j)
            if (!((c[j] >= 'A' && c[j] <= 'Z') || (c[j] >= 'a' && c[j] <= 'z') || (c[j] >= '0' && c[j] <= '9') || c[j] == '_')) return false;
    }
    return true;
}
__host__ __device__ constexpr bool str_eq(const char* a, const char* b) {
    int j = 0;
    while (a[j] && a[j] == b[j]) ++j;
    return a[j] == b[j];
}
__host__ __device__ constexpr bool sig_names_unique(const Sig& s) {
    for (int k = 0; k < s.n && k < MAX_PARAMS; ++k)
        for (int m = 0; m < k; ++m) if (str_eq(s.p[k].name, s.p[m].name)) return false;
    return true;
}
__host__ __device__ constexpr bool sig_no_context(const Sig& s) {
    for (int k = 0; k < s.n && k < MAX_PARAMS; ++k) if (str_eq(s.p[k].name, "context")) return false;
    return true;
}
// Python's order: positional-only, positional-or-keyword, at most one *args, keyword-only; among the positional
// parameters no required one after an optional one
__host__ __device__ constexpr bool sig_order_ok(const Sig& s) {
    bool opt_seen = false;
    for (int k = 0; k < s.n && k < MAX_PARAMS; ++k) {
        const Param& q = s.p[k];
        if (q.kind > P_KW_ONLY) return false;
        if (k && (q.kind < s.p[k - 1].kind || (q.kind == P_VAR_POS && s.p[k - 1].kind == P_VAR_POS))) return false;
        if (q.kind <= P_POS_OR_KW) { if (opt_seen && !q.opt) return false; opt_seen = opt_seen || q.opt; }
    }
    return true;
}

#define B9H_POS_ONLY(n)      b9h::Param(b9h::P_POS_ONLY, false, n)
#define B9H_POS_ONLY_OPT(n)  b9h::Param(b9h::P_POS_ONLY, true, n)
#define B9H_POS_OR_KW(n)     b9h::Param(b9h::P_POS_OR_KW, false, n)
#define B9H_POS_OR_KW_OPT(n) b9h::Param(b9h::P_POS_OR_KW, true, n)
#define B9H_VAR_POS(n)       b9h::Param(b9h::P_VAR_POS, true, n)
#define B9H_KW_ONLY(n)       b9h::Param(b9h::P_KW_ONLY, false, n)
#define B9H_KW_ONLY_OPT(n)   b9h::Param(b9h::P_KW_ONLY, true, n)
// Inside a handler struct: its Python signature, parameters in `def` order. Binding follows CPython's for
// handler(*args, **kwargs); an optional parameter left unbound reads as absent and the handler applies its default.
#define B9H_SIGNATURE(...)                                                                                                    \
    __host__ __device__ static constexpr b9h::Sig b9h_signature() { return b9h::make_sig(__VA_ARGS__); }                      \
    static_assert(b9h::make_sig(__VA_ARGS__).n <= b9h::MAX_PARAMS, "b9h: a signature has at most 8 parameters");             \
    static_assert(b9h::sig_names_ok(b9h::make_sig(__VA_ARGS__)), "b9h: parameter names are ASCII identifiers");              \
    static_assert(b9h::sig_names_unique(b9h::make_sig(__VA_ARGS__)), "b9h: duplicate parameter name");                       \
    static_assert(b9h::sig_no_context(b9h::make_sig(__VA_ARGS__)),                                                           \
                  "b9h: `context` is the runner's FunctionContext, which the device cannot bind");                           \
    static_assert(b9h::sig_order_ok(b9h::make_sig(__VA_ARGS__)),                                                             \
                  "b9h: parameters go positional-only, positional-or-keyword, *args, keyword-only, positional defaults last")

template <class...> struct void_t_ { typedef void type; };
template <class H, class = void> struct has_signature { static constexpr bool value = false; };
template <class H> struct has_signature<H, typename void_t_<decltype(H::b9h_signature())>::type> { static constexpr bool value = true; };

// Where a call's arguments are: the positional list p[a_off, a_off + a_len) (a_len 0: none) and the kwargs object
// p[k_off, k_off + k_len) (k_len 0: none). k_skip_args: the object is an HTTP body's top level, whose "args" members
// were taken as the positionals (SerializeHttpPayload deletes that key).
struct CallSrc { uint32_t a_off, a_len, k_off, k_len; uint8_t k_skip_args; };

// The bound call, by parameter index in the signature: c[i] is the bound value, c.has(i) whether there is one (an
// optional parameter not passed reads as absent), c.rest() the positionals *args collected.
class Call {
public:
    __device__ Arg operator[](int i) const { return Arg(p_, s_[i], e_[i], unsure_); }
    __device__ bool has(int i) const { return e_[i] != 0; }
    __device__ Items rest() const { Items it; it.p = rp_; it.i = ri_; it.e = re_; it.unsure = unsure_; return it; }

    // CPython's binding of handler(*args, **kwargs) to H's signature; false where it raises TypeError
    template <class H> __device__ bool bind(const uint8_t* p, const CallSrc& src, bool* unsure);

private:
    const uint8_t* p_; bool* unsure_;
    uint32_t s_[MAX_PARAMS], e_[MAX_PARAMS];
    const uint8_t* rp_; uint32_t ri_, re_;
};

template <class H> __device__ inline bool Call::bind(const uint8_t* p, const CallSrc& src, bool* unsure) {
    constexpr Sig S = H::b9h_signature();
    p_ = p; unsure_ = unsure;
#pragma unroll
    for (int k = 0; k < MAX_PARAMS; ++k) { s_[k] = 0; e_[k] = 0; }
    int npos = 0; bool var = false;
#pragma unroll
    for (int k = 0; k < S.n; ++k) { npos += S.p[k].kind <= P_POS_OR_KW; var = var || S.p[k].kind == P_VAR_POS; }
    // positionals: the first npos to the positional parameters, the others to *args
    int bound = 0;
    rp_ = (const uint8_t*)"]"; ri_ = 0; re_ = 1;
    if (src.a_len) {
        Items it; it.p = p; it.i = src.a_off + 1; it.e = src.a_off + src.a_len; it.unsure = unsure;
        Arg x;
#pragma unroll
        for (int k = 0; k < MAX_PARAMS; ++k) {
            if (k >= npos || !it.next(x)) break;
            s_[k] = x.s_; e_[k] = x.e_; ++bound;
        }
        rp_ = p; ri_ = it.i; re_ = it.e;
        if (!var && bound == npos && it.next(x)) return false;                    // too many positional arguments
    }
    // keywords: by decoded name, the last member of a name deciding
    if (src.k_len) {
        Members m{p, src.k_off + 1, src.k_off + src.k_len};
        uint32_t ks, ke, vs, ve;
        while (m.next(ks, ke, vs, ve)) {
            if (src.k_skip_args && b9::match_exact_key(p, ks, ke) == 1) continue;
            bool hit = false;
#pragma unroll
            for (int k = 0; k < S.n; ++k) {
                if (S.p[k].kind == P_VAR_POS || hit) continue;
                if (!key_eq(p, ks, ke, (const uint8_t*)S.p[k].name, cstr_len(S.p[k].name))) continue;
                if (S.p[k].kind == P_POS_ONLY || k < bound) return false;         // positional-only by keyword; multiple values
                s_[k] = vs; e_[k] = ve; hit = true;
            }
            if (!hit) return false;                                               // unexpected keyword argument
        }
    }
#pragma unroll
    for (int k = 0; k < S.n; ++k)
        if (S.p[k].kind != P_VAR_POS && !S.p[k].opt && !e_[k]) return false;     // missing required argument
    return true;
}

// Where rendering R's task p[0, n) with slot flags `flags` has its arguments (pr: user_parse's, ST_OK). flags 0: the SDK
// payload's args / kwargs as Go's struct decode kept them; B9_TF_TASK_MSG: the record's own; B9_TF_HTTP_BODY:
// SerializeHttpPayload -- a last "args" that is a list is the positionals, a last "kwargs" that is an object alone is
// the kwargs, otherwise every other top-level key of the body is a keyword argument.
__device__ inline CallSrc call_src(const uint8_t* p, uint32_t n, uint32_t flags, const b9::Parsed& pr) {
    CallSrc c; c.a_off = pr.args_off; c.a_len = pr.args_len; c.k_off = pr.kw_off; c.k_len = pr.kw_len; c.k_skip_args = 0;
    if (flags == B9_TF_HTTP_BODY && !pr.kw_len) {
        uint32_t i = 0;
        while (i < n && b9::is_ws(p[i])) ++i;
        if (i < n && p[i] == '{') {                                                // (else an empty or null body: no keys)
            uint32_t f = 0;
            c.k_off = i; c.k_len = (uint32_t)b9::skip_value(p, i, n, f) - i; c.k_skip_args = pr.args_len != 0;
        }
    }
    return c;
}

struct CallRec : UserRec {
    CallSrc src;                 // pass 2 of a string or container result binds the call again from here
};

// Phase A of a handler with a signature. A task-queue SDK payload whose "kwargs" came more than once as objects (Go
// merges those maps) is UNSUPPORTED.
template <class H, int R> __device__ inline void call_phase_a(const uint8_t* p, uint32_t n, uint32_t flags, const uint8_t* id, CallRec& rec) {
    const b9::Parsed pr = user_parse<R>(p, n, flags, id);
    rec.src_off = 0; rec.src_len = 0; rec.out_len = 0; rec.has = 0; rec.vk = VK_UNSET; rec.value = 0;
    if (pr.status != b9::ST_OK) { rec.status = pr.status; return; }
    if (flags == 0 && pr.kw_merged) { rec.status = b9::ST_UNSUPPORTED; return; }
    rec.src = call_src(p, n, flags, pr);
    bool unsure = false;
    Call c;
    if (!c.bind<H>(p, rec.src, &unsure)) { rec.status = b9::ST_ERROR; rec.value = B9_EXC_TYPE_ERROR; return; }
    CountSink<R> out;
    const int ret = H::call(c, out);
    phase_a_settle<R>(ret, unsure, out, rec);
}

template <class H, int R> __device__ inline bool call_phase_b(const uint8_t* p, const CallRec& rec, uint8_t* o) {
    if (rec.vk < VK_STR) { scalar_write<R>(rec.vk, rec.value, o); return true; }
    bool unsure = false;
    Call c;
    if (!c.bind<H>(p, rec.src, &unsure)) return false;
    WriteSink<R> out(o, rec.out_len);
    const int ret = H::call(c, out);
    return ret == 0 && !unsure && out.ok && out.done && out.n == rec.out_len;
}

// What the kernel runs for handler H: the one-Arg phases, or, for a handler with a signature, the bound call's
template <bool Signature> struct RecSel { typedef UserRec type; };
template <> struct RecSel<true> { typedef CallRec type; };
template <class H> using rec_t = typename RecSel<has_signature<H>::value>::type;
template <class H, int R> __device__ __forceinline__ void task_phase_a(const uint8_t* p, uint32_t n, uint32_t flags, const uint8_t* id, UserRec& rec) {
    user_phase_a<H, R>(p, user_parse<R>(p, n, flags, id), rec);
}
template <class H, int R> __device__ __forceinline__ bool task_phase_b(const uint8_t* p, const UserRec& rec, uint8_t* o) {
    return user_phase_b<H, R>(p, rec, o);
}
template <class H, int R> __device__ __forceinline__ void task_phase_a(const uint8_t* p, uint32_t n, uint32_t flags, const uint8_t* id, CallRec& rec) {
    call_phase_a<H, R>(p, n, flags, id, rec);
}
template <class H, int R> __device__ __forceinline__ bool task_phase_b(const uint8_t* p, const CallRec& rec, uint8_t* o) {
    return call_phase_b<H, R>(p, rec, o);
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
