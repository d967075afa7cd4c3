// Test-only user handlers (include/b9gpu_handler.cuh) that drive the header's whole contract: every sink call, every
// broken rule, every return value and every Arg accessor. Each struct has a Python twin in contract_twins.py; the host
// shim (tests/host_shim/contract_shim.cpp) and the device cubin (contract.cu, build.build_test_handlers) run the same
// source. Plain C++ behind CUDA qualifiers, as examples/handlers/handlers.cuh.
#pragma once
#include "b9gpu_handler.cuh"

namespace b9_contract {

// true for the sink of the writing pass: `script`'s ops 8 and 9 make the two passes disagree on purpose
template <class Out> struct is_write_sink { static constexpr bool value = false; };
template <int R> struct is_write_sink<b9h::WriteSink<R>> { static constexpr bool value = true; };

// ---- script: a sink-call interpreter --------------------------------------------------------------------------------
// ops is a list of int lists [code, a] or [code, hi, lo] (a 64-bit argument as two unsigned 32-bit halves: an int past
// 2^53 does not survive Go's float64 decode of the payload):
//   0 none()   1 boolean(a)   2 integer(a)   3 real(the double of bits a)   4 str_begin()   5 cp(a)   6 str_end()
//   7 return a   8 cp(a) in the writing pass only   9 cp(a) in the counting pass only
// Without a 7 it returns 0. A malformed script (not a list of 1-3 INTs with a known code) raises TypeError.
template <class Out> __device__ int run_script(const b9h::Arg& ops, Out& out) {
    if (ops.kind() != b9h::LIST) return B9_EXC_TYPE_ERROR;
    b9h::Items it = ops.items();
    b9h::Arg op;
    while (it.next(op)) {
        if (op.kind() != b9h::LIST) return B9_EXC_TYPE_ERROR;
        long long a[3] = {0, 0, 0};
        int n = 0;
        b9h::Items f = op.items();
        b9h::Arg x;
        while (f.next(x)) {
            double d;
            if (n == 3 || x.kind() != b9h::INT || x.number(&a[n], &d) != b9h::INT) return B9_EXC_TYPE_ERROR;
            ++n;
        }
        if (n == 0) return B9_EXC_TYPE_ERROR;
        const long long v = n == 3 ? (long long)(((unsigned long long)(uint32_t)a[1] << 32) | (uint32_t)a[2]) : a[1];
        switch (a[0]) {
        case 0: out.none(); break;
        case 1: out.boolean(v != 0); break;
        case 2: out.integer(v); break;
        case 3: out.real(b9::f64_from_bits((unsigned long long)v)); break;
        case 4: out.str_begin(); break;
        case 5: out.cp((uint32_t)v); break;
        case 6: out.str_end(); break;
        case 7: return (int)v;
        case 8: if (is_write_sink<Out>::value) out.cp((uint32_t)v); break;
        case 9: if (!is_write_sink<Out>::value) out.cp((uint32_t)v); break;
        default: return B9_EXC_TYPE_ERROR;
        }
    }
    return 0;
}

// def script(ops, /)
struct Script {
    template <class Out> __device__ static int call(const b9h::Arg& ops, Out& out) { return run_script(ops, out); }
};

// def script_sig(ops, *rest): the same script through the settle rules of a handler with a signature
struct ScriptSig {
    B9H_SIGNATURE(B9H_POS_OR_KW("ops"), B9H_VAR_POS("rest"));
    template <class Out> __device__ static int call(const b9h::Call& c, Out& out) { return run_script(c[0], out); }
};

// ---- inspect: what the header sees of an argument --------------------------------------------------------------------
constexpr int DEPTH = 3;           // containers deeper than this are described by their head only
constexpr int N_PROBES = 7;

// the keys a dict is probed with, as NUL-terminated UTF-8: a, values, é, €, 😀, "", a"b (1- to 4-byte code points)
__device__ inline const char* probe_key(int k) {
    switch (k) {
    case 0: return "a";
    case 1: return "values";
    case 2: return "\xc3\xa9";
    case 3: return "\xe2\x82\xac";
    case 4: return "\xf0\x9f\x98\x80";
    case 5: return "";
    default: return "a\"b";
    }
}

// one code point of valid UTF-8 (decoded here, independently of the header's key_eq)
__device__ inline uint32_t utf8_next(const char* s, int& i) {
    const uint8_t c = (uint8_t)s[i];
    const int l = c < 0x80 ? 1 : c < 0xE0 ? 2 : c < 0xF0 ? 3 : 4;
    uint32_t cp = l == 1 ? c : (c & (0x3Fu >> (l - 1)));
    for (int k = 1; k < l; ++k) cp = (cp << 6) | ((uint8_t)s[i + k] & 0x3Fu);
    i += l;
    return cp;
}

// the probe key a STR argument spells, or -1
__device__ inline int probe_of(const b9h::Arg& key) {
    if (key.kind() != b9h::STR) return -1;
    for (int k = 0; k < N_PROBES; ++k) {
        const char* s = probe_key(k);
        b9h::Chars c = key.chars();
        int i = 0;
        uint32_t cp;
        bool same = true;
        while (same && c.next(cp)) same = s[i] && utf8_next(s, i) == cp;
        if (same && !s[i]) return k;
    }
    return -1;
}

template <class Out> __device__ void put_hex(unsigned long long v, Out& out) {
    int sh = 60;
    while (sh > 0 && !((v >> sh) & 0xF)) sh -= 4;
    for (; sh >= 0; sh -= 4) out.cp((uint32_t)"0123456789abcdef"[(v >> sh) & 0xF]);
}

template <class Out> __device__ void put_dec(long long v, Out& out) {
    unsigned long long m = v < 0 ? 0ull - (unsigned long long)v : (unsigned long long)v;
    if (v < 0) out.cp('-');
    char d[20];
    int n = 0;
    do { d[n++] = (char)('0' + m % 10u); m /= 10u; } while (m);
    while (n) out.cp((uint32_t)d[--n]);
}

// a value's head: kind() as one of S I F B N L D, empty() as 1 / 0, number()'s answer (=i<decimal> or =f<hex bits>;
// nothing when it declines) and a STR's code points in hex (":61.e9")
template <class Out> __device__ void head(const b9h::Arg& v, Out& out) {
    const int k = v.kind();
    out.cp((uint32_t)"SIFBNLD"[k]);
    out.cp(v.empty() ? '1' : '0');
    long long i = 0;
    double f = 0.0;
    const int t = v.number(&i, &f);
    if (t == b9h::INT) { out.cp('='); out.cp('i'); put_dec(i, out); }
    else if (t == b9h::FLOAT) { out.cp('='); out.cp('f'); put_hex(b9::f64_to_bits(f), out); }
    if (k == b9h::STR) {
        out.cp(':');
        b9h::Chars c = v.chars();
        uint32_t cp;
        for (bool first = true; c.next(cp); first = false) {
            if (!first) out.cp('.');
            put_hex(cp, out);
        }
    }
}

// The description of a value: its head, then for a LIST its items' descriptions in [] (items()), for a DICT the
// descriptions of the probe keys' values in {} (get(const char*), "-" when absent), down to DEPTH containers. An
// explicit stack of DEPTH frames, no device recursion.
struct Frame {
    b9h::Arg d; b9h::Items it;
    int k;                         // < 0: a list, at its k = -1 first item or k = -2 later ones; else a dict's next probe
};

template <class Out> __device__ void enter(const b9h::Arg& v, Frame* st, int& top, Out& out) {
    head(v, out);
    const int k = v.kind();
    if ((k != b9h::LIST && k != b9h::DICT) || top == DEPTH) return;
    Frame& f = st[top++];
    f.d = v;
    f.k = k == b9h::LIST ? -1 : 0;
    if (k == b9h::LIST) f.it = v.items();
    out.cp(k == b9h::LIST ? '[' : '{');
}

template <class Out> __device__ void describe(const b9h::Arg& v, Out& out) {
    Frame st[DEPTH];
    int top = 0;
    enter(v, st, top, out);
    while (top) {
        Frame& f = st[top - 1];
        b9h::Arg x;
        if (f.k < 0) {
            if (!f.it.next(x)) { out.cp(']'); --top; continue; }
            if (f.k == -2) out.cp(',');
            f.k = -2;
            enter(x, st, top, out);
        } else {
            if (f.k == N_PROBES) { out.cp('}'); --top; continue; }
            if (f.k) out.cp(',');
            if (f.d.get(probe_key(f.k++), x)) enter(x, st, top, out);
            else out.cp('-');
        }
    }
}

// def inspect(v, /): contract_twins.describe(v)
struct Inspect {
    template <class Out> __device__ static int call(const b9h::Arg& v, Out& out) {
        out.str_begin();
        describe(v, out);
        out.str_end();
        return 0;
    }
};

// def inspect_keys(d, *keys): for every key, the description of what get(const Arg&) finds ("-": absent), and where the
// key spells a probe key, "|" and what get(const char*) finds for that probe; ";" between keys
struct InspectKeys {
    B9H_SIGNATURE(B9H_POS_OR_KW("d"), B9H_VAR_POS("keys"));
    template <class Out> __device__ static int call(const b9h::Call& c, Out& out) {
        const b9h::Arg d = c[0];
        b9h::Items it = c.rest();
        b9h::Arg key, v;
        out.str_begin();
        for (bool first = true; it.next(key); first = false) {
            if (!first) out.cp(';');
            if (d.get(key, v)) describe(v, out);
            else out.cp('-');
            const int pk = probe_of(key);
            if (pk >= 0) {
                out.cp('|');
                if (d.get(probe_key(pk), v)) describe(v, out);
                else out.cp('-');
            }
        }
        out.str_end();
        return 0;
    }
};

}  // namespace b9_contract
