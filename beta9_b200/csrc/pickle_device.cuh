// The function path beyond identity's one-str template (B9_DRAIN_PICKLE_FULL): the runner's loop over a cloudpickle
// argument blob for plain Python values, bit-exact against cloudpickle 3.1.2 on CPython 3.12.
//   runner  sdk/src/beta9/runner/function.py:236-283   payload = loads(blob); args = payload.get("args") or [];
//                                                      kwargs = payload.get("kwargs") or {}; kwargs.pop("callback_url");
//                                                      result = handler(*args, **kwargs); cloudpickle.dumps(result)
// One task = decode (pk_decode: a value graph in a PkScratch), the call rules and the handler (pk_prepare: status and
// result size), then the result's pickle (pk_write). pk_prepare's sizing walk and pk_write's walk are the same code.
// Plain C++ behind CUDA qualifiers: tests/host_shim/pickle_shim.cpp compiles this header for the CPU tests.
//
// Decoded opcodes (pickle protocol 5, at opcode boundaries): PROTO 5, FRAME (a bound check only, as CPython's C
// unpickler does), EMPTY_DICT / EMPTY_LIST / EMPTY_TUPLE, MARK, TUPLE1/2/3, TUPLE, APPEND(S), SETITEM(S), MEMOIZE,
// BINGET / LONG_BINGET, SHORT_BINUNICODE / BINUNICODE(8), SHORT_BINBYTES / BINBYTES(8), BININT1/2, BININT, LONG1,
// BINFLOAT, NONE, NEWTRUE / NEWFALSE, STOP (the last byte of the blob, one value on the stack, no open MARK).
// Everything else is declined (pk_decode returns -1); see include/b9gpu.h for the full list of declines.
#pragma once
#include <stdint.h>
#include "handlers_device.cuh"
#include "task_msg.cuh"

namespace b9 {

// Per-task scratch (28,744 bytes, 28.1 KiB): the graph of one blob. A blob that needs more of any of these is declined.
constexpr uint32_t PK_MAX_NODES  = 2048;    // values (a shared object is one node)
constexpr uint32_t PK_MAX_KIDS   = 2048;    // container members (a dict member counts twice: key, value)
constexpr uint32_t PK_MAX_CHUNKS = 256;     // runs of members added by one APPEND(S) / SETITEM(S) / TUPLE
constexpr uint32_t PK_MAX_MEMO   = 1024;    // MEMOIZE entries of the blob
constexpr uint32_t PK_MAX_MARKS  = 32;      // open MARKs
constexpr uint32_t PK_MAX_DEPTH  = 16;      // identity: containers nested in a result
constexpr uint32_t PK_MAX_MEMBERS = 64;     // members of one dict (PY_VALUE_MAX_MEMBERS of the JSON path)
constexpr uint32_t PK_FRAME_TARGET = 65536; // the pickler's FRAME_SIZE_TARGET: a result body this long is declined
constexpr uint16_t PK_NIL = 0xFFFFu;

enum : uint8_t { PK_NONE, PK_FALSE, PK_TRUE, PK_INT, PK_FLOAT, PK_STR, PK_BYTES, PK_LIST, PK_TUPLE, PK_DICT };

// scalars, str and bytes: x = offset of the opcode in the blob; containers: x = first chunk | last chunk << 16,
// n = members. fl bit 0: frozen (placed in a container or fetched from the memo: no longer mutable on the device)
struct PkNode { uint32_t x; uint16_t n; uint8_t kind; uint8_t fl; };
struct PkChunk { uint16_t start, count, next; };
struct PkScratch {
    PkNode node[PK_MAX_NODES];
    uint16_t kid[PK_MAX_KIDS];
    uint16_t stack[PK_MAX_NODES];       // the unpickler's stack while decoding; the result's memo index per node after
    uint16_t memo[PK_MAX_MEMO];
    PkChunk chunk[PK_MAX_CHUNKS];
    uint16_t sing[258];                 // CPython's str singletons ("" and one char of U+0000-U+00FF), then b""
    uint16_t mark[PK_MAX_MARKS];
    uint32_t n_nodes;
};

__device__ __forceinline__ uint32_t pk_u16(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }
__device__ __forceinline__ uint32_t pk_u32(const uint8_t* p) { return pk_u16(p) | (pk_u16(p + 2) << 16); }
__device__ __forceinline__ uint64_t pk_u64(const uint8_t* p) { return (uint64_t)pk_u32(p) | ((uint64_t)pk_u32(p + 4) << 32); }

// data of a str / bytes node: [*s, *s + *n)
__device__ inline void pk_data(const uint8_t* p, uint32_t op, uint32_t* s, uint32_t* n) {
    const uint8_t c = p[op];
    if (c == 0x8C || c == 'C') { *n = p[op + 1]; *s = op + 2; }
    else if (c == 'X' || c == 'B') { *n = pk_u32(p + op + 1); *s = op + 5; }
    else { *n = (uint32_t)pk_u64(p + op + 1); *s = op + 9; }                  // BINUNICODE8 / BINBYTES8
}

// LONG1's little-endian two's complement, shortened to the minimal length CPython writes
__device__ inline uint32_t pk_long_min(const uint8_t* b, uint32_t n) {
    while (n > 1 && ((b[n - 1] == 0x00 && !(b[n - 2] & 0x80)) || (b[n - 1] == 0xFF && (b[n - 2] & 0x80)))) --n;
    return n;
}
// value of an int node: true when it fits an int64 (*v), false for a longer LONG1 (its minimal bytes: *big, *nb)
__device__ inline bool pk_int(const uint8_t* p, uint32_t op, long long* v, const uint8_t** big, uint32_t* nb) {
    const uint8_t c = p[op];
    if (c == 'K') { *v = p[op + 1]; return true; }
    if (c == 'M') { *v = pk_u16(p + op + 1); return true; }
    if (c == 'J') { *v = (int32_t)pk_u32(p + op + 1); return true; }
    const uint32_t n0 = p[op + 1];
    const uint8_t* b = p + op + 2;
    if (n0 == 0) { *v = 0; return true; }
    const uint32_t n = pk_long_min(b, n0);
    if (n > 8) { *big = b; *nb = n; return false; }
    unsigned long long u = (b[n - 1] & 0x80) ? ~0ull : 0ull;
    for (uint32_t k = n; k-- > 0;) u = (u << 8) | b[k];
    *v = (long long)u;
    return true;
}
__device__ __forceinline__ double pk_float(const uint8_t* p, uint32_t op) {
    unsigned long long u = 0;
    for (int k = 1; k <= 8; ++k) u = (u << 8) | p[op + k];
    return f64_from_bits(u);
}

__device__ inline bool pk_truthy(const uint8_t* p, const PkNode& N) {
    switch (N.kind) {
    case PK_NONE: case PK_FALSE: return false;
    case PK_TRUE: return true;
    case PK_INT: { long long v = 0; const uint8_t* b = nullptr; uint32_t nb = 0; return !pk_int(p, N.x, &v, &b, &nb) || v != 0; }
    case PK_FLOAT: return (f64_to_bits(pk_float(p, N.x)) << 1) != 0ull;
    case PK_STR: case PK_BYTES: { uint32_t s, n; pk_data(p, N.x, &s, &n); return n != 0; }
    default: return N.n != 0;
    }
}

// ------------------------------------------------------------------------------------------------ decoder
// -> the root node, or -1 (declined: an opcode outside the list above, a truncated or ill-formed stream, str bytes that
// are not UTF-8 under "surrogatepass", a dict key that is not str / bytes / int / bool / float / None, a dict of more
// than 64 members, a list or dict mutated after it was placed in a container or fetched from the memo (which a cycle
// needs), or a scratch table full).
__device__ inline int pk_decode(const uint8_t* __restrict__ p, uint32_t len, PkScratch& S) {
    uint32_t i = 0, nn = 0, sp = 0, nm = 0, nmk = 0, nk = 0, nc = 0;
    for (uint32_t k = 0; k < 258; ++k) S.sing[k] = PK_NIL;
    S.n_nodes = 0;
    auto fence = [&]() -> uint32_t { return nmk ? S.mark[nmk - 1] : 0u; };
    auto node = [&](uint8_t kind, uint32_t x) -> int {
        if (nn >= PK_MAX_NODES) return -1;
        S.node[nn].x = x; S.node[nn].n = 0; S.node[nn].kind = kind; S.node[nn].fl = 0;
        return (int)nn++;
    };
    // appends k members (from the stack) to container c as one run
    auto add = [&](uint32_t c, const uint16_t* src, uint32_t k) -> bool {
        PkNode& C = S.node[c];
        if (k == 0) return true;
        if (nk + k > PK_MAX_KIDS) return false;
        for (uint32_t j = 0; j < k; ++j) { S.kid[nk + j] = src[j]; S.node[src[j]].fl |= 1u; }
        const uint32_t last = C.x >> 16;
        if (last != PK_NIL && S.chunk[last].start + S.chunk[last].count == nk) S.chunk[last].count = (uint16_t)(S.chunk[last].count + k);
        else {
            if (nc >= PK_MAX_CHUNKS) return false;
            S.chunk[nc].start = (uint16_t)nk; S.chunk[nc].count = (uint16_t)k; S.chunk[nc].next = PK_NIL;
            if (last == PK_NIL) C.x = nc | (nc << 16);
            else { S.chunk[last].next = (uint16_t)nc; C.x = (C.x & 0xFFFFu) | (nc << 16); }
            ++nc;
        }
        nk += k; C.n = (uint16_t)(C.n + k);
        return true;
    };
    auto key_ok = [&](uint32_t v) -> bool { const uint8_t t = S.node[v].kind; return t <= PK_BYTES; };
    for (;;) {
        if (i >= len) return -1;
        const uint32_t op = i;
        const uint8_t c = p[i++];
        const uint32_t rem = len - i;
        int push = -1;
        switch (c) {
        case 0x80: if (rem < 1 || p[i] != 5) return -1; ++i; continue;                                  // PROTO 5
        case 0x95: { if (rem < 8) return -1; const uint64_t fl = pk_u64(p + i); i += 8; if (fl > len - i) return -1; continue; }   // FRAME
        case '}': push = node(PK_DICT, 0xFFFFFFFFu); break;
        case ']': push = node(PK_LIST, 0xFFFFFFFFu); break;
        case ')': push = node(PK_TUPLE, 0xFFFFFFFFu); break;
        case 'N': push = node(PK_NONE, op); break;
        case 0x88: push = node(PK_TRUE, op); break;
        case 0x89: push = node(PK_FALSE, op); break;
        case 'K': if (rem < 1) return -1; i += 1; push = node(PK_INT, op); break;
        case 'M': if (rem < 2) return -1; i += 2; push = node(PK_INT, op); break;
        case 'J': if (rem < 4) return -1; i += 4; push = node(PK_INT, op); break;
        case 0x8A: if (rem < 1 || rem - 1 < p[i]) return -1; i += 1 + p[i]; push = node(PK_INT, op); break;
        case 'G': if (rem < 8) return -1; i += 8; push = node(PK_FLOAT, op); break;
        case 0x8C: case 'X': case 0x8D: case 'C': case 'B': case 0x8E: {
            const uint32_t h = (c == 0x8C || c == 'C') ? 1u : (c == 'X' || c == 'B') ? 4u : 8u;
            if (rem < h) return -1;
            const uint64_t n = h == 1 ? p[i] : h == 4 ? pk_u32(p + i) : pk_u64(p + i);
            if (n > rem - h) return -1;
            const uint32_t s = i + h;
            i = s + (uint32_t)n;
            const bool str = c == 0x8C || c == 'X' || c == 0x8D;
            if (str && !utf8_valid_surrogatepass(p + s, (uint32_t)n)) return -1;
            // CPython's singletons: "" and every one-character str of U+0000-U+00FF come back as one object each, and b""
            int sg = -1;
            if (!str) sg = n == 0 ? 257 : -1;
            else if (n == 0) sg = 0;
            else if (n == 1) sg = 1 + p[s];
            else if (n == 2 && (p[s] == 0xC2 || p[s] == 0xC3)) sg = 1 + (((p[s] & 3u) << 6) | (p[s + 1] & 0x3Fu));
            if (sg >= 0 && S.sing[sg] != PK_NIL) { push = S.sing[sg]; break; }
            push = node(str ? PK_STR : PK_BYTES, op);
            if (sg >= 0 && push >= 0) S.sing[sg] = (uint16_t)push;
            break;
        }
        case '(': if (nmk >= PK_MAX_MARKS) return -1; S.mark[nmk++] = (uint16_t)sp; continue;
        case 0x85: case 0x86: case 0x87: case 't': {                                                     // TUPLE1/2/3, TUPLE
            uint32_t base;
            if (c == 't') { if (!nmk) return -1; base = S.mark[--nmk]; }
            else { const uint32_t k = c - 0x84u; if (sp - fence() < k) return -1; base = sp - k; }
            push = node(PK_TUPLE, 0xFFFFFFFFu);
            if (push < 0 || !add((uint32_t)push, S.stack + base, sp - base)) return -1;
            sp = base;
            break;
        }
        case 'a': case 's': {                                                                            // APPEND, SETITEM
            const uint32_t k = c == 'a' ? 1u : 2u;
            if (sp - fence() < k + 1) return -1;
            const uint32_t t = S.stack[sp - k - 1];
            PkNode& T = S.node[t];
            if (T.kind != (c == 'a' ? PK_LIST : PK_DICT) || (T.fl & 1u)) return -1;
            if (c == 's' && (!key_ok(S.stack[sp - 2]) || T.n / 2u >= PK_MAX_MEMBERS)) return -1;
            if (!add(t, S.stack + sp - k, k)) return -1;
            sp -= k;
            continue;
        }
        case 'e': case 'u': {                                                                            // APPENDS, SETITEMS
            if (!nmk) return -1;
            const uint32_t m = S.mark[--nmk];
            if (m == 0 || m - 1 < fence()) return -1;
            const uint32_t t = S.stack[m - 1];
            PkNode& T = S.node[t];
            if (T.kind != (c == 'e' ? PK_LIST : PK_DICT) || (T.fl & 1u)) return -1;
            if (c == 'u') {
                if ((sp - m) & 1u) return -1;
                for (uint32_t q = m; q < sp; q += 2) if (!key_ok(S.stack[q])) return -1;
                if (T.n / 2u + (sp - m) / 2u > PK_MAX_MEMBERS) return -1;
            }
            if (!add(t, S.stack + m, sp - m)) return -1;
            sp = m;
            continue;
        }
        case 0x94: if (sp <= fence() || nm >= PK_MAX_MEMO) return -1; S.memo[nm++] = S.stack[sp - 1]; continue;   // MEMOIZE
        case 'h': case 'j': {                                                                            // BINGET, LONG_BINGET
            const uint32_t h = c == 'h' ? 1u : 4u;
            if (rem < h) return -1;
            const uint32_t ix = h == 1 ? p[i] : pk_u32(p + i);
            i += h;
            if (ix >= nm) return -1;
            push = S.memo[ix];
            S.node[push].fl |= 1u;
            break;
        }
        case '.':                                                                                        // STOP
            if (nmk || sp != 1 || i != len) return -1;
            S.n_nodes = nn;
            return S.stack[0];
        default: return -1;
        }
        if (push < 0 || sp >= PK_MAX_NODES) return -1;
        S.stack[sp++] = (uint16_t)push;
    }
}

// the str node is exactly `lit`
__device__ inline bool pk_is_str(const uint8_t* p, const PkNode& N, const char* lit, uint32_t n) {
    if (N.kind != PK_STR) return false;
    uint32_t s, m; pk_data(p, N.x, &s, &m);
    if (m != n) return false;
    for (uint32_t k = 0; k < n; ++k) if (p[s + k] != (uint8_t)lit[k]) return false;
    return true;
}
// member k of container c (in order), walking its runs
struct PkIter { uint32_t chunk, j; };
__device__ __forceinline__ PkIter pk_begin(const PkScratch& S, uint32_t c) { PkIter it; it.chunk = S.node[c].x & 0xFFFFu; it.j = 0; return it; }
__device__ __forceinline__ uint32_t pk_next(const PkScratch& S, PkIter& it) {
    const PkChunk& C = S.chunk[it.chunk];
    const uint32_t v = S.kid[C.start + it.j];
    if (++it.j == C.count) { it.chunk = C.next; it.j = 0; }
    return v;
}
// the value of the last member of dict d whose key is the str `lit` (what a dict with the duplicates merged holds), or -1
__device__ inline int pk_dict_get(const uint8_t* p, const PkScratch& S, uint32_t d, const char* lit, uint32_t n) {
    int r = -1;
    PkIter it = pk_begin(S, d);
    for (uint32_t q = 0; q < S.node[d].n; q += 2) {
        const uint32_t k = pk_next(S, it), v = pk_next(S, it);
        if (pk_is_str(p, S.node[k], lit, n)) r = (int)v;
    }
    return r;
}

// ------------------------------------------------------------------------------------------------ dict keys under ==
// an integral double as minimal two's complement bytes (|f| >= 2^63 here, so 9 to 129 bytes)
__device__ inline uint32_t pk_f64_int_bytes(double f, uint8_t* b) {
    const unsigned long long u = f64_to_bits(f);
    const int e = (int)((u >> 52) & 0x7FF) - 1075;                 // f = m * 2^e, e >= 11
    const unsigned long long m = (u & 0xFFFFFFFFFFFFFull) | (1ull << 52);
    const uint32_t nb = (uint32_t)(e / 8) + 9;
    for (uint32_t k = 0; k < nb; ++k) b[k] = 0;
    const uint32_t q = (uint32_t)(e / 8), r = (uint32_t)(e % 8);
    for (uint32_t k = 0; k < 8; ++k) {                             // m << r spans 8 bytes (m < 2^53, r < 8)
        const unsigned long long w = (m << r) >> (8 * k);
        b[q + k] = (uint8_t)w;
    }
    if (u >> 63) {                                                 // negate
        uint32_t carry = 1;
        for (uint32_t k = 0; k < nb; ++k) { const uint32_t t = (uint32_t)(uint8_t)~b[k] + carry; b[k] = (uint8_t)t; carry = t >> 8; }
    }
    return pk_long_min(b, nb);
}
// key nodes a, b of kinds str / bytes / int / bool / float / None: a == b in Python
__device__ inline bool pk_key_eq(const uint8_t* p, const PkScratch& S, uint32_t a, uint32_t b) {
    if (a == b) return true;
    const PkNode &A = S.node[a], &B = S.node[b];
    if (A.kind == PK_NONE || B.kind == PK_NONE) return A.kind == B.kind;
    if (A.kind == PK_STR || A.kind == PK_BYTES || B.kind == PK_STR || B.kind == PK_BYTES) {
        if (A.kind != B.kind) return false;
        uint32_t sa, na, sb, nb; pk_data(p, A.x, &sa, &na); pk_data(p, B.x, &sb, &nb);
        if (na != nb) return false;
        for (uint32_t k = 0; k < na; ++k) if (p[sa + k] != p[sb + k]) return false;
        return true;
    }
    // numbers: bool, int (int64 or longer), float
    struct Num { bool fl, big; long long i; double f; const uint8_t* b; uint32_t nb; };
    auto num = [&](const PkNode& N) -> Num {
        Num r; r.fl = false; r.big = false; r.i = 0; r.f = 0.0; r.b = nullptr; r.nb = 0;
        if (N.kind == PK_TRUE) r.i = 1;
        else if (N.kind == PK_INT) r.big = !pk_int(p, N.x, &r.i, &r.b, &r.nb);
        else if (N.kind == PK_FLOAT) { r.fl = true; r.f = pk_float(p, N.x); }
        return r;
    };
    Num x = num(A), y = num(B);
    if (x.fl && y.fl) return x.f == y.f;
    if (!x.fl && !y.fl) {
        if (x.big != y.big) return false;
        if (!x.big) return x.i == y.i;
        if (x.nb != y.nb) return false;
        for (uint32_t k = 0; k < x.nb; ++k) if (x.b[k] != y.b[k]) return false;
        return true;
    }
    if (y.fl) { Num t = x; x = y; y = t; }                         // x: the float, y: the int
    const unsigned long long u = f64_to_bits(x.f);
    if (((u >> 52) & 0x7FF) == 0x7FF) return false;                // inf, NaN
    const double lim = 9223372036854775808.0;                       // 2^63
    if (x.f < lim && x.f >= -lim) {
        if (y.big) return false;
        const long long t = (long long)x.f;
        return (double)t == x.f && t == y.i;
    }
    if (!y.big) return false;
    uint8_t fb[136];
    const uint32_t n = pk_f64_int_bytes(x.f, fb);
    if (n != y.nb) return false;
    for (uint32_t k = 0; k < n; ++k) if (fb[k] != y.b[k]) return false;
    return true;
}

// ------------------------------------------------------------------------------------------------ encoder
// Writes (o != nullptr) or sizes the body of a result pickle: every byte after PROTO, STOP included.
struct PkW {
    uint8_t* o; uint32_t n;
    __device__ __forceinline__ void put(uint32_t b) { if (o) o[n] = (uint8_t)b; ++n; }
    __device__ __forceinline__ void put_le(unsigned long long v, uint32_t k) { for (uint32_t j = 0; j < k; ++j) put((uint32_t)(v >> (8 * j)) & 0xFFu); }
    __device__ __forceinline__ void bytes(const uint8_t* s, uint32_t k) { if (o) for (uint32_t j = 0; j < k; ++j) o[n + j] = s[j]; n += k; }
};
// int: BININT1 / BININT2 for 0..65535, BININT within int32, else LONG1 of the minimal two's complement
__device__ inline void pk_put_int(PkW& w, long long v) {
    if (v >= 0 && v <= 0xFF) { w.put('K'); w.put((uint32_t)v); }
    else if (v >= 0 && v <= 0xFFFF) { w.put('M'); w.put_le((unsigned long long)v, 2); }
    else if (v >= -2147483648ll && v <= 2147483647ll) { w.put('J'); w.put_le((unsigned long long)v, 4); }
    else {
        uint8_t b[8];
        for (int k = 0; k < 8; ++k) b[k] = (uint8_t)((unsigned long long)v >> (8 * k));
        const uint32_t n = pk_long_min(b, 8);
        w.put(0x8A); w.put(n); w.bytes(b, n);
    }
}
__device__ inline void pk_put_float(PkW& w, unsigned long long bits) { w.put('G'); for (int k = 7; k >= 0; --k) w.put((uint32_t)(bits >> (8 * k)) & 0xFFu); }
// str (SHORT_BINUNICODE / BINUNICODE) or bytes (SHORT_BINBYTES / BINBYTES) header; lengths stay below the frame target
__device__ inline void pk_put_data_hdr(PkW& w, bool str, uint32_t n) {
    if (n < 256) { w.put(str ? 0x8C : 'C'); w.put(n); }
    else { w.put(str ? 'X' : 'B'); w.put_le(n, 4); }
}
__device__ inline void pk_put_get(PkW& w, uint32_t ix) {
    if (ix < 256) { w.put('h'); w.put(ix); } else { w.put('j'); w.put_le(ix, 4); }
}

// cloudpickle.dumps of node r's value, body only: the C pickler's choices (protocol 5): memoized str / bytes / list /
// dict / non-empty tuple, BINGET for every object seen before, lists in MARK ... APPENDS batches of 1000 (APPEND for a
// single member), dicts with SETITEM for one member, TUPLE1/2/3 or MARK ... TUPLE. false: declined (a dict with two
// keys equal under ==, containers nested deeper than PK_MAX_DEPTH, a body of PK_FRAME_TARGET bytes).
__device__ inline bool pk_encode(const uint8_t* __restrict__ p, PkScratch& S, uint32_t r, PkW& w) {
    uint16_t* memo_out = S.stack;                                  // (the decoder's stack is free now)
    for (uint32_t k = 0; k < S.n_nodes; ++k) memo_out[k] = PK_NIL;
    uint32_t n_memo = 0;
    struct Frame { uint32_t node, done; PkIter it; };
    Frame st[PK_MAX_DEPTH];
    uint32_t depth = 0;
    // a value that needs no frame: true when written
    auto leaf = [&](uint32_t v) -> bool {
        const PkNode& N = S.node[v];
        switch (N.kind) {
        case PK_NONE: w.put('N'); return true;
        case PK_TRUE: w.put(0x88); return true;
        case PK_FALSE: w.put(0x89); return true;
        case PK_INT: {
            long long iv = 0; const uint8_t* b = nullptr; uint32_t nb = 0;
            if (pk_int(p, N.x, &iv, &b, &nb)) pk_put_int(w, iv);
            else { w.put(0x8A); w.put(nb); w.bytes(b, nb); }
            return true;
        }
        case PK_FLOAT: pk_put_float(w, f64_to_bits(pk_float(p, N.x))); return true;
        default: break;
        }
        if (memo_out[v] != PK_NIL) { pk_put_get(w, memo_out[v]); return true; }
        if (N.kind == PK_STR || N.kind == PK_BYTES) {
            uint32_t s, n; pk_data(p, N.x, &s, &n);
            pk_put_data_hdr(w, N.kind == PK_STR, n);
            w.bytes(p + s, n);
            w.put(0x94); memo_out[v] = (uint16_t)n_memo++;
            return true;
        }
        if (N.kind == PK_TUPLE && N.n == 0) { w.put(')'); return true; }
        return false;
    };
    auto enter = [&](uint32_t v) -> bool {                         // a container's opening bytes and its frame
        if (depth >= PK_MAX_DEPTH) return false;
        const PkNode& N = S.node[v];
        if (N.kind == PK_DICT) {
            // Python's dict would have merged equal keys: a real dict never pickles to that
            PkIter a = pk_begin(S, v);
            for (uint32_t q = 0; q < N.n; q += 2) {
                const uint32_t ka = pk_next(S, a); pk_next(S, a);
                PkIter b = a;
                for (uint32_t q2 = q + 2; q2 < N.n; q2 += 2) { const uint32_t kb = pk_next(S, b); pk_next(S, b); if (pk_key_eq(p, S, ka, kb)) return false; }
            }
        }
        if (N.kind != PK_TUPLE) { w.put(N.kind == PK_LIST ? ']' : '}'); w.put(0x94); memo_out[v] = (uint16_t)n_memo++; }
        const bool batched = N.kind == PK_TUPLE ? N.n > 3 : N.kind == PK_LIST ? N.n > 1 : N.n > 2;
        if (N.n && batched) w.put('(');
        st[depth].node = v; st[depth].done = 0; st[depth].it = pk_begin(S, v);
        ++depth;
        return true;
    };
    if (!leaf(r) && !enter(r)) return false;
    while (depth) {
        if (w.n >= PK_FRAME_TARGET) return false;
        Frame& F = st[depth - 1];
        const PkNode& N = S.node[F.node];
        if (F.done == N.n) {                                       // close
            if (N.kind == PK_LIST) { if (N.n) w.put(N.n == 1 ? 'a' : 'e'); }
            else if (N.kind == PK_DICT) { if (N.n) w.put(N.n == 2 ? 's' : 'u'); }
            else {
                w.put(N.n <= 3 ? 0x84u + N.n : (uint32_t)'t');
                w.put(0x94); memo_out[F.node] = (uint16_t)n_memo++;
            }
            --depth;
            continue;
        }
        if (N.kind == PK_LIST && F.done && F.done % 1000u == 0) { w.put('e'); w.put('('); }   // the next batch
        const uint32_t v = pk_next(S, F.it);
        ++F.done;
        if (!leaf(v) && !enter(v)) return false;
    }
    w.put('.');
    return w.n < PK_FRAME_TARGET;
}

// ------------------------------------------------------------------------------------------------ json_sum's sum
// One term of CPython 3.12's builtin sum, the step sum_values_token (handlers_device.cuh) takes per JSON literal: ints
// and bools exactly in a C long while no float has come (`unsupported` where the total leaves that range), then float
// accumulation with Neumaier compensation for float terms. (Shared as one inlined helper, the step changed how nvcc
// scheduled drain3_kernel<3>'s comparisons; this copy keeps that kernel's code as it was.)
__device__ __forceinline__ void pk_sum_term(long long& acc, double& fs, double& comp, bool& fl, bool& unsupported, bool is_int, long long iv,
                                            double fv) {
    if (!fl) {
        if (is_int) {
            if (acc >= 0 ? (iv <= 9223372036854775807ll - acc) : (iv >= (-9223372036854775807ll - 1) - acc)) acc += iv;
            else unsupported = true;
        } else { fs = f64_add((double)acc, fv); comp = 0.0; fl = true; }
    } else if (is_int) fs = f64_add(fs, (double)iv);
    else {
        const double t = f64_add(fs, fv);
        if (f64_abs(fs) >= f64_abs(fv)) comp = f64_add(comp, f64_add(f64_add(fs, -t), fv));
        else comp = f64_add(comp, f64_add(f64_add(fv, -t), fs));
        fs = t;
    }
}

// ------------------------------------------------------------------------------------------------ one task
enum : uint8_t { PK_R_NODE, PK_R_INT, PK_R_FLOAT, PK_R_VADD };
struct PkPlan {
    uint8_t status;            // ST_OK / ST_ERROR / ST_UNSUPPORTED
    uint8_t kind;              // PK_R_*
    uint32_t node;             // PK_R_NODE: the value
    long long i;               // PK_R_INT
    unsigned long long bits;   // PK_R_FLOAT
    uint32_t src, src_len;     // PK_R_VADD: the base64 text, its decoded length
    uint32_t body;             // bytes after PROTO
    uint32_t out_len;          // the whole result (0 unless status == ST_OK)
};

// body of a scalar result (int, float, vadd's str) or of a node's value
__device__ inline bool pk_body(const uint8_t* p, PkScratch& S, const PkPlan& pl, PkW& w) {
    if (pl.kind == PK_R_NODE) return pk_encode(p, S, pl.node, w);
    if (pl.kind == PK_R_INT) pk_put_int(w, pl.i);
    else if (pl.kind == PK_R_FLOAT) pk_put_float(w, pl.bits);
    else {
        const uint32_t n = b64_encoded_len(pl.src_len / 2u);
        pk_put_data_hdr(w, true, n);
        // vadd_write puts a quote before and after the text: it lands on the header's last byte and on MEMOIZE, both
        // written again below
        if (w.o) {
            vadd_write(p, pl.src, pl.src_len / 8u, w.o + w.n - 1);
            w.o[w.n - 1] = n < 256 ? (uint8_t)n : (uint8_t)(n >> 24);
        }
        w.n += n;
        w.put(0x94);
    }
    w.put('.');
    return w.n < PK_FRAME_TARGET;
}

// Decode, the runner's call rules, the handler (0 identity, 1 crc32, 2 vadd_f32, 3 json_sum) and the result's size.
// crc_table: crc32's 256-entry byte table.
__device__ inline PkPlan pk_prepare(const uint8_t* __restrict__ p, uint32_t len, int handler, PkScratch& S, const uint32_t* crc_table) {
    PkPlan pl; pl.status = ST_UNSUPPORTED; pl.kind = PK_R_NODE; pl.node = 0; pl.i = 0; pl.bits = 0; pl.src = 0; pl.src_len = 0; pl.body = 0; pl.out_len = 0;
    const int root = pk_decode(p, len, S);
    if (root < 0) return pl;
    pl.status = ST_ERROR;                                          // from here on a Python exception is ERROR
    if (S.node[root].kind != PK_DICT) return pl;                   // payload.get: AttributeError
    const int av = pk_dict_get(p, S, (uint32_t)root, "args", 4), kv = pk_dict_get(p, S, (uint32_t)root, "kwargs", 6);
    if (kv >= 0 && pk_truthy(p, S.node[kv])) {
        if (S.node[kv].kind != PK_DICT) return pl;                 // kwargs.pop: AttributeError / TypeError
        PkIter it = pk_begin(S, (uint32_t)kv);
        for (uint32_t q = 0; q < S.node[kv].n; q += 2) {
            const uint32_t k = pk_next(S, it); pk_next(S, it);
            if (!pk_is_str(p, S.node[k], "callback_url", 12)) return pl;   // a keyword argument the handler does not take
        }
    }
    if (av < 0 || !pk_truthy(p, S.node[av])) return pl;            // handler(): a missing argument
    const PkNode& A = S.node[av];
    if (A.kind != PK_LIST && A.kind != PK_TUPLE) { pl.status = ST_UNSUPPORTED; return pl; }   // *args of a str, a dict, ...
    if (A.n != 1) return pl;
    PkIter it = pk_begin(S, (uint32_t)av);
    const uint32_t x = pk_next(S, it);
    const PkNode& X = S.node[x];
    if (handler == 0) { pl.kind = PK_R_NODE; pl.node = x; }
    else if (handler == 1) {                                       // zlib.crc32(x.encode())
        if (X.kind != PK_STR) return pl;
        uint32_t s, n; pk_data(p, X.x, &s, &n);
        uint32_t c = 0xFFFFFFFFu;
        for (uint32_t k = 0; k < n; ++k) {
            if (p[s + k] == 0xED && k + 1 < n && p[s + k + 1] >= 0xA0) return pl;   // a surrogate: UnicodeEncodeError
            c = crc_byte(c, p[s + k], crc_table);
        }
        pl.kind = PK_R_INT; pl.i = (long long)(~c);
    } else if (handler == 2) {                                     // base64.b64decode(x, validate=True), a + b, b64encode
        if (X.kind != PK_STR && X.kind != PK_BYTES) return pl;
        uint32_t s, n; pk_data(p, X.x, &s, &n);
        if (X.kind == PK_STR) for (uint32_t k = 0; k < n; ++k) if (p[s + k] >= 0x80) return pl;   // non-ASCII str: ValueError
        const int64_t rn = b64_decoded_len(p, s, s + n);
        if (rn < 0 || (rn & 7)) return pl;
        pl.kind = PK_R_VADD; pl.src = s; pl.src_len = (uint32_t)rn;
    } else {                                                       // sum(obj["values"])
        if (X.kind != PK_DICT) return pl;
        const int vv = pk_dict_get(p, S, x, "values", 6);
        if (vv < 0) return pl;                                     // KeyError
        const PkNode& V = S.node[vv];
        if (V.kind != PK_LIST && V.kind != PK_TUPLE) { pl.status = ST_UNSUPPORTED; return pl; }
        long long acc = 0; double fs = 0.0, comp = 0.0; bool fl = false, unsupported = false;
        PkIter vi = pk_begin(S, (uint32_t)vv);
        for (uint32_t q = 0; q < V.n; ++q) {
            const PkNode& T = S.node[pk_next(S, vi)];
            bool is_int = true; long long iv = 0; double fv = 0.0;
            if (T.kind == PK_TRUE) iv = 1;
            else if (T.kind == PK_FALSE) iv = 0;
            else if (T.kind == PK_INT) { const uint8_t* b = nullptr; uint32_t nb = 0; if (!pk_int(p, T.x, &iv, &b, &nb)) unsupported = true; }
            else if (T.kind == PK_FLOAT) { is_int = false; fv = pk_float(p, T.x); }
            else return pl;                                        // None, str, bytes, a container: TypeError
            if (!unsupported) pk_sum_term(acc, fs, comp, fl, unsupported, is_int, iv, fv);
        }
        if (unsupported) { pl.status = ST_UNSUPPORTED; return pl; }
        if (fl) {                                                  // the compensation, when non-zero and finite
            if (comp != 0.0 && (f64_to_bits(comp) & 0x7FF0000000000000ull) != 0x7FF0000000000000ull) fs = f64_add(fs, comp);
            pl.kind = PK_R_FLOAT; pl.bits = f64_to_bits(fs);
        } else { pl.kind = PK_R_INT; pl.i = acc; }
    }
    PkW w; w.o = nullptr; w.n = 0;
    if (!pk_body(p, S, pl, w)) { pl.status = ST_UNSUPPORTED; return pl; }
    pl.status = ST_OK;
    pl.body = w.n;
    pl.out_len = 2u + (w.n >= 4u ? 9u : 0u) + w.n;                // PROTO 5, a FRAME when the body is at least 4 bytes
    return pl;
}

// the result bytes of a ST_OK plan: o[0, pl.out_len)
__device__ inline void pk_write(const uint8_t* __restrict__ p, PkScratch& S, const PkPlan& pl, uint8_t* o) {
    o[0] = 0x80; o[1] = 0x05;
    uint32_t h = 2;
    if (pl.body >= 4u) { o[2] = 0x95; for (int k = 0; k < 8; ++k) o[3 + k] = (uint8_t)((unsigned long long)pl.body >> (8 * k)); h = 11; }
    PkW w; w.o = o + h; w.n = 0;
    pk_body(p, S, pl, w);
}

}  // namespace b9
