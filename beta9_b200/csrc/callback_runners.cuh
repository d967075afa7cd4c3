// The callback JSON of the function and endpoint runners (b9_set_callback_runners): the text D that the runner's
// send_callback wraps as {"data": D}, json.dumps with its defaults (", " / ": " separators, ensure_ascii=True). The signature
// over {"data": D} is cb_sign_record (callback_sign.cuh), run on the bytes written here.
//
// Reference behaviour realised per task:
//     send_callback   sdk/src/beta9/runner/common.py:406-481   body = {"data": payload}; sign_payload(json.dumps(body));
//                                                                requests.post(url, json=body) (allow_nan=False)
//     function        runner/function.py:235-343               payload = the handler's result itself (None -> null);
//                                                                url = kwargs.pop("callback_url") or the stub's
//     endpoint        middleware.py:29-78, runner/endpoint.py   payload = the handler's result, whose JSONResponse body E
//                                                                the endpoint drain already wrote (compact, ensure_ascii=False)
//
// Endpoint: D = T(E), a text transform of the record. Outside strings ',' -> ", " and ':' -> ": "; inside strings each
// UTF-8 sequence of U+0080 or above and the byte 0x7F -> \uXXXX (a surrogate pair above U+FFFF); every other byte, E's own
// escapes included, is copied. (E is well-formed; a malformed byte, which only a corrupted record has, becomes \u00XX.)
// Function: D = json.dumps of the result value, walked on the pickle pass's value graph (pickle_device.cuh).
// Plain C++ behind CUDA qualifiers: tests/host_shim/callback_runners_shim.cpp compiles it for the CPU tests.
#pragma once
#include <stdint.h>
#include "pickle_device.cuh"

namespace b9 {

// a record whose D would be longer is left to the host (B9_CB_HOST): it bounds one thread's walk of a value whose shared
// members repeat in the JSON, and keeps a warp's D bytes within 32 bits
constexpr uint32_t CBR_MAX_BODY = 1u << 20;

// Writes (o != nullptr) or sizes a D. n counts past CBR_MAX_BODY; the caller checks it.
struct CbrW {
    uint8_t* o; uint32_t n;
    __device__ __forceinline__ void put(uint32_t b) { if (o && n < CBR_MAX_BODY) o[n] = (uint8_t)b; ++n; }
    __device__ __forceinline__ void lit(const char* s, uint32_t k) { for (uint32_t j = 0; j < k; ++j) put((uint8_t)s[j]); }
    __device__ __forceinline__ bool full() const { return n > CBR_MAX_BODY; }
};

// ---- \uXXXX: the code point writer both runners share ----------------------------------------------------------------
__device__ __forceinline__ void cbr_put_u16(CbrW& w, uint32_t u) {
    w.put('\\'); w.put('u'); w.put(hexdig((u >> 12) & 15)); w.put(hexdig((u >> 8) & 15)); w.put(hexdig((u >> 4) & 15)); w.put(hexdig(u & 15));
}
// code point cp as json.dumps(ensure_ascii=True) spells it outside the short escapes: \uXXXX, a pair above U+FFFF
__device__ __forceinline__ void cbr_put_u(CbrW& w, uint32_t cp) {
    if (cp < 0x10000u) { cbr_put_u16(w, cp); return; }
    const uint32_t v = cp - 0x10000u;
    cbr_put_u16(w, 0xD800u + (v >> 10));
    cbr_put_u16(w, 0xDC00u + (v & 0x3FFu));
}

// the UTF-8 sequence at p[i] (p[i] >= 0x80), surrogates allowed ("surrogatepass"): its length and *cp, or 0 when malformed
__device__ inline uint32_t cbr_utf8(const uint8_t* __restrict__ p, uint32_t i, uint32_t end, uint32_t* cp) {
    const uint32_t c = p[i];
    auto cont = [&](uint32_t k, uint32_t lo, uint32_t hi) -> bool { return i + k < end && p[i + k] >= lo && p[i + k] <= hi; };
    if (c >= 0xC2 && c <= 0xDF) {
        if (!cont(1, 0x80, 0xBF)) return 0;
        *cp = ((c & 0x1Fu) << 6) | (p[i + 1] & 0x3Fu);
        return 2;
    }
    if (c >= 0xE0 && c <= 0xEF) {
        if (!cont(1, c == 0xE0 ? 0xA0 : 0x80, 0xBF) || !cont(2, 0x80, 0xBF)) return 0;
        *cp = ((c & 0x0Fu) << 12) | ((p[i + 1] & 0x3Fu) << 6) | (p[i + 2] & 0x3Fu);
        return 3;
    }
    if (c >= 0xF0 && c <= 0xF4) {
        if (!cont(1, c == 0xF0 ? 0x90 : 0x80, c == 0xF4 ? 0x8F : 0xBF) || !cont(2, 0x80, 0xBF) || !cont(3, 0x80, 0xBF)) return 0;
        *cp = ((c & 0x07u) << 18) | ((p[i + 1] & 0x3Fu) << 12) | ((p[i + 2] & 0x3Fu) << 6) | (p[i + 3] & 0x3Fu);
        return 4;
    }
    return 0;
}

// ---- endpoint: D = T(E) ------------------------------------------------------------------------------------------------
// o == nullptr: the length only. Returns |T(E)| (at most 6 |E|).
__device__ inline uint64_t cbr_endpoint_body(const uint8_t* __restrict__ e, uint32_t n, uint8_t* __restrict__ o) {
    uint64_t k = 0;
    auto put = [&](uint32_t b) { if (o) o[k] = (uint8_t)b; ++k; };
    bool in_str = false;
    uint32_t i = 0;
    while (i < n) {
        const uint32_t c = e[i];
        if (!in_str) {
            put(c);
            if (c == '"') in_str = true;
            else if (c == ',' || c == ':') put(' ');
            ++i;
        } else if (c == '\\') {                                   // E's escape: copied as it is
            put(c);
            if (i + 1 < n) put(e[i + 1]);
            i += 2;
        } else if (c == '"') { put(c); in_str = false; ++i; }
        else if (c < 0x7F) { put(c); ++i; }
        else {
            uint32_t cp = c, m = c >= 0x80 ? cbr_utf8(e, i, n, &cp) : 0;
            if (!m) { cp = c; m = 1; }
            CbrW w; w.o = o ? o + k : nullptr; w.n = 0;
            cbr_put_u(w, cp);
            k += w.n;
            i += m;
        }
    }
    return k;
}

// ---- function: json.dumps of a pickle-pass value ----------------------------------------------------------------------
enum : uint8_t { CBR_POST = 0, CBR_UNSENDABLE = 1, CBR_HOST = 2 };

// the str's UTF-8 (validated by the decoder under "surrogatepass") as an ensure_ascii JSON string
__device__ inline void cbr_str(CbrW& w, const uint8_t* __restrict__ s, uint32_t n) {
    w.put('"');
    uint32_t i = 0;
    while (i < n && !w.full()) {
        const uint32_t c = s[i];
        if (c >= 0x80) {
            uint32_t cp = c, m = cbr_utf8(s, i, n, &cp);
            if (!m) { cp = c; m = 1; }
            cbr_put_u(w, cp);
            i += m;
            continue;
        }
        uint32_t sc = 0;
        switch (c) { case '"': sc = '"'; break; case '\\': sc = '\\'; break; case '\b': sc = 'b'; break; case '\f': sc = 'f'; break;
                     case '\n': sc = 'n'; break; case '\r': sc = 'r'; break; case '\t': sc = 't'; break; }
        if (sc) { w.put('\\'); w.put(sc); }
        else if (c < 0x20 || c == 0x7F) cbr_put_u16(w, c);
        else w.put(c);
        ++i;
    }
    w.put('"');
}
__device__ inline void cbr_int(CbrW& w, long long v) {
    unsigned long long u = (unsigned long long)v;
    if (v < 0) { w.put('-'); u = 0ull - u; }
    uint8_t d[20];
    const uint32_t k = dec_len_u64(u);
    write_dec(d, u, k);
    for (uint32_t j = 0; j < k; ++j) w.put(d[j]);
}
// float.__repr__, NaN / Infinity / -Infinity included; false for those (requests refuses them)
__device__ inline bool cbr_float(CbrW& w, unsigned long long bits) {
    uint8_t d[32];
    const uint32_t k = py_json_float(bits, d);
    for (uint32_t j = 0; j < k; ++j) w.put(d[j]);
    return ((bits >> 52) & 0x7FFu) != 0x7FFu;
}

// What walking a value found: bytes (json.dumps raises TypeError), a non-finite float (requests raises ValueError), an
// int outside int64 or a D past CBR_MAX_BODY (the device does not write it).
struct CbrFound { bool bytes, nonfinite, host; };
__device__ __forceinline__ uint8_t cbr_kind(const CbrFound& f) { return (f.bytes || f.nonfinite) ? CBR_UNSENDABLE : f.host ? CBR_HOST : CBR_POST; }

// a scalar, str or bytes (as a value, or as a dict key when key = true: json.dumps's key coercion); false: a container
__device__ inline bool cbr_leaf(CbrW& w, const uint8_t* __restrict__ p, const PkNode& N, bool key, CbrFound& f) {
    switch (N.kind) {
    case PK_NONE: if (key) w.lit("\"null\"", 6); else w.lit("null", 4); return true;
    case PK_TRUE: if (key) w.lit("\"true\"", 6); else w.lit("true", 4); return true;
    case PK_FALSE: if (key) w.lit("\"false\"", 7); else w.lit("false", 5); return true;
    case PK_INT: {
        long long v = 0; const uint8_t* b = nullptr; uint32_t nb = 0;
        if (!pk_int(p, N.x, &v, &b, &nb)) { f.host = true; return true; }
        if (key) w.put('"');
        cbr_int(w, v);
        if (key) w.put('"');
        return true;
    }
    case PK_FLOAT: {
        if (key) w.put('"');
        if (!cbr_float(w, f64_to_bits(pk_float(p, N.x)))) f.nonfinite = true;
        if (key) w.put('"');
        return true;
    }
    case PK_STR: { uint32_t s, n; pk_data(p, N.x, &s, &n); cbr_str(w, p + s, n); return true; }
    case PK_BYTES: f.bytes = true; return true;
    default: return false;
    }
}

// json.dumps of node r (the decoder's graph in S; S.node, S.kid and S.chunk are read, nothing is written). Stops at the
// first bytes, past CBR_MAX_BODY, or deeper than PK_MAX_DEPTH (which the pickle pass has declined already).
__device__ inline CbrFound cbr_value(CbrW& w, const uint8_t* __restrict__ p, const PkScratch& S, uint32_t r) {
    CbrFound f; f.bytes = false; f.nonfinite = false; f.host = false;
    struct Frame { uint32_t node, done; PkIter it; };
    Frame st[PK_MAX_DEPTH];
    uint32_t depth = 0;
    auto enter = [&](uint32_t v) -> bool {
        if (depth >= PK_MAX_DEPTH) { f.host = true; return false; }
        const PkNode& N = S.node[v];
        w.put(N.kind == PK_DICT ? '{' : '[');
        st[depth].node = v; st[depth].done = 0; st[depth].it = pk_begin(S, v);
        ++depth;
        return true;
    };
    if (!cbr_leaf(w, p, S.node[r], false, f) && !enter(r)) return f;
    while (depth && !f.bytes && !w.full()) {
        Frame& F = st[depth - 1];
        const PkNode& N = S.node[F.node];
        if (F.done == N.n) { w.put(N.kind == PK_DICT ? '}' : ']'); --depth; continue; }
        if (F.done) w.lit(", ", 2);
        if (N.kind == PK_DICT) {
            cbr_leaf(w, p, S.node[pk_next(S, F.it)], true, f);     // (keys are scalars, str or bytes: the decoder's rule)
            w.lit(": ", 2);
            ++F.done;
        }
        const uint32_t v = pk_next(S, F.it);
        ++F.done;
        if (!cbr_leaf(w, p, S.node[v], false, f) && !enter(v)) break;
    }
    if (w.full()) f.host = true;
    return f;
}

// D of a ST_OK plan's result (pk_prepare): the value node, crc32's and json_sum's int or float, or vadd_f32's str
__device__ inline CbrFound cbr_result(CbrW& w, const uint8_t* __restrict__ p, const PkScratch& S, const PkPlan& pl) {
    if (pl.kind == PK_R_NODE) return cbr_value(w, p, S, pl.node);
    CbrFound f; f.bytes = false; f.nonfinite = false; f.host = false;
    if (pl.kind == PK_R_INT) cbr_int(w, pl.i);
    else if (pl.kind == PK_R_FLOAT) f.nonfinite = !cbr_float(w, pl.bits);
    else {                                                         // '"' + base64 + '"': ASCII that needs no escape
        const uint32_t n = b64_encoded_len(pl.src_len / 2u) + 2u;
        if (w.o) vadd_write(p, pl.src, pl.src_len / 8u, w.o + w.n);
        w.n += n;
    }
    if (w.full()) f.host = true;
    return f;
}

// The function runner's callback_url = kwargs.pop("callback_url", None) of a blob pk_decode accepted (root: its root, a
// dict when the call got as far as the handler). -1: absent or falsy (the stub's URL); -2: truthy but not a str the
// device posts to (another type, or a str with a surrogate that UTF-8 cannot carry); else the str node.
__device__ inline int cbr_callback_url(const uint8_t* __restrict__ p, const PkScratch& S, int root) {
    if (root < 0 || S.node[root].kind != PK_DICT) return -1;
    const int kv = pk_dict_get(p, S, (uint32_t)root, "kwargs", 6);
    if (kv < 0 || S.node[kv].kind != PK_DICT) return -1;          // (`or {}`: a truthy non-dict never reaches the handler)
    const int u = pk_dict_get(p, S, (uint32_t)kv, "callback_url", 12);
    if (u < 0 || !pk_truthy(p, S.node[u])) return -1;
    if (S.node[u].kind != PK_STR) return -2;
    uint32_t s, n; pk_data(p, S.node[u].x, &s, &n);
    for (uint32_t k = 0; k + 1 < n; ++k) if (p[s + k] == 0xED && p[s + k + 1] >= 0xA0) return -2;
    return u;
}

}  // namespace b9
