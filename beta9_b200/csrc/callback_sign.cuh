// The task callback's signature on the device: what the runner's send_callback posts for a drained task, and the
// gateway's SignPayload over it.
//
// Reference behaviour realised per record:
//     body        sdk/src/beta9/runner/taskqueue.py:391-397, runner/common.py:430-481: {"data": result or {}}, json.dumps
//     signature   pkg/auth/sign.go:17-35: hex(HMAC-SHA256(key, base64.StdEncoding(body) + ":" + decimal Unix seconds))
//
// The body of a record with result bytes R is exactly `{"data": ` + R + `}` (json.dumps of the dict writes the result
// with the same defaults serialize_result used for R), and `{"data": {}}` for a falsy result or an error. `{"data": `
// is 9 bytes, so the signed message is the constant "eyJkYXRhIjog", then base64(R + "}"), then ":" and the digits.
// Its base64 part starts at byte 12, a word boundary: every 4 base64 characters are one SHA-256 message word, and so are
// the 12 prefix bytes (3 words) and the drain's constant tail (":" digits, the 0x80 pad byte, zeros; CbSign::tail).
// The message is fed to the compression word by word from R; it is never materialised.
//
// HMAC as Go's hmac.New(sha256.New, key): a key longer than 64 bytes is hashed first; the ipad and opad blocks are
// compressed once per key (cb_midstates), so a record costs its inner blocks plus one outer block.
#pragma once
#include <stdint.h>
#include "json_device.cuh"

namespace b9 {

// enum b9_callback_kind (include/b9gpu.h)
constexpr uint8_t CB_NONE = 0, CB_POST = 1, CB_UNSENDABLE = 2, CB_HOST = 3;

// ---- SHA-256 (FIPS 180-4) ----------------------------------------------------------------------------------------
#define B9_SHA256_K { \
    0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u, \
    0xd807aa98u, 0x12835b01u, 0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u, \
    0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu, 0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau, \
    0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u, 0x06ca6351u, 0x14292967u, \
    0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u, \
    0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u, \
    0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu, 0x682e6ff3u, \
    0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u, 0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u }
__device__ __constant__ uint32_t CB_SHA_K_DEV[64] = B9_SHA256_K;
static const uint32_t CB_SHA_K_HOST[64] = B9_SHA256_K;
#undef B9_SHA256_K

__host__ __device__ __forceinline__ uint32_t cb_sha_k(int i) {
#ifdef __CUDA_ARCH__
    return CB_SHA_K_DEV[i];
#else
    return CB_SHA_K_HOST[i];
#endif
}

__host__ __device__ __forceinline__ uint32_t cb_rotr(uint32_t x, int n) { return (x >> n) | (x << (32 - n)); }

__host__ __device__ __forceinline__ void sha256_init(uint32_t h[8]) {
    h[0] = 0x6a09e667u; h[1] = 0xbb67ae85u; h[2] = 0x3c6ef372u; h[3] = 0xa54ff53au;
    h[4] = 0x510e527fu; h[5] = 0x9b05688cu; h[6] = 0x1f83d9abu; h[7] = 0x5be0cd19u;
}

// one block: h <- compress(h, w); w (16 big-endian message words) is used as the schedule's ring and overwritten
__host__ __device__ __forceinline__ void sha256_compress(uint32_t h[8], uint32_t w[16]) {
    uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], k = h[7];
#pragma unroll
    for (int i = 0; i < 64; ++i) {
        if (i >= 16) {
            const uint32_t w15 = w[(i - 15) & 15], w2 = w[(i - 2) & 15];
            const uint32_t s0 = cb_rotr(w15, 7) ^ cb_rotr(w15, 18) ^ (w15 >> 3);
            const uint32_t s1 = cb_rotr(w2, 17) ^ cb_rotr(w2, 19) ^ (w2 >> 10);
            w[i & 15] += s0 + w[(i - 7) & 15] + s1;
        }
        const uint32_t t1 = k + (cb_rotr(e, 6) ^ cb_rotr(e, 11) ^ cb_rotr(e, 25)) + ((e & f) ^ (~e & g)) + cb_sha_k(i) + w[i & 15];
        const uint32_t t2 = (cb_rotr(a, 2) ^ cb_rotr(a, 13) ^ cb_rotr(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
        k = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
    }
    h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += k;
}

// A byte-stream SHA-256 over a running state (the host's key hashing and midstates, the tests' reference path).
struct Sha256Stream {
    uint32_t h[8];
    uint8_t  buf[64];
    uint32_t fill;
    uint64_t total;       // bytes fed, including any block compressed into h before this stream took it over
};
__host__ __device__ inline void sha256_stream_init(Sha256Stream& s, const uint32_t* mid = nullptr, uint64_t fed = 0) {
    if (mid) { for (int i = 0; i < 8; ++i) s.h[i] = mid[i]; } else sha256_init(s.h);
    s.fill = 0; s.total = fed;
}
__host__ __device__ inline void sha256_stream_block(Sha256Stream& s) {
    uint32_t w[16];
    for (int i = 0; i < 16; ++i)
        w[i] = ((uint32_t)s.buf[4 * i] << 24) | ((uint32_t)s.buf[4 * i + 1] << 16) | ((uint32_t)s.buf[4 * i + 2] << 8) | s.buf[4 * i + 3];
    sha256_compress(s.h, w);
    s.fill = 0;
}
__host__ __device__ inline void sha256_stream_update(Sha256Stream& s, const uint8_t* p, uint64_t n) {
    for (uint64_t i = 0; i < n; ++i) {
        s.buf[s.fill++] = p[i];
        if (s.fill == 64) sha256_stream_block(s);
    }
    s.total += n;
}
// the padding with the 64-bit length of everything fed; out: 32 bytes
__host__ __device__ inline void sha256_stream_final(Sha256Stream& s, uint8_t out[32]) {
    const uint64_t bits = s.total * 8u;
    s.buf[s.fill++] = 0x80u;
    if (s.fill > 56) { while (s.fill < 64) s.buf[s.fill++] = 0; sha256_stream_block(s); }
    while (s.fill < 56) s.buf[s.fill++] = 0;
    for (int i = 0; i < 8; ++i) s.buf[56 + i] = (uint8_t)(bits >> (56 - 8 * i));
    sha256_stream_block(s);
    for (int i = 0; i < 8; ++i) { out[4 * i] = (uint8_t)(s.h[i] >> 24); out[4 * i + 1] = (uint8_t)(s.h[i] >> 16); out[4 * i + 2] = (uint8_t)(s.h[i] >> 8); out[4 * i + 3] = (uint8_t)s.h[i]; }
}
__host__ __device__ inline void sha256(const uint8_t* p, uint64_t n, uint8_t out[32]) {
    Sha256Stream s; sha256_stream_init(s); sha256_stream_update(s, p, n); sha256_stream_final(s, out);
}

// ---- HMAC-SHA256 ---------------------------------------------------------------------------------------------------
// mid[0..8): the state after the key's ipad block, mid[8..16): after its opad block
__host__ __device__ inline void cb_midstates(const uint8_t* key, uint32_t key_len, uint32_t mid[16]) {
    uint8_t k0[64];
    for (int i = 0; i < 64; ++i) k0[i] = 0;
    if (key_len > 64) sha256(key, key_len, k0);
    else for (uint32_t i = 0; i < key_len; ++i) k0[i] = key[i];
    for (int pass = 0; pass < 2; ++pass) {
        const uint8_t x = pass ? 0x5cu : 0x36u;
        uint32_t w[16];
        for (int i = 0; i < 16; ++i)
            w[i] = ((uint32_t)(k0[4 * i] ^ x) << 24) | ((uint32_t)(k0[4 * i + 1] ^ x) << 16) | ((uint32_t)(k0[4 * i + 2] ^ x) << 8) | (uint32_t)(k0[4 * i + 3] ^ x);
        uint32_t* h = mid + 8 * pass;
        sha256_init(h);
        sha256_compress(h, w);
    }
}
// the outer hash: one block over the inner digest (64 + 32 bytes in all)
__host__ __device__ __forceinline__ void cb_outer(const uint32_t mid[16], const uint32_t inner[8], uint32_t out[8]) {
    uint32_t w[16];
#pragma unroll
    for (int i = 0; i < 8; ++i) { w[i] = inner[i]; out[i] = mid[8 + i]; }
    w[8] = 0x80000000u;
#pragma unroll
    for (int i = 9; i < 15; ++i) w[i] = 0;
    w[15] = (64u + 32u) * 8u;
    sha256_compress(out, w);
}
// HMAC-SHA256 of any message (the tests' and the host's general path); out: 32 bytes
__host__ __device__ inline void hmac_sha256(const uint32_t mid[16], const uint8_t* msg, uint64_t n, uint8_t out[32]) {
    Sha256Stream s; sha256_stream_init(s, mid, 64);
    sha256_stream_update(s, msg, n);
    uint8_t d[32]; sha256_stream_final(s, d);
    uint32_t inner[8], o[8];
    for (int i = 0; i < 8; ++i) inner[i] = ((uint32_t)d[4 * i] << 24) | ((uint32_t)d[4 * i + 1] << 16) | ((uint32_t)d[4 * i + 2] << 8) | d[4 * i + 3];
    cb_outer(mid, inner, o);
    for (int i = 0; i < 8; ++i) { out[4 * i] = (uint8_t)(o[i] >> 24); out[4 * i + 1] = (uint8_t)(o[i] >> 16); out[4 * i + 2] = (uint8_t)(o[i] >> 8); out[4 * i + 3] = (uint8_t)o[i]; }
}

// ---- the signed message of one record ----------------------------------------------------------------------------
// What every record of one drain shares: the key's midstates and the tail ":" + decimal ts, 0x80, zero-padded to words.
struct CbSign {
    uint32_t mid[16];
    uint32_t tail[6];          // ":" + at most 19 digits + 0x80 = 21 bytes
    uint32_t tail_words;       // words of `tail` in use
    uint32_t tail_bytes;       // message bytes in the tail (":" and the digits, not 0x80)
};
// "eyJkYXRhIjog" = base64(`{"data": `), as three big-endian words
constexpr uint32_t CB_PREFIX_W0 = 0x65794a6bu, CB_PREFIX_W1 = 0x59585268u, CB_PREFIX_W2 = 0x496a6f67u;

__host__ __device__ inline void cb_sign_init(CbSign& s, const uint32_t mid[16], int64_t ts) {
    for (int i = 0; i < 16; ++i) s.mid[i] = mid[i];
    uint8_t t[24]; uint32_t n = 0;
    t[n++] = ':';
    char dg[20]; int nd = 0;
    uint64_t v = ts < 0 ? 0 : (uint64_t)ts;      // (Unix seconds; the host never passes a negative time)
    do { dg[nd++] = (char)('0' + v % 10u); v /= 10u; } while (v);
    while (nd) t[n++] = (uint8_t)dg[--nd];
    s.tail_bytes = n;
    t[n++] = 0x80u;
    while (n & 3u) t[n++] = 0;
    s.tail_words = n / 4;
    for (uint32_t i = 0; i < s.tail_words; ++i) s.tail[i] = ((uint32_t)t[4 * i] << 24) | ((uint32_t)t[4 * i + 1] << 16) | ((uint32_t)t[4 * i + 2] << 8) | t[4 * i + 3];
    for (uint32_t i = s.tail_words; i < 6; ++i) s.tail[i] = 0;
}

__host__ __device__ __forceinline__ uint32_t cb_b64_char(uint32_t v) {
    return v < 26 ? 'A' + v : v < 52 ? 'a' + (v - 26) : v < 62 ? '0' + (v - 52) : v == 62 ? '+' : '/';
}
// base64 quad q of S = R + "}" (|S| = len + 1) as one big-endian message word, '=' padded at the end
__host__ __device__ __forceinline__ uint32_t cb_b64_word(const uint8_t* __restrict__ r, uint32_t len, uint32_t q) {
    const uint32_t i = 3u * q, slen = len + 1u;
    const uint32_t b0 = i < len ? r[i] : '}';
    const uint32_t b1 = i + 1u < len ? r[i + 1u] : (i + 1u == len ? '}' : 0u);
    const uint32_t b2 = i + 2u < len ? r[i + 2u] : (i + 2u == len ? '}' : 0u);
    const uint32_t c0 = cb_b64_char(b0 >> 2), c1 = cb_b64_char(((b0 & 3u) << 4) | (b1 >> 4));
    const uint32_t c2 = i + 1u < slen ? cb_b64_char(((b1 & 15u) << 2) | (b2 >> 6)) : '=';
    const uint32_t c3 = i + 2u < slen ? cb_b64_char(b2 & 63u) : '=';
    return (c0 << 24) | (c1 << 16) | (c2 << 8) | c3;
}
// inner blocks of a record whose result bytes are `len` long (the ipad block not counted)
__host__ __device__ __forceinline__ uint32_t cb_inner_blocks(const CbSign& s, uint32_t len) {
    const uint32_t q = (len + 1u + 2u) / 3u;
    return (3u + q + s.tail_words + 2u + 15u) / 16u;
}
// HMAC-SHA256 of "eyJkYXRhIjog" + base64(R + "}") + ":" + ts for R = r[0, len); out: 8 big-endian digest words
__host__ __device__ inline void cb_sign_record(const CbSign& s, const uint8_t* __restrict__ r, uint32_t len, uint32_t out[8]) {
    const uint32_t q = (len + 1u + 2u) / 3u;                 // base64 words
    const uint32_t tail0 = 3u + q, tail_end = tail0 + s.tail_words;
    const uint32_t blocks = (tail_end + 2u + 15u) / 16u;
    const uint64_t bits = ((uint64_t)64u + 12u + 4ull * q + s.tail_bytes) * 8u;
    uint32_t h[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) h[i] = s.mid[i];
    for (uint32_t b = 0; b < blocks; ++b) {
        uint32_t w[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const uint32_t m = b * 16u + (uint32_t)i;
            uint32_t v;
            if (m >= 3u && m < tail0) v = cb_b64_word(r, len, m - 3u);
            else if (m < 3u) v = m == 0 ? CB_PREFIX_W0 : m == 1 ? CB_PREFIX_W1 : CB_PREFIX_W2;
            else if (m < tail_end) {                                  // (a select chain: no dynamic index, no local copy)
                const uint32_t ti = m - tail0;
                v = s.tail[0];
#pragma unroll
                for (uint32_t x = 1; x < 6; ++x) if (ti == x) v = s.tail[x];
            }
            else if (m == blocks * 16u - 2u) v = (uint32_t)(bits >> 32);
            else if (m == blocks * 16u - 1u) v = (uint32_t)bits;
            else v = 0;
            w[i] = v;
        }
        sha256_compress(h, w);
    }
    cb_outer(s.mid, h, out);
}

// R is a non-finite float: json.dumps wrote NaN / Infinity / -Infinity, which requests refuses to post (allow_nan=False)
__host__ __device__ __forceinline__ bool cb_nonfinite(const uint8_t* r, uint32_t len) {
    auto eq = [&](const char* t, uint32_t n) { if (len != n) return false; for (uint32_t i = 0; i < n; ++i) if (r[i] != (uint8_t)t[i]) return false; return true; };
    return eq("NaN", 3) || eq("Infinity", 8) || eq("-Infinity", 9);
}

// ---- does the handler's kwargs hold a "callback_url" key? ----------------------------------------------------------
// The runner reads override_callback_url = kwargs.get("callback_url"). Only the decoded key matters, as Python sees it
// after Go's re-encoding: Go's unquote (next_cp), compared with the 12 ASCII bytes.
__device__ inline bool cb_key_is_callback_url(const uint8_t* __restrict__ p, uint32_t s, uint32_t e) {
    const char* k = "callback_url";
    uint32_t i = s, n = 0;
    while (i < e) {
        const uint32_t cp = next_cp(p, i, e);
        if (n >= 12 || cp != (uint32_t)(uint8_t)k[n]) return false;
        ++n;
    }
    return n == 12;
}
// the members of a validated object p[s] == '{' .. e: any key "callback_url"?
__device__ inline bool cb_object_has_callback_url(const uint8_t* __restrict__ p, uint32_t s, uint32_t e) {
    uint32_t i = s + 1, f = 0;
    while (i < e && is_ws(p[i])) ++i;
    if (i >= e || p[i] == '}') return false;
    for (;;) {
        const uint32_t ks = i;
        const int64_t ke = scan_string(p, i, e, f); if (ke < 0) return false;
        if (cb_key_is_callback_url(p, ks + 1, (uint32_t)ke - 1)) return true;
        i = (uint32_t)ke;
        while (i < e && is_ws(p[i])) ++i;
        ++i;                                                                           // ':'
        while (i < e && is_ws(p[i])) ++i;
        const int64_t ve = skip_value(p, i, e, f); if (ve < 0) return false;
        i = (uint32_t)ve;
        while (i < e && is_ws(p[i])) ++i;
        if (i >= e || p[i] != ',') return false;
        ++i;
        while (i < e && is_ws(p[i])) ++i;
    }
}
// The kwargs the runner calls the handler with, for a payload the drain parsed (an ERROR's task). mode 0: an SDK put
// payload, Unmarshal into TaskPayload (case-folded "kwargs"; objects merge into the map, null resets it); mode 1: an HTTP
// body (SerializeHttpPayload: the last "kwargs" when it is an object, otherwise the body's remaining keys); mode 2: a
// TaskMessage record (one exact "kwargs", an object or null).
__device__ inline bool cb_kwargs_have_callback_url(const uint8_t* __restrict__ p, uint32_t n, int mode) {
    uint32_t i = 0, f = 0;
    while (i < n && is_ws(p[i])) ++i;
    if (i >= n || p[i] != '{') return false;
    ++i;
    while (i < n && is_ws(p[i])) ++i;
    if (i >= n || p[i] == '}') return false;
    bool found = false, top = false, kw_dict = false;
    for (;;) {
        const uint32_t ks = i;
        const int64_t ke = scan_string(p, i, n, f); if (ke < 0) return false;
        bool is_kw;
        if (mode == 0) is_kw = match_payload_key(p, ks + 1, (uint32_t)ke - 1) == 2;
        else if (mode == 1) { is_kw = match_exact_key(p, ks + 1, (uint32_t)ke - 1) == 2; top |= cb_key_is_callback_url(p, ks + 1, (uint32_t)ke - 1); }
        else is_kw = match_exact_key(p, ks + 1, (uint32_t)ke - 1) == 2;
        i = (uint32_t)ke;
        while (i < n && is_ws(p[i])) ++i;
        ++i;                                                                           // ':'
        while (i < n && is_ws(p[i])) ++i;
        const uint32_t vs = i;
        const int64_t ve = skip_value(p, i, n, f); if (ve < 0) return false;
        i = (uint32_t)ve;
        if (is_kw) {
            const bool obj = p[vs] == '{';
            const bool has = obj && cb_object_has_callback_url(p, vs, i);
            if (mode == 0) found = obj ? (found || has) : false;             // (a null map is reset; an object merges in)
            else if (mode == 1) { kw_dict = obj; found = has; }
            else found = has;
        }
        while (i < n && is_ws(p[i])) ++i;
        if (i >= n || p[i] != ',') break;
        ++i;
        while (i < n && is_ws(p[i])) ++i;
    }
    return mode == 1 ? (kw_dict ? found : top) : found;
}

}  // namespace b9
