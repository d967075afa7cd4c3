// Device-side JSON for the task payload: the deserialise and serialise halves of the hot path.
//
// What is restated here (behaviour only — written from scratch for the GPU):
//   * Go 1.23 encoding/json `Unmarshal` of `TaskQueuePutRequest.payload` into
//     `types.TaskPayload{Args []any; Kwargs map[string]any}`
//       (pkg/abstractions/taskqueue/taskqueue.go:213-214, pkg/types/task.go:13-16):
//     strict RFC 8259 validation of the whole document, case-folded struct keys, duplicate-key
//     rules, string unquoting with U+FFFD substitution for lone surrogates / invalid UTF-8.
//   * CPython `json.dumps` string escaping with ensure_ascii
//       (sdk/src/beta9/runner/common.py:484-489 `serialize_result`).
//   The Go re-encode (pkg/types/task.go:79-90) + runner `json.loads`
//   (sdk/src/beta9/runner/taskqueue.py:196) in between are value-preserving for everything the
//   device handlers accept, so they do not appear as code here; see DESIGN.md §"Why the wire
//   record does not have to be materialised to get the result".
#pragma once
#include <stdint.h>

namespace b9 {

enum ArgKind : uint8_t {
    AK_NONE = 0, AK_STR, AK_INT, AK_NUM, AK_TRUE, AK_FALSE, AK_NULL,
    AK_ARR_EMPTY, AK_ARR, AK_OBJ_EMPTY, AK_OBJ
};

// scan flags
constexpr uint32_t SF_ESC      = 1u << 0;  // string contains a backslash escape
constexpr uint32_t SF_NONPRINT = 1u << 1;  // string contains a byte >= 0x7F
constexpr uint32_t SF_NUM_EXP  = 1u << 2;  // a number with exponent or > 300 digits (may overflow float64)
constexpr uint32_t SF_DEEP     = 1u << 3;  // nesting deeper than the device stack
constexpr uint32_t SF_F64_OVER = 1u << 4;  // a number literal that strconv.ParseFloat rejects with ErrRange

constexpr int ST_OK = 0, ST_REJECTED = 3, ST_UNSUPPORTED = 4;

struct Parsed {
    uint8_t  status;          // ST_OK / ST_REJECTED / ST_UNSUPPORTED
    uint8_t  a0_kind;         // ArgKind of args[0]
    uint8_t  kwargs_nonempty;
    uint8_t  a0_flags;        // SF_* of args[0] when it is a string
    uint32_t nargs;
    uint32_t a0_off, a0_len;  // byte span of args[0]'s token inside the payload
    uint32_t args_off, args_len;   // span of the whole `args` value (last occurrence); len 0 = nil
    uint32_t kw_off, kw_len;       // span of the `kwargs` value; len 0 = nil
    uint8_t  kw_merged;            // kwargs appeared more than once with objects (Go merges the maps)
};

__device__ __forceinline__ bool is_ws(uint8_t c) { return c == ' ' || c == '\t' || c == '\r' || c == '\n'; }
__device__ __forceinline__ int hexval(uint8_t c) {
    if (c >= '0' && c <= '9') return c - '0';
    c |= 0x20;
    if (c >= 'a' && c <= 'f') return c - 'a' + 10;
    return -1;
}
__device__ __forceinline__ bool is_digit(uint8_t c) { return (uint8_t)(c - '0') <= 9; }

// p[i] == '"'. Returns the index just past the closing quote, or -1.
__device__ inline int64_t scan_string(const uint8_t* __restrict__ p, uint32_t i, uint32_t n, uint32_t& flags) {
    ++i;
    while (i < n) {
        uint8_t c = p[i];
        if (c == '"') return (int64_t)i + 1;
        if (c < 0x20) return -1;
        if (c == '\\') {
            flags |= SF_ESC;
            if (i + 1 >= n) return -1;
            uint8_t e = p[i + 1];
            if (e == 'u') {
                if (i + 6 > n) return -1;
                if ((hexval(p[i + 2]) | hexval(p[i + 3]) | hexval(p[i + 4]) | hexval(p[i + 5])) < 0) return -1;
                i += 6;
                continue;
            }
            if (e == '"' || e == '\\' || e == '/' || e == 'b' || e == 'f' || e == 'n' || e == 'r' || e == 't') { i += 2; continue; }
            return -1;
        }
        if (c >= 0x7F) flags |= SF_NONPRINT;
        ++i;
    }
    return -1;
}

// p[i] is '-' or a digit. Returns index past the number or -1. *simple_int: no frac/exp, <= 15 digits.
__device__ inline int64_t scan_number(const uint8_t* __restrict__ p, uint32_t i, uint32_t n, uint32_t& flags, bool* simple_int) {
    uint32_t s = i;
    bool simple = true;
    if (p[i] == '-') ++i;
    if (i >= n) return -1;
    uint32_t d0 = i;
    if (p[i] == '0') ++i;
    else if (p[i] >= '1' && p[i] <= '9') { while (i < n && is_digit(p[i])) ++i; }
    else return -1;
    uint32_t nd = i - d0;
    if (nd > 15) simple = false;
    if (nd > 300) flags |= SF_NUM_EXP;
    if (i < n && p[i] == '.') {
        simple = false; ++i;
        if (i >= n || !is_digit(p[i])) return -1;
        while (i < n && is_digit(p[i])) ++i;
    }
    if (i < n && (p[i] == 'e' || p[i] == 'E')) {
        simple = false; flags |= SF_NUM_EXP; ++i;
        if (i < n && (p[i] == '+' || p[i] == '-')) ++i;
        if (i >= n || !is_digit(p[i])) return -1;
        while (i < n && is_digit(p[i])) ++i;
    }
    (void)s;
    if (simple_int) *simple_int = simple;
    return i;
}


// ---- does a number literal overflow float64 (strconv.ParseFloat ErrRange -> Unmarshal error)? ----
// 2^1024 - 2^970, the smallest decimal that rounds (half-even) to +Inf: 309 digits.
__device__ __constant__ char F64_OVERFLOW_THRESHOLD[310] = {'1','7','9','7','6','9','3','1','3','4','8','6','2','3','1','5','8','0','7','9','3','7','2','8','9','7','1','4','0','5','3','0','3','4','1','5','0','7','9','9','3','4','1','3','2','7','1','0','0','3','7','8','2','6','9','3','6','1','7','3','7','7','8','9','8','0','4','4','4','9','6','8','2','9','2','7','6','4','7','5','0','9','4','6','6','4','9','0','1','7','9','7','7','5','8','7','2','0','7','0','9','6','3','3','0','2','8','6','4','1','6','6','9','2','8','8','7','9','1','0','9','4','6','5','5','5','5','4','7','8','5','1','9','4','0','4','0','2','6','3','0','6','5','7','4','8','8','6','7','1','5','0','5','8','2','0','6','8','1','9','0','8','9','0','2','0','0','0','7','0','8','3','8','3','6','7','6','2','7','3','8','5','4','8','4','5','8','1','7','7','1','1','5','3','1','7','6','4','4','7','5','7','3','0','2','7','0','0','6','9','8','5','5','5','7','1','3','6','6','9','5','9','6','2','2','8','4','2','9','1','4','8','1','9','8','6','0','8','3','4','9','3','6','4','7','5','2','9','2','7','1','9','0','7','4','1','6','8','4','4','4','3','6','5','5','1','0','7','0','4','3','4','2','7','1','1','5','5','9','6','9','9','5','0','8','0','9','3','0','4','2','8','8','0','1','7','7','9','0','4','1','7','4','4','9','7','7','9','2', 0};

// p[s..e) is a syntactically valid JSON number. Exact: compares the literal's significant digits
// against the threshold above when its magnitude is 10^308..10^309, otherwise decides by magnitude.
__device__ inline bool number_overflows_f64(const uint8_t* __restrict__ p, uint32_t s, uint32_t e) {
    uint32_t i = s;
    if (p[i] == '-') ++i;
    // significant digits = integer digits then fraction digits, leading zeros stripped
    uint32_t int_s = i;
    while (i < e && is_digit(p[i])) ++i;
    uint32_t int_e = i, frac_s = i, frac_e = i;
    if (i < e && p[i] == '.') { ++i; frac_s = i; while (i < e && is_digit(p[i])) ++i; frac_e = i; }
    long long ex = 0;
    if (i < e && (p[i] == 'e' || p[i] == 'E')) {
        ++i; bool neg = false;
        if (p[i] == '+') ++i; else if (p[i] == '-') { neg = true; ++i; }
        while (i < e) { if (ex < 100000000) ex = ex * 10 + (p[i] - '0'); ++i; }
        if (neg) ex = -ex;
    }
    // position of the first non-zero digit
    long long mag;                   // value = 0.d1d2.. x 10^mag
    uint32_t k = int_s;
    while (k < int_e && p[k] == '0') ++k;
    uint32_t first_in_frac = 0; bool in_frac = false;
    if (k < int_e) mag = (long long)(int_e - k) + ex;
    else {
        uint32_t z = frac_s;
        while (z < frac_e && p[z] == '0') ++z;
        if (z >= frac_e) return false;                     // the value is zero
        mag = -(long long)(z - frac_s) + ex;
        in_frac = true; first_in_frac = z;
    }
    if (mag <= 308) return false;
    if (mag >= 310) return true;
    // mag == 309: digit-wise compare against the 309-digit threshold (missing digits are zeros)
    uint32_t a = in_frac ? first_in_frac : k;              // walks the literal's digits, skipping '.'
    bool in_int = !in_frac;
    for (uint32_t t = 0; t < 309; ++t) {
        char d = '0';
        if (in_int) { if (a < int_e) d = (char)p[a++]; else { in_int = false; a = frac_s; if (a < frac_e) d = (char)p[a++]; } }
        else if (a < frac_e) d = (char)p[a++];
        char th = F64_OVERFLOW_THRESHOLD[t];
        if (d != th) return d > th;
    }
    return true;                                           // >= threshold in the first 309 digits
}

__device__ inline int64_t scan_literal(const uint8_t* __restrict__ p, uint32_t i, uint32_t n) {
    uint8_t c = p[i];
    if (c == 't') { if (i + 4 <= n && p[i + 1] == 'r' && p[i + 2] == 'u' && p[i + 3] == 'e') return i + 4; return -1; }
    if (c == 'f') { if (i + 5 <= n && p[i + 1] == 'a' && p[i + 2] == 'l' && p[i + 3] == 's' && p[i + 4] == 'e') return i + 5; return -1; }
    if (c == 'n') { if (i + 4 <= n && p[i + 1] == 'u' && p[i + 2] == 'l' && p[i + 3] == 'l') return i + 4; return -1; }
    return -1;
}

// Validates one JSON value whose first byte is p[i] (no leading whitespace); iterative, with the
// container kinds on a 64-entry bit stack. Returns the index past the value or -1 (syntax error).
// Documents nested deeper than 64 set SF_DEEP and are reported UNSUPPORTED by the caller.
__device__ inline int64_t skip_value(const uint8_t* __restrict__ p, uint32_t i, uint32_t n, uint32_t& flags) {
    uint64_t stack = 0;   // bit d: 1 = object at depth d+1
    int depth = 0;
    for (;;) {
        // ---- a value starts at i
        if (i >= n) return -1;
        uint8_t c = p[i];
        bool closed_empty = false;
        if (c == '{' || c == '[') {
            if (depth >= 64) { flags |= SF_DEEP; return -1; }
            stack = (stack << 1) | (c == '{' ? 1u : 0u);
            ++depth; ++i;
            while (i < n && is_ws(p[i])) ++i;
            if (i >= n) return -1;
            if (c == '{') {
                if (p[i] == '}') { ++i; closed_empty = true; }
            } else {
                if (p[i] == ']') { ++i; closed_empty = true; }
                else continue;                      // first array element
            }
            if (closed_empty) { stack >>= 1; --depth; }
        } else if (c == '"') {
            int64_t e = scan_string(p, i, n, flags); if (e < 0) return -1; i = (uint32_t)e;
        } else if (c == '-' || is_digit(c)) {
            uint32_t nf = 0;
            int64_t e = scan_number(p, i, n, nf, nullptr); if (e < 0) return -1;
            if ((nf & SF_NUM_EXP) && number_overflows_f64(p, i, (uint32_t)e)) nf |= SF_F64_OVER;
            flags |= nf; i = (uint32_t)e;
        } else {
            int64_t e = scan_literal(p, i, n); if (e < 0) return -1; i = (uint32_t)e;
        }
        bool need_key = (c == '{') && !closed_empty;
        // ---- after a value (or at the first key of a non-empty object)
        for (;;) {
            if (!need_key) {
                if (depth == 0) return i;
                while (i < n && is_ws(p[i])) ++i;
                if (i >= n) return -1;
                uint8_t d = p[i];
                bool in_obj = stack & 1u;
                if (d == ',') {
                    ++i;
                    while (i < n && is_ws(p[i])) ++i;
                    if (!in_obj) break;             // next array element
                    need_key = true;
                } else if (d == (in_obj ? '}' : ']')) {
                    ++i; stack >>= 1; --depth;
                    continue;
                } else return -1;
            }
            // object key
            if (i >= n || p[i] != '"') return -1;
            int64_t e = scan_string(p, i, n, flags); if (e < 0) return -1; i = (uint32_t)e;
            while (i < n && is_ws(p[i])) ++i;
            if (i >= n || p[i] != ':') return -1;
            ++i;
            while (i < n && is_ws(p[i])) ++i;
            need_key = false;
            break;                                  // value of this key
        }
    }
}

// One code point of a *validated* JSON string body p[i..end), as Go's unquote leaves it:
// escapes resolved, surrogate pairs joined, lone surrogates and invalid UTF-8 -> U+FFFD.
__device__ inline uint32_t next_cp(const uint8_t* __restrict__ p, uint32_t& i, uint32_t end) {
    uint8_t c = p[i];
    if (c == '\\') {
        uint8_t e = p[i + 1];
        if (e != 'u') {
            i += 2;
            switch (e) {
            case 'b': return 8; case 'f': return 12; case 'n': return 10; case 'r': return 13; case 't': return 9;
            default: return e;      // '"' '\\' '/'
            }
        }
        uint32_t r = (hexval(p[i + 2]) << 12) | (hexval(p[i + 3]) << 8) | (hexval(p[i + 4]) << 4) | hexval(p[i + 5]);
        i += 6;
        if (r - 0xD800u < 0x800u) {
            if (r < 0xDC00u && i + 6 <= end && p[i] == '\\' && p[i + 1] == 'u') {
                int h0 = hexval(p[i + 2]), h1 = hexval(p[i + 3]), h2 = hexval(p[i + 4]), h3 = hexval(p[i + 5]);
                if ((h0 | h1 | h2 | h3) >= 0) {
                    uint32_t r1 = (h0 << 12) | (h1 << 8) | (h2 << 4) | h3;
                    if (r1 - 0xDC00u < 0x400u) { i += 6; return 0x10000u + ((r - 0xD800u) << 10) + (r1 - 0xDC00u); }
                }
            }
            return 0xFFFDu;
        }
        return r;
    }
    if (c < 0x80) { ++i; return c; }
    // Go utf8.DecodeRune
    uint32_t rem = end - i;
    if (c >= 0xC2 && c <= 0xDF) {
        if (rem >= 2 && (p[i + 1] & 0xC0) == 0x80) { uint32_t r = ((c & 0x1Fu) << 6) | (p[i + 1] & 0x3Fu); i += 2; return r; }
    } else if (c >= 0xE0 && c <= 0xEF) {
        uint8_t lo = (c == 0xE0) ? 0xA0 : 0x80, hi = (c == 0xED) ? 0x9F : 0xBF;
        if (rem >= 3 && p[i + 1] >= lo && p[i + 1] <= hi && (p[i + 2] & 0xC0) == 0x80) {
            uint32_t r = ((c & 0x0Fu) << 12) | ((p[i + 1] & 0x3Fu) << 6) | (p[i + 2] & 0x3Fu); i += 3; return r;
        }
    } else if (c >= 0xF0 && c <= 0xF4) {
        uint8_t lo = (c == 0xF0) ? 0x90 : 0x80, hi = (c == 0xF4) ? 0x8F : 0xBF;
        if (rem >= 4 && p[i + 1] >= lo && p[i + 1] <= hi && (p[i + 2] & 0xC0) == 0x80 && (p[i + 3] & 0xC0) == 0x80) {
            uint32_t r = ((c & 0x07u) << 18) | ((p[i + 1] & 0x3Fu) << 12) | ((p[i + 2] & 0x3Fu) << 6) | (p[i + 3] & 0x3Fu); i += 4; return r;
        }
    }
    ++i;
    return 0xFFFDu;
}

// decoded keys a (body p[as..ae)) < b, bytewise on their UTF-8 (== code point order): the order Go's encoder
// writes map keys in
__device__ inline bool key_less(const uint8_t* __restrict__ p, uint32_t as, uint32_t ae, uint32_t bs, uint32_t be) {
    uint32_t i = as, j = bs;
    while (i < ae && j < be) {
        uint32_t a = next_cp(p, i, ae), b = next_cp(p, j, be);
        if (a != b) return a < b;
    }
    return i >= ae && j < be;
}

// encoding/json struct-key matching for TaskPayload: 1 = "args", 2 = "kwargs", 0 = neither.
// Exact match or equal under foldName (ASCII case, U+212A -> k, U+017F -> s). body = p[s..e).
__device__ inline int match_payload_key(const uint8_t* __restrict__ p, uint32_t s, uint32_t e) {
    const char A[] = "args", K[] = "kwargs";
    bool ma = true, mk = true;
    uint32_t k = 0, i = s;
    while (i < e) {
        uint32_t cp = next_cp(p, i, e);
        uint32_t f;
        if (cp < 0x80) f = (cp >= 'A' && cp <= 'Z') ? cp + 32 : cp;
        else if (cp == 0x212A) f = 'k';
        else if (cp == 0x017F) f = 's';
        else return 0;
        if (k >= 4 || f != (uint32_t)A[k]) ma = false;
        if (k >= 6 || f != (uint32_t)K[k]) mk = false;
        if (!ma && !mk) return 0;
        ++k;
    }
    if (ma && k == 4) return 1;
    if (mk && k == 6) return 2;
    return 0;
}

// map-key matching for an HTTP body decoded into map[string]interface{} (pkg/task/serialize.go:19-23,48-57):
// the DECODED key must be exactly "args" / "kwargs" — no case folding, that is a struct-field rule.
__device__ inline int match_exact_key(const uint8_t* __restrict__ p, uint32_t s, uint32_t e) {
    const char A[] = "args", K[] = "kwargs";
    bool ma = true, mk = true;
    uint32_t k = 0, i = s;
    while (i < e) {
        const uint32_t cp = next_cp(p, i, e);
        if (k >= 4 || cp != (uint32_t)A[k]) ma = false;
        if (k >= 6 || cp != (uint32_t)K[k]) mk = false;
        if (!ma && !mk) return 0;
        ++k;
    }
    if (ma && k == 4) return 1;
    if (mk && k == 6) return 2;
    return 0;
}

__device__ inline bool only_ws(const uint8_t* __restrict__ p, uint32_t s, uint32_t e) {
    for (uint32_t i = s; i < e; ++i) if (!is_ws(p[i])) return false;
    return true;
}

// Full, sequential (one thread) parse of a payload. The warp-level fast path in the drain kernel
// recognises the SDK's canonical frame without calling this; everything else lands here.
//
// http = false: TaskQueuePutRequest.payload, json.Unmarshal into the TaskPayload STRUCT (taskqueue.go:213-214).
// http = true (B9_TF_HTTP_BODY): an HTTP request body, SerializeHttpPayload (pkg/task/serialize.go:16-101) —
//   decoded into a MAP first: exact keys; "args" counts only if it is a list, "kwargs" only if it is an object,
//   otherwise every remaining key of the body becomes a keyword argument; an empty body is an empty payload;
//   every number of the document is converted (an overflow anywhere refuses the request).
__device__ inline Parsed parse_payload(const uint8_t* __restrict__ p, uint32_t n, bool http = false) {
    Parsed r; r.status = ST_OK; r.a0_kind = AK_NONE; r.kwargs_nonempty = 0; r.a0_flags = 0; r.nargs = 0; r.a0_off = 0; r.a0_len = 0;
    r.args_off = r.args_len = r.kw_off = r.kw_len = 0; r.kw_merged = 0;
    uint32_t i = 0, sub_flags = 0;
    // http: does the body's map still hold keys once "args" (a list) and "kwargs" (an object) are taken out?
    bool args_left = false, kwargs_left = false, others_left = false, kw_is_dict = false;
#define B9_REJECT() do { r.status = (sub_flags & SF_DEEP) ? ST_UNSUPPORTED : ST_REJECTED; return r; } while (0)
    while (i < n && is_ws(p[i])) ++i;
    if (i >= n) { if (http) return r; B9_REJECT(); }            // serialize.go:22-25 tolerates io.EOF: empty payload
    if (p[i] != '{') {
        // top-level null is a no-op for Unmarshal; any other value is a type or syntax error
        if (p[i] == 'n' && scan_literal(p, i, n) == (int64_t)i + 4) {
            i += 4;
            while (i < n && is_ws(p[i])) ++i;
            if (i == n) return r;
        }
        B9_REJECT();
    }
    ++i;
    while (i < n && is_ws(p[i])) ++i;
    if (i >= n) B9_REJECT();
    if (p[i] == '}') ++i;
    else for (;;) {
        if (i >= n || p[i] != '"') B9_REJECT();
        uint32_t kf = 0;
        uint32_t ks = i;
        int64_t e = scan_string(p, i, n, kf); if (e < 0) B9_REJECT();
        i = (uint32_t)e;
        int which = http ? match_exact_key(p, ks + 1, i - 1) : match_payload_key(p, ks + 1, i - 1);
        while (i < n && is_ws(p[i])) ++i;
        if (i >= n || p[i] != ':') B9_REJECT();
        ++i;
        while (i < n && is_ws(p[i])) ++i;
        if (i >= n) B9_REJECT();
        if (which == 1) {                                   // Args []interface{}
            if (p[i] == '[') {
                const uint32_t arr_start = i;
                ++i;
                uint32_t cnt = 0;
                r.a0_kind = AK_NONE; r.a0_flags = 0;
                while (i < n && is_ws(p[i])) ++i;
                if (i >= n) B9_REJECT();
                if (p[i] == ']') ++i;
                else for (;;) {
                    if (i >= n) B9_REJECT();
                    uint32_t es = i, ef = 0; uint8_t c = p[i]; bool simple = false;
                    int64_t ee;
                    if (c == '-' || is_digit(c)) {
                        ee = scan_number(p, i, n, ef, &simple);
                        if (ee >= 0 && (ef & SF_NUM_EXP) && number_overflows_f64(p, i, (uint32_t)ee)) ef |= SF_F64_OVER;
                    } else ee = skip_value(p, i, n, ef);
                    sub_flags |= ef & (SF_F64_OVER | SF_DEEP);
                    if (ee < 0) B9_REJECT();
                    i = (uint32_t)ee;
                    if (cnt == 0) {
                        r.a0_off = es; r.a0_len = i - es; r.a0_flags = (uint8_t)(ef & (SF_ESC | SF_NONPRINT));
                        switch (c) {
                        case '"': r.a0_kind = AK_STR; break;
                        case '{': r.a0_kind = only_ws(p, es + 1, i - 1) ? AK_OBJ_EMPTY : AK_OBJ; break;
                        case '[': r.a0_kind = only_ws(p, es + 1, i - 1) ? AK_ARR_EMPTY : AK_ARR; break;
                        case 't': r.a0_kind = AK_TRUE; break;
                        case 'f': r.a0_kind = AK_FALSE; break;
                        case 'n': r.a0_kind = AK_NULL; break;
                        default: r.a0_kind = simple ? AK_INT : AK_NUM; break;
                        }
                    }
                    ++cnt;
                    while (i < n && is_ws(p[i])) ++i;
                    if (i >= n) B9_REJECT();
                    if (p[i] == ',') { ++i; while (i < n && is_ws(p[i])) ++i; continue; }
                    if (p[i] == ']') { ++i; break; }
                    B9_REJECT();
                }
                r.nargs = cnt; r.args_off = arr_start; r.args_len = i - arr_start;
                args_left = false;
            } else if (http) {                              // "args" that is not a list stays in the map (a later "args" replaces it)
                uint32_t ef = 0;
                int64_t ee = skip_value(p, i, n, ef);
                sub_flags |= ef & (SF_F64_OVER | SF_DEEP);
                if (ee < 0) B9_REJECT();
                i = (uint32_t)ee;
                r.nargs = 0; r.a0_kind = AK_NONE; r.args_len = 0; args_left = true;
            } else if (p[i] == 'n' && scan_literal(p, i, n) >= 0) {
                i += 4; r.nargs = 0; r.a0_kind = AK_NONE; r.args_len = 0;
            } else B9_REJECT();                             // UnmarshalTypeError or syntax error
        } else if (which == 2) {                            // Kwargs map[string]interface{}
            if (p[i] == '{') {
                uint32_t vs = i, ef = 0;
                int64_t ee = skip_value(p, i, n, ef);
                sub_flags |= ef & (SF_F64_OVER | SF_DEEP);
                if (ee < 0) B9_REJECT();
                i = (uint32_t)ee;
                if (!only_ws(p, vs + 1, i - 1)) r.kwargs_nonempty = 1;   // a non-nil map is merged into
                if (http) { r.kwargs_nonempty = only_ws(p, vs + 1, i - 1) ? 0 : 1; kw_is_dict = true; kwargs_left = false; }   // map value: the last one wins
                else if (r.kw_len) r.kw_merged = 1;
                r.kw_off = vs; r.kw_len = i - vs;
            } else if (http) {                              // "kwargs" that is not an object stays in the map
                uint32_t ef = 0;
                int64_t ee = skip_value(p, i, n, ef);
                sub_flags |= ef & (SF_F64_OVER | SF_DEEP);
                if (ee < 0) B9_REJECT();
                i = (uint32_t)ee;
                kw_is_dict = false; kwargs_left = true; r.kw_len = 0;
            } else if (p[i] == 'n' && scan_literal(p, i, n) >= 0) {
                i += 4; r.kwargs_nonempty = 0; r.kw_len = 0; r.kw_merged = 0;
            } else B9_REJECT();
        } else {
            uint32_t ef = 0;
            int64_t ee = skip_value(p, i, n, ef);
            sub_flags |= ef & (http ? (SF_DEEP | SF_F64_OVER) : SF_DEEP);   // struct: numbers under ignored keys are never converted; map: all are
            if (ee < 0) B9_REJECT();
            i = (uint32_t)ee;
            others_left = true;
        }
        while (i < n && is_ws(p[i])) ++i;
        if (i >= n) B9_REJECT();
        if (p[i] == ',') { ++i; while (i < n && is_ws(p[i])) ++i; continue; }
        if (p[i] == '}') { ++i; break; }
        B9_REJECT();
    }
    while (i < n && is_ws(p[i])) ++i;
    if (i != n) B9_REJECT();
#undef B9_REJECT
    if (sub_flags & SF_F64_OVER) r.status = ST_REJECTED;     // "number out of range": Unmarshal error -> Ok:false
    if (http && !kw_is_dict) r.kwargs_nonempty = (args_left || kwargs_left || others_left) ? 1 : 0;   // serialize.go:57-60
    return r;
}

// ---- CPython json.dumps(str), ensure_ascii ----------------------------------------------------
__device__ __forceinline__ uint32_t py_escaped_len(uint32_t cp) {
    if (cp >= 0x20 && cp <= 0x7E) return (cp == '"' || cp == '\\') ? 2u : 1u;
    if (cp == '\n' || cp == '\r' || cp == '\t' || cp == '\b' || cp == '\f') return 2u;
    return cp >= 0x10000u ? 12u : 6u;
}

__device__ __forceinline__ uint8_t hexdig(uint32_t v) { return (uint8_t)(v < 10 ? '0' + v : 'a' + (v - 10)); }

__device__ inline uint32_t py_emit(uint32_t cp, uint8_t* __restrict__ o) {
    if (cp >= 0x20 && cp <= 0x7E) {
        if (cp == '"' || cp == '\\') { o[0] = '\\'; o[1] = (uint8_t)cp; return 2; }
        o[0] = (uint8_t)cp; return 1;
    }
    uint8_t sc = 0;
    switch (cp) { case '\n': sc = 'n'; break; case '\r': sc = 'r'; break; case '\t': sc = 't'; break; case '\b': sc = 'b'; break; case '\f': sc = 'f'; break; }
    if (sc) { o[0] = '\\'; o[1] = sc; return 2; }
    uint32_t u0 = cp, u1 = 0; uint32_t nu = 1;
    if (cp >= 0x10000u) { uint32_t x = cp - 0x10000u; u0 = 0xD800u | (x >> 10); u1 = 0xDC00u | (x & 0x3FFu); nu = 2; }
    for (uint32_t k = 0; k < nu; ++k) {
        uint32_t u = k ? u1 : u0;
        o[0] = '\\'; o[1] = 'u'; o[2] = hexdig((u >> 12) & 15); o[3] = hexdig((u >> 8) & 15); o[4] = hexdig((u >> 4) & 15); o[5] = hexdig(u & 15);
        o += 6;
    }
    return nu * 6;
}

}  // namespace b9
