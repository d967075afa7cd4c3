// TaskMessage records (B9_TF_TASK_MSG): the runner's half of the loop on the bytes TaskQueuePop hands over as
// `task_msg` (pkg/abstractions/taskqueue/taskqueue.go:238-309), i.e. what TaskMessage.Encode wrote
// (pkg/types/task.go:79-90). The runner does json.loads(task_msg), handler(*(args or []), **(kwargs or {})) and
// serialize_result (sdk/src/beta9/runner/taskqueue.py:196-201,349-378).
//
// The device answers a record only inside a domain on which CPython's reading of the record equals CPython's reading
// of Go's re-encoding of Go's decoding of it -- the value the payload handlers already compute -- so that the parse
// below fills the same `Parsed` as parse_payload and handler_phase_a runs unchanged:
//   * the whole record is UTF-8 as json.loads(bytes) decodes it ("surrogatepass");
//   * it is one JSON object as Python's strict decoder reads it, whose keys "task_id", "args" and "kwargs" each
//     appear exactly once (matched exactly; a top-level key with an escape is declined); other members are only
//     validated (exponent literals and nesting beyond 64 declined);
//   * task_id is the canonical lower-case text of the slot's 16-byte id; args is a list or null, kwargs an object
//     or null;
//   * inside args and kwargs: no lone-surrogate escape and no UTF-8-encoded surrogate in a string, every number is
//     exactly the text Go's float encoder writes for its float64, object keys strictly increase in Go's key order.
// Everything else is ST_UNSUPPORTED (never REJECTED: the task exists). Plain C++ behind CUDA qualifiers: the host
// shim tests/host_shim/task_msg_shim.cpp compiles it for the CPU tests.
#pragma once
#include <stdint.h>
#include "json_device.cuh"
#include "f64_device.cuh"

namespace b9 {

// UTF-8 as Python decodes it with "surrogatepass" (a pickled str, json.loads of bytes): the 3-byte encodings of
// U+D800..DFFF are accepted
__device__ __noinline__ bool utf8_valid_surrogatepass(const uint8_t* __restrict__ b, uint32_t n) {
    uint32_t i = 0;
    while (i < n) {
        const uint8_t c = b[i];
        if (c < 0x80) { ++i; continue; }
        if (c >= 0xC2 && c <= 0xDF) { if (i + 2 > n || (b[i + 1] & 0xC0) != 0x80) return false; i += 2; continue; }
        if (c >= 0xE0 && c <= 0xEF) {
            if (i + 3 > n) return false;
            const uint8_t lo = c == 0xE0 ? 0xA0 : 0x80;
            if (b[i + 1] < lo || b[i + 1] > 0xBF || (b[i + 2] & 0xC0) != 0x80) return false;
            i += 3; continue;
        }
        if (c >= 0xF0 && c <= 0xF4) {
            if (i + 4 > n) return false;
            const uint8_t lo = c == 0xF0 ? 0x90 : 0x80, hi = c == 0xF4 ? 0x8F : 0xBF;
            if (b[i + 1] < lo || b[i + 1] > hi || (b[i + 2] & 0xC0) != 0x80 || (b[i + 3] & 0xC0) != 0x80) return false;
            i += 4; continue;
        }
        return false;
    }
    return true;
}

// p[s, s + 36) is the canonical 8-4-4-4-12 lower-case text of the 16 raw id bytes (gofrs/uuid String())
__device__ inline bool uuid_text_matches(const uint8_t* __restrict__ p, uint32_t s, const uint8_t* __restrict__ id) {
    uint32_t k = s;
    for (int b = 0; b < 16; ++b) {
        if (b == 4 || b == 6 || b == 8 || b == 10) { if (p[k] != '-') return false; ++k; }
        if (p[k] != hexdig(id[b] >> 4) || p[k + 1] != hexdig(id[b] & 15u)) return false;
        k += 2;
    }
    return true;
}

// a validated string body p[s, e): no lone-surrogate escape, no UTF-8-encoded surrogate (ED A0..BF). Go would put
// U+FFFD in their place, Python keeps them.
__device__ inline bool task_msg_string_in_domain(const uint8_t* __restrict__ p, uint32_t s, uint32_t e) {
    uint32_t i = s;
    while (i < e) {
        const uint8_t c = p[i];
        if (c == '\\') {
            if (p[i + 1] != 'u') { i += 2; continue; }
            const uint32_t r = (hexval(p[i + 2]) << 12) | (hexval(p[i + 3]) << 8) | (hexval(p[i + 4]) << 4) | hexval(p[i + 5]);
            i += 6;
            if (r - 0xDC00u < 0x400u) return false;                              // a low surrogate nobody paired
            if (r - 0xD800u < 0x400u) {
                if (i + 6 > e || p[i] != '\\' || p[i + 1] != 'u') return false;
                const uint32_t r1 = (hexval(p[i + 2]) << 12) | (hexval(p[i + 3]) << 8) | (hexval(p[i + 4]) << 4) | hexval(p[i + 5]);
                if (r1 - 0xDC00u >= 0x400u) return false;
                i += 6;
            }
            continue;
        }
        if (c == 0xED && i + 1 < e && p[i + 1] >= 0xA0) return false;
        ++i;
    }
    return true;
}

// a valid number literal p[s, e) is exactly what Go's float encoder writes for its float64 value
__device__ inline bool task_msg_number_in_domain(const uint8_t* __restrict__ p, uint32_t s, uint32_t e) {
    if (e - s > 32u) return false;
    unsigned long long b = 0;
    if (!f64_parse(p, s, e, &b) || ((b >> 52) & 0x7FFull) == 0x7FFull) return false;
    uint8_t t[32];
    const uint32_t n = go_json_float(b, t);
    if (n != e - s) return false;
    for (uint32_t k = 0; k < n; ++k) if (t[k] != p[s + k]) return false;
    return true;
}

// The domain checks of args / kwargs: a walk over the value p[s, e) that skip_value accepted (so the bracket
// structure is sound and nesting is at most 64 below the list or object itself).
constexpr int TASK_MSG_MAX_DEPTH = 66;
__device__ __noinline__ bool task_msg_value_in_domain(const uint8_t* __restrict__ p, uint32_t s, uint32_t e) {
    uint32_t lks[TASK_MSG_MAX_DEPTH], lke[TASK_MSG_MAX_DEPTH];   // per open object: body of its previous key (lke 0: none yet)
    uint64_t obj_lo = 0, obj_hi = 0;                             // bit d: the container at depth d is an object
    int depth = 0;
    bool key_next = false;
    uint32_t i = s;
    while (i < e) {
        const uint8_t c = p[i];
        if (c == '{' || c == '[') {
            if (depth >= TASK_MSG_MAX_DEPTH) return false;
            const uint64_t bit = 1ull << (depth & 63);
            if (depth < 64) obj_lo = (c == '{') ? (obj_lo | bit) : (obj_lo & ~bit);
            else            obj_hi = (c == '{') ? (obj_hi | bit) : (obj_hi & ~bit);
            lke[depth] = 0;
            ++depth; key_next = c == '{'; ++i;
        } else if (c == '}' || c == ']') {
            --depth; key_next = false; ++i;
        } else if (c == ',') {
            const int d = depth - 1;
            key_next = ((d < 64 ? obj_lo : obj_hi) >> (d & 63)) & 1ull;
            ++i;
        } else if (c == ':' || is_ws(c)) {
            ++i;
        } else if (c == '"') {
            uint32_t f = 0;
            const int64_t q = scan_string(p, i, e, f);
            if (q < 0 || !task_msg_string_in_domain(p, i + 1, (uint32_t)q - 1)) return false;
            if (key_next) {
                const int d = depth - 1;
                if (lke[d] && !key_less(p, lks[d], lke[d], i + 1, (uint32_t)q - 1)) return false;   // unsorted or duplicate
                lks[d] = i + 1; lke[d] = (uint32_t)q - 1;
                key_next = false;
            }
            i = (uint32_t)q;
        } else if (c == '-' || is_digit(c)) {
            uint32_t f = 0;
            const int64_t q = scan_number(p, i, e, f, nullptr);
            if (q < 0 || !task_msg_number_in_domain(p, i, (uint32_t)q)) return false;
            i = (uint32_t)q;
        } else {
            const int64_t q = scan_literal(p, i, e);
            if (q < 0) return false;
            i = (uint32_t)q;
        }
    }
    return depth == 0;
}

__device__ inline bool bytes_eq(const uint8_t* __restrict__ p, uint32_t s, const char* k, uint32_t n) {
    for (uint32_t j = 0; j < n; ++j) if (p[s + j] != (uint8_t)k[j]) return false;
    return true;
}

// Sequential (one thread) parse of a TaskMessage record against the slot's id: the same Parsed as parse_payload
// gives for the payload the record was made from. status is ST_OK or ST_UNSUPPORTED.
__device__ __noinline__ Parsed parse_task_msg(const uint8_t* __restrict__ p, uint32_t n, const uint8_t* __restrict__ id) {
    Parsed r; r.status = ST_UNSUPPORTED; r.a0_kind = AK_NONE; r.kwargs_nonempty = 0; r.a0_flags = 0; r.nargs = 0; r.a0_off = 0; r.a0_len = 0;
    r.args_off = r.args_len = r.kw_off = r.kw_len = 0; r.kw_merged = 0;
    if (!utf8_valid_surrogatepass(p, n)) return r;
    uint32_t i = 0, seen_id = 0, seen_args = 0, seen_kw = 0;
    while (i < n && is_ws(p[i])) ++i;
    if (i >= n || p[i] != '{') return r;
    ++i;
    while (i < n && is_ws(p[i])) ++i;
    for (;;) {
        if (i >= n || p[i] != '"') return r;                                // (an empty object lacks the keys)
        uint32_t kf = 0;
        const uint32_t ks = i;
        const int64_t ke = scan_string(p, i, n, kf);
        if (ke < 0 || (kf & SF_ESC)) return r;
        i = (uint32_t)ke;
        const uint32_t kl = i - ks - 2;
        const int which = (kl == 7 && bytes_eq(p, ks + 1, "task_id", 7)) ? 1 : (kl == 4 && bytes_eq(p, ks + 1, "args", 4)) ? 2
                        : (kl == 6 && bytes_eq(p, ks + 1, "kwargs", 6)) ? 3 : 0;
        while (i < n && is_ws(p[i])) ++i;
        if (i >= n || p[i] != ':') return r;
        ++i;
        while (i < n && is_ws(p[i])) ++i;
        if (i >= n) return r;
        if (which == 1) {
            if (seen_id++) return r;
            if (p[i] != '"' || i + 38u > n || p[i + 37] != '"' || !uuid_text_matches(p, i + 1, id)) return r;
            i += 38;
        } else if (which == 2) {
            if (seen_args++) return r;
            if (p[i] == '[') {
                const uint32_t arr_start = i;
                uint32_t cnt = 0;
                ++i;
                while (i < n && is_ws(p[i])) ++i;
                if (i >= n) return r;
                if (p[i] == ']') ++i;
                else for (;;) {
                    if (i >= n) return r;
                    const uint32_t es = i; uint32_t ef = 0; const uint8_t c = p[i]; bool simple = false;
                    const int64_t ee = (c == '-' || is_digit(c)) ? scan_number(p, i, n, ef, &simple) : skip_value(p, i, n, ef);
                    if (ee < 0) return r;
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
                    if (i >= n) return r;
                    if (p[i] == ',') { ++i; while (i < n && is_ws(p[i])) ++i; continue; }
                    if (p[i] == ']') { ++i; break; }
                    return r;
                }
                r.nargs = cnt; r.args_off = arr_start; r.args_len = i - arr_start;
            } else if (p[i] == 'n' && scan_literal(p, i, n) >= 0) {
                i += 4;                                                     // None: `args or []`
            } else return r;                                                // *args of a str / dict / number: declined
        } else if (which == 3) {
            if (seen_kw++) return r;
            if (p[i] == '{') {
                const uint32_t vs = i; uint32_t ef = 0;
                const int64_t ee = skip_value(p, i, n, ef);
                if (ee < 0) return r;
                i = (uint32_t)ee;
                r.kwargs_nonempty = only_ws(p, vs + 1, i - 1) ? 0 : 1;
                r.kw_off = vs; r.kw_len = i - vs;
            } else if (p[i] == 'n' && scan_literal(p, i, n) >= 0) {
                i += 4;                                                     // None: `kwargs or {}`
            } else return r;
        } else {
            uint32_t ef = 0;
            const int64_t ee = skip_value(p, i, n, ef);
            if (ee < 0 || (ef & SF_NUM_EXP)) return r;                      // (an exponent or a > 300-digit literal: int() limits)
            i = (uint32_t)ee;
        }
        while (i < n && is_ws(p[i])) ++i;
        if (i >= n) return r;
        if (p[i] == ',') { ++i; while (i < n && is_ws(p[i])) ++i; continue; }
        if (p[i] == '}') { ++i; break; }
        return r;
    }
    while (i < n && is_ws(p[i])) ++i;
    if (i != n || !seen_id || !seen_args || !seen_kw) return r;
    if (r.args_len && !task_msg_value_in_domain(p, r.args_off, r.args_off + r.args_len)) return r;
    if (r.kw_len && !task_msg_value_in_domain(p, r.kw_off, r.kw_off + r.kw_len)) return r;
    r.status = ST_OK;
    return r;
}

}  // namespace b9
