// The sequential (one thread per task) half of the drain: what a parsed payload means to each handler
// (phase A: status, result size, how the bytes will be produced) and the byte producers that are not plain
// copies (phase B). No CUDA builtins in here: tests/host_shim/host_parse.cpp compiles this file, the parser
// and the handlers for the host, so that the device's slow path is fuzzed against the oracle on a CPU
// (tests/test_device_parser_on_host.py). The warp-cooperative fast paths live in drain2.cuh.
#pragma once
#include <stdint.h>
#include "json_device.cuh"
#include "handlers_device.cuh"

namespace b9 {

// what phase A leaves for phase B, per task of the tile
enum OutMode : uint8_t { OM_NONE = 0, OM_COPY, OM_STR_ESC /* one thread walks the token */, OM_U32_DEC, OM_I64_DEC, OM_VADD,
                         OM_STR_PAR /* warp transcodes the framed body in 32 chunks (drain2) */,
                         OM_DEFER /* identity main kernel: left to drain_slow_kernel */,
                         OM_PY_NUM /* identity of a number: py_json_go_number(value) */,
                         OM_PY_FLOAT /* json_sum's float result: py_json_float(value) */,
                         OM_PY_VALUE /* identity of a non-empty list / object: py_value_json over the token */ };
struct TaskRec {
    uint32_t src_off;    // OM_COPY / OM_STR_ESC / OM_VADD / OM_PY_VALUE: byte offset inside the payload
    uint32_t src_len;
    uint32_t out_len;
    uint8_t  status, has, mode, ready;
    long long value;     // OM_U32_DEC / OM_I64_DEC; the float64's bits for OM_PY_NUM / OM_PY_FLOAT; status ERROR: the
                         // exception class the handler raised (one EXC_* bit), for the retry policy (retry_settle)
};

// the exception classes of include/b9gpu.h's B9_EXC_* (the retry policy matches them exactly, as retry_on_errors does)
constexpr uint8_t EXC_TYPE = 0x01, EXC_ATTRIBUTE = 0x02, EXC_UNICODE_ENCODE = 0x04, EXC_KEY = 0x08, EXC_VALUE = 0x10, EXC_BINASCII = 0x20;

// base64.b64decode(s, validate=True) of a str that is not valid base64: `s.encode('ascii')` comes first, so a non-ASCII
// character anywhere is ValueError, otherwise binascii.Error. p[s..e) is the validated string token, quotes included.
__device__ inline uint8_t b64_str_error_class(const uint8_t* __restrict__ p, uint32_t s, uint32_t e) {
    uint32_t i = s + 1;
    while (i < e - 1) if (next_cp(p, i, e - 1) >= 0x80) return EXC_VALUE;
    return EXC_BINASCII;
}

// String token p[s..e) (quotes included, validated): does the Python-escaped form equal a plain
// copy?  Computes the json.dumps length either way. One thread.
__device__ inline uint32_t py_string_len(const uint8_t* __restrict__ p, uint32_t s, uint32_t e) {
    uint32_t i = s + 1, end = e - 1, out = 2;
    while (i < end) out += py_escaped_len(next_cp(p, i, end));
    return out;
}
__device__ inline uint32_t py_string_write(const uint8_t* __restrict__ p, uint32_t s, uint32_t e, uint8_t* __restrict__ o) {
    uint32_t i = s + 1, end = e - 1, n = 1;
    o[0] = '"';
    while (i < end) n += py_emit(next_cp(p, i, end), o + n);
    o[n] = '"';
    return n + 1;
}

// Go's encoding/json of a string token p[s..e) (quotes included, validated) as Go decoded it: go_emit per code point
__device__ inline uint32_t go_string_len(const uint8_t* __restrict__ p, uint32_t s, uint32_t e) {
    uint32_t i = s + 1, end = e - 1, out = 2;
    while (i < end) out += go_emit_len(next_cp(p, i, end));
    return out;
}
__device__ inline uint32_t go_string_write(const uint8_t* __restrict__ p, uint32_t s, uint32_t e, uint8_t* __restrict__ o) {
    uint32_t i = s + 1, end = e - 1, n = 1;
    o[0] = '"';
    while (i < end) n += go_emit(next_cp(p, i, end), o + n);
    o[n] = '"';
    return n + 1;
}

// How value_json writes what the walk visits: separators, strings (token with its quotes), numbers (o == nullptr: size)
struct PyJsonWriter {       // CPython json.dumps (ensure_ascii, separators ", " / ": ") of what json.loads makes of Go's text
    static constexpr bool SPACED = true;
    __device__ static __forceinline__ uint32_t string_len(const uint8_t* __restrict__ p, uint32_t s, uint32_t e) { return py_string_len(p, s, e); }
    __device__ static __forceinline__ uint32_t string_write(const uint8_t* __restrict__ p, uint32_t s, uint32_t e, uint8_t* __restrict__ o) {
        return py_string_write(p, s, e, o);
    }
    __device__ static __forceinline__ uint32_t number(unsigned long long bits, uint8_t* o) { return py_json_go_number(bits, o); }
};
struct GoJsonWriter {       // Go encoding/json (TaskMessage.Encode): no white space, HTML-safe strings, float64 text
    static constexpr bool SPACED = false;
    __device__ static __forceinline__ uint32_t string_len(const uint8_t* __restrict__ p, uint32_t s, uint32_t e) { return go_string_len(p, s, e); }
    __device__ static __forceinline__ uint32_t string_write(const uint8_t* __restrict__ p, uint32_t s, uint32_t e, uint8_t* __restrict__ o) {
        return go_string_write(p, s, e, o);
    }
    __device__ static __forceinline__ uint32_t number(unsigned long long bits, uint8_t* o) { return go_json_float(bits, o); }
};

// The value Go decodes from the validated, non-empty JSON list or object p[s..e), written by W: object members in Go's
// map order -- keys sorted bytewise by their decoded UTF-8 (escapes resolved, invalid UTF-8 and lone surrogates as
// U+FFFD), the last of duplicate keys winning. That order needs no storage: each step scans the object for the
// smallest key after the one emitted last (among equal keys the last occurrence), which is quadratic in the member
// count. drop_args: leave out the top-level object's member "args" (exact decoded key; an HTTP body's remaining map).
// o == nullptr: size only. Returns the byte count, or -1 where the device DECLINES: nesting deeper than
// PY_VALUE_MAX_DEPTH, an object with more than PY_VALUE_MAX_MEMBERS members, a number f64_parse cannot settle.
// Instantiated out of line below: py_value_json (identity's result) and go_value_json (the wire record).
constexpr int PY_VALUE_MAX_DEPTH = 16;
constexpr uint32_t PY_VALUE_MAX_MEMBERS = 64;
template <class W>
__device__ __forceinline__ int64_t value_json(const uint8_t* __restrict__ p, uint32_t s, uint32_t e, uint8_t* __restrict__ o, bool drop_args) {
    uint32_t pos[PY_VALUE_MAX_DEPTH];              // list: the next element (or ','); object: just past its '{'
    uint32_t lks[PY_VALUE_MAX_DEPTH], lke[PY_VALUE_MAX_DEPTH];   // object: body of the key emitted last
    uint32_t is_obj = 0, started = 0;              // bit d: the container at depth d is an object / has emitted a member
    int depth = 0;
    int64_t n = 0;
    uint32_t vs = s, ve = e;                       // the value to emit next
    bool have = true;
    for (;;) {
        if (have) {
            have = false;
            const uint8_t c = p[vs];
            if (c == '{' || c == '[') {
                if (o) o[n] = c;
                ++n;
                if (only_ws(p, vs + 1, ve - 1)) { if (o) o[n] = (c == '{') ? '}' : ']'; ++n; }
                else {
                    if (depth == PY_VALUE_MAX_DEPTH) return -1;
                    const uint32_t bit = 1u << depth;
                    pos[depth] = vs + 1; started &= ~bit;
                    if (c == '{') is_obj |= bit; else is_obj &= ~bit;
                    ++depth;
                }
            } else if (c == '"') n += o ? W::string_write(p, vs, ve, o + n) : W::string_len(p, vs, ve);
            else if (c == 't' || c == 'n') { if (o) for (int k = 0; k < 4; ++k) o[n + k] = p[vs + k]; n += 4; }
            else if (c == 'f') { if (o) for (int k = 0; k < 5; ++k) o[n + k] = p[vs + k]; n += 5; }
            else {
                unsigned long long b = 0;
                if (!f64_parse(p, vs, ve, &b)) return -1;
                n += W::number(b, o ? o + n : nullptr);
            }
        }
        if (depth == 0) return n;
        const int d = depth - 1;
        const uint32_t bit = 1u << d;
        uint32_t f = 0;
        if (!(is_obj & bit)) {                     // list: the next element in order
            uint32_t i = pos[d];
            while (is_ws(p[i])) ++i;
            if (p[i] == ']') { if (o) o[n] = ']'; ++n; --depth; continue; }
            if (p[i] == ',') { ++i; while (is_ws(p[i])) ++i; }
            if (started & bit) { if (o) { o[n] = ','; if (W::SPACED) o[n + 1] = ' '; } n += W::SPACED ? 2 : 1; }
            started |= bit;
            vs = i; ve = (uint32_t)skip_value(p, i, e, f); pos[d] = ve; have = true;
            continue;
        }
        // object: the smallest key after the last one emitted
        uint32_t i = pos[d], members = 0, bks = 0, bke = 0, bvs = 0, bve = 0;
        bool found = false;
        for (;;) {
            while (is_ws(p[i])) ++i;
            if (p[i] == '}') break;
            if (p[i] == ',') { ++i; while (is_ws(p[i])) ++i; }
            const uint32_t ks = i;
            i = (uint32_t)scan_string(p, i, e, f);
            const uint32_t ke = i;
            while (is_ws(p[i])) ++i;
            ++i;                                   // ':'
            while (is_ws(p[i])) ++i;
            const uint32_t v0 = i;
            i = (uint32_t)skip_value(p, i, e, f);
            if (++members > PY_VALUE_MAX_MEMBERS) return -1;
            if ((started & bit) && !key_less(p, lks[d], lke[d], ks + 1, ke - 1)) continue;   // emitted already
            if (drop_args && d == 0 && match_exact_key(p, ks + 1, ke - 1) == 1) continue;
            if (!found || !key_less(p, bks + 1, bke - 1, ks + 1, ke - 1)) { found = true; bks = ks; bke = ke; bvs = v0; bve = i; }
        }
        if (!found) { if (o) o[n] = '}'; ++n; --depth; continue; }
        if (started & bit) { if (o) { o[n] = ','; if (W::SPACED) o[n + 1] = ' '; } n += W::SPACED ? 2 : 1; }
        started |= bit;
        lks[d] = bks + 1; lke[d] = bke - 1;
        n += o ? W::string_write(p, bks, bke, o + n) : W::string_len(p, bks, bke);
        if (o) { o[n] = ':'; if (W::SPACED) o[n + 1] = ' '; }
        n += W::SPACED ? 2 : 1;
        vs = bvs; ve = bve; have = true;
    }
}
// json.dumps of the value as the runner's json.loads reads it back from Go's encoding (identity's result)
__device__ __noinline__ int64_t py_value_json(const uint8_t* __restrict__ p, uint32_t s, uint32_t e, uint8_t* __restrict__ o) {
    return value_json<PyJsonWriter>(p, s, e, o, false);
}
// Go's json.Marshal of the value (TaskMessage.Encode's args / kwargs)
__device__ __noinline__ int64_t go_value_json(const uint8_t* __restrict__ p, uint32_t s, uint32_t e, uint8_t* __restrict__ o, bool drop_args) {
    return value_json<GoJsonWriter>(p, s, e, o, drop_args);
}

// Lane 0: classify args[0] for the handler and fill the record. `pr` is the parse of the payload.
__device__ inline void handler_phase_a(int handler, const uint8_t* __restrict__ p, const Parsed& pr, TaskRec& rec,
                                       const uint32_t* __restrict__ crc_table = nullptr) {
    rec.has = 0; rec.mode = OM_NONE; rec.out_len = 0; rec.src_off = 0; rec.src_len = 0; rec.value = 0;
    if (pr.status != ST_OK) { rec.status = pr.status; return; }
    // handler(*args, **kwargs) with a positional-only one-parameter handler
    if (pr.nargs != 1 || pr.kwargs_nonempty) { rec.status = ST_ERROR; rec.value = EXC_TYPE; return; }
    rec.status = 0;
    switch (handler) {
    case 0: {   // identity: result = args[0]; `serialize_result(result) if result else None`
        switch (pr.a0_kind) {
        case AK_STR:
            if (pr.a0_len == 2) return;                                     // "" is falsy
            rec.src_off = pr.a0_off; rec.src_len = pr.a0_len; rec.has = 1;
            if (!(pr.a0_flags & (SF_ESC | SF_NONPRINT))) { rec.mode = OM_COPY; rec.out_len = pr.a0_len; }
            else { rec.mode = OM_STR_ESC; rec.out_len = py_string_len(p, pr.a0_off, pr.a0_off + pr.a0_len); }
            return;
        case AK_NULL: case AK_FALSE: case AK_ARR_EMPTY: case AK_OBJ_EMPTY: return;   // falsy
        case AK_TRUE: rec.src_off = pr.a0_off; rec.src_len = 4; rec.out_len = 4; rec.mode = OM_COPY; rec.has = 1; return;
        case AK_INT: {
            // float64 integer -> Go prints the digits -> Python int -> same digits; "-0"/"0" falsy
            bool zero = true;
            for (uint32_t k = 0; k < pr.a0_len; ++k) { uint8_t c = p[pr.a0_off + k]; if (c != '-' && c != '0') zero = false; }
            if (zero) return;
            rec.src_off = pr.a0_off; rec.src_len = pr.a0_len; rec.out_len = pr.a0_len; rec.mode = OM_COPY; rec.has = 1; return;
        }
        case AK_NUM: {
            // any other number: its float64, as Python reads Go's text of it; +-0 (also by underflow) is falsy
            unsigned long long b = 0;
            if (!f64_parse(p, pr.a0_off, pr.a0_off + pr.a0_len, &b)) { rec.status = ST_UNSUPPORTED; return; }
            if ((b << 1) == 0) return;
            rec.value = (long long)b; rec.mode = OM_PY_NUM; rec.out_len = py_json_go_number(b, nullptr); rec.has = 1;
            return;
        }
        case AK_ARR: case AK_OBJ: {                                          // non-empty: truthy
            const int64_t n = py_value_json(p, pr.a0_off, pr.a0_off + pr.a0_len, nullptr);
            if (n < 0) { rec.status = ST_UNSUPPORTED; return; }
            rec.src_off = pr.a0_off; rec.src_len = pr.a0_len; rec.out_len = (uint32_t)n; rec.mode = OM_PY_VALUE; rec.has = 1;
            return;
        }
        default: rec.status = ST_UNSUPPORTED; return;
        }
    }
    case 1: {   // crc32: zlib.crc32(s.encode()); a non-str has no .encode -> AttributeError
        if (pr.a0_kind != AK_STR) { rec.status = ST_ERROR; rec.value = EXC_ATTRIBUTE; return; }
        uint32_t c = crc32_of_string_token(p, pr.a0_off, pr.a0_off + pr.a0_len, pr.a0_flags, crc_table);
        if (c == 0) return;                                                 // 0 is falsy
        rec.value = (long long)c; rec.out_len = dec_len_u64(c); rec.mode = OM_U32_DEC; rec.has = 1;
        return;
    }
    case 2: {   // vadd_f32: base64 -> fp32 a||b -> a+b -> base64
        if (pr.a0_kind != AK_STR) { rec.status = ST_ERROR; rec.value = EXC_TYPE; return; }
        if (pr.a0_flags & SF_NONPRINT) {                                    // non-ASCII / DEL: ValueError / binascii.Error
            rec.status = ST_ERROR; rec.value = b64_str_error_class(p, pr.a0_off, pr.a0_off + pr.a0_len); return;
        }
        if (pr.a0_flags & SF_ESC) {
            // escaped text: any decoded character outside the base64 alphabet is an error for sure;
            // a fully valid escaped base64 string (only "\/" can do that) is not produced by the SDK
            uint32_t i = pr.a0_off + 1, end = pr.a0_off + pr.a0_len - 1;
            while (i < end) {
                uint32_t cp = next_cp(p, i, end);
                if (cp >= 0x80 || (b64_val((uint8_t)cp) < 0 && cp != '=')) {
                    rec.status = ST_ERROR; rec.value = b64_str_error_class(p, pr.a0_off, pr.a0_off + pr.a0_len); return;
                }
            }
            rec.status = ST_UNSUPPORTED; return;
        }
        int64_t rn = b64_decoded_len(p, pr.a0_off + 1, pr.a0_off + pr.a0_len - 1);
        if (rn < 0 || (rn % 8)) { rec.status = ST_ERROR; rec.value = rn < 0 ? EXC_BINASCII : EXC_VALUE; return; }
        uint32_t n = (uint32_t)(rn / 8);
        if (n == 0) return;                                                 // "" is falsy
        rec.src_off = pr.a0_off + 1; rec.src_len = n; rec.out_len = 2 + b64_encoded_len(4 * n); rec.mode = OM_VADD; rec.has = 1;
        return;
    }
    case 3: {   // json_sum: sum(obj["values"])
        if (pr.a0_kind != AK_OBJ) { rec.status = ST_ERROR; rec.value = pr.a0_kind == AK_OBJ_EMPTY ? EXC_KEY : EXC_TYPE; return; }
        PySum ps;
        bool no_key = false;
        int st = json_sum_object(p, pr.a0_off, pr.a0_off + pr.a0_len, &ps, &no_key);
        if (st) { rec.status = (uint8_t)st; if (st == ST_ERROR) rec.value = no_key ? EXC_KEY : EXC_TYPE; return; }
        if (ps.is_float) {                                                  // 0.0 / -0.0 are falsy, NaN is not
            const unsigned long long b = f64_to_bits(ps.f);
            if ((b << 1) == 0) return;
            rec.value = (long long)b; rec.mode = OM_PY_FLOAT; rec.out_len = py_json_float(b, nullptr); rec.has = 1;
            return;
        }
        const long long sum = ps.i;
        if (sum == 0) return;
        rec.value = sum; rec.mode = OM_I64_DEC; rec.has = 1;
        // the magnitude is negated in unsigned arithmetic: a total of exactly LLONG_MIN has no signed negation
        const unsigned long long mag = sum < 0 ? 0ull - (unsigned long long)sum : (unsigned long long)sum;
        rec.out_len = dec_len_u64(mag) + (sum < 0 ? 1u : 0u);
        return;
    }
    default:
        rec.status = ST_UNSUPPORTED; return;
    }
}

// phase B of the float64 and container modes, out of line (one call site in the kernels' main loops)
__device__ __noinline__ void seq_emit_py(const uint8_t* __restrict__ p, const TaskRec& rec, uint8_t* __restrict__ o) {
    if (rec.mode == OM_PY_NUM) py_json_go_number((unsigned long long)rec.value, o);
    else if (rec.mode == OM_PY_FLOAT) py_json_float((unsigned long long)rec.value, o);
    else py_value_json(p, rec.src_off, rec.src_off + rec.src_len, o);
}

// phase B for the modes that are not plain copies: writes exactly rec.out_len bytes at o. PY = false leaves out the
// float64 / container modes (only identity's deferred tasks and json_sum make them), and with them a call in the other loops.
template <bool PY = true>
__device__ inline void seq_emit(const uint8_t* __restrict__ p, const TaskRec& rec, uint8_t* __restrict__ o) {
    if (PY && rec.mode >= OM_PY_NUM) seq_emit_py(p, rec, o);
    else if (rec.mode == OM_VADD) vadd_write(p, rec.src_off, rec.src_len, o);
    else if (rec.mode == OM_U32_DEC || rec.mode == OM_I64_DEC) {
        unsigned long long v = (unsigned long long)rec.value; uint32_t l = rec.out_len;
        if (rec.value < 0) { *o++ = '-'; --l; v = 0ull - v; }     // (unsigned: LLONG_MIN's magnitude fits)
        write_dec(o, v, l);
    } else if (rec.mode == OM_STR_ESC) {                          // string the sequential parser sized (non-canonical frame)
        py_string_write(p, rec.src_off, rec.src_off + rec.src_len, o);
    }
}

}  // namespace b9
