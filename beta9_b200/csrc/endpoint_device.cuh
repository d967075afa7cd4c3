// The sequential (one thread per task) half of the endpoint drain (b9_endpoint_drain_launch): what an HTTP request body
// means to the endpoint runner and the bytes of its response. Reference behaviour realised per task:
//     gateway      pkg/abstractions/endpoint/buffer.go:460-572 (SerializeHttpPayload -> json.Marshal(TaskPayload))
//     runner       sdk/src/beta9/runner/endpoint.py:202-306 (json.loads, args / kwargs None -> [] / {},
//                  handler(*args, **kwargs), JSONResponse(result))
//     rendering    Starlette's JSONResponse: json.dumps(ensure_ascii=False, allow_nan=False, separators=(",", ":"))
// Unlike the task-queue runner there is no falsy rule: every answered request has a body ("" -> `""`, 0 -> `0`, [] -> `[]`).
// Plain C++ behind CUDA qualifiers: tests/host_shim/endpoint_shim.cpp compiles it for the host
// (tests/test_endpoint_on_host.py). The kernel is endpoint_drain.cu.
#pragma once
#include <stdint.h>
#include "handler_seq.cuh"

namespace b9 {

// ---- CPython json.dumps(str) with ensure_ascii=False ------------------------------------------------------------------
// '"' and '\\' and the short forms \n \r \t \b \f are escaped, other code points below 0x20 become \u00xx (lower-case hex);
// everything else is raw UTF-8 (non-ASCII, DEL, U+2028 / U+2029, '<' '>' '&'). The string is what Go decoded, so invalid
// UTF-8 and lone surrogates are U+FFFD (EF BF BD) by then (next_cp).
__device__ __forceinline__ uint32_t ep_emit_len(uint32_t cp) {
    if (cp < 0x80) {
        if (cp == '"' || cp == '\\' || cp == '\n' || cp == '\r' || cp == '\t' || cp == '\b' || cp == '\f') return 2;
        return cp < 0x20 ? 6u : 1u;
    }
    return cp < 0x800 ? 2u : (cp < 0x10000 ? 3u : 4u);
}
__device__ inline uint32_t ep_emit(uint32_t cp, uint8_t* __restrict__ o) {
    if (cp < 0x80) {
        uint8_t sc = 0;
        switch (cp) { case '"': sc = '"'; break; case '\\': sc = '\\'; break; case '\b': sc = 'b'; break; case '\f': sc = 'f'; break;
                      case '\n': sc = 'n'; break; case '\r': sc = 'r'; break; case '\t': sc = 't'; break; }
        if (sc) { o[0] = '\\'; o[1] = sc; return 2; }
        if (cp < 0x20) { o[0] = '\\'; o[1] = 'u'; o[2] = '0'; o[3] = '0'; o[4] = hexdig(cp >> 4); o[5] = hexdig(cp & 15); return 6; }
        o[0] = (uint8_t)cp; return 1;
    }
    if (cp < 0x800) { o[0] = 0xC0 | (cp >> 6); o[1] = 0x80 | (cp & 0x3F); return 2; }
    if (cp < 0x10000) { o[0] = 0xE0 | (cp >> 12); o[1] = 0x80 | ((cp >> 6) & 0x3F); o[2] = 0x80 | (cp & 0x3F); return 3; }
    o[0] = 0xF0 | (cp >> 18); o[1] = 0x80 | ((cp >> 12) & 0x3F); o[2] = 0x80 | ((cp >> 6) & 0x3F); o[3] = 0x80 | (cp & 0x3F); return 4;
}
// string token p[s..e) (quotes included, validated)
__device__ inline uint32_t ep_string_len(const uint8_t* __restrict__ p, uint32_t s, uint32_t e) {
    uint32_t i = s + 1, end = e - 1, out = 2;
    while (i < end) out += ep_emit_len(next_cp(p, i, end));
    return out;
}
__device__ inline uint32_t ep_string_write(const uint8_t* __restrict__ p, uint32_t s, uint32_t e, uint8_t* __restrict__ o) {
    uint32_t i = s + 1, end = e - 1, n = 1;
    o[0] = '"';
    while (i < end) n += ep_emit(next_cp(p, i, end), o + n);
    o[n] = '"';
    return n + 1;
}

// value_json's writer for the response body: compact separators, ensure_ascii=False strings, numbers as json.loads read
// Go's text of them (py_json_go_number: "-0" is the int 0, 1e21 is the float 1e+21)
struct EpJsonWriter {
    static constexpr bool SPACED = false;
    __device__ static __forceinline__ uint32_t string_len(const uint8_t* __restrict__ p, uint32_t s, uint32_t e) { return ep_string_len(p, s, e); }
    __device__ static __forceinline__ uint32_t string_write(const uint8_t* __restrict__ p, uint32_t s, uint32_t e, uint8_t* __restrict__ o) {
        return ep_string_write(p, s, e, o);
    }
    __device__ static __forceinline__ uint32_t number(unsigned long long bits, uint8_t* o) { return py_json_go_number(bits, o); }
};
// JSONResponse(value).body for the validated JSON value p[s..e) as the runner received it; -1 where value_json declines
__device__ __noinline__ int64_t ep_value_json(const uint8_t* __restrict__ p, uint32_t s, uint32_t e, uint8_t* __restrict__ o) {
    return value_json<EpJsonWriter>(p, s, e, o, false);
}

// How a record's bytes are produced (TaskRec.mode of the endpoint drain). EM_COPY is a verbatim copy of
// p[src_off .. src_off + src_len), which the kernel does warp-cooperatively; endpoint_emit writes the others.
enum EpMode : uint8_t {
    EM_NONE = 0,
    EM_COPY,     // the argument's token as it is: a string without escapes whose bytes are valid UTF-8, true / false / null, an int
    EM_STR,      // a string: ep_string_write over the token
    EM_VALUE,    // a list / object: ep_value_json over the token
    EM_NUM,      // a number argument: py_json_go_number(value)
    EM_FLOAT,    // json_sum's float total: py_json_float(value)
    EM_DEC,      // crc32's / json_sum's int: the decimal digits of (signed) value
    EM_VADD      // vadd_f32: '"' + base64(a + b) + '"' for src_len floats per vector from the base64 body at src_off
};

// The tasks an endpoint drain answers: exactly B9_TF_HTTP_BODY (a body the gateway would run SerializeHttpPayload on).
// Without it the task is a pre-marshalled payload, and B9_TF_PICKLE / B9_TF_TASK_MSG are other paths: UNSUPPORTED.
__device__ __forceinline__ bool endpoint_accepts(uint32_t flags) { return flags == 0x02u; }

// Phase A for one request: `pr` is parse_payload(p, n, /*http=*/true). Fills status / has / out_len / mode:
//   COMPLETE, has = 1   the handler returned and JSONResponse rendered it (200): out_len bytes, falsy results included
//   REJECTED            SerializeHttpPayload failed: the gateway's 400
//   ERROR               the handler raised (TypeError for a call that does not bind one positional argument, KeyError,
//                       ValueError, ...): the runner's 500
//   UNSUPPORTED         a render failure (json_sum's non-finite total: allow_nan=False raises, 500 with the task Complete),
//                       or what the parse and handlers decline (more than 19 significant digits at a rounding boundary,
//                       nesting deeper than 16, more than 64 members, json_sum ints outside a C long)
__device__ inline void endpoint_phase_a(int handler, const uint8_t* __restrict__ p, const Parsed& pr, TaskRec& rec,
                                        const uint32_t* __restrict__ crc_table = nullptr) {
    rec.has = 0; rec.mode = EM_NONE; rec.out_len = 0; rec.src_off = 0; rec.src_len = 0; rec.value = 0;
    if (pr.status != ST_OK) { rec.status = pr.status; return; }
    // args None -> [], kwargs None -> {} (endpoint.py:271-277), then handler(*args, **kwargs) with a positional-only
    // one-parameter handler: anything but one argument and no keyword is a TypeError
    if (pr.nargs != 1 || pr.kwargs_nonempty) { rec.status = 1; return; }
    rec.status = 0;
    switch (handler) {
    case 0: {   // identity: JSONResponse(args[0])
        const uint32_t s = pr.a0_off, e = pr.a0_off + pr.a0_len;
        switch (pr.a0_kind) {
        case AK_STR:
            rec.src_off = s; rec.src_len = pr.a0_len; rec.has = 1;
            if (!(pr.a0_flags & (SF_ESC | SF_NONPRINT))) { rec.out_len = pr.a0_len; rec.mode = EM_COPY; return; }   // printable ASCII
            rec.out_len = ep_string_len(p, s, e);
            // no escape: each code point is written as the bytes it was read from, unless it was invalid UTF-8 (one byte
            // read, three written), so an unchanged length means an unchanged token
            rec.mode = (!(pr.a0_flags & SF_ESC) && rec.out_len == pr.a0_len) ? EM_COPY : EM_STR;
            return;
        case AK_NULL: case AK_TRUE: case AK_FALSE:
            rec.src_off = s; rec.src_len = pr.a0_len; rec.out_len = pr.a0_len; rec.mode = EM_COPY; rec.has = 1; return;
        case AK_INT: {
            // <= 15 digits: Go prints the float64's digits again and json.loads makes an int of them; "-0" is the int 0
            bool zero = true;
            for (uint32_t k = 0; k < pr.a0_len; ++k) { const uint8_t c = p[s + k]; if (c != '-' && c != '0') zero = false; }
            rec.has = 1;
            if (zero) { rec.value = 0; rec.out_len = 1; rec.mode = EM_DEC; return; }
            rec.src_off = s; rec.src_len = pr.a0_len; rec.out_len = pr.a0_len; rec.mode = EM_COPY; return;
        }
        case AK_NUM: {
            unsigned long long b = 0;
            if (!f64_parse(p, s, e, &b)) { rec.status = ST_UNSUPPORTED; return; }
            rec.value = (long long)b; rec.mode = EM_NUM; rec.out_len = py_json_go_number(b, nullptr); rec.has = 1;
            return;
        }
        case AK_ARR_EMPTY: case AK_OBJ_EMPTY: case AK_ARR: case AK_OBJ: {
            const int64_t n = ep_value_json(p, s, e, nullptr);
            if (n < 0) { rec.status = ST_UNSUPPORTED; return; }
            rec.src_off = s; rec.src_len = pr.a0_len; rec.out_len = (uint32_t)n; rec.mode = EM_VALUE; rec.has = 1;
            return;
        }
        default: rec.status = ST_UNSUPPORTED; return;
        }
    }
    case 1: {   // crc32: zlib.crc32(s.encode()), 0 included
        if (pr.a0_kind != AK_STR) { rec.status = 1; return; }               // AttributeError
        const uint32_t c = crc32_of_string_token(p, pr.a0_off, pr.a0_off + pr.a0_len, pr.a0_flags, crc_table);
        rec.value = (long long)c; rec.out_len = dec_len_u64(c); rec.mode = EM_DEC; rec.has = 1;
        return;
    }
    case 2: {   // vadd_f32: base64 -> fp32 a||b -> a+b -> base64; "" -> ""
        if (pr.a0_kind != AK_STR) { rec.status = 1; return; }               // TypeError
        if (pr.a0_flags & SF_NONPRINT) { rec.status = 1; return; }          // non-ASCII / DEL: ValueError / binascii.Error
        if (pr.a0_flags & SF_ESC) {                                         // as the task-queue drain: see handler_phase_a
            uint32_t i = pr.a0_off + 1, end = pr.a0_off + pr.a0_len - 1;
            while (i < end) { uint32_t cp = next_cp(p, i, end); if (cp >= 0x80 || (b64_val((uint8_t)cp) < 0 && cp != '=')) { rec.status = 1; return; } }
            rec.status = ST_UNSUPPORTED; return;
        }
        const int64_t rn = b64_decoded_len(p, pr.a0_off + 1, pr.a0_off + pr.a0_len - 1);
        if (rn < 0 || (rn % 8)) { rec.status = 1; return; }
        const uint32_t n = (uint32_t)(rn / 8);
        rec.src_off = pr.a0_off + 1; rec.src_len = n; rec.out_len = 2 + b64_encoded_len(4 * n); rec.mode = EM_VADD; rec.has = 1;
        return;
    }
    case 3: {   // json_sum: sum(obj["values"])
        if (pr.a0_kind != AK_OBJ) { rec.status = 1; return; }               // TypeError, or KeyError for {}
        PySum ps;
        const int st = json_sum_object(p, pr.a0_off, pr.a0_off + pr.a0_len, &ps);
        if (st) { rec.status = (uint8_t)st; return; }
        if (ps.is_float) {
            const unsigned long long b = f64_to_bits(ps.f);
            if ((b & 0x7FF0000000000000ull) == 0x7FF0000000000000ull) { rec.status = ST_UNSUPPORTED; return; }   // allow_nan=False
            rec.value = (long long)b; rec.mode = EM_FLOAT; rec.out_len = py_json_float(b, nullptr); rec.has = 1;
            return;
        }
        const long long sum = ps.i;
        rec.value = sum; rec.mode = EM_DEC; rec.has = 1;
        const unsigned long long mag = sum < 0 ? 0ull - (unsigned long long)sum : (unsigned long long)sum;
        rec.out_len = dec_len_u64(mag) + (sum < 0 ? 1u : 0u);
        return;
    }
    default:
        rec.status = ST_UNSUPPORTED; return;
    }
}

// Phase B for every mode but EM_COPY: writes exactly rec.out_len bytes at o
__device__ __noinline__ void endpoint_emit(const uint8_t* __restrict__ p, const TaskRec& rec, uint8_t* __restrict__ o) {
    switch (rec.mode) {
    case EM_STR: ep_string_write(p, rec.src_off, rec.src_off + rec.src_len, o); break;
    case EM_VALUE: ep_value_json(p, rec.src_off, rec.src_off + rec.src_len, o); break;
    case EM_NUM: py_json_go_number((unsigned long long)rec.value, o); break;
    case EM_FLOAT: py_json_float((unsigned long long)rec.value, o); break;
    case EM_VADD: vadd_write(p, rec.src_off, rec.src_len, o); break;
    case EM_DEC: {
        unsigned long long v = (unsigned long long)rec.value; uint32_t l = rec.out_len;
        if (rec.value < 0) { *o++ = '-'; --l; v = 0ull - v; }
        write_dec(o, v, l);
        break;
    }
    default: break;
    }
}

}  // namespace b9
