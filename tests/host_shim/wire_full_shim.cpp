// TEST INFRASTRUCTURE: compiles what b9_wire_encode_full writes for a task's Args and Kwargs -- the payload parser, the
// ordered Go walk (go_value_json, handler_seq.cuh), go_transcode and the HTTP kwargs rule (wire_full_values,
// wire_encode.cuh) -- for the host, so that they can be compared with the oracle's Go encoder on a CPU
// (tests/test_wire_full_on_host.py).
#include <stdint.h>
#include <string.h>
#include <vector>
#define __device__
#define __host__
#define __forceinline__ inline
#define __constant__ static const
static inline float __uint_as_float(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline uint32_t __float_as_uint(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline float __fadd_rn(float a, float b) { volatile float z = a + b; return z; }     // IEEE binary32, round to nearest even
static inline uint32_t __funnelshift_r(uint32_t lo, uint32_t hi, uint32_t sh) { return (uint32_t)(((((uint64_t)hi) << 32) | lo) >> (sh & 31u)); }
#include "../../beta9_b200/csrc/handler_seq.cuh"
#define B9_WIRE_ENCODE_HELPERS_ONLY 1
#include "../../beta9_b200/csrc/wire_encode.cuh"

// One task as b9_wire_encode_full sees it: status 0 (args and kwargs written), 3 (Go refuses the payload) or 4 (declined).
static uint8_t task(const uint8_t* p, uint32_t n, bool http, b9::GoVal& a, b9::GoVal& k, uint8_t* kw_merged) {
    const b9::Parsed pr = b9::parse_payload(p, n, http);
    *kw_merged = pr.kw_merged;
    if (pr.status != b9::ST_OK) return pr.status;
    return b9::wire_full_values(p, n, http, pr, a, k) ? 0 : b9::ST_UNSUPPORTED;
}

// Where go_transcode wrote v: 1 = the walk writes the same bytes, 2 = the walk declines (its limits), 0 = other bytes.
static uint8_t walk_agrees(const uint8_t* p, const b9::GoVal& v, const uint8_t* written) {
    if (v.mode != b9::GV_TRANSCODE) return 1;
    const int64_t need = b9::go_value_json(p, v.s, v.e, nullptr, false);
    if (need < 0) return 2;
    std::vector<uint8_t> w((size_t)need + 1);
    return need == v.len && b9::go_value_json(p, v.s, v.e, w.data(), false) == v.len && memcmp(w.data(), written, (size_t)v.len) == 0;
}

// n payloads blob[off[i] .. off[i+1]). out == nullptr: fills out_off (n + 1 entries) with the sizes of the records and
// returns the total. Otherwise writes record i = args bytes, a 0 byte, kwargs bytes (empty for status != 0) at
// out[out_off[i]..out_off[i+1]). status[i], kw_merged[i], mode[2i], mode[2i+1] (GoValMode of args / kwargs), and
// agree[i]: 0 where go_transcode answered a value and the walk over the same span wrote other bytes, 2 where the walk
// declined such a value, else 1.
extern "C" uint64_t b9_wf_batch(const uint8_t* blob, const uint64_t* off, uint32_t n, int http, uint8_t* status, uint8_t* kw_merged,
                                uint8_t* mode, uint8_t* agree, uint8_t* out, uint64_t* out_off) {
    uint64_t total = 0;
    for (uint32_t i = 0; i < n; ++i) {
        const uint8_t* p = blob + off[i];
        const uint32_t len = (uint32_t)(off[i + 1] - off[i]);
        b9::GoVal a, k;
        status[i] = task(p, len, http != 0, a, k, &kw_merged[i]);
        mode[2 * i] = mode[2 * i + 1] = 0xFF;
        if (!out) {
            out_off[i] = total;
            total += status[i] == 0 ? (uint64_t)a.len + 1 + (uint64_t)k.len : 0;
            continue;
        }
        agree[i] = 1;
        if (status[i] != 0) continue;
        mode[2 * i] = a.mode; mode[2 * i + 1] = k.mode;
        uint8_t* o = out + out_off[i];
        const uint32_t la = b9::go_val_write(p, a, o);
        agree[i] = walk_agrees(p, a, o);
        o += la;
        *o++ = 0;
        const uint32_t lk = b9::go_val_write(p, k, o);
        const uint8_t ak = walk_agrees(p, k, o);
        if (agree[i] == 0 || ak == 0) agree[i] = 0; else if (ak == 2) agree[i] = 2;
        o += lk;
        total += (uint64_t)(o - (out + out_off[i]));
    }
    if (!out) out_off[n] = total;
    return total;
}

// The ordered Go walk alone over one validated, non-empty list or object: bytes written, -1 where it declines,
// -2 if `cap` is too small or the sizing and writing passes disagree.
extern "C" long b9_wf_walk(const uint8_t* p, uint32_t n, int drop_args, uint8_t* out, uint32_t cap) {
    const int64_t need = b9::go_value_json(p, 0, n, nullptr, drop_args != 0);
    if (need < 0) return -1;
    if ((uint64_t)need > cap) return -2;
    const int64_t got = b9::go_value_json(p, 0, n, out, drop_args != 0);
    return got == need ? (long)got : -2;
}

// go_transcode alone (the copy-like path): bytes written, or -1 where it declines.
extern "C" long b9_wf_transcode(const uint8_t* p, uint32_t n, uint8_t* out, uint32_t cap) {
    const int64_t need = b9::go_transcode(p, 0, n, nullptr);
    if (need < 0) return -1;
    if ((uint64_t)need > cap) return -2;
    return (long)b9::go_transcode(p, 0, n, out);
}
