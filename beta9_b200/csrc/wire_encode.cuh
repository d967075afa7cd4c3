// Device-side `TaskMessage.Encode` (pkg/types/task.go:55-65,79-90): the bytes client.Push RPUSHes
// (pkg/abstractions/taskqueue/client.go:29-41) and Dispatcher.Send stores as task state
// (pkg/task/dispatch.go:105-112) — the durable record the Go host keeps in Redis.
//
//   {"task_id":"<uuid>","workspace_name":…,"stub_id":…,"executor":…,"args":[…],"kwargs":{…}|null,
//    "policy":{"max_retries":N,"timeout":N,"expires":"<RFC3339Nano>","ttl":N},"retries":N,"timestamp":N}
//
// Go 1.23 encoding/json rules restated for the values a payload can hold: strings HTML-safe escaped
// (< > & -> < > &, U+2028/9, \b \f \n \r \t short forms, other controls \u00XX, the rest
// raw UTF-8), map keys sorted, no whitespace, nil Args -> [], nil Kwargs -> null, integer-valued
// float64 printed as digits. PARITY UNPINNED like the oracle's restatement (DESIGN.md §3).
//
// Two entry points share one kernel, wire_encode_kernel<FULL>:
//   * b9_wire_encode (FULL = false). Device domain: numbers must be plain integers of <= 15 digits (anything else
//     needs strconv's shortest-float formatting), object keys must already be in strictly increasing byte order (Go
//     would sort them), SDK payloads only. Everything else is reported B9_ST_UNSUPPORTED, never approximated.
//   * b9_wire_encode_full (FULL = true): go_transcode where it answers (the copy-like path of canonical payloads),
//     else the ordered walk go_value_json (handler_seq.cuh): every number go_json_float(f64_parse(literal)), objects
//     in Go's map order, duplicates last-wins; HTTP bodies by SerializeHttpPayload's map rules (wire_full_values).
//     Declines: merged struct kwargs, a literal f64_parse cannot settle, the walk's depth / member limits, TASK_MSG
//     and PICKLE tasks.
// One thread per task: a sizing walk, one warp_reserve_bytes per warp (drain_kernel.cuh), an emitting walk.
#pragma once
#include <stdint.h>
#ifdef B9_WIRE_ENCODE_HELPERS_ONLY      // tests/host_shim builds the value encoders below for the host
#include "handler_seq.cuh"
#else
#include "drain_kernel.cuh"
#endif

namespace b9 {

struct WireEnv {
    // pre-quoted, constant per queue: `","workspace_name":"ws","stub_id":"…","executor":"taskqueue","args":`
    uint8_t mid[512]; uint32_t mid_len;
    uint32_t max_retries; int32_t timeout; uint32_t ttl;
};

// Re-encode the validated JSON value p[s..e) by Go's rules. o == nullptr: size only.
// Returns the byte count, or -1 if the value is outside the device domain.
__device__ inline int64_t go_transcode(const uint8_t* __restrict__ p, uint32_t s, uint32_t e, uint8_t* __restrict__ o) {
    constexpr int MAXD = 16;
    uint32_t prev_ks[MAXD], prev_ke[MAXD];          // previous key (body span) of the object open at each depth
    uint32_t has_prev = 0;                          // bit d: prev_k*[d] is set
    uint64_t is_obj = 0;
    int depth = 0;
    int64_t n = 0;
    uint32_t i = s;
    bool expect_key = false;
    while (i < e) {
        const uint8_t c = p[i];
        if (is_ws(c)) { ++i; continue; }
        if (c == '"') {
            uint32_t f = 0;
            const uint32_t ts = i;
            i = (uint32_t)scan_string(p, i, e, f);
            const uint32_t bs = ts + 1, be = i - 1;
            if (expect_key) {
                if (((has_prev >> (depth - 1)) & 1u) && !key_less(p, prev_ks[depth - 1], prev_ke[depth - 1], bs, be)) return -1;   // Go would reorder / dedupe
                prev_ks[depth - 1] = bs; prev_ke[depth - 1] = be; has_prev |= 1u << (depth - 1);
                expect_key = false;
            }
            if (o) o[n] = '"';
            ++n;
            uint32_t k = bs;
            while (k < be) { const uint32_t cp = next_cp(p, k, be); if (o) n += go_emit(cp, o + n); else n += go_emit_len(cp); }
            if (o) o[n] = '"';
            ++n;
            continue;
        }
        if (c == '-' || is_digit(c)) {
            uint32_t f = 0; bool simple = false;
            const uint32_t ts = i;
            i = (uint32_t)scan_number(p, i, e, f, &simple);
            if (!simple) return -1;
            if (o) for (uint32_t k = ts; k < i; ++k) o[n + (k - ts)] = p[k];
            n += i - ts;
            continue;
        }
        if (c == 't' || c == 'n') { if (o) for (int k = 0; k < 4; ++k) o[n + k] = p[i + k]; n += 4; i += 4; continue; }
        if (c == 'f') { if (o) for (int k = 0; k < 5; ++k) o[n + k] = p[i + k]; n += 5; i += 5; continue; }
        if (c == '{' || c == '[') {
            if (depth >= MAXD) return -1;
            is_obj = (is_obj << 1) | (c == '{' ? 1u : 0u);
            has_prev &= ~(1u << depth);
            ++depth;
            expect_key = c == '{';
        } else if (c == '}' || c == ']') {
            is_obj >>= 1; --depth; expect_key = false;
        } else if (c == ',') {
            expect_key = (is_obj & 1u) != 0;
        }
        // ':' and the structural characters above are copied as they are
        if (o) o[n] = c;
        ++n; ++i;
    }
    return n;
}

// ---- b9_wire_encode_full: what TaskMessage.Encode writes for Args and Kwargs ----------------------------------
// How one of the two values is written: a span of the payload (go_transcode, or the ordered walk), or a constant.
enum GoValMode : uint8_t { GV_TRANSCODE = 0, GV_WALK, GV_WALK_NO_ARGS /* an HTTP body's map minus "args" */,
                           GV_LIST_NIL /* [] */, GV_MAP_NIL /* null */, GV_MAP_EMPTY /* {} */ };
struct GoVal { uint32_t s, e; int64_t len; uint8_t mode; };

// Sizes the value p[s..e): go_transcode where it answers, the walk where it declines. len < 0: the walk declines too.
__device__ inline GoVal go_val_plan(const uint8_t* __restrict__ p, uint32_t s, uint32_t e, bool drop_args) {
    GoVal v; v.s = s; v.e = e; v.len = -1; v.mode = drop_args ? GV_WALK_NO_ARGS : GV_TRANSCODE;
    if (!drop_args) v.len = go_transcode(p, s, e, nullptr);
    if (v.len < 0) { if (!drop_args) v.mode = GV_WALK; v.len = go_value_json(p, s, e, nullptr, drop_args); }
    return v;
}
__device__ inline GoVal go_val_const(uint8_t mode) { GoVal v; v.s = v.e = 0; v.mode = mode; v.len = mode == GV_MAP_NIL ? 4 : 2; return v; }

// Writes what go_val_plan sized: exactly v.len bytes.
__device__ inline uint32_t go_val_write(const uint8_t* __restrict__ p, const GoVal& v, uint8_t* __restrict__ o) {
    switch (v.mode) {
    case GV_TRANSCODE: return (uint32_t)go_transcode(p, v.s, v.e, o);
    case GV_WALK: case GV_WALK_NO_ARGS: return (uint32_t)go_value_json(p, v.s, v.e, o, v.mode == GV_WALK_NO_ARGS);
    case GV_LIST_NIL: o[0] = '['; o[1] = ']'; return 2;
    case GV_MAP_NIL: o[0] = 'n'; o[1] = 'u'; o[2] = 'l'; o[3] = 'l'; return 4;
    default: o[0] = '{'; o[1] = '}'; return 2;
    }
}

// Args and Kwargs of a payload the parser accepted (pr.status == ST_OK; pr = parse_payload(p, n, http)), as
// TaskMessage.Encode writes them. Returns false where the device declines: struct kwargs objects Go merges
// (pr.kw_merged), or a value the walk declines.
//   SDK payload (struct decode into TaskPayload): nil Args -> [], nil Kwargs -> null.
//   HTTP body (SerializeHttpPayload, pkg/task/serialize.go:16-101): Args = the last "args" if it is a list, else nil
//   ([]). Kwargs is never nil: the last "kwargs" if it is an object; otherwise the body's remaining map -- the whole
//   top-level object minus "args" when that was taken as Args; {} for an empty or null body.
__device__ inline bool wire_full_values(const uint8_t* __restrict__ p, uint32_t n, bool http, const Parsed& pr, GoVal& a, GoVal& k) {
    if (pr.kw_merged) return false;
    a = pr.args_len ? go_val_plan(p, pr.args_off, pr.args_off + pr.args_len, false) : go_val_const(GV_LIST_NIL);
    if (pr.kw_len) k = go_val_plan(p, pr.kw_off, pr.kw_off + pr.kw_len, false);
    else if (!http) k = go_val_const(GV_MAP_NIL);
    else {
        uint32_t s = 0, e = n;
        while (s < e && is_ws(p[s])) ++s;
        while (e > s && is_ws(p[e - 1])) --e;
        k = (s == e || p[s] == 'n') ? go_val_const(GV_MAP_EMPTY) : go_val_plan(p, s, e, pr.args_len != 0);
    }
    return a.len >= 0 && k.len >= 0;
}

__device__ __forceinline__ void civil_from_days_dev(long long z, long long* y, int* m, int* d) {
    z += 719468;
    const long long era = (z >= 0 ? z : z - 146096) / 146097;
    const long long doe = z - era * 146097;
    const long long yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
    *y = yoe + era * 400;
    const long long doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
    const long long mp = (5 * doy + 2) / 153;
    *d = (int)(doy - (153 * mp + 2) / 5 + 1);
    *m = (int)(mp < 10 ? mp + 3 : mp - 9);
    if (*m <= 2) ++*y;
}
__device__ __forceinline__ void put2(uint8_t* o, int v) { o[0] = (uint8_t)('0' + v / 10); o[1] = (uint8_t)('0' + v % 10); }

// time.Time.MarshalJSON body at UTC: 2006-01-02T15:04:05.999999999Z (fraction trimmed / omitted). <= 30 bytes.
__device__ inline uint32_t rfc3339nano(long long unix_ns, uint8_t* o) {
    long long secs = unix_ns / 1000000000ll, ns = unix_ns % 1000000000ll;
    if (ns < 0) { ns += 1000000000ll; --secs; }
    long long days = secs / 86400, sod = secs % 86400;
    if (sod < 0) { sod += 86400; --days; }
    long long y; int m, d; civil_from_days_dev(days, &y, &m, &d);
    o[0] = (uint8_t)('0' + (y / 1000) % 10); o[1] = (uint8_t)('0' + (y / 100) % 10); o[2] = (uint8_t)('0' + (y / 10) % 10); o[3] = (uint8_t)('0' + y % 10);
    o[4] = '-'; put2(o + 5, m); o[7] = '-'; put2(o + 8, d); o[10] = 'T';
    put2(o + 11, (int)(sod / 3600)); o[13] = ':'; put2(o + 14, (int)(sod % 3600 / 60)); o[16] = ':'; put2(o + 17, (int)(sod % 60));
    uint32_t n = 19;
    if (ns) {
        uint8_t f[9]; long long t = ns;
        for (int k = 8; k >= 0; --k) { f[k] = (uint8_t)('0' + t % 10); t /= 10; }
        int e = 9; while (e > 0 && f[e - 1] == '0') --e;
        o[n++] = '.';
        for (int k = 0; k < e; ++k) o[n++] = f[k];
    }
    o[n++] = 'Z';
    return n;
}

// (not inlined: with its three call sites in wire_encode_kernel inlined, the sm_90a optimizer of CUDA 12.9 does not
// finish compiling the kernel)
__device__ __attribute__((noinline)) uint32_t put_dec_ll(uint8_t* o, long long v) {
    uint32_t n = 0;
    if (v < 0) { o[n++] = '-'; v = -v; }
    const uint32_t l = dec_len_u64((unsigned long long)v);
    write_dec(o + n, (unsigned long long)v, l);
    return n + l;
}

#ifndef B9_WIRE_ENCODE_HELPERS_ONLY
struct WireArgs {
    const uint8_t* payload; const uint64_t* off; const uint64_t* hdr; const uint4* ids; const int64_t* ts; const int64_t* exp;
    uint32_t slot_mask; uint64_t first_task; uint32_t n_tasks;
    DrainOut out;
};

// FULL = false: b9_wire_encode; FULL = true: b9_wire_encode_full (the header comment above), instantiated in wire_full.cu
template <bool FULL>
__global__ void __launch_bounds__(128) wire_encode_kernel(WireArgs a, const WireEnv* __restrict__ envp) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const bool valid = t < a.n_tasks;
    const WireEnv& env = *envp;
    uint32_t status = 0, total = 0;
    Parsed pr; pr.status = ST_OK; pr.args_len = 0; pr.kw_len = 0; pr.args_off = 0; pr.kw_off = 0; pr.kw_merged = 0;
    const uint8_t* p = nullptr;
    uint32_t slot = 0; uint64_t h = 0;
    int64_t la = 2, lk = 4;                      // "[]" / "null"
    GoVal ga, gk;                                // FULL: how args / kwargs are written
    uint8_t tail[96]; uint32_t tail_len = 0;     // ,"policy":{…},"retries":N,"timestamp":N}
    if (valid) {
        slot = (uint32_t)((a.first_task + t) & a.slot_mask);
        h = a.hdr[slot];
        p = a.payload + a.off[slot];
        if (FULL) {
            const bool http = (hdr_flags(h) & B9_TF_HTTP_BODY_BIT) != 0;
            pr = parse_payload(p, hdr_len(h), http);
            status = pr.status;
            if (hdr_flags(h) & (B9_TF_TASK_MSG_BIT | B9_TF_PICKLE_BIT)) status = ST_UNSUPPORTED;   // a record already / not JSON
            if (status == ST_OK) {
                if (!wire_full_values(p, hdr_len(h), http, pr, ga, gk)) status = ST_UNSUPPORTED;
                la = ga.len; lk = gk.len;
            }
        } else {
            pr = parse_payload(p, hdr_len(h));
            status = pr.status;
            if (hdr_flags(h) & B9_TF_HTTP_BODY_BIT) status = ST_UNSUPPORTED;     // an HTTP body's TaskPayload follows the map rules: not encoded here
            if (hdr_flags(h) & B9_TF_TASK_MSG_BIT) status = ST_UNSUPPORTED;      // already a record: nothing to encode
            if (status == ST_OK) {
                if (pr.kw_merged) status = ST_UNSUPPORTED;                       // Go merges duplicate kwargs maps
                if (pr.args_len) la = go_transcode(p, pr.args_off, pr.args_off + pr.args_len, nullptr);
                if (pr.kw_len) lk = go_transcode(p, pr.kw_off, pr.kw_off + pr.kw_len, nullptr);
                if (la < 0 || lk < 0) status = ST_UNSUPPORTED;
            }
        }
        if (status == ST_OK) {
            // the tail is small and per task: build it once in registers/local memory
            const char P0[] = ",\"policy\":{\"max_retries\":";
            for (int k = 0; P0[k]; ++k) tail[tail_len++] = (uint8_t)P0[k];
            tail_len += put_dec_ll(tail + tail_len, (long long)env.max_retries);
            const char P1[] = ",\"timeout\":";
            for (int k = 0; P1[k]; ++k) tail[tail_len++] = (uint8_t)P1[k];
            tail_len += put_dec_ll(tail + tail_len, (long long)env.timeout);
            total = 12 /* {"task_id":" */ + 36 + env.mid_len + (uint32_t)la + 10 /* ,"kwargs": */ + (uint32_t)lk + tail_len;
        }
    }
    // the rest of the tail depends on per-task slot words; sized exactly below
    uint8_t tbuf[40]; uint32_t tlen = 0; long long ts = 0; uint32_t retries = 0;
    if (valid && status == ST_OK) {
        const long long ex = a.exp[slot];
        if (ex) tlen = rfc3339nano(ex, tbuf);
        else { const char Z[] = "0001-01-01T00:00:00Z"; for (tlen = 0; Z[tlen]; ++tlen) tbuf[tlen] = (uint8_t)Z[tlen]; }   // time.Time{}
        ts = a.ts[slot]; retries = (uint32_t)(h >> 40) & 0xFFu;
        uint8_t scratch[24];
        total += 12 /* ,"expires":" */ + tlen + 8 /* ","ttl": */ + put_dec_ll(scratch, (long long)env.ttl) + 12 /* },"retries": */
               + put_dec_ll(scratch, (long long)retries) + 13 /* ,"timestamp": */ + put_dec_ll(scratch, ts) + 1 /* } */;
    }
    // one cursor add per warp
    const uint32_t mine = (valid && status == ST_OK) ? total : 0u;
    const uint32_t inc = warp_incl_scan(mine, lane);
    const Reservation r = warp_reserve_bytes(a.out, __shfl_sync(0xffffffffu, inc, 31), lane);
    if (!valid) return;
    const unsigned long long ob = r.base + (inc - mine);
    store_record_id(a.out, t, a.ids + slot);                           // (a no-op: records are 1:1 with the window's tasks)
    store_record(a.out, t, r.fits, ob, mine, (uint8_t)status, mine ? 1 : 0);
    if (!mine || !r.fits) return;
    uint8_t* o = a.out.payload + ob;
    const char H0[] = "{\"task_id\":\"";
    for (int k = 0; k < 12; ++k) *o++ = (uint8_t)H0[k];
    {
        const uint4 idv = a.ids[slot];
        const uint32_t w[4] = {idv.x, idv.y, idv.z, idv.w};
        for (int b = 0; b < 16; ++b) {
            if (b == 4 || b == 6 || b == 8 || b == 10) *o++ = '-';
            const uint32_t byte = (w[b >> 2] >> (8 * (b & 3))) & 0xFFu;
            *o++ = hexdig(byte >> 4); *o++ = hexdig(byte & 15);
        }
    }
    for (uint32_t k = 0; k < env.mid_len; ++k) *o++ = env.mid[k];
    const char K0[] = ",\"kwargs\":";
    if (FULL) {
        o += go_val_write(p, ga, o);
        for (int k = 0; k < 10; ++k) *o++ = (uint8_t)K0[k];
        o += go_val_write(p, gk, o);
    } else {
        if (pr.args_len) o += go_transcode(p, pr.args_off, pr.args_off + pr.args_len, o); else { *o++ = '['; *o++ = ']'; }
        for (int k = 0; k < 10; ++k) *o++ = (uint8_t)K0[k];
        if (pr.kw_len) o += go_transcode(p, pr.kw_off, pr.kw_off + pr.kw_len, o); else { *o++ = 'n'; *o++ = 'u'; *o++ = 'l'; *o++ = 'l'; }
    }
    for (uint32_t k = 0; k < tail_len; ++k) *o++ = tail[k];
    const char E0[] = ",\"expires\":\"";
    for (int k = 0; k < 12; ++k) *o++ = (uint8_t)E0[k];
    for (uint32_t k = 0; k < tlen; ++k) *o++ = tbuf[k];
    const char E1[] = "\",\"ttl\":";
    for (int k = 0; k < 8; ++k) *o++ = (uint8_t)E1[k];
    o += put_dec_ll(o, (long long)env.ttl);
    const char E2[] = "},\"retries\":";
    for (int k = 0; k < 12; ++k) *o++ = (uint8_t)E2[k];
    o += put_dec_ll(o, (long long)retries);
    const char E3[] = ",\"timestamp\":";
    for (int k = 0; k < 13; ++k) *o++ = (uint8_t)E3[k];
    o += put_dec_ll(o, ts);
    *o++ = '}';
}

#endif

}  // namespace b9
