// TEST INFRASTRUCTURE: compiles the device's sequential path for TaskMessage records (task_msg.cuh: parse_task_msg and
// its domain checks) together with the payload parser and the handlers for the host, so that the record path can be
// compared with the oracle and with the payload path on a CPU (tests/test_task_msg_on_host.py).
#include <stdint.h>
#include <string.h>
#define __device__
#define __host__
#define __forceinline__ inline
#define __constant__ static const
static inline float __uint_as_float(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline uint32_t __float_as_uint(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline float __fadd_rn(float a, float b) { volatile float z = a + b; return z; }     // IEEE binary32, round to nearest even
static inline uint32_t __funnelshift_r(uint32_t lo, uint32_t hi, uint32_t sh) { return (uint32_t)(((((uint64_t)hi) << 32) | lo) >> (sh & 31u)); }
#include "../../beta9_b200/csrc/handler_seq.cuh"
#include "../../beta9_b200/csrc/task_msg.cuh"

static const uint32_t* crc_table() {
    static uint32_t table[256];
    static bool have = false;
    if (!have) { for (uint32_t i = 0; i < 256; ++i) table[i] = b9::crc_table_entry(i); have = true; }
    return table;
}

// one task through parse (record: parse_task_msg against `id`, else parse_payload) -> handler_phase_a -> result bytes.
// Returns the result length (0 with *has == 0: no result bytes), or -1 if `cap` is too small.
extern "C" long b9_tm_run(const uint8_t* p, uint32_t n, int record, const uint8_t* id, int handler, uint8_t* status, uint8_t* has,
                          uint8_t* out, uint32_t cap) {
    const b9::Parsed pr = record ? b9::parse_task_msg(p, n, id) : b9::parse_payload(p, n, false);
    b9::TaskRec rec; memset(&rec, 0, sizeof rec); rec.ready = 1;
    b9::handler_phase_a(handler, p, pr, rec, crc_table());
    *status = rec.status; *has = rec.has;
    if (!rec.has) return 0;
    if (rec.out_len > cap) return -1;
    if (rec.mode == b9::OM_COPY) memcpy(out, p + rec.src_off, rec.src_len);
    else b9::seq_emit(p, rec, out);
    return (long)rec.out_len;
}

extern "C" int b9_tm_utf8_surrogatepass(const uint8_t* p, uint32_t n) { return b9::utf8_valid_surrogatepass(p, n) ? 1 : 0; }
