// TEST INFRASTRUCTURE: compiles the device's sequential path (the payload parser, parse_task_msg, the handlers and
// handler_phase_a) for the host and reports, per task, the status and the exception class the drain kernels hand to
// the retry policy (an ERROR record's TaskRec::value, a B9_EXC_* bit), so that the class can be compared with the
// oracle's type(e) on a CPU (tests/test_retry_on_host.py).
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

// kind: 0 = an SDK put payload, 1 = an HTTP body (B9_TF_HTTP_BODY), 2 = a TaskMessage record of the task `id` (B9_TF_TASK_MSG)
extern "C" void b9_retry_classify(const uint8_t* p, uint32_t n, int kind, const uint8_t* id, int handler, uint8_t* status, uint8_t* exc) {
    static uint32_t table[256];
    static bool have = false;
    if (!have) { for (uint32_t i = 0; i < 256; ++i) table[i] = b9::crc_table_entry(i); have = true; }
    const b9::Parsed pr = kind == 2 ? b9::parse_task_msg(p, n, id) : b9::parse_payload(p, n, kind == 1);
    b9::TaskRec rec; memset(&rec, 0, sizeof rec); rec.ready = 1;
    b9::handler_phase_a(handler, p, pr, rec, table);
    *status = rec.status; *exc = rec.status == b9::ST_ERROR ? (uint8_t)rec.value : 0;
}
