// TEST INFRASTRUCTURE: the device's float64 codec (beta9_b200/csrc/f64_device.cuh) compiled for the host, in batch
// entry points, so that tests/test_f64_on_host.py can hold it against Python's float() and repr() by the million.
#include <stdint.h>
#include <string.h>
#define __device__
#define __host__
#define __forceinline__ inline
#define __constant__ static const
#include "../../beta9_b200/csrc/f64_device.cuh"

// literals buf[off[i]..off[i+1]) -> bits[i], ok[i] (0: declined), over[i] (number_overflows_f64)
extern "C" void b9_f64_parse_batch(const uint8_t* buf, const uint64_t* off, uint64_t n, uint64_t* bits, uint8_t* ok, uint8_t* over) {
    for (uint64_t i = 0; i < n; ++i) {
        const uint32_t s = (uint32_t)off[i], e = (uint32_t)off[i + 1];
        unsigned long long b = 0;
        ok[i] = (uint8_t)b9::f64_parse(buf, s, e, &b);
        bits[i] = b;
        over[i] = b9::number_overflows_f64(buf, s, e) ? 1 : 0;
    }
}

// which = 0 go_json_float, 1 py_json_float, 2 py_json_go_number; the texts joined by '\n'. Returns the bytes written.
extern "C" uint64_t b9_f64_format_batch(const uint64_t* bits, uint64_t n, int which, uint8_t* out) {
    uint64_t k = 0;
    for (uint64_t i = 0; i < n; ++i) {
        uint32_t want = which == 0 ? b9::go_json_float(bits[i], nullptr) : which == 1 ? b9::py_json_float(bits[i], nullptr) : b9::py_json_go_number(bits[i], nullptr);
        uint32_t got = which == 0 ? b9::go_json_float(bits[i], out + k) : which == 1 ? b9::py_json_float(bits[i], out + k) : b9::py_json_go_number(bits[i], out + k);
        if (got != want) return 0;                 // the sizing pass and the writing pass disagree
        k += got;
        out[k++] = '\n';
    }
    return k;
}
