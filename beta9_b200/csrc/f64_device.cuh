// binary64 <-> decimal on the device: the number half of the JSON round trip a task's argument makes.
//
// Every JSON number of a payload is a float64 in the reference's path (Go's decoder), is written again by Go's
// encoder (`TaskMessage.Encode`) and read by the runner's `json.loads`, which makes it a Python int when Go's text has
// no '.' or exponent and a float otherwise; `json.dumps` finally writes the int's digits or the float's repr. So
// what the device needs is:
//   * f64_parse: a correctly rounded decimal -> binary64 parse (Go's strconv.ParseFloat), by Eisel-Lemire with a
//     128-bit table of powers of five (D. Lemire, "Number parsing at a gigabyte per second", 2021; without the
//     fallback: N. Mushtak, D. Lemire, "Fast number parsing without fallback", 2023). A literal of more than 19
//     significant digits is rounded from its first 19 digits w and from w + 1: when both give the same double that
//     is the answer, otherwise the parse is DECLINED (the caller reports B9_ST_UNSUPPORTED, it never guesses).
//   * f64_shortest: the shortest decimal that rounds back to the double, the closest one when there are several,
//     ties to an even last digit -- what CPython's repr and Go's strconv (precision -1) both produce. Schubfach
//     (R. Giulietti, "The Schubfach way to render doubles", 2020), without Java's two-digit minimum.
//   * three writers on those digits: go_json_float (Go encoding/json's float64 encoder), py_json_float
//     (CPython json.dumps of a float: repr, Infinity, NaN) and py_json_go_number (json.dumps of what json.loads
//     makes of Go's text: int digits or repr).
// Plain C++ behind CUDA qualifiers: tests/host_shim compiles this file for the host (tests/test_f64_on_host.py).
// The entry points are out of line so that the kernels' main loops keep their register allocation.
#pragma once
#include <stdint.h>
#include "json_device.cuh"
#include "f64_tables.cuh"
#ifndef __noinline__
#define __noinline__ __attribute__((noinline))     // (host build)
#endif

namespace b9 {

// ---- decimal digits of unsigned integers --------------------------------------------------------------------
// (Round 1 divided by ten in 64 bits, one lane per task while 31 idle: 6-9 % of the crc32 and json_sum
// kernels' instructions went into printing ~10 digits. Now: compares against powers
// of ten and 32-bit multiply-shift division by 10, in at most three 9-digit limbs.)
__device__ __forceinline__ uint32_t dec_len_u32(uint32_t v) {
    return 1u + (v >= 10u) + (v >= 100u) + (v >= 1000u) + (v >= 10000u) + (v >= 100000u) + (v >= 1000000u) + (v >= 10000000u) + (v >= 100000000u) + (v >= 1000000000u);
}
__device__ __forceinline__ uint32_t dec_len_u64(unsigned long long v) {
    if (v < 4294967296ull) return dec_len_u32((uint32_t)v);
    const unsigned long long hi = v / 1000000000ull;                    // >= 4: v has more than 9 digits
    if (hi < 4294967296ull) return 9u + dec_len_u32((uint32_t)hi);
    return 18u + dec_len_u32((uint32_t)(hi / 1000000000ull));
}
// exactly n digits of x (x < 10^n), most significant first, zero-padded on the left
__device__ __forceinline__ void write_dec_u32(uint8_t* o, uint32_t x, uint32_t n) {
    for (uint32_t k = n; k-- > 0;) {
        const uint32_t q = (uint32_t)(((unsigned long long)x * 0xCCCCCCCDull) >> 35);   // x / 10
        o[k] = (uint8_t)('0' + (x - q * 10u));
        x = q;
    }
}
__device__ inline void write_dec(uint8_t* o, unsigned long long v, uint32_t len) {
    if (v < 4294967296ull) { write_dec_u32(o, (uint32_t)v, len); return; }
    const unsigned long long hi = v / 1000000000ull;
    write_dec_u32(o + (len - 9u), (uint32_t)(v - hi * 1000000000ull), 9u);
    if (hi < 4294967296ull) { write_dec_u32(o, (uint32_t)hi, len - 9u); return; }
    const unsigned long long top = hi / 1000000000ull;
    write_dec_u32(o + (len - 18u), (uint32_t)(hi - top * 1000000000ull), 9u);
    write_dec_u32(o, (uint32_t)top, len - 18u);
}

// ---- 64-bit helpers that the host build gets from the compiler ----------------------------------------------
__device__ __forceinline__ unsigned long long f64_mulhi(unsigned long long a, unsigned long long b) {
#ifdef __CUDA_ARCH__
    return __umul64hi(a, b);
#else
    return (unsigned long long)(((unsigned __int128)a * b) >> 64);
#endif
}
__device__ __forceinline__ int f64_clz64(unsigned long long x) {      // x != 0
#ifdef __CUDA_ARCH__
    return __clzll((long long)x);
#else
    return __builtin_clzll(x);
#endif
}
__device__ __forceinline__ double f64_from_bits(unsigned long long b) {
#ifdef __CUDA_ARCH__
    return __longlong_as_double((long long)b);
#else
    double d; __builtin_memcpy(&d, &b, 8); return d;
#endif
}
__device__ __forceinline__ unsigned long long f64_to_bits(double d) {
#ifdef __CUDA_ARCH__
    return (unsigned long long)__double_as_longlong(d);
#else
    unsigned long long b; __builtin_memcpy(&b, &d, 8); return b;
#endif
}

// ---- decimal -> binary64 --------------------------------------------------------------------------------------
// w * 10^q, w != 0 with at most 19 digits, rounded to nearest even: the bits of the magnitude (+Inf on overflow,
// 0 on underflow). Eisel-Lemire as in fast_float's compute_float for binary64; exact for every such w and q
// (Mushtak & Lemire 2023), so there is no fallback.
__device__ inline unsigned long long f64_eisel_lemire(unsigned long long w, long long q) {
    if (q < F64_POW5_QMIN) return 0ull;
    if (q > F64_POW5_QMAX) return 0x7FF0000000000000ull;
    const int lz = f64_clz64(w);
    w <<= lz;
    const int idx = (int)(q - F64_POW5_QMIN);
    const unsigned long long t_hi = F64_POW5_128[idx][0], t_lo = F64_POW5_128[idx][1];
    unsigned long long hi = f64_mulhi(w, t_hi), lo = w * t_hi;
    if ((hi & 0x1FFull) == 0x1FFull) {                                  // the low half of the table entry can carry in
        const unsigned long long h2 = f64_mulhi(w, t_lo);
        lo += h2;
        if (lo < h2) ++hi;
    }
    const int upper = (int)(hi >> 63);
    const int shift = upper + 9;
    unsigned long long m = hi >> shift;
    int p2 = (int)((((152170 + 65536) * q) >> 16) + 63) + upper - lz + 1023;
    if (p2 <= 0) {                                                      // subnormal (or zero)
        if (-p2 + 1 >= 64) return 0ull;
        m >>= -p2 + 1;
        m += m & 1ull; m >>= 1;
        // rounding may carry into the smallest normal exponent
        return (m < (1ull << 52)) ? m : ((1ull << 52) | (m & ((1ull << 52) - 1ull)));
    }
    // exactly between two doubles: only possible while 5^q fits in 64 bits (q in [-4, 23]); round to even
    if (lo <= 1ull && q >= -4 && q <= 23 && (m & 3ull) == 1ull && (m << shift) == hi) m &= ~1ull;
    m += m & 1ull; m >>= 1;
    if (m >= (2ull << 52)) { m = 1ull << 52; ++p2; }
    m &= ~(1ull << 52);
    if (p2 >= 0x7FF) return 0x7FF0000000000000ull;
    return ((unsigned long long)p2 << 52) | m;
}

// p[s..e) is a syntactically valid JSON number. 1: *bits is strconv.ParseFloat's result (+-Inf where it reports
// ErrRange, which agrees with number_overflows_f64; +-0 on underflow). 0: DECLINED -- the literal has more than 19
// significant digits and its first 19 (w) and w + 1 round to different doubles.
__device__ __noinline__ int f64_parse(const uint8_t* __restrict__ p, uint32_t s, uint32_t e, unsigned long long* bits) {
    uint32_t i = s;
    const bool neg = p[i] == '-';
    if (neg) ++i;
    unsigned long long w = 0;
    uint32_t nd = 0;                          // significant digits taken into w (<= 19)
    long long dp = 0;                         // value = w * 10^(dp - nd) * 10^ex (before the dropped digits)
    bool dropped_nonzero = false, seen = false;
    for (; i < e && is_digit(p[i]); ++i) {
        const uint32_t d = p[i] - '0';
        if (!seen && d == 0) continue;
        seen = true;
        if (nd < 19) { w = w * 10 + d; ++nd; } else if (d) dropped_nonzero = true;
        ++dp;
    }
    if (i < e && p[i] == '.') {
        for (++i; i < e && is_digit(p[i]); ++i) {
            const uint32_t d = p[i] - '0';
            if (!seen && d == 0) { --dp; continue; }
            seen = true;
            if (nd < 19) { w = w * 10 + d; ++nd; } else if (d) dropped_nonzero = true;
        }
    }
    long long ex = 0;
    if (i < e && (p[i] == 'e' || p[i] == 'E')) {
        ++i; bool en = false;
        if (p[i] == '+') ++i; else if (p[i] == '-') { en = true; ++i; }
        for (; i < e; ++i) if (ex < 100000000) ex = ex * 10 + (p[i] - '0');
        if (en) ex = -ex;
    }
    const unsigned long long sign = neg ? (1ull << 63) : 0ull;
    if (w == 0) { *bits = sign; return 1; }
    const long long q = dp - (long long)nd + ex;
    unsigned long long r = f64_eisel_lemire(w, q);
    if (dropped_nonzero && f64_eisel_lemire(w + 1, q) != r) return 0;   // the true value lies in (w, w + 1) * 10^q
    *bits = sign | r;
    return 1;
}

// ---- binary64 -> shortest decimal -----------------------------------------------------------------------------
struct F64Dec {
    unsigned long long f;     // the digits, no trailing zeros (0 for zero / Inf / NaN)
    int n;                    // how many
    int dp;                   // |x| = 0.d1d2..dn x 10^dp
    uint8_t neg, cls;         // cls: 0 finite non-zero, 1 zero, 2 infinity, 3 NaN
};

__device__ __forceinline__ long long f64_flog10pow2(long long e) { return (e * 661971961083ll) >> 41; }
__device__ __forceinline__ long long f64_flog10_34pow2(long long e) { return (e * 661971961083ll - 274743187321ll) >> 41; }
__device__ __forceinline__ long long f64_flog2pow10(long long e) { return (e * 913124641741ll) >> 38; }
// g * cp / 2^127 rounded down, with the lowest bit set when the quotient is inexact (Giulietti's rop)
__device__ __forceinline__ unsigned long long f64_rop(unsigned long long g1, unsigned long long g0, unsigned long long cp) {
    const unsigned long long x1 = f64_mulhi(g0, cp), y0 = g1 * cp, y1 = f64_mulhi(g1, cp);
    const unsigned long long z = (y0 >> 1) + x1;
    const unsigned long long vbp = y1 + (z >> 63);
    return vbp | (((z & 0x7FFFFFFFFFFFFFFFull) + 0x7FFFFFFFFFFFFFFFull) >> 63);
}

__device__ __noinline__ F64Dec f64_shortest(unsigned long long bits) {
    F64Dec r; r.neg = (uint8_t)(bits >> 63); r.f = 0; r.n = 0; r.dp = 0; r.cls = 0;
    const unsigned long long t = bits & ((1ull << 52) - 1ull);
    const int bq = (int)((bits >> 52) & 0x7FFu);
    if (bq == 0x7FF) { r.cls = t ? 3 : 2; return r; }
    if (bq == 0 && t == 0) { r.cls = 1; return r; }
    unsigned long long c; long long q;
    if (bq) { c = t | (1ull << 52); q = bq - 1075; } else { c = t; q = -1074; }
    unsigned long long f; long long k10;
    if (q < 0 && q > -53 && ((c >> -q) << -q) == c) { f = c >> -q; k10 = 0; }   // an integer below 2^53: its own digits
    else {
        const unsigned long long cb = c << 2, cbr = cb + 2;
        unsigned long long cbl; long long k;
        if (c != (1ull << 52) || q == -1074) { cbl = cb - 2; k = f64_flog10pow2(q); }
        else { cbl = cb - 1; k = f64_flog10_34pow2(q); }                // the gap below a power of two is half the one above
        const int h = (int)(q + f64_flog2pow10(-k) + 2);
        const unsigned long long g1 = F64_G_126[k - F64_G_KMIN][0], g0 = F64_G_126[k - F64_G_KMIN][1];
        const unsigned long long vb = f64_rop(g1, g0, cb << h), vbl = f64_rop(g1, g0, cbl << h), vbr = f64_rop(g1, g0, cbr << h);
        const unsigned long long s = vb >> 2, out = c & 1ull;
        // one digit fewer: at most one multiple of ten lies in the rounding interval (it is < 10 units wide)
        const unsigned long long sp10 = (s / 10u) * 10u, tp10 = sp10 + 10u;
        const bool upin = vbl + out <= (sp10 << 2), wpin = (tp10 << 2) + out <= vbr;
        if (upin != wpin) { f = upin ? sp10 : tp10; k10 = k; }
        else {
            const unsigned long long tt = s + 1;
            const bool uin = vbl + out <= (s << 2), win = (tt << 2) + out <= vbr;
            if (uin != win) f = uin ? s : tt;
            else {
                const long long cmp = (long long)(vb - ((s + tt) << 1));
                f = (cmp < 0 || (cmp == 0 && (s & 1ull) == 0)) ? s : tt;
            }
            k10 = k;
        }
    }
    while (f % 10u == 0) { f /= 10u; ++k10; }
    r.f = f; r.n = (int)dec_len_u64(f); r.dp = (int)(r.n + k10);
    return r;
}

// ---- writers: o == nullptr sizes only; all return the byte count ---------------------------------------------
// d1..dn as `ip.fp` with the decimal point at position dp (fixed notation, no exponent); add_dot0: "x.0" for integers
__device__ inline uint32_t f64_put_fixed(const F64Dec& d, uint8_t* o, bool add_dot0) {
    uint32_t n = 0;
    if (d.dp <= 0) {                                                    // 0.000ddd
        const uint32_t z = (uint32_t)(-d.dp);
        if (o) { o[0] = '0'; o[1] = '.'; for (uint32_t k = 0; k < z; ++k) o[2 + k] = '0'; write_dec(o + 2 + z, d.f, (uint32_t)d.n); }
        return 2u + z + (uint32_t)d.n;
    }
    if (d.dp >= d.n) {                                                  // ddd000[.0]
        const uint32_t z = (uint32_t)(d.dp - d.n);
        if (o) { write_dec(o, d.f, (uint32_t)d.n); for (uint32_t k = 0; k < z; ++k) o[d.n + k] = '0'; if (add_dot0) { o[d.dp] = '.'; o[d.dp + 1] = '0'; } }
        n = (uint32_t)d.dp + (add_dot0 ? 2u : 0u);
        return n;
    }
    if (o) {                                                            // dd.ddd
        uint8_t* t = o + 1;                                             // digits one place right, then the integer part moves left
        write_dec(t, d.f, (uint32_t)d.n);
        for (int k = 0; k < d.dp; ++k) o[k] = t[k];
        o[d.dp] = '.';
    }
    return (uint32_t)d.n + 1u;
}
// d1[.d2..dn] 'e' sign exponent, at least min_exp_digits exponent digits
__device__ inline uint32_t f64_put_sci(const F64Dec& d, uint8_t* o, uint32_t min_exp_digits) {
    const int x = d.dp - 1;
    const uint32_t ax = (uint32_t)(x < 0 ? -x : x);
    uint32_t el = dec_len_u32(ax);
    if (el < min_exp_digits) el = min_exp_digits;
    const uint32_t mant = d.n > 1 ? (uint32_t)d.n + 1u : 1u;
    if (o) {
        if (d.n > 1) { write_dec(o + 1, d.f, (uint32_t)d.n); o[0] = o[1]; o[1] = '.'; }
        else o[0] = (uint8_t)('0' + d.f);
        o[mant] = 'e'; o[mant + 1] = x < 0 ? '-' : '+';
        write_dec_u32(o + mant + 2, ax, el);
    }
    return mant + 2u + el;
}
__device__ __forceinline__ uint32_t f64_put_str(const char* s, uint32_t n, uint8_t* o) { if (o) for (uint32_t k = 0; k < n; ++k) o[k] = (uint8_t)s[k]; return n; }

// Go encoding/json, float64 (encode.go floatEncoder): strconv 'f' with the shortest digits, 'e' when |x| < 1e-6 or
// |x| >= 1e21, "e-07" shortened to "e-7"; zero is "0" / "-0". Only finite values (Go refuses Inf and NaN).
__device__ __noinline__ uint32_t go_json_float(unsigned long long bits, uint8_t* o) {
    const F64Dec d = f64_shortest(bits);
    uint32_t n = 0;
    if (d.neg) { if (o) o[0] = '-'; n = 1; }
    if (d.cls == 1) return n + f64_put_str("0", 1, o ? o + n : nullptr);
    // |x| < 1e-6 <=> dp <= -6;  |x| >= 1e21 <=> dp >= 22
    if (d.dp <= -6 || d.dp >= 22) return n + f64_put_sci(d, o ? o + n : nullptr, (d.dp - 1 < 0) ? 1u : 2u);
    return n + f64_put_fixed(d, o ? o + n : nullptr, false);
}

// CPython json.dumps(float): float.__repr__ ('r' format: scientific when the exponent dp - 1 is < -4 or >= 16, two or
// more exponent digits; "x.0" for integral fixed output), and Infinity / -Infinity / NaN for the non-finite values.
__device__ __noinline__ uint32_t py_json_float(unsigned long long bits, uint8_t* o) {
    const F64Dec d = f64_shortest(bits);
    if (d.cls == 3) return f64_put_str("NaN", 3, o);
    uint32_t n = 0;
    if (d.neg) { if (o) o[0] = '-'; n = 1; }
    uint8_t* const t = o ? o + n : nullptr;
    if (d.cls == 2) return n + f64_put_str("Infinity", 8, t);
    if (d.cls == 1) return n + f64_put_str("0.0", 3, t);
    if (d.dp <= -4 || d.dp > 16) return n + f64_put_sci(d, t, 2u);
    return n + f64_put_fixed(d, t, true);
}

// json.dumps(json.loads(<go_json_float text>)) for a finite x: Python makes an int of Go's text when it has no '.' and
// no exponent (x integral and |x| < 1e21, or zero: "-0" is the int 0), a float equal to x otherwise.
__device__ __noinline__ uint32_t py_json_go_number(unsigned long long bits, uint8_t* o) {
    const F64Dec d = f64_shortest(bits);
    if (d.cls == 1) return f64_put_str("0", 1, o);
    if (d.dp >= d.n && d.dp < 22) {                                     // Go wrote digits only: the int's digits
        uint32_t n = 0;
        if (d.neg) { if (o) o[0] = '-'; n = 1; }
        return n + f64_put_fixed(d, o ? o + n : nullptr, false);
    }
    return py_json_float(bits, o);
}

}  // namespace b9
