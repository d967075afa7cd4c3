// Example user handlers (include/b9gpu_handler.cuh). Each struct is the device form of the Python function in
// handlers.py next to it, its twin: the tests run both over the same tasks and compare the records byte for byte.
// Plain C++ behind CUDA qualifiers, so that tests/host_shim/user_handler_shim.cpp compiles them with g++ as well.
#pragma once
#include "b9gpu_handler.cuh"

namespace b9_examples {

// def echo_str(s, /): if type(s) is not str: raise TypeError; return s
struct EchoStr {
    template <class Out> __device__ static int call(const b9h::Arg& s, Out& out) {
        if (s.kind() != b9h::STR) return B9_EXC_TYPE_ERROR;
        out.str_begin();
        b9h::Chars c = s.chars();
        uint32_t cp;
        while (c.next(cp)) out.cp(cp);
        out.str_end();
        return 0;
    }
};

// def crc32_str(s, /): return zlib.crc32(s.encode())     (a non-str has no .encode: AttributeError)
// The CRC-32 of the string's UTF-8 bytes, bit by bit (reflected polynomial 0xEDB88320).
struct Crc32Str {
    __device__ static uint32_t crc_byte(uint32_t c, uint32_t b) {
        c ^= b;
        for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1u)));
        return c;
    }
    template <class Out> __device__ static int call(const b9h::Arg& s, Out& out) {
        if (s.kind() != b9h::STR) return B9_EXC_ATTRIBUTE_ERROR;
        uint32_t c = 0xFFFFFFFFu, cp;
        b9h::Chars it = s.chars();
        while (it.next(cp)) {
            if (cp < 0x80) c = crc_byte(c, cp);
            else if (cp < 0x800) { c = crc_byte(c, 0xC0 | (cp >> 6)); c = crc_byte(c, 0x80 | (cp & 0x3F)); }
            else if (cp < 0x10000) {
                c = crc_byte(c, 0xE0 | (cp >> 12)); c = crc_byte(c, 0x80 | ((cp >> 6) & 0x3F)); c = crc_byte(c, 0x80 | (cp & 0x3F));
            } else {
                c = crc_byte(c, 0xF0 | (cp >> 18)); c = crc_byte(c, 0x80 | ((cp >> 12) & 0x3F));
                c = crc_byte(c, 0x80 | ((cp >> 6) & 0x3F)); c = crc_byte(c, 0x80 | (cp & 0x3F));
            }
        }
        out.integer((long long)(~c));
        return 0;
    }
};

// def word_count(s, /): return len(s.split())
// str.split() with no separator splits on runs of the code points CPython's Py_UNICODE_ISSPACE accepts.
struct WordCount {
    __device__ static bool is_space(uint32_t c) {
        if (c < 0x80) return c == ' ' || (c >= 0x09 && c <= 0x0D) || (c >= 0x1C && c <= 0x1F);
        return c == 0x85 || c == 0xA0 || c == 0x1680 || (c >= 0x2000 && c <= 0x200A) || c == 0x2028 || c == 0x2029 ||
               c == 0x202F || c == 0x205F || c == 0x3000;
    }
    template <class Out> __device__ static int call(const b9h::Arg& s, Out& out) {
        if (s.kind() != b9h::STR) return B9_EXC_ATTRIBUTE_ERROR;
        long long n = 0;
        bool in_word = false;
        uint32_t cp;
        b9h::Chars it = s.chars();
        while (it.next(cp)) {
            const bool sp = is_space(cp);
            if (!sp && !in_word) ++n;
            in_word = !sp;
        }
        out.integer(n);
        return 0;
    }
};

// def prod(xs, /):
//     p = 1
//     for x in xs:
//         if type(x) not in (int, float, bool): raise TypeError
//         p *= x
//     return p
// ints multiply exactly while the product fits in int64 (past it the device declines: Python goes on with a big int);
// from the first float on, the product is a float64 multiplied in IEEE round-to-nearest. A str or dict argument iterates
// its characters / keys (str: TypeError, unless empty); other non-iterables raise TypeError.
struct Prod {
    template <class Out> __device__ static int call(const b9h::Arg& xs, Out& out) {
        const int k = xs.kind();
        if (k == b9h::STR || k == b9h::DICT) {
            if (!xs.empty()) return B9_EXC_TYPE_ERROR;
            out.integer(1);
            return 0;
        }
        if (k != b9h::LIST) return B9_EXC_TYPE_ERROR;
        long long pi = 1; double pf = 1.0; bool fl = false;
        b9h::Items it = xs.items();
        b9h::Arg x;
        while (it.next(x)) {
            const int kx = x.kind();
            if (kx != b9h::INT && kx != b9h::FLOAT && kx != b9h::BOOL) return B9_EXC_TYPE_ERROR;
            long long vi = 0; double vf = 0.0;
            const int t = x.number(&vi, &vf);
            if (t == B9H_DECLINE) return B9H_DECLINE;
            if (t == b9h::FLOAT) {
                if (!fl) { pf = (double)pi; fl = true; }
                pf = b9h::mul_rn(pf, vf);
            } else if (fl) {
                pf = b9h::mul_rn(pf, (double)vi);
            } else {
                const __int128 r = (__int128)pi * vi;
                if (r > (__int128)9223372036854775807ll || r < -(__int128)9223372036854775807ll - 1) return B9H_DECLINE;
                pi = (long long)r;
            }
        }
        if (fl) out.real(pf);
        else out.integer(pi);
        return 0;
    }
};

}  // namespace b9_examples
