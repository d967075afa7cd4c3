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

// ---- handlers with a declared signature (B9H_SIGNATURE): `call` receives the bound call -------------------------------
template <class Out> __device__ void put_str(const b9h::Arg& s, Out& out) {
    b9h::Chars c = s.chars();
    uint32_t cp;
    while (c.next(cp)) out.cp(cp);
}
template <class Out> __device__ void put_ascii(const char* s, Out& out) { for (; *s; ++s) out.cp((uint8_t)*s); }

// def greet(name, greeting="Hello", *, punct="!"): return greeting + ", " + name + punct
// (str + a non-str raises TypeError)
struct Greet {
    B9H_SIGNATURE(B9H_POS_OR_KW("name"), B9H_POS_OR_KW_OPT("greeting"), B9H_KW_ONLY_OPT("punct"));
    template <class Out> __device__ static int call(const b9h::Call& c, Out& out) {
        for (int i = 0; i < 3; ++i)
            if (c.has(i) && c[i].kind() != b9h::STR) return B9_EXC_TYPE_ERROR;
        out.str_begin();
        if (c.has(1)) put_str(c[1], out); else put_ascii("Hello", out);
        put_ascii(", ", out);
        put_str(c[0], out);
        if (c.has(2)) put_str(c[2], out); else put_ascii("!", out);
        out.str_end();
        return 0;
    }
};

// def join(sep, *parts):
//     if type(sep) is not str or any(type(p) is not str for p in parts): raise TypeError
//     return sep.join(parts)
struct Join {
    B9H_SIGNATURE(B9H_POS_OR_KW("sep"), B9H_VAR_POS("parts"));
    template <class Out> __device__ static int call(const b9h::Call& c, Out& out) {
        if (c[0].kind() != b9h::STR) return B9_EXC_TYPE_ERROR;
        b9h::Items it = c.rest();
        b9h::Arg x;
        while (it.next(x)) if (x.kind() != b9h::STR) return B9_EXC_TYPE_ERROR;
        out.str_begin();
        it = c.rest();
        for (bool first = true; it.next(x); first = false) {
            if (!first) put_str(c[0], out);
            put_str(x, out);
        }
        out.str_end();
        return 0;
    }
};

// def field_sum(rows, *, field):
//     total = 0
//     for row in rows:
//         if type(row) is not dict: raise TypeError
//         v = row[field]                                   (KeyError when the row has no such key)
//         if type(v) not in (int, float, bool): raise TypeError
//         total += v
//     return total
// A field that is not a str raises TypeError before the loop. ints add exactly while the sum fits in int64 (past it
// the device declines: Python goes on with a big int); from the first float on, the sum is a float64 added left to right
// in IEEE round-to-nearest. A str or dict `rows` iterates its characters / keys (TypeError, unless empty); other
// non-iterables raise TypeError.
struct FieldSum {
    B9H_SIGNATURE(B9H_POS_OR_KW("rows"), B9H_KW_ONLY("field"));
    template <class Out> __device__ static int call(const b9h::Call& c, Out& out) {
        const b9h::Arg rows = c[0], field = c[1];
        if (field.kind() != b9h::STR) return B9_EXC_TYPE_ERROR;
        const int k = rows.kind();
        if (k == b9h::STR || k == b9h::DICT) {
            if (!rows.empty()) return B9_EXC_TYPE_ERROR;
            out.integer(0);
            return 0;
        }
        if (k != b9h::LIST) return B9_EXC_TYPE_ERROR;
        long long si = 0; double sf = 0.0; bool fl = false;
        b9h::Items it = rows.items();
        b9h::Arg row, v;
        while (it.next(row)) {
            if (row.kind() != b9h::DICT) return B9_EXC_TYPE_ERROR;
            if (!row.get(field, v)) return B9_EXC_KEY_ERROR;
            const int kv = v.kind();
            if (kv != b9h::INT && kv != b9h::FLOAT && kv != b9h::BOOL) return B9_EXC_TYPE_ERROR;
            long long vi = 0; double vf = 0.0;
            const int t = v.number(&vi, &vf);
            if (t == B9H_DECLINE) return B9H_DECLINE;
            if (t == b9h::FLOAT) {
                if (!fl) { sf = (double)si; fl = true; }
                sf = b9h::add_rn(sf, vf);
            } else if (fl) {
                sf = b9h::add_rn(sf, (double)vi);
            } else {
                const __int128 r = (__int128)si + vi;
                if (r > (__int128)9223372036854775807ll || r < -(__int128)9223372036854775807ll - 1) return B9H_DECLINE;
                si = (long long)r;
            }
        }
        if (fl) out.real(sf);
        else out.integer(si);
        return 0;
    }
};

// ---- handlers that return lists and dicts -----------------------------------------------------------------------------
// The words of the code points c[i, end) as strings of a list, split as str.split() does (WordCount::is_space)
template <class Out> __device__ void put_words(const b9h::Chars& c, Out& out) {
    b9h::Chars it = c;
    bool in_word = false;
    uint32_t cp;
    out.list_begin();
    while (it.next(cp)) {
        const bool sp = WordCount::is_space(cp);
        if (!sp && !in_word) out.str_begin();
        if (sp && in_word) out.str_end();
        if (!sp) out.cp(cp);
        in_word = !sp;
    }
    if (in_word) out.str_end();
    out.list_end();
}

// def tokens(s, /): return s.split()                     (a non-str has no .split: AttributeError)
struct Tokens {
    template <class Out> __device__ static int call(const b9h::Arg& s, Out& out) {
        if (s.kind() != b9h::STR) return B9_EXC_ATTRIBUTE_ERROR;
        put_words(s.chars(), out);
        return 0;
    }
};

// def grid(s, /): return [line.split() for line in s.split("\n")]
// s.split("\n") splits on U+000A alone: one line more than the string has line feeds.
struct Grid {
    template <class Out> __device__ static int call(const b9h::Arg& s, Out& out) {
        if (s.kind() != b9h::STR) return B9_EXC_ATTRIBUTE_ERROR;
        b9h::Chars it = s.chars(), line = it;
        uint32_t cp;
        out.list_begin();
        for (;;) {
            const uint32_t at = it.i;
            const bool more = it.next(cp);
            if (more && cp != '\n') continue;
            line.end = at;
            put_words(line, out);
            if (!more) break;
            line.i = it.i;
            line.end = it.end;
        }
        out.list_end();
        return 0;
    }
};

template <class Out> __device__ void put_key(const char* k, Out& out) { out.str_begin(); put_ascii(k, out); out.str_end(); }

// def describe(x, /): return {"type": type(x).__name__, "value": x}
struct Describe {
    template <class Out> __device__ static int call(const b9h::Arg& x, Out& out) {
        static const char* const names[] = {"str", "int", "float", "bool", "NoneType", "list", "dict"};
        out.dict_begin();
        put_key("type", out);
        put_key(names[x.kind()], out);
        put_key("value", out);
        out.value(x);
        out.dict_end();
        return 0;
    }
};

// def pick(d, /, *keys):
//     if type(d) is not dict: raise TypeError
//     return {k: d[k] for k in keys}
// A list or dict key is unhashable (TypeError); any other key the dict lacks, a non-str one included, is KeyError. A
// key given twice makes two equal keys in the built dict: the device declines it (UNSUPPORTED).
struct Pick {
    B9H_SIGNATURE(B9H_POS_ONLY("d"), B9H_VAR_POS("keys"));
    template <class Out> __device__ static int call(const b9h::Call& c, Out& out) {
        const b9h::Arg d = c[0];
        if (d.kind() != b9h::DICT) return B9_EXC_TYPE_ERROR;
        b9h::Items it = c.rest();
        b9h::Arg k, v;
        while (it.next(k)) {
            const int kk = k.kind();
            if (kk == b9h::LIST || kk == b9h::DICT) return B9_EXC_TYPE_ERROR;
            if (!d.get(k, v)) return B9_EXC_KEY_ERROR;
        }
        out.dict_begin();
        it = c.rest();
        while (it.next(k)) {
            d.get(k, v);
            out.str_begin(); put_str(k, out); out.str_end();
            out.value(v);
        }
        out.dict_end();
        return 0;
    }
};

}  // namespace b9_examples
