// Test-only user handler (include/b9gpu_handler.cuh) that drives the container calls of the sinks: lists, dicts and
// value(). Its Python twin is container_twins.py; the host shim (tests/host_shim/user_containers_shim.cpp) and the
// device cubin (containers.cu, build.build_test_handlers) run the same source. Plain C++ behind CUDA qualifiers, as
// examples/handlers/handlers.cuh.
#pragma once
#include "b9gpu_handler.cuh"

namespace b9_containers {

template <class Out> struct is_write_sink { static constexpr bool value = false; };
template <int R> struct is_write_sink<b9h::WriteSink<R>> { static constexpr bool value = true; };

// def cscript(ops, *rest): a sink-call interpreter. ops is a list of int lists [code, a] or [code, hi, lo] (a 64-bit
// argument as two unsigned 32-bit halves), with contract.cuh's codes
//   0 none()   1 boolean(a)   2 integer(a)   3 real(the double of bits a)   4 str_begin()   5 cp(a)   6 str_end()
//   7 return a   8 cp(a) in the writing pass only   9 cp(a) in the counting pass only
// and the container calls
//   10 list_begin()   11 list_end()   12 dict_begin()   13 dict_end()   14 value(rest[a])
// Without a 7 it returns 0. A malformed script (not a list of 1-3 INTs with a known code, or a 14 past the end of rest)
// raises TypeError.
struct CScript {
    B9H_SIGNATURE(B9H_POS_OR_KW("ops"), B9H_VAR_POS("rest"));
    template <class Out> __device__ static int call(const b9h::Call& c, Out& out) {
        const b9h::Arg ops = c[0];
        if (ops.kind() != b9h::LIST) return B9_EXC_TYPE_ERROR;
        b9h::Items it = ops.items();
        b9h::Arg op;
        while (it.next(op)) {
            if (op.kind() != b9h::LIST) return B9_EXC_TYPE_ERROR;
            long long a[3] = {0, 0, 0};
            int n = 0;
            b9h::Items f = op.items();
            b9h::Arg x;
            while (f.next(x)) {
                double d;
                if (n == 3 || x.kind() != b9h::INT || x.number(&a[n], &d) != b9h::INT) return B9_EXC_TYPE_ERROR;
                ++n;
            }
            if (n == 0) return B9_EXC_TYPE_ERROR;
            const long long v = n == 3 ? (long long)(((unsigned long long)(uint32_t)a[1] << 32) | (uint32_t)a[2]) : a[1];
            switch (a[0]) {
            case 0: out.none(); break;
            case 1: out.boolean(v != 0); break;
            case 2: out.integer(v); break;
            case 3: out.real(b9::f64_from_bits((unsigned long long)v)); break;
            case 4: out.str_begin(); break;
            case 5: out.cp((uint32_t)v); break;
            case 6: out.str_end(); break;
            case 7: return (int)v;
            case 8: if (is_write_sink<Out>::value) out.cp((uint32_t)v); break;
            case 9: if (!is_write_sink<Out>::value) out.cp((uint32_t)v); break;
            case 10: out.list_begin(); break;
            case 11: out.list_end(); break;
            case 12: out.dict_begin(); break;
            case 13: out.dict_end(); break;
            case 14: {
                b9h::Items r = c.rest();
                b9h::Arg y;
                bool found = false;
                for (long long k = 0; k <= v && (found = r.next(y)); ++k) {}
                if (v < 0 || !found) return B9_EXC_TYPE_ERROR;
                out.value(y);
                break;
            }
            default: return B9_EXC_TYPE_ERROR;
            }
        }
        return 0;
    }
};

}  // namespace b9_containers
