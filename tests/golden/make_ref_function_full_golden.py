"""Runs the REFERENCE's own function path for plain Python values under all four handlers and freezes what it produced.

    B9_REFERENCE_SDK=<beta9 checkout>/sdk/src python tests/golden/make_ref_function_full_golden.py   (from the repo root)

The same harness as make_ref_function_golden.py: the unmodified `_CallableWrapper._call_remote`
(sdk/src/beta9/abstractions/function.py:198-232) frames each call, the unmodified `invoke_function`
(sdk/src/beta9/runner/function.py:236-283) runs it (cloudpickle.loads, `callback_url` popped, handler(*args, **kwargs),
cloudpickle.dumps); only the gRPC stubs are replaced. The inputs are the domain of B9_DRAIN_PICKLE_FULL
(include/b9gpu.h): configs[4] documents and float documents, floats, bytes and base64 bytes for vadd_f32, shared objects
and separate equal objects (CPython's str singletons), `callback_url`-only keyword arguments, the integer opcode
boundaries. Output: tests/golden/ref_function_full_golden.json, checked by tests/test_pickle_on_host.py (oracle and the
host build of the codec) and tests/test_gpu_function_full.py (the device)."""
import asyncio
import base64
import json
import math
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_ref_runner_golden import load_reference_runner  # noqa: E402

HANDLERS = ["identity", "crc32", "vadd_f32", "json_sum"]


def calls():
    """(args tuple, kwargs dict) of each `_call_remote`"""
    from beta9_b200 import synth
    out = []
    for b in (synth.json_batch(6), synth.json_float_batch(4)):
        raw = b.payload.tobytes()
        out += [((json.loads(raw[int(b.offsets[i]):int(b.offsets[i + 1])])["args"][0],), {}) for i in range(b.n)]
    ints = [0, 1, 255, 256, 65535, 65536, 2**31 - 1, 2**31, -1, -2**31, -2**31 - 1, 2**32, 2**63 - 1, 2**63, -2**63 - 1, 10**30]
    floats = [0.0, -0.0, 1.5, math.inf, -math.inf, math.nan, 5e-324, 1e308]
    vadd_raw = [bytes(range(8)), bytes(range(16, 48)), b""]
    ab1, ab2 = "".join(["a", "b"]), "".join(["a", "b"])             # two equal, separate str objects
    e1, e2 = "".join(["\xe9"]), "".join(["\xe9"])                   # "é": CPython's singleton
    shared = ["s", 1]
    vals = ints + floats + [None, True, False, "", "a", "é", "\ud83d", "x" * 300, b"", b"x", b"raw bytes",
                            [ab1, ab2], [e1, e2], [shared, shared], (shared, shared), [b"", b""], (), (1,), (1, 2, 3, 4),
                            list(range(1001)), [str(i) for i in range(300)], {"a": 1, "b": [2.5, None]},
                            {1: "i", 2.5: "f", None: "n", b"k": "b"}, [[[[1]]]]]
    vals += [base64.b64encode(r) for r in vadd_raw] + [base64.b64encode(r).decode() for r in vadd_raw] + ["AAA=", "é"]
    vals += [{"values": v} for v in ([1, 2.5, True], (1, 2), [2**63 - 1], [0.1] * 10, [1, None], [], "ab", None)]
    out += [((v,), {}) for v in vals]
    out += [(("cb",), {"callback_url": "http://callback"}), (({"values": [3, 4]},), {"callback_url": "u"}),
            (("x",), {"k": 1}), (("a", "b"), {}), ((), {})]
    return out


def main():
    load_reference_runner()
    os.environ["STUB_TYPE"] = "function"
    import beta9.abstractions.function as af
    import beta9.runner.function as rf
    import beta9.runner.common as rc
    import beta9.clients.function as cf
    from oracle.pyoracle import handlers as H
    out = {"source": "reference function path: abstractions/function.py:198-232 (framing), runner/function.py:236-283 (loop)", "cases": []}

    captured = []

    class InvokeStub:
        def function_invoke(self, req):
            captured.append(bytes(req.args))
            yield af.FunctionInvokeResponse(done=True, exit_code=0, result=b"", task_id="t")

    parent = af.Function.__new__(af.Function)
    parent.function_stub = InvokeStub()
    parent.stub_id = "stub"; parent.headless = False; parent.handler = "mod:f"
    w = af._CallableWrapper(H.identity, parent)
    for args, kwargs in calls():
        captured.clear()
        w._call_remote(*args, **kwargs)
        assert len(captured) == 1
        out["cases"].append({"input_repr": repr((args, kwargs))[:80], "args_pickle": base64.b64encode(captured[0]).decode(), "results": {}})

    for h in HANDLERS:
        fw = af._CallableWrapper(getattr(H, h), parent)
        mod = types.ModuleType("ref_fn_handlers"); setattr(mod, h, fw)
        sys.modules["ref_fn_handlers"] = mod
        rc.config.handler = f"ref_fn_handlers:{h}"
        for c in out["cases"]:
            args_bytes = base64.b64decode(c["args_pickle"])
            got = {}

            class FnStub:
                def function_get_args(self, req):
                    return cf.FunctionGetArgsResponse(ok=True, args=args_bytes)

                def function_set_result(self, req):
                    got["result"] = bytes(req.result)
                    return cf.FunctionSetResultResponse(ok=True)

            ctx = rc.FunctionContext.new(config=rc.config, task_id="00000000-0000-4000-8000-000000000000", on_start_value=None)
            res = asyncio.run(rf.invoke_function(FnStub(), ctx, "00000000-0000-4000-8000-000000000000"))
            ok = res.exception is None
            c["results"][h] = {"ok": ok, "result_pickle": base64.b64encode(got["result"]).decode() if ok and "result" in got else None,
                               "exception": None if ok else type(res.exception).__name__}
    path = os.path.join(ROOT, "tests", "golden", "ref_function_full_golden.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
    print(path, len(out["cases"]), "inputs x", len(HANDLERS), "handlers through the reference function runner")


if __name__ == "__main__":
    main()
