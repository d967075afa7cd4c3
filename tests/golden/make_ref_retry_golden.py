"""Runs the REFERENCE's own runner loop with a stub `retry_for` and freezes which tasks it reports Retry.

    B9_REFERENCE_SDK=<beta9 checkout>/sdk/src python tests/golden/make_ref_retry_golden.py   (run from the repo root)

The same harness as make_ref_runner_golden.py: the unmodified `TaskQueueWorker.process_tasks`
(sdk/src/beta9/runner/taskqueue.py:297-404) pops the given `task_msg` bytes, calls the user handler and reports
TaskStatus.Retry instead of Error when `retry_on_errors(handler.parent_abstraction.retry_for, e)` holds (:352-361,
407-408). Here the handler's `parent.retry_for` is set to each exception class a device handler can raise, one at a
time, over the golden wire records (hot_path_golden.json) and the wire records of the seeded fuzz payloads
(ref_fuzz_golden.json's n_payloads / seed). Retry is reported exactly when type(e) is that class, so the class a task
raised is the one whose run answered Retry (none: it completed, or raised a class outside the six).
Output: tests/golden/ref_retry_golden.json, checked on every CPU run by tests/test_retry_on_host.py. Per handler and
class, one status letter per task (C = COMPLETE, E = ERROR, R = RETRY) in corpus order.
"""
import binascii
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from tests.golden.make_ref_runner_golden import HANDLERS, fuzz_payloads, load_reference_runner, run_reference_worker  # noqa: E402

CLASSES = {"TypeError": TypeError, "AttributeError": AttributeError, "UnicodeEncodeError": UnicodeEncodeError,
           "KeyError": KeyError, "ValueError": ValueError, "binascii.Error": binascii.Error}
LETTER = {"COMPLETE": "C", "ERROR": "E", "RETRY": "R"}


def corpus_wires(handler: str):
    """The wire records every check of this golden runs: the golden cases that became tasks, then the fuzz payloads'."""
    import base64
    from oracle.pyoracle import loop
    golden = json.load(open(os.path.join(HERE, "hot_path_golden.json")))
    wires = [base64.b64decode(c["wire"]) for cases in golden["groups"].values() for c in cases if c["wire"] is not None]
    fz = json.load(open(os.path.join(HERE, "ref_fuzz_golden.json")))
    payloads, ids = fuzz_payloads(fz["n_payloads"], fz["seed"])
    wires += [w.wire for w in loop.run_task_loop(payloads, ids, handler, keep_wire=True) if w.wire is not None]
    return wires


def main():
    rt, rc = load_reference_runner()
    import ref_handlers
    out = {"source": "reference runner loop (sdk/src/beta9/runner/taskqueue.py:297-404) with parent.retry_for = [class], "
                     "over hot_path_golden.json's wires and ref_fuzz_golden.json's fuzz payload wires", "handlers": {}}
    for h in HANDLERS:
        wires = corpus_wires(h)
        per = {}
        for name, cls in CLASSES.items():
            getattr(ref_handlers, h).parent.retry_for = [cls]
            done = run_reference_worker(rt, rc, h, wires)
            assert len(done) == len(wires), (h, name, len(done), len(wires))
            per[name] = "".join(LETTER[str(st)] for _, st, _ in done)
        getattr(ref_handlers, h).parent.retry_for = []
        out["handlers"][h] = {"n": len(wires), "status": per}
    path = os.path.join(HERE, "ref_retry_golden.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
    print(path, sum(v["n"] for v in out["handlers"].values()) * len(CLASSES), "task executions through the reference runner")


if __name__ == "__main__":
    main()
