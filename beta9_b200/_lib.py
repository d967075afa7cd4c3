"""ctypes binding of libb9gpu.so (include/b9gpu.h). No fallback: if the library is missing or no
CUDA device is visible, the calls raise."""
from __future__ import annotations

import ctypes as C
import os

PKG = os.path.dirname(os.path.abspath(__file__))
SO = os.environ.get("B9GPU_LIB") or os.path.join(PKG, "libb9gpu.so")     # B9GPU_LIB: an alternative build, for A/B timing

B9_OK, B9_EINVAL, B9_ENOMEM, B9_ENOSPC, B9_E2BIG, B9_EIO, B9_ENODEV, B9_ENOSYS, B9_ENOENT = 0, -22, -12, -28, -7, -5, -19, -38, -2
H_IDENTITY, H_CRC32, H_VADD_F32, H_JSON_SUM = 0, 1, 2, 3
ST_COMPLETE, ST_ERROR, ST_RETRY, ST_REJECTED, ST_UNSUPPORTED = 0, 1, 2, 3, 4
TF_CANCELLED = 0x01
TF_HTTP_BODY, TF_PICKLE, TF_TASK_MSG = 0x02, 0x04, 0x08


class Opts(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("device", C.c_int32), ("ring_bytes", C.c_uint64),
                ("ring_tasks", C.c_uint32), ("max_drain_tasks", C.c_uint32), ("max_result_bytes", C.c_uint64),
                ("max_task_bytes", C.c_uint32), ("flags", C.c_uint32)]


class PushMeta(C.Structure):
    _fields_ = [("timestamp_unix", C.c_void_p), ("expires_unix_ns", C.c_void_p),
                ("retries", C.c_void_p), ("flags", C.c_void_p)]


class Results(C.Structure):
    _fields_ = [("task_ids", C.c_void_p), ("status", C.c_void_p), ("has_result", C.c_void_p),
                ("offsets", C.c_void_p), ("lengths", C.c_void_p), ("payload", C.c_void_p), ("cap_tasks", C.c_uint32),
                ("cap_bytes", C.c_uint64), ("n_results", C.c_uint32), ("n_popped", C.c_uint32),
                ("n_bytes", C.c_uint64), ("need_bytes", C.c_uint64), ("task_duration", C.c_float), ("reserved_", C.c_uint32)]


class Stats(C.Structure):
    _fields_ = [("tasks_pushed", C.c_uint64), ("tasks_drained", C.c_uint64), ("bytes_h2d", C.c_uint64),
                ("bytes_d2h", C.c_uint64), ("kernel_launches", C.c_uint64), ("drains", C.c_uint64),
                ("last_push_h2d_ms", C.c_float), ("last_drain_kernel_ms", C.c_float),
                ("last_drain_d2h_ms", C.c_float), ("last_drain_tiles", C.c_uint32), ("sm_count", C.c_uint32),
                ("last_drain_in_bytes", C.c_uint64), ("last_drain_out_bytes", C.c_uint64)]


class SinkRecord(C.Structure):
    _fields_ = [("task_id", C.c_void_p), ("data", C.c_void_p), ("length", C.c_uint32), ("index", C.c_uint32),
                ("status", C.c_uint8), ("has_result", C.c_uint8)]


class WireEnv(C.Structure):
    _fields_ = [("workspace_name", C.c_char_p), ("stub_id", C.c_char_p), ("executor", C.c_char_p),
                ("max_retries", C.c_uint32), ("timeout", C.c_int32), ("ttl", C.c_uint32)]


class RebalanceInfo(C.Structure):
    _fields_ = [("world", C.c_uint32), ("rank", C.c_uint32), ("tasks_before", C.c_uint64), ("bytes_before", C.c_uint64),
                ("tasks_sent", C.c_uint64), ("bytes_sent", C.c_uint64), ("tasks_received", C.c_uint64),
                ("bytes_received", C.c_uint64), ("tasks_after", C.c_uint64), ("bytes_after", C.c_uint64)]


# every symbol include/b9gpu.h declares: (restype, argtypes)
SYMBOLS = {
    "b9_abi_version": (C.c_uint32, []),
    "b9_device_count": (C.c_int, []),
    "b9_ctx_create": (C.c_int, [C.POINTER(Opts), C.POINTER(C.c_void_p)]),
    "b9_ctx_destroy": (None, [C.c_void_p]),
    "b9_last_error": (C.c_char_p, [C.c_void_p]),
    "b9_handler_name": (C.c_char_p, [C.c_int]),
    "b9_handler_id": (C.c_int, [C.c_char_p]),
    "b9_host_alloc": (C.c_void_p, [C.c_void_p, C.c_uint64]),
    "b9_host_free": (None, [C.c_void_p, C.c_void_p]),
    "b9_batch_push": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(PushMeta)]),
    "b9_batch_push_async": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(PushMeta)]),
    "b9_batch_push_v": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(PushMeta)]),
    "b9_submit": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint8]),
    "b9_flush": (C.c_int64, [C.c_void_p]),
    "b9_buffered": (C.c_uint64, [C.c_void_p]),
    "b9_depth": (C.c_uint64, [C.c_void_p]),
    "b9_running": (C.c_uint64, [C.c_void_p]),
    "b9_depth_bytes": (C.c_uint64, [C.c_void_p]),
    "b9_expire": (C.c_int64, [C.c_void_p, C.c_int64]),
    "b9_drain": (C.c_int64, [C.c_void_p, C.c_int, C.c_uint32, C.POINTER(Results)]),
    "b9_drain_launch": (C.c_int64, [C.c_void_p, C.c_int, C.c_uint32, C.c_int]),
    "b9_drain_fetch": (C.c_int64, [C.c_void_p, C.POINTER(Results)]),
    "b9_wire_encode": (C.c_int64, [C.c_void_p, C.POINTER(WireEnv), C.c_uint32]),
    "b9_comm_unique_id": (C.c_int, [C.c_void_p]),
    "b9_comm_init": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int]),
    "b9_rebalance": (C.c_int, [C.c_void_p, C.POINTER(RebalanceInfo)]),
    "b9_rebalance_plan": (C.c_int, [C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]),
    "b9_sink_object_bytes": (C.c_uint64, [C.c_uint32, C.c_uint64]),
    "b9_sink_pack": (C.c_int64, [C.POINTER(Results), C.c_void_p, C.c_uint64]),
    "b9_drain_fetch_object": (C.c_int64, [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]),
    "b9_sink_get": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint32, C.POINTER(SinkRecord)]),
    "b9_sink_find": (C.c_int, [C.c_void_p, C.c_uint64, C.c_void_p, C.POINTER(SinkRecord)]),
    "b9_sink_result_json": (C.c_int64, [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64]),
    "b9_stats_get": (C.c_int, [C.c_void_p, C.POINTER(Stats)]),
    "b9_sync": (C.c_int, [C.c_void_p]),
    "b9_task_queue_scale": (C.c_int, [C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.POINTER(C.c_int)]),
}

_lib = None


class B9Error(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"b9gpu error {code}: {msg}")
        self.code = code


def load() -> C.CDLL:
    """dlopen libb9gpu.so and bind every declared symbol. Raises if the library is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(SO):
        raise B9Error(B9_ENODEV, f"{SO} is not built — run `python -m beta9_b200.build` (there is no CPU fallback)")
    lib = C.CDLL(SO)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)      # AttributeError if the .so does not export it
        fn.restype = res
        fn.argtypes = args
    if lib.b9_abi_version() != 2:
        raise B9Error(B9_EINVAL, "ABI version mismatch")
    _lib = lib
    return lib


def last_error(ctx=None) -> str:
    s = load().b9_last_error(ctx)
    return s.decode("utf-8", "replace") if s else ""
