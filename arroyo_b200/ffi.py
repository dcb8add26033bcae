"""ctypes binding of libarroyo_b200.so (include/arroyo_b200.h).

This is the Python twin of the `extern "C"` block a Rust shim would declare (INTEGRATION.md).
There is no fallback: if the library is missing, importing raises."""
import ctypes as C
import os

from . import build as _build

ABI_VERSION = 2  # 2: OpConfig gained `frame` at its end
MAX_AGGS = 8
MAX_COLS = 16

OK, INVALID_ARGUMENT, UNSUPPORTED, RUNTIME, FATAL, PANIC = 0, 1, 2, 3, 4, 5
TUMBLING_AGGREGATE, SLIDING_AGGREGATE, SESSION_AGGREGATE, INSTANT_JOIN, UPDATING_AGGREGATE, TTL_JOIN = 1, 2, 3, 4, 5, 6
INSTANT_AGGREGATE = 7
WINDOW_FUNCTION = 8
FN_ROW_NUMBER, FN_RANK, FN_DENSE_RANK, FN_AGGREGATE = 1, 2, 3, 4
FN_LAG, FN_LEAD, FN_FIRST_VALUE, FN_LAST_VALUE, FN_NTH_VALUE, FN_PERCENT_RANK, FN_CUME_DIST = 5, 6, 7, 8, 9, 10, 11
ORDER_ASC, ORDER_DESC = 16, 17
FN_ARGUMENT = 18
FRAME_DEFAULT, FRAME_ROWS, FRAME_RANGE, FRAME_GROUPS = 0, 1, 2, 3
BOUND_UNBOUNDED_PRECEDING, BOUND_PRECEDING, BOUND_CURRENT_ROW, BOUND_FOLLOWING, BOUND_UNBOUNDED_FOLLOWING = 1, 2, 3, 4, 5
MAX_ORDER_KEYS = 4
AGG_COUNT_STAR, AGG_SUM_I64, AGG_AVG_I64, AGG_MIN_I64, AGG_MAX_I64 = 1, 2, 3, 4, 5
JOIN_INNER, JOIN_LEFT, JOIN_RIGHT, JOIN_FULL = 0, 1, 2, 3
FLAG_PROFILE, FLAG_REMERGE_ONLY, FLAG_COMBINE, FLAG_AVG_F64, FLAG_NO_COMBINE, FLAG_ZERO_COPY = 1, 2, 4, 8, 16, 32
FLAG_NO_DIRECT = 64  # accepted and ignored since round 2
FLAG_NO_TWO_PASS = 128
FLAG_TWO_PASS_ALWAYS = 256
FLAG_UPDATING_INPUT = 512
FLAG_FN_DEFAULT = 1024
NO_WATERMARK = -(1 << 63)
INT64_MIN = -(1 << 63)
INT64_MAX = (1 << 63) - 1


class ArrowSchema(C.Structure):
    pass


class ArrowArray(C.Structure):
    pass


ArrowSchema._fields_ = [
    ("format", C.c_char_p), ("name", C.c_char_p), ("metadata", C.c_char_p), ("flags", C.c_int64),
    ("n_children", C.c_int64), ("children", C.POINTER(C.POINTER(ArrowSchema))),
    ("dictionary", C.POINTER(ArrowSchema)), ("release", C.c_void_p), ("private_data", C.c_void_p),
]
ArrowArray._fields_ = [
    ("length", C.c_int64), ("null_count", C.c_int64), ("offset", C.c_int64), ("n_buffers", C.c_int64),
    ("n_children", C.c_int64), ("buffers", C.POINTER(C.c_void_p)),
    ("children", C.POINTER(C.POINTER(ArrowArray))), ("dictionary", C.POINTER(ArrowArray)),
    ("release", C.c_void_p), ("private_data", C.c_void_p),
]


class Agg(C.Structure):
    _fields_ = [("kind", C.c_int32), ("input_col", C.c_int32)]


class WindowFrame(C.Structure):
    _fields_ = [("units", C.c_int32), ("start_kind", C.c_int32), ("end_kind", C.c_int32), ("pad", C.c_int32),
                ("start_offset", C.c_int64), ("end_offset", C.c_int64)]


class OpConfig(C.Structure):
    _fields_ = [
        ("kind", C.c_int32), ("device", C.c_int32), ("stream", C.c_uint64),
        ("task_index", C.c_uint32), ("parallelism", C.c_uint32),
        ("width_ns", C.c_int64), ("slide_ns", C.c_int64), ("gap_ns", C.c_int64),
        ("n_cols", C.c_int32), ("timestamp_col", C.c_int32), ("n_key_cols", C.c_int32), ("key_col", C.c_int32),
        ("n_aggs", C.c_int32), ("aggs", Agg * MAX_AGGS),
        ("final_projection", C.c_int32), ("window_index", C.c_int32),
        ("join_type", C.c_int32), ("right_n_cols", C.c_int32), ("right_timestamp_col", C.c_int32),
        ("left_key_col", C.c_int32), ("right_key_col", C.c_int32),
        ("left_n_routing", C.c_int32), ("right_n_routing", C.c_int32),
        ("partial_count_col_plus1", C.c_int32), ("window_fn", C.c_int32),
        ("expected_keys", C.c_uint64), ("flags", C.c_uint32), ("reserved", C.c_uint32),
        ("frame", WindowFrame),
    ]


class Batches(C.Structure):
    _fields_ = [("n_batches", C.c_int64), ("arrays", C.POINTER(ArrowArray)), ("schemas", C.POINTER(ArrowSchema)),
                ("private_data", C.c_void_p)]


class DeviceBatch(C.Structure):
    _fields_ = [("n_rows", C.c_int64), ("n_cols", C.c_int32), ("reserved", C.c_int32),
                ("cols", C.c_uint64 * MAX_COLS)]


class Stats(C.Structure):
    _fields_ = [
        ("rows_in", C.c_uint64), ("rows_late", C.c_uint64), ("rows_deferred", C.c_uint64), ("rows_out", C.c_uint64),
        ("windows_out", C.c_uint64), ("n_keys", C.c_uint64), ("kernel_launches", C.c_uint64),
        ("ingest_launches", C.c_uint64), ("emit_launches", C.c_uint64), ("h2d_bytes", C.c_uint64),
        ("d2h_bytes", C.c_uint64), ("ingest_ms", C.c_double), ("emit_ms", C.c_double),
        ("ingest_rows_timed", C.c_uint64), ("emit_rows_timed", C.c_uint64),
        ("host_process_ms", C.c_double), ("host_watermark_ms", C.c_double),
    ]

    def as_dict(self):
        return {f: getattr(self, f) for f, _ in self._fields_}


# every symbol include/arroyo_b200.h declares: (name, restype, argtypes)
_VP = C.c_void_p
SYMBOLS = [
    ("arroyo_b200_abi_version", C.c_int32, []),
    ("arroyo_b200_device_count", C.c_int32, []),
    ("arroyo_b200_host_alloc", _VP, [C.c_uint64]),
    ("arroyo_b200_host_free", None, [_VP]),
    ("arroyo_b200_op_create", C.c_int32, [C.POINTER(OpConfig), C.POINTER(_VP), C.c_char_p, C.c_uint64]),
    ("arroyo_b200_op_destroy", None, [_VP]),
    ("arroyo_b200_op_last_error", C.c_char_p, [_VP]),
    ("arroyo_b200_op_name", C.c_char_p, [_VP]),
    ("arroyo_b200_op_on_start", C.c_int32, [_VP, C.POINTER(ArrowArray), C.POINTER(ArrowSchema), C.c_int64,
                                            C.c_int64, C.c_int64]),
    ("arroyo_b200_op_process_batch", C.c_int32, [_VP, C.c_uint32, C.c_uint32, C.POINTER(ArrowArray),
                                                 C.POINTER(ArrowSchema)]),
    ("arroyo_b200_op_process_device_batch", C.c_int32, [_VP, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint64),
                                                        C.c_int32, C.c_int64]),
    ("arroyo_b200_op_process_device_batches", C.c_int32, [_VP, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint64),
                                                          C.c_int32, C.POINTER(C.c_int64), C.c_int64]),
    ("arroyo_b200_op_handle_watermark", C.c_int32, [_VP, C.c_int64, C.POINTER(Batches)]),
    ("arroyo_b200_op_handle_watermark_begin", C.c_int32, [_VP, C.c_int64]),
    ("arroyo_b200_op_handle_watermark_poll", C.c_int32, [_VP, C.c_int32, C.POINTER(Batches), C.POINTER(C.c_int32)]),
    ("arroyo_b200_op_run_batches", C.c_int32, [_VP, C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64), C.c_int32,
                                               C.POINTER(Batches), C.POINTER(C.c_int64)]),
    ("arroyo_b200_op_handle_watermark_device", C.c_int32, [_VP, C.c_int64, C.POINTER(DeviceBatch), C.c_int64,
                                                           C.POINTER(C.c_int64)]),
    ("arroyo_b200_op_handle_watermark_device_begin", C.c_int32, [_VP, C.c_int64]),
    ("arroyo_b200_op_handle_watermark_device_poll", C.c_int32, [_VP, C.POINTER(DeviceBatch), C.c_int64,
                                                                C.POINTER(C.c_int64)]),
    ("arroyo_b200_op_handle_checkpoint", C.c_int32, [_VP, C.c_int64, C.POINTER(Batches)]),
    ("arroyo_b200_op_checkpoint_state", C.c_int32, [_VP, C.POINTER(Batches)]),
    ("arroyo_b200_op_set_clock", C.c_int32, [_VP, C.c_int64]),
    ("arroyo_b200_op_on_close", C.c_int32, [_VP, C.c_int32, C.POINTER(Batches)]),
    ("arroyo_b200_op_handle_tick", C.c_int32, [_VP, C.POINTER(Batches)]),
    ("arroyo_b200_op_process_batch_emit", C.c_int32, [_VP, C.c_uint32, C.c_uint32, C.POINTER(ArrowArray), C.POINTER(ArrowSchema),
                                                      C.POINTER(Batches)]),
    ("arroyo_b200_op_restore_side", C.c_int32, [_VP, C.c_uint32, C.POINTER(ArrowArray), C.POINTER(ArrowSchema),
                                                C.c_int64]),
    ("arroyo_b200_op_flush", C.c_int32, [_VP]),
    ("arroyo_b200_op_submit", C.c_int32, [_VP]),
    ("arroyo_b200_release_batches", None, [C.POINTER(Batches)]),
    ("arroyo_b200_op_stats", C.c_int32, [_VP, C.POINTER(Stats)]),
    ("arroyo_b200_partitioner_create", C.c_int32, [C.c_int32, C.c_uint64, C.c_int32, C.c_int32, C.c_int32,
                                                   C.c_int64, C.POINTER(_VP)]),
    ("arroyo_b200_partitioner_destroy", None, [_VP]),
    ("arroyo_b200_partition", C.c_int32, [_VP, C.POINTER(C.c_uint64), C.c_int64, C.POINTER(C.c_uint64),
                                          C.c_uint64, C.c_uint64]),
    ("arroyo_b200_partition_packed", C.c_int32, [_VP, C.POINTER(C.c_uint64), C.c_int64, C.c_uint64, C.c_uint64,
                                                 C.c_uint64]),
    ("arroyo_b200_ts_minmax", C.c_int32, [C.c_int32, C.c_uint64, C.c_uint64, C.c_int64, C.POINTER(C.c_int64),
                                          C.POINTER(C.c_int64)]),
    ("arroyo_b200_hash_key", C.c_uint64, [C.c_int64]),
    ("arroyo_b200_server_for_hash", C.c_uint32, [C.c_uint64, C.c_uint32]),
    ("arroyo_b200_bin_start", C.c_int64, [C.c_int64, C.c_int64]),
    ("arroyo_b200_plan_sliding", C.c_int64, [C.c_int64, C.c_int64, C.POINTER(C.c_int64), C.c_int64,
                                             C.POINTER(C.c_int64), C.c_int64]),
    ("arroyo_b200_plan_tumbling", C.c_int64, [C.c_int64, C.POINTER(C.c_int64), C.c_int64, C.POINTER(C.c_int64),
                                              C.c_int64]),
]

_lib = None


def lib_path() -> str:
    return _build.LIB


def load():
    """Loads (never builds) the shared library; raises if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if not os.path.exists(path):
        raise ImportError(
            f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(arroyo_b200 has no CPU fallback)")
    lib = C.CDLL(path)
    for name, res, args in SYMBOLS:
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    v = lib.arroyo_b200_abi_version()
    if v != ABI_VERSION:
        raise ImportError(f"libarroyo_b200 ABI {v} != binding {ABI_VERSION}")
    _lib = lib
    return lib


class ArroyoB200Error(RuntimeError):
    def __init__(self, status: int, message: str):
        super().__init__(f"[status {status}] {message}")
        self.status = status
        self.message = message


class UnsupportedPlan(ArroyoB200Error):
    """The plan is outside the supported subset: fall through to the stock operator."""
