"""The C-ABI shared library loads and exports every symbol include/arroyo_b200.h declares.
No compute calls: this runs on a box without a GPU."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from arroyo_b200 import ffi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    text = open(os.path.join(ROOT, "include", "arroyo_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(arroyo_b200_\w+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    lib = ffi.load()
    declared = header_symbols()
    assert len(declared) >= 25
    bound = {name for name, _, _ in ffi.SYMBOLS}
    assert set(declared) == bound, (set(declared) ^ bound)
    for name in declared:
        assert getattr(lib, name) is not None


def test_abi_version_and_struct_layout():
    lib = ffi.load()
    assert lib.arroyo_b200_abi_version() == ffi.ABI_VERSION
    # sizes the C compiler produces for the same declarations (natural alignment)
    assert C.sizeof(ffi.ArrowArray) == 80 and C.sizeof(ffi.ArrowSchema) == 72
    assert C.sizeof(ffi.OpConfig) % 8 == 0
    assert C.sizeof(ffi.DeviceBatch) == 16 + 8 * ffi.MAX_COLS


def test_no_cpu_fallback_without_gpu():
    lib = ffi.load()
    if lib.arroyo_b200_device_count() > 0:
        pytest.skip("a CUDA device is present")
    cfg = ffi.OpConfig()
    cfg.kind = ffi.TUMBLING_AGGREGATE
    cfg.width_ns = 10**9
    cfg.n_cols = 2
    cfg.timestamp_col = 1
    cfg.n_key_cols = 1
    cfg.n_aggs = 1
    cfg.aggs[0].kind = ffi.AGG_COUNT_STAR
    h = C.c_void_p()
    err = C.create_string_buffer(256)
    st = lib.arroyo_b200_op_create(C.byref(cfg), C.byref(h), err, 256)
    assert st == ffi.FATAL and not h
    assert b"no CPU fallback" in err.value


def test_bad_config_is_rejected_before_touching_cuda():
    lib = ffi.load()
    cfg = ffi.OpConfig()
    cfg.kind = ffi.SLIDING_AGGREGATE
    cfg.width_ns = 10 * 10**9
    cfg.slide_ns = 3 * 10**9  # width not a multiple of slide
    cfg.n_cols = 2
    cfg.timestamp_col = 1
    cfg.n_aggs = 1
    cfg.aggs[0].kind = ffi.AGG_COUNT_STAR
    h = C.c_void_p()
    err = C.create_string_buffer(256)
    st = lib.arroyo_b200_op_create(C.byref(cfg), C.byref(h), err, 256)
    assert st == ffi.INVALID_ARGUMENT and b"multiple of the slide" in err.value
    cfg.kind = 99
    assert lib.arroyo_b200_op_create(C.byref(cfg), C.byref(h), err, 256) == ffi.INVALID_ARGUMENT
    cfg.kind = ffi.TUMBLING_AGGREGATE
    cfg.width_ns = 0  # instant window: outside the supported subset
    assert lib.arroyo_b200_op_create(C.byref(cfg), C.byref(h), err, 256) == ffi.UNSUPPORTED
    # a group-by key column outside the input, for each aggregating operator
    cfg.width_ns = cfg.slide_ns = cfg.gap_ns = 10 * 10**9
    cfg.n_key_cols = 1
    cfg.key_col = 2
    for kind in (ffi.TUMBLING_AGGREGATE, ffi.SESSION_AGGREGATE, ffi.UPDATING_AGGREGATE):
        cfg.kind = kind
        st = lib.arroyo_b200_op_create(C.byref(cfg), C.byref(h), err, 256)
        assert st == ffi.INVALID_ARGUMENT and b"key_col" in err.value and not h, (kind, st, err.value)


def test_bin_start_fast_division_matches_modulo():
    """K1: bin = ts - ts % width with the kernel's multiply-high division."""
    lib = ffi.load()
    rng = np.random.default_rng(7)
    widths = [2, 3, 1000, 10**6, 10**9, 2 * 10**9, 3600 * 10**9, 30 * 86400 * 10**9, 2**40, 2**40 + 1,
              999_999_937, 2**62 - 57]
    for w in widths:
        ts = np.concatenate([rng.integers(0, 2**62, 200), [0, 1, w - 1, w, w + 1, 2**63 - 1, 1_700_000_000 * 10**9]])
        for t in ts.tolist():
            assert lib.arroyo_b200_bin_start(t, w) == t - t % w, (t, w)


def test_server_for_hash_matches_reference_formula():
    """dest = (h / (u64::MAX / n)) % n  (arroyo-operator/src/lib.rs:30-41) and our routing hash equals
    the oracle's restatement."""
    from oracle import arroyo_oracle as O
    lib = ffi.load()
    rng = np.random.default_rng(3)
    keys = rng.integers(-2**63, 2**63 - 1, 500, dtype=np.int64)
    h = O.mix64(keys.view(np.uint64))
    for k, hv in zip(keys.tolist(), h.tolist()):
        assert lib.arroyo_b200_hash_key(k) == hv
    for n in (1, 2, 3, 6, 8):
        want = O.server_for_hash_array(h, n)
        for hv, w in zip(h.tolist(), want.tolist()):
            assert lib.arroyo_b200_server_for_hash(hv, n) == w
        assert lib.arroyo_b200_server_for_hash(2**64 - 1, n) == ((2**64 - 1) // ((2**64 - 1) // n)) % n
