"""TFGNN_PREPARE_TRANSPOSE_OWNED (the backward CSR of a target-range shard): the header and the Python binding agree on
it, and prepare_sharded validates its arguments with the flag set before any CUDA call."""
import ctypes
import os
import re

from tf2_gnn_b200 import _ffi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_transpose_owned_flag_matches_header():
    with open(os.path.join(ROOT, "include", "tfgnn_b200.h")) as f:
        text = f.read()
    m = re.search(r"TFGNN_PREPARE_TRANSPOSE_OWNED\s*=\s*1u\s*<<\s*(\d+)", text)
    assert m and _ffi.PREPARE_TRANSPOSE_OWNED == 1 << int(m.group(1))
    flags = (_ffi.PREPARE_VALIDATE, _ffi.PREPARE_TRANSPOSE, _ffi.PREPARE_TRANSPOSE_OWNED)
    assert len({*flags}) == 3 and all(f & (f - 1) == 0 for f in flags)


def test_transpose_owned_rejects_a_range_outside_the_graph():
    lib = _ffi.lib()
    out = ctypes.c_void_p()
    rc = lib.tfgnn_b200_prepare_sharded(None, None, 0, 10, 8, 5, _ffi.PREPARE_TRANSPOSE_OWNED, ctypes.byref(out), None)
    assert rc == _ffi.ERR_INVALID_ARGUMENT
    assert b"target range" in lib.tfgnn_b200_last_error()
    assert not out.value


def test_backward_entries_reject_missing_batches():
    lib = _ffi.lib()
    rc = lib.tfgnn_b200_rgcn_bwd(None, None, None, 4, None, 4, 0, 0, 0, None, None, None, None, None)
    assert rc == _ffi.ERR_INVALID_ARGUMENT
    rc = lib.tfgnn_b200_ggnn_bwd(None, None, None, 4, None, 4, 0, 0, None, None, None, None, None, None, None, None,
                                 None, None)
    assert rc == _ffi.ERR_INVALID_ARGUMENT
