"""tfgnn_b200_gru_update_fwd / tfgnn_b200_gru_update_bwd (GGNN's node update on its own): the header and the Python binding
agree on them, and both validate their arguments before any CUDA call (no GPU needed)."""
import os
import re

import pytest

from tf2_gnn_b200 import _ffi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 16   # a non-NULL stand-in address: every call below fails its checks before it could be dereferenced


@pytest.mark.parametrize("name,nargs", [("tfgnn_b200_gru_update_fwd", 10), ("tfgnn_b200_gru_update_bwd", 14)])
def test_gru_update_entries_are_declared_and_bound(name, nargs):
    with open(os.path.join(ROOT, "include", "tfgnn_b200.h")) as f:
        text = f.read()
    m = re.search(r"TFGNN_API int " + name + r"\(([^;]*)\);", text)
    assert m, f"{name} is not declared"
    assert len(m.group(1).split(",")) == nargs
    assert name in _ffi.EXPORTED_SYMBOLS
    assert len(getattr(_ffi.lib(), name).argtypes) == nargs


def _fwd(rows=8, H=8, path=_ffi.PATH["auto"], agg=P, h=P, out=P, k=P):
    return _ffi.lib().tfgnn_b200_gru_update_fwd(agg, h, rows, H, k, P, P, path, out, None)


def _bwd(rows=8, H=8, agg=P, h=P, g=P, gk=P):
    return _ffi.lib().tfgnn_b200_gru_update_bwd(agg, h, rows, H, P, P, P, g, P, P, gk, P, P, None)


def test_gru_update_fwd_rejects_bad_arguments():
    for kw in (dict(rows=-1), dict(H=0), dict(H=-8), dict(path=7), dict(path=-1), dict(agg=None), dict(h=None),
               dict(out=None), dict(k=None)):
        assert _fwd(**kw) == _ffi.ERR_INVALID_ARGUMENT, kw
    assert _fwd(path=_ffi.PATH["atomic"]) == _ffi.ERR_UNSUPPORTED
    assert _fwd(rows=0) == _ffi.OK   # nothing to update


def test_gru_update_bwd_rejects_bad_arguments():
    for kw in (dict(rows=-1), dict(H=0), dict(agg=None), dict(h=None), dict(g=None), dict(gk=None)):
        assert _bwd(**kw) == _ffi.ERR_INVALID_ARGUMENT, kw
    assert b"NULL" in _ffi.lib().tfgnn_b200_last_error()


def test_gru_update_bwd_returns_unsupported_for_odd_widths():
    """hidden_dim % 4 != 0: GGNN trains that update through the per-op GRU cell instead."""
    for H in (30, 6, 1):
        assert _bwd(H=H) == _ffi.ERR_UNSUPPORTED
        assert b"gru_update_bwd" in _ffi.lib().tfgnn_b200_last_error()
