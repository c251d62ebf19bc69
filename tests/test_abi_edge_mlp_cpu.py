"""tfgnn_b200_edge_mlp_bwd: the header and the Python binding agree on it, and it validates its arguments before any CUDA
call (no GPU needed)."""
import os
import re

from tf2_gnn_b200 import _ffi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_edge_mlp_bwd_is_declared_and_bound():
    with open(os.path.join(ROOT, "include", "tfgnn_b200.h")) as f:
        text = f.read()
    m = re.search(r"TFGNN_API int tfgnn_b200_edge_mlp_bwd\(([^;]*)\);", text)
    assert m, "tfgnn_b200_edge_mlp_bwd is not declared"
    assert len(m.group(1).split(",")) == 15
    assert "tfgnn_b200_edge_mlp_bwd" in _ffi.EXPORTED_SYMBOLS
    assert len(_ffi.lib().tfgnn_b200_edge_mlp_bwd.argtypes) == 15


def _call(D=4, H=4, n_hidden=1, flags=0, agg=_ffi.AGG["sum"], act=_ffi.ACT["relu"]):
    return _ffi.lib().tfgnn_b200_edge_mlp_bwd(None, None, None, D, None, n_hidden, H, flags, agg, act, None, None, None,
                                              None, None)


def test_edge_mlp_bwd_rejects_missing_batches():
    assert _call() == _ffi.ERR_INVALID_ARGUMENT
    assert b"NULL" in _ffi.lib().tfgnn_b200_last_error()
    assert _call(flags=_ffi.FLAG_NORMALIZE | _ffi.FLAG_USE_TARGET, agg=_ffi.AGG["sqrt_n"]) == _ffi.ERR_INVALID_ARGUMENT


def test_edge_mlp_bwd_rejects_bad_codes_and_shapes():
    assert _call(act=99) == _ffi.ERR_INVALID_ARGUMENT
    assert _call(agg=17) == _ffi.ERR_INVALID_ARGUMENT
    assert _call(D=0) == _ffi.ERR_INVALID_ARGUMENT
    assert _call(H=-4) == _ffi.ERR_INVALID_ARGUMENT
    assert _call(n_hidden=-1) == _ffi.ERR_INVALID_ARGUMENT


def test_edge_mlp_bwd_returns_unsupported_outside_its_math():
    """0 or 2 hidden layers, activation before aggregation, max aggregation, D or H not a multiple of 4: the other fused
    backward's and the literal path's configurations."""
    for kw in (dict(n_hidden=0), dict(n_hidden=2), dict(flags=_ffi.FLAG_ACT_BEFORE_AGG),
               dict(flags=_ffi.FLAG_ACT_BEFORE_AGG | _ffi.FLAG_USE_TARGET), dict(agg=_ffi.AGG["max"]), dict(D=6),
               dict(H=6)):
        assert _call(**kw) == _ffi.ERR_UNSUPPORTED, kw
        assert b"edge_mlp_bwd" in _ffi.lib().tfgnn_b200_last_error()
