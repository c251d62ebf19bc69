"""tfgnn_b200_film_bwd: the header and the Python binding agree on it, and it validates its arguments before any CUDA
call (no GPU needed)."""
import os
import re

from tf2_gnn_b200 import _ffi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_film_bwd_is_declared_and_bound():
    with open(os.path.join(ROOT, "include", "tfgnn_b200.h")) as f:
        text = f.read()
    m = re.search(r"TFGNN_API int tfgnn_b200_film_bwd\(([^;]*)\);", text)
    assert m, "tfgnn_b200_film_bwd is not declared"
    assert len(m.group(1).split(",")) == 16
    assert "tfgnn_b200_film_bwd" in _ffi.EXPORTED_SYMBOLS
    assert len(_ffi.lib().tfgnn_b200_film_bwd.argtypes) == 16


def _call(D=4, H=4, flags=0, agg=_ffi.AGG["sum"], act=_ffi.ACT["relu"]):
    return _ffi.lib().tfgnn_b200_film_bwd(None, None, None, D, None, None, H, flags, agg, act, None, None, None, None,
                                          None, None)


def test_film_bwd_rejects_missing_batches():
    assert _call() == _ffi.ERR_INVALID_ARGUMENT
    assert b"NULL" in _ffi.lib().tfgnn_b200_last_error()
    assert _call(flags=_ffi.FLAG_NORMALIZE | _ffi.FLAG_USE_TARGET, agg=_ffi.AGG["sqrt_n"]) == _ffi.ERR_INVALID_ARGUMENT


def test_film_bwd_rejects_bad_codes_and_shapes():
    assert _call(act=99) == _ffi.ERR_INVALID_ARGUMENT
    assert _call(agg=17) == _ffi.ERR_INVALID_ARGUMENT
    assert _call(D=0) == _ffi.ERR_INVALID_ARGUMENT
    assert _call(H=-4) == _ffi.ERR_INVALID_ARGUMENT


def test_film_bwd_returns_unsupported_outside_its_math():
    """Activation before aggregation, max aggregation, D or H not a multiple of 4: the literal path's configurations."""
    for kw in (dict(flags=_ffi.FLAG_ACT_BEFORE_AGG), dict(flags=_ffi.FLAG_ACT_BEFORE_AGG | _ffi.FLAG_USE_TARGET),
               dict(agg=_ffi.AGG["max"]), dict(D=6), dict(H=10)):
        assert _call(**kw) == _ffi.ERR_UNSUPPORTED, kw
        assert b"film_bwd" in _ffi.lib().tfgnn_b200_last_error()
