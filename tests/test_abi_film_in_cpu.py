"""tfgnn_b200_film_in_fwd / _bwd (GNN-FiLM with a per-type FiLM input): the header and the Python binding agree on them,
and they validate their arguments before any CUDA call (no GPU needed)."""
import os
import re

import pytest

from tf2_gnn_b200 import _ffi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("name,nargs", [("tfgnn_b200_film_in_fwd", 15), ("tfgnn_b200_film_in_bwd", 19)])
def test_film_in_entries_are_declared_and_bound(name, nargs):
    with open(os.path.join(ROOT, "include", "tfgnn_b200.h")) as f:
        text = f.read()
    m = re.search(r"TFGNN_API int " + name + r"\(([^;]*)\);", text)
    assert m, f"{name} is not declared"
    assert len(m.group(1).split(",")) == nargs
    assert name in _ffi.EXPORTED_SYMBOLS
    assert len(getattr(_ffi.lib(), name).argtypes) == nargs


def _fwd(D=4, H=4, S=8, flags=0, agg=_ffi.AGG["sum"], act=_ffi.ACT["relu"]):
    return _ffi.lib().tfgnn_b200_film_in_fwd(None, None, D, None, 0, None, S, None, H, flags, agg, act, 0, None, None)


def _bwd(D=4, H=4, S=8, flags=0, agg=_ffi.AGG["sum"], act=_ffi.ACT["relu"]):
    return _ffi.lib().tfgnn_b200_film_in_bwd(None, None, None, D, None, None, S, None, H, flags, agg, act, None, None,
                                             None, None, None, None, None)


def _last_error():
    return _ffi.lib().tfgnn_b200_last_error()


@pytest.mark.parametrize("call", [_fwd, _bwd])
def test_film_in_rejects_missing_batches(call):
    assert call() == _ffi.ERR_INVALID_ARGUMENT
    assert b"NULL" in _last_error()
    assert call(flags=_ffi.FLAG_NORMALIZE | _ffi.FLAG_USE_TARGET, agg=_ffi.AGG["sqrt_n"]) == _ffi.ERR_INVALID_ARGUMENT


def test_film_in_bwd_rejects_bad_codes_and_shapes():
    for kw in (dict(act=99), dict(agg=17), dict(D=0), dict(H=-4), dict(S=0), dict(S=-8)):
        assert _bwd(**kw) == _ffi.ERR_INVALID_ARGUMENT, kw
        assert b"film_in_bwd" in _last_error(), kw


def test_film_in_bwd_returns_unsupported_outside_its_math():
    """Activation before aggregation, max aggregation, D, H or S not a multiple of 4: the literal path's configurations."""
    for kw in (dict(flags=_ffi.FLAG_ACT_BEFORE_AGG), dict(flags=_ffi.FLAG_ACT_BEFORE_AGG | _ffi.FLAG_USE_TARGET),
               dict(agg=_ffi.AGG["max"]), dict(D=6), dict(H=10), dict(S=30)):
        assert _bwd(**kw) == _ffi.ERR_UNSUPPORTED, kw
        assert b"film_in_bwd" in _last_error(), kw
