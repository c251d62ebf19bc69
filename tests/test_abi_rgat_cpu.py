"""tfgnn_b200_rgat_bwd: the header and the Python binding agree on it, and it validates its arguments before any CUDA
call (no GPU needed)."""
import os
import re

from tf2_gnn_b200 import _ffi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_rgat_bwd_is_declared_and_bound():
    with open(os.path.join(ROOT, "include", "tfgnn_b200.h")) as f:
        text = f.read()
    m = re.search(r"TFGNN_API int tfgnn_b200_rgat_bwd\(([^;]*)\);", text)
    assert m, "tfgnn_b200_rgat_bwd is not declared"
    assert len(m.group(1).split(",")) == 16
    assert "tfgnn_b200_rgat_bwd" in _ffi.EXPORTED_SYMBOLS
    assert len(_ffi.lib().tfgnn_b200_rgat_bwd.argtypes) == 16


def _call(D=8, H=16, K=4, act=_ffi.ACT["tanh"], path=_ffi.PATH["auto"]):
    return _ffi.lib().tfgnn_b200_rgat_bwd(None, None, None, D, None, None, H, K, act, path, None, None, None, None, None,
                                          None)


def test_rgat_bwd_rejects_missing_batches():
    assert _call() == _ffi.ERR_INVALID_ARGUMENT
    assert b"NULL" in _ffi.lib().tfgnn_b200_last_error()
    assert _call(act=_ffi.ACT["gelu"], K=1) == _ffi.ERR_INVALID_ARGUMENT


def test_rgat_bwd_rejects_bad_codes_and_shapes():
    assert _call(act=99) == _ffi.ERR_INVALID_ARGUMENT
    assert _call(D=0) == _ffi.ERR_INVALID_ARGUMENT
    assert _call(H=-4) == _ffi.ERR_INVALID_ARGUMENT
    assert _call(K=0) == _ffi.ERR_INVALID_ARGUMENT
    assert _call(H=18, K=4) == _ffi.ERR_INVALID_ARGUMENT     # hidden_dim not divisible by num_heads


def test_rgat_bwd_returns_unsupported_outside_its_scope():
    """D or the per-head width not a multiple of 4, hidden_dim above 512, the atomic path: the literal path's shapes."""
    for kw in (dict(D=6), dict(H=24, K=4), dict(H=12, K=1, D=5), dict(H=528, K=4), dict(path=_ffi.PATH["atomic"])):
        assert _call(**kw) == _ffi.ERR_UNSUPPORTED, kw
        assert b"rgat_bwd" in _ffi.lib().tfgnn_b200_last_error()
