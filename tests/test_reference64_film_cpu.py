"""The scalable float64 GNN-FiLM reference (reference64_film.py) against float64 torch autograd of the reference's literal
per-edge op order, on small graphs with empty types, isolated nodes, duplicate edges and self-loops.  CPU only."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

import reference64_film as rf  # noqa: E402
from test_reference64_cpu import close, small_graph  # noqa: E402


def _autograd(h, adjs, Ws, Fs, g, **kw):
    h64 = torch.from_numpy(h).requires_grad_()
    W64 = [torch.from_numpy(w).requires_grad_() for w in Ws]
    F64 = [torch.from_numpy(f).requires_grad_() for f in Fs]
    out = rf.film_autograd(h64, [torch.from_numpy(a) for a in adjs], W64, F64, **kw)
    out.backward(torch.from_numpy(g))
    return out.detach(), h64.grad, [w.grad for w in W64], [f.grad for f in F64]


@pytest.mark.parametrize("agg", ["sum", "mean", "sqrt_n"])
@pytest.mark.parametrize("act", [None, "relu", "tanh", "elu", "gelu"])
@pytest.mark.parametrize("normalize,use_target", [(False, False), (True, False), (False, True), (True, True)])
def test_film_reference_matches_autograd(agg, act, normalize, use_target):
    rng = np.random.default_rng(len(agg) + 7 * len(act or "") + 2 * normalize + use_target)
    V, D, H, L = 60, 12, 8, 3
    adjs = small_graph(rng, V, L)
    h = rng.uniform(-1, 1, (V, D))
    Ws = [rng.uniform(-0.5, 0.5, (2 * D if use_target else D, H)) for _ in range(L)]
    Fs = [rng.uniform(-0.5, 0.5, (D, 2 * H)) for _ in range(L)]
    g = rng.uniform(-1, 1, (V, H))
    kw = dict(agg=agg, act=act, normalize=normalize, use_target=use_target)
    got = rf.film_layer(h, adjs, Ws, Fs, g, **kw)
    out, gh, gW, gF = _autograd(h, adjs, Ws, Fs, g, **kw)
    close(got["out"], out)
    close(got["grad_h"], gh)
    assert len(got["grad_W"]) == len(got["grad_F"]) == L
    for a, b in zip(got["grad_W"], gW):
        close(a, b)
    for a, b in zip(got["grad_F"], gF):
        close(a, b)
    assert np.all(got["grad_W"][1].numpy() == 0.0) and np.all(got["grad_F"][1].numpy() == 0.0)   # the empty type
    assert np.all(got["grad_h"][V - 5:].numpy() == 0.0)                                          # isolated nodes


@pytest.mark.parametrize("use_target", [False, True])
def test_film_abs_mode_bounds_every_result(use_target):
    """absval=True dominates |out| (relu), |grad_h|, |grad_W| and |grad_F| element-wise, and partial_max covers them."""
    rng = np.random.default_rng(19)
    V, D, H, L = 80, 8, 12, 3
    adjs = small_graph(rng, V, L)
    h = rng.integers(-1, 2, (V, D)).astype(np.float64)
    Ws = [rng.integers(-1, 2, (2 * D if use_target else D, H)).astype(np.float64) for _ in range(L)]
    Fs = [rng.integers(-1, 2, (D, 2 * H)).astype(np.float64) for _ in range(L)]
    g = rng.integers(-1, 2, (V, H)).astype(np.float64)
    val = rf.film_layer(h, adjs, Ws, Fs, g, use_target=use_target)
    bnd = rf.film_layer(h, adjs, Ws, Fs, g, use_target=use_target, absval=True)
    assert np.all(np.abs(val["out"].numpy()) <= bnd["out"].numpy())
    assert np.all(np.abs(val["grad_h"].numpy()) <= bnd["grad_h"].numpy())
    for key in ("grad_W", "grad_F"):
        for a, b in zip(val[key], bnd[key]):
            assert np.all(np.abs(a.numpy()) <= b.numpy())
    tables = [bnd["out"], bnd["grad_h"], *bnd["grad_W"], *bnd["grad_F"]]
    assert bnd["partial_max"] >= max(float(t.max()) for t in tables)
    for x in [val["out"], val["grad_h"], *val["grad_W"], *val["grad_F"]]:   # integer inputs give integer results
        assert np.array_equal(x.numpy(), np.round(x.numpy()))
