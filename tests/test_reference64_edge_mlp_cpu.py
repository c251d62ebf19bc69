"""The scalable float64 reference of the one-hidden-layer edge MLP (reference64_edge_mlp.py) against float64 torch autograd
of the reference's literal per-edge op order, on small graphs with empty types, isolated nodes, duplicate edges,
self-loops and exact zeros in the hidden pre-activations.  CPU only."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

import reference64_edge_mlp as rm  # noqa: E402
from test_reference64_cpu import close, small_graph  # noqa: E402


def _autograd(h, adjs, Us, W2s, g, aggr=None, **kw):
    h64 = torch.from_numpy(h).requires_grad_()
    U64 = [torch.from_numpy(u).requires_grad_() for u in Us]
    W64 = [torch.from_numpy(w).requires_grad_() for w in W2s]
    M64 = [torch.from_numpy(m).requires_grad_() for m in (aggr or [])]
    out = rm.edge_mlp_autograd(h64, [torch.from_numpy(a) for a in adjs], U64, W64, aggr_ws=M64, **kw)
    out.backward(torch.from_numpy(g))
    return out.detach(), h64.grad, [u.grad for u in U64], [w.grad for w in W64], [m.grad for m in M64]


def _check(got, ref, L, n_aggr):
    out, gh, gU, gW, gM = ref
    close(got["out"], out)
    close(got["grad_h"], gh)
    assert len(got["grad_U"]) == len(got["grad_W2"]) == L and len(got["grad_aggr"]) == n_aggr
    for a, b in zip(got["grad_U"] + got["grad_W2"] + got["grad_aggr"], gU + gW + gM):
        close(a, b)


@pytest.mark.parametrize("agg", ["sum", "mean", "sqrt_n"])
@pytest.mark.parametrize("act", [None, "relu", "tanh", "leaky_relu", "elu", "selu", "gelu"])
@pytest.mark.parametrize("normalize,use_target", [(False, False), (True, False), (False, True), (True, True)])
def test_edge_mlp_reference_matches_autograd(agg, act, normalize, use_target):
    rng = np.random.default_rng(len(agg) + 7 * len(act or "") + 2 * normalize + use_target)
    V, D, H, L = 60, 12, 8, 3
    adjs = small_graph(rng, V, L)
    h = rng.uniform(-1, 1, (V, D))
    Us = [rng.uniform(-0.5, 0.5, (2 * D if use_target else D, H)) for _ in range(L)]
    W2s = [rng.uniform(-0.5, 0.5, (H, H)) for _ in range(L)]
    g = rng.uniform(-1, 1, (V, H))
    kw = dict(agg=agg, act=act, normalize=normalize, use_target=use_target)
    got = rm.edge_mlp_layer(h, adjs, Us, W2s, g, chunk=7, **kw)   # chunks smaller than most types
    _check(got, _autograd(h, adjs, Us, W2s, g, **kw), L, 0)
    assert np.all(got["grad_U"][1].numpy() == 0.0) and np.all(got["grad_W2"][1].numpy() == 0.0)   # the empty type
    assert np.all(got["grad_h"][V - 5:].numpy() == 0.0)                                            # isolated nodes


@pytest.mark.parametrize("n_aggr", [1, 2, 3])   # 0, 1 and 2 hidden layers in the aggregation MLP
@pytest.mark.parametrize("act", ["relu", "tanh", "gelu"])
def test_rgin_reference_with_aggregation_mlp_matches_autograd(n_aggr, act):
    rng = np.random.default_rng(11 * n_aggr + len(act))
    V, D, H, L = 50, 8, 12, 3
    adjs = small_graph(rng, V, L)
    h = rng.uniform(-1, 1, (V, D))
    Us = [rng.uniform(-0.5, 0.5, (D, H)) for _ in range(L)]
    W2s = [rng.uniform(-0.5, 0.5, (H, H)) for _ in range(L)]
    Ms = [rng.uniform(-0.5, 0.5, (H, H)) for _ in range(n_aggr)]
    g = rng.uniform(-1, 1, (V, H))
    got = rm.edge_mlp_layer(h, adjs, Us, W2s, g, act=act, aggr_ws=Ms, chunk=16)
    _check(got, _autograd(h, adjs, Us, W2s, g, aggr=Ms, act=act), L, n_aggr)


@pytest.mark.parametrize("use_target", [False, True])
def test_relu_mask_at_exact_zero_is_zero(use_target):
    """Integer inputs put many hidden pre-activations exactly at 0; both the reference and autograd take derivative 0
    there (TF's ReluGrad), and min_abs_P reports the zeros."""
    rng = np.random.default_rng(3 + use_target)
    V, D, H, L = 40, 6, 8, 2
    adjs = small_graph(rng, V, L)
    h = rng.integers(-1, 2, (V, D)).astype(np.float64)
    Us = [rng.integers(-1, 2, (2 * D if use_target else D, H)).astype(np.float64) for _ in range(L)]
    W2s = [rng.uniform(-1, 1, (H, H)) for _ in range(L)]
    g = rng.uniform(-1, 1, (V, H))
    got = rm.edge_mlp_layer(h, adjs, Us, W2s, g, act="tanh", use_target=use_target)
    assert got["min_abs_P"] == 0.0
    _check(got, _autograd(h, adjs, Us, W2s, g, act="tanh", use_target=use_target), L, 0)


@pytest.mark.parametrize("use_target,n_aggr", [(False, 0), (True, 0), (False, 2)])
def test_edge_mlp_abs_mode_bounds_every_result(use_target, n_aggr):
    """absval=True dominates |out| (relu), |grad_h| and every weight gradient element-wise, partial_max covers them, and
    operand_max covers the inputs."""
    rng = np.random.default_rng(19 + n_aggr)
    V, D, H, L = 80, 8, 12, 3
    adjs = small_graph(rng, V, L)
    ints = lambda shape: rng.integers(-1, 2, shape).astype(np.float64)
    h, g = ints((V, D)), ints((V, H))
    Us = [ints((2 * D if use_target else D, H)) for _ in range(L)]
    W2s = [ints((H, H)) for _ in range(L)]
    Ms = [ints((H, H)) for _ in range(n_aggr)]
    val = rm.edge_mlp_layer(h, adjs, Us, W2s, g, use_target=use_target, aggr_ws=Ms)
    bnd = rm.edge_mlp_layer(h, adjs, Us, W2s, g, use_target=use_target, aggr_ws=Ms, absval=True)
    assert np.all(np.abs(val["out"].numpy()) <= bnd["out"].numpy())
    assert np.all(np.abs(val["grad_h"].numpy()) <= bnd["grad_h"].numpy())
    for key in ("grad_U", "grad_W2", "grad_aggr"):
        for a, b in zip(val[key], bnd[key]):
            assert np.all(np.abs(a.numpy()) <= b.numpy())
    tables = [bnd["out"], bnd["grad_h"], *bnd["grad_U"], *bnd["grad_W2"], *bnd["grad_aggr"]]
    assert bnd["partial_max"] >= max(float(t.max()) for t in tables)
    assert bnd["operand_max"] >= 1.0
    for x in [val["out"], val["grad_h"], *val["grad_U"], *val["grad_W2"], *val["grad_aggr"]]:   # integers stay integers
        assert np.array_equal(x.numpy(), np.round(x.numpy()))
