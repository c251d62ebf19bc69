"""The scalable float64 reference (reference64.py) against the float64 autograd restatements of test_gpu_parity.py on
small graphs with empty types, isolated nodes, duplicate edges and self-loops.  CPU only."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

import reference64 as r64  # noqa: E402
from test_gpu_parity import _torch_reference_ggnn, _torch_reference_layer  # noqa: E402

BAR = 1e-12


def small_graph(rng, V, L):
    adjs = []
    for l in range(L):
        if l == 1:
            adjs.append(np.zeros((0, 2), np.int32))        # empty type
            continue
        a = rng.integers(0, V - 5, size=(4 * V, 2)).astype(np.int32)   # the last 5 nodes are isolated
        a[:6] = a[0]                                       # duplicate edges
        a[6:12, 1] = a[6:12, 0]                            # self-loops
        a[12:40, 1] = 3                                    # a small hub target
        a[40:70, 0] = 7                                    # a small hub source
        adjs.append(a)
    return adjs


def close(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape
    scale = max(np.abs(ref).max() if ref.size else 0.0, 1e-30)
    err = np.abs(got - ref).max() if ref.size else 0.0
    assert err <= BAR * scale, f"{err:.3e} > {BAR:g} * {scale:.3e}"


@pytest.mark.parametrize("agg", ["sum", "mean", "sqrt_n"])
@pytest.mark.parametrize("act", ["relu", "tanh", "leaky_relu", "elu", "selu", "gelu"])
@pytest.mark.parametrize("normalize,use_target", [(False, False), (True, False), (False, True), (True, True)])
def test_rgcn_reference_matches_autograd(agg, act, normalize, use_target):
    rng = np.random.default_rng(len(agg) + 7 * len(act) + 2 * normalize + use_target)
    V, D, H, L = 60, 12, 8, 3
    adjs = small_graph(rng, V, L)
    h = rng.uniform(-1, 1, (V, D))
    Ws = [rng.uniform(-0.5, 0.5, (2 * D if use_target else D, H)) for _ in range(L)]
    g = rng.uniform(-1, 1, (V, H))
    got = r64.rgcn_layer(h, adjs, Ws, g, agg=agg, act=act, normalize=normalize, use_target=use_target)
    h64 = torch.from_numpy(h).requires_grad_()
    W64 = [torch.from_numpy(w).requires_grad_() for w in Ws]
    ref = _torch_reference_layer(h64, [torch.from_numpy(a) for a in adjs], W64, normalize, agg, act, use_target)
    ref.backward(torch.from_numpy(g))
    close(got["out"], ref.detach())
    close(got["grad_h"], h64.grad)
    assert len(got["grad_W"]) == L
    for gw, w in zip(got["grad_W"], W64):
        close(gw, w.grad)
    assert np.all(got["grad_W"][1].numpy() == 0.0)              # the empty type
    assert np.all(got["grad_h"][V - 5:].numpy() == 0.0)          # isolated nodes get nothing


@pytest.mark.parametrize("agg,normalize", [("sum", True), ("mean", False), ("sqrt_n", True), ("sum", False)])
def test_ggnn_reference_matches_autograd(agg, normalize):
    rng = np.random.default_rng(3 + len(agg) + normalize)
    V, H, L = 50, 8, 3
    adjs = small_graph(rng, V, L)
    h = rng.uniform(-1, 1, (V, H))
    Ws = [rng.uniform(-0.5, 0.5, (H, H)) for _ in range(L)]
    K, U = rng.uniform(-0.5, 0.5, (H, 3 * H)), rng.uniform(-0.5, 0.5, (H, 3 * H))
    b = rng.uniform(-0.2, 0.2, (2, 3 * H))
    g = rng.uniform(-1, 1, (V, H))
    got = r64.ggnn_layer(h, adjs, Ws, K, U, b, g, agg=agg, normalize=normalize)
    h64 = torch.from_numpy(h).requires_grad_()
    W64 = [torch.from_numpy(w).requires_grad_() for w in Ws]
    K64, U64, b64 = (torch.from_numpy(x).requires_grad_() for x in (K, U, b))
    ref = _torch_reference_ggnn(h64, [torch.from_numpy(a) for a in adjs], W64, K64, U64, b64, normalize, agg)
    ref.backward(torch.from_numpy(g))
    close(got["out"], ref.detach())
    close(got["grad_h"], h64.grad)
    close(got["grad_K"], K64.grad)
    close(got["grad_U"], U64.grad)
    close(got["grad_b"], b64.grad)
    for gw, w in zip(got["grad_W"], W64):
        close(gw, w.grad)


@pytest.mark.parametrize("use_target", [False, True])
def test_abs_mode_bounds_every_result(use_target):
    """absval=True dominates |out| (relu), |grad_h| and |grad_W| element-wise: the premise of the exact-arithmetic bounds."""
    rng = np.random.default_rng(9)
    V, D, H, L = 80, 8, 12, 3
    adjs = small_graph(rng, V, L)
    h = rng.integers(-1, 2, (V, D)).astype(np.float64)
    Ws = [rng.integers(-1, 2, (2 * D if use_target else D, H)).astype(np.float64) for _ in range(L)]
    g = rng.integers(-1, 2, (V, H)).astype(np.float64)
    val = r64.rgcn_layer(h, adjs, Ws, g, use_target=use_target)
    bnd = r64.rgcn_layer(h, adjs, Ws, g, use_target=use_target, absval=True)
    assert np.all(np.abs(val["out"].numpy()) <= bnd["out"].numpy())
    assert np.all(np.abs(val["grad_h"].numpy()) <= bnd["grad_h"].numpy())
    for a, b in zip(val["grad_W"], bnd["grad_W"]):
        assert np.all(np.abs(a.numpy()) <= b.numpy())
    assert val["max_abs_A"] <= bnd["max_abs_A"]
    # integer inputs give integer results
    for x in [val["out"], val["grad_h"], *val["grad_W"]]:
        assert np.array_equal(x.numpy(), np.round(x.numpy()))
