"""The steps of the fused transform-then-aggregate backward (max aggregation and / or activation before aggregation, edge
MLPs without hidden layer; csrc/backward.cu transform_aggregate_bwd), restated in float64 numpy
(reference64_transform_aggregate.backward), against float64 torch autograd of the reference's literal op order: ties from
duplicate edges share the gradient as tf.math.unsorted_segment_max's gradient shares it, empty segments pass none, and the
contributions of target-range shards sum to the whole."""
import numpy as np
import pytest
import torch

import reference64_transform_aggregate as ta

V, D, H, L = 40, 6, 5, 3


def _graph(rng, empty_target=True):
    """L edge lists with duplicate edges (real ties under max) and, optionally, target 7 without incoming edges."""
    adjs = []
    for _ in range(L):
        a = rng.integers(0, V, size=(90, 2))
        a = np.concatenate([a, a[:25]])            # duplicates
        if empty_target:
            a = a[a[:, 1] != 7]
        adjs.append(a.astype(np.int32))
    return adjs


def _inputs(seed, use_target, empty_target=True):
    rng = np.random.default_rng(seed)
    adjs = _graph(rng, empty_target)
    h = rng.integers(-3, 4, size=(V, D)).astype(np.float64)
    Ws = [rng.integers(-2, 3, size=((2 if use_target else 1) * D, H)).astype(np.float64) for _ in range(L)]
    g = rng.uniform(-1, 1, (V, H))
    return adjs, h, Ws, g


def _autograd(adjs, h, Ws, g, **kw):
    ht = torch.from_numpy(h).requires_grad_()
    Wt = [torch.from_numpy(w).requires_grad_() for w in Ws]
    out = ta.literal_autograd(ht, adjs, Wt, **kw)
    out.backward(torch.from_numpy(g))
    return out.detach().numpy(), ht.grad.numpy(), [w.grad.numpy() for w in Wt]


def _close(a, b, what):
    scale = max(float(np.abs(b).max()), 1.0)
    assert np.abs(np.asarray(a) - np.asarray(b)).max() <= 1e-10 * scale, what


CASES = ([dict(agg="max", act=act, act_before=False, normalize=n) for act in ("relu", "tanh", "gelu") for n in (False, True)]
         + [dict(agg="max", act=act, act_before=True, normalize=n) for act in ("tanh", "gelu") for n in (False, True)]
         + [dict(agg=agg, act=act, act_before=True, normalize=n)
            for agg, act, n in (("sum", "tanh", False), ("mean", "gelu", True), ("sqrt_n", "relu", False),
                                ("sqrt_n", "tanh", True), ("mean", "elu", False))])


@pytest.mark.parametrize("use_target", [False, True])
@pytest.mark.parametrize("kw", CASES, ids=lambda kw: "-".join(str(v) for v in kw.values()))
def test_fused_steps_match_autograd_of_the_literal_order(kw, use_target):
    adjs, h, Ws, g = _inputs(len(kw["act"]) + 3 * kw["normalize"], use_target)
    kw = dict(kw, use_target=use_target)
    out, gh, gw = ta.backward(h, adjs, Ws, g, **kw)
    r_out, r_gh, r_gw = _autograd(adjs, h, Ws, g, **kw)
    _close(out, r_out, "out")
    _close(gh, r_gh, "grad_h")
    for a, b in zip(gw, r_gw):
        _close(a, b, "grad_W")
    if kw["agg"] == "max":
        _, ties = ta.max_margin(h, adjs, Ws, **{k: kw[k] for k in ("act", "act_before", "normalize", "use_target")})
        assert ties > 0                                  # the case exercises the tie rule
        assert np.all(out[7] == (ta.LOWEST if kw["act_before"] else ta._act(torch.tensor(ta.LOWEST), kw["act"]).item()))


def test_tied_messages_share_the_gradient():
    """One target, two identical messages and a smaller one: each tied message gets half of the gradient."""
    h = np.array([[1.0], [1.0], [0.5], [0.0]])
    W = [np.array([[2.0]])]
    adjs = [np.array([[0, 3], [1, 3], [2, 3]], np.int32)]
    g = np.array([[0.0], [0.0], [0.0], [4.0]])
    _, gh, gw = ta.backward(h, adjs, W, g, agg="max", act=None)
    assert np.array_equal(gh[:, 0], [4.0, 4.0, 0.0, 0.0])     # 4 / 2 ties * W = 2 * 2
    assert np.array_equal(gw[0], [[4.0]])                      # h_0 * 2 + h_1 * 2
    _, r_gh, r_gw = _autograd(adjs, h, W, g, agg="max", act=None)
    assert np.array_equal(gh, r_gh) and np.array_equal(gw[0], r_gw[0])


@pytest.mark.parametrize("kw", [dict(agg="max", act="tanh", act_before=False, normalize=True, use_target=True),
                                dict(agg="max", act="gelu", act_before=True, normalize=False, use_target=False),
                                dict(agg="sqrt_n", act="tanh", act_before=True, normalize=True, use_target=True)],
                         ids=["max-target", "max-before", "sqrt_n-before-target"])
def test_target_range_contributions_sum_to_the_whole(kw):
    adjs, h, Ws, g = _inputs(11, kw["use_target"])
    out, gh, gw = ta.backward(h, adjs, Ws, g, **kw)
    for bounds in ([(0, 17), (17, V)], [(0, 9), (9, 9), (9, 30), (30, V)]):   # the second world has an empty shard
        sum_h = np.zeros_like(gh)
        sum_w = [np.zeros_like(w) for w in gw]
        outs = []
        for lo, hi in bounds:
            o, a, ws = ta.backward(h, adjs, Ws, g[lo:hi], lo=lo, hi=hi, **kw)
            if lo == hi:
                assert not a.any() and not any(w.any() for w in ws)
            outs.append(o)
            sum_h += a
            for s, w in zip(sum_w, ws):
                s += w
        _close(np.concatenate(outs), out, "out")
        _close(sum_h, gh, "grad_h")
        for s, w in zip(sum_w, gw):
            _close(s, w, "grad_W")
