"""The element-wise criterion of tests/bounds64.py tested on its own, without a GPU.

(a) float32 evaluations of every configuration of test_gpu_elementwise.py stay within 1e-5 of their bound: the bound is
    not too tight for a correct float32 computation.
(b) planted defects of the kinds a kernel can have are rejected.
(c) two of them pass the max-scaled criterion of the parity tests: the gap this criterion closes.  If that criterion is
    ever tightened, (c) says so.
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

import bounds64 as b64  # noqa: E402
import reference64 as r64  # noqa: E402
import reference64_edge_mlp as rm  # noqa: E402
import elementwise_cases as ge  # noqa: E402
from oracle import message_passing_oracle as mo  # noqa: E402
# (c) is about the parity tests' own criterion, so it is taken from them, not restated here.
from test_gpu_parity import assert_states_close  # noqa: E402

REL = 1e-5


# ---- (a) the float32 oracle passes -----------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ge.RGCN_CASES, ids=[c[0] for c in ge.RGCN_CASES])
def test_float32_oracle_rgcn_within_bound(case):
    name, path, V, D, H, L, agg, act, env = case
    p, w, h, adjs = ge.rgcn_case(V, D, H, L, agg, act, seed=V + H)
    ref = mo.message_passing_forward("rgcn", p, w, h, adjs, dtype=np.float64)
    got = mo.message_passing_forward("rgcn", p, w, h, adjs, dtype=np.float32)
    b64.assert_within_bound(got, ref, b64.forward_bound("rgcn", p, w, h, adjs), REL, what=name)


@pytest.mark.parametrize("V,act", ge.LAYERNORM_CASES)
def test_float32_oracle_layernorm_within_bound(V, act):
    p, w, h, adjs, ln = ge.layernorm_case(V, act)
    ref, bound = ge.layernorm_reference(p, w, h, adjs, ln)
    got, _ = ge.layernorm_reference(p, w, h, adjs, ln, dtype=np.float32)
    b64.assert_within_bound(got, ref, bound, REL, what="layernorm")


@pytest.mark.parametrize("name,kind,extra", ge.FAMILY_CASES, ids=[c[0] for c in ge.FAMILY_CASES])
def test_float32_oracle_family_within_bound(name, kind, extra):
    p, w, h, adjs = ge.family_case(kind, extra)
    ref = mo.message_passing_forward(kind, p, w, h, adjs, dtype=np.float64)
    got = mo.message_passing_forward(kind, p, w, h, adjs, dtype=np.float32)
    b64.assert_within_bound(got, ref, b64.forward_bound(kind, p, w, h, adjs), REL, what=name)


def _weighted(x, w, ids, G, K, dtype):
    x = x.astype(dtype)
    return mo.unsorted_segment_sum((x.reshape(-1, K, x.shape[1] // K) * w.astype(dtype)[:, :, None]).reshape(x.shape),
                                   ids, G)


def test_float32_reductions_within_bound():
    K = 4
    ptr, x, scores = ge.reduction_inputs(K=K)
    G = len(ptr) - 1
    ids = b64.graph_ids(ptr)
    for agg in ("sum", "mean", "sqrt_n", "max"):
        fn = mo.get_aggregation_function(agg)
        b64.assert_within_bound(fn(x, ids, G), fn(x.astype(np.float64), ids, G), b64.segment_bound(x, ptr, agg=agg), REL,
                                what=agg)
    sig = (1.0 / (1.0 + np.exp(-scores.astype(np.float64)))).astype(np.float32)
    b64.assert_within_bound(_weighted(x, sig, ids, G, K, np.float32), _weighted(x, sig, ids, G, K, np.float64),
                            b64.segment_bound(x, ptr, weights=sig, num_heads=K), REL, what="sigmoid")
    a32 = np.stack([mo.unsorted_segment_softmax(scores[:, k], ids, G) for k in range(K)], 1)
    a64 = np.stack([mo.unsorted_segment_softmax(scores[:, k].astype(np.float64), ids, G) for k in range(K)], 1)
    b64.assert_within_bound(_weighted(x, a32, ids, G, K, np.float32), _weighted(x, a64, ids, G, K, np.float64),
                            b64.softmax_segment_bound(x, scores, ptr, K), REL, what="softmax")


def _grads32(fn, tensors, g):
    leaves = [torch.from_numpy(np.asarray(t, np.float32)).requires_grad_() for t in tensors]
    out = fn(*leaves)
    out.backward(torch.from_numpy(np.asarray(g, np.float32)))
    return [out.detach().numpy()] + [x.grad.numpy() for x in leaves]


@pytest.mark.parametrize("act", ["tanh", "gelu"])
@pytest.mark.parametrize("V,K,N,bias", ge.DENSE_BWD_CASES)
def test_float32_dense_backward_within_bound(act, V, K, N, bias):
    x, W, b, g = ge.dense_bwd_inputs(V, K, N, bias)
    b = b if bias else np.zeros(W.shape[1], np.float32)
    fn = lambda x_, W_, b_: r64.act_and_grad(x_ @ W_ + b_, act)[0]   # noqa: E731
    got = _grads32(fn, (x, W, b), g)
    leaves = [torch.from_numpy(a).double().requires_grad_() for a in (x, W, b)]
    out = fn(*leaves)
    out.backward(torch.from_numpy(g).double())
    ref = [out.detach().numpy()] + [t.grad.numpy() for t in leaves]
    bd = b64.dense_backward_bound(x, W, b if bias else None, g, act)
    for key, a, r in zip(("out", "grad_x", "grad_W", "grad_bias"), got, ref):
        b64.assert_within_bound(a, r, bd[key], REL, what=key)


@pytest.mark.parametrize("act", ["tanh", "gelu"])
@pytest.mark.parametrize("V,D,H,agg,normalize", ge.RGCN_BWD_CASES)
def test_float32_rgcn_backward_within_bound(act, V, D, H, agg, normalize):
    h, adjs, Ws, g = ge.rgcn_bwd_inputs(V, D, H)
    L = len(Ws)
    a_t = [torch.from_numpy(a) for a in adjs]
    got = _grads32(lambda h_, *W_: rm.edge_mlp_autograd(h_, a_t, W_, None, agg=agg, act=act, normalize=normalize),
                   (h, *Ws), g)
    ref = r64.rgcn_layer(h, adjs, Ws, g, agg=agg, act=act, normalize=normalize)
    bd = b64.rgcn_backward_bound(h, adjs, Ws, g, agg=agg, act=act, normalize=normalize)
    b64.assert_within_bound(got[0], ref["out"].numpy(), bd["out"], REL, what="out")
    b64.assert_within_bound(got[1], ref["grad_h"].numpy(), bd["grad_h"], REL, what="grad_h")
    for l in range(L):
        b64.assert_within_bound(got[2 + l], ref["grad_W"][l].numpy(), bd["grad_W"][l], REL, what=f"grad_W[{l}]")


@pytest.mark.parametrize("act,agg,use_target", ge.EDGE_MLP_BWD_CASES)
def test_float32_edge_mlp_backward_within_bound(act, agg, use_target):
    h, adjs, Us, W2s, g = ge.edge_mlp_bwd_inputs(use_target)
    L = len(Us)
    a_t = [torch.from_numpy(a) for a in adjs]
    got = _grads32(lambda h_, *w_: rm.edge_mlp_autograd(h_, a_t, w_[:L], w_[L:], agg=agg, act=act, use_target=use_target),
                   (h, *Us, *W2s), g)
    ref = rm.edge_mlp_layer(h, adjs, Us, W2s, g, agg=agg, act=act, use_target=use_target)
    bd = b64.edge_mlp_backward_bound(h, adjs, Us, W2s, g, agg=agg, act=act, normalize=False, use_target=use_target)
    b64.assert_within_bound(got[0], ref["out"].numpy(), bd["out"], REL, what="out")
    b64.assert_within_bound(got[1], ref["grad_h"].numpy(), bd["grad_h"], REL, what="grad_h")
    for l in range(L):
        b64.assert_within_bound(got[2 + l], ref["grad_U"][l].numpy(), bd["grad_U"][l], REL, what=f"grad_U[{l}]")
        b64.assert_within_bound(got[2 + L + l], ref["grad_W2"][l].numpy(), bd["grad_W2"][l], REL, what=f"grad_W2[{l}]")


# ---- (b) planted defects fail, (c) two of them pass the max-scaled criterion -------------------------------------------
def _tf32(x):
    """Round to the 10-bit mantissa of TF32 (round to nearest even on the dropped 13 bits)."""
    b = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    b = (b + 0xFFF + ((b >> 13) & 1)) & ~np.uint64(0x1FFF)
    return b.astype(np.uint32).view(np.float32)


@pytest.fixture(scope="module")
def hub_case():
    """RGCN V=5000, D=H=128, L=4, target hub and duplicate edges, sum, relu, not normalised."""
    rng = np.random.default_rng(1)
    V, D, H, L = 5000, 128, 128, 4
    adjs = ge.random_graph(rng, V, L, 30000, hub=True, dups=True)
    p = mo.default_hyperparameters("rgcn")
    p.update(hidden_dim=H, aggregation_function="sum", message_activation_function="relu", normalize_by_num_incoming=False)
    w = mo.make_weights("rgcn", p, D, L, rng)
    h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    ref = mo.message_passing_forward("rgcn", p, w, h, adjs, dtype=np.float64)
    bound = b64.forward_bound("rgcn", p, w, h, adjs)
    return p, w, h, adjs, ref, bound


def test_hub_case_spans_two_orders_of_magnitude(hub_case):
    *_, ref, _ = hub_case
    assert np.abs(ref).max() > 100 * np.median(np.abs(ref).max(axis=1))


def test_tf32_tile_is_rejected_and_passes_the_max_scaled_check(hub_case):
    """Rows 128..255 computed from TF32-rounded h and W: a 3xTF32 tile that dropped its correction products."""
    p, w, h, adjs, ref, bound = hub_case
    w_tf32 = {"edge_mlps": [[_tf32(m[0])] for m in w["edge_mlps"]]}
    bad = mo.message_passing_forward("rgcn", p, w_tf32, _tf32(h), adjs, dtype=np.float64)
    got = ref.astype(np.float32)
    got[128:256] = bad[128:256]
    with pytest.raises(AssertionError, match="128-row tile 1"):
        b64.assert_within_bound(got, ref, bound, REL, what="tf32 tile", tiles=True)
    assert_states_close(got, ref)          # (c): the max-scaled criterion does not see it


def test_dropped_edge_is_rejected(hub_case):
    p, w, h, adjs, ref, bound = hub_case
    deg = ge.in_degree(len(h), adjs)
    v = int(np.flatnonzero((deg >= 8) & (deg <= 50))[0])
    l = next(i for i, a in enumerate(adjs) if np.any(a[:, 1] == v))
    e = int(np.flatnonzero(adjs[l][:, 1] == v)[0])
    dropped = [a if i != l else np.delete(a, e, axis=0) for i, a in enumerate(adjs)]
    got = ref.astype(np.float32)
    got[v] = mo.message_passing_forward("rgcn", p, w, h, dropped, dtype=np.float64)[v]
    with pytest.raises(AssertionError, match=f"row {v}"):
        b64.assert_within_bound(got, ref, bound, REL, what="dropped edge", row_sizes=deg)


def test_one_node_graph_error_is_rejected_and_passes_the_max_scaled_check():
    ptr, x, _ = ge.reduction_inputs()
    G = len(ptr) - 1
    ids = b64.graph_ids(ptr)
    ref = mo.unsorted_segment_sum(x.astype(np.float64), ids, G)
    got = ref.astype(np.float32)
    one = int(np.flatnonzero(np.diff(ptr) == 1)[0])
    got[one] *= np.float32(1 + 1e-3)
    with pytest.raises(AssertionError, match="graph size 1"):
        b64.assert_within_bound(got, ref, b64.segment_bound(x, ptr), REL, what="one-node graph",
                                row_sizes=np.diff(ptr), row_label="graph size")
    assert_states_close(got, ref)          # (c)


def test_nan_element_is_rejected(hub_case):
    *_, ref, bound = hub_case
    got = ref.astype(np.float32)
    got[17, 3] = np.nan
    with pytest.raises(AssertionError, match="row 17, column 3"):
        b64.assert_within_bound(got, ref, bound, REL, what="nan")


def test_stale_row_is_rejected(hub_case):
    """A row the kernel never wrote, holding what the buffer held before: here the previous row's result."""
    *_, ref, bound = hub_case
    got = ref.astype(np.float32)
    got[1001] = got[1000]
    with pytest.raises(AssertionError, match="row 1001"):
        b64.assert_within_bound(got, ref, bound, REL, what="stale row")


def test_exact_elements_and_the_max_identity():
    """bound == 0 demands float32(ref) exactly; the unsorted_segment_max identity must be finfo(float32).min."""
    ref = np.array([[0.0, 1.0], [np.finfo(np.float64).min, 2.0]])
    bound = np.array([[0.0, 1.0], [0.0, 1.0]])
    ok = np.array([[0.0, 1.0], [np.finfo(np.float32).min, 2.0]], np.float32)
    assert b64.assert_within_bound(ok, ref, bound) == 0.0
    for bad in (np.array([[1e-30, 1.0], [b64.LOWEST, 2.0]], np.float32),
                np.array([[0.0, 1.0], [-3e38, 2.0]], np.float32)):
        with pytest.raises(AssertionError):
            b64.assert_within_bound(bad, ref, bound)


def test_activation_constants():
    assert b64.lipschitz("relu") == 1.0 and b64.lipschitz("tanh") == pytest.approx(1.0)
    assert b64.lipschitz("gelu") == pytest.approx(1.129, abs=1e-3)
    assert b64.lipschitz("selu") == pytest.approx(mo.SELU_SCALE * mo.SELU_ALPHA, rel=1e-4)
    assert b64.act2max("tanh") == pytest.approx(4 / 3 ** 1.5, rel=1e-3)
    assert b64.act2max("gelu") == pytest.approx(0.798, abs=1e-3)
    with pytest.raises(ValueError):
        b64.act2max("relu")
