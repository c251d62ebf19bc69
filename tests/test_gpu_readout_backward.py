"""Training of the graph readout, the three global exchanges and WASGraphRepresentation on graph row ranges
(layers/graph_autograd.py, tfgnn_b200_segment_sum_rows / readout_bwd / gru_gate_bwd_indexed) against the float64 reference
of reference64_readout.py: entry by entry, exact cases, layer gradients, training forward == inference forward, bitwise
reproducibility, dropout masks, scale, and routing away from the atomic segment reduce."""
import os
import sys

import numpy as np
import pytest

torch = pytest.importorskip("torch")
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import reference64_readout as r64  # noqa: E402
from oracle import message_passing_oracle as mo  # noqa: E402

pytestmark = pytest.mark.gpu
TOL = 3e-5


@pytest.fixture(autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def close(got, ref, tol=TOL, what="", floor=1e-30):
    got = np.asarray(got.detach().cpu().numpy() if isinstance(got, torch.Tensor) else got, np.float64)
    ref = np.asarray(ref.detach().numpy() if isinstance(ref, torch.Tensor) else ref, np.float64)
    assert got.shape == ref.shape, f"{what}: shape {got.shape} vs {ref.shape}"
    err, scale = np.linalg.norm(got - ref), max(np.linalg.norm(ref), floor)
    assert err <= tol * scale, f"{what}: |err| {err:.3e} > {tol:g} * {scale:.3e}"


def close_variables(gots, wants, what):
    """Every variable's gradient at the bar, measured against its own norm or, where that is smaller, the largest norm among
    the layer's variables: under softmax weighting the gradient of the scoring MLP's output bias is exactly zero (a shift of a
    head's scores changes no weight), and what float32 leaves there is the rounding of sums whose terms are not small."""
    wants = list(wants)
    floor = max(np.linalg.norm(w) for w in wants)
    for got, want in zip(gots, wants):
        close(got, want, what=what, floor=floor)


def dev(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(device="cuda", dtype=dtype)


def graph_sizes(layout: str, rng):
    """Row counts per graph for the layouts a user meets and the corner cases of the chunked sum."""
    if layout == "many_short":
        return rng.integers(1, 30, size=700)
    if layout == "three_long":
        return np.array([2100, 3300, 2600])
    if layout == "one":
        return np.array([5000])
    if layout == "empty_first_middle_last":
        return np.array([0, 0, 70, 0, 129, 64, 0, 1, 300, 0, 0])
    if layout == "chunk_aligned":
        return np.array([64, 128, 64, 1, 63])
    raise ValueError(layout)


def f32(bound):
    """A bound as the kernels see it (a float32): a float32 value equal to it is a tie, not a cut."""
    return None if bound is None else float(np.float32(bound))


def n2g_of(sizes):
    return np.repeat(np.arange(len(sizes)), sizes).astype(np.int32)


LAYOUTS = ["many_short", "three_long", "one", "empty_first_middle_last", "chunk_aligned"]


def ptr_of(n2g_t, G):
    from tf2_gnn_b200.layers import node_ops
    return node_ops.graph_offsets(n2g_t, G, validate=True)


# ---- 1 / 2: the entries alone ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("C", [1, 30, 96, 320 * 3])
def test_segment_sum_rows_against_float64(layout, C):
    from tf2_gnn_b200.layers import graph_autograd
    rng = np.random.default_rng(C)
    sizes = graph_sizes(layout, rng)
    n2g = n2g_of(sizes)
    data = rng.uniform(-1, 1, (len(n2g), C)).astype(np.float32)
    n2g_t = dev(n2g, torch.int32)
    got = graph_autograd.segment_sum_rows(dev(data), n2g_t, ptr_of(n2g_t, len(sizes)))
    ptr = r64.graph_ptr_of(n2g, len(sizes))
    ref = np.stack([data[ptr[g]:ptr[g + 1]].astype(np.float64).sum(0) for g in range(len(sizes))])
    close(got, ref, tol=1e-6, what="segment_sum_rows")
    # the documented order of additions, in float32 on the host: bitwise
    if len(n2g) <= 1000:
        assert np.array_equal(got.cpu().numpy(), r64.segment_sum_rows_chunked(data, ptr))


@pytest.mark.parametrize("layout", LAYOUTS)
def test_segment_sum_rows_is_exact_on_integers(layout):
    from tf2_gnn_b200.layers import graph_autograd
    rng = np.random.default_rng(1)
    sizes = graph_sizes(layout, rng)
    n2g = n2g_of(sizes)
    for C in (7, 64):
        data = rng.integers(-8, 9, size=(len(n2g), C)).astype(np.float32)
        n2g_t = dev(n2g, torch.int32)
        got = graph_autograd.segment_sum_rows(dev(data), n2g_t, ptr_of(n2g_t, len(sizes))).cpu().numpy()
        ptr = r64.graph_ptr_of(n2g, len(sizes))
        ref = np.stack([data[ptr[g]:ptr[g + 1]].astype(np.float64).sum(0) for g in range(len(sizes))])
        assert np.array_equal(got.astype(np.float64), ref)


def test_segment_sum_rows_without_rows_or_graphs():
    from tf2_gnn_b200.layers import graph_autograd
    empty = torch.zeros((0, 8), device="cuda")
    ids = torch.zeros((0,), dtype=torch.int32, device="cuda")
    out = graph_autograd.segment_sum_rows(empty, ids, torch.zeros(4, dtype=torch.int32, device="cuda"))
    assert out.shape == (3, 8) and not out.any()
    assert graph_autograd.segment_sum_rows(empty, ids, torch.zeros(1, dtype=torch.int32, device="cuda")).shape == (0, 8)


def _readout_bwd(reprs, weights, n2g, G, K, mode, out, grad_out, lower=None, upper=None):
    from tf2_gnn_b200 import _ffi
    from tf2_gnn_b200.runtime import stream_ptr
    n2g_t = dev(n2g, torch.int32)
    ptr = ptr_of(n2g_t, G)
    r, go = dev(reprs), dev(grad_out)
    w = dev(weights) if weights is not None else None
    o = dev(out) if out is not None else None
    gr = torch.empty_like(r)
    gs = torch.empty_like(w) if w is not None else None
    p = lambda t: 0 if t is None else t.data_ptr()
    _ffi.check(_ffi.lib().tfgnn_b200_readout_bwd(
        r.data_ptr(), p(w), n2g_t.data_ptr(), ptr.data_ptr(), p(o), go.data_ptr(), r.shape[0], G, r.shape[1], K,
        _ffi.READOUT_MODE[mode], float(lower or 0.0), float(upper or 0.0), int(lower is not None), int(upper is not None),
        gr.data_ptr(), p(gs), stream_ptr()))
    torch.cuda.synchronize()
    return gs, gr


@pytest.mark.parametrize("mode", ["softmax", "sigmoid", "none", "average"])
@pytest.mark.parametrize("layout,GD,K,bounds", [("many_short", 64, 4, (None, None)), ("three_long", 320, 4, (-0.3, 0.4)),
                                                ("one", 30, 3, (None, 0.2)), ("empty_first_middle_last", 15, 1, (0.1, None)),
                                                ("many_short", 12, 12, (None, None))])
def test_readout_bwd_entry_against_float64(mode, layout, GD, K, bounds):
    rng = np.random.default_rng(GD + K)
    bounds = (f32(bounds[0]), f32(bounds[1]))
    sizes = graph_sizes(layout, rng)
    n2g, G = n2g_of(sizes), len(sizes)
    V = len(n2g)
    scores = rng.uniform(-2, 2, (V, K)).astype(np.float32)
    reprs = rng.uniform(-1, 1, (V, GD)).astype(np.float32)
    grad_out = rng.uniform(-1, 1, (G, GD)).astype(np.float32)
    weights = out = None
    if mode in ("softmax", "sigmoid"):
        # the forward's own weights and result, as the layer saves them
        with torch.no_grad():
            fwd = r64.readout_from_scores(torch.from_numpy(scores).double(), torch.from_numpy(reprs).double(), n2g, G, K, mode,
                                          *bounds)
            out = fwd.numpy().astype(np.float32)
        s = scores.astype(np.float64)
        if mode == "sigmoid":
            weights = (1 / (1 + np.exp(-s))).astype(np.float32)
        else:
            ids = n2g.astype(np.int64)
            mx = np.full((G, K), -np.inf)
            np.maximum.at(mx, ids, s)
            e = np.exp(s - mx[ids])
            z = np.zeros((G, K))
            np.add.at(z, ids, e)
            weights = (e / z[ids]).astype(np.float32)
    gs_ref, gr_ref = r64.readout_backward_closed_form(scores, reprs, n2g, G, K, mode, grad_out, *bounds)
    gs, gr = _readout_bwd(reprs, weights, n2g, G, K, mode, out, grad_out, *bounds)
    close(gr, gr_ref, what=f"grad_reprs {mode}")
    if gs_ref is not None:
        close(gs, gs_ref, what=f"grad_scores {mode}")


@pytest.mark.parametrize("mode", ["softmax", "sigmoid", "none", "average"])
def test_readout_bwd_is_exact_on_small_integers_and_passes_the_gradient_at_a_clamp_tie(mode):
    """Dyadic weights, small integers and graphs of 1, 2, 4 or 8 nodes: every product, sum and quotient is exact in float32,
    so the entry must equal the float64 closed form bit for bit.  reprs equal to a bound keep their gradient (tf.maximum /
    tf.minimum pass it to their first argument on a tie); reprs beyond a bound lose it."""
    rng = np.random.default_rng(8)
    sizes = np.array([4, 0, 8, 1, 2, 64, 128, 0])
    n2g, G, GD, K = n2g_of(sizes), len(sizes), 24, 3
    V = len(n2g)
    lower, upper = -2.0, 3.0
    reprs = rng.integers(-4, 6, size=(V, GD)).astype(np.float32)          # hits both bounds exactly and crosses them
    assert (reprs == lower).any() and (reprs == upper).any() and (reprs < lower).any() and (reprs > upper).any()
    grad_out = rng.integers(-3, 4, size=(G, GD)).astype(np.float32)
    weights = out = None
    if mode in ("softmax", "sigmoid"):
        weights = rng.choice([0.25, 0.5, 0.75], size=(V, K)).astype(np.float32)
        R = np.clip(reprs, lower, upper).astype(np.float64)
        o = np.zeros((G, K, GD // K))
        np.add.at(o, n2g.astype(np.int64), weights.astype(np.float64)[:, :, None] * R.reshape(V, K, -1))
        out = o.reshape(G, GD).astype(np.float32)
    gs_ref, gr_ref = r64.readout_backward_closed_form(None, reprs, n2g, G, K, mode, grad_out, lower, upper, weights=weights)
    gs, gr = _readout_bwd(reprs, weights, n2g, G, K, mode, out, grad_out, lower, upper)
    assert np.array_equal(gr.cpu().numpy().astype(np.float64), gr_ref)
    if gs_ref is not None:
        assert np.array_equal(gs.cpu().numpy().astype(np.float64), gs_ref)
    tie = (reprs == lower) | (reprs == upper)
    cut = (reprs < lower) | (reprs > upper)
    got = gr.cpu().numpy()
    assert not got[cut].any()
    assert np.array_equal(got[tie], gr_ref[tie].astype(np.float32)) and got[tie].any()


@pytest.mark.parametrize("layout,H", [("many_short", 32), ("three_long", 100), ("empty_first_middle_last", 7)])
def test_gru_gate_bwd_indexed_against_float64(layout, H):
    from tf2_gnn_b200 import _ffi
    from tf2_gnn_b200.runtime import stream_ptr
    rng = np.random.default_rng(H)
    sizes = graph_sizes(layout, rng)
    n2g, G = n2g_of(sizes), len(sizes)
    V = len(n2g)
    gx, gh = rng.uniform(-1, 1, (G, 3 * H)).astype(np.float32), rng.uniform(-1, 1, (V, 3 * H)).astype(np.float32)
    h, go = rng.uniform(-1, 1, (V, H)).astype(np.float32), rng.uniform(-1, 1, (V, H)).astype(np.float32)
    gx64, gh64, h64 = r64.leaf(gx), r64.leaf(gh), r64.leaf(h)
    x = gx64[torch.from_numpy(n2g).long()]
    z = torch.sigmoid(x[:, :H] + gh64[:, :H])
    r = torch.sigmoid(x[:, H:2 * H] + gh64[:, H:2 * H])
    out = z * h64.detach() + (1 - z) * torch.tanh(x[:, 2 * H:] + r * gh64[:, 2 * H:])
    (out * torch.from_numpy(go).double()).sum().backward()
    n2g_t = dev(n2g, torch.int32)
    ptr = ptr_of(n2g_t, G)
    t = [dev(a) for a in (gx, gh, h, go)]
    dgx, dgh, dh = torch.empty_like(t[0]), torch.empty_like(t[1]), torch.empty_like(t[2])
    _ffi.check(_ffi.lib().tfgnn_b200_gru_gate_bwd_indexed(t[0].data_ptr(), n2g_t.data_ptr(), ptr.data_ptr(), t[1].data_ptr(),
                                                          t[2].data_ptr(), t[3].data_ptr(), V, G, H, dgx.data_ptr(),
                                                          dgh.data_ptr(), dh.data_ptr(), stream_ptr()))
    close(dgx, gx64.grad, what="grad_gx per graph")
    close(dgh, gh64.grad, what="grad_gh")
    close(dh, torch.from_numpy(go).double() * z.detach(), what="direct state path")


# ---- 3 / 4: layers ----------------------------------------------------------------------------------------------
def _assign(mlp, kernels, biases=None):
    for var, m in zip(mlp.kernels, kernels):
        var.assign(np.asarray(m, np.float32))
    if biases is not None:
        for var, m in zip(mlp.biases, biases):
            var.assign(np.asarray(m, np.float32))


def _load_readout(layer, w):
    if "scoring_mlp" in w:
        _assign(layer._scoring_mlp, w["scoring_mlp"], w.get("scoring_biases"))
    _assign(layer._transformation_mlp, w["transformation_mlp"], w.get("transformation_biases"))


def _readout_grads(layer):
    """In the order of r64.flat_grads (sorted keys of the weight dict)."""
    out = []
    if layer._scoring_mlp is not None:
        out += [v.grad for v in (layer._scoring_mlp.biases or [])] + [v.grad for v in layer._scoring_mlp.kernels]
    out += [v.grad for v in (layer._transformation_mlp.biases or [])] + [v.grad for v in layer._transformation_mlp.kernels]
    return out


def _readout_weights(rng, D, GD, K, mode, biases):
    w = {"transformation_mlp": [mo.glorot_uniform(rng, (D, 24)), mo.glorot_uniform(rng, (24, GD))]}
    if mode in ("softmax", "sigmoid"):
        w["scoring_mlp"] = [mo.glorot_uniform(rng, (D, 20)) * 2, mo.glorot_uniform(rng, (20, K)) * 2]
    if biases:
        w["transformation_biases"] = [rng.uniform(-.2, .2, 24).astype(np.float32), rng.uniform(-.2, .2, GD).astype(np.float32)]
        if "scoring_mlp" in w:
            w["scoring_biases"] = [rng.uniform(-.2, .2, 20).astype(np.float32), rng.uniform(-.2, .2, K).astype(np.float32)]
    return w


def _make_readout(D, GD, K, mode, w, regression_task: bool):
    from tf2_gnn_b200.layers import NodesToGraphRepresentationInput, WeightedSumGraphRepresentation
    kw = dict(scoring_mlp_layers=[20], transformation_mlp_layers=[24])
    if regression_task:      # biases, ELU, bounded transformation results: what graph_regression_task.py configures
        kw.update(scoring_mlp_activation_fun="elu", scoring_mlp_use_biases=True, transformation_mlp_activation_fun="elu",
                  transformation_mlp_use_biases=True, transformation_mlp_result_lower_bound=-0.3,
                  transformation_mlp_result_upper_bound=0.4)
    layer = WeightedSumGraphRepresentation(GD, K, mode, **kw)
    layer.build(NodesToGraphRepresentationInput((None, D), None, None))
    _load_readout(layer, w)
    for v in layer.variables:
        v.requires_grad_(True)
    return layer


@pytest.mark.parametrize("mode", ["softmax", "sigmoid", "none", "average"])
@pytest.mark.parametrize("regression_task", [False, True])
def test_readout_layer_gradients_and_training_forward(mode, regression_task):
    from tf2_gnn_b200.layers import NodesToGraphRepresentationInput, differentiable
    rng = np.random.default_rng(11)
    D, GD, K = 32, 16, 4
    sizes = rng.integers(0, 40, size=60)
    n2g, G = n2g_of(sizes), len(sizes)
    V = len(n2g)
    x = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    R = rng.uniform(-1, 1, (G, GD)).astype(np.float32)
    w = _readout_weights(rng, D, GD, K, mode, regression_task)
    layer = _make_readout(D, GD, K, mode, w, regression_task)
    xt = dev(x).requires_grad_()
    inp = NodesToGraphRepresentationInput(xt, dev(n2g, torch.int32), G)
    out = layer(inp, training=False)
    (out * dev(R)).sum().backward()
    with torch.no_grad():
        assert torch.equal(layer(inp, training=False), out.detach())          # training forward == inference forward
    L, x64 = r64.leaves_of(w), r64.leaf(x)
    acts, bounds = (("elu", "elu"), (f32(-0.3), f32(0.4))) if regression_task else (("relu", "relu"), (None, None))
    ref = r64.readout_layer(x64, L, n2g, G, K, mode, *acts, *bounds)
    (ref * torch.from_numpy(R).double()).sum().backward()
    close(out, ref, tol=1e-5, what="readout forward")
    close(xt.grad, x64.grad, what="readout grad_x")
    close_variables(_readout_grads(layer), r64.flat_grads(L), f"readout {mode} variable gradient")
    if not regression_task:
        # the literal op order stays importable and correct
        for v in layer.variables:
            v.value.grad = None
        x2 = dev(x).requires_grad_()
        lit = differentiable.weighted_sum_graph_representation(layer, x2, dev(n2g, torch.int32), G, False)
        (lit * dev(R)).sum().backward()
        close(lit, ref, tol=1e-5, what="literal readout forward")
        close(x2.grad, x64.grad, what="literal readout grad_x")
        close_variables(_readout_grads(layer), r64.flat_grads(L), f"literal readout {mode} variable gradient")


def _make_exchange(mode, H, K, weighting, w, dropout_rate=0.0, seed=None):
    from tf2_gnn_b200.layers import (GraphGlobalExchangeInput, GraphGlobalGRUExchange, GraphGlobalMeanExchange,
                                     GraphGlobalMLPExchange, node_ops)
    cls = {"mean": GraphGlobalMeanExchange, "gru": GraphGlobalGRUExchange, "mlp": GraphGlobalMLPExchange}[mode]
    ex = cls(hidden_dim=H, weighting_fun=weighting, num_heads=K, dropout_rate=dropout_rate)
    ex.build(GraphGlobalExchangeInput((None, H), (None,), ()))
    _load_readout(ex._node_to_graph_representation_layer, w)
    if mode == "gru":
        ex._gru_kernel.assign(w["gru_kernel"])
        ex._gru_recurrent_kernel.assign(w["gru_recurrent_kernel"])
        ex._gru_bias.assign(w["gru_bias"])
    if mode == "mlp":
        _assign(ex._mlp, w["mlp"])
    if seed is not None:
        ex.dropout_state = node_ops.DropoutState(seed)
    for v in ex.variables:
        v.requires_grad_(True)
    return ex


def _exchange_grads(ex, mode):
    """In the order of r64.flat_grads: gru_bias, gru_kernel, gru_recurrent_kernel | mlp, then the readout's."""
    out = []
    if mode == "gru":
        out += [ex._gru_bias.grad, ex._gru_kernel.grad, ex._gru_recurrent_kernel.grad]
    if mode == "mlp":
        out += [v.grad for v in ex._mlp.kernels]
    return out + _readout_grads(ex._node_to_graph_representation_layer)


@pytest.mark.parametrize("mode", ["mean", "gru", "mlp"])
@pytest.mark.parametrize("weighting", ["softmax", "sigmoid"])
def test_exchange_gradients_and_training_forward(mode, weighting):
    from tf2_gnn_b200.layers import GraphGlobalExchangeInput
    rng = np.random.default_rng(len(mode) + len(weighting))
    H, K = 32, 4
    sizes = rng.integers(0, 30, size=40)
    n2g, G = n2g_of(sizes), len(sizes)
    V = len(n2g)
    x = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    R = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    w = mo.make_exchange_weights(mode, H, K, rng, weighting)
    ex = _make_exchange(mode, H, K, weighting, w)
    xt = dev(x).requires_grad_()
    inp = GraphGlobalExchangeInput(xt, dev(n2g, torch.int32), G)
    out = ex(inp, training=False)
    (out * dev(R)).sum().backward()
    with torch.no_grad():
        assert torch.equal(ex(inp, training=False), out.detach())
    L, x64 = r64.leaves_of(w), r64.leaf(x)
    ref = r64.exchange(mode, x64, L, n2g, G, K, weighting)
    (ref * torch.from_numpy(R).double()).sum().backward()
    close(out, ref, tol=1e-5, what=f"exchange {mode} forward")
    close(xt.grad, x64.grad, what=f"exchange {mode} grad_x")
    close_variables(_exchange_grads(ex, mode), r64.flat_grads(L), f"exchange {mode} {weighting} variable gradient")


def test_was_graph_representation_trains():
    from tf2_gnn_b200.layers import NodesToGraphRepresentationInput, WASGraphRepresentation
    rng = np.random.default_rng(12)
    D, GD, K = 24, 16, 4
    sizes = rng.integers(0, 30, size=50)
    n2g, G = n2g_of(sizes), len(sizes)
    x = rng.uniform(-1, 1, (len(n2g), D)).astype(np.float32)
    R = rng.uniform(-1, 1, (G, GD)).astype(np.float32)
    layer = WASGraphRepresentation(GD, K, pooling_mlp_layers=[20, 12])
    layer.build(NodesToGraphRepresentationInput((None, D), None, None))
    names = [v.name for v in layer.variables]
    assert "WASGraphRepresentation/WeightedAvgGraphRepresentation/WeightedSumGraphRepresentation/ScoringMLP/dense_0/kernel:0" in names
    assert "WASGraphRepresentation/WeightedSumGraphRepresentation/WeightedSumGraphRepresentation/TransformationMLP/dense_2/bias:0" in names

    def weights():
        sizes_s, sizes_t = [D, 20, 12, K], [D, 20, 12, GD]
        return {"scoring_mlp": [mo.glorot_uniform(rng, (a, b)) for a, b in zip(sizes_s, sizes_s[1:])],
                "scoring_biases": [rng.uniform(-.2, .2, b).astype(np.float32) for b in sizes_s[1:]],
                "transformation_mlp": [mo.glorot_uniform(rng, (a, b)) for a, b in zip(sizes_t, sizes_t[1:])],
                "transformation_biases": [rng.uniform(-.2, .2, b).astype(np.float32) for b in sizes_t[1:]]}

    w_avg, w_sum = weights(), weights()
    P = mo.glorot_uniform(rng, (2 * GD, GD))
    _load_readout(layer._weighted_avg_graph_repr_layer, w_avg)
    _load_readout(layer._weighted_sum_graph_repr_layer, w_sum)
    layer._out_projection.assign(P)
    for v in layer.variables:
        v.requires_grad_(True)
    xt = dev(x).requires_grad_()
    inp = NodesToGraphRepresentationInput(xt, dev(n2g, torch.int32), G)
    out = layer(inp, training=False)
    (out * dev(R)).sum().backward()
    with torch.no_grad():
        assert torch.equal(layer(inp, training=False), out.detach())
    L_avg, L_sum, P64, x64 = r64.leaves_of(w_avg), r64.leaves_of(w_sum), r64.leaf(P), r64.leaf(x)
    ref = r64.was(x64, L_avg, L_sum, P64, n2g, G, K)
    (ref * torch.from_numpy(R).double()).sum().backward()
    close(out, ref, tol=1e-5, what="WAS forward")
    close(xt.grad, x64.grad, what="WAS grad_x")
    close(layer._out_projection.grad, P64.grad, what="WAS projection gradient")
    for sub, L in ((layer._weighted_avg_graph_repr_layer, L_avg), (layer._weighted_sum_graph_repr_layer, L_sum)):
        close_variables(_readout_grads(sub), r64.flat_grads(L), "WAS variable gradient")


# ---- 5: reproducibility at the shape where the atomic path collided most ------------------------------------------------
PPI = dict(sizes=np.array([2400, 3500, 2100]), H=320, K=4)


def _ppi_inputs(rng):
    n2g = n2g_of(PPI["sizes"])
    return n2g, rng.uniform(-1, 1, (len(n2g), PPI["H"])).astype(np.float32)


@pytest.mark.parametrize("mode", ["readout", "mean", "gru", "mlp"])
def test_two_identical_steps_give_bitwise_identical_gradients_at_ppi_shape(mode):
    from tf2_gnn_b200.layers import GraphGlobalExchangeInput, NodesToGraphRepresentationInput
    rng = np.random.default_rng(13)
    n2g, x = _ppi_inputs(rng)
    H, K, G = PPI["H"], PPI["K"], 3
    if mode == "readout":
        w = _readout_weights(rng, H, H, K, "softmax", False)
        layer = _make_readout(H, H, K, "softmax", w, False)
        make_input = lambda xt: NodesToGraphRepresentationInput(xt, dev(n2g, torch.int32), G)
    else:
        layer = _make_exchange(mode, H, K, "softmax", mo.make_exchange_weights(mode, H, K, rng, "softmax"))
        make_input = lambda xt: GraphGlobalExchangeInput(xt, dev(n2g, torch.int32), G)
    runs = []
    for _ in range(2):
        for v in layer.variables:
            v.value.grad = None
        xt = dev(x).requires_grad_()
        out = layer(make_input(xt), training=False)
        (out * out).sum().backward()
        runs.append([xt.grad.clone()] + [v.grad.clone() for v in layer.variables])
    for a, b in zip(*runs):
        assert torch.equal(a, b)
        assert torch.isfinite(a).all()


def test_default_gnn_with_dropout_is_bitwise_reproducible():
    """GNN.get_default_hyperparameters(): RGCN + GRU exchange every second layer, exchange dropout 0.2."""
    from tf2_gnn_b200.layers import GNN, GNNInput
    rng = np.random.default_rng(14)
    V, F, L = 8000, 50, 2
    n2g = n2g_of(np.array([2600, 2900, 2500]))
    params = GNN.get_default_hyperparameters()
    params.update(hidden_dim=64, layer_input_dropout_rate=0.1, b200_dropout_seed=21)
    adjs = tuple(dev(rng.integers(0, V, size=(40000, 2)).astype(np.int32), torch.int32) for _ in range(L))
    feats = dev(rng.uniform(-1, 1, (V, F)).astype(np.float32))
    runs = []
    for _ in range(2):
        torch.manual_seed(0)
        gnn = GNN(params)
        gnn.build(GNNInput((None, F), tuple((None, 2) for _ in range(L)), (None,), ()))
        for v in gnn.variables:
            v.requires_grad_(True)
        out = gnn(GNNInput(feats, adjs, dev(n2g, torch.int32), 3), training=True)
        (out * out).sum().backward()
        runs.append([out.detach().clone()] + [v.grad.clone() for v in gnn.variables])
    for a, b in zip(*runs):
        assert torch.equal(a, b) and torch.isfinite(a).all()


# ---- 6: the exchange's own dropout ----------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["mean", "gru", "mlp"])
def test_exchange_dropout_gradients_match_float64_with_the_same_masks(mode):
    from tf2_gnn_b200.layers import GraphGlobalExchangeInput, differentiable, node_ops
    rng = np.random.default_rng(15)
    H, K, rate, seed = 32, 4, 0.2, 99
    sizes = rng.integers(1, 30, size=30)
    n2g, G = n2g_of(sizes), len(sizes)
    V = len(n2g)
    x = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    R = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    w = mo.make_exchange_weights(mode, H, K, rng, "softmax")
    ex = _make_exchange(mode, H, K, "softmax", w, dropout_rate=rate, seed=seed)
    xt = dev(x).requires_grad_()
    n2g_t = dev(n2g, torch.int32)
    out = ex(GraphGlobalExchangeInput(xt, n2g_t, G), training=True)
    (out * dev(R)).sum().backward()
    # the masks, read off ones tables in the order the layer takes them: scoring MLP (two layer inputs, the MLPs' class default
    # rate 0.2), transformation MLP (two layer inputs), the per-node graph representations
    state = node_ops.DropoutState(seed)
    masks = [node_ops.dropout(torch.ones((V, n), device="cuda"), r, state).cpu().numpy()
             for n, r in ((H, 0.2), (H, 0.2), (H, 0.2), (128, 0.2), (H, rate))]
    assert all(0.1 < (m == 0).mean() < 0.3 for m in masks)
    L, x64 = r64.leaves_of(w), r64.leaf(x)
    ref = r64.exchange(mode, x64, L, n2g, G, K, "softmax", per_node_mask=masks[4], scoring_masks=masks[0:2],
                       transformation_masks=masks[2:4])
    (ref * torch.from_numpy(R).double()).sum().backward()
    close(out, ref, tol=1e-5, what=f"exchange {mode} forward under dropout")
    close(xt.grad, x64.grad, what=f"exchange {mode} grad_x under dropout")
    close_variables(_exchange_grads(ex, mode), r64.flat_grads(L), f"exchange {mode} variable gradient under dropout")
    # the literal path draws the same masks from the same seed
    ex.dropout_state = node_ops.DropoutState(seed)
    with torch.enable_grad():
        lit = differentiable.per_node_graph_representations(ex, dev(x).requires_grad_(), n2g_t, G, True)
    close(lit, r64.readout_layer(x64, L, n2g, G, K, "softmax", scoring_masks=masks[0:2], transformation_masks=masks[2:4])
          .detach()[torch.from_numpy(n2g).long()] * torch.from_numpy(masks[4]).double(), tol=1e-5,
          what="literal per-node representations under dropout")


# ---- 7: scale -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", ["qm9", "one_graph"])
def test_exchange_step_at_scale(shape):
    """One GRU exchange step at QM9 shape (500k nodes in 27.8k graphs, H = 128) and on a single graph of 1M nodes (H = 256):
    finite gradients; node-state gradients of the first graphs against float64 (a graph's rows depend on no other graph) at
    QM9 shape; the segment sum of sampled graphs against float64 at both."""
    from tf2_gnn_b200.layers import GraphGlobalExchangeInput, graph_autograd
    rng = np.random.default_rng(16)
    if shape == "qm9":
        G, H, K = 27800, 128, 4
        sizes = rng.integers(9, 30, size=G)
        sizes[-1] += 500_000 - sizes.sum() if sizes.sum() < 500_000 else 0
    else:
        G, H, K = 1, 256, 4
        sizes = np.array([1_000_000])
    n2g = n2g_of(sizes)
    V = len(n2g)
    x = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    R = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    w = mo.make_exchange_weights("gru", H, K, rng, "softmax")
    ex = _make_exchange("gru", H, K, "softmax", w)
    xt = dev(x).requires_grad_()
    n2g_t = dev(n2g, torch.int32)
    out = ex(GraphGlobalExchangeInput(xt, n2g_t, G), training=False)
    (out * dev(R)).sum().backward()
    assert torch.isfinite(xt.grad).all() and all(torch.isfinite(v.grad).all() for v in ex.variables)
    if shape == "qm9":
        n, g = int(sizes[:12].sum()), 12
        x64 = r64.leaf(x[:n])
        ref = r64.exchange("gru", x64, r64.leaves_of(w), n2g[:n], g, K, "softmax")
        (ref * torch.from_numpy(R[:n]).double()).sum().backward()
        close(out[:n], ref, tol=1e-5, what="exchange forward of the first graphs")
        close(xt.grad[:n], x64.grad, what="exchange grad_x of the first graphs")
    data = torch.rand((V, 3 * H), device="cuda") - 0.5
    got = graph_autograd.segment_sum_rows(data, n2g_t, ptr_of(n2g_t, G))
    ptr = r64.graph_ptr_of(n2g, G)
    for g in sorted({0, G // 2, G - 1}):
        close(got[g], data[ptr[g]:ptr[g + 1]].double().sum(0).cpu(), tol=1e-5, what=f"segment sum of graph {g}")


# ---- 8: routing ---------------------------------------------------------------------------------------------------
class _CountingLib:
    def __init__(self, real):
        self._real, self.calls = real, {}

    def __getattr__(self, name):
        self.calls[name] = self.calls.get(name, 0) + 1
        return getattr(self._real, name)


@pytest.fixture
def counting_lib(monkeypatch):
    from tf2_gnn_b200 import _ffi
    proxy = _CountingLib(_ffi.lib())
    monkeypatch.setattr(_ffi, "_lib", proxy)
    return proxy


@pytest.mark.parametrize("mode", ["readout", "mean", "gru", "mlp"])
@pytest.mark.parametrize("training", [False, True])
def test_training_never_reaches_the_atomic_segment_reduce(counting_lib, mode, training):
    from tf2_gnn_b200.layers import GraphGlobalExchangeInput, NodesToGraphRepresentationInput
    rng = np.random.default_rng(17)
    H, K = 32, 4
    sizes = rng.integers(0, 30, size=20)
    n2g, G = n2g_of(sizes), len(sizes)
    x = dev(rng.uniform(-1, 1, (len(n2g), H)).astype(np.float32)).requires_grad_()
    if mode == "readout":
        layer = _make_readout(H, H, K, "softmax", _readout_weights(rng, H, H, K, "softmax", False), False)
        inp = NodesToGraphRepresentationInput(x, dev(n2g, torch.int32), G)
    else:
        layer = _make_exchange(mode, H, K, "softmax", mo.make_exchange_weights(mode, H, K, rng, "softmax"),
                               dropout_rate=0.2 if training else 0.0, seed=3)
        inp = GraphGlobalExchangeInput(x, dev(n2g, torch.int32), G)
    layer(inp, training=training).sum().backward()
    assert "tfgnn_b200_unsorted_segment_reduce" not in counting_lib.calls
    assert counting_lib.calls.get("tfgnn_b200_readout_bwd") == 1
    if mode != "readout":
        assert counting_lib.calls.get("tfgnn_b200_segment_sum_rows", 0) + counting_lib.calls.get(
            "tfgnn_b200_gru_gate_bwd_indexed", 0) >= 1


def test_gru_exchange_keeps_no_per_node_input_table():
    """Without dropout the GRU's input half lives per graph: the step's peak is lower than the literal path's by more than the
    [V, 3H] table that path keeps (it also keeps the [V, H] copies of the graph representations and their gradients)."""
    from tf2_gnn_b200.layers import GraphGlobalExchangeInput, differentiable
    rng = np.random.default_rng(18)
    n2g, x = _ppi_inputs(rng)
    H, K, G = PPI["H"], PPI["K"], 3
    V = len(n2g)
    ex = _make_exchange("gru", H, K, "softmax", mo.make_exchange_weights("gru", H, K, rng, "softmax"))
    n2g_t = dev(n2g, torch.int32)

    def peak(step):
        for v in ex.variables:
            v.value.grad = None
        xt = dev(x).requires_grad_()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        step(xt).sum().backward()
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base

    def literal(xt):
        per_node = differentiable.per_node_graph_representations(ex, xt, n2g_t, G, False)
        return differentiable.gru_cell(per_node, xt, ex._gru_kernel.value, ex._gru_recurrent_kernel.value, ex._gru_bias.value)

    new = peak(lambda xt: ex(GraphGlobalExchangeInput(xt, n2g_t, G), training=False))
    old = peak(literal)
    assert new + V * 3 * H * 4 <= old, (new, old)
