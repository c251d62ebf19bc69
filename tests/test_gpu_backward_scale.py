"""Layer gradients at BASELINE sizes against the float64 reference of reference64.py (whole tables, no sampling).

Exact-arithmetic cases: RGCN-style layer, sum aggregation, no normalisation, relu, and h, W, grad_out with entries in
{-1, 0, 1}.  Every intermediate (gathered rows, Z, out, dZ, dW, dA, grad_h, the target-state coefficients) is then an
integer.  The tf32 hi part of an integer of magnitude <= 2048 is the integer itself and its lo part is 0, so the
correction products of both 3xTF32 schemes (bf16 pair in the fused kernel, two tf32 MMAs in the GEMM) add exactly 0, and
fp32 sums of integers are exact in any order while every partial sum stays below 2^24.  So the GPU result must equal
float32(reference) exactly.  The test proves the premises first, from the abs-value evaluation of the same products
(max |A| <= 2048; |S||h||W|, (|S||h|)^T |dZ| and |S|^T (|dZ||W|^T) below 2^24 everywhere), and only then compares.

Tolerance cases cover what cannot be exact (mean / sqrt_n, normalisation, tanh / gelu, the GRU): the norm-wise bars of
test_gpu_parity.py, plus a per-row bar on the largest-degree rows, whose error a norm-wise bar over the whole table can
hide.
"""
import os
import resource
import sys
import time

import numpy as np
import pytest

torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import reference64 as r64  # noqa: E402
from oracle import message_passing_oracle as mo  # noqa: E402

pytestmark = pytest.mark.gpu

TWO24 = float(2 ** 24)
OUT_TOL, GRAD_TOL, ROW_TOL = 1e-5, 2e-5, 1e-4


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def source_hub_graph(seed, V=1_000_000, E=5_000_000, L=3):
    """Out-degrees ~ Zipf(2.1) capped at 1e5 (the same weights for every type, so hubs add up over types), uniform
    targets: the source-keyed CSR of the dh reduce holds segments of ~1e5 edges."""
    rng = np.random.default_rng(seed)
    deg = np.minimum(rng.zipf(2.1, size=V), 100_000).astype(np.float64)
    p = deg / deg.sum()
    return [np.stack([rng.choice(V, size=E, p=p).astype(np.int32), rng.integers(0, V, size=E, dtype=np.int32)], axis=1)
            for _ in range(L)]


def exact_workload(name):
    """(V, D, H, adjs, use_target, fraction of non-zero weights)"""
    import bench
    if name == "source_hub":
        return 1_000_000, 128, 128, source_hub_graph(11), False, 1.0 / 32
    if name == "target_state":
        rng = np.random.default_rng(12)
        V = 200_000
        return V, 128, 128, [rng.integers(0, V, size=(2_000_000, 2), dtype=np.int32) for _ in range(2)], True, 1.0
    wl = bench.WORKLOADS[name]
    _, adjs, _ = bench.make_inputs(wl, seed=0)   # the benchmark's graph; its node states and weights are replaced
    return wl["V"], wl["H"], wl["H"], adjs, False, 1.0


def ternary(rng, shape, density=1.0):
    """Entries in {-1, 0, 1}; with density < 1 only that fraction is non-zero."""
    x = rng.choice(np.array([-1.0, 1.0], np.float32), size=shape)
    keep = rng.random(shape) < (2.0 / 3.0 if density >= 1.0 else density)
    return np.where(keep, x, 0.0).astype(np.float32)


def rgcn_on_gpu(V, D, H, adjs, h, Ws, g, agg="sum", act="relu", normalize=False, use_target=False, path="auto"):
    """out, grad_h, [grad_W] of the RGCN layer through its autograd hook, and whether a second backward gave the same
    bits."""
    from tf2_gnn_b200.layers import MessagePassingInput, RGCN
    from tf2_gnn_b200.runtime import PreparedBatch
    p = RGCN.get_default_hyperparameters()
    p.update(hidden_dim=H, aggregation_function=agg, message_activation_function=act, normalize_by_num_incoming=normalize,
             use_target_state_as_input=use_target, b200_path=path)
    layer = RGCN(p)
    layer.build(MessagePassingInput((None, D), tuple((None, 2) for _ in range(len(adjs)))))
    layer.set_weights_from_oracle_dict({"edge_mlps": [[w] for w in Ws]})
    weights = [v.value.requires_grad_() for v in layer.variables]
    adj_dev = tuple(torch.from_numpy(a).cuda() for a in adjs)
    ht = torch.from_numpy(h).cuda().requires_grad_()
    out = layer(MessagePassingInput(ht, adj_dev), prepared=PreparedBatch(adj_dev, V), training=True)
    gt = torch.from_numpy(g).cuda()
    first = torch.autograd.grad(out, [ht] + weights, gt, retain_graph=True)
    second = torch.autograd.grad(out, [ht] + weights, gt)
    same = all(torch.equal(a, b) for a, b in zip(first, second))
    res = (out.detach().cpu(), first[0].cpu(), [x.cpu() for x in first[1:]], same)
    del out, first, second, ht, layer
    torch.cuda.empty_cache()
    return res


@pytest.mark.parametrize("name", ["cfg2", "h320", "cfg1", "source_hub", "target_state"])
def test_rgcn_backward_exact_at_scale(name):
    _need_gpu()
    t0 = time.time()
    V, D, H, adjs, use_target, density = exact_workload(name)
    L = len(adjs)
    rng = np.random.default_rng(5)
    h = ternary(rng, (V, D))
    Ws = [ternary(rng, (2 * D if use_target else D, H), density) for _ in range(L)]
    g = ternary(rng, (V, H))
    graph = r64.Graph(adjs, V)
    bound = r64.rgcn_layer(h, adjs, Ws, g, use_target=use_target, absval=True, graph=graph)
    b_a, b_fwd = bound["max_abs_A"], float(bound["out"].max())
    b_dh, b_dw = float(bound["grad_h"].max()), max(float(x.max()) for x in bound["grad_W"])
    del bound
    assert b_a <= 2048, f"max |A| = {b_a:g}: the tf32 split of A is not exact"
    assert max(b_fwd, b_dh, b_dw) < TWO24, f"partial sums may exceed 2^24: fwd {b_fwd:g}, dW {b_dw:g}, dh {b_dh:g}"
    ref = r64.rgcn_layer(h, adjs, Ws, g, use_target=use_target, graph=graph)
    t_ref = time.time() - t0
    out, grad_h, grad_W, same = rgcn_on_gpu(V, D, H, adjs, h, Ws, g, use_target=use_target)
    assert same, "a second backward gave different bits"
    assert torch.equal(out, ref["out"].float()), f"out differs in {int((out != ref['out'].float()).sum())} elements"
    diff = grad_h != ref["grad_h"].float()
    assert not bool(diff.any()), (f"grad_h differs in {int(diff.sum())} elements over {int(diff.any(1).sum())} rows, "
                                  f"max |err| {float((grad_h.double() - ref['grad_h']).abs().max()):g}")
    for l in range(L):
        assert tuple(grad_W[l].shape) == tuple(Ws[l].shape)
        assert torch.equal(grad_W[l], ref["grad_W"][l].float()), f"grad_W[{l}] differs"
    idle = (graph.out_degree == 0) & ((graph.in_degree == 0) if use_target else True)
    assert bool((grad_h[idle] == 0).all())
    if name == "source_hub":
        assert int(idle.sum()) > 0 and int(graph.out_degree.max()) > 50_000
    print(f"{name}: exact; bounds max|A| {b_a:g}, fwd {b_fwd:g}, dW {b_dw:g}, dh {b_dh:g} (< 2^24 = {TWO24:g}); "
          f"max out-degree {int(graph.out_degree.max())}; reference {t_ref:.0f} s, total {time.time() - t0:.0f} s, "
          f"host peak RSS {resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2 ** 20:.1f} GiB")


def rel_err(got, ref):
    got, ref = got.double(), ref.double()
    return float((got - ref).abs().max()) / max(float(ref.abs().max()), 1e-30)


def worst_row_ratio(got, ref, rows):
    """max over `rows` of max|err| in the row / max|ref| in the row."""
    got, ref = got[rows].double(), ref[rows].double()
    return float(((got - ref).abs().amax(1) / ref.abs().amax(1).clamp(min=1e-30)).max())


def check_tolerances(name, out, grad_h, grad_W, ref, graph, extra=()):
    top_in = torch.argsort(graph.in_degree)[-8:]
    top_out = torch.argsort(graph.out_degree)[-8:]
    r = {"out": rel_err(out, ref["out"]), "grad_h": rel_err(grad_h, ref["grad_h"]),
         "grad_W": max(rel_err(a, b) for a, b in zip(grad_W, ref["grad_W"])),
         "out_hub_rows": worst_row_ratio(out, ref["out"], top_in),
         "grad_h_hub_rows": worst_row_ratio(grad_h, ref["grad_h"], top_out)}
    for key, got in extra:
        r[key] = rel_err(got, ref[key])
    print(f"{name}: " + ", ".join(f"{k} {v:.2e}" for k, v in r.items()))
    assert r["out"] <= OUT_TOL
    for k, v in r.items():
        if k.endswith("hub_rows"):
            assert v <= ROW_TOL, f"{k}: {v:.3e} > {ROW_TOL:g}"
        elif k != "out":
            assert v <= GRAD_TOL, f"{k}: {v:.3e} > {GRAD_TOL:g}"


@pytest.mark.parametrize("name,agg,act,normalize", [("cfg2", "mean", "tanh", True), ("h320", "sqrt_n", "gelu", False)])
def test_rgcn_backward_tolerance_at_scale(name, agg, act, normalize):
    _need_gpu()
    V, D, H, adjs, _, _ = exact_workload(name)
    L = len(adjs)
    rng = np.random.default_rng(6)
    h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    Ws = [mo.glorot_uniform(rng, (D, H)) for _ in range(L)]
    g = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    out, grad_h, grad_W, same = rgcn_on_gpu(V, D, H, adjs, h, Ws, g, agg=agg, act=act, normalize=normalize)
    assert same, "a second backward gave different bits"
    graph = r64.Graph(adjs, V)
    ref = r64.rgcn_layer(h, adjs, Ws, g, agg=agg, act=act, normalize=normalize, graph=graph)
    check_tolerances(f"{name} {agg} {act} normalize={normalize}", out, grad_h, grad_W, ref, graph)


def test_ggnn_backward_tolerance_at_scale():
    """cfg4 (GGNN, 500k nodes, 5 types) with the fused-GRU forward."""
    _need_gpu()
    import bench
    from tf2_gnn_b200.layers import GGNN, MessagePassingInput
    from tf2_gnn_b200.runtime import PreparedBatch
    wl = bench.WORKLOADS["cfg4"]
    V, H = wl["V"], wl["H"]
    _, adjs, _ = bench.make_inputs(wl, seed=0)
    L = len(adjs)
    rng = np.random.default_rng(8)
    h = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    Ws = [mo.glorot_uniform(rng, (H, H)) for _ in range(L)]
    K, U = mo.glorot_uniform(rng, (H, 3 * H)), mo.glorot_uniform(rng, (H, 3 * H))
    b = rng.uniform(-0.2, 0.2, (2, 3 * H)).astype(np.float32)
    g = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    p = GGNN.get_default_hyperparameters()
    p.update(hidden_dim=H)
    layer = GGNN(p)
    layer.build(MessagePassingInput((None, H), tuple((None, 2) for _ in range(L))))
    layer.set_weights_from_oracle_dict({"edge_mlps": [[w] for w in Ws], "gru_kernel": K, "gru_recurrent_kernel": U,
                                        "gru_bias": b})
    by_name = {v.name: v.value for v in layer.variables}
    pick = lambda suffix: [t for n, t in by_name.items() if n.endswith(suffix)][0]   # noqa: E731
    weights = [m.layers[0].value for m in layer._edge_type_mlps] + [pick("gru_cell/kernel:0"),
                                                                    pick("gru_cell/recurrent_kernel:0"),
                                                                    pick("gru_cell/bias:0")]
    for t in weights:
        t.requires_grad_()
    adj_dev = tuple(torch.from_numpy(a).cuda() for a in adjs)
    ht = torch.from_numpy(h).cuda().requires_grad_()
    out = layer(MessagePassingInput(ht, adj_dev), prepared=PreparedBatch(adj_dev, V), training=True)
    gt = torch.from_numpy(g).cuda()
    first = torch.autograd.grad(out, [ht] + weights, gt, retain_graph=True)
    second = torch.autograd.grad(out, [ht] + weights, gt)
    assert all(torch.equal(x, y) for x, y in zip(first, second)), "a second backward gave different bits"
    first = [x.cpu() for x in first]
    graph = r64.Graph(adjs, V)
    ref = r64.ggnn_layer(h, adjs, Ws, K, U, b, g, agg=p["aggregation_function"],
                         normalize=p["normalize_by_num_incoming"], graph=graph)
    check_tolerances("cfg4 ggnn", out.detach().cpu(), first[0], first[1:1 + L], ref, graph,
                     extra=(("grad_K", first[1 + L]), ("grad_U", first[2 + L]), ("grad_b", first[3 + L])))
