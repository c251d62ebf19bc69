"""Training of edge MLPs with one hidden layer (GNN_Edge_MLP and RGIN defaults) through tfgnn_b200_edge_mlp_bwd (hoisted
hidden layer, no per-edge tensors), and of RGIN through the fused backward in general: gradients of the node states and
every kernel against float64 references, exactly on integer data at scale, against the literal per-edge path, on
target-range shards, through a GNN stack, and one cfg2-sized training step.

The hidden ReLU's derivative flips when a pre-activation P_e lies within rounding of 0, which no tolerance can absorb.
So every tolerance case either puts h and U on a dyadic grid on which every P_e is exact in fp32 and in 3xTF32 (the GPU's
mask is then the float64 mask; `_prove_exact_hidden` shows it from the bounds), or asserts a float64 margin
min |P_e| >= 1e-5 * scale (stacked layers, whose inputs are not on a grid)."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

import reference64_edge_mlp as rm  # noqa: E402
from oracle import message_passing_oracle as mo  # noqa: E402
from reference64 import Graph  # noqa: E402
from test_gpu_backward_scale import source_hub_graph, ternary  # noqa: E402
from test_gpu_parity import _need_gpu, assert_states_close, make_layer, random_graph  # noqa: E402
from test_gpu_shard_backward import _check_shards  # noqa: E402

pytestmark = pytest.mark.gpu

TOL = 3e-5   # the norm-wise bar of the FiLM backward tests
FUSED = "_EdgeMLPLayerFunctionBackward"
GRID = 64    # h and U are multiples of 1/GRID in [-1, 1]


def dyadic(rng, shape):
    return (rng.integers(-GRID, GRID + 1, size=shape) / GRID).astype(np.float32)


def _prove_exact_hidden(h, Us):
    """h and U on the 1/64 grid in [-1, 1]: every product h_d U_dc is a multiple of 2^-12 of magnitude <= 1, so every partial
    sum of P_e = sum_d h_u,d U^s_dc + sum_d h_v,d U^t_dc is a multiple of 2^-12 of magnitude <= D_in < 2^12 and needs at most
    24 significant bits: exact in fp32, in any order.  Each operand has at most 7 significant bits, so 3xTF32 splits it
    with a zero low part and its products are exact too.  The GPU's mask [P_e > 0] therefore equals the float64 mask."""
    for x in (h, *Us):
        assert np.all(np.abs(x) <= 1.0) and np.array_equal(x * GRID, np.round(x * GRID))
    D_in = max(u.shape[0] for u in Us)
    assert D_in * GRID * GRID < 2 ** 24


def _weights(kind, D, H, L, rng, use_target, n_edge_hidden=1, n_aggr=None):
    """{"edge_mlps": [[U, W2] or [W]], "aggr_mlp": [...] or None}: U dyadic, every other kernel a random float."""
    d_in = (2 if use_target else 1) * D
    if n_edge_hidden == 1:
        edge = [[dyadic(rng, (d_in, H)), mo.glorot_uniform(rng, (H, H))] for _ in range(L)]
    else:
        edge = [[mo.glorot_uniform(rng, (d_in, H))] for _ in range(L)]
    w = {"edge_mlps": edge}
    if kind == "rgin":
        w["aggr_mlp"] = None if n_aggr is None else [mo.glorot_uniform(rng, (H, H)) for _ in range(n_aggr + 1)]
    return w


def _layer(kind, D, H, L, weights, **hyper):
    p = mo.default_hyperparameters(kind)
    p.update(hidden_dim=H, **hyper)
    layer = make_layer(kind, p, D, L, weights)
    for v in layer.variables:
        v.requires_grad_()
    return layer, p


def _params(layer):
    out = [v for m in layer._edge_type_mlps for v in m.layers]
    return out + list(getattr(layer, "_aggregation_mlp", None) or [])


def _uses_fused(out):
    seen, todo = set(), [out.grad_fn]
    while todo:
        f = todo.pop()
        if f is None or f in seen:
            continue
        seen.add(f)
        if type(f).__name__ == FUSED:
            return True
        todo.extend(n for n, _ in f.next_functions)
    return False


def _run(layer, h, adjs, g, prepared=None):
    """(out, grad_h, [grad of every kernel]) of one fused forward + backward."""
    from tf2_gnn_b200.layers import MessagePassingInput
    ht = torch.from_numpy(h).cuda().requires_grad_()
    for p in _params(layer):
        p.value.grad = None
    out = layer(MessagePassingInput(ht, tuple(torch.from_numpy(a).cuda() for a in adjs)), prepared=prepared)
    assert _uses_fused(out)
    out.backward(torch.from_numpy(g).cuda())
    torch.cuda.synchronize()
    return out.detach().cpu().numpy(), ht.grad.cpu().numpy(), [p.value.grad.cpu().numpy() for p in _params(layer)]


def _autograd64(h, adjs, w, g, p, n_edge_hidden=1):
    h64 = torch.from_numpy(h).double().requires_grad_()
    U64 = [torch.from_numpy(m[0]).double().requires_grad_() for m in w["edge_mlps"]]
    W64 = [torch.from_numpy(m[1]).double().requires_grad_() for m in w["edge_mlps"]] if n_edge_hidden else None
    M64 = [torch.from_numpy(m).double().requires_grad_() for m in (w.get("aggr_mlp") or [])]
    out = rm.edge_mlp_autograd(h64, [torch.from_numpy(a) for a in adjs], U64, W64, agg=p["aggregation_function"],
                               act=p["message_activation_function"], normalize=p["normalize_by_num_incoming"],
                               use_target=p["use_target_state_as_input"], aggr_ws=M64)
    out.backward(torch.from_numpy(g).double())
    leaves = [x for pair in zip(U64, W64) for x in pair] if W64 else U64
    return out.detach().numpy(), h64.grad.numpy(), [x.grad.numpy() for x in leaves + M64]


def _close_all(got, ref, tol=TOL):
    (o, gh, gw), (ro, rgh, rgw) = got, ref
    assert_states_close(o, ro, tol=tol)
    assert_states_close(gh, rgh, tol=tol)
    assert len(gw) == len(rgw)
    for a, b in zip(gw, rgw):
        assert_states_close(a, b, tol=tol)


def _same_bits(a, b):
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert all(np.array_equal(x, y) for x, y in zip(a[2], b[2]))


def _aggr_margin(h, adjs, w, p):
    """float64 margin of the aggregation MLP's hidden ReLUs (their inputs are not on a grid)."""
    if not w.get("aggr_mlp") or len(w["aggr_mlp"]) < 2:
        return
    ref = rm.edge_mlp_layer(h, adjs, [m[0] for m in w["edge_mlps"]], [m[1] for m in w["edge_mlps"]],
                            agg=p["aggregation_function"], act=p["message_activation_function"],
                            normalize=p["normalize_by_num_incoming"], use_target=p["use_target_state_as_input"],
                            aggr_ws=w["aggr_mlp"])
    assert ref["min_abs_aggr_pre"] >= 1e-5 * float(np.abs(ref["out"].numpy()).max()), ref["min_abs_aggr_pre"]


# Smooth output activations only (DESIGN.md §5); relu output is covered by the exact tests.
@pytest.mark.parametrize("kind,V,D,H,L,E,agg,act,normalize,use_target,empty,hub,n_aggr", [
    ("gnn_edge_mlp", 600, 32, 36, 3, 4000, "sum", "tanh", False, True, None, False, None),
    ("gnn_edge_mlp", 600, 32, 36, 3, 4000, "mean", "gelu", True, False, 1, True, None),
    ("gnn_edge_mlp", 800, 64, 96, 4, 5000, "sqrt_n", "elu", False, True, 2, True, None),
    ("gnn_edge_mlp", 800, 64, 96, 4, 5000, "sum", "elu", True, True, None, True, None),
    ("gnn_edge_mlp", 500, 320, 320, 2, 3000, "mean", "tanh", True, True, None, True, None),
    # unnormalised: a hub's relu sum stays below 2^12, where fp32 sums of these dyadic values are still exact (a
    # 3000-edge hub rounds, and every rounding is a tie: 1e-2 on a sum of 6000, 6e-5 of the dW2 scale)
    ("gnn_edge_mlp", 1500, 64, 64, 7, 2000, "sqrt_n", "gelu", False, True, 3, True, None),
    ("gnn_edge_mlp", 900, 32, 480, 1, 3000, "mean", "tanh", True, False, None, True, None),
    ("rgin", 700, 48, 32, 5, 4000, "mean", "elu", False, False, 0, True, None),
    ("rgin", 700, 48, 32, 3, 4000, "sum", "tanh", False, False, None, False, 0),
    ("rgin", 740, 32, 64, 3, 4000, "sqrt_n", "gelu", True, False, 1, False, 1),
    ("rgin", 600, 32, 32, 2, 3000, "mean", "tanh", False, True, None, True, 2),
])
def test_edge_mlp_backward_matches_float64_autograd(kind, V, D, H, L, E, agg, act, normalize, use_target, empty, hub,
                                                    n_aggr):
    _need_gpu()
    rng = np.random.default_rng(V + D + H + L + (n_aggr or 0))
    adjs = random_graph(rng, V, L, E, empty_type=empty, hub=hub, dups=True, self_loops=True)
    w = _weights(kind, D, H, L, rng, use_target, n_aggr=n_aggr)
    layer, p = _layer(kind, D, H, L, w, aggregation_function=agg, message_activation_function=act,
                      normalize_by_num_incoming=normalize, use_target_state_as_input=use_target,
                      **({"num_aggr_MLP_hidden_layers": n_aggr} if kind == "rgin" else {}))
    h = dyadic(rng, (V, D))
    g = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    _prove_exact_hidden(h, [m[0] for m in w["edge_mlps"]])
    _aggr_margin(h, adjs, w, p)
    got = _run(layer, h, adjs, g)
    _close_all(got, _autograd64(h, adjs, w, g, p))
    _same_bits(got, _run(layer, h, adjs, g))   # a second backward gives the same bits
    if empty is not None:
        assert not got[2][2 * empty].any() and not got[2][2 * empty + 1].any()


@pytest.mark.parametrize("n_aggr,agg,act", [(None, "sum", "tanh"), (0, "mean", "gelu"), (2, "sqrt_n", "elu")])
def test_rgin_without_edge_mlp_hidden_layer_trains_fused(n_aggr, agg, act):
    """RGIN with 0 hidden layers in its edge MLPs: tfgnn_b200_rgcn_bwd, then the aggregation MLP through node_ops.dense."""
    _need_gpu()
    rng = np.random.default_rng(41 + (n_aggr or 0))
    V, D, H, L = 700, 32, 48, 3
    # no hub under unnormalised sum: a plain fp32 sum of 2000 rows alone exceeds the bar (DESIGN.md §5)
    adjs = random_graph(rng, V, L, 4000, empty_type=1, hub=agg != "sum", dups=True)
    w = _weights("rgin", D, H, L, rng, False, n_edge_hidden=0, n_aggr=n_aggr)
    layer, p = _layer("rgin", D, H, L, w, aggregation_function=agg, message_activation_function=act,
                      num_edge_MLP_hidden_layers=0, num_aggr_MLP_hidden_layers=n_aggr)
    h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    g = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    got = _run(layer, h, adjs, g)
    _close_all(got, _autograd64(h, adjs, w, g, p, n_edge_hidden=0))
    _same_bits(got, _run(layer, h, adjs, g))


@pytest.mark.parametrize("kind,n_aggr,use_target", [("rgin", None, False), ("rgin", 1, False), ("gnn_edge_mlp", None, True),
                                                    ("rgin", 0, True)])
def test_training_output_equals_inference_output(kind, n_aggr, use_target):
    """The training forward is the inference forward: the same bits."""
    _need_gpu()
    from tf2_gnn_b200.layers import MessagePassingInput
    rng = np.random.default_rng(3 + (n_aggr or 0))
    V, D, H, L = 2000, 64, 64, 3
    adjs = random_graph(rng, V, L, 12000, hub=True, dups=True)
    w = _weights(kind, D, H, L, rng, use_target, n_aggr=n_aggr)
    layer, _ = _layer(kind, D, H, L, w, use_target_state_as_input=use_target, aggregation_function="mean",
                      **({"num_aggr_MLP_hidden_layers": n_aggr} if kind == "rgin" else {}))
    ht = torch.from_numpy(rng.uniform(-1, 1, (V, D)).astype(np.float32)).cuda()
    adj_dev = tuple(torch.from_numpy(a).cuda() for a in adjs)
    with torch.no_grad():
        inf = layer(MessagePassingInput(ht, adj_dev))
    train = layer(MessagePassingInput(ht.clone().requires_grad_(), adj_dev))
    assert _uses_fused(train)
    assert torch.equal(inf, train.detach())


# ---- exact at scale ----------------------------------------------------------------------------------------------------
def exact_case(name):
    """(kind, V, D, H, adjs, use_target, densities of h / U / W2 / grad_out)."""
    import bench
    if name == "cfg2_rgin":
        wl = bench.WORKLOADS["cfg2"]
        _, adjs, _ = bench.make_inputs(wl, seed=0)   # the benchmark's graph; states and weights are replaced
        return "rgin", wl["V"], wl["H"], wl["H"], adjs, False, (1 / 8, 1 / 8, 1 / 8, 1 / 16)
    if name == "target_state":
        rng = np.random.default_rng(12)
        V = 200_000
        return ("gnn_edge_mlp", V, 128, 128, [rng.integers(0, V, size=(2_000_000, 2), dtype=np.int32) for _ in range(2)],
                True, (1 / 4, 1 / 4, 1 / 8, 1 / 8))
    if name == "source_hub":   # ~1e5-edge segments in the source-keyed kernel
        return "gnn_edge_mlp", 1_000_000, 128, 128, source_hub_graph(11), True, (1 / 8, 1 / 8, 1 / 32, 1 / 2048)
    raise ValueError(name)


def exact_inputs(name, seed=0):
    kind, V, D, H, adjs, use_target, (dh, du, dw, dg) = exact_case(name)
    rng = np.random.default_rng(seed)
    L = len(adjs)
    h = ternary(rng, (V, D), dh)
    g = ternary(rng, (V, H), dg)
    Us = [ternary(rng, ((2 if use_target else 1) * D, H), du) for _ in range(L)]
    W2s = [ternary(rng, (H, H), dw) for _ in range(L)]
    return kind, V, D, H, adjs, use_target, h, g, Us, W2s


def exact_bounds(name):
    """The abs-value run of the reference for an exact case: (operand_max, partial_max)."""
    kind, V, D, H, adjs, use_target, h, g, Us, W2s = exact_inputs(name)
    b = rm.edge_mlp_layer(h, adjs, Us, W2s, g, use_target=use_target, absval=True, graph=Graph(adjs, V))
    return b["operand_max"], b["partial_max"]


@pytest.mark.parametrize("name", ["cfg2_rgin", "target_state", "source_hub"])
def test_edge_mlp_backward_exact_at_scale(name, trimmed_pool):
    """sum / relu / no normalisation with sparse ternary h, U, W2 and grad_out.  Once the abs-value run shows every
    tensor-core operand <= 2048 (exact in 3xTF32) and every partial sum < 2^24, out, grad_h and every weight gradient must
    equal float32(reference) bit for bit."""
    kind, V, D, H, adjs, use_target, h, g, Us, W2s = exact_inputs(name)
    L = len(adjs)
    graph = Graph(adjs, V)
    bound = rm.edge_mlp_layer(h, adjs, Us, W2s, g, use_target=use_target, absval=True, graph=graph)
    assert bound["operand_max"] <= 2048, bound["operand_max"]
    assert bound["partial_max"] < 2 ** 24, bound["partial_max"]
    del bound
    w = {"edge_mlps": [[u, w2] for u, w2 in zip(Us, W2s)], "aggr_mlp": None}
    layer, _ = _layer(kind, D, H, L, w, aggregation_function="sum", message_activation_function="relu",
                      normalize_by_num_incoming=False, use_target_state_as_input=use_target)
    got = _run(layer, h, adjs, g)
    _same_bits(got, _run(layer, h, adjs, g))
    torch.cuda.empty_cache()
    ref = rm.edge_mlp_layer(h, adjs, Us, W2s, g, act="relu", use_target=use_target, graph=graph)
    out, gh, gw = got
    f32 = lambda t: t.numpy().astype(np.float32)
    assert np.array_equal(out, f32(ref["out"]))
    assert np.array_equal(gh, f32(ref["grad_h"]))
    refs = [x for pair in zip(ref["grad_U"], ref["grad_W2"]) for x in pair]
    assert len(gw) == len(refs)
    for i, (a, b) in enumerate(zip(gw, refs)):
        assert np.array_equal(a, f32(b)), i
    assert np.abs(gh).max() > 0 and all(np.abs(a).max() > 0 for a in gw)


# ---- the literal path: still the path of everything else ---------------------------------------------------------------
@pytest.mark.parametrize("kind,agg,act,normalize,use_target,n_aggr", [
    ("gnn_edge_mlp", "sum", "tanh", True, True, None), ("gnn_edge_mlp", "mean", "gelu", False, False, None),
    ("rgin", "sqrt_n", "elu", False, False, 1)])
def test_fused_and_literal_paths_agree_with_float64(kind, agg, act, normalize, use_target, n_aggr):
    """The literal per-edge path (layers/differentiable.py), called directly, stays covered for the configurations that now
    train through the fused backward; both meet the same bar against float64 autograd."""
    _need_gpu()
    from tf2_gnn_b200.layers.differentiable import edge_mlp_family_forward
    from tf2_gnn_b200.runtime import PreparedBatch
    rng = np.random.default_rng(31 + len(agg))
    V, D, H, L = 900, 32, 48, 3
    adjs = random_graph(rng, V, L, 6000, empty_type=2, hub=True, dups=True)
    w = _weights(kind, D, H, L, rng, use_target, n_aggr=n_aggr)
    layer, p = _layer(kind, D, H, L, w, aggregation_function=agg, message_activation_function=act,
                      normalize_by_num_incoming=normalize, use_target_state_as_input=use_target,
                      **({"num_aggr_MLP_hidden_layers": n_aggr} if kind == "rgin" else {}))
    h = dyadic(rng, (V, D))
    g = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    _prove_exact_hidden(h, [m[0] for m in w["edge_mlps"]])
    ref = _autograd64(h, adjs, w, g, p)
    _close_all(_run(layer, h, adjs, g), ref)
    ht = torch.from_numpy(h).cuda().requires_grad_()
    adj_dev = tuple(torch.from_numpy(a).cuda() for a in adjs)
    for q in _params(layer):
        q.value.grad = None
    aggr = [v.value for v in layer._aggregation_mlp] if kind == "rgin" and layer._aggregation_mlp else None
    out = edge_mlp_family_forward(layer, ht, PreparedBatch(adj_dev, V), activation_before=False, aggr_kernels=aggr)
    assert not _uses_fused(out)
    out.backward(torch.from_numpy(g).cuda())
    _close_all((out.detach().cpu().numpy(), ht.grad.cpu().numpy(), [q.value.grad.cpu().numpy() for q in _params(layer)]),
               ref)


@pytest.mark.parametrize("kind,extra,D", [
    ("gnn_edge_mlp", dict(num_edge_MLP_hidden_layers=2), 32),
    ("rgin", dict(num_edge_MLP_hidden_layers=2), 32),
    ("gnn_edge_mlp", dict(aggregation_function="max"), 32),
    ("rgin", dict(aggregation_function="max"), 32),
    ("gnn_edge_mlp", dict(message_activation_before_aggregation=True, message_activation_function="tanh"), 32),
    ("gnn_edge_mlp", {}, 30),
    ("rgin", {}, 30),
])
def test_configurations_outside_the_fused_backward_keep_the_literal_path(kind, extra, D):
    _need_gpu()
    from tf2_gnn_b200.layers import MessagePassingInput
    from tf2_gnn_b200.runtime import PreparedBatch
    rng = np.random.default_rng(5)
    V, H, L = 400, 32, 2
    adjs = random_graph(rng, V, L, 2000)
    p = mo.default_hyperparameters(kind)
    p.update(hidden_dim=H, **extra)
    layer = make_layer(kind, p, D, L, mo.make_weights(kind, p, D, L, rng))
    for v in layer.variables:
        v.requires_grad_()
    ht = torch.from_numpy(rng.uniform(-1, 1, (V, D)).astype(np.float32)).cuda().requires_grad_()
    adj_dev = tuple(torch.from_numpy(a).cuda() for a in adjs)
    out = layer(MessagePassingInput(ht, adj_dev))
    assert not _uses_fused(out)
    out.sum().backward()
    assert torch.isfinite(ht.grad).all()
    with pytest.raises(NotImplementedError, match="target-range shard"):
        layer(MessagePassingInput(ht, adj_dev), prepared=PreparedBatch(adj_dev, V, target_range=(0, V // 2)))


# ---- shards ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,D,H,agg,act,normalize,use_target,n_aggr", [
    ("gnn_edge_mlp", 64, 64, "mean", "tanh", True, True, None),
    ("gnn_edge_mlp", 32, 48, "sum", "gelu", True, False, None),
    ("gnn_edge_mlp", 64, 32, "sqrt_n", "elu", False, True, None),
    ("rgin", 32, 36, "mean", "tanh", False, False, 1),
])
def test_edge_mlp_shard_backward_sums_to_full(kind, D, H, agg, act, normalize, use_target, n_aggr):
    """Worlds of 2 and 3 and a world with an empty shard (test_gpu_shard_backward._check_shards)."""
    _need_gpu()
    V, L = 700, 3
    rng = np.random.default_rng(D + H + 7)
    adjs = random_graph(rng, V, L, 5000, hub=True, dups=True, self_loops=use_target)
    w = _weights(kind, D, H, L, rng, use_target, n_aggr=n_aggr)
    layer, p = _layer(kind, D, H, L, w, aggregation_function=agg, message_activation_function=act,
                      normalize_by_num_incoming=normalize, use_target_state_as_input=use_target,
                      **({"num_aggr_MLP_hidden_layers": n_aggr} if kind == "rgin" else {}))
    h = dyadic(rng, (V, D))
    g = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    _prove_exact_hidden(h, [m[0] for m in w["edge_mlps"]])
    _, ref_h, ref_w = _autograd64(h, adjs, w, g, p)
    _check_shards(layer, _params(layer), h, adjs, g, (ref_h, ref_w))


# ---- a PPI_RGIN-shaped stack -------------------------------------------------------------------------------------------
def _rgin_stack_reference(params, w, feats, adjs, dtype=torch.float64):
    """torch restatement of gnn.py:276-329 for an RGIN stack with inter-layer LayerNorm, without exchange or dropout
    (differentiable); also returns min |P_e| / scale over every hidden ReLU of every layer (float64)."""
    t = lambda a: torch.from_numpy(np.asarray(a)).to(dtype).requires_grad_()
    leaves = {"proj": t(w["initial_projection"]),
              "U": [[t(m[0]) for m in wi["edge_mlps"]] for wi in w["mp"]],
              "W2": [[t(m[1]) for m in wi["edge_mlps"]] for wi in w["mp"]],
              "ln": [(t(g), t(b)) for g, b in w["layernorm"]],
              "dense": {i: t(d) for i, d in w["dense"].items()}}
    acts = {"tanh": torch.tanh, "relu": torch.relu, "gelu": lambda x: rm.act_and_grad(x, "gelu")[0]}
    cur = acts[params["initial_node_representation_activation"]](torch.from_numpy(feats).to(dtype) @ leaves["proj"])
    last = cur
    margin = float("inf")
    for i in range(params["num_layers"]):
        if i % params["residual_every_num_layers"] == 0:
            tmp = cur
            if i > 0:
                cur = (cur + last) / 2
            last = tmp
        if dtype == torch.float64:
            with torch.no_grad():
                ref = rm.edge_mlp_layer(cur, adjs, leaves["U"][i], leaves["W2"][i], agg=params["aggregation_function"],
                                        act=params["message_activation_function"],
                                        normalize=params["normalize_by_num_incoming"],
                                        use_target=params["use_target_state_as_input"])
                scale = max(float((cur.abs() @ leaves["U"][i][0].abs()).max()), 1e-30)
                margin = min(margin, ref["min_abs_P"] / scale)
        cur = rm.edge_mlp_autograd(cur, adjs, leaves["U"][i], leaves["W2"][i], agg=params["aggregation_function"],
                                   act=params["message_activation_function"],
                                   normalize=params["normalize_by_num_incoming"],
                                   use_target=params["use_target_state_as_input"])
        g_, b_ = leaves["ln"][i]
        mu = cur.mean(dim=1, keepdim=True)
        var = ((cur - mu) ** 2).mean(dim=1, keepdim=True)
        cur = (cur - mu) / torch.sqrt(var + 1e-3) * g_ + b_
        if i % params["dense_every_num_layers"] == 0:
            cur = acts[params["dense_intermediate_layer_activation"]](cur @ leaves["dense"][i])
    return cur, leaves, margin


def test_training_step_of_a_ppi_rgin_stack_matches_float64_autograd():
    """PPI_RGIN.json-shaped: 5 RGIN layers (one hidden layer, sum, relu-free smooth output), residual every 2 layers,
    inter-layer LayerNorm, dropout off; one SGD step's gradients against float64 autograd, with the hidden-ReLU margin
    asserted in float64."""
    _need_gpu()
    from tf2_gnn_b200.layers import GNN, GNNInput
    from test_gpu_graph_ops import _build_gnn
    # small enough that the float64 margin holds: over N (edge, column) pairs the expected number of |P_e| below
    # 1e-5 * scale grows like 3e-5 * N
    rng = np.random.default_rng(0)
    V, F, H, L = 100, 16, 16, 2
    params = GNN.get_default_hyperparameters("rgin")
    params.update(hidden_dim=H, num_layers=5, global_exchange_every_num_layers=10000, layer_input_dropout_rate=0.0,
                  dense_every_num_layers=10000, residual_every_num_layers=2, use_inter_layer_layernorm=True,
                  num_edge_MLP_hidden_layers=1, num_aggr_MLP_hidden_layers=None, message_activation_function="tanh",
                  aggregation_function="sum", use_target_state_as_input=False, normalize_by_num_incoming=True)
    adjs = [rng.integers(0, V, size=(150, 2)).astype(np.int32) for _ in range(L)]
    feats = rng.uniform(-1, 1, (V, F)).astype(np.float32)
    R = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    gnn, w = _build_gnn(params, F, L, rng, False)
    for v in gnn.variables:
        v.requires_grad_(True)
    inp = GNNInput(torch.from_numpy(feats).cuda(), tuple(torch.from_numpy(a).cuda() for a in adjs),
                   torch.zeros(V, dtype=torch.int32).cuda(), 1)
    out = gnn(inp, training=True)
    (out * torch.from_numpy(R).cuda()).sum().backward()
    refs = {}
    for dt in (torch.float64, torch.float32):
        ref_out, leaves, margin = _rgin_stack_reference(params, w, feats, adjs, dt)
        if dt == torch.float64:
            assert margin >= 1e-5, margin   # precondition (b): no hidden pre-activation within rounding of 0
        (ref_out * torch.from_numpy(R).to(dt)).sum().backward()
        refs[dt] = [ref_out.detach(), leaves["proj"].grad]
        for i in range(len(leaves["U"])):
            refs[dt] += [x.grad for pair in zip(leaves["U"][i], leaves["W2"][i]) for x in pair]
            refs[dt] += [leaves["ln"][i][0].grad, leaves["ln"][i][1].grad]
    got = [out.detach(), gnn._initial_projection_layer.kernel.grad]
    for i, mp in enumerate(gnn._mp_layers):
        got += [v.grad for m in mp._edge_type_mlps for v in m.layers]
        got += [gnn._inter_layer_layernorms[i].gamma.grad, gnn._inter_layer_layernorms[i].beta.grad]
    assert len(got) == len(refs[torch.float64]) and all(x is not None for x in got)
    # the FiLM stack test's bar: 1e-5 per stage of the chain relative to the scale, or within 3x of the fp32
    # restatement's own error
    tol = 1e-5 * (2 * params["num_layers"] + 2)
    for i, (x, r64, r32) in enumerate(zip(got, refs[torch.float64], refs[torch.float32])):
        x, r64, r32 = x.cpu().double().numpy(), r64.numpy(), r32.double().numpy()
        scale = max(np.abs(r64).max(), 1e-30)
        err, fp32_err = np.abs(x - r64).max(), np.abs(r32 - r64).max()
        assert err <= max(tol * scale, 3.0 * fp32_err), (i, err, fp32_err, scale)


# ---- cfg2 size ---------------------------------------------------------------------------------------------------------
@pytest.fixture
def trimmed_pool():
    """Start and leave a large case with the library's memory pool and torch's cache handed back to the driver."""
    import gc
    from tf2_gnn_b200 import _ffi
    from tf2_gnn_b200.runtime import clear_prepared_batch_cache
    _need_gpu()
    clear_prepared_batch_cache()
    gc.collect()
    torch.cuda.empty_cache()
    _ffi.lib().tfgnn_b200_release_device_state()
    yield
    clear_prepared_batch_cache()
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    _ffi.lib().tfgnn_b200_release_device_state()


@pytest.mark.parametrize("kind", ["rgin", "gnn_edge_mlp"])
def test_cfg2_training_step_fits_one_gpu_and_repeats_bitwise(kind, trimmed_pool, record_property, capsys):
    """bench.py's cfg2 graph (1M nodes, 4 types of 5M edges, D = H = 256): one training step of an RGIN layer with the
    PPI_RGIN hyper-parameters (one hidden layer, normalised, sum, relu) and of a GNN_Edge_MLP layer with its class
    defaults (target-state input) fits one 80 GB H100, is finite, and a second step gives the same bits."""
    from tf2_gnn_b200.layers import MessagePassingInput
    from tf2_gnn_b200.runtime import PreparedBatch
    V, D, L, E = 1_000_000, 256, 4, 5_000_000
    gen = torch.Generator(device="cuda")
    gen.manual_seed(7)
    adj = tuple(torch.randint(0, V, (E, 2), generator=gen, device="cuda", dtype=torch.int32) for _ in range(L))
    h = (torch.rand((V, D), generator=gen, device="cuda") * 2 - 1).requires_grad_()
    g = torch.rand((V, D), generator=gen, device="cuda") * 2 - 1
    rng = np.random.default_rng(7)
    p = mo.default_hyperparameters(kind)
    p.update(hidden_dim=D)
    if kind == "rgin":
        p.update(normalize_by_num_incoming=True, aggregation_function="sum", message_activation_function="relu")
    layer = make_layer(kind, p, D, L, mo.make_weights(kind, p, D, L, rng))
    for v in layer.variables:
        v.requires_grad_()
    prepared = PreparedBatch(adj, V)
    runs = []
    torch.cuda.reset_peak_memory_stats()
    for _ in range(2):
        h.grad = None
        for q in _params(layer):
            q.value.grad = None
        out = layer(MessagePassingInput(h, adj), prepared=prepared)
        assert _uses_fused(out)
        out.backward(g)
        torch.cuda.synchronize()
        runs.append((h.grad.cpu(), [q.value.grad.cpu() for q in _params(layer)]))
        del out
    free, total = torch.cuda.mem_get_info()
    used = (total - free) / 1e9
    record_property("device_memory_in_use_GB", round(used, 2))
    with capsys.disabled():
        print(f"\n[{kind} cfg2 step] device memory in use {used:.1f} GB "
              f"(torch peak {torch.cuda.max_memory_allocated() / 1e9:.1f} GB)")
    del prepared, adj, h, g
    assert used < 80
    (h1, w1), (h2, w2) = runs
    assert torch.isfinite(h1).all() and all(torch.isfinite(x).all() for x in w1)
    assert h1.abs().max() > 0
    assert torch.equal(h1, h2) and all(torch.equal(a, b) for a, b in zip(w1, w2))
