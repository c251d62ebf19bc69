"""Training of edge MLPs without hidden layer under max aggregation or activation before aggregation (the
transform-then-aggregate form) through tfgnn_b200_rgcn_bwd, and of GGNN under max aggregation through tfgnn_b200_ggnn_bwd:
no per-edge tensors.  Gradients against float64 torch autograd of the reference's literal op order, on target-range shards,
and one step at the cfg2 size.

The max picks one message per (target, column); fp32 and float64 must pick the same ones.  So h and W are small integers,
every segment holds 0, 7 or 11 edges (x / 7 and x' / 11 never coincide for |x|, |x'| <= 8 unless both are 0), duplicate
edges make real ties, and `_margin` asserts in float64 that every message below a maximum lies more than 1e-6 below it."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

import reference64_transform_aggregate as ta  # noqa: E402
from oracle import message_passing_oracle as mo  # noqa: E402
from test_gpu_edge_mlp_backward import trimmed_pool  # noqa: E402,F401  (fixture)
from test_gpu_parity import _need_gpu, assert_states_close, make_layer  # noqa: E402
from test_gpu_shard_backward import _check_shards  # noqa: E402

pytestmark = pytest.mark.gpu

TOL = 3e-5
FUSED = {"ggnn": "_GGNNFunctionBackward"}
# name -> (layer kind, target-state input, D, H): H covers 1 to 4 float4 column groups per lane
KINDS = {"rgcn": ("rgcn", False, 4, 36), "gnn_edge_mlp": ("gnn_edge_mlp", False, 4, 260),
         "gnn_edge_mlp_target": ("gnn_edge_mlp", True, 4, 132), "rgin": ("rgin", False, 4, 420),
         "ggnn": ("ggnn", False, 8, 8), "rgcn_target": ("rgcn", True, 4, 64)}
GRID_KINDS = ("rgcn", "gnn_edge_mlp", "gnn_edge_mlp_target", "rgin", "ggnn")
MAX = [dict(agg="max", act=a, before=False, normalize=n) for a in ("relu", "tanh", "gelu") for n in (False, True)]
BEFORE = [dict(agg=agg, act=a, before=True, normalize=(i + j) % 2 == 1)
          for i, agg in enumerate(("sum", "mean", "sqrt_n")) for j, a in enumerate(("tanh", "gelu", "relu"))]


def _grid():
    for name in GRID_KINDS:
        if name == "ggnn":          # GGNN has neither a message activation nor activation before aggregation
            yield from ((name, c) for c in MAX if c["act"] == "relu")
        elif name == "rgin":        # RGIN ignores activation before aggregation
            yield from ((name, c) for c in MAX)
        else:
            yield from ((name, c) for c in MAX + BEFORE)


def degree_graph(rng, V, L, empty=3):
    """L edge lists: every (type, target) segment holds 0, 7 or 11 edges, its second edge repeats its first, targets
    [0, empty) have none at all; the lists are shuffled.  empty=None: no segment is empty."""
    adjs = []
    for _ in range(L):
        deg = rng.choice([0, 7, 11], size=V, p=[0.3, 0.35, 0.35] if empty is not None else [0.0, 0.5, 0.5])
        deg[:empty or 0] = 0
        tgt = np.repeat(np.arange(V), deg)
        src = rng.integers(0, V, size=tgt.size)
        first = (np.cumsum(deg) - deg)[deg > 0]
        src[first + 1] = src[first]
        adjs.append(np.stack([src, tgt], 1)[rng.permutation(tgt.size)].astype(np.int32))
    return adjs


def _inputs(name, cfg, seed):
    kind, use_target, D, H = KINDS[name]
    rng = np.random.default_rng(seed)
    V, L = 500, 3
    # GGNN feeds the maximum to the GRU: every target gets an edge (an empty max segment holds the lowest float)
    adjs = degree_graph(rng, V, L, empty=None if kind == "ggnn" else 3)
    small = lambda shape: rng.integers(-1, 2, size=shape).astype(np.float32)
    h = small((V, D))
    Ws = [small(((2 if use_target else 1) * D, H)) for _ in range(L)]
    w = {"edge_mlps": [[x] for x in Ws]}
    if kind == "ggnn":
        w.update(gru_kernel=0.3 * mo.glorot_uniform(rng, (H, 3 * H)), gru_recurrent_kernel=mo.glorot_uniform(rng, (H, 3 * H)),
                 gru_bias=rng.uniform(-0.1, 0.1, (2, 3 * H)).astype(np.float32))
    if kind == "rgin":
        w["aggr_mlp"] = None
    p = mo.default_hyperparameters(kind)
    p.update(hidden_dim=H, aggregation_function=cfg["agg"], message_activation_function=cfg["act"],
             message_activation_before_aggregation=cfg["before"], normalize_by_num_incoming=cfg["normalize"],
             num_edge_MLP_hidden_layers=0, use_target_state_as_input=use_target)
    g = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    return kind, p, adjs, h, w, g


def _margin(kind, p, adjs, h, w):
    if p["aggregation_function"] != "max":
        return
    before = p["message_activation_before_aggregation"] and kind in ("rgcn", "gnn_edge_mlp")
    gap, ties = ta.max_margin(h, adjs, [m[0] for m in w["edge_mlps"]], act=p["message_activation_function"],
                              act_before=before, normalize=p["normalize_by_num_incoming"],
                              use_target=p["use_target_state_as_input"])
    assert gap > 1e-6, gap
    assert ties > 0


def _layer(kind, p, D, L, w):
    layer = make_layer(kind, p, D, L, w)
    for v in layer.variables:
        v.requires_grad_()
    params = [m.layers[0] for m in layer._edge_type_mlps]
    if kind == "ggnn":
        params += [layer._gru_kernel, layer._gru_recurrent_kernel, layer._gru_bias]
    return layer, params


def _reference(kind, p, adjs, h, w, g):
    """(out, grad_out masked on empty max segments, grad_h, [grads]) of float64 autograd of the literal op order."""
    t = lambda x: torch.from_numpy(np.asarray(x)).double().requires_grad_()
    h64 = t(h)
    leaves = [t(m[0]) for m in w["edge_mlps"]]
    if kind == "ggnn":
        gru = [t(w[k]) for k in ("gru_kernel", "gru_recurrent_kernel", "gru_bias")]
        out = ta.ggnn_autograd(h64, adjs, leaves, *gru, agg=p["aggregation_function"],
                               normalize=p["normalize_by_num_incoming"])
        leaves += gru
    else:
        before = p["message_activation_before_aggregation"] and kind != "rgin"
        out = ta.literal_autograd(h64, adjs, leaves, agg=p["aggregation_function"], act=p["message_activation_function"],
                                  act_before=before, normalize=p["normalize_by_num_incoming"],
                                  use_target=p["use_target_state_as_input"])
    sentinel = (out.detach() < -1e38).numpy()   # empty max segments (no gradient flows there)
    g = np.where(sentinel, 0.0, g).astype(np.float32)
    out.backward(torch.from_numpy(g).double())
    return out.detach().numpy(), g, h64.grad.numpy(), [x.grad.numpy() for x in leaves]


def _uses(out, name):
    seen, todo = set(), [out.grad_fn]
    while todo:
        f = todo.pop()
        if f is None or f in seen:
            continue
        seen.add(f)
        if type(f).__name__ == name:
            return True
        todo.extend(n for n, _ in f.next_functions)
    return False


def _run(kind, layer, params, h, adjs, g, prepared=None):
    from tf2_gnn_b200.layers import MessagePassingInput
    ht = torch.from_numpy(h).cuda().requires_grad_()
    for q in params:
        q.value.grad = None
    out = layer(MessagePassingInput(ht, tuple(torch.from_numpy(a).cuda() for a in adjs)), prepared=prepared)
    assert _uses(out, FUSED.get(kind, "_EdgeMLPLayerFunctionBackward"))
    out.backward(torch.from_numpy(g).cuda())
    torch.cuda.synchronize()
    return out.detach().cpu().numpy(), ht.grad.cpu().numpy(), [q.value.grad.cpu().numpy() for q in params]


@pytest.mark.parametrize("name,cfg", list(_grid()),
                         ids=[f"{n}-{'-'.join(str(v) for v in c.values())}" for n, c in _grid()])
def test_transform_aggregate_backward_matches_float64_autograd(name, cfg):
    _need_gpu()
    kind, p, adjs, h, w, g = _inputs(name, cfg, seed=len(name) + 7 * MAX.index(cfg) if cfg in MAX else 100 + BEFORE.index(cfg))
    _margin(kind, p, adjs, h, w)
    layer, params = _layer(kind, p, h.shape[1], len(adjs), w)
    ref_out, g, ref_h, ref_w = _reference(kind, p, adjs, h, w, g)
    got = _run(kind, layer, params, h, adjs, g)
    assert_states_close(got[0], ref_out, tol=TOL)
    assert_states_close(got[1], ref_h, tol=TOL)
    assert len(got[2]) == len(ref_w)
    for a, b in zip(got[2], ref_w):
        assert_states_close(a, b, tol=TOL)
    again = _run(kind, layer, params, h, adjs, g)   # a second backward gives the same bits
    assert np.array_equal(got[1], again[1]) and all(np.array_equal(a, b) for a, b in zip(got[2], again[2]))


@pytest.mark.parametrize("name,cfg", [
    ("rgcn", dict(agg="max", act="tanh", before=False, normalize=True)),
    ("rgcn_target", dict(agg="mean", act="gelu", before=True, normalize=True)),
    ("rgcn_target", dict(agg="max", act="tanh", before=True, normalize=False)),
    ("ggnn", dict(agg="max", act="relu", before=False, normalize=True)),
])
def test_transform_aggregate_shard_backward_sums_to_full(name, cfg):
    """Worlds of 2 and 3 and a world with an empty middle shard (test_gpu_shard_backward._check_shards)."""
    _need_gpu()
    kind, p, adjs, h, w, g = _inputs(name, cfg, seed=5 + len(name))
    _margin(kind, p, adjs, h, w)
    layer, params = _layer(kind, p, h.shape[1], len(adjs), w)
    _, g, ref_h, ref_w = _reference(kind, p, adjs, h, w, g)
    _check_shards(layer, params, h, adjs, g, (ref_h, ref_w))


def test_ggnn_with_max_aggregation_trains():
    """GGNN with max aggregation: out.backward() runs tfgnn_b200_ggnn_bwd and matches float64 autograd."""
    _need_gpu()
    kind, p, adjs, h, w, g = _inputs("ggnn", MAX[1], seed=9)
    layer, params = _layer(kind, p, h.shape[1], len(adjs), w)
    got = _run(kind, layer, params, h, adjs, g)
    _, g, ref_h, ref_w = _reference(kind, p, adjs, h, w, g)
    assert_states_close(got[1], ref_h, tol=TOL)
    for a, b in zip(got[2], ref_w):
        assert_states_close(a, b, tol=TOL)


# ---- cfg2 size ---------------------------------------------------------------------------------------------------------
def _float64_max_backward(h, adj, Ws, g, rows, chunk=1 << 21):
    """float64 on the device, chunked over edges: grad_h[rows] and every dW of an RGCN layer with max aggregation, relu after
    it, no normalisation (tf.math.unsorted_segment_max's gradient: grad / tie count to every message at the maximum)."""
    V, H = h.shape[0], Ws[0].shape[1]
    h64 = h.double()
    P = [h64 @ W.double() for W in Ws]
    z = torch.full((V, H), ta.LOWEST, dtype=torch.float64, device=h.device)
    for a, Pl in zip(adj, P):
        for c0 in range(0, a.shape[0], chunk):
            s, t = a[c0:c0 + chunk, 0].long(), a[c0:c0 + chunk, 1].long()
            z.scatter_reduce_(0, t[:, None].expand(-1, H), Pl[s], reduce="amax")
    n = torch.zeros_like(z)
    for a, Pl in zip(adj, P):
        for c0 in range(0, a.shape[0], chunk):
            s, t = a[c0:c0 + chunk, 0].long(), a[c0:c0 + chunk, 1].long()
            n.index_add_(0, t, (Pl[s] == z[t]).double())
    dz = torch.where(n > 0, g.double() * (z > 0).double() / n.clamp(min=1), torch.zeros_like(z))
    grad_h = torch.zeros((rows.numel(), h.shape[1]), dtype=torch.float64, device=h.device)
    grad_W = []
    for a, Pl, W in zip(adj, P, Ws):
        dP = torch.zeros_like(z)
        for c0 in range(0, a.shape[0], chunk):
            s, t = a[c0:c0 + chunk, 0].long(), a[c0:c0 + chunk, 1].long()
            dP.index_add_(0, s, dz[t] * (Pl[s] == z[t]).double())
        grad_W.append(h64.T @ dP)
        grad_h += dP[rows] @ W.double().T
        del dP
    return grad_h, grad_W


def test_cfg2_max_training_step_without_per_edge_tensors(trimmed_pool, record_property, capsys):
    """bench.py's cfg2 graph (1M nodes, 4 types of 5M edges, D = H = 256), RGCN with max aggregation: one forward and
    backward step through the fused path raises the device memory in use by less than one [M, H] fp32 tensor (what the
    literal path holds several of), and grad_h (sampled rows) and every dW match float64."""
    import bench
    from tf2_gnn_b200.layers import MessagePassingInput
    from tf2_gnn_b200.runtime import PreparedBatch
    wl = bench.WORKLOADS["cfg2"]
    _, adjs, _ = bench.make_inputs(wl, seed=0)   # the benchmark's graph; states and weights are small integers
    V, H, L = wl["V"], wl["H"], len(adjs)
    M = sum(a.shape[0] for a in adjs)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(3)
    small = lambda shape: torch.randint(-1, 2, shape, generator=gen, device="cuda").float()
    h = small((V, H)).requires_grad_()
    Ws = [small((H, H)) for _ in range(L)]
    g = torch.rand((V, H), generator=gen, device="cuda") * 2 - 1
    adj = tuple(torch.from_numpy(a).cuda() for a in adjs)
    del adjs
    p = mo.default_hyperparameters("rgcn")
    p.update(hidden_dim=H, aggregation_function="max", message_activation_function="relu", normalize_by_num_incoming=False)
    layer, params = _layer("rgcn", p, H, L, {"edge_mlps": [[w.cpu().numpy()] for w in Ws]})
    prepared = PreparedBatch(adj, V)
    prepared.transposed()
    torch.cuda.synchronize()
    free0, total = torch.cuda.mem_get_info()
    out = layer(MessagePassingInput(h, adj), prepared=prepared)
    assert _uses(out, "_EdgeMLPLayerFunctionBackward")
    out.backward(g)
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    rise = (free0 - free1) / 1e9
    record_property("device_memory_rise_GB", round(rise, 2))
    with capsys.disabled():
        print(f"\n[rgcn max cfg2 step] device memory rose by {rise:.1f} GB; one [M, H] fp32 tensor is "
              f"{4 * M * H / 1e9:.1f} GB")
    assert rise * 1e9 < 4.0 * M * H
    grad_h, grad_w = h.grad.detach(), [q.value.grad.detach() for q in params]
    del out, prepared
    h.grad = None
    for q in params:
        q.value.grad = None
    torch.cuda.empty_cache()
    rows = torch.randperm(V, generator=gen, device="cuda")[:4096]
    ref_h, ref_w = _float64_max_backward(h.detach(), adj, Ws, g, rows)
    assert_states_close(grad_h[rows].cpu().numpy(), ref_h.cpu().numpy(), tol=TOL)
    for a, b in zip(grad_w, ref_w):
        assert_states_close(a.cpu().numpy(), b.cpu().numpy(), tol=TOL)
    assert grad_h.abs().max() > 0
