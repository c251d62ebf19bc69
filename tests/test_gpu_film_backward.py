"""GNN-FiLM training through tfgnn_b200_film_bwd (aggregate-then-transform, no per-edge tensors): gradients of the node
states, the edge-MLP kernels and the FiLM kernels against float64 references, exactly on integer data, against the literal
per-edge path, on target-range shards, through a GNN stack, and at scale."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

import reference64_film as rf  # noqa: E402
from oracle import message_passing_oracle as mo  # noqa: E402
from reference64 import Graph  # noqa: E402
from test_gpu_parity import _need_gpu, assert_states_close, make_layer, random_graph  # noqa: E402
from test_gpu_shard_backward import _check_shards  # noqa: E402

pytestmark = pytest.mark.gpu

TOL = 3e-5   # the literal path's norm-wise bar for FiLM gradients (test_gpu_graph_ops.py)
FUSED = "_FilmLayerFunctionBackward"


def _film(D, H, L, rng, weights=None, **hyper):
    p = mo.default_hyperparameters("gnn_film")
    p.update(hidden_dim=H, **hyper)
    if weights is None:
        Ws = [mo.glorot_uniform(rng, ((2 if p["use_target_state_as_input"] else 1) * D, H)) for _ in range(L)]
        Fs = [mo.glorot_uniform(rng, (D, 2 * H)) for _ in range(L)]
    else:
        Ws, Fs = weights
    layer = make_layer("gnn_film", p, D, L, {"edge_mlps": [[w] for w in Ws], "film_mlps": [[f] for f in Fs]})
    for v in layer.variables:
        v.requires_grad_()
    return layer, p, Ws, Fs


def _params(layer):
    return ([m.layers[0] for m in layer._edge_type_mlps]
            + [m.layers[0] for m in layer._edge_type_film_layer_computations])


def _run(layer, h, adjs, g, prepared=None):
    """(out, grad_h, [grad of every edge-MLP kernel, then every FiLM kernel]) of one fused forward + backward."""
    from tf2_gnn_b200.layers import MessagePassingInput
    ht = torch.from_numpy(h).cuda().requires_grad_()
    for p in _params(layer):
        p.value.grad = None
    out = layer(MessagePassingInput(ht, tuple(torch.from_numpy(a).cuda() for a in adjs)), prepared=prepared)
    assert type(out.grad_fn).__name__ == FUSED
    out.backward(torch.from_numpy(g).cuda())
    torch.cuda.synchronize()
    return out.detach().cpu().numpy(), ht.grad.cpu().numpy(), [p.value.grad.cpu().numpy() for p in _params(layer)]


def _autograd64(h, adjs, Ws, Fs, g, p):
    h64 = torch.from_numpy(h).double().requires_grad_()
    W64 = [torch.from_numpy(w).double().requires_grad_() for w in Ws]
    F64 = [torch.from_numpy(f).double().requires_grad_() for f in Fs]
    out = rf.film_autograd(h64, [torch.from_numpy(a) for a in adjs], W64, F64, agg=p["aggregation_function"],
                           act=p["message_activation_function"], normalize=p["normalize_by_num_incoming"],
                           use_target=p["use_target_state_as_input"])
    out.backward(torch.from_numpy(g).double())
    return out.detach().numpy(), h64.grad.numpy(), [x.grad.numpy() for x in W64 + F64]


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


# Smooth activations only: with relu a pre-activation within rounding of 0 may take the other derivative (DESIGN.md §5).
@pytest.mark.parametrize("V,D,H,L,E,agg,act,normalize,use_target,empty,hub", [
    (600, 32, 36, 3, 4000, "sum", "tanh", False, False, None, False),
    (600, 32, 36, 3, 4000, "mean", "gelu", True, False, 1, True),
    (800, 64, 96, 4, 5000, "sqrt_n", "elu", False, True, 2, True),
    (800, 64, 96, 4, 5000, "sum", None, True, True, None, True),
    (500, 320, 320, 2, 3000, "mean", "tanh", True, True, None, True),
    (1500, 64, 64, 7, 6000, "sqrt_n", "gelu", False, True, 3, True),
    (700, 48, 32, 5, 4000, "mean", "elu", False, False, 0, True),
    (20000, 128, 128, 3, 120000, "sum", "tanh", True, False, None, True),
])
def test_film_backward_matches_float64_autograd(V, D, H, L, E, agg, act, normalize, use_target, empty, hub):
    _need_gpu()
    rng = np.random.default_rng(V + D + H + L)
    adjs = random_graph(rng, V, L, E, empty_type=empty, hub=hub, dups=True, self_loops=use_target)
    layer, p, Ws, Fs = _film(D, H, L, rng, aggregation_function=agg, message_activation_function=act,
                             normalize_by_num_incoming=normalize, use_target_state_as_input=use_target)
    h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    g = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    got = _run(layer, h, adjs, g)
    _close_all(got, _autograd64(h, adjs, Ws, Fs, g, p))
    _same_bits(got, _run(layer, h, adjs, g))   # a second backward gives the same bits
    if empty is not None:
        assert not got[2][empty].any() and not got[2][L + empty].any()


@pytest.mark.parametrize("V,D,H,L,E,use_target", [(4000, 64, 64, 3, 24000, False), (3000, 32, 48, 4, 15000, True),
                                                   (12000, 128, 128, 2, 60000, True)])
def test_film_backward_exact_on_integer_data(V, D, H, L, E, use_target):
    """sum / relu / no normalisation with h, W, F and grad_out in {-1, 0, 1}: once every partial sum is shown to stay below
    2^24, every output and gradient must equal float32(reference) bit for bit."""
    _need_gpu()
    rng = np.random.default_rng(V + L)
    adjs = random_graph(rng, V, L, E, empty_type=1 if L > 2 else None, dups=True)
    adjs[0][:300, 1] = V // 3                 # an in-degree hub (one long target segment)
    adjs[-1][:300, 0] = 7                     # an out-degree hub (one long segment of the source-keyed reduce)
    ints = lambda shape: rng.integers(-1, 2, shape).astype(np.float32)
    h, g = ints((V, D)), ints((V, H))
    Ws = [ints(((2 if use_target else 1) * D, H)) for _ in range(L)]
    Fs = [ints((D, 2 * H)) for _ in range(L)]
    graph = Graph(adjs, V)
    bound = rf.film_layer(h, adjs, Ws, Fs, g, use_target=use_target, absval=True, graph=graph)
    assert bound["partial_max"] < 2 ** 24, bound["partial_max"]
    ref = rf.film_layer(h, adjs, Ws, Fs, g, agg="sum", act="relu", use_target=use_target, graph=graph)
    layer, _, _, _ = _film(D, H, L, rng, weights=(Ws, Fs), aggregation_function="sum",
                           message_activation_function="relu", normalize_by_num_incoming=False,
                           use_target_state_as_input=use_target)
    out, gh, gw = _run(layer, h, adjs, g)
    f32 = lambda t: t.numpy().astype(np.float32)
    assert np.array_equal(out, f32(ref["out"]))
    assert np.array_equal(gh, f32(ref["grad_h"]))
    for a, b in zip(gw, ref["grad_W"] + ref["grad_F"]):
        assert np.array_equal(a, f32(b))


@pytest.mark.parametrize("agg,act,normalize,use_target", [("sum", "tanh", True, True), ("mean", "gelu", False, False),
                                                          ("sqrt_n", "elu", True, False)])
def test_fused_and_literal_paths_agree_with_float64(agg, act, normalize, use_target):
    """The literal per-edge path (layers/differentiable.py), called directly, stays covered for the configurations that now
    train through the fused backward; both meet the same bar against float64 autograd."""
    _need_gpu()
    from tf2_gnn_b200.layers.differentiable import edge_mlp_family_forward
    from tf2_gnn_b200.runtime import PreparedBatch
    rng = np.random.default_rng(31 + len(agg))
    V, D, H, L = 900, 32, 48, 3
    # no hub: the literal path sums beta once per edge in fp32, which at a 3000-edge hub alone exceeds the bar
    adjs = random_graph(rng, V, L, 6000, empty_type=2, dups=True)
    layer, p, Ws, Fs = _film(D, H, L, rng, aggregation_function=agg, message_activation_function=act,
                             normalize_by_num_incoming=normalize, use_target_state_as_input=use_target)
    h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    g = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    ref = _autograd64(h, adjs, Ws, Fs, g, p)
    _close_all(_run(layer, h, adjs, g), ref)
    ht = torch.from_numpy(h).cuda().requires_grad_()
    adj_dev = tuple(torch.from_numpy(a).cuda() for a in adjs)
    for q in _params(layer):
        q.value.grad = None
    out = edge_mlp_family_forward(layer, ht, PreparedBatch(adj_dev, V),
                                  film_kernels=[[v.value for v in m.layers] for m in layer._edge_type_film_layer_computations])
    assert type(out.grad_fn).__name__ != FUSED
    out.backward(torch.from_numpy(g).cuda())
    _close_all((out.detach().cpu().numpy(), ht.grad.cpu().numpy(), [q.value.grad.cpu().numpy() for q in _params(layer)]),
               ref)


@pytest.mark.parametrize("extra,D", [(dict(num_edge_MLP_hidden_layers=1), 32), (dict(film_parameter_MLP_hidden_layers=[16]), 32),
                                     (dict(aggregation_function="max"), 32),
                                     (dict(message_activation_before_aggregation=True, message_activation_function="tanh"), 32),
                                     ({}, 30)])
def test_configurations_outside_the_fused_backward_keep_the_literal_path(extra, D):
    _need_gpu()
    from tf2_gnn_b200.layers import MessagePassingInput
    from tf2_gnn_b200.runtime import PreparedBatch
    rng = np.random.default_rng(5)
    V, H, L = 400, 32, 2
    adjs = random_graph(rng, V, L, 2000)
    p = mo.default_hyperparameters("gnn_film")
    p.update(hidden_dim=H, **extra)
    layer = make_layer("gnn_film", p, D, L, mo.make_weights("gnn_film", p, D, L, rng))
    for v in layer.variables:
        v.requires_grad_()
    ht = torch.from_numpy(rng.uniform(-1, 1, (V, D)).astype(np.float32)).cuda().requires_grad_()
    adj_dev = tuple(torch.from_numpy(a).cuda() for a in adjs)
    out = layer(MessagePassingInput(ht, adj_dev))
    assert type(out.grad_fn).__name__ != FUSED
    out.sum().backward()
    assert torch.isfinite(ht.grad).all()
    with pytest.raises(NotImplementedError, match="target-range shard"):
        layer(MessagePassingInput(ht, adj_dev), prepared=PreparedBatch(adj_dev, V, target_range=(0, V // 2)))


@pytest.mark.parametrize("D,H,agg,act,normalize,use_target", [
    (64, 64, "mean", "tanh", True, True),
    (32, 48, "sum", "gelu", True, False),
    (64, 32, "sqrt_n", "elu", True, True),
    (32, 36, "mean", "tanh", False, False),
])
def test_film_shard_backward_sums_to_full(D, H, agg, act, normalize, use_target):
    """Worlds of 2 and 3 and a world with an empty shard (test_gpu_shard_backward._check_shards)."""
    _need_gpu()
    V, L = 700, 3
    rng = np.random.default_rng(D + H + 7)
    adjs = random_graph(rng, V, L, 5000, hub=True, dups=True, self_loops=use_target)
    layer, p, Ws, Fs = _film(D, H, L, rng, aggregation_function=agg, message_activation_function=act,
                             normalize_by_num_incoming=normalize, use_target_state_as_input=use_target)
    h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    g = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    _, ref_h, ref_w = _autograd64(h, adjs, Ws, Fs, g, p)
    _check_shards(layer, _params(layer), h, adjs, g, (ref_h, ref_w))


def _film_stack_reference(params, w, feats, adjs, dtype=torch.float64):
    """torch restatement of gnn.py:276-329 for a GNN-FiLM stack without exchange, LayerNorm or dropout (differentiable)."""
    t = lambda a: torch.from_numpy(np.asarray(a)).to(dtype).requires_grad_()
    leaves = {"proj": t(w["initial_projection"]), "mp": [[t(m[0]) for m in wi["edge_mlps"]] for wi in w["mp"]],
              "film": [[t(m[0]) for m in wi["film_mlps"]] for wi in w["mp"]],
              "dense": {i: t(d) for i, d in w["dense"].items()}}
    acts = {"tanh": torch.tanh, "relu": torch.relu}
    cur = acts[params["initial_node_representation_activation"]](torch.from_numpy(feats).to(dtype) @ leaves["proj"])
    last = cur
    for i in range(params["num_layers"]):
        if i % params["residual_every_num_layers"] == 0:
            tmp = cur
            if i > 0:
                cur = (cur + last) / 2
            last = tmp
        cur = rf.film_autograd(cur, adjs, leaves["mp"][i], leaves["film"][i], agg=params["aggregation_function"],
                               act=params["message_activation_function"], normalize=params["normalize_by_num_incoming"],
                               use_target=params["use_target_state_as_input"])
        if i % params["dense_every_num_layers"] == 0:
            cur = acts[params["dense_intermediate_layer_activation"]](cur @ leaves["dense"][i])
    return cur, leaves


def test_training_step_of_a_film_stack_matches_float64_autograd():
    """A PPI_GNN_FiLM.json-shaped stack: dense every layer, residual every 2 layers, target-state input, normalised."""
    _need_gpu()
    from tf2_gnn_b200.layers import GNNInput
    from test_gpu_graph_ops import _build_gnn
    from tf2_gnn_b200.layers import GNN
    rng = np.random.default_rng(13)
    V, F, H, L = 700, 48, 64, 3
    params = GNN.get_default_hyperparameters("gnn_film")
    params.update(hidden_dim=H, num_layers=4, global_exchange_every_num_layers=10000, layer_input_dropout_rate=0.0,
                  dense_every_num_layers=1, residual_every_num_layers=2, use_target_state_as_input=True,
                  normalize_by_num_incoming=True, use_inter_layer_layernorm=False)
    adjs = [rng.integers(0, V, size=(4000, 2)).astype(np.int32) for _ in range(L)]
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
        ref_out, leaves = _film_stack_reference(params, w, feats, adjs, dt)
        (ref_out * torch.from_numpy(R).to(dt)).sum().backward()
        refs[dt] = [ref_out.detach()] + [leaves["proj"].grad] + [x.grad for i in range(len(leaves["mp"]))
                                                                 for x in leaves["mp"][i] + leaves["film"][i]]
        refs[dt] += [leaves["dense"][i].grad for i in sorted(leaves["dense"])]
    got = [out.detach(), gnn._initial_projection_layer.kernel.grad]
    for mp in gnn._mp_layers:
        got += [m.layers[0].grad for m in mp._edge_type_mlps] + [m.layers[0].grad for m in mp._edge_type_film_layer_computations]
    got += [gnn._dense_layers[str(i)].kernel.grad for i in sorted(int(k) for k in gnn._dense_layers)]
    assert len(got) == len(refs[torch.float64]) and all(x is not None for x in got)
    # Through four FiLM layers the fp32 restatement itself drifts from the exact result (test_gnn_stack_parity): the bar is
    # 1e-5 per stage of the chain relative to the scale, or within 3x of the fp32 restatement's own error.
    tol = 1e-5 * (2 * params["num_layers"] + 2)
    for i, (x, r64, r32) in enumerate(zip(got, refs[torch.float64], refs[torch.float32])):
        x, r64, r32 = x.cpu().double().numpy(), r64.numpy(), r32.double().numpy()
        scale = max(np.abs(r64).max(), 1e-30)
        err, fp32_err = np.abs(x - r64).max(), np.abs(r32 - r64).max()
        assert err <= max(tol * scale, 3.0 * fp32_err), (i, err, fp32_err, scale)


def _row_close(got, ref, row, tol=TOL):
    g, r = np.asarray(got[row], np.float64), np.asarray(ref[row], np.float64)
    scale = max(np.abs(r).max(), 1e-30)
    assert np.abs(g - r).max() <= tol * scale, (row, np.abs(g - r).max(), scale)


@pytest.fixture
def trimmed_pool():
    """Start and leave a large case with the library's memory pool and torch's cache handed back to the driver."""
    import gc
    from tf2_gnn_b200 import _ffi
    from tf2_gnn_b200.runtime import clear_prepared_batch_cache
    _need_gpu()
    # batches of earlier cases (the layer call's prepared-batch cache, reference cycles) hold their CSR, and the pool keeps
    # the blocks earlier calls freed
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


def test_film_backward_at_scale_against_float64(monkeypatch, trimmed_pool):
    """1M nodes, 6 types of 1.5M edges, D = H = 256 (mean / tanh / normalised), with an in-degree and an out-degree hub of
    20,000 edges; norm-wise bars plus per-row bars on the largest in-degree and out-degree rows.  The forward runs in the
    aggregate-then-transform form (the form the backward differentiates, and the one shards use): the projected-table form
    sums beta once per edge in fp32, which loses 1e-4 at the 20,000-edge hub."""
    _need_gpu()
    monkeypatch.setenv("TFGNN_B200_FILM_ATT", "1")
    V, D, H, L, E = 1_000_000, 256, 256, 6, 1_500_000
    rng = np.random.default_rng(2024)
    adjs = [rng.integers(0, V, size=(E, 2)).astype(np.int32) for _ in range(L)]
    adjs[0][:20000, 1] = V // 3
    adjs[1][:20000, 0] = 7
    layer, p, Ws, Fs = _film(D, H, L, rng, aggregation_function="mean", message_activation_function="tanh",
                             normalize_by_num_incoming=True, use_target_state_as_input=False)
    h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    g = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    out, gh, gw = _run(layer, h, adjs, g)
    torch.cuda.empty_cache()
    graph = Graph(adjs, V)
    ref = rf.film_layer(h, adjs, Ws, Fs, g, agg="mean", act="tanh", normalize=True, graph=graph)
    ref_out, ref_h = ref["out"].numpy(), ref["grad_h"].numpy()
    assert_states_close(out, ref_out, tol=TOL)
    assert_states_close(gh, ref_h, tol=TOL)
    for a, b in zip(gw, ref["grad_W"] + ref["grad_F"]):
        assert_states_close(a, b.numpy(), tol=TOL)
    in_row, out_row = int(graph.in_degree.argmax()), int(graph.out_degree.argmax())
    assert in_row == V // 3 and out_row == 7
    _row_close(out, ref_out, in_row)
    _row_close(gh, ref_h, in_row)
    _row_close(gh, ref_h, out_row)


def test_film_cfg5_shard_forward_and_backward_fit_one_gpu(trimmed_pool):
    """bench.py's cfg5_shard (2M nodes, 6 types of 5.33M edges, D = H = 320, the class defaults): one training step fits
    one 80 GB H100, is finite, and a second step gives the same bits."""
    _need_gpu()
    from tf2_gnn_b200.layers import MessagePassingInput
    from tf2_gnn_b200.runtime import PreparedBatch
    V, D, L, E = 2_000_000, 320, 6, 5_333_333
    gen = torch.Generator(device="cuda")
    gen.manual_seed(5)
    adj = tuple(torch.randint(0, V, (E, 2), generator=gen, device="cuda", dtype=torch.int32) for _ in range(L))
    h = (torch.rand((V, D), generator=gen, device="cuda") * 2 - 1).requires_grad_()
    g = torch.rand((V, D), generator=gen, device="cuda") * 2 - 1
    layer, _, _, _ = _film(D, D, L, np.random.default_rng(5))
    prepared = PreparedBatch(adj, V)
    runs = []
    for _ in range(2):
        h.grad = None
        for q in _params(layer):
            q.value.grad = None
        out = layer(MessagePassingInput(h, adj), prepared=prepared)
        assert type(out.grad_fn).__name__ == FUSED
        out.backward(g)
        torch.cuda.synchronize()
        runs.append((h.grad.cpu(), [q.value.grad.cpu() for q in _params(layer)]))
        del out
    free, total = torch.cuda.mem_get_info()
    del prepared, adj, h, g
    assert total - free < 80e9
    (h1, w1), (h2, w2) = runs
    assert torch.isfinite(h1).all() and all(torch.isfinite(x).all() for x in w1)
    assert h1.abs().max() > 0
    assert torch.equal(h1, h2) and all(torch.equal(a, b) for a, b in zip(w1, w2))
