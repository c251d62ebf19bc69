"""GGNN training with any message MLP: hidden layers in the edge MLPs, target-state input, hidden_dim % 4 != 0.

GGNN.call composes the messages (GNN_Edge_MLP's own routing without activation: the fused _EdgeMLPLayerFunction where
it has a backward, else the literal op order of layers/differentiable.py) with the GRU update on its own
(tfgnn_b200_gru_update_fwd / _bwd, or the per-op GRU cell where hidden_dim % 4 != 0).  Gradients against float64 autograd
of the reference's op order (ggnn.py:68-89) at the bars of the existing GGNN tests, on target-range shards, and one
training step at the cfg4 size.

The hidden ReLU's derivative flips when a pre-activation lies within rounding of 0, which no tolerance absorbs.  So the fused
one-hidden-layer cases put h and the first kernels on the dyadic grid of test_gpu_edge_mlp_backward, on which every
pre-activation is exact (`_prove_exact_hidden`)."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

from oracle import message_passing_oracle as mo  # noqa: E402
from test_gpu_edge_mlp_backward import _prove_exact_hidden, dyadic, trimmed_pool  # noqa: E402,F401  (fixture)
from test_gpu_parity import _need_gpu, assert_states_close, make_layer, random_graph  # noqa: E402
from test_gpu_shard_backward import _check_shards  # noqa: E402
from test_gpu_transform_aggregate_backward import _uses  # noqa: E402

pytestmark = pytest.mark.gpu

OUT_TOL, GRAD_TOL = 1e-5, 2e-5

# name -> (hidden layers in the message MLPs, aggregation, normalize_by_num_incoming, use_target_state_as_input, H)
CASES = {
    "h1-sum-norm": (1, "sum", True, False, 32),
    "h1-sum": (1, "sum", False, False, 64),
    "h1-mean-target": (1, "mean", False, True, 32),
    "h1-sqrt_n-norm-target": (1, "sqrt_n", True, True, 48),
    "h0-target-norm": (0, "sum", True, True, 32),
    "h0-mean-target": (0, "mean", False, True, 36),
    "h2-sum-norm": (2, "sum", True, False, 32),
    "h3-mean-target": (3, "mean", False, True, 32),
    "h1-max": (1, "max", False, False, 32),
    "H30": (0, "sum", True, False, 30),
    "H30-h1-target": (1, "sum", True, True, 30),
}


def _fused_messages(n_hidden, agg, H):
    return H % 4 == 0 and (n_hidden == 0 or (n_hidden == 1 and agg != "max"))


def _inputs(name, seed, V=400, L=3):
    n_hidden, agg, normalize, use_target, H = CASES[name]
    rng = np.random.default_rng(seed)
    # max: every target gets an edge (self-loops in type 0; an empty max segment holds the lowest float) and no duplicate
    # edges (ties); otherwise hubs, duplicates and an empty type
    if agg == "max":
        adjs = random_graph(rng, V, L, 6 * V, self_loops=True)
    else:
        adjs = random_graph(rng, V, L, 6 * V, hub=True, dups=True, empty_type=1)
    exact = n_hidden == 1 and _fused_messages(n_hidden, agg, H)
    h = dyadic(rng, (V, H)) if exact else rng.uniform(-1, 1, (V, H)).astype(np.float32)
    dims = [(2 if use_target else 1) * H] + [H] * n_hidden + [H]
    mlps = [[dyadic(rng, (dims[0], dims[1])) if exact and i == 0 else mo.glorot_uniform(rng, (dims[i], dims[i + 1]))
             for i in range(len(dims) - 1)] for _ in range(L)]
    if exact:
        _prove_exact_hidden(h, [m[0] for m in mlps])
    w = {"edge_mlps": mlps, "gru_kernel": mo.glorot_uniform(rng, (H, 3 * H)),
         "gru_recurrent_kernel": mo.glorot_uniform(rng, (H, 3 * H)),
         "gru_bias": rng.uniform(-0.2, 0.2, (2, 3 * H)).astype(np.float32)}
    p = mo.default_hyperparameters("ggnn")
    p.update(hidden_dim=H, aggregation_function=agg, normalize_by_num_incoming=normalize,
             use_target_state_as_input=use_target, num_edge_MLP_hidden_layers=n_hidden)
    g = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    return p, adjs, h, w, g


def ggnn64(h, adjs, mlps, K, U, b, *, agg, normalize, use_target):
    """GGNN (ggnn.py:68-89) in the reference's op order: per-edge MLP messages (bias-free, ReLU hidden layers, linear output,
    gnn_edge_mlp.py:93-106), aggregation without activation, Keras GRUCell reset_after=True.  All float64 leaves."""
    V, H = h.shape
    msgs, tgts = [], []
    for adj, Ws in zip(adjs, mlps):
        a = torch.from_numpy(adj).long()
        src, tgt = a[:, 0], a[:, 1]
        x = h.index_select(0, src)
        if use_target:
            x = torch.cat([x, h.index_select(0, tgt)], 1)
        for i, W in enumerate(Ws):
            x = x @ W
            if i < len(Ws) - 1:
                x = torch.relu(x)
        if normalize:
            c = torch.zeros(V, dtype=h.dtype).index_add_(0, tgt, torch.ones(len(tgt), dtype=h.dtype))
            x = x / (c.index_select(0, tgt) + 1e-7).unsqueeze(-1)
        msgs.append(x)
        tgts.append(tgt)
    M, T = torch.cat(msgs), torch.cat(tgts)
    if agg == "max":
        aggd = torch.zeros((V, H), dtype=h.dtype).scatter_reduce(0, T[:, None].expand(-1, H), M, "amax",
                                                                 include_self=False)
    else:
        aggd = torch.zeros((V, H), dtype=h.dtype).index_add_(0, T, M)
        if agg in ("mean", "sqrt_n"):
            n = torch.zeros(V, dtype=h.dtype).index_add_(0, T, torch.ones(len(T), dtype=h.dtype)).clamp(min=1)
            aggd = aggd / (n if agg == "mean" else n.sqrt()).unsqueeze(-1)
    gx = aggd @ K + b[0]
    gh = h @ U + b[1]
    z = torch.sigmoid(gx[:, :H] + gh[:, :H])
    r = torch.sigmoid(gx[:, H:2 * H] + gh[:, H:2 * H])
    hh = torch.tanh(gx[:, 2 * H:] + r * gh[:, 2 * H:])
    return z * h + (1 - z) * hh


def _reference(p, adjs, h, w, g):
    """(out, grad_h, [grads of the message weights type-major, then K, U, b]) of float64 autograd."""
    t = lambda x: torch.from_numpy(np.asarray(x)).double().requires_grad_()   # noqa: E731
    h64 = t(h)
    mlps = [[t(W) for W in Ws] for Ws in w["edge_mlps"]]
    gru = [t(w[k]) for k in ("gru_kernel", "gru_recurrent_kernel", "gru_bias")]
    out = ggnn64(h64, adjs, mlps, *gru, agg=p["aggregation_function"], normalize=p["normalize_by_num_incoming"],
                 use_target=p["use_target_state_as_input"])
    out.backward(torch.from_numpy(g).double())
    leaves = [W for Ws in mlps for W in Ws] + gru
    return out.detach().numpy(), h64.grad.numpy(), [x.grad.numpy() for x in leaves]


def _layer(p, H, L, w):
    layer = make_layer("ggnn", p, H, L, w)
    for v in layer.variables:
        v.requires_grad_()
    params = [v for m in layer._edge_type_mlps for v in m.layers]
    params += [layer._gru_kernel, layer._gru_recurrent_kernel, layer._gru_bias]
    return layer, params


def _run(layer, params, h, adjs, g):
    from tf2_gnn_b200.layers import MessagePassingInput
    ht = torch.from_numpy(h).cuda().requires_grad_()
    for q in params:
        q.value.grad = None
    out = layer(MessagePassingInput(ht, tuple(torch.from_numpy(a).cuda() for a in adjs)))
    routes = {n: _uses(out, n) for n in ("_GGNNFunctionBackward", "_EdgeMLPLayerFunctionBackward",
                                         "_GruUpdateFunctionBackward", "_GruGateFunctionBackward")}
    out.backward(torch.from_numpy(g).cuda())
    torch.cuda.synchronize()
    return out.detach().cpu().numpy(), ht.grad.cpu().numpy(), [q.value.grad.cpu().numpy() for q in params], routes


@pytest.mark.parametrize("name", list(CASES))
def test_ggnn_mlp_backward_matches_float64_autograd(name):
    _need_gpu()
    n_hidden, agg, _, _, H = CASES[name]
    p, adjs, h, w, g = _inputs(name, seed=len(name))
    layer, params = _layer(p, H, len(adjs), w)
    ref_out, ref_h, ref_w = _reference(p, adjs, h, w, g)
    out, gh, gw, routes = _run(layer, params, h, adjs, g)
    assert not routes["_GGNNFunctionBackward"]
    assert routes["_EdgeMLPLayerFunctionBackward"] == _fused_messages(n_hidden, agg, H)
    assert routes["_GruUpdateFunctionBackward"] == (H % 4 == 0)
    assert routes["_GruGateFunctionBackward"] == (H % 4 != 0)
    assert_states_close(out, ref_out, tol=OUT_TOL)
    assert_states_close(gh, ref_h, tol=GRAD_TOL)
    assert len(gw) == len(ref_w)
    for a, b in zip(gw, ref_w):
        assert_states_close(a, b, tol=GRAD_TOL)
    if _fused_messages(n_hidden, agg, H):   # a second backward gives the same bits (the literal path's reductions do not)
        again = _run(layer, params, h, adjs, g)
        assert np.array_equal(out, again[0]) and np.array_equal(gh, again[1])
        assert all(np.array_equal(a, b) for a, b in zip(gw, again[2]))


@pytest.mark.parametrize("name", ["h1-sum-norm", "h1-sqrt_n-norm-target", "h0-target-norm"])
@pytest.mark.parametrize("fused_gru", ["1", "0"])
def test_training_output_is_the_inference_output(name, fused_gru, monkeypatch):
    """On the fused message paths the composed training forward runs tfgnn_b200_ggnn_fwd's kernels in its order."""
    _need_gpu()
    monkeypatch.setenv("TFGNN_B200_GGNN_FUSED_GRU", fused_gru)
    from tf2_gnn_b200.layers import MessagePassingInput
    p, adjs, h, w, _ = _inputs(name, seed=3)
    layer, _ = _layer(p, h.shape[1], len(adjs), w)
    inp = MessagePassingInput(torch.from_numpy(h).cuda().requires_grad_(), tuple(torch.from_numpy(a).cuda() for a in adjs))
    train = layer(inp)
    assert _uses(train, "_GruUpdateFunctionBackward")
    with torch.no_grad():
        infer = layer(inp)
    assert torch.equal(train.detach(), infer)


@pytest.mark.parametrize("name", ["h1-sum-norm", "h1-mean-target", "h0-target-norm"])
def test_ggnn_mlp_shard_backward_sums_to_full(name):
    """Worlds of 2 and 3 and a world with an empty middle shard (test_gpu_shard_backward._check_shards)."""
    _need_gpu()
    p, adjs, h, w, g = _inputs(name, seed=11)
    layer, params = _layer(p, h.shape[1], len(adjs), w)
    _, ref_h, ref_w = _reference(p, adjs, h, w, g)
    _check_shards(layer, params, h, adjs, g, (ref_h, ref_w))


@pytest.mark.parametrize("name", ["h2-sum-norm", "h1-max", "H30"])
def test_literal_message_paths_raise_on_a_shard(name):
    _need_gpu()
    from tf2_gnn_b200.layers import MessagePassingInput
    from tf2_gnn_b200.runtime import PreparedBatch
    p, adjs, h, w, _ = _inputs(name, seed=5)
    layer, _ = _layer(p, h.shape[1], len(adjs), w)
    V = h.shape[0]
    adj_t = tuple(torch.from_numpy(a).cuda() for a in adjs)
    with pytest.raises(NotImplementedError):
        layer(MessagePassingInput(torch.from_numpy(h).cuda().requires_grad_(), adj_t),
              prepared=PreparedBatch(adj_t, V, target_range=(0, V // 2)))


@pytest.mark.parametrize("name", ["h0-target-norm", "h0-mean-target"])
def test_ggnn_bwd_with_target_state_input(name):
    """tfgnn_b200_ggnn_bwd called directly with TFGNN_FLAG_USE_TARGET_STATE ([2H, H] message weights; GGNN.call trains these
    configurations through the composed path): whole batch against float64 autograd, and the shard contributions of worlds
    of 2 and 3 (the middle shard empty) sum to it."""
    _need_gpu()
    from tf2_gnn_b200 import _ffi
    from tf2_gnn_b200.runtime import PreparedBatch, stream_ptr
    p, adjs, h, w, g = _inputs(name, seed=17)
    _, ref_h, ref_w = _reference(p, adjs, h, w, g)
    V, H = h.shape
    flags = _ffi.FLAG_USE_TARGET | (_ffi.FLAG_NORMALIZE if p["normalize_by_num_incoming"] else 0)
    cuda = lambda x: torch.from_numpy(np.asarray(x, np.float32)).cuda()   # noqa: E731
    adj_t = tuple(torch.from_numpy(a).cuda() for a in adjs)
    ht, gt = cuda(h), cuda(g)
    Ws = [cuda(m[0]) for m in w["edge_mlps"]]
    gru = [cuda(w[k]) for k in ("gru_kernel", "gru_recurrent_kernel", "gru_bias")]

    def backward(lo, hi):
        pb = PreparedBatch(adj_t, V, target_range=(lo, hi))
        gh = torch.empty_like(ht)
        gw = [torch.empty_like(x) for x in Ws + gru]
        _ffi.check(_ffi.lib().tfgnn_b200_ggnn_bwd(
            pb.handle, pb.transposed().handle, ht.data_ptr(), H, _ffi.ptr_array(Ws), H, flags,
            _ffi.AGG[p["aggregation_function"]], *(x.data_ptr() for x in gru), gt[lo:hi].contiguous().data_ptr(),
            gh.data_ptr(), _ffi.ptr_array(gw[:len(Ws)]), *(x.data_ptr() for x in gw[len(Ws):]), stream_ptr()))
        torch.cuda.synchronize()
        return gh.cpu().double().numpy(), [x.cpu().double().numpy() for x in gw]

    full_h, full_w = backward(0, V)
    assert_states_close(full_h, ref_h, tol=GRAD_TOL)
    assert len(full_w) == len(ref_w)
    for a, b in zip(full_w, ref_w):
        assert_states_close(a, b, tol=GRAD_TOL)
    cut = V // 3
    for bounds in ([(0, V // 2), (V // 2, V)], [(0, cut), (cut, cut), (cut, V)]):
        parts = [backward(lo, hi) for lo, hi in bounds]
        sum_h = sum(x[0] for x in parts)
        assert_states_close(sum_h, full_h, tol=2e-6)
        for i, ref in enumerate(full_w):
            assert_states_close(sum(x[1][i] for x in parts), ref, tol=2e-6)
        if len(bounds) == 3:
            assert not parts[1][0].any() and not any(x.any() for x in parts[1][1])


def _device_bytes_in_use():
    torch.cuda.synchronize()
    free, total = torch.cuda.mem_get_info()
    return total - free


def _trim():
    """Hand torch's cache and the library's memory pool back to the driver."""
    import gc
    from tf2_gnn_b200 import _ffi
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    _ffi.lib().tfgnn_b200_release_device_state()


def _cfg4_steps(edge_scale):
    """Two training steps of a one-hidden-layer GGNN on bench.py's cfg4 graph with every edge list `edge_scale` times as long:
    (device-memory rise over the steps, measured with the pool and torch's cache trimmed before them, [(grad_h, grads)])."""
    import bench
    from tf2_gnn_b200.layers import GGNN, MessagePassingInput
    from tf2_gnn_b200.runtime import PreparedBatch
    wl = bench.WORKLOADS["cfg4"]
    wl = dict(wl, E=[e * edge_scale for e in wl["E"]])
    V, H = wl["V"], wl["H"]
    _, adjs, _ = bench.make_inputs(wl, seed=0)
    L = len(adjs)
    p = GGNN.get_default_hyperparameters()
    p.update(hidden_dim=H, num_edge_MLP_hidden_layers=1)
    rng = np.random.default_rng(4)
    layer, params = _layer(p, H, L, mo.make_weights("ggnn", p, H, L, rng))
    adj = tuple(torch.from_numpy(a).cuda() for a in adjs)
    prepared = PreparedBatch(adj, V)
    prepared.transposed()   # the backward's CSR belongs to the batch, not to the step
    h = torch.from_numpy(rng.uniform(-1, 1, (V, H)).astype(np.float32)).cuda().requires_grad_()
    g = torch.from_numpy(rng.uniform(-1, 1, (V, H)).astype(np.float32)).cuda()
    _trim()
    base = _device_bytes_in_use()
    runs = []
    for _ in range(2):
        h.grad = None
        for q in params:
            q.value.grad = None
        out = layer(MessagePassingInput(h, adj), prepared=prepared)
        assert _uses(out, "_EdgeMLPLayerFunctionBackward") and _uses(out, "_GruUpdateFunctionBackward")
        out.backward(g)
        runs.append((h.grad.cpu(), [q.value.grad.cpu() for q in params]))
        del out
    rise = _device_bytes_in_use() - base
    del layer, params, adj, prepared, h, g
    _trim()
    return rise, runs, sum(int(a.shape[0]) for a in adjs), V, H


def test_cfg4_training_step_with_a_hidden_layer(trimmed_pool, record_property, capsys):
    """bench.py's cfg4 graph (500k nodes, 5 types, 1.5M edges, H = 128), one hidden layer in the message MLPs: the step takes
    the fused message path, is finite, and a second step gives the same bits.  No temporary has a per-edge dimension: with
    four times the edges on the same nodes, the step's device-memory rise (torch's tensors and the library's pool, both
    trimmed before the steps) grows by less than one [3E, H] fp32 table.  The rise itself is several [V, H] tables (the
    edge-MLP backward's [V, L*H] operands, the GRU's [V, 3H] gate tables, the layer's [V, H] inputs and outputs), which at
    cfg4 (E = 3 V, L = 5) is more than one [E, H] table."""
    rise1, runs, E, V, H = _cfg4_steps(1)
    rise4, _, E4, _, _ = _cfg4_steps(4)
    record_property("device_memory_rise_GB", round(rise1 / 1e9, 3))
    record_property("device_memory_rise_4x_edges_GB", round(rise4 / 1e9, 3))
    with capsys.disabled():
        print(f"\n[ggnn cfg4 step, 1 hidden layer] device-memory rise {rise1 / 1e9:.3f} GB; with 4x the edges "
              f"{rise4 / 1e9:.3f} GB; one [E, H] fp32 table = {E * H * 4 / 1e9:.3f} GB, one [V, H] = {V * H * 4 / 1e9:.3f} GB")
    assert rise4 - rise1 < (E4 - E) * H * 4
    (h1, w1), (h2, w2) = runs
    assert torch.isfinite(h1).all() and all(torch.isfinite(x).all() for x in w1)
    assert h1.abs().max() > 0
    assert torch.equal(h1, h2) and all(torch.equal(a, b) for a, b in zip(w1, w2))
