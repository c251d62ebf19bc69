"""The stream contract of the library (include/tfgnn_b200.h, INTEGRATION.md): every call is enqueued on the caller's stream,
a batch may move to another stream between calls (the library orders the streams), entry points are re-entrant and the last
error is thread-local.

Torch's side streams are created non-blocking: unlike the legacy default stream they wait for nothing, so a launch on the
wrong stream, an internal stream that is not joined, or a buffer freed on the wrong stream races there.  No test here loops
to catch a race; each makes the race window long instead.  A case first runs on the default stream (the warm-up, whose
results are the reference bits), then fills its inputs with a huge finite poison and, on a side stream, sleeps before it
copies the real values back and makes the same calls.  A kernel that runs early reads the poison (or, for a CSR, a pool
block that held another graph) and the result differs from the reference bits.  Each delayed case asserts that its sleep
was still pending when its last call was enqueued: otherwise a pass would prove nothing."""
import threading
import time

import numpy as np
import pytest

torch = pytest.importorskip("torch")

import reference64 as r64  # noqa: E402
import reference64_readout as r64r  # noqa: E402
from oracle import adjacency_oracle as ao  # noqa: E402
from oracle import message_passing_oracle as mo  # noqa: E402
from test_gpu_parity import _need_gpu, assert_states_close, make_layer, random_graph  # noqa: E402
from test_gpu_readout_backward import _load_readout, _make_exchange, _make_readout, _readout_weights, n2g_of  # noqa: E402
from test_gpu_transform_aggregate_backward import _uses  # noqa: E402

pytestmark = pytest.mark.gpu

SLEEP_CYCLES = 150_000_000     # about 75-90 ms at the H100's 1.7-2.0 GHz SM clock
POISON = 1e30                  # finite: fmaxf would drop a NaN and hide it from max aggregation
GRAD_TOL = 2e-5                # test_gpu_parity.py's bar for gradients through one layer


@pytest.fixture(autouse=True)
def _gpu():
    _need_gpu()


# ---- the harness ------------------------------------------------------------------------------------------------------
def _poison(bufs):
    """Fill every buffer with the poison (index tensors with 0: a valid node id, so an early read gives a wrong graph, never
    an out-of-range access) and return copies of the real values."""
    saved = [b.detach().clone() for b in bufs]
    with torch.no_grad():
        for b in bufs:
            b.fill_(POISON if b.is_floating_point() else 0)
    torch.cuda.synchronize()
    return saved


def _sleep_then_restore(bufs, saved):
    """On the current stream: the sleep, an event behind it, then the real values into the poisoned buffers."""
    torch.cuda._sleep(SLEEP_CYCLES)
    ev = torch.cuda.Event()
    ev.record()
    with torch.no_grad():
        for b, v in zip(bufs, saved):
            b.copy_(v)
    return ev


def _assert_window_open(ev):
    assert not ev.query(), "the sleep had ended before the last call was enqueued: the race window was not open"


def run_delayed(bufs, fn, stream=None):
    """fn() on a side stream behind the sleep, with `bufs` poisoned until then.  Returns (results, snapshots taken on the
    side stream right after the calls), both after a device synchronisation."""
    saved = _poison(bufs)
    s = stream or torch.cuda.Stream()
    with torch.cuda.stream(s):
        ev = _sleep_then_restore(bufs, saved)
        res = fn()
        snap = [r.clone() for r in res]
    _assert_window_open(ev)
    torch.cuda.synchronize()
    return res, snap


def check_side_stream(bufs, fn, bitwise=True):
    """Warm-up on the default stream, then the delayed run on a side stream: every result must equal its snapshot and,
    with `bitwise`, the warm-up's bits.  Paths that sum with float atomics (bitwise=False) are left to the float64
    comparison of the caller.  Returns the side stream's results."""
    ref = [r.detach().clone() for r in fn()]
    torch.cuda.synchronize()
    res, snap = run_delayed(bufs, fn)
    assert len(res) == len(ref)
    for i, (a, b, c) in enumerate(zip(ref, res, snap)):
        assert torch.equal(b, c), f"result {i} was still being written after the calls returned to the stream"
        if bitwise:
            assert torch.equal(a, b), f"result {i} differs from the default-stream run"
    return res


def _grads(out, inputs, g):
    return [x for x in torch.autograd.grad(out, inputs, g, allow_unused=True) if x is not None]


def _np(t):
    return t.detach().cpu().numpy()


class _MP:
    """One message-passing layer with its device inputs.  h, grad_out and the weights are poisoned for the delayed run; the
    adjacency is not: the batch (and its transpose) the warm-up prepared stays cached, so the delayed run moves a built,
    synchronised CSR to the side stream, and a kernel that runs early reads poisoned values through valid indices.  A
    prepare on another stream is the subject of the batch-moves tests below."""

    def __init__(self, kind, params, V, D, L, E, seed, graph=None, path="auto", grads=True, **graph_opts):
        from tf2_gnn_b200.layers import MessagePassingInput
        rng = np.random.default_rng(seed)
        self.kind, self.V, self.D, self.L = kind, V, D, L
        self.p = dict(params, b200_path=path)
        self.adjs = graph if graph is not None else random_graph(rng, V, L, E, **graph_opts)
        self.w = mo.make_weights(kind, self.p, D, L, rng)
        self.layer = make_layer(kind, self.p, D, L, self.w)
        self.h_np = rng.uniform(-1, 1, (V, D)).astype(np.float32)
        H = int(self.p["hidden_dim"])
        self.g_np = rng.uniform(-1, 1, (V, H)).astype(np.float32)
        self.h = torch.from_numpy(self.h_np).cuda()
        self.g = torch.from_numpy(self.g_np).cuda()
        self.adj = tuple(torch.from_numpy(a).cuda() for a in self.adjs)
        self.weights = [v.value for v in self.layer.variables]
        self.grads = grads
        if grads:
            self.h.requires_grad_()
            for t in self.weights:
                t.requires_grad_()
        self.inp = MessagePassingInput(self.h, self.adj)

    @property
    def bufs(self):
        return [self.h, self.g, *self.weights]

    def step(self, prepared=None):
        """Forward and, with gradients on, backward: [out, grad_h, *grad_weights]."""
        if not self.grads:
            with torch.no_grad():
                return [self.layer(self.inp, prepared=prepared)]
        out = self.layer(self.inp, training=True, prepared=prepared)
        return [out.detach()] + _grads(out, [self.h] + self.weights, self.g)

    def forward64(self):
        return mo.message_passing_forward(self.kind, self.p, self.w, self.h_np, self.adjs, dtype=np.float64)

    def check_rgcn64(self, res, agg, act, normalize):
        """out, grad_h and every grad_W against the float64 RGCN layer."""
        ref = r64.rgcn_layer(self.h_np, self.adjs, [m[0] for m in self.w["edge_mlps"]], self.g_np, agg=agg, act=act,
                             normalize=normalize)
        assert_states_close(_np(res[0]), ref["out"].numpy())
        assert_states_close(_np(res[1]), ref["grad_h"].numpy(), tol=GRAD_TOL)
        assert len(res) == 2 + self.L
        for got, want in zip(res[2:], ref["grad_W"]):
            assert_states_close(_np(got), want.numpy(), tol=GRAD_TOL)


def _rgcn_params(H, agg="sum", act="tanh", normalize=False, **extra):
    p = mo.default_hyperparameters("rgcn")
    p.update(hidden_dim=H, aggregation_function=agg, message_activation_function=act,
             normalize_by_num_incoming=normalize, **extra)
    return p


# ---- 1: every family on a side stream ------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,V,D,H,L,E,agg,path,env", [
    ("fused_rows_h256", 3000, 256, 256, 3, 12000, "mean", "auto", {}),
    ("fused_split_tiles", 2000, 128, 128, 3, 8000, "mean", "fused_tc", {"TFGNN_B200_FUSED_SPLIT": "1"}),
    ("fused_multipass_h320", 2000, 64, 320, 3, 8000, "sqrt_n", "fused_tc", {}),
    ("sorted", 1000, 64, 64, 3, 6000, "mean", "sorted", {}),
    ("sorted_tc", 1000, 64, 64, 3, 6000, "sum", "sorted_tc", {}),
    ("atomic", 1000, 64, 64, 3, 6000, "sum", "atomic", {}),
])
def test_rgcn_on_a_side_stream(monkeypatch, name, V, D, H, L, E, agg, path, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    normalize = agg == "mean"
    c = _MP("rgcn", _rgcn_params(H, agg, normalize=normalize), V, D, L, E, seed=V + H, path=path, hub=True, dups=True)
    res = check_side_stream(c.bufs, c.step, bitwise=path != "atomic")   # the atomic path sums in arrival order
    c.check_rgcn64(res, agg, "tanh", normalize)


def test_rgcn_pipeline_forks_its_streams_on_a_side_stream(monkeypatch):
    """The gather || GEMM pipeline over 256-row chunks (D = 36: the fused kernel refuses it), its two internal streams
    forked from and joined to a side stream."""
    from tf2_gnn_b200 import _ffi
    monkeypatch.setenv("TFGNN_B200_PIPE_CHUNK_ROWS", "256")
    V, D, H, L = 1500, 36, 64, 3
    c = _MP("rgcn", _rgcn_params(H, "mean", normalize=True), V, D, L, 6000, seed=3, hub=True, self_loops=True)
    res = check_side_stream(c.bufs, c.step)
    c.check_rgcn64(res, "mean", "tanh", True)
    with torch.no_grad():
        n0 = _ffi.launch_count()
        c.layer(c.inp)
        launches = _ffi.launch_count() - n0
    assert launches >= 2 * -(-V // 256), f"{launches} launches: the pipeline did not run"


def test_rgcn_layernorm_epilogue_on_a_side_stream():
    """tfgnn_b200_rgcn_ln_fwd: LayerNorm in the fused kernel's epilogue."""
    V, D, H, L = 3000, 256, 256, 3
    c = _MP("rgcn", _rgcn_params(H, act="relu"), V, D, L, 9000, seed=4, grads=False)
    rng = np.random.default_rng(5)
    gamma = torch.from_numpy(rng.uniform(0.5, 1.5, H).astype(np.float32)).cuda()
    beta = torch.from_numpy(rng.uniform(-0.2, 0.2, H).astype(np.float32)).cuda()
    fn = lambda: [c.layer.call_with_layernorm(c.inp, gamma, beta, 1e-3)]
    res = check_side_stream(c.bufs + [gamma, beta], fn)
    with torch.no_grad():
        plain = c.layer(c.inp)
    ref = mo.layer_norm(_np(plain).astype(np.float64), _np(gamma).astype(np.float64), _np(beta).astype(np.float64))
    assert_states_close(_np(res[0]), ref)


@pytest.mark.parametrize("agg,before", [("max", False), ("sum", True)])
def test_transform_aggregate_backward_on_a_side_stream(agg, before):
    """Max aggregation and activation before aggregation: the transform-then-aggregate forward and its fused backward."""
    p = _rgcn_params(64, agg, normalize=True, message_activation_before_aggregation=before)
    c = _MP("rgcn", p, 800, 64, 3, 5000, seed=6, hub=True)
    res = check_side_stream(c.bufs, c.step)
    out = c.layer(c.inp, training=True)
    assert _uses(out, "_EdgeMLPLayerFunctionBackward")
    assert_states_close(_np(res[0]), c.forward64())


@pytest.mark.parametrize("fused_gru", ["1", "0"])
def test_ggnn_on_a_side_stream(monkeypatch, fused_gru):
    monkeypatch.setenv("TFGNN_B200_GGNN_FUSED_GRU", fused_gru)
    p = mo.default_hyperparameters("ggnn")
    p["hidden_dim"] = 64
    c = _MP("ggnn", p, 1000, 64, 3, 4000, seed=7, hub=True)
    res = check_side_stream(c.bufs, c.step)
    w = c.w
    ref = r64.ggnn_layer(c.h_np, c.adjs, [m[0] for m in w["edge_mlps"]], w["gru_kernel"], w["gru_recurrent_kernel"],
                         w["gru_bias"], c.g_np, agg=p["aggregation_function"], normalize=p["normalize_by_num_incoming"])
    assert_states_close(_np(res[0]), ref["out"].numpy())
    assert_states_close(_np(res[1]), ref["grad_h"].numpy(), tol=GRAD_TOL)


@pytest.mark.parametrize("kind,extra,env", [
    ("rgin", dict(normalize_by_num_incoming=True), {}),
    ("gnn_film", dict(normalize_by_num_incoming=True), {"TFGNN_B200_FILM_ATT": "1"}),
    ("gnn_film", dict(normalize_by_num_incoming=True), {"TFGNN_B200_FILM_ATT": "0"}),
    ("gnn_edge_mlp", dict(num_edge_MLP_hidden_layers=1, use_target_state_as_input=True), {}),
    ("gnn_edge_mlp", dict(num_edge_MLP_hidden_layers=2, message_activation_function="tanh"), {}),   # the literal path
])
def test_edge_mlp_families_on_a_side_stream(monkeypatch, kind, extra, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    p = mo.default_hyperparameters(kind)
    p.update(hidden_dim=48, **extra)
    c = _MP(kind, p, 700, 32, 3, 4000, seed=len(kind) + len(env), hub=True, dups=True)
    # the literal per-edge path sums its messages with unsorted_segment_reduce's float atomics: float64 only
    res = check_side_stream(c.bufs, c.step, bitwise=extra.get("num_edge_MLP_hidden_layers") != 2)
    assert_states_close(_np(res[0]), c.forward64())


def test_rgat_with_a_hub_on_a_side_stream():
    """3 heads and one target with more than 2048 incoming edges per type: the hub work list, the chunk partials and their
    in-order combine, forward and backward."""
    p = mo.default_hyperparameters("rgat")
    p.update(hidden_dim=48, num_heads=3, message_activation_function="tanh")
    c = _MP("rgat", p, 900, 32, 2, 6000, seed=8, hub=True)
    assert max(np.bincount(a[:, 1]).max() for a in c.adjs) > 2048
    res = check_side_stream(c.bufs, c.step)
    assert_states_close(_np(res[0]), c.forward64())


def test_generic_plugin_path_on_a_side_stream():
    """A user plugin (MessagePassing subclass): in_degree, gather_rows and unsorted_segment_reduce."""
    from tf2_gnn_b200.layers import MessagePassing, MessagePassingInput

    class MeanOfSources(MessagePassing):
        def __init__(self):
            params = super().get_default_hyperparameters()
            params.update(hidden_dim=24, message_activation_function="relu", aggregation_function="sum")
            super().__init__(params)

        def _message_function(self, edge_source_states, edge_target_states, num_incoming_to_node_per_message,
                              edge_type_idx, training):
            return edge_source_states / num_incoming_to_node_per_message.unsqueeze(-1)

    rng = np.random.default_rng(9)
    V, D, L = 500, 24, 2
    adjs = random_graph(rng, V, L, 3000, hub=True)
    h_np = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    h = torch.from_numpy(h_np).cuda()
    adj = tuple(torch.from_numpy(a).cuda() for a in adjs)
    layer = MeanOfSources()
    # the adjacency is poisoned too: the delayed run prepares its own batch on the side stream.  The messages are summed
    # with float atomics, so the result is checked against float64 only.
    res = check_side_stream([h, *adj], lambda: [layer(MessagePassingInput(h, adj))], bitwise=False)
    ref = np.zeros((V, D))
    for a in adjs:
        deg = np.bincount(a[:, 1], minlength=V)
        np.add.at(ref, a[:, 1], h_np[a[:, 0]].astype(np.float64) / deg[a[:, 1], None])
    assert_states_close(_np(res[0]), np.maximum(ref, 0.0))


def test_dense_and_layer_norm_on_a_side_stream():
    from tf2_gnn_b200.layers import node_ops
    from tf2_gnn_b200.utils.param_helpers import get_activation_function
    rng = np.random.default_rng(10)
    V, K, N = 2000, 64, 96
    x_np, W_np = rng.uniform(-1, 1, (V, K)).astype(np.float32), mo.glorot_uniform(rng, (K, N))
    b_np, R_np = rng.uniform(-.3, .3, N).astype(np.float32), rng.uniform(-1, 1, (V, N)).astype(np.float32)
    ga_np, be_np = rng.uniform(0.5, 1.5, N).astype(np.float32), rng.uniform(-.2, .2, N).astype(np.float32)
    x, W, b, R, ga, be = (torch.from_numpy(a).cuda() for a in (x_np, W_np, b_np, R_np, ga_np, be_np))
    leaves = [x, W, b, ga, be]
    for t in leaves:
        t.requires_grad_()

    def fn():
        y = node_ops.layer_norm(node_ops.dense(x, W, b, get_activation_function("tanh")), ga, be, 1e-3)
        return [y.detach()] + _grads(y, leaves, R)

    res = check_side_stream([*leaves, R], fn)
    t64 = [torch.from_numpy(a).double().requires_grad_() for a in (x_np, W_np, b_np, ga_np, be_np)]
    y64 = torch.nn.functional.layer_norm(torch.tanh(t64[0] @ t64[1] + t64[2]), (N,), t64[3], t64[4], eps=1e-3)
    (y64 * torch.from_numpy(R_np).double()).sum().backward()
    assert_states_close(_np(res[0]), y64.detach().numpy())
    for got, want in zip(res[1:], t64):
        assert_states_close(_np(got), want.grad.numpy(), tol=GRAD_TOL)


def _graph_inputs(rng, D):
    sizes = np.concatenate([rng.integers(0, 40, size=60), [2500]])   # many short graphs and one long one
    n2g = n2g_of(sizes)
    return n2g, len(sizes), torch.from_numpy(rng.uniform(-1, 1, (len(n2g), D)).astype(np.float32)).cuda()


@pytest.mark.parametrize("mode", ["softmax", "sigmoid", "none", "average"])
def test_readout_on_a_side_stream(mode):
    """WeightedSumGraphRepresentation through graph_autograd: the row-range segment sums and the readout backward."""
    from tf2_gnn_b200.layers import NodesToGraphRepresentationInput
    rng = np.random.default_rng(11)
    D, GD, K = 32, 16, 4
    n2g, G, x = _graph_inputs(rng, D)
    w = _readout_weights(rng, D, GD, K, mode, False)
    layer = _make_readout(D, GD, K, mode, w, regression_task=False)
    R = torch.from_numpy(rng.uniform(-1, 1, (G, GD)).astype(np.float32)).cuda()
    n2g_t = torch.from_numpy(n2g).cuda()
    x.requires_grad_()
    weights = [v.value for v in layer.variables]

    def fn():
        out = layer(NodesToGraphRepresentationInput(x, n2g_t, G), training=False)
        return [out.detach()] + _grads(out, [x] + weights, R)

    res = check_side_stream([x, R, *weights], fn)
    x64 = r64r.leaf(_np(x))
    ref = r64r.readout_layer(x64, r64r.leaves_of(w), n2g, G, K, mode, "relu", "relu", None, None)
    (ref * r64r.leaf(_np(R))).sum().backward()
    assert_states_close(_np(res[0]), ref.detach().numpy())
    assert_states_close(_np(res[1]), x64.grad.numpy(), tol=GRAD_TOL)


def test_was_readout_on_a_side_stream():
    from tf2_gnn_b200.layers import NodesToGraphRepresentationInput, WASGraphRepresentation
    rng = np.random.default_rng(12)
    D, GD, K = 24, 16, 4
    n2g, G, x = _graph_inputs(rng, D)
    layer = WASGraphRepresentation(GD, K, pooling_mlp_layers=[20])
    layer.build(NodesToGraphRepresentationInput((None, D), None, None))

    def weights():
        s, t = [D, 20, K], [D, 20, GD]
        return {"scoring_mlp": [mo.glorot_uniform(rng, (a, b)) for a, b in zip(s, s[1:])],
                "scoring_biases": [rng.uniform(-.2, .2, b).astype(np.float32) for b in s[1:]],
                "transformation_mlp": [mo.glorot_uniform(rng, (a, b)) for a, b in zip(t, t[1:])],
                "transformation_biases": [rng.uniform(-.2, .2, b).astype(np.float32) for b in t[1:]]}

    w_avg, w_sum, P = weights(), weights(), mo.glorot_uniform(rng, (2 * GD, GD))
    _load_readout(layer._weighted_avg_graph_repr_layer, w_avg)
    _load_readout(layer._weighted_sum_graph_repr_layer, w_sum)
    layer._out_projection.assign(P)
    R = torch.from_numpy(rng.uniform(-1, 1, (G, GD)).astype(np.float32)).cuda()
    n2g_t = torch.from_numpy(n2g).cuda()
    x.requires_grad_()
    wts = [v.value.requires_grad_() for v in layer.variables]

    def fn():
        out = layer(NodesToGraphRepresentationInput(x, n2g_t, G), training=False)
        return [out.detach()] + _grads(out, [x] + wts, R)

    res = check_side_stream([x, R, *wts], fn)
    x64 = r64r.leaf(_np(x))
    ref = r64r.was(x64, r64r.leaves_of(w_avg), r64r.leaves_of(w_sum), r64r.leaf(P), n2g, G, K)
    (ref * r64r.leaf(_np(R))).sum().backward()
    assert_states_close(_np(res[0]), ref.detach().numpy())
    assert_states_close(_np(res[1]), x64.grad.numpy(), tol=GRAD_TOL)


@pytest.mark.parametrize("dropout", [0.0, 0.2])
@pytest.mark.parametrize("mode", ["mean", "gru", "mlp"])
def test_global_exchange_on_a_side_stream(mode, dropout):
    """The three global exchanges through graph_autograd; with dropout, the masks are drawn again from the same seed for each
    run (float64 parity of the masked exchange is test_gpu_readout_backward.py's)."""
    from tf2_gnn_b200.layers import GraphGlobalExchangeInput, node_ops
    rng = np.random.default_rng(13 + len(mode))
    H, K, seed = 32, 4, 99
    n2g, G, x = _graph_inputs(rng, H)
    w = mo.make_exchange_weights(mode, H, K, rng, "softmax")
    ex = _make_exchange(mode, H, K, "softmax", w, dropout_rate=dropout, seed=seed if dropout else None)
    R = torch.from_numpy(rng.uniform(-1, 1, tuple(x.shape)).astype(np.float32)).cuda()
    n2g_t = torch.from_numpy(n2g).cuda()
    x.requires_grad_()
    weights = [v.value for v in ex.variables]

    def fn():
        if dropout:
            ex.dropout_state = node_ops.DropoutState(seed)
        out = ex(GraphGlobalExchangeInput(x, n2g_t, G), training=bool(dropout))
        return [out.detach()] + _grads(out, [x] + weights, R)

    res = check_side_stream([x, R, *weights], fn)
    if not dropout:
        x64 = r64r.leaf(_np(x))
        ref = r64r.exchange(mode, x64, r64r.leaves_of(w), n2g, G, K, "softmax")
        (ref * r64r.leaf(_np(R))).sum().backward()
        assert_states_close(_np(res[0]), ref.detach().numpy())
        assert_states_close(_np(res[1]), x64.grad.numpy(), tol=GRAD_TOL)


def test_minibatch_from_the_device_graph_store_on_a_side_stream():
    """DeviceGraphStore.batch (tfgnn_b200_assemble_batch and the feature gather) feeding an RGCN training step."""
    from tf2_gnn_b200.data import DeviceGraphStore
    from tf2_gnn_b200.layers import MessagePassingInput
    from test_gpu_batch_builder import _random_graphs
    rng = np.random.default_rng(14)
    T, F, H = 2, 32, 32
    graphs = _random_graphs(rng, 80, T, 25, F)
    store = DeviceGraphStore(graphs, T)
    ids = next(iter(store.iter_batch_graph_ids(max_nodes_per_batch=600)))
    p = _rgcn_params(H)
    w = mo.make_weights("rgcn", p, F, T, rng)
    layer = make_layer("rgcn", p, F, T, w)
    weights = [v.value.requires_grad_() for v in layer.variables]

    def fn():
        b = store.batch(ids)
        h = b["node_features"].requires_grad_()
        out = layer(MessagePassingInput(h, tuple(b[f"adjacency_list_{t}"] for t in range(T))), training=True)
        g = torch.ones_like(out)
        return [b["node_features"].detach(), b["node_to_graph_map"], *[b[f"adjacency_list_{t}"] for t in range(T)],
                out.detach()] + _grads(out, [h] + weights, g)

    res = check_side_stream([store.node_features, *store.edges, *weights], fn)
    hb = ao.assemble_batch([graphs[i] for i in ids], T)
    assert np.array_equal(_np(res[0]), np.asarray(hb["node_features"], np.float32))
    assert np.array_equal(_np(res[1]), np.asarray(hb["node_to_graph_map"], np.int32))
    adjs = [np.asarray(hb[f"adjacency_list_{t}"], np.int32).reshape(-1, 2) for t in range(T)]
    for t in range(T):
        assert np.array_equal(_np(res[2 + t]), adjs[t])
    ref = r64.rgcn_layer(_np(res[0]), adjs, [m[0] for m in w["edge_mlps"]], np.ones((len(res[1]), H), np.float32),
                         agg="sum", act="tanh")
    assert_states_close(_np(res[2 + T]), ref["out"].numpy())
    assert_states_close(_np(res[3 + T]), ref["grad_h"].numpy(), tol=GRAD_TOL)


# ---- 2 / 3: one batch on many streams ------------------------------------------------------------------------------------
def _decoy(rng, adjs, V):
    """A graph with the same sizes (so its CSR takes the same pool blocks) and different degrees: every edge into a few
    targets."""
    return [np.stack([a[:, 0], rng.integers(0, 8, size=len(a))], 1).astype(np.int32) for a in adjs]


def test_one_batch_moves_across_five_streams():
    """Prepare on A behind a sleep, the forward on B, transposed() and a training step on C, in_degree() on D, csr() on E:
    every result equals the single-stream run bitwise.  A decoy of the same sizes was prepared and freed just before, so a
    read that overtakes the prepare finds a plausible but wrong CSR in the pool block."""
    from tf2_gnn_b200.runtime import PreparedBatch
    V, D, H, L = 3000, 64, 64, 3
    c = _MP("rgcn", _rgcn_params(H, "mean", normalize=True), V, D, L, 9000, seed=15, hub=True)

    def ref_run():
        pb = PreparedBatch(c.adj, V)
        with torch.no_grad():
            fwd = c.layer(c.inp, prepared=pb)
        pb.transposed()
        return pb, [fwd, *c.step(prepared=pb), pb.in_degree(), *pb.csr()]

    _, ref = ref_run()
    ref = [r.clone() for r in ref]
    decoy = tuple(torch.from_numpy(a).cuda() for a in _decoy(np.random.default_rng(16), c.adjs, V))
    d = PreparedBatch(decoy, V)
    d.transposed()
    del d
    torch.cuda.synchronize()
    A, B, C, Dst, E = (torch.cuda.Stream() for _ in range(5))
    with torch.cuda.stream(A):
        torch.cuda._sleep(SLEEP_CYCLES)
        ev = torch.cuda.Event()
        ev.record()
        pb = PreparedBatch(c.adj, V)
    with torch.cuda.stream(B), torch.no_grad():
        fwd = c.layer(c.inp, prepared=pb)
    with torch.cuda.stream(C):
        pb.transposed()
        step = c.step(prepared=pb)
    with torch.cuda.stream(Dst):
        deg = pb.in_degree()
    with torch.cuda.stream(E):
        csr = pb.csr()
    _assert_window_open(ev)
    torch.cuda.synchronize()
    got = [fwd, *step, deg, *csr]
    names = ["forward on B", "training forward on C", "grad_h"] + [f"grad_W{l}" for l in range(L)] + \
            ["in_degree on D", "row_ptr on E", "src_sorted on E"]
    for n, a, b in zip(names, ref, got):
        assert torch.equal(a, b), f"{n} differs from the single-stream run"
    assert np.array_equal(_np(deg), mo.calculate_type_to_num_incoming_edges(V, c.adjs))


def test_free_after_a_read_on_another_stream():
    """A read on B behind a sleep, then the batch is freed and a decoy of the same sizes prepared on A: the free must wait
    for B's read, or the decoy's CSR lands in the block B is about to read."""
    from tf2_gnn_b200.runtime import PreparedBatch
    rng = np.random.default_rng(17)
    V, L = 4000, 3
    adjs = random_graph(rng, V, L, 12000, hub=True)
    adj = tuple(torch.from_numpy(a).cuda() for a in adjs)
    decoy = tuple(torch.from_numpy(a).cuda() for a in _decoy(rng, adjs, V))
    expected = mo.calculate_type_to_num_incoming_edges(V, adjs)
    A, B = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(A):
        pb = PreparedBatch(adj, V)
        assert np.array_equal(_np(pb.in_degree()), expected)
    torch.cuda.synchronize()
    with torch.cuda.stream(B):
        torch.cuda._sleep(SLEEP_CYCLES)
        ev = torch.cuda.Event()
        ev.record()
        deg = pb.in_degree()
        row_ptr, _ = pb.csr()
    del pb                                   # tfgnn_b200_free_batch
    with torch.cuda.stream(A):
        d = PreparedBatch(decoy, V)
    _assert_window_open(ev)
    torch.cuda.synchronize()
    assert np.array_equal(_np(deg), expected), "in_degree read a CSR freed and reused before the read ran"
    counts = np.concatenate([np.bincount(a[:, 1], minlength=V) for a in adjs])
    assert np.array_equal(_np(row_ptr), np.concatenate([[0], np.cumsum(counts)]).astype(np.int32))
    del d


# ---- 4: concurrent batches ------------------------------------------------------------------------------------------------
def test_four_batches_run_concurrently_on_four_streams():
    """Two persistent fused RGCN kernels (row tiling with more tiles than SMs, and the multi-pass H = 320 form), RGAT with a
    hub and GGNN, each on its own stream and graph, forward and backward interleaved for three rounds without a host sync.
    The fused kernels have a static tile assignment and no dependency between clusters, so co-running them must not wait
    on each other: the host waits with a deadline."""
    pg = mo.default_hyperparameters("ggnn")
    pg["hidden_dim"] = 64
    pa = mo.default_hyperparameters("rgat")
    pa.update(hidden_dim=48, num_heads=3, message_activation_function="tanh")
    cases = [_MP("rgcn", _rgcn_params(256), 20000, 128, 3, 60000, seed=18, path="fused_tc"),
             _MP("rgcn", _rgcn_params(320, "mean", normalize=True), 6000, 64, 3, 20000, seed=19, path="fused_tc", hub=True),
             _MP("rgat", pa, 900, 32, 2, 6000, seed=20, hub=True),
             _MP("ggnn", pg, 3000, 64, 3, 9000, seed=21)]
    ref = [[r.clone() for r in c.step()] for c in cases]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in cases]
    rounds = []
    for _ in range(3):
        row = []
        for c, s in zip(cases, streams):
            with torch.cuda.stream(s):
                row.append(c.step())
        rounds.append(row)
    done = []
    for s in streams:
        ev = torch.cuda.Event()
        ev.record(s)
        done.append(ev)
    deadline = time.monotonic() + 60.0
    while not all(e.query() for e in done):
        if time.monotonic() > deadline:
            pytest.fail("the concurrent batches did not finish within 60 s: kernels on different streams wait on each other")
        time.sleep(0.005)
    torch.cuda.synchronize()
    for r, row in enumerate(rounds):
        for i, (want, got) in enumerate(zip(ref, row)):
            for j, (a, b) in enumerate(zip(want, got)):
                assert torch.equal(a, b), f"round {r}, batch {i} ({cases[i].kind}), result {j} differs from the sequential run"


# ---- 5: HostPipeline -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("depth", [1, 2, 3])
def test_host_pipeline_returns_each_steps_own_result(depth):
    """bench.py's end-to-end layer (RGCN, fused path, D = H = 256, 4 edge types, 5 edges per node) at reduced V over a
    sequence of distinct host batches: every out_host equals the device-resident call on that batch, bitwise."""
    from tf2_gnn_b200.layers import MessagePassingInput
    from tf2_gnn_b200.runtime import HostPipeline
    rng = np.random.default_rng(22 + depth)
    D = H = 256
    L = 4
    p = _rgcn_params(H, act="relu")
    layer = make_layer("rgcn", p, D, L, mo.make_weights("rgcn", p, D, L, rng))
    steps = []
    for i in range(6):
        V = 12000 - 1500 * i
        h = torch.from_numpy(rng.uniform(-1, 1, (V, D)).astype(np.float32)).pin_memory()
        adj = tuple(torch.from_numpy(rng.integers(0, V, size=(5 * V, 2)).astype(np.int32)).pin_memory() for _ in range(L))
        steps.append((MessagePassingInput(h, adj), torch.empty((V, H), dtype=torch.float32).pin_memory()))
    with torch.no_grad():
        want = [_np(layer(MessagePassingInput(b.node_embeddings.cuda(), tuple(a.cuda() for a in b.adjacency_lists))))
                for b, _ in steps]
        pipe = HostPipeline(lambda b: layer(b), depth=depth)
        for b, out_host in steps:
            pipe.submit(b, out_host)
        pipe.drain()
    for i, ((_, out_host), w) in enumerate(zip(steps, want)):
        assert np.array_equal(out_host.numpy(), w), f"step {i}: out_host is not that step's result"


# ---- 6: host threads -----------------------------------------------------------------------------------------------------
def test_two_host_threads_train_concurrently_and_keep_their_own_errors():
    """Two threads, each with its own stream and batches, run training steps at once (ctypes releases the GIL, so the calls
    overlap) while a third keeps failing an argument check: results equal the sequential runs bitwise, and every thread's
    exception carries its own message (tfgnn_b200_last_error is thread-local)."""
    from tf2_gnn_b200 import _ffi
    pg = mo.default_hyperparameters("ggnn")
    pg["hidden_dim"] = 64
    cases = [_MP("rgcn", _rgcn_params(128, "mean", normalize=True), 5000, 128, 3, 20000, seed=30, hub=True),
             _MP("ggnn", pg, 3000, 64, 3, 9000, seed=31)]
    ref = [[r.clone() for r in c.step()] for c in cases]
    torch.cuda.synchronize()
    n_steps = 5
    results = [[] for _ in cases]
    errors = []
    stop = threading.Event()
    dummy = torch.zeros(16, device="cuda")

    def worker(i):
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                for _ in range(n_steps):
                    results[i].append(cases[i].step())
                    with pytest.raises(ValueError) as e:   # an error of this thread's own
                        _ffi.check(_ffi.lib().tfgnn_b200_axpby(dummy.data_ptr(), 1.0, None, 0.0, -1 - i, dummy.data_ptr(),
                                                               s.cuda_stream))
                    assert "negative size" in str(e.value), str(e.value)
                s.synchronize()
        except BaseException as e:  # noqa: BLE001  (reported by the main thread)
            errors.append(e)

    def failer():
        n = 0
        try:
            while not stop.is_set() or n < 50:
                with pytest.raises(ValueError) as e:
                    _ffi.check(_ffi.lib().tfgnn_b200_activation(dummy.data_ptr(), 16, 99, dummy.data_ptr(), None))
                assert "bad activation arguments" in str(e.value), str(e.value)
                n += 1
        except BaseException as e:  # noqa: BLE001
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(i,)) for i in range(len(cases))]
    f = threading.Thread(target=failer)
    f.start()
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    stop.set()
    f.join()
    torch.cuda.synchronize()
    assert not errors, errors
    for i, runs in enumerate(results):
        assert len(runs) == n_steps
        for k, run in enumerate(runs):
            for j, (a, b) in enumerate(zip(ref[i], run)):
                assert torch.equal(a, b), f"thread {i}, step {k}, result {j} differs from the sequential run"
