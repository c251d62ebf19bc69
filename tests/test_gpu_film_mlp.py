"""GNN-FiLM with hidden FiLM-MLP layers (film_parameter_MLP_hidden_layers): the hidden chain runs at node level and its last
activation feeds tfgnn_b200_film_in_fwd / _bwd.  Inference against the oracle (both forward forms, target-range shards),
training against float64 autograd of the reference's per-edge op order, exactly on integer data, the entry's shard
contributions, memory that does not grow with the edge count, and a task model end to end."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

import reference64_film_mlp as rfm  # noqa: E402
from oracle import message_passing_oracle as mo  # noqa: E402
from test_gpu_parity import _need_gpu, assert_states_close, make_layer, random_graph  # noqa: E402

pytestmark = pytest.mark.gpu

TOL = 3e-5   # the FiLM gradients' norm-wise bar (test_gpu_film_backward.py)
FUSED = "_FilmInLayerFunctionBackward"


def _hidden_list(hidden, H):
    """An int is that many hidden layers of width 2H (dpu_utils' MLP); the oracle takes the list."""
    return [2 * H] * hidden if isinstance(hidden, int) else list(hidden)


def _setup(hidden, V, D, H, L, E, seed, *, empty=None, hub=False, ints=False, quantize=False, **hyper):
    rng = np.random.default_rng(seed)
    adjs = random_graph(rng, V, L, E, empty_type=empty, hub=hub, dups=True,
                        self_loops=hyper.get("use_target_state_as_input", False))
    p = mo.default_hyperparameters("gnn_film")
    p.update(hidden_dim=H, **hyper)
    w = mo.make_weights("gnn_film", dict(p, film_parameter_MLP_hidden_layers=_hidden_list(hidden, H)), D, L, rng)
    if ints:
        w = {k: [[rng.integers(-1, 2, m.shape).astype(np.float32) for m in ms] for ms in v] for k, v in w.items()}
        h = rng.integers(-1, 2, (V, D)).astype(np.float32)
        g = rng.integers(-1, 2, (V, H)).astype(np.float32)
    else:
        h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
        g = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    if quantize:   # h in multiples of 1/8, hidden FiLM kernels in multiples of 1/64 (relu_quantum)
        h = np.round(h * 8) / 8
        w["film_mlps"] = [[np.round(m * 64) / 64 for m in ms[:-1]] + [ms[-1]] for ms in w["film_mlps"]]
    p["film_parameter_MLP_hidden_layers"] = hidden
    return p, w, h, g, adjs


def _layer(p, w, D, L, train=False):
    layer = make_layer("gnn_film", p, D, L, w)
    if train:
        for v in layer.variables:
            v.requires_grad_()
    return layer


def _oracle(p, w, h, adjs, H):
    return mo.message_passing_forward("gnn_film", dict(p, film_parameter_MLP_hidden_layers=_hidden_list(
        p["film_parameter_MLP_hidden_layers"], H)), w, h, adjs, dtype=np.float64)


# ---- 1. inference ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("att", ["0", "1"])
@pytest.mark.parametrize("hidden,extra", [
    ([16], {}),
    ([48, 24], dict(use_target_state_as_input=True, normalize_by_num_incoming=True)),
    (1, dict(aggregation_function="mean", message_activation_function="gelu")),
    ([30], dict(normalize_by_num_incoming=True, aggregation_function="sqrt_n")),
    ([16], dict(num_edge_MLP_hidden_layers=1, use_target_state_as_input=True)),
    ([48, 24], dict(aggregation_function="max")),
    ([16], dict(message_activation_before_aggregation=True, message_activation_function="tanh")),
    ([30], dict(num_edge_MLP_hidden_layers=2, aggregation_function="max", message_activation_before_aggregation=True)),
])
def test_film_mlp_inference_matches_oracle(monkeypatch, att, hidden, extra):
    _need_gpu()
    from tf2_gnn_b200.layers import MessagePassingInput
    monkeypatch.setenv("TFGNN_B200_FILM_ATT", att)
    V, D, H, L = 500, 64, 64, 4
    p, w, h, _, adjs = _setup(hidden, V, D, H, L, 3000, 8, empty=2, hub=True, **extra)
    layer = _layer(p, w, D, L)
    with torch.no_grad():
        out = layer(MessagePassingInput(torch.from_numpy(h).cuda(), tuple(torch.from_numpy(a).cuda() for a in adjs)))
    assert_states_close(out.cpu().numpy(), _oracle(p, w, h, adjs, H))


@pytest.mark.parametrize("hidden,extra", [([16], dict(use_target_state_as_input=True)),
                                          ([30], dict(normalize_by_num_incoming=True)),
                                          (1, dict(num_edge_MLP_hidden_layers=1))])
def test_film_mlp_target_range_shards_match_oracle(hidden, extra):
    """Worlds of 2 and 3: the concatenated shard rows meet the oracle, and unfiltered and pre-filtered edge lists give the
    same bits (as test_gpu_parity.test_target_range_shards_match_full)."""
    _need_gpu()
    from tf2_gnn_b200 import sharding
    from tf2_gnn_b200.layers import MessagePassingInput
    from tf2_gnn_b200.runtime import PreparedBatch
    V, D, H, L = 700, 64, 64, 3
    p, w, h, _, adjs = _setup(hidden, V, D, H, L, 5000, 21, hub=True, **extra)
    layer = _layer(p, w, D, L)
    ref = _oracle(p, w, h, adjs, H)
    ht = torch.from_numpy(h).cuda()
    adj_t = tuple(torch.from_numpy(a).cuda() for a in adjs)
    deg = sum(np.bincount(a[:, 1], minlength=V) for a in adjs)
    with torch.no_grad():
        for world in (2, 3):
            parts = []
            for lo, hi in sharding.partition_target_range(V, world, deg):
                got = {}
                for filtered in (False, True):
                    a_in = adj_t if not filtered else tuple(
                        torch.from_numpy(a).cuda() for a in sharding.filter_edges_by_target(adjs, lo, hi))
                    out = layer(MessagePassingInput(ht, a_in), prepared=PreparedBatch(a_in, V, target_range=(lo, hi)))
                    assert tuple(out.shape) == (hi - lo, H)
                    got[filtered] = out.cpu().numpy()
                assert np.array_equal(got[False], got[True])
                parts.append(got[True])
            assert_states_close(np.concatenate(parts, axis=0), ref)


# ---- 2. training against float64 -----------------------------------------------------------------------------------
def _params(layer):
    return ([v for m in layer._edge_type_mlps for v in m.layers]
            + [v for m in layer._edge_type_film_layer_computations for v in m.layers])


def _run(layer, h, adjs, g):
    from tf2_gnn_b200.layers import MessagePassingInput
    ht = torch.from_numpy(h).cuda().requires_grad_()
    for q in _params(layer):
        q.value.grad = None
    out = layer(MessagePassingInput(ht, tuple(torch.from_numpy(a).cuda() for a in adjs)))
    assert type(out.grad_fn).__name__ == FUSED
    out.backward(torch.from_numpy(g).cuda())
    torch.cuda.synchronize()
    return out.detach().cpu().numpy(), ht.grad.cpu().numpy(), [q.value.grad.cpu().numpy() for q in _params(layer)]


def _autograd64(p, w, h, adjs, g):
    t = lambda a: torch.from_numpy(np.asarray(a)).double().requires_grad_()
    h64 = t(h)
    E64 = [[t(m) for m in ms] for ms in w["edge_mlps"]]
    F64 = [[t(m) for m in ms] for ms in w["film_mlps"]]
    out = rfm.film_mlp_autograd(h64, [torch.from_numpy(a) for a in adjs], E64, F64, agg=p["aggregation_function"],
                                act=p["message_activation_function"], normalize=p["normalize_by_num_incoming"],
                                use_target=p["use_target_state_as_input"])
    out.backward(torch.from_numpy(g).double())
    return (out.detach().numpy(), h64.grad.numpy(),
            [x.grad.numpy() for ms in E64 for x in ms] + [x.grad.numpy() for ms in F64 for x in ms])


TRAIN_CASES = [   # hidden, V, D, H, L, E, agg, act, normalize, use_target, empty, hub, seed
    ([16], 600, 32, 36, 3, 4000, "sum", "tanh", False, False, None, False, 1),
    ([48, 24], 600, 32, 36, 3, 4000, "mean", "gelu", True, False, 1, True, 2),
    (1, 800, 64, 32, 4, 5000, "sqrt_n", "elu", False, True, 2, True, 3),
    ([20], 800, 64, 96, 4, 5000, "sum", None, True, True, None, True, 4),
]


def _train_case(case, **over):
    hidden, V, D, H, L, E, agg, act, normalize, use_target, empty, hub, seed = case
    return _setup(hidden, V, D, H, L, E, seed, empty=empty, hub=hub, quantize=True, aggregation_function=agg,
                  message_activation_function=act, normalize_by_num_incoming=normalize,
                  use_target_state_as_input=use_target, **over)


def relu_quantum(w, h):
    """With quantised h and hidden FiLM kernels every hidden pre-activation is a short dyadic number that float32 holds
    exactly.  Checks that, and returns the smallest non-zero |pre-activation|.  Exact zeros occur (the values are
    discrete); gpu_chain_is_exact shows that the GPU's hidden chain reproduces every value, zeros included, so both sides
    see the same ReLU masks."""
    pre = rfm.hidden_preactivations(torch.from_numpy(h).double(),
                                    [[torch.from_numpy(m).double() for m in ms] for ms in w["film_mlps"]])
    smallest = np.inf
    for x in pre.values():
        x = x.numpy()
        assert np.array_equal(x, x.astype(np.float32).astype(np.float64))
        assert np.abs(x).max() < 2.0 ** 8
        nz = np.abs(x[x != 0])
        smallest = min(smallest, float(nz.min()))
    return smallest


def gpu_chain_is_exact(w, h):
    """Every hidden layer of every FiLM MLP through node_ops.dense (the 3xTF32 GEMM with the ReLU in its epilogue) equals
    relu of the float64 product of its own input bit for bit.  The backward's mask comes from that output (> 0), so it
    equals the float64 reference's mask, exact zeros included."""
    from tf2_gnn_b200.layers.node_ops import dense
    from tf2_gnn_b200.utils.param_helpers import get_activation_function
    relu = get_activation_function("relu")
    for ms in w["film_mlps"]:
        x = torch.from_numpy(h).cuda()
        for m in ms[:-1]:
            with torch.no_grad():
                y = dense(x, torch.from_numpy(m).cuda(), None, relu)
            exact = torch.relu(x.double().cpu() @ torch.from_numpy(m).double())
            if not torch.equal(y.cpu().double(), exact):
                return False
            x = y
    return True


@pytest.mark.parametrize("case", TRAIN_CASES)
def test_film_mlp_training_matches_float64_autograd(case):
    _need_gpu()
    from tf2_gnn_b200.layers import MessagePassingInput
    p, w, h, g, adjs = _train_case(case)
    assert relu_quantum(w, h) >= 2.0 ** -15   # float32 rounding of these pre-activations is exactly 0
    assert gpu_chain_is_exact(w, h)
    D, L = h.shape[1], len(adjs)
    layer = _layer(p, w, D, L, train=True)
    got = _run(layer, h, adjs, g)
    ref = _autograd64(p, w, h, adjs, g)
    assert_states_close(got[0], ref[0], tol=TOL)
    assert_states_close(got[1], ref[1], tol=TOL)
    assert len(got[2]) == len(ref[2])
    for a, b in zip(got[2], ref[2]):
        assert_states_close(a, b, tol=TOL)
    again = _run(layer, h, adjs, g)   # a second backward gives the same bits
    assert np.array_equal(got[0], again[0]) and np.array_equal(got[1], again[1])
    assert all(np.array_equal(a, b) for a, b in zip(got[2], again[2]))
    with torch.no_grad():             # the training forward gives the inference forward's bits
        inf = layer(MessagePassingInput(torch.from_numpy(h).cuda(), tuple(torch.from_numpy(a).cuda() for a in adjs)))
    assert np.array_equal(inf.cpu().numpy(), got[0])


# ---- 3. exact integer data -----------------------------------------------------------------------------------------
def _node_level_abs_peak(w, h, g, adjs, use_target):
    """The largest entry of every node-level table and gradient of the fused computation, evaluated on |h|, |W|, |F|,
    |grad_out| with identity activations (ReLU is the identity there).  All terms are then non-negative, so every partial
    sum the kernels form is bounded by one of these tables."""
    t = lambda a: torch.from_numpy(np.abs(np.asarray(a, np.float64))).requires_grad_()
    V = h.shape[0]
    ha = t(h)
    Ws = [t(ms[0]) for ms in w["edge_mlps"]]
    Fs = [[t(m) for m in ms] for ms in w["film_mlps"]]
    tables = []

    def keep(x):
        x.retain_grad()
        tables.append(x)
        return x

    Z = 0
    for adj, W, F in zip(adjs, Ws, Fs):
        src, tgt = torch.from_numpy(adj[:, 0]).long(), torch.from_numpy(adj[:, 1]).long()
        c = torch.bincount(tgt, minlength=V).double()
        A = keep(torch.zeros_like(ha).index_add(0, tgt, ha.index_select(0, src)))
        X = keep(torch.cat([A, c[:, None] * ha], dim=1)) if use_target else A
        Q = keep(X @ W)
        z = ha
        for Fk in F[:-1]:
            z = keep(z @ Fk)
        GB = keep(z @ F[-1])
        H = GB.shape[1] // 2
        Z = Z + GB[:, :H] * Q + c[:, None] * GB[:, H:]
        Z = keep(Z)
    (Z * torch.from_numpy(np.abs(g).astype(np.float64))).sum().backward()
    peak = max(float(x.detach().abs().max()) for x in tables)
    peak = max([peak, float(ha.grad.max())] + [float(x.grad.max()) for x in tables if x.grad is not None]
               + [float(x.grad.max()) for x in Ws] + [float(x.grad.max()) for F in Fs for x in F])
    return peak


@pytest.mark.parametrize("hidden,V,D,H,L,E,use_target", [([16], 3000, 32, 48, 3, 15000, False),
                                                         ([8, 8], 2000, 16, 16, 3, 8000, True)])
def test_film_mlp_exact_on_integer_data(hidden, V, D, H, L, E, use_target):
    """sum / relu / no normalisation with h, W, F and grad_out in {-1, 0, 1}: once every partial sum is shown to stay below
    2^24, every output and gradient must equal float32(reference) bit for bit."""
    _need_gpu()
    p, w, h, g, adjs = _setup(hidden, V, D, H, L, E, V + L, empty=1, ints=True, aggregation_function="sum",
                              message_activation_function="relu", normalize_by_num_incoming=False,
                              use_target_state_as_input=use_target)
    adjs[0][:300, 1] = V // 3    # an in-degree hub
    adjs[-1][:300, 0] = 7        # an out-degree hub
    assert _node_level_abs_peak(w, h, g, adjs, use_target) < 2 ** 24
    layer = _layer(p, w, D, L, train=True)
    got = _run(layer, h, adjs, g)
    ref = _autograd64(p, w, h, adjs, g)
    f32 = lambda a: np.asarray(a).astype(np.float32)
    assert np.array_equal(got[0], f32(ref[0]))
    assert np.array_equal(got[1], f32(ref[1]))
    for a, b in zip(got[2], ref[2]):
        assert np.array_equal(a, f32(b))


# ---- 4. the entry's shard contributions ----------------------------------------------------------------------------
def _entry(pb, h, film_in, S, Ws, Fs, H, flags, agg, act, grad_out):
    """tfgnn_b200_film_in_fwd then _bwd on one prepared batch: (out, grad_h, grad_film_in, grad_W, grad_F)."""
    from tf2_gnn_b200 import _ffi
    from tf2_gnn_b200.runtime import stream_ptr
    L = len(Ws)
    out = torch.empty((pb.num_nodes, H), device="cuda")
    lib = _ffi.lib()
    _ffi.check(lib.tfgnn_b200_film_in_fwd(pb.handle, h.data_ptr(), int(h.shape[1]), _ffi.ptr_array(Ws), 0,
                                          film_in.data_ptr(), S, _ffi.ptr_array(Fs), H, flags, agg, act, 0,
                                          out.data_ptr(), stream_ptr()))
    gh, gin = torch.empty_like(h), torch.empty_like(film_in)
    gW, gF = [torch.empty_like(x) for x in Ws], [torch.empty_like(x) for x in Fs]
    _ffi.check(lib.tfgnn_b200_film_in_bwd(pb.handle, pb.transposed().handle, h.data_ptr(), int(h.shape[1]),
                                          _ffi.ptr_array(Ws), film_in.data_ptr(), S, _ffi.ptr_array(Fs), H, flags, agg,
                                          act, out.data_ptr(), grad_out.contiguous().data_ptr(), gh.data_ptr(),
                                          gin.data_ptr(), _ffi.ptr_array(gW), _ffi.ptr_array(gF), stream_ptr()))
    torch.cuda.synchronize()
    return [x.cpu().numpy() for x in [out, gh, gin] + gW + gF]


@pytest.mark.parametrize("S,agg,act,normalize,use_target", [(16, "mean", "tanh", True, True), (40, "sum", "gelu", False, False),
                                                            (24, "sqrt_n", "elu", True, False)])
def test_film_in_bwd_shard_contributions_sum_to_full(S, agg, act, normalize, use_target):
    _need_gpu()
    from tf2_gnn_b200 import _ffi, sharding
    from tf2_gnn_b200.runtime import PreparedBatch
    rng = np.random.default_rng(S + len(agg))
    V, D, H, L = 700, 32, 48, 3
    adjs = random_graph(rng, V, L, 5000, hub=True, dups=True, self_loops=use_target)
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()
    h = cu(rng.uniform(-1, 1, (V, D)))
    film_in = cu(rng.uniform(0, 1, (V, L * S)))
    Ws = [cu(mo.glorot_uniform(rng, ((2 if use_target else 1) * D, H))) for _ in range(L)]
    Fs = [cu(mo.glorot_uniform(rng, (S, 2 * H))) for _ in range(L)]
    g = cu(rng.uniform(-1, 1, (V, H)))
    flags = (_ffi.FLAG_NORMALIZE if normalize else 0) | (_ffi.FLAG_USE_TARGET if use_target else 0)
    args = (S, Ws, Fs, H, flags, _ffi.AGG[agg], _ffi.ACT[act])
    adj_t = tuple(torch.from_numpy(a).cuda() for a in adjs)
    full = _entry(PreparedBatch(adj_t, V), h, film_in, *args, g)
    deg = sum(np.bincount(a[:, 1], minlength=V) for a in adjs)
    worlds = [sharding.partition_target_range(V, n, deg) for n in (2, 3)] + [[(0, 300), (300, 300), (300, V)]]
    for bounds in worlds:
        sums = [np.zeros_like(x, dtype=np.float64) for x in full[1:2] + full[3:]]
        gin_rows = []
        for lo, hi in bounds:
            pb = PreparedBatch(adj_t, V, target_range=(lo, hi))
            got = _entry(pb, h, film_in[lo:hi].contiguous(), *args, g[lo:hi])
            again = _entry(pb, h, film_in[lo:hi].contiguous(), *args, g[lo:hi])
            assert all(np.array_equal(a, b) for a, b in zip(got, again))
            if hi == lo:
                assert not got[1].any() and not any(x.any() for x in got[3:])
            gin_rows.append(got[2])
            for s, x in zip(sums, got[1:2] + got[3:]):
                s += x
        assert_states_close(np.concatenate(gin_rows, axis=0), full[2].astype(np.float64), tol=TOL)
        for s, x in zip(sums, full[1:2] + full[3:]):
            assert_states_close(s, x.astype(np.float64), tol=TOL)


# ---- 5. memory -----------------------------------------------------------------------------------------------------
def test_film_mlp_training_memory_does_not_grow_with_edges():
    """A training step with [H] hidden FiLM layers: the rise in device memory in use (torch and the library's pool,
    trimmed first) on a graph and on the same nodes with four times the edges."""
    _need_gpu()
    import gc
    from tf2_gnn_b200 import _ffi
    from tf2_gnn_b200.layers import MessagePassingInput
    from tf2_gnn_b200.runtime import PreparedBatch, clear_prepared_batch_cache
    V, D, H, L, E = 200_000, 64, 64, 3, 400_000
    rises = []
    for mult in (1, 4):
        p, w, _, _, _ = _setup([H], 10, D, H, L, 10, 3)
        layer = _layer(p, w, D, L, train=True)
        gen = torch.Generator(device="cuda")
        gen.manual_seed(mult)
        adj = tuple(torch.randint(0, V, (mult * E, 2), generator=gen, device="cuda", dtype=torch.int32) for _ in range(L))
        h = (torch.rand((V, D), generator=gen, device="cuda") * 2 - 1).requires_grad_()
        g = torch.rand((V, H), generator=gen, device="cuda") * 2 - 1
        prepared = PreparedBatch(adj, V)
        prepared.transposed()
        clear_prepared_batch_cache()
        gc.collect()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        _ffi.lib().tfgnn_b200_release_device_state()
        free0, _ = torch.cuda.mem_get_info()
        out = layer(MessagePassingInput(h, adj), prepared=prepared)
        assert type(out.grad_fn).__name__ == FUSED
        out.backward(g)
        torch.cuda.synchronize()
        free1, _ = torch.cuda.mem_get_info()
        rises.append(free0 - free1)
        del out, prepared, adj, h, g, layer
    assert rises[1] <= 1.1 * rises[0] + (32 << 20), rises


# ---- 6. a task model end to end ------------------------------------------------------------------------------------
def test_node_multiclass_task_with_film_mlp_trains_validates_and_predicts():
    _need_gpu()
    import random
    from test_gpu_task_models import _load_jsonl
    from tf2_gnn_b200.data import DeviceGraphStore
    from tf2_gnn_b200.models import NodeMulticlassTask
    random.seed(0)
    np.random.seed(0)
    torch.manual_seed(0)
    rng = np.random.default_rng(0)
    samples, T = _load_jsonl("train.jsonl.gz")
    for s in samples:
        n = len(s["node_features"])
        s["node_labels"] = (rng.uniform(size=(n, 5)) < 0.3).astype(np.float32)
    store = DeviceGraphStore(samples, T)
    params = NodeMulticlassTask.get_default_hyperparameters("gnn_film")
    params.update(gnn_hidden_dim=32, gnn_num_layers=2, gnn_global_exchange_every_num_layers=10000,
                  gnn_film_parameter_MLP_hidden_layers=[32], optimizer="Adam", learning_rate=0.005)
    model = NodeMulticlassTask(params, dataset=store)
    order = np.random.permutation(store.num_graphs)
    train_loss, _, _ = model.run_one_epoch(store, store.iter_batch_graph_ids(10000, order), training=True)
    valid_loss, _, results = model.run_one_epoch(store, store.iter_batch_graph_ids(10000), training=False)
    assert np.isfinite(train_loss) and np.isfinite(valid_loss)
    assert np.isfinite(model.compute_epoch_metrics(results)[0])
    preds = model.predict(store, store.iter_batch_graph_ids(10000))
    preds = preds.cpu().numpy() if hasattr(preds, "cpu") else np.asarray(preds)
    assert preds.shape[0] == sum(len(s["node_features"]) for s in samples) and np.isfinite(preds).all()
