"""The task models (NodeMulticlassTask, GraphRegressionTask, GraphBinaryClassificationTask) trained on target-range shards:
every rank is a spawned process on one GPU, joined over gloo with host-staged collectives (NCCL refuses two ranks on one
device; the library's collectives all go through sharding.all_gather_into_tensor / reduce_scatter_tensor, which the workers
replace).

Each rank builds its model from a different seed and takes rank 0's weights with sharding.broadcast_variables, assembles
its part of the batch with store.shard_batch, and runs train_step(shard=...).  Rank 0 also runs the unsharded step.  The
tests check that loss and metrics hold the same bits on every rank and match the unsharded step (F1 counts and the number
of correct predictions exactly), that the summed gradients hold the same bits on every rank and match the unsharded ones,
that one SGD step matches and three Adam steps with global-norm clipping keep every rank on the same bits, run after run;
and that the row-window batch holds what the sharded layers need."""
import gzip
import json
import os
import socket
import sys

import numpy as np
import pytest

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu
TOL = 3e-5
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


# ---- host-staged collectives (gloo moves host tensors) ---------------------------------------------------------------
def _host_all_gather_into_tensor(out, inp, group=None):
    import torch.distributed as dist
    world = dist.get_world_size(group)
    src = inp.detach().contiguous().cpu()
    parts = [torch.empty_like(src) for _ in range(world)]
    dist.all_gather(parts, src, group=group)
    out.copy_(torch.cat([p.reshape(-1) for p in parts]).reshape(out.shape))


def _host_reduce_scatter_tensor(out, inp, group=None):
    import torch.distributed as dist
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    src = inp.detach().contiguous().cpu()
    parts = [torch.empty_like(src) for _ in range(world)]
    dist.all_gather(parts, src, group=group)
    acc = parts[0].reshape(world, -1)[rank].clone()
    for p in parts[1:]:
        acc += p.reshape(world, -1)[rank]
    out.copy_(acc.reshape(out.shape))


# ---- the cases -----------------------------------------------------------------------------------------------------
PPI = dict(gnn_hidden_dim=64, gnn_layer_input_dropout_rate=0.1, gnn_dense_every_num_layers=10000,
           gnn_global_exchange_every_num_layers=10000, gnn_initial_node_representation_activation="tanh",
           gnn_dense_intermediate_layer_activation="tanh", gnn_aggregation_function="sum")
CASES = [
    dict(name="ppi_rgcn", task="node", style="rgcn",
         hyper=dict(PPI, gnn_num_layers=4, gnn_normalize_by_num_incoming=True, gnn_num_edge_MLP_hidden_layers=0,
                    gnn_residual_every_num_layers=10000, gnn_use_inter_layer_layernorm=False,
                    gnn_message_activation_function="relu")),
    dict(name="ppi_rgin", task="node", style="rgin",
         hyper=dict(PPI, gnn_num_layers=5, gnn_normalize_by_num_incoming=True, gnn_num_edge_MLP_hidden_layers=1,
                    gnn_num_aggr_MLP_hidden_layers=None, gnn_residual_every_num_layers=2,
                    gnn_use_inter_layer_layernorm=True, gnn_message_activation_function="relu")),
    dict(name="ppi_rgat", task="node", style="rgat",
         hyper=dict(PPI, gnn_num_layers=3, gnn_num_heads=4, gnn_residual_every_num_layers=10000,
                    gnn_use_inter_layer_layernorm=False, gnn_message_activation_function="tanh")),
    dict(name="regression_defaults", task="regression", style=None, hyper={}),
    dict(name="binary_defaults", task="binary", style=None, hyper={}),
]
SGD_LR = 0.05
METRICS = ("loss", "f1_score", "f1_counts", "mae", "num_correct")


def _store(case, seed):
    from tf2_gnn_b200.data import DeviceGraphStore
    rng = np.random.default_rng(seed)
    node_task = case["task"] == "node"
    num_graphs, (n_lo, n_hi), F, L = (3, (250, 400), 50, 3) if node_task else (40, (9, 30), 15, 3)
    graphs = []
    for _ in range(num_graphs):
        n = int(rng.integers(n_lo, n_hi))
        s = {"node_features": rng.uniform(-1, 1, (n, F)).astype(np.float32),
             "adjacency_lists": [rng.integers(0, n, (4 * n, 2)).astype(np.int32) for _ in range(L)]}
        if node_task:
            s["node_labels"] = (rng.uniform(size=(n, 121)) < 0.3).astype(np.float32)
        elif case["task"] == "binary":
            s["target_value"] = float(rng.uniform() < 0.5)
        else:
            s["target_value"] = float(rng.normal(3.0, 1.0))
        graphs.append(s)
    return DeviceGraphStore(graphs, L), F


def _model(case, store, F, optimizer, seed):
    from tf2_gnn_b200.models import GraphBinaryClassificationTask, GraphRegressionTask, NodeMulticlassTask
    cls = {"node": NodeMulticlassTask, "regression": GraphRegressionTask, "binary": GraphBinaryClassificationTask}[case["task"]]
    params = cls.get_default_hyperparameters(case["style"])
    params.update(case["hyper"])
    if optimizer == "sgd":
        params.update(optimizer="SGD", learning_rate=SGD_LR, momentum=0.0)
    else:
        params.update(optimizer="Adam", learning_rate=0.01, gradient_clip_global_norm=1.0)
    torch.manual_seed(seed)
    model = cls(params, dataset=store)
    shapes = {"node_features": (None, F)}
    shapes.update({f"adjacency_list_{t}": (None, 2) for t in range(store.num_edge_types)})
    model.build(shapes)
    return model


def _record_gradients(model):
    """The gradients the optimizer step receives (after the sum over ranks), in trainable_variables order."""
    seen = []
    apply = model._apply_gradients

    def recording(pairs):
        pairs = list(pairs)
        seen.append([None if g is None else g.detach().cpu().numpy() for g, _ in pairs])
        apply(pairs)

    model._apply_gradients = recording
    return seen


def _metrics(m):
    out = {"loss": np.array(m["loss"].detach().cpu().numpy())}
    for k in METRICS[1:]:
        if k in m:
            out[k] = np.array(m[k].detach().cpu().numpy())
    return out


def _run(case, seed, shard, rank):
    """(results of one SGD step, parameters after three Adam steps with global-norm clipping); shard None = unsharded."""
    from tf2_gnn_b200 import sharding
    store, F = _store(case, seed)
    ids = np.arange(store.num_graphs)
    if shard is None:
        feats, labels = store.batch(ids), store.batch_labels(ids)
    else:
        feats, labels = store.shard_batch(ids, shard), store.shard_batch_labels(ids, shard)
    res = {}
    model = _model(case, store, F, "sgd", seed + (0 if shard is None else 7 * rank))   # different seeds on every rank
    if shard is not None:
        sharding.broadcast_variables(model.trainable_variables, shard.group)
    res["w0"] = [v.value.detach().cpu().numpy() for v in model.trainable_variables]
    seen = _record_gradients(model)
    for k, v in _metrics(model.train_step(feats, labels, shard=shard)).items():
        res[f"sgd_{k}"] = v
    res["sgd_grads"] = seen[0]
    res["sgd_w1"] = [v.value.detach().cpu().numpy() for v in model.trainable_variables]
    if shard is not None:
        model = _model(case, store, F, "adam", seed + 7 * rank)
        sharding.broadcast_variables(model.trainable_variables, shard.group)
        res["adam_losses"] = np.array([model.train_step(feats, labels, shard=shard)["loss"].item() for _ in range(3)])
        res["adam_w3"] = [v.value.detach().cpu().numpy() for v in model.trainable_variables]
        res["adam_iterations"] = np.array(model._optimizer.iterations)
        slots = [model._optimizer.slots(v.value) for v in model.trainable_variables]
        res["adam_slots"] = [s.cpu().numpy() for pair in slots for s in pair if s is not None]
    return res


def _bounds(kind, store_bounds, V, world):
    if kind == "store":
        return store_bounds
    if kind == "empty":
        cut = V // 3 + 7
        return [(0, cut), (cut, cut), (cut, V)]
    cuts = [0] + [int(V * r / world) + 5 * r + 1 for r in range(1, world)] + [V]   # cuts inside graphs
    return [(cuts[r], cuts[r + 1]) for r in range(world)]


def _check_shard_batch(store, ids, shard):
    """shard_batch against store.batch: rows, labels, the edges filtered by target and the prepared CSR."""
    from tf2_gnn_b200 import sharding
    from tf2_gnn_b200.runtime import PreparedBatch
    lo, hi = shard.lo, shard.hi
    full, full_labels = store.batch(ids), store.batch_labels(ids)
    part, part_labels = store.shard_batch(ids, shard), store.shard_batch_labels(ids, shard)
    checks = {"keys": set(part) == set(full) and part["num_graphs_in_batch"] == full["num_graphs_in_batch"],
              "node_features": torch.equal(part["node_features"], full["node_features"][lo:hi]),
              "node_to_graph_map": torch.equal(part["node_to_graph_map"], full["node_to_graph_map"][lo:hi])}
    for k in full_labels:
        checks[k] = torch.equal(part_labels[k], full_labels[k][lo:hi] if k == "node_labels" else full_labels[k])
    T = store.num_edge_types
    full_adj = [full[f"adjacency_list_{t}"].cpu().numpy() for t in range(T)]
    part_adj = [part[f"adjacency_list_{t}"].cpu().numpy() for t in range(T)]
    filtered = sharding.filter_edges_by_target(full_adj, lo, hi)
    # a superset of the edges filtered by target, in the same order
    checks["edges"] = all(np.array_equal(sharding.filter_edges_by_target([part_adj[t]], lo, hi)[0], filtered[t])
                          for t in range(T))
    Vb = int(full["node_to_graph_map"].shape[0])
    csr_part = PreparedBatch(tuple(part[f"adjacency_list_{t}"] for t in range(T)), Vb, target_range=(lo, hi)).csr()
    csr_filt = PreparedBatch(tuple(torch.from_numpy(a).cuda() for a in filtered), Vb, target_range=(lo, hi)).csr()
    checks["csr_row_ptr"] = torch.equal(csr_part[0], csr_filt[0])
    kept = int(csr_filt[0][-1])                     # the export also copies the unused tail of a list with dropped edges
    checks["csr_sources"] = torch.equal(csr_part[1][:kept], csr_filt[1][:kept])
    extra = sum(len(p) - len(f) for p, f in zip(part_adj, filtered))
    return {k: bool(v) for k, v in checks.items()}, extra


def _world1_loss_bits(group):
    """A world of one: the sharded node loss gives the bits of the unsharded entries (loss, F1, counts, gradient)."""
    from tf2_gnn_b200 import sharding
    from tf2_gnn_b200.models import task_ops
    rng = np.random.default_rng(3)
    x = torch.from_numpy(rng.normal(0, 4, (5000, 121)).astype(np.float32)).cuda()
    y = torch.from_numpy((rng.uniform(size=(5000, 121)) < 0.3).astype(np.float32)).cuda()
    shard = sharding.TargetRangeShard([(0, 5000)], 0, group)
    a, b = x.clone().requires_grad_(), x.clone().requires_grad_()
    got = task_ops.node_multiclass_loss(a, y, shard)
    want = task_ops.node_multiclass_loss(b, y)
    (ga,), (gb,) = torch.autograd.grad(got[0], a), torch.autograd.grad(want[0], b)
    same = all(torch.equal(g, w) for g, w in zip(got, want)) and torch.equal(ga, gb)
    return bool(same)


def _film_raises(rank, world):
    from tf2_gnn_b200 import sharding
    from tf2_gnn_b200.models import NodeMulticlassTask
    store, F = _store(CASES[0], 5)
    ids = np.arange(store.num_graphs)
    shard = sharding.TargetRangeShard(store.shard_bounds(ids, world), rank)
    params = NodeMulticlassTask.get_default_hyperparameters("gnn_film")
    params.update(gnn_hidden_dim=32, gnn_num_layers=2)
    model = NodeMulticlassTask(params, dataset=store)
    try:
        model.train_step(store.shard_batch(ids, shard), store.shard_batch_labels(ids, shard), shard=shard)
    except NotImplementedError:
        return True
    return False


def _load_jsonl(name):
    from tf2_gnn_b200.data import get_tied_edge_types, process_adjacency_lists
    tied = get_tied_edge_types(True, 3)
    num_edge_types = 2 * 3 - len(tied) + 1
    samples = []
    with gzip.open(os.path.join(GOLDEN, name), "rt") as f:
        for line in f:
            d = json.loads(line)
            nf = d["graph"]["node_features"]
            adjs, _ = process_adjacency_lists(d["graph"]["adjacency_lists"], len(nf), True, tied)
            samples.append({"node_features": nf, "adjacency_lists": [a.cpu().numpy() for a in adjs[:num_edge_types]],
                            "target_value": float(d["Property"])})
    return samples, num_edge_types


def _sharded_train_improvement():
    """test_train_improvement (test_gpu_task_models.py) with every epoch on target-range shards over the world."""
    import torch.distributed as dist
    from tf2_gnn_b200 import sharding
    from tf2_gnn_b200.data import DeviceGraphStore
    from tf2_gnn_b200.models import GraphRegressionTask
    np.random.seed(0)
    torch.manual_seed(0)
    train_s, T = _load_jsonl("train.jsonl.gz")
    valid_s, _ = _load_jsonl("valid.jsonl.gz")
    train, valid = DeviceGraphStore(train_s, T), DeviceGraphStore(valid_s, T)
    model = GraphRegressionTask(GraphRegressionTask.get_default_hyperparameters(), dataset=train)
    shapes = {"node_features": (None, int(train.node_features.shape[1]))}
    shapes.update({f"adjacency_list_{t}": (None, 2) for t in range(T)})
    model.build(shapes)
    sharding.broadcast_variables(model.trainable_variables)
    group = dist.group.WORLD

    def epoch(store, training):
        order = np.random.permutation(store.num_graphs) if training else None
        loss, _, results = model.run_one_epoch(store, store.iter_batch_graph_ids(10000, order), training=training,
                                               shard_group=group)
        return loss, model.compute_epoch_metrics(results)[0]

    out = [epoch(valid, False), epoch(train, True), epoch(valid, False), epoch(train, True)]
    return np.array(out, dtype=np.float64)


def _worker(rank, world, port, tmp, cut_kinds):
    import torch.distributed as dist
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        torch.cuda.set_device(0)
        from tf2_gnn_b200 import sharding
        sharding.all_gather_into_tensor = _host_all_gather_into_tensor
        sharding.reduce_scatter_tensor = _host_reduce_scatter_tensor
        results = {}
        for ci, kind in enumerate(cut_kinds):
            for i, case in enumerate(CASES):
                key = f"{kind}/{i}"
                seed = 100 + i
                store, _ = _store(case, seed)
                ids = np.arange(store.num_graphs)
                V = int(store.node_offsets_host[-1])
                bounds = _bounds(kind, store.shard_bounds(ids, world), V, world)
                shard = sharding.TargetRangeShard(bounds, rank)
                results[f"{key}/bounds"] = np.array(bounds)
                checks, extra = _check_shard_batch(store, ids, shard)
                for name, ok in checks.items():
                    results[f"{key}/shard_batch/{name}"] = np.array(ok)
                results[f"{key}/extra_edges"] = np.array(extra)
                got = _run(case, seed, shard, rank)
                again = _run(case, seed, shard, rank)
                same = all(np.array_equal(a, b) for a, b in zip(got["adam_w3"], again["adam_w3"]))
                same &= np.array_equal(got["adam_losses"], again["adam_losses"])
                same &= all(np.array_equal(a, b) for a, b in zip(got["sgd_w1"], again["sgd_w1"]))
                results[f"{key}/rerun_same_bits"] = np.array(same)
                if rank == 0:
                    full = _run(case, seed, None, 0)
                    for k, v in full.items():
                        got[f"full_{k}"] = v
                for k, v in got.items():
                    if isinstance(v, list):
                        results[f"{key}/{k}/n"] = np.array(len(v))
                        for j, a in enumerate(v):
                            if a is not None:
                                results[f"{key}/{k}/{j}"] = a
                    else:
                        results[f"{key}/{k}"] = v
        results["film_raises"] = np.array(_film_raises(rank, world))
        if world == 2:
            solo = dist.new_group([0])                                    # every rank joins the call, rank 0 uses it
            results["world1_loss_bits"] = np.array(_world1_loss_bits(solo) if rank == 0 else True)
            results["train_improvement"] = _sharded_train_improvement()
        np.savez(os.path.join(tmp, f"rank{rank}.npz"), **results)
    finally:
        dist.destroy_process_group()


WORLDS = {"world2": (2, ("store", "inside")), "world3": (3, ("store", "inside")), "world3_empty_shard": (3, ("empty",))}


@pytest.fixture(scope="module")
def worlds(tmp_path_factory):
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import torch.multiprocessing as mp
    out = {}
    for name, (world, kinds) in WORLDS.items():
        tmp = str(tmp_path_factory.mktemp(name))
        mp.spawn(_worker, args=(world, _free_port(), tmp, kinds), nprocs=world, join=True)
        out[name] = [dict(np.load(os.path.join(tmp, f"rank{r}.npz"))) for r in range(world)]
    return out


def close(got, ref, tol=TOL, what="", floor=1e-30):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape, f"{what}: shape {got.shape} vs {ref.shape}"
    err, scale = np.linalg.norm(got - ref), max(np.linalg.norm(ref), floor)
    assert err <= tol * scale, f"{what}: |err| {err:.3e} > {tol:g} * {scale:.3e}"


def _list(r, key):
    n = int(r[f"{key}/n"])
    return [r.get(f"{key}/{j}") for j in range(n)]


RUNS = [(w, kind, i) for w, (_, kinds) in WORLDS.items() for kind in kinds for i in range(len(CASES))]


@pytest.mark.parametrize("world,kind,i", RUNS, ids=[f"{w}-{k}-{CASES[i]['name']}" for w, k, i in RUNS])
def test_sharded_train_step_matches_the_unsharded_step(worlds, world, kind, i):
    ranks = worlds[world]
    r0 = ranks[0]
    key = f"{kind}/{i}"
    bounds = r0[f"{key}/bounds"]
    if kind == "empty":
        assert any(lo == hi for lo, hi in bounds)
    # the row-window batch: rows and labels of store.batch, a superset of the edges filtered by target, the same CSR
    for r in ranks:
        checks = {k.rsplit("/", 1)[1]: bool(v) for k, v in r.items() if k.startswith(f"{key}/shard_batch/")}
        assert len(checks) == 7 and all(checks.values()), checks
    # broadcast_variables: every rank starts from rank 0's bits (built from a different seed), which are the unsharded ones
    for r in ranks:
        for a, b in zip(_list(r, f"{key}/w0"), _list(r0, f"{key}/full_w0")):
            assert np.array_equal(a, b)
    # loss and metrics: the same bits on every rank, the unsharded values (counts exactly)
    metric_keys = [m for m in METRICS if f"{key}/sgd_{m}" in r0]
    assert "loss" in metric_keys
    for m in metric_keys:
        for r in ranks:
            assert np.array_equal(r[f"{key}/sgd_{m}"], r0[f"{key}/sgd_{m}"], equal_nan=True), m
    close(r0[f"{key}/sgd_loss"], r0[f"{key}/full_sgd_loss"], what="loss")
    for m in ("f1_counts", "f1_score", "num_correct"):
        if m in metric_keys:
            assert np.array_equal(r0[f"{key}/sgd_{m}"], r0[f"{key}/full_sgd_{m}"], equal_nan=True), m
    if "mae" in metric_keys:
        close(r0[f"{key}/sgd_mae"], r0[f"{key}/full_sgd_mae"], what="mae")
    # gradients after the sum over ranks: the same bits on every rank, the unsharded gradients at the bar
    grads = _list(r0, f"{key}/sgd_grads")
    wants = _list(r0, f"{key}/full_sgd_grads")
    assert len(grads) == len(wants) and sum(g is not None for g in wants) >= len(wants) - 2
    floor = max(np.linalg.norm(w) for w in wants if w is not None)
    for j, (g, w) in enumerate(zip(grads, wants)):
        for r in ranks:
            gr = _list(r, f"{key}/sgd_grads")[j]
            assert (gr is None) == (g is None) and (g is None or np.array_equal(gr, g)), f"gradient {j} differs between ranks"
        assert (g is None) == (w is None), f"gradient {j}: presence differs from the unsharded step"
        if w is not None:
            close(g, w, what=f"gradient {j}", floor=floor)
    # one SGD step: within the bar of the unsharded step, the same bits on every rank
    for j, (a, b) in enumerate(zip(_list(r0, f"{key}/sgd_w1"), _list(r0, f"{key}/full_sgd_w1"))):
        for r in ranks:
            assert np.array_equal(_list(r, f"{key}/sgd_w1")[j], a)
        close(a, b, what=f"variable {j} after one SGD step", floor=floor * SGD_LR)
    # three Adam steps with global-norm clipping: every rank holds the same variables, slots and step count
    for r in ranks:
        assert np.array_equal(r[f"{key}/adam_losses"], r0[f"{key}/adam_losses"])
        assert int(r[f"{key}/adam_iterations"]) == 3
        for name in ("adam_w3", "adam_slots"):
            for a, b in zip(_list(r, f"{key}/{name}"), _list(r0, f"{key}/{name}")):
                assert np.array_equal(a, b), name
        assert bool(r[f"{key}/rerun_same_bits"])


def test_boundary_graph_edges_are_included(worlds):
    """Cuts inside graphs hand a rank edges whose targets lie on another rank; the CSR test above shows they are dropped."""
    for name in ("world2", "world3"):
        assert any(int(r[f"inside/{i}/extra_edges"]) > 0 for r in worlds[name] for i in range(len(CASES)))


def test_world_of_one_gives_the_bits_of_the_unsharded_loss(worlds):
    assert bool(worlds["world2"][0]["world1_loss_bits"])


def test_gnn_film_raises_on_every_rank(worlds):
    for ranks in worlds.values():
        assert all(bool(r["film_raises"]) for r in ranks)


def test_sharded_train_improvement(worlds):
    """The assertions of test_train_improvement, with every epoch on shards over two ranks; both ranks see the same
    losses and metrics."""
    r0, r1 = worlds["world2"]
    assert np.array_equal(r0["train_improvement"], r1["train_improvement"])
    (valid0_loss, valid0_metric), (train1_loss, train1_metric), (valid1_loss, valid1_metric), (train2_loss, train2_metric) = \
        r0["train_improvement"]
    assert valid0_loss > valid1_loss
    assert valid0_metric > valid1_metric
    assert train1_loss > train2_loss
    assert train1_metric > train2_metric
