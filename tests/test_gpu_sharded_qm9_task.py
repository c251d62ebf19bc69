"""QM9RegressionTask trained on target-range shards: every rank is a spawned process on one GPU, joined over gloo with
host-staged collectives (as in test_gpu_sharded_task_models.py), on a QM9Dataset of seeded synthetic molecules.

Each rank builds its model from a different seed and takes rank 0's weights with sharding.broadcast_variables, assembles
its part of the batch with store.shard_batch and runs train_step(shard=...) with QM9_RGCN.json's model parameters and
out-layer dropout.  The tests check that loss and metrics hold the same bits on every rank and match the unsharded step,
that the summed gradients hold the same bits on every rank and match the unsharded ones, that one SGD step matches and three
RMSProp steps with value clipping keep every rank on the same variables, slots and step count, run after run; and that a
sharded training run improves the validation MAE."""
import os
import socket
import sys

import numpy as np
import pytest

torch = pytest.importorskip("torch")

import reference64_qm9 as rq
from reference64_qm9 import QM9_RGCN

pytestmark = pytest.mark.gpu
TOL = 3e-5
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SGD_LR = 0.05
METRICS = ("loss", "batch_squared_error", "batch_absolute_error")
HYPER = dict(QM9_RGCN, gnn_num_layers=4, out_layer_dropout_keep_prob=0.1)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


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


def _dataset(data_dir):
    from tf2_gnn_b200.data import QM9Dataset
    ds = QM9Dataset(QM9Dataset.get_default_hyperparameters())
    ds.load_data(data_dir)
    return ds


def _model(ds, optimizer, seed, **hyper):
    from tf2_gnn_b200.models import QM9RegressionTask
    params = QM9RegressionTask.get_default_hyperparameters()
    params.update(HYPER, **hyper)
    if optimizer == "sgd":
        params.update(optimizer="SGD", learning_rate=SGD_LR, momentum=0.0, gradient_clip_value=None)
    torch.manual_seed(seed)
    model = QM9RegressionTask(params, ds)
    shapes = {"node_features": (None, rq.NUM_FEATURES)}
    shapes.update({f"adjacency_list_{t}": (None, 2) for t in range(ds.num_edge_types)})
    model.build(shapes)
    return model


def _run(ds, ids, seed, shard, rank):
    """(results of one SGD step, parameters after three RMSProp steps); shard None = unsharded."""
    from tf2_gnn_b200 import sharding
    from tf2_gnn_b200.data import DataFold
    store = ds.store(DataFold.TRAIN)
    if shard is None:
        feats, labels = store.batch(ids), store.batch_labels(ids)
    else:
        feats, labels = store.shard_batch(ids, shard), store.shard_batch_labels(ids, shard)
    res = {}
    model = _model(ds, "sgd", seed + (0 if shard is None else 7 * rank))
    if shard is not None:
        sharding.broadcast_variables(model.trainable_variables, shard.group)
    res["w0"] = [v.value.detach().cpu().numpy() for v in model.trainable_variables]
    seen = []
    apply = model._apply_gradients

    def recording(pairs):
        pairs = list(pairs)
        seen.append([None if g is None else g.detach().cpu().numpy() for g, _ in pairs])
        apply(pairs)

    model._apply_gradients = recording
    m = model.train_step(feats, labels, shard=shard)
    for k in METRICS:
        res[f"sgd_{k}"] = np.array(m[k].detach().cpu().numpy())
    res["sgd_grads"] = seen[0]
    res["sgd_w1"] = [v.value.detach().cpu().numpy() for v in model.trainable_variables]
    if shard is not None:
        model = _model(ds, "rmsprop", seed + 7 * rank)
        sharding.broadcast_variables(model.trainable_variables, shard.group)
        res["rms_losses"] = np.array([model.train_step(feats, labels, shard=shard)["loss"].item() for _ in range(3)])
        res["rms_w3"] = [v.value.detach().cpu().numpy() for v in model.trainable_variables]
        res["rms_iterations"] = np.array(model._optimizer.iterations)
        slots = [model._optimizer.slots(v.value) for v in model.trainable_variables]
        res["rms_slots"] = [s.cpu().numpy() for pair in slots for s in pair if s is not None]
    return res


def _bounds(kind, store_bounds, V, world):
    if kind == "store":
        return store_bounds
    if kind == "empty":
        cut = V // 3 + 7
        return [(0, cut), (cut, cut), (cut, V)]
    cuts = [0] + [int(V * r / world) + 5 * r + 1 for r in range(1, world)] + [V]   # cuts inside graphs
    return [(cuts[r], cuts[r + 1]) for r in range(world)]


def _sharded_train_improvement(ds):
    """test_train_improvement (test_gpu_qm9_task.py) with every epoch on target-range shards over the world."""
    import torch.distributed as dist
    from tf2_gnn_b200 import sharding
    from tf2_gnn_b200.data import DataFold
    np.random.seed(0)
    model = _model(ds, "rmsprop", 0, learning_rate=0.001, out_layer_dropout_keep_prob=0.0)
    sharding.broadcast_variables(model.trainable_variables)
    group = dist.group.WORLD

    def epoch(store, training):
        order = np.random.permutation(store.num_graphs) if training else None
        loss, _, results = model.run_one_epoch(store, store.iter_batch_graph_ids(2000, order), training=training,
                                               shard_group=group)
        return loss, model.compute_epoch_metrics(results)[0]

    train, valid = ds.store(DataFold.TRAIN), ds.store(DataFold.VALIDATION)
    out = [epoch(valid, False)] + [epoch(train, True) for _ in range(3)] + [epoch(valid, False)]
    return np.array(out, dtype=np.float64)


def _film_raises(ds, rank, world):
    from tf2_gnn_b200 import sharding
    from tf2_gnn_b200.data import DataFold
    from tf2_gnn_b200.models import QM9RegressionTask
    store = ds.store(DataFold.TRAIN)
    ids = np.arange(20)
    shard = sharding.TargetRangeShard(store.shard_bounds(ids, world), rank)
    params = QM9RegressionTask.get_default_hyperparameters("gnn_film")
    params.update(gnn_hidden_dim=32, gnn_num_layers=2, out_layer_dropout_keep_prob=0.0)
    model = QM9RegressionTask(params, ds)
    try:
        model.train_step(store.shard_batch(ids, shard), store.shard_batch_labels(ids, shard), shard=shard)
    except NotImplementedError:
        return True
    return False


def _worker(rank, world, port, tmp, data_dir, cut_kinds):
    import torch.distributed as dist
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        torch.cuda.set_device(0)
        from tf2_gnn_b200 import sharding
        from tf2_gnn_b200.data import DataFold
        sharding.all_gather_into_tensor = _host_all_gather_into_tensor
        sharding.reduce_scatter_tensor = _host_reduce_scatter_tensor
        ds = _dataset(data_dir)
        store = ds.store(DataFold.TRAIN)
        ids = np.arange(40)
        V = int(sum(store.node_offsets_host[g + 1] - store.node_offsets_host[g] for g in ids))
        results = {}
        for kind in cut_kinds:
            seed = 100
            shard = sharding.TargetRangeShard(_bounds(kind, store.shard_bounds(ids, world), V, world), rank)
            results[f"{kind}/bounds"] = np.array(shard.bounds)
            got = _run(ds, ids, seed, shard, rank)
            again = _run(ds, ids, seed, shard, rank)
            same = all(np.array_equal(a, b) for a, b in zip(got["rms_w3"], again["rms_w3"]))
            same &= np.array_equal(got["rms_losses"], again["rms_losses"])
            same &= all(np.array_equal(a, b) for a, b in zip(got["sgd_w1"], again["sgd_w1"]))
            results[f"{kind}/rerun_same_bits"] = np.array(same)
            if rank == 0:
                got.update({f"full_{k}": v for k, v in _run(ds, ids, seed, None, 0).items()})
            for k, v in got.items():
                if isinstance(v, list):
                    results[f"{kind}/{k}/n"] = np.array(len(v))
                    results.update({f"{kind}/{k}/{j}": a for j, a in enumerate(v) if a is not None})
                else:
                    results[f"{kind}/{k}"] = v
        results["film_raises"] = np.array(_film_raises(ds, rank, world))
        if world == 2:
            results["train_improvement"] = _sharded_train_improvement(ds)
        np.savez(os.path.join(tmp, f"rank{rank}.npz"), **results)
    finally:
        dist.destroy_process_group()


WORLDS = {"world2": (2, ("store", "inside")), "world3": (3, ("store", "inside")), "world3_empty_shard": (3, ("empty",))}


@pytest.fixture(scope="module")
def worlds(tmp_path_factory):
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import torch.multiprocessing as mp
    data_dir = str(tmp_path_factory.mktemp("qm9"))
    rq.write_dataset(data_dir, np.random.default_rng(9), (600, 100, 10))
    out = {}
    for name, (world, kinds) in WORLDS.items():
        tmp = str(tmp_path_factory.mktemp(name))
        mp.spawn(_worker, args=(world, _free_port(), tmp, data_dir, kinds), nprocs=world, join=True)
        out[name] = [dict(np.load(os.path.join(tmp, f"rank{r}.npz"))) for r in range(world)]
    return out


def close(got, ref, tol=TOL, what="", floor=1e-30):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape, f"{what}: shape {got.shape} vs {ref.shape}"
    err, scale = np.linalg.norm(got - ref), max(np.linalg.norm(ref), floor)
    assert err <= tol * scale, f"{what}: |err| {err:.3e} > {tol:g} * {scale:.3e}"


def _list(r, key):
    return [r.get(f"{key}/{j}") for j in range(int(r[f"{key}/n"]))]


RUNS = [(w, kind) for w, (_, kinds) in WORLDS.items() for kind in kinds]


@pytest.mark.parametrize("world,kind", RUNS, ids=[f"{w}-{k}" for w, k in RUNS])
def test_sharded_train_step_matches_the_unsharded_step(worlds, world, kind):
    ranks = worlds[world]
    r0 = ranks[0]
    if kind == "empty":
        assert any(lo == hi for lo, hi in r0[f"{kind}/bounds"])
    for r in ranks:   # every rank starts from rank 0's bits, which are the unsharded ones
        for a, b in zip(_list(r, f"{kind}/w0"), _list(r0, f"{kind}/full_w0")):
            assert np.array_equal(a, b)
    for m in METRICS:
        for r in ranks:
            assert np.array_equal(r[f"{kind}/sgd_{m}"], r0[f"{kind}/sgd_{m}"]), m
        close(r0[f"{kind}/sgd_{m}"], r0[f"{kind}/full_sgd_{m}"], what=m)
    grads, wants = _list(r0, f"{kind}/sgd_grads"), _list(r0, f"{kind}/full_sgd_grads")
    assert len(grads) == len(wants) and sum(g is not None for g in wants) >= len(wants) - 2
    floor = max(np.linalg.norm(w) for w in wants if w is not None)
    for j, (g, w) in enumerate(zip(grads, wants)):
        for r in ranks:
            gr = _list(r, f"{kind}/sgd_grads")[j]
            assert (gr is None) == (g is None) and (g is None or np.array_equal(gr, g)), f"gradient {j} differs between ranks"
        assert (g is None) == (w is None), f"gradient {j}: presence differs from the unsharded step"
        if w is not None:
            close(g, w, what=f"gradient {j}", floor=floor)
    for j, (a, b) in enumerate(zip(_list(r0, f"{kind}/sgd_w1"), _list(r0, f"{kind}/full_sgd_w1"))):
        for r in ranks:
            assert np.array_equal(_list(r, f"{kind}/sgd_w1")[j], a)
        close(a, b, what=f"variable {j} after one SGD step", floor=floor * SGD_LR)
    for r in ranks:   # three RMSProp steps with value clipping: the same variables, slots and step count on every rank
        assert np.array_equal(r[f"{kind}/rms_losses"], r0[f"{kind}/rms_losses"])
        assert int(r[f"{kind}/rms_iterations"]) == 3
        for name in ("rms_w3", "rms_slots"):
            for a, b in zip(_list(r, f"{kind}/{name}"), _list(r0, f"{kind}/{name}")):
                assert np.array_equal(a, b), name
        assert bool(r[f"{kind}/rerun_same_bits"])


def test_gnn_film_raises_on_every_rank(worlds):
    for ranks in worlds.values():
        assert all(bool(r["film_raises"]) for r in ranks)


def test_sharded_train_improvement(worlds):
    """Validation MAE and loss improve after three sharded training epochs; both ranks see the same values."""
    r0, r1 = worlds["world2"]
    assert np.array_equal(r0["train_improvement"], r1["train_improvement"])
    valid0, valid1 = r0["train_improvement"][0], r0["train_improvement"][-1]
    assert valid1[1] < valid0[1] and valid1[0] < valid0[0], r0["train_improvement"]
