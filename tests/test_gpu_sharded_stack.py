"""A GNN, its readout and its global exchanges on target-range shards (sharding.TargetRangeShard): every rank is a spawned
process on one GPU, joined over gloo with host-staged collectives (NCCL refuses two ranks on one device; the library's
collectives all go through sharding.all_gather_into_tensor / reduce_scatter_tensor, which the workers replace).

Each world runs every case once sharded and once unsharded (the unsharded run is the one the rest of the suite checks
against float64 autograd) and saves what it got; the tests then compare the ranks' rows and gradients with the unsharded
run at the float64 bar of test_gpu_readout_backward.py, check that all ranks hold the same bits for per-graph rows and for
the weight gradients after sharding.sum_gradients_over_ranks, and that a second run gives the same bits."""
import os
import socket
import sys

import numpy as np
import pytest

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu
TOL = 3e-5
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


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
def _graph(kind, rng):
    """(V, n2g, G, adjacency lists in global ids): one graph split across every rank, or many QM9-sized graphs."""
    if kind == "one":
        V = 3000
        sizes = np.array([V])
    else:
        sizes = rng.integers(9, 30, size=150)
        V = int(sizes.sum())
    n2g = np.repeat(np.arange(len(sizes)), sizes).astype(np.int32)
    starts = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    adjs = []
    for _ in range(2):
        g = rng.integers(0, len(sizes), size=4 * V)
        src = starts[g] + rng.integers(0, 1 << 30, size=4 * V) % sizes[g]
        tgt = starts[g] + rng.integers(0, 1 << 30, size=4 * V) % sizes[g]
        adjs.append(np.stack([src, tgt], 1).astype(np.int32))
    return V, n2g, len(sizes), adjs


def _bounds(V, world, empty):
    if empty:
        cut = V // 3 + 7
        return [(0, cut), (cut, cut), (cut, V)]
    cuts = [0] + [int(V * r / world) + 5 * r + 1 for r in range(1, world)] + [V]   # cuts inside graphs
    return [(cuts[r], cuts[r + 1]) for r in range(world)]


def _readout_case(weighting, graph):
    return dict(kind="readout", weighting=weighting, graph=graph)


def _exchange_case(mode, weighting, graph):
    return dict(kind="exchange", mode=mode, weighting=weighting, graph=graph)


def _stack_case(name, graph, **hyper):
    return dict(kind="stack", name=name, graph=graph, hyper=hyper)


CASES = ([_readout_case(w, g) for w in ("softmax", "sigmoid") for g in ("one", "many")]
         + [_exchange_case(m, w, "many") for m in ("mean", "gru", "mlp") for w in ("softmax", "sigmoid")]
         + [_exchange_case("gru", "softmax", "one")]
         + [_stack_case("default_rgcn", "many", layer_input_dropout_rate=0.1),
            _stack_case("default_rgcn_one_graph", "one", layer_input_dropout_rate=0.1),
            _stack_case("layernorm_residual_dense_mean", "many", use_inter_layer_layernorm=True, global_exchange_mode="mean",
                        global_exchange_weighting_fun="sigmoid", num_layers=5, layer_input_dropout_rate=0.2)])


def _case_id(c):
    return "-".join(str(c[k]) for k in ("kind", "name", "mode", "weighting", "graph") if k in c)


def _run_case(case, shard, seed):
    """(rows or per-graph output, grad of the input rows, weight gradients) of one training step; shard None = unsharded."""
    from tf2_gnn_b200 import sharding
    from tf2_gnn_b200.layers import (GNN, GNNInput, GraphGlobalExchangeInput, GraphGlobalGRUExchange,
                                     GraphGlobalMeanExchange, GraphGlobalMLPExchange, NodesToGraphRepresentationInput,
                                     WeightedSumGraphRepresentation, node_ops)
    rng = np.random.default_rng(seed)
    V, n2g, G, adjs = _graph(case["graph"], rng)
    H, F = 32, 24
    feats = rng.uniform(-1, 1, (V, F if case["kind"] == "stack" else H)).astype(np.float32)
    lo, hi = (shard.lo, shard.hi) if shard is not None else (0, V)
    torch.manual_seed(1234)
    if case["kind"] == "readout":
        layer = WeightedSumGraphRepresentation(graph_representation_size=H, num_heads=4, weighting_fun=case["weighting"],
                                               scoring_mlp_layers=[H], transformation_mlp_layers=[H],
                                               scoring_mlp_use_biases=True)
        layer.build(NodesToGraphRepresentationInput((None, H), None, None))
        layer.dropout_state = node_ops.DropoutState(seed)
        variables = layer.variables
    elif case["kind"] == "exchange":
        cls = {"mean": GraphGlobalMeanExchange, "gru": GraphGlobalGRUExchange, "mlp": GraphGlobalMLPExchange}[case["mode"]]
        layer = cls(hidden_dim=H, weighting_fun=case["weighting"], num_heads=4, dropout_rate=0.2)
        layer.build(GraphGlobalExchangeInput((None, H), (None,), ()))
        layer.dropout_state = node_ops.DropoutState(seed)
        variables = layer.variables
    else:
        params = GNN.get_default_hyperparameters(case["hyper"].get("message_calculation_class"))
        params.update(hidden_dim=H, b200_dropout_seed=seed)
        params.update(case["hyper"])
        layer = GNN(params)
        layer.build(GNNInput((None, F), tuple((None, 2) for _ in adjs), None, None))
        variables = layer.variables
    for v in variables:
        v.requires_grad_(True)
    x = torch.from_numpy(feats[lo:hi].copy()).cuda().requires_grad_()
    n2g_t = torch.from_numpy(n2g[lo:hi].copy()).cuda()
    R = torch.from_numpy(rng.uniform(-1, 1, (G if case["kind"] == "readout" else V, H)).astype(np.float32)).cuda()
    if case["kind"] == "readout":
        out = layer(NodesToGraphRepresentationInput(x, n2g_t, G), training=True, shard=shard)
        # the loss of the replicated graph rows is counted once: on rank 0 (the backward sums the ranks' parts)
        weight = R if shard is None or shard.rank == 0 else torch.zeros_like(R)
    elif case["kind"] == "exchange":
        out = layer(GraphGlobalExchangeInput(x, n2g_t, G), training=True, shard=shard)
        weight = R[lo:hi]
    else:
        inp = GNNInput(x, tuple(torch.from_numpy(a).cuda() for a in adjs), n2g_t, G)
        ctx = sharding.regather_saved_tables() if shard is not None else None
        if ctx:
            ctx.__enter__()
        out = layer(inp, training=True, shard=shard)
        if ctx:
            ctx.__exit__(None, None, None)
        weight = R[lo:hi]
    (out * weight).sum().backward()
    if shard is not None:
        sharding.sum_gradients_over_ranks(variables, shard.group)
    torch.cuda.synchronize()
    grads = [v.grad.detach().cpu().numpy() if v.grad is not None else np.zeros(tuple(v.value.shape), np.float32)
             for v in variables]
    return out.detach().cpu().numpy(), x.grad.detach().cpu().numpy(), grads


def _memory_rise(shard, edge_factor):
    """Rise of torch's peak allocated bytes over one default-GNN training step under regather_saved_tables()."""
    from tf2_gnn_b200 import sharding
    from tf2_gnn_b200.layers import GNN, GNNInput
    rng = np.random.default_rng(11)
    V, H, G = 40000, 64, 400
    n2g = np.repeat(np.arange(G), V // G).astype(np.int32)
    adjs = [rng.integers(0, V, size=(4 * edge_factor * V, 2)).astype(np.int32) for _ in range(2)]
    adjs = sharding.filter_edges_by_target(adjs, shard.lo, shard.hi)
    params = GNN.get_default_hyperparameters()
    params.update(hidden_dim=H, layer_input_dropout_rate=0.1)
    torch.manual_seed(0)
    gnn = GNN(params)
    gnn.build(GNNInput((None, H), tuple((None, 2) for _ in adjs), None, None))
    for v in gnn.variables:
        v.requires_grad_(True)
    x = torch.from_numpy(rng.uniform(-1, 1, (shard.hi - shard.lo, H)).astype(np.float32)).cuda().requires_grad_()
    inp = GNNInput(x, tuple(torch.from_numpy(a).cuda() for a in adjs), torch.from_numpy(n2g[shard.lo:shard.hi]).cuda(), G)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    with sharding.regather_saved_tables():
        out = gnn(inp, training=True, shard=shard)
    out.sum().backward()
    sharding.sum_gradients_over_ranks(gnn.variables, shard.group)
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def _worker(rank, world, port, tmp, empty):
    import torch.distributed as dist
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        torch.cuda.set_device(0)
        from tf2_gnn_b200 import sharding
        sharding.all_gather_into_tensor = _host_all_gather_into_tensor
        sharding.reduce_scatter_tensor = _host_reduce_scatter_tensor
        from tf2_gnn_b200.layers import graph_autograd
        merged = []
        shard_readout = graph_autograd.shard_readout

        def recording_shard_readout(*args, **kwargs):             # every merged [G, GD] table of a step, in call order
            out = shard_readout(*args, **kwargs)
            merged.append(out.detach().cpu().numpy().reshape(-1))
            return out

        graph_autograd.shard_readout = recording_shard_readout
        results = {}
        for i, case in enumerate(CASES):
            seed = 100 + i
            V = _graph(case["graph"], np.random.default_rng(seed))[0]
            shard = sharding.TargetRangeShard(_bounds(V, world, empty), rank)
            merged.clear()
            out, gx, gw = _run_case(case, shard, seed)
            results[f"{i}/merged"] = np.concatenate(merged) if merged else np.zeros(0, np.float32)
            again = _run_case(case, shard, seed)
            results[f"{i}/out"], results[f"{i}/gx"] = out, gx
            for j, g in enumerate(gw):
                results[f"{i}/gw{j}"] = g
            results[f"{i}/repeat_same_bits"] = np.array(
                np.array_equal(out, again[0]) and np.array_equal(gx, again[1])
                and all(np.array_equal(a, b) for a, b in zip(gw, again[2])))
            results[f"{i}/bounds"] = np.array(shard.bounds)
            if rank == 0:
                full = _run_case(case, None, seed)
                results[f"{i}/full_out"], results[f"{i}/full_gx"] = full[0], full[1]
                for j, g in enumerate(full[2]):
                    results[f"{i}/full_gw{j}"] = g
        if world == 2 and not empty:
            small = _memory_rise(sharding.TargetRangeShard([(0, 20000), (20000, 40000)], rank), 1)
            large = _memory_rise(sharding.TargetRangeShard([(0, 20000), (20000, 40000)], rank), 4)
            results["memory"] = np.array([small, large])
        np.savez(os.path.join(tmp, f"rank{rank}.npz"), **results)
    finally:
        dist.destroy_process_group()


WORLDS = {"world2": (2, False), "world3": (3, False), "world3_empty_shard": (3, True)}


@pytest.fixture(scope="module")
def worlds(tmp_path_factory):
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import torch.multiprocessing as mp
    out = {}
    for name, (world, empty) in WORLDS.items():
        tmp = str(tmp_path_factory.mktemp(name))
        mp.spawn(_worker, args=(world, _free_port(), tmp, empty), nprocs=world, join=True)
        out[name] = [dict(np.load(os.path.join(tmp, f"rank{r}.npz"))) for r in range(world)]
    return out


def close(got, ref, tol=TOL, what="", floor=1e-30):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape, f"{what}: shape {got.shape} vs {ref.shape}"
    err, scale = np.linalg.norm(got - ref), max(np.linalg.norm(ref), floor)
    assert err <= tol * scale, f"{what}: |err| {err:.3e} > {tol:g} * {scale:.3e}"


@pytest.mark.parametrize("world", list(WORLDS))
@pytest.mark.parametrize("i", range(len(CASES)), ids=[_case_id(c) for c in CASES])
def test_sharded_step_matches_the_unsharded_step(worlds, world, i):
    ranks = worlds[world]
    r0 = ranks[0]
    case = CASES[i]
    bounds = r0[f"{i}/bounds"]
    if case["kind"] == "readout":
        for r in ranks:                                              # merged graph rows: the same bits on every rank
            assert np.array_equal(r[f"{i}/out"], r0[f"{i}/out"])
        close(r0[f"{i}/out"], r0[f"{i}/full_out"], what="merged graph rows")
    else:
        close(np.concatenate([r[f"{i}/out"] for r in ranks]), r0[f"{i}/full_out"], what="output rows")
    close(np.concatenate([r[f"{i}/gx"] for r in ranks]), r0[f"{i}/full_gx"], what="grad of the input rows")
    assert sum(int(hi - lo) for lo, hi in bounds) == r0[f"{i}/full_gx"].shape[0]
    n = sum(1 for k in r0 if k.startswith(f"{i}/gw"))
    assert n > 0
    wants = [r0[f"{i}/full_gw{j}"] for j in range(n)]
    floor = max(np.linalg.norm(w) for w in wants)
    for j in range(n):
        for r in ranks:                                              # after sum_gradients_over_ranks: the same bits
            assert np.array_equal(r[f"{i}/gw{j}"], r0[f"{i}/gw{j}"]), f"weight gradient {j} differs between ranks"
        close(r0[f"{i}/gw{j}"], wants[j], what=f"weight gradient {j}", floor=floor)
    assert all(bool(r[f"{i}/repeat_same_bits"]) for r in ranks)
    for r in ranks:                               # every merged per-graph table of the step: the same bits on every rank
        assert np.array_equal(r[f"{i}/merged"], r0[f"{i}/merged"])
    hyper = case.get("hyper", {})
    if case["kind"] != "stack" or hyper.get("global_exchange_every_num_layers", 2) < hyper.get("num_layers", 4):
        assert r0[f"{i}/merged"].size, "no merged per-graph table was recorded"


def test_no_temporary_grows_with_the_edge_count(worlds):
    """Four times the edges on the same nodes: a training step under regather_saved_tables() raises the peak of torch's
    allocator by about the same amount, so no tensor the stack, the readout merge or the exchanges create grows with the
    edge count.  This sees torch's allocations only: the library's own pool (the prepared CSR, kernel scratch) is not
    measured here; the layer backward tests bound that part for each fused layer."""
    for r in worlds["world2"]:
        small, large = (int(v) for v in r["memory"])
        assert large <= 1.15 * small + (8 << 20), (small, large)


def test_shard_dropout_draws_the_unsharded_masks():
    """node_ops.dropout(rows=(lo, V)) on rows [lo, hi) of a [V, H] table gives rows [lo, hi) of the unsharded masks, with
    the same stream offset consumed; lo * H % 4 != 0 included."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    sys.path.insert(0, ROOT)
    from tf2_gnn_b200.layers import node_ops
    V, H = 1001, 7
    x = torch.rand((V, H), device="cuda") + 0.5
    for rate in (0.1, 0.5):
        full_state = node_ops.DropoutState(77)
        full_state.offset = 5
        full = node_ops.dropout(x, rate, full_state)
        for lo, hi in [(0, 1), (1, 2), (3, 500), (333, 1001), (1000, 1001), (17, 17)]:
            st = node_ops.DropoutState(77)
            st.offset = 5
            part = node_ops.dropout(x[lo:hi], rate, st, rows=(lo, V))
            assert st.offset == full_state.offset
            assert torch.equal(part, full[lo:hi]), (lo, hi)
            # backward draws the same mask
            xs = x[lo:hi].clone().requires_grad_()
            st = node_ops.DropoutState(77)
            st.offset = 5
            node_ops.dropout(xs, rate, st, rows=(lo, V)).sum().backward()
            assert torch.equal((xs.grad != 0), (full[lo:hi] != 0))
    with pytest.raises(ValueError):              # rows outside the table would take the next call's Philox counters
        node_ops.dropout(x[990:], 0.5, node_ops.DropoutState(77), rows=(995, V))
