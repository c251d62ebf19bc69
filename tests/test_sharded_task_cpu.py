"""Task models on target-range shards, without a GPU: the new loss and batch-window entries are exported, bound and reject
invalid arguments before any CUDA call; a float64 restatement of the node loss shows that the ranks' partial sums over the
batch's row count are the unsharded loss, that micro-F1 from the summed counts is the unsharded F1, and that each rank's
gradient rows are the unsharded ones; the store's cut rule on its host tables is partition_target_range over the batch's
in-degree."""
import ctypes
import math

import numpy as np
import pytest

import reference64_task as rt
from tf2_gnn_b200 import _ffi, sharding
from tf2_gnn_b200.data.graph_store import shard_bounds_from_tables, stored_in_degree

ENTRIES = ("tfgnn_b200_node_multiclass_loss_partial", "tfgnn_b200_node_multiclass_loss_merge",
           "tfgnn_b200_node_multiclass_loss_bwd_rows", "tfgnn_b200_assemble_batch_rows")
FAKE = 0x1000   # never dereferenced: every call below fails validation first


def test_entries_are_exported_and_bound():
    lib = _ffi.lib()
    for name in ENTRIES:
        assert name in _ffi.EXPORTED_SYMBOLS
        assert getattr(lib, name).argtypes, f"{name} has no argtypes"
    assert lib.tfgnn_b200_abi_version() == 1


def _rejects(name, *args, says=None):
    lib = _ffi.lib()
    rc = getattr(lib, name)(*args)
    assert rc == _ffi.ERR_INVALID_ARGUMENT, f"{name}: rc {rc}"
    msg = lib.tfgnn_b200_last_error().decode()
    assert name in msg, msg
    if says:
        assert says in msg, msg


def test_node_loss_entries_validate_sizes_and_pointers():
    part = "tfgnn_b200_node_multiclass_loss_partial"
    _rejects(part, FAKE, FAKE, 10, 0, FAKE, FAKE, None, says="num_labels")
    _rejects(part, FAKE, FAKE, -1, 3, FAKE, FAKE, None, says="bad sizes")
    _rejects(part, None, FAKE, 10, 3, FAKE, FAKE, None, says="NULL")
    _rejects(part, FAKE, FAKE, 10, 3, None, FAKE, None, says="NULL")
    _rejects(part, FAKE, FAKE, 0, 3, FAKE, None, None, says="NULL")
    merge = "tfgnn_b200_node_multiclass_loss_merge"
    _rejects(merge, FAKE, FAKE, 0, 10, FAKE, FAKE, FAKE, None, says="world")
    _rejects(merge, FAKE, FAKE, -2, 10, FAKE, FAKE, FAKE, None, says="world")
    _rejects(merge, FAKE, FAKE, 2, -1, FAKE, FAKE, FAKE, None, says="total_rows")
    _rejects(merge, None, FAKE, 2, 10, FAKE, FAKE, FAKE, None, says="NULL")
    _rejects(merge, FAKE, FAKE, 2, 10, FAKE, None, FAKE, None, says="NULL")
    bwd = "tfgnn_b200_node_multiclass_loss_bwd_rows"
    _rejects(bwd, FAKE, FAKE, 10, 0, 20, FAKE, FAKE, None, says="num_labels")
    _rejects(bwd, FAKE, FAKE, -1, 3, 20, FAKE, FAKE, None, says="bad sizes")
    _rejects(bwd, FAKE, FAKE, 10, 3, 9, FAKE, FAKE, None, says="total_rows")
    _rejects(bwd, FAKE, FAKE, 10, 3, 20, None, FAKE, None, says="NULL")
    # an empty rank's backward is a no-op (no launch, no GPU needed)
    assert _ffi.lib().tfgnn_b200_node_multiclass_loss_bwd_rows(None, None, 0, 3, 20, None, None, None) == _ffi.OK


def _rows_call(row_begin, row_count, num_nodes=100, T=2, null_offsets=False, num_graphs=5):
    ptrs = lambda: ctypes.cast((ctypes.c_void_p * T)(*([FAKE] * T)), _ffi._PP)   # noqa: E731
    Eb = (ctypes.c_int64 * T)(*([7] * T))
    return ("tfgnn_b200_assemble_batch_rows", None if null_offsets else FAKE, ptrs(), ptrs(), T, 9, FAKE, num_graphs,
            num_nodes, Eb, row_begin, row_count, FAKE, FAKE, ptrs(), FAKE, None)


def test_assemble_batch_rows_validates_the_window():
    _rejects(*_rows_call(-1, 5), says="row window")
    _rejects(*_rows_call(0, -1), says="row window")
    _rejects(*_rows_call(96, 5), says="row window")
    _rejects(*_rows_call(101, 0), says="row window")
    _rejects(*_rows_call(0, 5, num_nodes=-1), says="negative")
    _rejects(*_rows_call(0, 5, T=_ffi.MAX_EDGE_TYPES + 1), says="edge types")
    _rejects(*_rows_call(0, 5, null_offsets=True), says="NULL")
    lib = _ffi.lib()
    name, *args = _rows_call(100, 0)                    # an empty window at the end of the batch writes nothing
    assert getattr(lib, name)(*args) == _ffi.OK
    name, *args = _rows_call(0, 0, num_nodes=0, num_graphs=0)
    assert getattr(lib, name)(*args) == _ffi.OK


# ---- the node loss over ranks, restated in float64 ---------------------------------------------------------------------
def _cuts(V, world, empty):
    if empty:
        return [(0, V // 3), (V // 3, V // 3), (V // 3, V)]
    c = [0] + [V * r // world + 3 * r for r in range(1, world)] + [V]
    return [(c[r], c[r + 1]) for r in range(world)]


@pytest.mark.parametrize("world,empty", [(1, False), (2, False), (3, False), (3, True)])
def test_partials_over_the_total_row_count_are_the_unsharded_loss(world, empty):
    rng = np.random.default_rng(world + 10 * empty)
    V, C = 901, 121
    x = rng.normal(0, 3, (V, C)).astype(np.float32)
    y = (rng.uniform(size=(V, C)) < 0.3).astype(np.float32)
    loss, grad, counts, f1 = rt.node_multiclass_loss(x, y)
    sums, parts = [], []
    for lo, hi in _cuts(V, world, empty):
        l_r, g_r, c_r, _ = rt.node_multiclass_loss(x[lo:hi], y[lo:hi])
        sums.append(l_r * (hi - lo) if hi > lo else 0.0)        # the raw partial sum of the rank's rows
        parts.append(c_r)
        if hi > lo:                                               # the rank's backward: 1 / total rows, no collective
            np.testing.assert_allclose(g_r * (hi - lo) / V, grad[lo:hi], rtol=1e-12, atol=0)
    merged = sum(sums) / V
    assert merged == pytest.approx(loss, rel=1e-12)
    summed = tuple(int(sum(c[k] for c in parts)) for k in range(3))
    assert summed == counts
    assert rt.micro_f1(summed) == f1 or (math.isnan(f1) and math.isnan(rt.micro_f1(summed)))


# ---- the store's cut rule ------------------------------------------------------------------------------------------
def _graphs(rng, n):
    out = []
    for _ in range(n):
        v = int(rng.integers(1, 40))
        out.append([rng.integers(0, v, (int(rng.integers(0, 5 * v)), 2)).astype(np.int32) for _ in range(3)] + [v])
    return out


@pytest.mark.parametrize("world", [1, 2, 3, 5])
def test_store_cut_rule_is_partition_target_range_of_the_batch(world):
    rng = np.random.default_rng(world)
    graphs = _graphs(rng, 60)
    counts = [g[-1] for g in graphs]
    node_offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    edges = [[g[t] for g in graphs] for t in range(3)]
    deg_table = stored_in_degree(node_offsets, edges)
    for ids in (rng.permutation(60)[:17], np.arange(60), np.array([5]), np.array([], dtype=np.int64)):
        # the batch as assemble_batch builds it: node ids offset by the running node count, in batch order
        Vb, tgts = 0, []
        for g in ids:
            for t in range(3):
                tgts.append(graphs[g][t][:, 1].astype(np.int64) + Vb)
            Vb += counts[g]
        deg = np.bincount(np.concatenate(tgts), minlength=Vb) if tgts else np.zeros(Vb, np.int64)
        want = sharding.partition_target_range(Vb, world, deg)
        assert shard_bounds_from_tables(node_offsets, deg_table, ids, world) == want
        assert want[0][0] == 0 and want[-1][1] == Vb
