"""The readout on target-range shards without a GPU: the new entries are exported, bound and validate their arguments
before any CUDA call, and a float64 restatement of the per-graph partials (fixed row chunks, pieces combined in chunk
order) and of their rank-ordered merge gives the unsharded readout for any cut of the rows, graphs split across ranks and
empty shards included."""
import ctypes
import zlib

import numpy as np
import pytest

torch = pytest.importorskip("torch")

from tf2_gnn_b200 import _ffi, sharding  # noqa: E402

NEW = ("tfgnn_b200_readout_partial", "tfgnn_b200_readout_merge", "tfgnn_b200_dropout_at")


def test_new_entries_are_exported_and_bound():
    raw = ctypes.CDLL(_ffi.library_path())
    lib = _ffi.lib()
    for name in NEW:
        assert hasattr(raw, name) and name in _ffi.EXPORTED_SYMBOLS
        assert getattr(lib, name).argtypes, f"{name} has no argtypes in _ffi.py"


def test_invalid_arguments_are_reported_before_any_cuda_call():
    lib = _ffi.lib()
    p = 64     # never dereferenced: validation fails first
    bad = _ffi.ERR_INVALID_ARGUMENT

    def partial(scores=p, reprs=p, n2g=p, ptr=p, V=10, G=3, GD=8, K=4, mode=0, out=p):
        return lib.tfgnn_b200_readout_partial(scores, reprs, n2g, ptr, V, G, GD, K, mode, out, None)

    assert partial(GD=10) == bad
    assert b"num_heads must divide" in lib.tfgnn_b200_last_error()
    assert partial(V=-1) == bad
    assert partial(mode=3) == bad
    assert b"average is not built for shards" in lib.tfgnn_b200_last_error()
    assert partial(scores=None, mode=0) == bad
    assert partial(scores=None, mode=1) == bad
    assert partial(reprs=None) == bad
    assert partial(ptr=None) == bad
    assert partial(out=None) == bad
    assert partial(G=0) == 0                                     # no graphs: nothing to do

    def merge(parts=p, world=2, G=3, GD=8, K=4, mode=0, out=p, m=p, s=p):
        return lib.tfgnn_b200_readout_merge(parts, world, G, GD, K, mode, out, m, s, None)

    assert merge(world=0) == bad
    assert merge(GD=6) == bad
    assert merge(mode=3) == bad
    assert merge(m=None) == bad                                  # softmax needs the normaliser outputs
    assert merge(parts=None) == bad
    assert merge(G=0) == 0
    with pytest.raises(ValueError):
        _ffi.check(merge(out=None, mode=1))

    assert lib.tfgnn_b200_dropout_at(p, 10, 1.0, 0, 0, 3, p, None) == bad
    assert lib.tfgnn_b200_dropout_at(p, 10, 0.5, 0, 0, -1, p, None) == bad
    assert lib.tfgnn_b200_dropout_at(None, 10, 0.5, 0, 0, 3, p, None) == bad
    assert lib.tfgnn_b200_dropout_at(p, 0, 0.5, 0, 0, 3, None, None) == 0


# ---- float64 restatement of tfgnn_b200_readout_partial / _merge ------------------------------------------------------
CHUNK_ROWS = 256


def _combine(a, b, softmax):
    """(m, s, S) pieces; m, s [K], S [K, d].  The online-softmax rescale, neutral = (-inf, 0, 0)."""
    if not softmax:
        return a[0], a[1], a[2] + b[2]
    m = np.maximum(a[0], b[0])
    with np.errstate(invalid="ignore"):
        ea = np.where(np.isneginf(m), 0.0, np.exp(a[0] - m))
        eb = np.where(np.isneginf(m), 0.0, np.exp(b[0] - m))
    return m, a[1] * ea + b[1] * eb, a[2] * ea[:, None] + b[2] * eb[:, None]


def _neutral(K, d):
    return np.full(K, -np.inf), np.zeros(K), np.zeros((K, d))


def readout_partial(w, reprs, n2g, G, K, softmax, chunk_rows=CHUNK_ROWS):
    """One rank's partial of every graph: its rows cut into fixed chunks, each chunk's rows in order, a graph's chunk
    pieces combined in chunk order."""
    V, GD = reprs.shape
    d = GD // K
    out = [_neutral(K, d) for _ in range(G)]
    for c0 in range(0, V, chunk_rows):
        pieces = {}
        for v in range(c0, min(V, c0 + chunk_rows)):
            g = int(n2g[v])
            t = reprs[v].reshape(K, d)
            x = w[v] if w is not None else np.ones(K)
            row = (x, np.ones(K), t) if softmax else (None, None, x[:, None] * t)
            pieces[g] = _combine(pieces.get(g, _neutral(K, d)), row, softmax)
        for g, piece in pieces.items():                    # chunks in order
            out[g] = _combine(out[g], piece, softmax)
    return out


def readout_merge(partials, softmax):
    """partials[r][g] in rank order -> ([G, GD], max [G, K], sum [G, K])."""
    G = len(partials[0])
    res, ms, ss = [], [], []
    for g in range(G):
        acc = partials[0][g]
        for r in range(1, len(partials)):
            acc = _combine(acc, partials[r][g], softmax)
        m, s, S = acc
        if softmax:
            S = np.where(s[:, None] > 0, S / np.where(s > 0, s, 1.0)[:, None], 0.0)
        res.append(S.reshape(-1))
        ms.append(m)
        ss.append(s)
    return np.stack(res), np.stack(ms), np.stack(ss)


def _unsharded(scores, reprs, n2g, G, K, weighting):
    V, GD = reprs.shape
    d = GD // K
    out = np.zeros((G, GD))
    for g in range(G):
        rows = np.nonzero(n2g == g)[0]
        if not len(rows):
            continue
        if weighting == "softmax":
            e = np.exp(scores[rows] - scores[rows].max(0))
            w = e / e.sum(0)
        elif weighting == "sigmoid":
            w = 1.0 / (1.0 + np.exp(-scores[rows]))
        else:
            w = np.ones((len(rows), K))
        out[g] = (w[:, :, None] * reprs[rows].reshape(-1, K, d)).sum(0).reshape(-1)
    return out


def _cuts(V, rng, world):
    inner = np.sort(rng.integers(0, V + 1, size=world - 1))
    return [0] + [int(c) for c in inner] + [V]


@pytest.mark.parametrize("weighting", ["softmax", "sigmoid", "none"])
@pytest.mark.parametrize("layout", ["one_graph", "many_small", "empty_graphs"])
@pytest.mark.parametrize("world", [1, 2, 3, 5])
def test_partials_merged_in_rank_order_are_the_unsharded_readout(weighting, layout, world):
    rng = np.random.default_rng(zlib.crc32(f"{weighting}/{layout}/{world}".encode()))
    K = 1 if weighting == "none" else 2
    GD = 4 * K
    if layout == "one_graph":
        sizes = np.array([700])
    elif layout == "many_small":
        sizes = rng.integers(9, 30, size=40)
    else:
        sizes = np.array([0, 0, 300, 0, 5, 1, 0, 290, 0])
    G, V = len(sizes), int(sizes.sum())
    n2g = np.repeat(np.arange(G), sizes)
    scores = rng.uniform(-30, 30, (V, K))                  # large spread: the rescale matters
    reprs = rng.uniform(-1, 1, (V, GD))
    want = _unsharded(scores, reprs, n2g, G, K, weighting)
    w = scores if weighting == "softmax" else (1.0 / (1.0 + np.exp(-scores)) if weighting == "sigmoid" else None)
    cuts = _cuts(V, rng, world)
    if world == 3:
        cuts[1] = cuts[2]                                  # an empty shard
    parts = [readout_partial(None if w is None else w[lo:hi], reprs[lo:hi], n2g[lo:hi], G, K, weighting == "softmax",
                             chunk_rows=37)
             for lo, hi in zip(cuts[:-1], cuts[1:])]
    got, gmax, gsum = readout_merge(parts, weighting == "softmax")
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)
    if weighting == "softmax":                            # the merged normaliser is the global one
        for g in range(G):
            rows = n2g == g
            if rows.any():
                np.testing.assert_array_equal(gmax[g], scores[rows].max(0))
                np.testing.assert_allclose(gsum[g], np.exp(scores[rows] - gmax[g]).sum(0), rtol=1e-12)
                # the backward's weights from the merged normaliser are the unsharded softmax weights
                wts = np.exp(scores[rows] - gmax[g]) / gsum[g]
                np.testing.assert_allclose(wts.sum(0), np.ones(K), rtol=1e-12)
            else:
                assert np.isneginf(gmax[g]).all() and not gsum[g].any()


def test_target_range_shard_checks_its_bounds():
    s = sharding.TargetRangeShard([(0, 4), (4, 4), (4, 9)], 2)
    assert (s.lo, s.hi, s.num_nodes, s.world_size, s.rows) == (4, 9, 9, 3, (4, 9))
    for bad in ([(1, 4), (4, 9)], [(0, 4), (5, 9)], [(0, 5), (5, 3)]):
        with pytest.raises(ValueError):
            sharding.TargetRangeShard(bad, 0)
    with pytest.raises(ValueError):
        sharding.TargetRangeShard([(0, 4), (4, 9)], 2)


def test_a_film_stack_on_a_shard_raises_before_any_device_work():
    from tf2_gnn_b200.layers import GNN, GNNInput
    params = GNN.get_default_hyperparameters("gnn_film")
    params.update(hidden_dim=8)
    gnn = GNN(params)
    gnn.build(GNNInput((None, 4), ((None, 2),), None, None))
    shard = sharding.TargetRangeShard([(0, 3), (3, 6)], 0)
    inp = GNNInput(np.zeros((3, 4), np.float32), (np.zeros((0, 2), np.int32),), np.zeros(3, np.int32), 1)
    with pytest.raises(NotImplementedError, match="GNN-FiLM stack on target-range shards"):
        gnn(inp, training=True, shard=shard)
