"""Parity at BASELINE.json's FULL sizes (VERDICT r1, next-round #1a): the layer runs once on the whole graph of each
config and the float64 oracle is evaluated on a sample of target rows — all their incoming edges of every type, so
the sampled rows of the sub-problem are exactly the rows of the full problem (in-degree scaling, softmax over all
incoming edges, GRU / FiLM target terms included) — in seconds of CPU time and without any [E, H] materialisation.
Covers what the small tests cannot: the CTA-pair default rule (m_tiles >= SMs), thousands of tiles per launch, the
two-N-pass path at H = 320, byte offsets beyond 2^31, power-law hubs of 1e5 edges.  Tolerance: the north_star's 1e-5
(norm-wise over the sampled rows)."""
import os
import sys

import numpy as np
import pytest

torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import message_passing_oracle as mo  # noqa: E402

pytestmark = pytest.mark.gpu
TOL = 1e-5


def sampled_subproblem(h, adjs, rows):
    """All incoming edges of `rows` (every type, original order), nodes relabelled compactly.
    Returns (h_sub, adjs_sub, positions of `rows` in the sub-problem)."""
    V = h.shape[0]
    mask = np.zeros(V, dtype=bool)
    mask[rows] = True
    kept = [a[mask[a[:, 1]]] for a in adjs]
    nodes = np.unique(np.concatenate([rows] + [a[:, 0] for a in kept]))
    remap = np.full(V, -1, dtype=np.int64)
    remap[nodes] = np.arange(nodes.shape[0])
    sub_adjs = [np.stack([remap[a[:, 0]], remap[a[:, 1]]], axis=1).astype(np.int32) for a in kept]
    return h[nodes], sub_adjs, remap[rows]


def check_sampled_rows(kind, params, weights, h, adjs, out_gpu, rows, tol=TOL):
    h_sub, adjs_sub, pos = sampled_subproblem(h, adjs, rows)
    ref = mo.message_passing_forward(kind, params, weights, h_sub, adjs_sub, dtype=np.float64)[pos]
    got = out_gpu[torch.from_numpy(rows).to(out_gpu.device)].cpu().numpy().astype(np.float64)
    scale = max(np.abs(ref).max(), 1e-30)
    err = np.abs(got - ref).max()
    assert np.isfinite(got).all()
    assert err <= tol * scale, f"max abs err {err:.3e} > {tol:g} * {scale:.3e} over {len(rows)} sampled rows"
    return err / scale


def pick_rows(rng, V, adjs, n=2000, hubs=8):
    """n random targets + the `hubs` largest in-degree targets + the first and last tile of the graph."""
    deg = np.zeros(V, dtype=np.int64)
    for a in adjs:
        deg += np.bincount(a[:, 1], minlength=V)
    top = np.argsort(deg)[-hubs:]
    edge = np.concatenate([np.arange(0, 130), np.arange(V - 130, V)])
    rows = np.unique(np.concatenate([rng.choice(V, size=min(n, V), replace=False), top, edge]))
    return rows.astype(np.int64)


@pytest.mark.parametrize("name", ["cfg1", "cfg2", "h320", "cfg4", "cfg3", "cfg5_shard"])
def test_baseline_scale_sampled_rows(name):
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import bench
    from tf2_gnn_b200.layers import MessagePassingInput
    from tf2_gnn_b200.runtime import PreparedBatch
    wl = bench.WORKLOADS[name]
    kind, V, H, L = wl["kind"], wl["V"], wl["H"], len(wl["E"])
    h, adjs, _ = bench.make_inputs(wl, seed=0)
    layer, params = bench.build_layer(wl, 0)
    rng = np.random.default_rng(123)
    weights = mo.make_weights(kind, params, H, L, rng)
    layer.set_weights_from_oracle_dict(weights)
    dev = torch.device("cuda")
    adj_dev = tuple(torch.from_numpy(a).to(dev) for a in adjs)
    prepared = PreparedBatch(adj_dev, V)
    out = layer(MessagePassingInput(torch.from_numpy(h).to(dev), adj_dev), prepared=prepared)
    torch.cuda.synchronize()
    assert tuple(out.shape) == (V, H)
    rows = np.arange(V, dtype=np.int64) if V <= 10_000 else pick_rows(rng, V, adjs)
    rel = check_sampled_rows(kind, params, weights, h, adjs, out, rows)
    # run-to-run determinism at full size (CSR order, no atomics on these paths)
    out2 = layer(MessagePassingInput(torch.from_numpy(h).to(dev), adj_dev), prepared=prepared)
    assert torch.equal(out, out2)
    print(f"{name}: rel err {rel:.2e} over {len(rows)} rows")
