"""The row tiling of the fused RGCN kernel (fused_rgcn_rows_kernel: 64-row x H tiles in one N pass, CTA pairs sharing
each weight stage), taken by the full-size launch for 64 < H <= 256 with H % 32 == 0.

Every case runs with split-tile mode off, so the launch takes the row tiling, and checks it against the float64 oracle and
run to run.  Batches with fewer 128-row tiles than SMs / 2 can also run split-tile mode, which keeps the multi-pass tiling
of fused_rgcn_kernel; there the two tilings must give the same bits (the K order of every output element is the same).
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

from oracle import message_passing_oracle as mo
from test_gpu_parity import _need_gpu, make_layer, random_graph, run_case

pytestmark = pytest.mark.gpu


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("V,D,H,L,E,agg,act,graph", [
    (64 * 37 + 5, 128, 256, 4, 30000, "sum", "relu", dict(hub=True, dups=True)),          # 38 tiles: idle CTA, tail
    (64 * 51, 256, 96, 3, 25000, "mean", "tanh", dict(hub=True, empty_type=1)),          # 51 tiles, empty type
    (64 * 80 + 63, 256, 128, 4, 40000, "sqrt_n", "gelu", dict(hub=True, self_loops=True)),
    (64 * 45 + 1, 512, 192, 2, 20000, "sum", "leaky_relu", dict(hub=True, empty_type=0)),  # D = 512: Q = 4 ring
    (64 * 300 + 17, 256, 256, 4, 120000, "mean", "tanh", dict(hub=True, dups=True)),     # 301 tiles: several per CTA
    (40, 128, 160, 3, 200, "sum", "relu", dict()),                                         # one tile, V < 64
])
def test_rows_tiling_oracle_and_reproducible(monkeypatch, V, D, H, L, E, agg, act, graph):
    _need_gpu()
    rng = np.random.default_rng(V + D + H)
    adjs = random_graph(rng, V, L, E, **graph)
    p = mo.default_hyperparameters("rgcn")
    p.update(hidden_dim=H, aggregation_function=agg, message_activation_function=act)
    monkeypatch.setenv("TFGNN_B200_FUSED_SPLIT", "0")
    a = run_case("rgcn", p, V, D, L, adjs, seed=V, path="fused_tc")
    b = run_case("rgcn", p, V, D, L, adjs, seed=V, path="fused_tc")
    assert np.array_equal(a.cpu().numpy().view(np.uint32), b.cpu().numpy().view(np.uint32))


@pytest.mark.parametrize("V,D,H,L,E,act", [
    (128 * 66 - 40, 256, 256, 4, 60000, "relu"),    # 66 128-row tiles: split-tile mode on 132 SMs
    (128 * 40 + 3, 256, 256, 4, 40000, "tanh"),     # tanh: corrections as two tf32 MMAs
    (128 * 30, 128, 192, 3, 20000, "gelu"),
    (128 * 21 + 9, 384, 96, 2, 9000, "relu"),
])
def test_rows_tiling_matches_multi_pass_tiling_bitwise(monkeypatch, V, D, H, L, E, act):
    _need_gpu()
    if 2 * ((V + 127) // 128) > min(_sms(), 160):
        pytest.skip("split-tile mode needs fewer 128-row tiles than SMs / 2")
    rng = np.random.default_rng(V + H)
    adjs = random_graph(rng, V, L, E, hub=True, dups=True)
    p = mo.default_hyperparameters("rgcn")
    p.update(hidden_dim=H, aggregation_function="mean", message_activation_function=act)
    monkeypatch.setenv("TFGNN_B200_FUSED_SPLIT", "1")
    old = run_case("rgcn", p, V, D, L, adjs, seed=V, path="fused_tc")
    monkeypatch.setenv("TFGNN_B200_FUSED_SPLIT", "0")
    new = run_case("rgcn", p, V, D, L, adjs, seed=V, path="fused_tc")
    assert np.array_equal(old.cpu().numpy().view(np.uint32), new.cpu().numpy().view(np.uint32))


@pytest.mark.parametrize("V,lo,hi", [(20000, 64 * 100, 20000 - 77), (9001, 0, 64 * 41 + 7)])
def test_rows_tiling_allgather_replica_stores(monkeypatch, V, lo, hi):
    """tfgnn_b200_rgcn_fwd_allgather on one GPU through the row tiling: every replica gets exactly the rows of the plain
    sharded call, at rows [lo, hi), and nothing else (the shard's last cluster has an idle CTA)."""
    _need_gpu()
    from tf2_gnn_b200.layers import MessagePassingInput
    from tf2_gnn_b200.runtime import PreparedBatch
    D, H, L = 256, 256, 4
    monkeypatch.setenv("TFGNN_B200_FUSED_SPLIT", "0")
    rng = np.random.default_rng(V + lo)
    adjs = random_graph(rng, V, L, 8 * V, hub=True)
    p = mo.default_hyperparameters("rgcn")
    p.update(hidden_dim=H)
    w = mo.make_weights("rgcn", p, D, L, rng)
    layer = make_layer("rgcn", p, D, L, w)
    h = torch.from_numpy(rng.uniform(-1, 1, (V, D)).astype(np.float32)).cuda()
    adj_t = tuple(torch.from_numpy(a).cuda() for a in adjs)
    shard = PreparedBatch(adj_t, V, target_range=(lo, hi))
    ref = layer(MessagePassingInput(h, adj_t), prepared=shard)
    tables = [torch.full((V, H), -7.0, device="cuda") for _ in range(3)]
    layer.call_allgather(h, shard, [t.data_ptr() for t in tables], own_rank=1)
    torch.cuda.synchronize()
    for t in tables:
        assert torch.equal(t[lo:hi], ref)
        assert bool((t[:lo] == -7.0).all()) and bool((t[hi:] == -7.0).all())
