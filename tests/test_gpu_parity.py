"""Parity of the CUDA path (through the Python facade -> ctypes -> C ABI) against the oracle.

Tolerance for node states (north_star: 1e-5 relative fp32): |got - ref64| <= 1e-5 * max|ref64|,
where ref64 is the float64 evaluation of the oracle (norm-wise criterion, SURVEY.md §7: element-wise
relative error is ill-defined next to ReLU zero crossings).  Index bookkeeping is bit-exact.
"""
import json
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")

from oracle import message_passing_oracle as mo

pytestmark = pytest.mark.gpu

TOL = 1e-5
LOWEST = np.finfo(np.float32).min


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def assert_states_close(got, ref64, tol=TOL):
    got = np.asarray(got, dtype=np.float64)
    ref64 = np.asarray(ref64, dtype=np.float64)
    assert got.shape == ref64.shape
    sentinel = ref64 <= LOWEST * 0.99  # unsorted_segment_max identity on empty segments
    assert np.array_equal(sentinel, got <= LOWEST * 0.99)
    r = np.where(sentinel, 0.0, ref64)
    g = np.where(sentinel, 0.0, got)
    scale = max(np.abs(r).max() if r.size else 0.0, 1e-30)
    err = np.abs(g - r).max() if r.size else 0.0
    assert err <= tol * scale, f"max abs err {err:.3e} > {tol:g} * {scale:.3e}"


def random_graph(rng, V, L, edges_per_type, empty_type=None, hub=False, self_loops=False, dups=False):
    adjs = []
    for l in range(L):
        E = int(edges_per_type if np.isscalar(edges_per_type) else edges_per_type[l])
        if empty_type is not None and l == empty_type:
            adjs.append(np.zeros((0, 2), np.int32))
            continue
        a = rng.integers(0, V, size=(E, 2)).astype(np.int32)
        if hub and E:
            a[: E // 2, 1] = V // 3  # half of the edges hit one target
        if self_loops and l == 0:
            ids = np.arange(V, dtype=np.int32)
            a = np.stack([ids, ids], axis=1)
        if dups and E >= 4:
            a[1] = a[0]
            a[3] = a[0]
        adjs.append(a)
    return adjs


def make_layer(kind, params, D, L, weights):
    from tf2_gnn_b200.layers import MessagePassingInput, get_message_passing_class
    layer = get_message_passing_class(kind)(params)
    layer.build(MessagePassingInput((None, D), tuple((None, 2) for _ in range(L))))
    layer.set_weights_from_oracle_dict(weights)
    return layer


def run_case(kind, params, V, D, L, adjs, seed=0, path="auto"):
    from tf2_gnn_b200.layers import MessagePassingInput
    rng = np.random.default_rng(seed)
    h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    w = mo.make_weights(kind, params, D, L, rng)
    params = dict(params, b200_path=path)
    layer = make_layer(kind, params, D, L, w)
    out = layer(MessagePassingInput(torch.from_numpy(h).cuda(), tuple(torch.from_numpy(a).cuda() for a in adjs)))
    torch.cuda.synchronize()
    assert tuple(out.shape) == (V, int(params["hidden_dim"])) and out.dtype == torch.float32
    ref64 = mo.message_passing_forward(kind, params, w, h, adjs, dtype=np.float64)
    assert_states_close(out.cpu().numpy(), ref64)
    return out


# ------------------------------------------------------------------------------------------
# Golden vectors of the reference's own tests
# ------------------------------------------------------------------------------------------
def test_golden_pass_source_states(golden_dir):
    """tf2_gnn/test/layers/test_message_passing.py:11-84 on the generic plugin path."""
    _need_gpu()
    from tf2_gnn_b200.layers import MessagePassing, MessagePassingInput

    class PassSourceStates(MessagePassing):
        def __init__(self):
            params = super().get_default_hyperparameters()
            params["message_activation_function"] = "relu"
            params["aggregation_function"] = "sum"
            super().__init__(params)

        def _message_function(self, edge_source_states, edge_target_states, num_incoming_to_node_per_message,
                              edge_type_idx, training):
            return edge_source_states

    with open(os.path.join(golden_dir, "message_passing_golden.json")) as f:
        g = json.load(f)
    for case in g["pass_source_states"]:
        layer = PassSourceStates()
        inp = MessagePassingInput(
            node_embeddings=torch.tensor(case["node_embeddings"], dtype=torch.float32).cuda(),
            adjacency_lists=tuple(torch.tensor(a, dtype=torch.int32).cuda() for a in case["adjacency_lists"]))
        out = layer(inp, training=False)
        expected = np.array(case["aggregated_states"], np.float32)
        assert tuple(out.shape) == expected.shape
        np.testing.assert_array_almost_equal(out.cpu().numpy(), expected)


def test_golden_in_degree_doctest(golden_dir):
    """message_passing.py:238-249 — exact."""
    _need_gpu()
    from tf2_gnn_b200.layers.message_passing import calculate_type_to_num_incoming_edges
    with open(os.path.join(golden_dir, "message_passing_golden.json")) as f:
        d = json.load(f)["in_degree_doctest"]
    got = calculate_type_to_num_incoming_edges(
        torch.zeros((d["num_nodes"], 3)).cuda(),
        [torch.tensor(a, dtype=torch.int32).cuda() for a in d["adjacency_lists"]])
    assert got.dtype == torch.float32
    assert np.array_equal(got.cpu().numpy(), np.array(d["type_to_num_incoming_edges"], np.float32))


def test_in_degree_on_process_adjacency_golden(golden_dir):
    """In-degree of every golden processed adjacency (test/data/test_utils.py:50-115) — exact."""
    _need_gpu()
    from tf2_gnn_b200.layers.message_passing import calculate_type_to_num_incoming_edges
    with open(os.path.join(golden_dir, "process_adjacency_lists_golden.json")) as f:
        g = json.load(f)
    for case in g["cases"]:
        n = case["input"]["num_nodes"]
        adjs = [torch.tensor(np.array(a, np.int32).reshape(-1, 2)).cuda() for a in case["adjacency_lists"]]
        got = calculate_type_to_num_incoming_edges(torch.zeros((n, 1)).cuda(), adjs).cpu().numpy()
        assert np.array_equal(got, np.array(case["type_to_num_incoming_edges"], np.float32).reshape(len(adjs), n))


# ------------------------------------------------------------------------------------------
# Index bookkeeping: bit-exact
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V,L,E", [(1, 1, 1), (37, 3, 200), (5000, 4, 40000), (300, 2, 9000), (2000, 2, 300001)])
def test_csr_is_bit_exact(V, L, E):
    _need_gpu()
    from tf2_gnn_b200.runtime import PreparedBatch
    rng = np.random.default_rng(V + L + E)
    adjs = random_graph(rng, V, L, E, empty_type=1 if L > 2 else None, hub=True, dups=True)
    pb = PreparedBatch([torch.from_numpy(a).cuda() for a in adjs], V)
    row_ptr, src = (t.cpu().numpy() for t in pb.csr())
    counts = np.concatenate([np.bincount(a[:, 1], minlength=V) for a in adjs])
    expect_ptr = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    assert np.array_equal(row_ptr, expect_ptr)
    for l, a in enumerate(adjs):
        order = np.argsort(a[:, 1], kind="stable")
        by_tgt = a[order]
        for v in np.unique(a[:, 1])[:200]:
            seg = src[row_ptr[l * V + v]: row_ptr[l * V + v + 1]]
            ref = np.sort(by_tgt[by_tgt[:, 1] == v, 0])
            assert np.array_equal(seg, ref)  # canonical ascending order, hubs included
    indeg = pb.in_degree().cpu().numpy()
    assert np.array_equal(indeg, mo.calculate_type_to_num_incoming_edges(V, adjs))


def test_out_of_range_index_raises_with_validation():
    _need_gpu()
    from tf2_gnn_b200.runtime import PreparedBatch
    adj = torch.tensor([[0, 1], [5, 1]], dtype=torch.int32).cuda()
    with pytest.raises(IndexError):
        PreparedBatch([adj], 3, validate=True)
    pb = PreparedBatch([adj], 3, validate=False)  # dropped, like TF on GPU
    assert pb.in_degree().cpu().numpy().tolist() == [[0.0, 1.0, 0.0]]


# ------------------------------------------------------------------------------------------
# RGCN (primary target)
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V,D,H,L,E,opts", [
    (5, 3, 12, 3, 3, {}),                        # doctest-sized (scalar fallback kernels)
    (64, 7, 7, 14, 50, {}),                      # test_RGCN.py shape case: 14 edge types, odd dims
    (500, 64, 64, 3, 4000, dict(self_loops=True)),
    (1000, 128, 128, 4, 6000, dict(hub=True, dups=True)),
    (2000, 320, 320, 3, 20000, dict(self_loops=True)),   # PPI-like hidden size
    (3000, 256, 256, 4, 15000, dict(empty_type=2)),      # cfg2-like hidden size, one empty type
    (257, 100, 36, 2, 1000, {}),                 # D%4==0, H%4==0 but not tile multiples
])
@pytest.mark.parametrize("path", ["sorted", "auto"])
def test_rgcn_parity(V, D, H, L, E, opts, path):
    _need_gpu()
    rng = np.random.default_rng(V * 7 + D)
    adjs = random_graph(rng, V, L, E, **opts)
    p = mo.default_hyperparameters("rgcn")
    p["hidden_dim"] = H
    run_case("rgcn", p, V, D, L, adjs, seed=V, path=path)


@pytest.mark.parametrize("chunk_rows,V", [(256, 3000), (128, 1000), (None, 160000)])
def test_rgcn_pipelined_two_stream(chunk_rows, V, monkeypatch):
    """gather || tensor-core-GEMM pipeline over node chunks (triple-buffered) == oracle.  D = 36 (D % 4 == 0, D % 32 != 0):
    the fused kernel refuses the shape, so `auto` takes the pipeline, which makes one gather and one GEMM launch per chunk
    more than the one-shot path."""
    from tf2_gnn_b200 import _ffi
    _need_gpu()
    rows = chunk_rows if chunk_rows is not None else 2 * 132 * 128
    if chunk_rows is not None:
        monkeypatch.setenv("TFGNN_B200_PIPE_CHUNK_ROWS", str(chunk_rows))
    rng = np.random.default_rng(V)
    D, H = 36, 64
    L = 3
    adjs = random_graph(rng, V, L, V * 3, hub=True, self_loops=True)
    p = mo.default_hyperparameters("rgcn")
    p.update(hidden_dim=H, aggregation_function="mean", message_activation_function="tanh")
    n0 = _ffi.launch_count()
    a = run_case("rgcn", p, V, D, L, adjs, seed=2, path="auto")
    n1 = _ffi.launch_count()
    monkeypatch.setenv("TFGNN_B200_PIPE_CHUNK_ROWS", str(1 << 24))   # disables the pipeline
    b = run_case("rgcn", p, V, D, L, adjs, seed=2, path="sorted_tc")
    n2 = _ffi.launch_count()
    assert_states_close(a.cpu().numpy(), b.cpu().numpy().astype(np.float64), tol=1e-6)
    chunks = -(-V // rows)
    assert (n1 - n0) - (n2 - n1) >= 2 * (chunks - 1), f"{n1 - n0} vs {n2 - n1} launches: the pipeline did not run"


@pytest.mark.parametrize("V,D,H,L,E,opts,agg", [
    (100, 32, 16, 1, 300, {}, "sum"),
    (129, 64, 64, 3, 1000, dict(self_loops=True), "sum"),
    (5000, 128, 128, 4, 30000, dict(hub=True, dups=True), "mean"),
    (3000, 256, 256, 4, 15000, dict(empty_type=2), "sum"),
    (40000, 256, 256, 3, 150000, dict(hub=True), "sqrt_n"),
    (20000, 320, 256, 2, 60000, {}, "sum"),
    (1000, 96, 48, 5, 4000, {}, "sum"),
    (3000, 320, 320, 3, 20000, dict(self_loops=True), "sum"),     # PPI hidden size: two N passes over the ring
    (20000, 320, 320, 3, 100000, dict(hub=True), "mean"),
    (2500, 128, 512, 2, 9000, {}, "sum"),
])
def test_rgcn_fused_kernel(V, D, H, L, E, opts, agg):
    """fused_rgcn_kernel: gather -> segment-sum -> wgmma 3xTF32 -> activation in one persistent kernel."""
    _need_gpu()
    rng = np.random.default_rng(V + D + H)
    adjs = random_graph(rng, V, L, E, **opts)
    p = mo.default_hyperparameters("rgcn")
    p.update(hidden_dim=H, aggregation_function=agg, message_activation_function="tanh")
    a = run_case("rgcn", p, V, D, L, adjs, seed=V, path="fused_tc")
    b = run_case("rgcn", p, V, D, L, adjs, seed=V, path="sorted")
    assert_states_close(a.cpu().numpy(), b.cpu().numpy().astype(np.float64), tol=1e-5)
    a2 = run_case("rgcn", p, V, D, L, adjs, seed=V, path="fused_tc")
    assert np.array_equal(a.cpu().numpy(), a2.cpu().numpy())   # bitwise reproducible


@pytest.mark.parametrize("pair", ["0", "2"])
@pytest.mark.parametrize("V,D,H,L,E,agg", [
    (300, 32, 16, 2, 1500, "sum"),            # 3 tiles: the peer CTA of the last pair has no tile
    (1000, 96, 48, 5, 4000, "mean"),
    (5000, 256, 256, 4, 30000, "sum"),
    (3000, 320, 320, 3, 20000, "sqrt_n"),     # two N passes, 80 weight rows per CTA
    (25000, 64, 80, 2, 80000, "sum"),         # 196 tiles > SM count: pairs by the default rule as well
])
def test_rgcn_fused_kernel_cta_pairs(monkeypatch, pair, V, D, H, L, E, agg):
    """The fused kernel under both settings of TFGNN_B200_FUSED_PAIR (the CTA-pair switch of earlier builds, which the
    kernel now ignores) against the fp32 CSR path and run to run."""
    _need_gpu()
    monkeypatch.setenv("TFGNN_B200_FUSED_PAIR", pair)
    rng = np.random.default_rng(V + D + H + 1)
    adjs = random_graph(rng, V, L, E, hub=True, self_loops=True)
    p = mo.default_hyperparameters("rgcn")
    p.update(hidden_dim=H, aggregation_function=agg, message_activation_function="relu")
    a = run_case("rgcn", p, V, D, L, adjs, seed=V, path="fused_tc")
    b = run_case("rgcn", p, V, D, L, adjs, seed=V, path="sorted")
    assert_states_close(a.cpu().numpy(), b.cpu().numpy().astype(np.float64), tol=1e-5)
    a2 = run_case("rgcn", p, V, D, L, adjs, seed=V, path="fused_tc")
    assert np.array_equal(a.cpu().numpy(), a2.cpu().numpy())


@pytest.mark.parametrize("V,D,H,L,E,agg,act", [
    (129, 64, 64, 3, 1000, "sum", "relu"),          # 2 tiles, the second with a single row
    (8000, 320, 320, 3, 120000, "sum", "relu"),      # BASELINE cfg1 shape (63 tiles): H/2 = 160 columns per CTA
    (5000, 128, 128, 4, 30000, "mean", "tanh"),      # tanh -> two-tf32-MMA corrections in the split kernel
    (9000, 256, 256, 4, 40000, "sqrt_n", "gelu"),    # 71 tiles: just under SMs / 2
    (2500, 128, 512, 2, 9000, "sum", "relu"),        # H/2 = 256: full-width accumulators per CTA
    (700, 96, 64, 5, 6000, "sum", "leaky_relu"),     # D = 96: three 32-float K blocks per type
])
def test_rgcn_fused_kernel_split_tiles(monkeypatch, V, D, H, L, E, agg, act):
    """Split-tile mode of the fused kernel (batches with fewer tiles than SMs / 2: two CTAs of a cluster share a tile, half
    of the gathered rows and half of the output columns each) against the oracle, against the one-CTA-per-tile kernel
    (same bits: the K order of every output element is unchanged) and run to run."""
    _need_gpu()
    rng = np.random.default_rng(V + H)
    adjs = random_graph(rng, V, L, E, hub=True, self_loops=True, dups=True)
    p = mo.default_hyperparameters("rgcn")
    p.update(hidden_dim=H, aggregation_function=agg, message_activation_function=act)
    monkeypatch.setenv("TFGNN_B200_FUSED_SPLIT", "1")
    a = run_case("rgcn", p, V, D, L, adjs, seed=V, path="fused_tc")
    a2 = run_case("rgcn", p, V, D, L, adjs, seed=V, path="fused_tc")
    assert np.array_equal(a.cpu().numpy(), a2.cpu().numpy())
    monkeypatch.setenv("TFGNN_B200_FUSED_SPLIT", "0")
    b = run_case("rgcn", p, V, D, L, adjs, seed=V, path="fused_tc")
    assert np.array_equal(a.cpu().numpy(), b.cpu().numpy())


@pytest.mark.parametrize("q", ["1", "2", "3", "8"])
def test_rgcn_fused_kernel_gather_ring_depths(monkeypatch, q):
    """The rolling cp.async gather ring with Q = 1..8 row slots per warp: long segments (hubs > 32 edges cross the
    index-block boundary), empty types, a last tile with a single node; all depths give the same bits."""
    _need_gpu()
    V, D, H, L = 128 * 37 + 1, 128, 64, 4
    rng = np.random.default_rng(77)
    adjs = random_graph(rng, V, L, 60000, hub=True, dups=True, empty_type=2, self_loops=True)
    p = mo.default_hyperparameters("rgcn")
    p.update(hidden_dim=H, aggregation_function="mean", message_activation_function="tanh")
    monkeypatch.setenv("TFGNN_B200_GATHER_Q", q)
    a = run_case("rgcn", p, V, D, L, adjs, seed=5, path="fused_tc")
    monkeypatch.setenv("TFGNN_B200_GATHER_Q", "4")
    b = run_case("rgcn", p, V, D, L, adjs, seed=5, path="fused_tc")
    assert np.array_equal(a.cpu().numpy(), b.cpu().numpy())


def test_rgcn_atomic_path_matches():
    _need_gpu()
    rng = np.random.default_rng(5)
    V, D, H, L = 1500, 128, 128, 3
    adjs = random_graph(rng, V, L, 12000, hub=True)
    p = mo.default_hyperparameters("rgcn")
    p["hidden_dim"] = H
    a = run_case("rgcn", p, V, D, L, adjs, seed=1, path="atomic")
    b = run_case("rgcn", p, V, D, L, adjs, seed=1, path="sorted")
    assert_states_close(a.cpu().numpy(), b.cpu().numpy().astype(np.float64))


def test_rgcn_isolated_nodes_and_no_edges():
    _need_gpu()
    p = mo.default_hyperparameters("rgcn")
    p["hidden_dim"] = 16
    adjs = [np.zeros((0, 2), np.int32), np.array([[0, 1]], np.int32)]
    out = run_case("rgcn", p, 10, 16, 2, adjs)
    assert np.all(out.cpu().numpy()[2:] == 0.0)  # sigma(0) for nodes without incoming edges
    run_case("rgcn", p, 10, 16, 2, [np.zeros((0, 2), np.int32)] * 2)


def test_rgcn_is_deterministic_run_to_run():
    _need_gpu()
    from tf2_gnn_b200.layers import MessagePassingInput
    rng = np.random.default_rng(3)
    V, D, H, L = 4000, 128, 128, 3
    adjs = [torch.from_numpy(a).cuda() for a in random_graph(rng, V, L, 60000, hub=True)]
    h = torch.from_numpy(rng.uniform(-1, 1, (V, D)).astype(np.float32)).cuda()
    p = mo.default_hyperparameters("rgcn")
    p["hidden_dim"] = H
    layer = make_layer("rgcn", p, D, L, mo.make_weights("rgcn", p, D, L, rng))
    a = layer(MessagePassingInput(h, tuple(adjs))).cpu().numpy()
    b = layer(MessagePassingInput(h, tuple(adjs))).cpu().numpy()
    assert np.array_equal(a, b)


# ------------------------------------------------------------------------------------------
# Edge-MLP family over its hyper-parameter grid
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("agg", ["sum", "mean", "max", "sqrt_n"])
@pytest.mark.parametrize("act_before", [False, True])
@pytest.mark.parametrize("use_target,normalize,n_hidden", [
    (False, True, 0), (True, False, 0), (True, True, 0), (False, False, 1), (True, True, 1)])
def test_edge_mlp_grid(agg, act_before, use_target, normalize, n_hidden):
    _need_gpu()
    rng = np.random.default_rng(11)
    V, D, H, L = 300, 32, 48, 3
    adjs = random_graph(rng, V, L, 2500, hub=True, dups=True)
    p = mo.default_hyperparameters("gnn_edge_mlp")
    p.update(hidden_dim=H, aggregation_function=agg, message_activation_before_aggregation=act_before,
             use_target_state_as_input=use_target, normalize_by_num_incoming=normalize,
             num_edge_MLP_hidden_layers=n_hidden, message_activation_function="tanh")
    # n_hidden >= 1 with max / act-before runs the literal per-edge path (literal.cu)
    run_case("gnn_edge_mlp", p, V, D, L, adjs)


@pytest.mark.parametrize("kind,extra", [
    ("gnn_edge_mlp", dict(num_edge_MLP_hidden_layers=2)),
    ("gnn_edge_mlp", dict(num_edge_MLP_hidden_layers=3, aggregation_function="max", use_target_state_as_input=False)),
    ("rgin", dict(num_edge_MLP_hidden_layers=2, num_aggr_MLP_hidden_layers=1)),
    ("gnn_film", dict(num_edge_MLP_hidden_layers=1, normalize_by_num_incoming=True)),
    ("gnn_film", dict(num_edge_MLP_hidden_layers=2, message_activation_before_aggregation=True,
                      use_target_state_as_input=True, aggregation_function="mean")),
    ("ggnn", dict(num_edge_MLP_hidden_layers=2)),
])
def test_literal_per_edge_path(kind, extra):
    """Hyper-parameter combinations whose per-edge non-linearity cannot be hoisted to node level."""
    _need_gpu()
    rng = np.random.default_rng(31)
    V, D, H, L = 250, 48, 48, 3
    adjs = random_graph(rng, V, L, 1800, hub=True, dups=True, empty_type=1)
    p = mo.default_hyperparameters(kind)
    p.update(hidden_dim=H, message_activation_function="tanh")
    p.update(extra)
    run_case(kind, p, V, D, L, adjs)


@pytest.mark.parametrize("act", ["relu", "tanh", "leaky_relu", "elu", "selu", "gelu"])
def test_activations(act):
    _need_gpu()
    rng = np.random.default_rng(2)
    adjs = random_graph(rng, 200, 2, 1500)
    p = mo.default_hyperparameters("rgcn")
    p.update(hidden_dim=32, message_activation_function=act)
    run_case("rgcn", p, 200, 32, 2, adjs)
    p["message_activation_before_aggregation"] = True
    run_case("rgcn", p, 200, 32, 2, adjs)


@pytest.mark.parametrize("fused_gru", ["1", "0"])
@pytest.mark.parametrize("V,H", [(700, 128), (1000, 96), (257, 32), (300, 40)])
def test_ggnn_parity(V, H, fused_gru, monkeypatch):
    """GGNN layer (ggnn.py:68-89).  fused_gru=1: the GRU update is ONE tensor-core contraction over [agg | h] with the gate math
    in its epilogue (hidden_dim % 32 == 0; 40 falls back); 0: two GEMMs + the gate kernel.  Same oracle, same bar."""
    _need_gpu()
    monkeypatch.setenv("TFGNN_B200_GGNN_FUSED_GRU", fused_gru)
    rng = np.random.default_rng(4)
    L = 5
    adjs = random_graph(rng, V, L, 3 * V, self_loops=True)
    p = mo.default_hyperparameters("ggnn")
    p["hidden_dim"] = H
    run_case("ggnn", p, V, H, L, adjs)
    p["normalize_by_num_incoming"] = False   # PPI_GGNN.json:9
    run_case("ggnn", p, V, H, L, adjs)


@pytest.mark.parametrize("n_aggr", [None, 0, 2])
def test_rgin_parity(n_aggr):
    _need_gpu()
    rng = np.random.default_rng(6)
    V, D, H, L = 400, 64, 64, 3
    adjs = random_graph(rng, V, L, 3000)
    p = mo.default_hyperparameters("rgin")
    p.update(hidden_dim=H, num_aggr_MLP_hidden_layers=n_aggr, normalize_by_num_incoming=True)
    run_case("rgin", p, V, D, L, adjs)


@pytest.mark.parametrize("use_target,act_before,agg", [(False, False, "sum"), (True, False, "sum"),
                                                        (False, True, "sum"), (True, True, "max")])
@pytest.mark.parametrize("att", ["0", "1"])
def test_film_parity(monkeypatch, att, use_target, act_before, agg):
    """att = 1: aggregate-then-transform with the FiLM modulation chained through the GEMM epilogue (the form target-range
    shards use); att = 0: projected tables + per-edge modulation.  (max / activation-before always take the latter.)"""
    _need_gpu()
    monkeypatch.setenv("TFGNN_B200_FILM_ATT", att)
    rng = np.random.default_rng(8)
    V, D, H, L = 500, 64, 64, 4
    adjs = random_graph(rng, V, L, 3000, hub=True)
    p = mo.default_hyperparameters("gnn_film")
    p.update(hidden_dim=H, use_target_state_as_input=use_target, message_activation_before_aggregation=act_before,
             aggregation_function=agg, normalize_by_num_incoming=True)
    run_case("gnn_film", p, V, D, L, adjs)


@pytest.mark.parametrize("fused_scores", ["1", "0"])
@pytest.mark.parametrize("V,D,H,K,L,E", [(5, 3, 12, 3, 3, 3), (400, 64, 64, 4, 3, 3000), (300, 32, 36, 3, 2, 2000),
                                         (1000, 128, 128, 4, 3, 8000), (700, 64, 256, 8, 2, 5000),
                                         (600, 32, 64, 2, 5, 4000)])
def test_rgat_parity(V, D, H, K, L, E, fused_scores, monkeypatch):
    """fused_scores=1: the attention score halves come out of the projection GEMM's epilogue where the tile layout allows
    it (per-head dim % 16 == 0: (64,4), (128,4), (256,8), (64,2)); 0: the separate score kernel.  Same oracle, same bar."""
    _need_gpu()
    monkeypatch.setenv("TFGNN_B200_RGAT_FUSED_SCORES", fused_scores)
    rng = np.random.default_rng(V + H)
    adjs = random_graph(rng, V, L, E, hub=V > 100, dups=True)
    p = mo.default_hyperparameters("rgat")
    p.update(hidden_dim=H, num_heads=K, message_activation_function="tanh")
    run_case("rgat", p, V, D, L, adjs)


@pytest.mark.parametrize("kind,extra", [
    ("rgcn", dict(dense_every_num_layers=10000, residual_every_num_layers=10000)),          # PPI_RGCN.json shape
    ("rgcn", dict(use_inter_layer_layernorm=True, message_activation_function="leaky_relu")),  # QM9_RGCN.json
    ("gnn_film", dict(dense_every_num_layers=1, residual_every_num_layers=2, use_target_state_as_input=True)),
    ("ggnn", dict(num_layers=3, normalize_by_num_incoming=False, message_activation_function="tanh")),
])
def test_gnn_stack_parity(kind, extra):
    """GNN._internal_call (gnn.py:276-329): projection, residuals, MP layers, LayerNorm, Dense."""
    _need_gpu()
    from tf2_gnn_b200.layers import GNN, GNNInput
    rng = np.random.default_rng(17)
    V, F, H, L = 600, 50, 64, 3
    adjs = random_graph(rng, V, L, 4000, self_loops=True)
    params = GNN.get_default_hyperparameters(kind)
    params.update(hidden_dim=H, global_exchange_every_num_layers=10000)
    params.update(extra)
    feats = rng.uniform(-1, 1, (V, F)).astype(np.float32)
    gnn = GNN(params)
    gnn.build(GNNInput((None, F), tuple((None, 2) for _ in range(L)), (None,), ()))
    w = {"initial_projection": mo.glorot_uniform(rng, (F, H)), "mp": [], "dense": {}, "layernorm": []}
    gnn._initial_projection_layer.kernel.assign(w["initial_projection"])
    for i, mp in enumerate(gnn._mp_layers):
        wi = mo.make_weights(kind, params, H, L, rng)
        mp.set_weights_from_oracle_dict(wi)
        w["mp"].append(wi)
        if params["use_inter_layer_layernorm"]:
            g, b = rng.uniform(0.5, 1.5, H).astype(np.float32), rng.uniform(-0.2, 0.2, H).astype(np.float32)
            gnn._inter_layer_layernorms[i].gamma.assign(g)
            gnn._inter_layer_layernorms[i].beta.assign(b)
            w["layernorm"].append((g, b))
        if str(i) in gnn._dense_layers:
            w["dense"][i] = mo.glorot_uniform(rng, (H, H))
            gnn._dense_layers[str(i)].kernel.assign(w["dense"][i])
    inp = GNNInput(torch.from_numpy(feats).cuda(), tuple(torch.from_numpy(a).cuda() for a in adjs),
                   torch.zeros(V, dtype=torch.int32).cuda(), 1)
    out, all_reps = gnn(inp, training=False, return_all_representations=True)
    ref, ref_all = mo.gnn_forward(params, w, feats, adjs, dtype=np.float64)
    ref32, ref32_all = mo.gnn_forward(params, w, feats, adjs, dtype=np.float32)
    assert len(all_reps) == len(ref_all) == params["num_layers"] + 1

    def close_as_fp32(got, r64, r32):
        # Through a deep stack the fp32 reference itself drifts from the exact result (FiLM: 1e-4 after 4
        # layers); the bar is 1e-5 relative OR within 3x of the fp32 restatement's own error.
        fp32_err = np.abs(r32.astype(np.float64) - r64).max()
        scale = max(np.abs(r64).max(), 1e-30)
        err = np.abs(got.astype(np.float64) - r64).max()
        assert err <= max(1e-5 * scale, 3.0 * fp32_err), f"err {err:.3e}, fp32 oracle err {fp32_err:.3e}, scale {scale:.3e}"

    close_as_fp32(out.cpu().numpy(), ref, ref32)
    for a, b, c in zip(all_reps, ref_all, ref32_all):
        close_as_fp32(a.cpu().numpy(), b, c)
    # Without per-layer representations the stack may fuse LayerNorm into the layer kernel's epilogue: a
    # different rounding order, so the same parity bar (not bit equality) against the oracle; repeated calls
    # of the same path are bit-identical.
    out2 = gnn(inp)
    close_as_fp32(out2.cpu().numpy(), ref, ref32)
    assert np.array_equal(gnn(inp).cpu().numpy(), out2.cpu().numpy())


@pytest.mark.parametrize("kind,extra", [("rgcn", {}), ("gnn_film", dict(use_target_state_as_input=True)),
                                        ("ggnn", {}), ("rgat", dict(num_heads=4)),
                                        ("gnn_edge_mlp", dict(aggregation_function="max", num_edge_MLP_hidden_layers=0))])
def test_target_range_shards_match_full(kind, extra):
    """SURVEY.md §8e case 2 on one GPU: each target-range shard (tfgnn_b200_prepare_sharded) computes its
    rows from the full source table; the concatenation equals the unsharded layer."""
    _need_gpu()
    from tf2_gnn_b200 import sharding
    from tf2_gnn_b200.layers import MessagePassingInput
    from tf2_gnn_b200.runtime import PreparedBatch
    rng = np.random.default_rng(21)
    V, D, H, L = 700, 64, 64, 3
    adjs = random_graph(rng, V, L, 5000, hub=True)
    p = mo.default_hyperparameters(kind)
    p.update(hidden_dim=H)
    p.update(extra)
    w = mo.make_weights(kind, p, D, L, rng)
    h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    layer = make_layer(kind, p, D, L, w)
    ht = torch.from_numpy(h).cuda()
    adj_t = tuple(torch.from_numpy(a).cuda() for a in adjs)
    full = layer(MessagePassingInput(ht, adj_t)).cpu().numpy()
    assert_states_close(full, mo.message_passing_forward(kind, p, w, h, adjs, dtype=np.float64))
    deg = sum(np.bincount(a[:, 1], minlength=V) for a in adjs)
    for world in (2, 3):
        bounds = sharding.partition_target_range(V, world, deg)
        parts = []
        for lo, hi in bounds:
            for filtered in (False, True):
                a_in = adj_t if not filtered else tuple(
                    torch.from_numpy(a).cuda() for a in sharding.filter_edges_by_target(adjs, lo, hi))
                pb = PreparedBatch(a_in, V, target_range=(lo, hi))
                out = layer(MessagePassingInput(ht, a_in), prepared=pb)
                assert tuple(out.shape) == (hi - lo, H)
                if filtered:
                    parts.append(out.cpu().numpy())
                else:
                    first = out.cpu().numpy()
            assert np.array_equal(first, parts[-1])  # unfiltered and pre-filtered edge lists agree
        got = np.concatenate(parts, axis=0)
        assert_states_close(got, mo.message_passing_forward(kind, p, w, h, adjs, dtype=np.float64))
        if kind != "gnn_film":   # FiLM shards use the aggregate-then-transform form, the full batch the projected tables
            assert_states_close(got, full.astype(np.float64), tol=2e-6)


def _torch_reference_layer(h, adjs, Ws, normalize, agg, act, use_target=False):
    """float64 autograd restatement of the RGCN layer (reference op order) for gradient parity."""
    V = h.shape[0]
    msgs, tgts = [], []
    for adj, W in zip(adjs, Ws):
        src, tgt = adj[:, 0].long(), adj[:, 1].long()
        x = h.index_select(0, src)
        if use_target:   # gnn_edge_mlp.py:93-98: MLP input = [h_src || h_tgt]
            x = torch.cat([x, h.index_select(0, tgt)], dim=-1)
        m = x @ W
        if normalize:
            c = torch.zeros(V, dtype=h.dtype).index_add_(0, tgt, torch.ones(len(tgt), dtype=h.dtype))
            m = (1.0 / (c.index_select(0, tgt) + 1e-7)).unsqueeze(-1) * m
        msgs.append(m)
        tgts.append(tgt)
    M, T = torch.cat(msgs), torch.cat(tgts)
    out = torch.zeros((V, Ws[0].shape[1]), dtype=h.dtype).index_add_(0, T, M)
    if agg in ("mean", "sqrt_n"):
        n = torch.zeros(V, dtype=h.dtype).index_add_(0, T, torch.ones(len(T), dtype=h.dtype)).clamp(min=1)
        out = out / (n if agg == "mean" else n.sqrt()).unsqueeze(-1)
    def gelu(x):   # utils/activation.py:7-14
        return x * 0.5 * (1.0 + torch.tanh(0.7978845608028654 * (x + 0.044715 * x ** 3)))
    return {"relu": torch.relu, "tanh": torch.tanh, "elu": torch.nn.functional.elu, "selu": torch.selu, "gelu": gelu,
            "leaky_relu": lambda x: torch.nn.functional.leaky_relu(x, 0.2)}[act](out)


@pytest.mark.parametrize("V,D,H,L,E,agg,act,normalize", [
    (300, 32, 48, 3, 2500, "sum", "relu", True),
    (1000, 64, 64, 2, 9000, "mean", "tanh", True),
    (20000, 128, 128, 4, 150000, "sum", "tanh", False),
    (400, 64, 32, 2, 2500, "sum", "leaky_relu", False),
    (700, 256, 256, 3, 5000, "sqrt_n", "elu", True),
    (500, 36, 20, 2, 3000, "sum", "selu", True),
    (900, 64, 48, 3, 7000, "mean", "gelu", True),
])
def test_rgcn_backward_matches_autograd_reference(V, D, H, L, E, agg, act, normalize):
    """SURVEY.md §8f-1: gradients w.r.t. node states and per-type weights vs float64 autograd of the
    reference op order (tf.GradientTape in the reference, graph_task_model.py:338-365)."""
    _need_gpu()
    from tf2_gnn_b200.layers import MessagePassingInput, RGCN
    rng = np.random.default_rng(V + H)
    adjs = random_graph(rng, V, L, E, hub=True, dups=True)
    p = RGCN.get_default_hyperparameters()
    p.update(hidden_dim=H, aggregation_function=agg, message_activation_function=act,
             normalize_by_num_incoming=normalize)
    h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    Ws = [mo.glorot_uniform(rng, (D, H)) for _ in range(L)]
    g = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    layer = make_layer("rgcn", p, D, L, {"edge_mlps": [[w] for w in Ws]})
    for v in layer.variables:
        v.requires_grad_()
    ht = torch.from_numpy(h).cuda().requires_grad_()
    out = layer(MessagePassingInput(ht, tuple(torch.from_numpy(a).cuda() for a in adjs)), training=True)
    out.backward(torch.from_numpy(g).cuda())
    # float64 reference
    h64 = torch.from_numpy(h).double().requires_grad_()
    W64 = [torch.from_numpy(w).double().requires_grad_() for w in Ws]
    ref = _torch_reference_layer(h64, [torch.from_numpy(a) for a in adjs], W64, normalize, agg, act)
    ref.backward(torch.from_numpy(g).double())
    assert_states_close(out.detach().cpu().numpy(), ref.detach().numpy())
    assert_states_close(ht.grad.cpu().numpy(), h64.grad.numpy(), tol=2e-5)
    for var, w64 in zip(layer.variables, W64):
        assert_states_close(var.grad.cpu().numpy(), w64.grad.numpy(), tol=2e-5)


def _torch_reference_ggnn(h, adjs, Ws, K, U, b, normalize, agg):
    """float64 autograd restatement of GGNN (ggnn.py:68-89): messages, aggregation, Keras GRUCell reset_after=True."""
    V, H = h.shape
    msgs, tgts = [], []
    for adj, W in zip(adjs, Ws):
        src, tgt = adj[:, 0].long(), adj[:, 1].long()
        m = h.index_select(0, src) @ W
        if normalize:
            c = torch.zeros(V, dtype=h.dtype).index_add_(0, tgt, torch.ones(len(tgt), dtype=h.dtype))
            m = (1.0 / (c.index_select(0, tgt) + 1e-7)).unsqueeze(-1) * m
        msgs.append(m)
        tgts.append(tgt)
    M, T = torch.cat(msgs), torch.cat(tgts)
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


@pytest.mark.parametrize("V,H,L,E,agg,normalize", [
    (300, 32, 3, 2500, "sum", True),
    (1000, 64, 2, 9000, "mean", False),
    (20000, 128, 5, 60000, "sum", True),
    (700, 36, 2, 4000, "sqrt_n", True),
])
def test_ggnn_backward_matches_autograd_reference(V, H, L, E, agg, normalize):
    """SURVEY.md §8f-1: GGNN gradients w.r.t. node states, message weights and the GRU parameters vs float64 autograd
    of the reference op order."""
    _need_gpu()
    from tf2_gnn_b200.layers import GGNN, MessagePassingInput
    rng = np.random.default_rng(V + H + L)
    adjs = random_graph(rng, V, L, E, hub=True, dups=True)
    p = GGNN.get_default_hyperparameters()
    p.update(hidden_dim=H, aggregation_function=agg, normalize_by_num_incoming=normalize)
    h = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    Ws = [mo.glorot_uniform(rng, (H, H)) for _ in range(L)]
    K, U = mo.glorot_uniform(rng, (H, 3 * H)), mo.glorot_uniform(rng, (H, 3 * H))
    b = rng.uniform(-0.2, 0.2, (2, 3 * H)).astype(np.float32)
    g = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    layer = make_layer("ggnn", p, H, L, {"edge_mlps": [[w] for w in Ws], "gru_kernel": K, "gru_recurrent_kernel": U,
                                         "gru_bias": b})
    for v in layer.variables:
        v.requires_grad_()
    ht = torch.from_numpy(h).cuda().requires_grad_()
    out = layer(MessagePassingInput(ht, tuple(torch.from_numpy(a).cuda() for a in adjs)))
    out.backward(torch.from_numpy(g).cuda())
    h64 = torch.from_numpy(h).double().requires_grad_()
    W64 = [torch.from_numpy(w).double().requires_grad_() for w in Ws]
    K64, U64, b64 = (torch.from_numpy(x).double().requires_grad_() for x in (K, U, b))
    ref = _torch_reference_ggnn(h64, [torch.from_numpy(a) for a in adjs], W64, K64, U64, b64, normalize, agg)
    ref.backward(torch.from_numpy(g).double())
    assert_states_close(out.detach().cpu().numpy(), ref.detach().numpy())
    assert_states_close(ht.grad.cpu().numpy(), h64.grad.numpy(), tol=2e-5)
    grads = {v.name: v.grad.cpu().numpy() for v in layer.variables}
    assert_states_close(grads[[n for n in grads if n.endswith("gru_cell/kernel:0")][0]], K64.grad.numpy(), tol=2e-5)
    assert_states_close(grads[[n for n in grads if n.endswith("gru_cell/recurrent_kernel:0")][0]], U64.grad.numpy(),
                        tol=2e-5)
    assert_states_close(grads[[n for n in grads if n.endswith("gru_cell/bias:0")][0]], b64.grad.numpy(), tol=2e-5)
    assert len(layer._edge_type_mlps) == L
    for l, mlp in enumerate(layer._edge_type_mlps):
        assert_states_close(mlp.layers[0].grad.cpu().numpy(), W64[l].grad.numpy(), tol=2e-5)


@pytest.mark.parametrize("V,D,H,L,E,agg,act,normalize", [
    (300, 32, 48, 3, 2500, "sum", "tanh", True),
    (2000, 64, 64, 2, 15000, "mean", "elu", False),
    (700, 128, 36, 4, 6000, "sqrt_n", "tanh", True),
])
def test_rgcn_backward_with_target_state_input(V, D, H, L, E, agg, act, normalize):
    """use_target_state_as_input=True (the [2D, H] kernels of test_RGCN.py:40-65): gradients incl. the target half."""
    _need_gpu()
    from tf2_gnn_b200.layers import MessagePassingInput, RGCN
    rng = np.random.default_rng(V + D + H)
    adjs = random_graph(rng, V, L, E, hub=True, dups=True, self_loops=True)
    p = RGCN.get_default_hyperparameters()
    p.update(hidden_dim=H, aggregation_function=agg, message_activation_function=act,
             normalize_by_num_incoming=normalize, use_target_state_as_input=True)
    h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    Ws = [mo.glorot_uniform(rng, (2 * D, H)) for _ in range(L)]
    g = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    layer = make_layer("rgcn", p, D, L, {"edge_mlps": [[w] for w in Ws]})
    for v in layer.variables:
        v.requires_grad_()
    ht = torch.from_numpy(h).cuda().requires_grad_()
    out = layer(MessagePassingInput(ht, tuple(torch.from_numpy(a).cuda() for a in adjs)))
    out.backward(torch.from_numpy(g).cuda())
    h64 = torch.from_numpy(h).double().requires_grad_()
    W64 = [torch.from_numpy(w).double().requires_grad_() for w in Ws]
    ref = _torch_reference_layer(h64, [torch.from_numpy(a) for a in adjs], W64, normalize, agg, act, use_target=True)
    ref.backward(torch.from_numpy(g).double())
    assert_states_close(out.detach().cpu().numpy(), ref.detach().numpy())
    assert_states_close(ht.grad.cpu().numpy(), h64.grad.numpy(), tol=2e-5)
    for var, w64 in zip(layer.variables, W64):
        assert tuple(var.grad.shape) == (2 * D, H)
        assert_states_close(var.grad.cpu().numpy(), w64.grad.numpy(), tol=2e-5)


def _forward_backward_twice(layer, h, adjs, g, weights):
    """Two independent forward + backward runs through the autograd hook; they must agree bit for bit.
    Returns [out, grad_h, *grad_weights] as numpy arrays."""
    from tf2_gnn_b200.layers import MessagePassingInput
    adj_dev = tuple(torch.from_numpy(a).cuda() for a in adjs)
    runs = []
    for _ in range(2):
        ht = torch.from_numpy(h).cuda().requires_grad_()
        out = layer(MessagePassingInput(ht, adj_dev), training=True)
        grads = torch.autograd.grad(out, [ht] + weights, torch.from_numpy(g).cuda())
        runs.append([out.detach().cpu().numpy()] + [x.cpu().numpy() for x in grads])
    for a, b in zip(*runs):
        assert np.array_equal(a, b)
    return runs[0]


@pytest.mark.parametrize("V,D,H,L,E,agg,act,normalize,opts", [
    (3000, 384, 64, 3, 15000, "sum", "tanh", True, {}),             # NV = 3 (D in 257..384), split-tile mode
    (3000, 384, 320, 3, 15000, "mean", "elu", False, {}),
    (9000, 448, 64, 3, 30000, "sqrt_n", "tanh", False, {}),         # NV = 4, 71 tiles: one CTA per tile
    (9000, 448, 320, 3, 30000, "sum", "gelu", True, {}),
    (20000, 512, 64, 3, 60000, "mean", "tanh", False, {}),          # D = 512: 2 stages, 7 gather slots per warp
    (20000, 512, 320, 3, 60000, "sum", "elu", False, {}),
    (3000, 64, 128, 7, 8000, "sum", "tanh", True, {}),              # several N passes: the ring at its 8-slot limit
    (3000, 64, 512, 7, 8000, "mean", "gelu", False, {}),
    (9000, 64, 512, 7, 20000, "sum", "tanh", False, {}),
    (2000, 32, 64, 14, 3000, "sum", "tanh", True, {}),              # one N pass, 14 types on the tensor cores
    (2000, 64, 16, 3, 8000, "sum", "tanh", False, {}),              # BN = 16, one pass
    (2000, 64, 80, 3, 8000, "mean", "tanh", True, {}),              # BN = 16, 5 passes
    (9000, 64, 112, 3, 30000, "sqrt_n", "elu", False, {}),          # BN = 16, 7 passes
    (8191, 64, 64, 2, 24000, "sum", "tanh", False, {}),             # around the 8192-row chunks of the dW reduction
    (8192, 64, 64, 2, 24000, "mean", "tanh", True, {}),
    (8193, 64, 64, 2, 24000, "mean", "tanh", False, dict(hub=True)),
    (16385, 64, 64, 2, 50000, "sum", "elu", False, {}),
    (3000, 128, 128, 4, 12000, "sum", "tanh", True, dict(empty_type=2)),
])
def test_rgcn_backward_shape_limits(V, D, H, L, E, agg, act, normalize, opts):
    """Fused-kernel instantiations and backward tilings at their limits: forward forced to fused_tc, backward through the
    autograd hook, both against the float64 reference; two runs give the same bits.  Only activations with a continuous
    derivative: with relu / leaky_relu / selu, a pre-activation within rounding of 0 takes the other derivative in fp32
    and moves a whole gradient row by |grad_out| |W| (0.06 of a 6.5 scale measured at D = 512, H = 320), so the kinked
    activations are checked by the exact-arithmetic tests of test_gpu_backward_scale.py instead."""
    _need_gpu()
    import reference64 as r64
    from tf2_gnn_b200.layers import RGCN
    rng = np.random.default_rng(V + D + H + L)
    adjs = random_graph(rng, V, L, E, **opts)
    p = RGCN.get_default_hyperparameters()
    p.update(hidden_dim=H, aggregation_function=agg, message_activation_function=act, normalize_by_num_incoming=normalize,
             b200_path="fused_tc")
    h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    Ws = [mo.glorot_uniform(rng, (D, H)) for _ in range(L)]
    g = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    layer = make_layer("rgcn", p, D, L, {"edge_mlps": [[w] for w in Ws]})
    weights = [v.value.requires_grad_() for v in layer.variables]
    out, grad_h, *grad_W = _forward_backward_twice(layer, h, adjs, g, weights)
    ref = r64.rgcn_layer(h, adjs, Ws, g, agg=agg, act=act, normalize=normalize)
    assert_states_close(out, ref["out"].numpy())
    assert_states_close(grad_h, ref["grad_h"].numpy(), tol=2e-5)
    for l in range(L):
        if opts.get("empty_type") == l:
            assert np.all(grad_W[l] == 0.0)
        else:
            assert_states_close(grad_W[l], ref["grad_W"][l].numpy(), tol=2e-5)


def test_rgcn_fused_refuses_eight_types_with_several_passes():
    """L = 8 with H > 64 needs 9 ring slots: fused_tc raises instead of computing something else, and auto (which then
    takes another path) still matches the float64 reference, gradients included."""
    _need_gpu()
    import reference64 as r64
    from tf2_gnn_b200.layers import MessagePassingInput, RGCN
    V, D, H, L = 3000, 64, 128, 8
    rng = np.random.default_rng(88)
    adjs = random_graph(rng, V, L, 6000)
    h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    Ws = [mo.glorot_uniform(rng, (D, H)) for _ in range(L)]
    g = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    p = RGCN.get_default_hyperparameters()
    p.update(hidden_dim=H, aggregation_function="sum", message_activation_function="tanh", normalize_by_num_incoming=False,
             b200_path="fused_tc")
    layer = make_layer("rgcn", p, D, L, {"edge_mlps": [[w] for w in Ws]})
    with pytest.raises(NotImplementedError):
        layer(MessagePassingInput(torch.from_numpy(h).cuda(), tuple(torch.from_numpy(a).cuda() for a in adjs)))
    layer = make_layer("rgcn", dict(p, b200_path="auto"), D, L, {"edge_mlps": [[w] for w in Ws]})
    weights = [v.value.requires_grad_() for v in layer.variables]
    out, grad_h, *grad_W = _forward_backward_twice(layer, h, adjs, g, weights)
    ref = r64.rgcn_layer(h, adjs, Ws, g, act="tanh")
    assert_states_close(out, ref["out"].numpy())
    assert_states_close(grad_h, ref["grad_h"].numpy(), tol=2e-5)
    for l in range(L):
        assert_states_close(grad_W[l], ref["grad_W"][l].numpy(), tol=2e-5)


@pytest.mark.parametrize("H", [160, 320])
def test_ggnn_backward_wide_gru_epilogue(H, monkeypatch):
    """GGNN with more than 4 GRU N tiles (fused-GRU forward) against the float64 reference; two runs give the same bits."""
    _need_gpu()
    import reference64 as r64
    from tf2_gnn_b200.layers import GGNN
    monkeypatch.setenv("TFGNN_B200_GGNN_FUSED_GRU", "1")
    V, L = 3000, 3
    rng = np.random.default_rng(H)
    adjs = random_graph(rng, V, L, 3 * V, hub=True, dups=True)
    p = GGNN.get_default_hyperparameters()
    p.update(hidden_dim=H, b200_path="fused_tc")
    h = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    Ws = [mo.glorot_uniform(rng, (H, H)) for _ in range(L)]
    K, U = mo.glorot_uniform(rng, (H, 3 * H)), mo.glorot_uniform(rng, (H, 3 * H))
    b = rng.uniform(-0.2, 0.2, (2, 3 * H)).astype(np.float32)
    g = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    layer = make_layer("ggnn", p, H, L, {"edge_mlps": [[w] for w in Ws], "gru_kernel": K, "gru_recurrent_kernel": U,
                                         "gru_bias": b})
    by_name = {v.name: v.value for v in layer.variables}
    gru = [[t for n, t in by_name.items() if n.endswith(s)][0]
           for s in ("gru_cell/kernel:0", "gru_cell/recurrent_kernel:0", "gru_cell/bias:0")]
    weights = [t.requires_grad_() for t in [m.layers[0].value for m in layer._edge_type_mlps] + gru]
    out, grad_h, *grads = _forward_backward_twice(layer, h, adjs, g, weights)
    ref = r64.ggnn_layer(h, adjs, Ws, K, U, b, g, agg=p["aggregation_function"], normalize=p["normalize_by_num_incoming"])
    assert_states_close(out, ref["out"].numpy())
    assert_states_close(grad_h, ref["grad_h"].numpy(), tol=2e-5)
    for l in range(L):
        assert_states_close(grads[l], ref["grad_W"][l].numpy(), tol=2e-5)
    for got, key in zip(grads[L:], ("grad_K", "grad_U", "grad_b")):
        assert_states_close(got, ref[key].numpy(), tol=2e-5)


# ------------------------------------------------------------------------------------------
# Node-level dense and error behaviour
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V,K,N", [(1, 1, 1), (130, 50, 17), (1000, 320, 320), (777, 96, 256)])
def test_dense_fwd(V, K, N):
    _need_gpu()
    from tf2_gnn_b200 import _ffi
    from tf2_gnn_b200.runtime import stream_ptr
    rng = np.random.default_rng(V)
    x = rng.uniform(-1, 1, (V, K)).astype(np.float32)
    w = rng.uniform(-0.3, 0.3, (K, N)).astype(np.float32)
    xt, wt = torch.from_numpy(x).cuda(), torch.from_numpy(w).cuda()
    out = torch.empty((V, N), dtype=torch.float32, device="cuda")
    _ffi.check(_ffi.lib().tfgnn_b200_dense_fwd(xt.data_ptr(), wt.data_ptr(), out.data_ptr(), V, K, N,
                                                _ffi.ACT["tanh"], 0, stream_ptr()))
    assert_states_close(out.cpu().numpy(), np.tanh(x.astype(np.float64) @ w.astype(np.float64)))


@pytest.mark.parametrize("V,K,N", [(128, 32, 64), (129, 64, 16), (1000, 320, 320), (300, 1024, 256),
                                   (5000, 960, 320), (500, 100, 48), (70000, 256, 1024)])
def test_dense_fwd_tensor_core_3xtf32(V, K, N):
    """wgmma 3xTF32 GEMM keeps fp32-level accuracy (plain TF32 would be ~1e-3)."""
    _need_gpu()
    from tf2_gnn_b200 import _ffi
    from tf2_gnn_b200.runtime import stream_ptr
    rng = np.random.default_rng(V + K)
    x = rng.uniform(-1, 1, (V, K)).astype(np.float32)
    w = rng.uniform(-0.3, 0.3, (K, N)).astype(np.float32)
    xt, wt = torch.from_numpy(x).cuda(), torch.from_numpy(w).cuda()
    out = torch.full((V, N), float("nan"), dtype=torch.float32, device="cuda")
    _ffi.check(_ffi.lib().tfgnn_b200_dense_fwd(xt.data_ptr(), wt.data_ptr(), out.data_ptr(), V, K, N,
                                                _ffi.ACT["relu"], _ffi.PATH["sorted_tc"], stream_ptr()))
    torch.cuda.synchronize()
    ref = np.maximum(x.astype(np.float64) @ w.astype(np.float64), 0.0)
    # measured: 4e-7 (K=32) .. 3.2e-6 (K=1024): accumulate-truncation bias of the tensor core, see gemm_tc.cu
    assert_states_close(out.cpu().numpy(), ref, tol=5e-6)


@pytest.mark.parametrize("N", [16, 32, 48, 64, 80, 96, 112, 128, 176, 384])
def test_dense_fwd_tensor_core_3xtf32_tiles_and_tails(N):
    """Every BN instantiation of the wgmma GEMM (N = 176: BN = 16, 11 column tiles), M tails around the 64-row consumer
    halves and 128-row tiles, M = 33921 (every CTA runs several tiles, so the stage ring wraps inside a tile), and K from
    one partial K block to 32 (K = 160: 5 K blocks over a 3- or 4-stage ring).  Integer inputs in [-8, 8] must come out
    exact; random inputs within 1e-5 of (|x||w| + |b|) element by element."""
    _need_gpu()
    from tf2_gnn_b200 import _ffi
    from tf2_gnn_b200.runtime import stream_ptr
    lib = _ffi.lib()
    rng = np.random.default_rng(N)
    for M in (1, 63, 64, 65, 128, 129, 33921):
        for K in (4, 36, 160, 1024):
            for integer in (True, False):
                if integer:
                    x, w, bias = (rng.integers(-8, 9, s).astype(np.float32) for s in ((M, K), (K, N), (N,)))
                else:
                    x = rng.uniform(-1, 1, (M, K)).astype(np.float32)
                    w = rng.uniform(-0.3, 0.3, (K, N)).astype(np.float32)
                    bias = rng.uniform(-0.5, 0.5, N).astype(np.float32)
                x64, w64 = x.astype(np.float64), w.astype(np.float64)
                ref = x64 @ w64
                bound = np.abs(x64) @ np.abs(w64)
                xt, wt, bt = (torch.from_numpy(a).cuda() for a in (x, w, bias))
                for with_bias in (False, True):
                    out = torch.full((M, N), float("nan"), dtype=torch.float32, device="cuda")
                    if with_bias:
                        _ffi.check(lib.tfgnn_b200_dense_bias_fwd(xt.data_ptr(), wt.data_ptr(), bt.data_ptr(), out.data_ptr(),
                                                                 M, K, N, 0, _ffi.PATH["sorted_tc"], stream_ptr()))
                    else:
                        _ffi.check(lib.tfgnn_b200_dense_fwd(xt.data_ptr(), wt.data_ptr(), out.data_ptr(), M, K, N, 0,
                                                            _ffi.PATH["sorted_tc"], stream_ptr()))
                    got = out.cpu().numpy().astype(np.float64)
                    want = ref + bias.astype(np.float64) if with_bias else ref
                    what = f"M={M} K={K} N={N} {'integer' if integer else 'random'} bias={with_bias}"
                    if integer:
                        assert np.array_equal(got, want), what
                    else:
                        bnd = bound + np.abs(bias.astype(np.float64)) if with_bias else bound
                        excess = np.abs(got - want) - 1e-5 * bnd
                        assert np.isfinite(got).all() and excess.max() <= 0.0, \
                            f"{what}: worst |err| / (|x||w|) = {(np.abs(got - want) / bnd).max():.3e}"


def test_unknown_names_raise_like_the_reference():
    from tf2_gnn_b200.layers import get_message_passing_class
    from tf2_gnn_b200.utils import get_activation_function, get_aggregation_function
    with pytest.raises(ValueError):
        get_message_passing_class("gcn2")
    with pytest.raises(ValueError):
        get_activation_function("linear")
    with pytest.raises(ValueError):
        get_aggregation_function("median")
    assert get_message_passing_class("RGCN").__name__ == "RGCN"


def test_launch_counter_moves():
    _need_gpu()
    from tf2_gnn_b200 import _ffi
    before = _ffi.launch_count()
    rng = np.random.default_rng(0)
    p = mo.default_hyperparameters("rgcn")
    p["hidden_dim"] = 32
    run_case("rgcn", p, 100, 32, 2, random_graph(rng, 100, 2, 500))
    assert _ffi.launch_count() > before


@pytest.mark.parametrize("V,D,H,L,E,split", [(9000, 64, 64, 3, 40000, "1"), (30000, 128, 256, 4, 150000, "0"),
                                             (3000, 320, 320, 3, 20000, "1")])
def test_rgcn_fwd_allgather_replica_stores(monkeypatch, V, D, H, L, E, split):
    """tfgnn_b200_rgcn_fwd_allgather on ONE GPU: the replicas are three local tables, the batch is a target-range shard.
    Every replica must receive exactly the rows the plain sharded layer call produces, at rows [lo, hi), and nothing else
    (multi-GPU: the same stores go to NVLink-mapped peer tables; tools / bench.py --gpus N exercise that)."""
    _need_gpu()
    from tf2_gnn_b200.layers import MessagePassingInput
    from tf2_gnn_b200.runtime import PreparedBatch
    monkeypatch.setenv("TFGNN_B200_FUSED_SPLIT", split)
    rng = np.random.default_rng(V)
    adjs = random_graph(rng, V, L, E, hub=True)
    p = mo.default_hyperparameters("rgcn")
    p.update(hidden_dim=H)
    w = mo.make_weights("rgcn", p, D, L, rng)
    layer = make_layer("rgcn", p, D, L, w)
    h = torch.from_numpy(rng.uniform(-1, 1, (V, D)).astype(np.float32)).cuda()
    adj_t = tuple(torch.from_numpy(a).cuda() for a in adjs)
    lo, hi = (V // 3) // 128 * 128, V - 77
    shard = PreparedBatch(adj_t, V, target_range=(lo, hi))
    ref = layer(MessagePassingInput(h, adj_t), prepared=shard)
    tables = [torch.full((V, H), -7.0, device="cuda") for _ in range(3)]
    layer.call_allgather(h, shard, [t.data_ptr() for t in tables], own_rank=1)
    torch.cuda.synchronize()
    for t in tables:
        assert torch.equal(t[lo:hi], ref)
        assert bool((t[:lo] == -7.0).all()) and bool((t[hi:] == -7.0).all())
    # a layer with a target-state input cannot take the fused kernel: the entry refuses instead of computing something else
    p2 = dict(p, use_target_state_as_input=True)
    layer2 = make_layer("gnn_edge_mlp", dict(mo.default_hyperparameters("gnn_edge_mlp"), hidden_dim=H), D, L,
                        mo.make_weights("gnn_edge_mlp", dict(mo.default_hyperparameters("gnn_edge_mlp"), hidden_dim=H), D, L, rng))
    with pytest.raises(NotImplementedError):
        layer2.call_allgather(h, shard, [t.data_ptr() for t in tables], own_rank=0)
    del p2
