"""Inputs of the element-wise bound tests: the case tables and graph builders shared by test_gpu_elementwise.py (the
kernels against the bounds) and test_bounds64_cpu.py (float32 evaluations of the same cases against the same bounds).
numpy, torch on the CPU and the float64 references only; nothing here needs a GPU."""
from __future__ import annotations

import numpy as np

import bounds64 as b64
from oracle import message_passing_oracle as mo

GRID = 64    # dyadic(): multiples of 1/GRID in [-1, 1]


# ---- graph and input builders --------------------------------------------------------------------------------------
def random_graph(rng, V, L, edges_per_type, empty_type=None, hub=False, dups=False):
    """L edge lists of uniform random edges; hub: half of each type's edges go to node V // 3; dups: edges 1 and 3
    repeat edge 0; empty_type: that type has no edges."""
    adjs = []
    for l in range(L):
        if l == empty_type:
            adjs.append(np.zeros((0, 2), np.int32))
            continue
        E = int(edges_per_type)
        a = rng.integers(0, V, size=(E, 2)).astype(np.int32)
        if hub and E:
            a[: E // 2, 1] = V // 3
        if dups and E >= 4:
            a[1] = a[0]
            a[3] = a[0]
        adjs.append(a)
    return adjs


def source_hub_graph(seed, V, E, L=3):
    """Out-degrees ~ Zipf(2.1) (the same weights for every type, so hubs add up over types), uniform targets: the
    source-keyed CSR of the dh reduction holds segments of thousands of edges."""
    rng = np.random.default_rng(seed)
    deg = np.minimum(rng.zipf(2.1, size=V), 100_000).astype(np.float64)
    p = deg / deg.sum()
    return [np.stack([rng.choice(V, size=E, p=p).astype(np.int32), rng.integers(0, V, size=E, dtype=np.int32)], axis=1)
            for _ in range(L)]


def dyadic(rng, shape):
    return (rng.integers(-GRID, GRID + 1, size=shape) / GRID).astype(np.float32)


def in_degree(V, adjs):
    return sum(np.bincount(np.asarray(a)[:, 1], minlength=V) for a in adjs)


def out_degree(V, adjs):
    return sum(np.bincount(np.asarray(a)[:, 0], minlength=V) for a in adjs)


# ---- RGCN forward --------------------------------------------------------------------------------------------------
# (name, path, V, D, H, L, aggregation, activation, environment).  Each fused_tc case names the kernel the launch rule of
# csrc/fused_rgcn.cu picks for it:
#   tiles      fused_rgcn_kernel, one CTA per 128-row tile, one N pass (H <= 64)
#   multipass  fused_rgcn_kernel, one CTA per 128-row tile, several N passes over the ring (H > 256)
#   rows       fused_rgcn_rows_kernel, 128 x H tiles in one N pass, each split by columns over a CTA pair that gathers
#              64 rows apiece (64 < H <= 256)
#   split      split-tile mode (fewer than SMs / 2 tiles): two CTAs share each 128-row tile
# TFGNN_B200_FUSED_SPLIT=0 keeps a small batch off split-tile mode; fused_rows_default is large enough for the default
# rule to choose row tiling (its 321-row shard, three tiles, takes split-tile mode).  The CTA-pair switch of earlier
# builds, TFGNN_B200_FUSED_PAIR, is no longer read by the kernel and has no case here.  V = 128k + 1 / 63 / 65 leaves 1,
# 63 or 65 rows in the last 128-row tile (1 in the last 64-row tile for 2561, 5185 and 10305).  Every graph: no
# normalisation, a target hub, duplicate edges, the last type empty.
NO_SPLIT = {"TFGNN_B200_FUSED_SPLIT": "0"}
SPLIT = {"TFGNN_B200_FUSED_SPLIT": "1"}
RGCN_CASES = [
    ("fused_tiles_h64", "fused_tc", 3903, 96, 64, 3, "sum", "elu", NO_SPLIT),
    ("fused_multipass_h320", "fused_tc", 2561, 128, 320, 3, "sum", "tanh", NO_SPLIT),
    ("fused_multipass_h512", "fused_tc", 5185, 128, 512, 2, "sum", "relu", NO_SPLIT),
    ("fused_rows_h128", "fused_tc", 2561, 128, 128, 4, "mean", "selu", NO_SPLIT),
    ("fused_rows_h256", "fused_tc", 3903, 64, 256, 3, "sqrt_n", "gelu", NO_SPLIT),
    ("fused_rows_default", "fused_tc", 10305, 64, 192, 3, "sum", "tanh", {}),
    ("fused_split_h128", "fused_tc", 2561, 128, 128, 4, "mean", "selu", SPLIT),
    ("fused_split_h320", "fused_tc", 3903, 64, 320, 3, "sum", "tanh", SPLIT),
    ("sorted", "sorted", 2561, 96, 48, 3, "sum", "leaky_relu", {}),
    ("atomic", "atomic", 3903, 64, 64, 3, "sum", "tanh", {}),
    ("pipeline", "auto", 5185, 36, 64, 3, "mean", "tanh", {"TFGNN_B200_PIPE_CHUNK_ROWS": "128"}),   # D % 32 != 0
]


def rgcn_case(V, D, H, L, agg, act, seed):
    """(params, weights, h, adjs) of an unnormalised RGCN layer on a hub graph with duplicates and an empty type."""
    rng = np.random.default_rng(seed)
    adjs = random_graph(rng, V, L, 4 * V, empty_type=L - 1, hub=True, dups=True)
    p = mo.default_hyperparameters("rgcn")
    p.update(hidden_dim=H, aggregation_function=agg, message_activation_function=act, normalize_by_num_incoming=False)
    w = mo.make_weights("rgcn", p, D, L, rng)
    h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    return p, w, h, adjs


def shard_range(V):
    """A target range around the hub (V // 3) whose ends are not tile multiples."""
    return V // 3 - 70, V // 3 + 251


# ---- LayerNorm-fused entry -----------------------------------------------------------------------------------------
LAYERNORM_CASES = [(3903, "relu"), (2561, "tanh")]


def layernorm_case(V, act, H=64, eps=1e-3):
    p, w, h, adjs = rgcn_case(V, 64, H, 3, "sum", act, seed=V)
    rng = np.random.default_rng(V + 1)
    return p, w, h, adjs, (rng.uniform(0.5, 1.5, H).astype(np.float32), rng.uniform(-0.2, 0.2, H).astype(np.float32), eps)


def layernorm_reference(p, w, h, adjs, ln, dtype=np.float64):
    """(LayerNorm of the layer output evaluated in `dtype`, the float64 element bound).

    With y_j = gamma_j x_hat_j + beta_j, x_hat = (x - mu) / sigma, an input error dx moves y_j by
    gamma_j / sigma (dx_j - d mu - x_hat_j d sigma), and |d mu|, |d sigma| <= max_j |dx_j| (mean |x_hat| <= 1).  So the
    bound of y_j is |gamma_j| / sigma * (2 + |x_hat_j|) * (the row's largest input bound), plus |gamma_j x_hat_j| +
    |beta_j| for the rounding of the normalisation itself.  A row without edges is the constant 0: y = beta exactly."""
    gamma, beta, eps = ln
    x64 = mo.message_passing_forward("rgcn", p, w, h, adjs, dtype=np.float64)
    x = mo.message_passing_forward("rgcn", p, w, h, adjs, dtype=dtype)
    ref = mo.layer_norm(x, gamma.astype(dtype), beta.astype(dtype), eps)
    sigma = np.sqrt(x64.var(axis=1) + eps)[:, None]
    x_hat = np.abs(x64 - x64.mean(axis=1, keepdims=True)) / sigma
    pre = b64.forward_bound("rgcn", p, w, h, adjs).max(axis=1)[:, None]
    g, b = np.abs(gamma.astype(np.float64)), np.abs(beta.astype(np.float64))
    bound = np.where(pre > 0, g / sigma * (2.0 + x_hat) * pre + g * x_hat + b, 0.0)
    return ref, bound


# ---- edge-MLP family and RGAT --------------------------------------------------------------------------------------
def family_case(kind, extra, seed=7, V=700, D=64, H=64, L=3):
    rng = np.random.default_rng(seed)
    adjs = random_graph(rng, V, L, 5 * V, empty_type=L - 1, hub=True, dups=True)
    p = mo.default_hyperparameters(kind)
    p.update(hidden_dim=H, normalize_by_num_incoming=False, message_activation_function="tanh")
    p.update(extra)
    w = mo.make_weights(kind, p, D, L, rng)
    h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    return p, w, h, adjs


ACT_OF_AGG = {"sum": "tanh", "sqrt_n": "gelu", "max": "relu"}
FAMILY_CASES = (
    [(f"{kind}_h{n}_{agg}{'_tgt' if tgt else ''}", kind,
      dict(num_edge_MLP_hidden_layers=n, aggregation_function=agg, use_target_state_as_input=tgt,
           message_activation_function=ACT_OF_AGG[agg]))
     for kind in ("rgin", "gnn_edge_mlp") for n in (0, 1) for agg in ("sum", "sqrt_n", "max") for tgt in (False, True)]
    + [("literal_h2_sum", "gnn_edge_mlp", dict(num_edge_MLP_hidden_layers=2)),
       ("literal_h2_max_before", "gnn_edge_mlp", dict(num_edge_MLP_hidden_layers=2, aggregation_function="max",
                                                      message_activation_before_aggregation=True,
                                                      use_target_state_as_input=False)),
       ("film", "gnn_film", dict(use_target_state_as_input=True)),
       ("film_mlp", "gnn_film", dict(film_parameter_MLP_hidden_layers=[32], aggregation_function="sqrt_n",
                                     message_activation_function="gelu")),
       ("rgat_k4", "rgat", dict(num_heads=4)),
       ("rgat_k8_h256", "rgat", dict(num_heads=8, hidden_dim=256, message_activation_function="elu"))])


# ---- graph reductions ----------------------------------------------------------------------------------------------
SEG_ROWS, PART_ROWS = 64, 256     # the fixed row chunks of segment_sum_rows and of readout_partial (csrc/graph_ops.cu)


def reduction_layout(seed=3):
    """graph_ptr of one batch: empty graphs first, in the middle and last, one-node graphs, a 100 000-node graph, and
    short graphs that straddle the 64-row and the 256-row chunk borders."""
    rng = np.random.default_rng(seed)
    small = lambda n: list(rng.choice([0, 1, 1, 2, 37, 63, 65, 130, 200], size=n))   # noqa: E731
    sizes = [0, 0, 1] + small(30) + [0, 1, 100_000, 1, 0] + small(30) + [1, 0]
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)


def straddles(ptr, chunk):
    """Graphs shorter than a chunk that cross a chunk border."""
    lo, hi = ptr[:-1].astype(np.int64), ptr[1:].astype(np.int64)
    return np.flatnonzero((hi - lo < chunk) & (hi - lo > 0) & (lo // chunk != (hi - 1) // chunk))


def reduction_inputs(C=64, K=4, seed=3):
    ptr = reduction_layout(seed)
    rng = np.random.default_rng(seed + 1)
    x = rng.uniform(-1, 1, (int(ptr[-1]), C)).astype(np.float32)
    scores = rng.uniform(-3, 3, (int(ptr[-1]), K)).astype(np.float32)
    return ptr, x, scores


# ---- backward ------------------------------------------------------------------------------------------------------
DENSE_BWD_CASES = [(9000, 64, 96, True), (1000, 33, 7, False), (4097, 320, 128, True)]
RGCN_BWD_CASES = [(20000, 128, 128, "sum", False), (9001, 64, 320, "mean", True)]
EDGE_MLP_BWD_CASES = [("tanh", "sum", True), ("gelu", "sqrt_n", False)]


def dense_bwd_inputs(V, K, N, bias):
    """(x, W, bias or None, grad_out)."""
    rng = np.random.default_rng(V + N)
    x = rng.uniform(-1, 1, (V, K)).astype(np.float32)
    W = mo.glorot_uniform(rng, (K, N))
    b = rng.uniform(-0.3, 0.3, N).astype(np.float32) if bias else None
    return x, W, b, rng.uniform(-1, 1, (V, N)).astype(np.float32)


def rgcn_bwd_inputs(V, D, H, L=3):
    """(h, adjs, [W_l], grad_out) on a graph with Zipf source hubs."""
    adjs = source_hub_graph(V, V=V, E=3 * V, L=L)
    rng = np.random.default_rng(V + H)
    h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    Ws = [mo.glorot_uniform(rng, (D, H)) for _ in range(L)]
    return h, adjs, Ws, np.random.default_rng(V).uniform(-1, 1, (V, H)).astype(np.float32)


def edge_mlp_bwd_inputs(use_target, V=6000, D=32, H=64, L=3):
    """(h, adjs, [U_l], [W2_l], grad_out): h and U on the 1/64 grid, so every hidden pre-activation is exact in fp32 and
    in 3xTF32 (|h U| partial sums are multiples of 2^-12 below 2^12) and a kernel's relu mask is the float64 one."""
    adjs = source_hub_graph(V + 1, V=V, E=3 * V, L=L)
    rng = np.random.default_rng(V + D)
    h = dyadic(rng, (V, D))
    Us = [dyadic(rng, ((2 if use_target else 1) * D, H)) for _ in range(L)]
    assert max(u.shape[0] for u in Us) * GRID * GRID < 2 ** 24
    W2s = [mo.glorot_uniform(rng, (H, H)) for _ in range(L)]
    return h, adjs, Us, W2s, np.random.default_rng(V).uniform(-1, 1, (V, H)).astype(np.float32)
