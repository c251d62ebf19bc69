"""Training of RGAT layers through tfgnn_b200_rgat_bwd (no per-edge tensors, no float atomics): gradients against the
float64 reference (reference64_rgat), bitwise reproducibility, target-range shards, a PPI_RGAT-shaped stack step and one step
at bench.py's cfg3 size.

Each case asserts in float64 that every edge's score argument x_e lies at least 1e-5 * max |x_e| from 0, so that no kink of
leaky_relu decides the result."""
import time

import numpy as np
import pytest

torch = pytest.importorskip("torch")

import reference64_rgat as r64  # noqa: E402
from oracle import message_passing_oracle as mo  # noqa: E402
from test_gpu_edge_mlp_backward import trimmed_pool  # noqa: E402,F401  (fixture)
from test_gpu_parity import _need_gpu, assert_states_close, make_layer  # noqa: E402
from test_gpu_shard_backward import _check_shards  # noqa: E402
from test_gpu_transform_aggregate_backward import _uses  # noqa: E402

pytestmark = pytest.mark.gpu

TOL = 3e-5
HUB_EDGES = 5300   # > 2048 (the hub threshold): 6 chunks of 1024 edges
# (K, d, D, L, activation, hub): K in {1, 3, 4, 8}, d in {4, 32, 80}, D != H, L = 1..7 with an empty type, every lane count
# (NV = 1..4 float4 groups per lane), heads straddling lane groups (d = 80) and heads wider than a warp's row (d = 256)
CASES = [
    (1, 4, 8, 1, None, False),
    (3, 32, 20, 3, "tanh", True),
    (4, 80, 64, 2, "gelu", True),
    (8, 4, 12, 7, "relu", False),
    (4, 32, 128, 4, "relu", True),
    (1, 32, 16, 5, "tanh", False),
    (8, 32, 36, 2, None, True),
    (3, 80, 8, 3, "relu", False),
    (4, 4, 4, 6, "gelu", False),
    (8, 4, 24, 2, "tanh", True),
    (1, 256, 8, 2, "tanh", False),
    (2, 256, 12, 3, "gelu", True),
]


def graph(rng, V, L, E, hub):
    """L edge lists with duplicates and self-loops; the last of several types is empty; hub=True sends HUB_EDGES more edges
    into target V // 3."""
    adjs = []
    for l in range(L):
        if L > 1 and l == L - 1:
            adjs.append(np.zeros((0, 2), np.int32))
            continue
        a = rng.integers(0, V, size=(E, 2))
        a[1] = a[0]
        a[3] = a[0]
        a[5:25, 1] = a[5:25, 0]
        adjs.append(a)
    if hub:
        n = max(L - 1, 1)
        for l, part in enumerate(np.array_split(rng.integers(0, V, size=HUB_EDGES), n)):
            adjs[l] = np.concatenate([adjs[l], np.stack([part, np.full_like(part, V // 3)], 1)])
    return [a[rng.permutation(len(a))].astype(np.int32) for a in adjs]


def _inputs(case, seed, V=600, E=3000):
    """Inputs of the first seed in seed, seed + 1000, .. whose scores keep the margin from leaky_relu's kink."""
    K, d, D, L, act, hub = case
    H = K * d
    E = min(E, 20000 // (K * max(L - 1, 1)))   # at most ~20k (edge, head) scores, so that a margin is likely
    for s in range(seed, seed + 20000, 1000):
        rng = np.random.default_rng(s)
        adjs = graph(rng, V, L, E, hub)
        p = mo.default_hyperparameters("rgat")
        p.update(hidden_dim=H, num_heads=K, message_activation_function=act)
        w = mo.make_weights("rgat", p, D, L, rng)
        h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
        g = rng.uniform(-1, 1, (V, H)).astype(np.float32)
        lo, hi = _score_abs_range(adjs, h, w)
        if lo >= 1e-5 * hi:
            return p, adjs, h, w, g
    raise AssertionError("no seed keeps the scores away from leaky_relu's kink")


def _reference(adjs, h, w, g, act, device="cpu"):
    t = lambda x: torch.from_numpy(np.asarray(x)).to(device)
    out, grad_h, dW, da, margin = r64.forward_backward(t(h), [t(a) for a in adjs], [t(x) for x in w["edge_kernels"]],
                                                       [t(x) for x in w["edge_attention"]], t(g), act)
    assert margin >= 1e-5 * _score_abs_range(adjs, h, w)[1], margin
    return out.cpu().numpy(), grad_h.cpu().numpy(), [x.cpu().numpy() for x in dW + da]


def _score_abs_range(adjs, h, w):
    """(min, max) over all edges and heads of |x_e| in float64."""
    h = h.astype(np.float64)
    lo, hi = np.inf, 0.0
    for a, W, A in zip(adjs, w["edge_kernels"], w["edge_attention"]):
        if not len(a):
            continue
        K = A.shape[0]
        P = (h @ W.astype(np.float64)).reshape(len(h), K, -1)
        d = P.shape[2]
        x = np.abs((P * A[:, :d]).sum(-1)[a[:, 0]] + (P * A[:, d:]).sum(-1)[a[:, 1]])
        lo, hi = min(lo, x.min()), max(hi, x.max())
    return lo, hi


def _layer(p, D, L, w):
    layer = make_layer("rgat", p, D, L, w)
    for v in layer.variables:
        v.requires_grad_()
    params = list(layer._edge_type_to_message_computation_layer) + list(layer._edge_type_to_attention_parameters)
    return layer, params


def _run(layer, params, h, adjs, g, prepared=None, twice=False):
    from tf2_gnn_b200.layers import MessagePassingInput
    ht = torch.from_numpy(h).cuda().requires_grad_()
    for q in params:
        q.value.grad = None
    out = layer(MessagePassingInput(ht, tuple(torch.from_numpy(a).cuda() for a in adjs)), prepared=prepared)
    assert _uses(out, "_RgatLayerFunctionBackward")
    gt = torch.from_numpy(g).cuda()
    out.backward(gt, retain_graph=twice)
    torch.cuda.synchronize()
    got = out.detach().cpu().numpy(), ht.grad.cpu().numpy(), [q.value.grad.cpu().numpy() for q in params]
    if not twice:
        return got
    ht.grad = None
    for q in params:
        q.value.grad = None
    out.backward(gt)   # a second backward of the same forward
    torch.cuda.synchronize()
    return got, (ht.grad.cpu().numpy(), [q.value.grad.cpu().numpy() for q in params])


@pytest.mark.parametrize("case", CASES, ids=[f"K{c[0]}-d{c[1]}-D{c[2]}-L{c[3]}-{c[4]}{'-hub' if c[5] else ''}"
                                             for c in CASES])
def test_rgat_backward_matches_float64(case):
    _need_gpu()
    p, adjs, h, w, g = _inputs(case, seed=CASES.index(case))
    ref_out, ref_h, ref_w = _reference(adjs, h, w, g, case[4])
    layer, params = _layer(p, h.shape[1], len(adjs), w)
    got, again = _run(layer, params, h, adjs, g, twice=True)
    assert_states_close(got[0], ref_out, tol=TOL)
    assert_states_close(got[1], ref_h, tol=TOL)
    assert len(got[2]) == len(ref_w)
    for a, b in zip(got[2], ref_w):
        assert_states_close(a, b, tol=TOL)
    assert np.array_equal(got[1], again[0]) and all(np.array_equal(a, b) for a, b in zip(got[2], again[1]))


@pytest.mark.parametrize("hub", [False, True])
def test_training_forward_equals_inference(hub):
    """The training forward is tfgnn_b200_rgat_fwd: bitwise equal to inference, hub rows included."""
    _need_gpu()
    from tf2_gnn_b200.layers import MessagePassingInput
    case = (4, 32, 64, 3, "tanh", hub)
    p, adjs, h, w, g = _inputs(case, seed=21)
    layer, params = _layer(p, h.shape[1], len(adjs), w)
    train = _run(layer, params, h, adjs, g)[0]
    with torch.no_grad():
        inp = MessagePassingInput(torch.from_numpy(h).cuda(), tuple(torch.from_numpy(a).cuda() for a in adjs))
        infer = layer(inp).cpu().numpy()
    assert np.array_equal(train, infer)


@pytest.mark.parametrize("case", [(3, 8, 20, 3, "tanh", False), (4, 32, 64, 3, "relu", True)])
def test_fused_matches_literal_path(case):
    """The fused backward and the literal rgat_forward (layers/differentiable.py) agree with each other and with float64."""
    _need_gpu()
    from tf2_gnn_b200.layers import MessagePassingInput
    from tf2_gnn_b200.layers.differentiable import rgat_forward
    from tf2_gnn_b200.runtime import PreparedBatch
    p, adjs, h, w, g = _inputs(case, seed=31, E=1500)
    _, ref_h, ref_w = _reference(adjs, h, w, g, case[4])
    layer, params = _layer(p, h.shape[1], len(adjs), w)
    fused = _run(layer, params, h, adjs, g)
    ht = torch.from_numpy(h).cuda().requires_grad_()
    for q in params:
        q.value.grad = None
    adj = tuple(torch.from_numpy(a).cuda() for a in adjs)
    out = rgat_forward(layer, ht, PreparedBatch(adj, h.shape[0]))
    assert not _uses(out, "_RgatLayerFunctionBackward")
    out.backward(torch.from_numpy(g).cuda())
    literal = ht.grad.cpu().numpy(), [q.value.grad.cpu().numpy() for q in params]
    assert_states_close(fused[1], literal[0].astype(np.float64), tol=TOL)
    assert_states_close(literal[0], ref_h, tol=TOL)
    for a, b, r in zip(fused[2], literal[1], ref_w):
        assert_states_close(a, b.astype(np.float64), tol=TOL)
        assert_states_close(b, r, tol=TOL)


@pytest.mark.parametrize("route", ["inference", "fused", "literal"])
def test_every_route_rejects_a_batch_with_other_edge_types(route):
    """The layer checks its shapes before it picks a path: inference, the fused backward and the literal path (D not a
    multiple of 4) raise the same ValueError."""
    _need_gpu()
    from tf2_gnn_b200.layers import MessagePassingInput
    p, adjs, h, w, _ = _inputs((4, 8, 18 if route == "literal" else 32, 3, "tanh", False), seed=51)
    layer, _ = _layer(p, h.shape[1], len(adjs), w)
    ht = torch.from_numpy(h).cuda().requires_grad_(route != "inference")
    with pytest.raises(ValueError, match="number of adjacency lists"):
        layer(MessagePassingInput(ht, tuple(torch.from_numpy(a).cuda() for a in adjs[:-1])))


@pytest.mark.parametrize("case", [(4, 32, 64, 3, "relu", True), (3, 80, 16, 2, None, True), (8, 4, 12, 4, "tanh", False)])
def test_rgat_shard_backward_sums_to_full(case):
    """Worlds of 2 and 3 and a world with an empty middle shard (test_gpu_shard_backward._check_shards).  Each shard runs its
    own forward, whose hub rows are combined in chunk order, so the backward's bits do not depend on the run."""
    _need_gpu()
    p, adjs, h, w, g = _inputs(case, seed=41)
    layer, params = _layer(p, h.shape[1], len(adjs), w)
    _, ref_h, ref_w = _reference(adjs, h, w, g, case[4])
    _check_shards(layer, params, h, adjs, g, (ref_h, ref_w))


def test_ppi_rgat_shaped_stack_step():
    """PPI_RGAT.json's layer shape (H = 320, 4 heads, tanh) in a stack of 3 layers: one training step through the fused
    backward matches float64 layer by layer."""
    _need_gpu()
    from tf2_gnn_b200.layers import MessagePassingInput
    rng = np.random.default_rng(5)
    V, D, H, K, L, n_layers = 800, 64, 320, 4, 3, 3
    adjs = graph(rng, V, L + 1, 4000, True)[:L]
    p = mo.default_hyperparameters("rgat")
    p.update(hidden_dim=H, num_heads=K, message_activation_function="tanh")
    ws = [mo.make_weights("rgat", p, D if i == 0 else H, L, rng) for i in range(n_layers)]
    layers = [_layer(p, D if i == 0 else H, L, w) for i, w in enumerate(ws)]
    h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    g = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    adj = tuple(torch.from_numpy(a).cuda() for a in adjs)
    ht = torch.from_numpy(h).cuda().requires_grad_()
    x, states = ht, [h.astype(np.float64)]
    for layer, _ in layers:
        x = layer(MessagePassingInput(x, adj))
        assert _uses(x, "_RgatLayerFunctionBackward")
        states.append(x.detach().cpu().numpy().astype(np.float64))
    x.backward(torch.from_numpy(g).cuda())
    # float64: forward layer by layer from the fp32 states, backward from the top
    t = lambda a: torch.from_numpy(np.asarray(a, np.float64))
    dout = t(g)
    for i in reversed(range(n_layers)):
        w = ws[i]
        out, gh, dW, da, _ = r64.forward_backward(t(states[i]), [t(a) for a in adjs], [t(m) for m in w["edge_kernels"]],
                                                  [t(m) for m in w["edge_attention"]], dout, "tanh")
        assert_states_close(states[i + 1], out.numpy(), tol=TOL)
        params = layers[i][1]
        for q, r in zip(params, dW + da):
            assert_states_close(q.value.grad.cpu().numpy(), r.numpy(), tol=1e-4)
        dout = gh
    assert_states_close(ht.grad.cpu().numpy(), dout.numpy(), tol=1e-4)


def test_cfg3_training_step_without_per_edge_tensors(trimmed_pool, record_property, capsys):
    """bench.py's cfg3 graph (2M nodes, power-law, 3 x 20M edges, D = H = 128, 4 heads): one forward and backward step
    through the fused path raises the device memory in use by less than one [M, H] fp32 tensor, and grad_W, grad_attention
    and sampled rows of grad_h match the float64 reference.

    Among 240M (edge, head) scores of random sign, hundreds would lie within fp32 rounding of leaky_relu's kink, and each
    one that fp32 and float64 put on different sides moves its rows by ~1e-3.  So states and projections are positive and
    the attention parameters of types 0 and 2 positive, of type 1 negative: every score lies far from 0 on a known side
    (both branches of leaky_relu are taken), which the float64 reference asserts."""
    import resource

    import bench
    from tf2_gnn_b200.layers import MessagePassingInput
    from tf2_gnn_b200.runtime import PreparedBatch
    t0 = time.time()
    wl = bench.WORKLOADS["cfg3"]
    h_np, adjs, _ = bench.make_inputs(wl, seed=0)
    V, H, L = wl["V"], wl["H"], len(adjs)
    M = sum(a.shape[0] for a in adjs)
    p = mo.default_hyperparameters("rgat")
    p.update(hidden_dim=H, **wl["params"])
    D = h_np.shape[1]
    rng = np.random.default_rng(7)
    K = int(p["num_heads"])
    sign = [1.0, -1.0, 1.0]
    w = {"edge_kernels": [rng.uniform(0.01, 0.1, (D, H)).astype(np.float32) for _ in range(L)],
         "edge_attention": [(sign[l % 3] * rng.uniform(0.001, 0.01, (K, 2 * H // K))).astype(np.float32) for l in range(L)]}
    layer, params = _layer(p, D, L, w)
    h = (torch.from_numpy(np.abs(h_np)).cuda() * 0.9 + 0.1).requires_grad_()
    del h_np
    adj = tuple(torch.from_numpy(a).cuda() for a in adjs)
    del adjs
    gen = torch.Generator(device="cuda")
    gen.manual_seed(3)
    g = torch.rand((V, H), generator=gen, device="cuda") * 2 - 1
    prepared = PreparedBatch(adj, V)
    prepared.transposed()
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    out = layer(MessagePassingInput(h, adj), prepared=prepared)
    assert _uses(out, "_RgatLayerFunctionBackward")
    out.backward(g)
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    rise = (free0 - free1) / 1e9
    grad_h, grad_w = h.grad.detach(), [q.value.grad.detach() for q in params]
    del out, prepared
    torch.cuda.empty_cache()
    rows = torch.randperm(V, generator=gen, device="cuda")[:4096]
    _, ref_h, dW, da, margin = r64.forward_backward(h.detach(), adj, [q.value.detach() for q in params[:L]],
                                                    [q.value.detach() for q in params[L:]], g,
                                                    p["message_activation_function"], chunk=1 << 22, grad_h_rows=rows)
    wall = time.time() - t0
    rss = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1e6
    record_property("device_memory_rise_GB", round(rise, 2))
    with capsys.disabled():
        print(f"\n[rgat cfg3 step] device memory rose by {rise:.1f} GB; one [M, H] fp32 tensor is {4 * M * H / 1e9:.1f} GB; "
              f"min |x_e| {margin:.3g}; test wall time {wall:.0f} s, host max RSS {rss:.1f} GB")
    assert margin > 1e-2
    assert rise * 1e9 < 4.0 * M * H
    assert_states_close(grad_h[rows].cpu().numpy(), ref_h.cpu().numpy(), tol=TOL)
    for a, b in zip(grad_w, dW + da):
        assert_states_close(a.cpu().numpy(), b.cpu().numpy(), tol=TOL)
