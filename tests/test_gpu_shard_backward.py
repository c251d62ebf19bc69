"""Backward through target-range shards (DESIGN.md §6): each shard's tfgnn_b200_rgcn_bwd / tfgnn_b200_ggnn_bwd over its
TFGNN_PREPARE_TRANSPOSE_OWNED batch writes its contribution to the full grad_h table and to the weight gradients; the
contributions of all shards sum to the unsharded backward."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

from oracle import message_passing_oracle as mo
from test_gpu_parity import (_need_gpu, _torch_reference_ggnn, _torch_reference_layer, assert_states_close, make_layer,
                             random_graph)

pytestmark = pytest.mark.gpu


def _shard_bounds(V, deg):
    """world 2 and 3 balanced by in-degree, and a world of 3 whose middle shard is empty."""
    from tf2_gnn_b200 import sharding
    cut = V // 3
    return [sharding.partition_target_range(V, 2, deg), sharding.partition_target_range(V, 3, deg),
            [(0, cut), (cut, cut), (cut, V)]]


def _backward(layer, params, ht, adj, g, prepared=None):
    """(grad_h, [grad of each param]) of one layer call and out.backward(g)."""
    from tf2_gnn_b200.layers import MessagePassingInput
    h = ht.detach().clone().requires_grad_()
    for p in params:
        p.value.grad = None
    out = layer(MessagePassingInput(h, adj), prepared=prepared)
    out.backward(g)
    torch.cuda.synchronize()
    return h.grad.cpu().numpy(), [p.value.grad.cpu().numpy() for p in params]


def _check_shards(layer, params, h, adjs, g, ref64):
    """Every world of _shard_bounds: filtered / unfiltered edge lists agree bit for bit, each shard is reproducible, an
    empty shard gives zeros, and the summed contributions equal the unsharded backward and the float64 reference."""
    from tf2_gnn_b200 import sharding
    from tf2_gnn_b200.runtime import PreparedBatch
    V = h.shape[0]
    ht = torch.from_numpy(h).cuda()
    adj_t = tuple(torch.from_numpy(a).cuda() for a in adjs)
    gt = torch.from_numpy(g).cuda()
    full_h, full_w = _backward(layer, params, ht, adj_t, gt)
    ref_h, ref_w = ref64
    assert_states_close(full_h, ref_h, tol=2e-5)
    deg = sum(np.bincount(a[:, 1], minlength=V) for a in adjs)
    for bounds in _shard_bounds(V, deg):
        sum_h = np.zeros(full_h.shape, np.float64)
        sum_w = [np.zeros(w.shape, np.float64) for w in full_w]
        for lo, hi in bounds:
            got = {}
            for filtered in (False, True):
                a_in = adj_t if not filtered else tuple(
                    torch.from_numpy(a).cuda() for a in sharding.filter_edges_by_target(adjs, lo, hi))
                pb = PreparedBatch(a_in, V, target_range=(lo, hi))
                got[filtered] = _backward(layer, params, ht, a_in, gt[lo:hi], prepared=pb)
                again = _backward(layer, params, ht, a_in, gt[lo:hi], prepared=pb)
                assert np.array_equal(got[filtered][0], again[0])                 # bitwise reproducible
                assert all(np.array_equal(a, b) for a, b in zip(got[filtered][1], again[1]))
            assert np.array_equal(got[False][0], got[True][0])
            assert all(np.array_equal(a, b) for a, b in zip(got[False][1], got[True][1]))
            gh, gw = got[True]
            assert gh.shape == full_h.shape
            if hi == lo:
                assert not gh.any() and not any(w.any() for w in gw)
            sum_h += gh
            for s, w in zip(sum_w, gw):
                s += w
        assert_states_close(sum_h, full_h.astype(np.float64), tol=2e-6)
        assert_states_close(sum_h, ref_h, tol=2e-5)
        for s, w, r in zip(sum_w, full_w, ref_w):
            assert_states_close(s, w.astype(np.float64), tol=2e-6)
            assert_states_close(s, r, tol=2e-5)


@pytest.mark.parametrize("D,H,agg,act,normalize,use_target", [
    (64, 64, "sum", "relu", True, False),
    (32, 48, "mean", "tanh", False, False),
    (64, 32, "sqrt_n", "gelu", True, False),
    (64, 64, "sum", "tanh", True, True),
    (32, 36, "mean", "relu", False, True),
    (64, 64, "sqrt_n", "relu", False, True),
])
def test_rgcn_shard_backward_sums_to_full(D, H, agg, act, normalize, use_target):
    _need_gpu()
    from tf2_gnn_b200.layers import RGCN
    V, L = 700, 3
    rng = np.random.default_rng(D + H + L)
    adjs = random_graph(rng, V, L, 5000, hub=True, dups=True, self_loops=use_target)
    p = RGCN.get_default_hyperparameters()
    p.update(hidden_dim=H, aggregation_function=agg, message_activation_function=act,
             normalize_by_num_incoming=normalize, use_target_state_as_input=use_target)
    h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    Ws = [mo.glorot_uniform(rng, ((2 if use_target else 1) * D, H)) for _ in range(L)]
    g = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    layer = make_layer("rgcn", p, D, L, {"edge_mlps": [[w] for w in Ws]})
    params = [mlp.layers[0] for mlp in layer._edge_type_mlps]
    for v in layer.variables:
        v.requires_grad_()
    h64 = torch.from_numpy(h).double().requires_grad_()
    W64 = [torch.from_numpy(w).double().requires_grad_() for w in Ws]
    _torch_reference_layer(h64, [torch.from_numpy(a) for a in adjs], W64, normalize, agg, act,
                           use_target=use_target).backward(torch.from_numpy(g).double())
    _check_shards(layer, params, h, adjs, g, (h64.grad.numpy(), [w.grad.numpy() for w in W64]))


@pytest.mark.parametrize("H,agg,normalize", [(64, "sum", True), (32, "mean", False), (36, "sqrt_n", True)])
def test_ggnn_shard_backward_sums_to_full(H, agg, normalize):
    _need_gpu()
    from tf2_gnn_b200.layers import GGNN
    V, L = 600, 2
    rng = np.random.default_rng(H + L)
    adjs = random_graph(rng, V, L, 4000, hub=True, dups=True)
    p = GGNN.get_default_hyperparameters()
    p.update(hidden_dim=H, aggregation_function=agg, normalize_by_num_incoming=normalize)
    h = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    Ws = [mo.glorot_uniform(rng, (H, H)) for _ in range(L)]
    K, U = mo.glorot_uniform(rng, (H, 3 * H)), mo.glorot_uniform(rng, (H, 3 * H))
    b = rng.uniform(-0.2, 0.2, (2, 3 * H)).astype(np.float32)
    g = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    layer = make_layer("ggnn", p, H, L, {"edge_mlps": [[w] for w in Ws], "gru_kernel": K, "gru_recurrent_kernel": U,
                                         "gru_bias": b})
    params = [mlp.layers[0] for mlp in layer._edge_type_mlps] + [layer._gru_kernel, layer._gru_recurrent_kernel,
                                                                 layer._gru_bias]
    for v in layer.variables:
        v.requires_grad_()
    h64 = torch.from_numpy(h).double().requires_grad_()
    W64 = [torch.from_numpy(w).double().requires_grad_() for w in Ws]
    K64, U64, b64 = (torch.from_numpy(x).double().requires_grad_() for x in (K, U, b))
    _torch_reference_ggnn(h64, [torch.from_numpy(a) for a in adjs], W64, K64, U64, b64, normalize,
                          agg).backward(torch.from_numpy(g).double())
    _check_shards(layer, params, h, adjs, g,
                  (h64.grad.numpy(), [w.grad.numpy() for w in W64] + [x.grad.numpy() for x in (K64, U64, b64)]))


@pytest.mark.parametrize("filtered", [False, True])
def test_owned_transpose_csr_is_bit_exact(filtered):
    """TFGNN_PREPARE_TRANSPOSE_OWNED: edges into [lo, hi), segments (type, global source), local target ids ascending."""
    _need_gpu()
    from tf2_gnn_b200 import sharding
    from tf2_gnn_b200.runtime import PreparedBatch
    rng = np.random.default_rng(3)
    V, L = 5000, 3
    adjs = random_graph(rng, V, L, [40000, 0, 25000], hub=True, dups=True)
    for lo, hi in [(0, V), (0, 1700), (1700, 1700), (1700, 3301), (3301, V)]:
        a_np = sharding.filter_edges_by_target(adjs, lo, hi) if filtered else adjs
        pb = PreparedBatch(tuple(torch.from_numpy(a).cuda() for a in a_np), V, target_range=(lo, hi))
        row_ptr, vals = (t.cpu().numpy() for t in pb.transposed().csr())
        keys, values = [], []
        for l, a in enumerate(adjs):
            keep = (a[:, 1] >= lo) & (a[:, 1] < hi)
            keys.append(l * V + a[keep, 0].astype(np.int64))
            values.append(a[keep, 1] - lo)
        keys, values = np.concatenate(keys), np.concatenate(values).astype(np.int32)
        order = np.lexsort((values, keys))
        ref_ptr = np.concatenate([[0], np.cumsum(np.bincount(keys, minlength=L * V))]).astype(np.int32)
        assert np.array_equal(row_ptr, ref_ptr)
        assert np.array_equal(vals[: len(order)], values[order])
