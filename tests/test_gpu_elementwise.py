"""Kernel results checked element by element against float64 error bounds (tests/bounds64.py).

The parity tests scale their tolerance by the largest element of a tensor, so wherever rows differ a lot in magnitude
(unnormalised sums into a hub, a 100 000-node graph next to one-node graphs, source hubs in dh) the ordinary rows are held
to a bar 100x or more looser than 1e-5.  Here every element meets |got - ref64| <= 1e-5 * bound, the bound being the same
computation on absolute values; rows without edges and empty graphs must come out exact.  Every output a test allocates
for a direct library call starts out as NaN, so a row the kernel leaves unwritten cannot pass.

Each check prints "RATIO <case> <largest error / bound>" (pytest -s shows them): about 1e-7 is float32 rounding, a
3xTF32 product that lost its correction terms shows up at 5e-5.
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

import bounds64 as b64  # noqa: E402
import reference64 as r64  # noqa: E402
import reference64_edge_mlp as rm  # noqa: E402
from elementwise_cases import (DENSE_BWD_CASES, EDGE_MLP_BWD_CASES, FAMILY_CASES, LAYERNORM_CASES, PART_ROWS,  # noqa: E402
                               RGCN_BWD_CASES, RGCN_CASES, SEG_ROWS, dense_bwd_inputs, edge_mlp_bwd_inputs, family_case,
                               in_degree, layernorm_case, layernorm_reference, out_degree, reduction_inputs,
                               reduction_layout, rgcn_bwd_inputs, rgcn_case, shard_range, straddles)
from oracle import message_passing_oracle as mo  # noqa: E402
from test_gpu_parity import _need_gpu, make_layer  # noqa: E402

pytestmark = pytest.mark.gpu

REL = 1e-5
NAN = float("nan")


def report(name, ratio):
    print(f"RATIO {name} {ratio:.3e}")


def nan_out(*shape):
    return torch.full(shape, NAN, dtype=torch.float32, device="cuda")


# ------------------------------------------------------------------------------------------------------------------
# RGCN forward on every path
# ------------------------------------------------------------------------------------------------------------------
def rgcn_abi(p, w, h, adjs, path, target_range=None, ln=None):
    """tfgnn_b200_rgcn_fwd (or _rgcn_ln_fwd with ln = (gamma, beta, eps)) into a NaN-filled output."""
    from tf2_gnn_b200 import _ffi
    from tf2_gnn_b200.runtime import PreparedBatch, stream_ptr
    V, D = h.shape
    H = int(p["hidden_dim"])
    adj_dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in adjs]
    pb = PreparedBatch(adj_dev, V, target_range=target_range)
    ht = torch.from_numpy(h).cuda()
    Ws = [torch.from_numpy(m[0]).cuda() for m in w["edge_mlps"]]
    out = nan_out(pb.num_nodes, H)
    flags = _ffi.FLAG_NORMALIZE if p["normalize_by_num_incoming"] else 0
    args = (pb.handle, ht.data_ptr(), D, _ffi.ptr_array(Ws), H, flags, _ffi.AGG[p["aggregation_function"]],
            _ffi.ACT[p["message_activation_function"]], _ffi.PATH[path])
    if ln is None:
        _ffi.check(_ffi.lib().tfgnn_b200_rgcn_fwd(*args, out.data_ptr(), stream_ptr()))
    else:
        gamma, beta, eps = (torch.from_numpy(ln[0]).cuda(), torch.from_numpy(ln[1]).cuda(), ln[2])
        _ffi.check(_ffi.lib().tfgnn_b200_rgcn_ln_fwd(*args, gamma.data_ptr(), beta.data_ptr(), float(eps), out.data_ptr(),
                                                    stream_ptr()))
    torch.cuda.synchronize()
    return out.cpu().numpy()


def split_tiles(V, env):
    """Whether the fused kernel's launch rule (csrc/fused_rgcn.cu) takes split-tile mode for V rows: fewer 128-row tiles
    than half the SMs (at most 160 counted), unless TFGNN_B200_FUSED_SPLIT=0.  Every H of RGCN_CASES allows it."""
    sms = min(torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count, 160)
    return env.get("TFGNN_B200_FUSED_SPLIT", "1") != "0" and 2 * -(-V // 128) <= sms


@pytest.mark.parametrize("name,path,V,D,H,L,agg,act,env", RGCN_CASES, ids=[c[0] for c in RGCN_CASES])
def test_rgcn_forward_within_bound(monkeypatch, name, path, V, D, H, L, agg, act, env):
    """Whole batch and a target-range shard (its rows against the matching slice of the full bound).  A fused case must
    reach the kernel its name gives (elementwise_cases.RGCN_CASES): split-tile mode for the split cases only."""
    _need_gpu()
    monkeypatch.delenv("TFGNN_B200_FUSED_SPLIT", raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    if path == "fused_tc":
        assert split_tiles(V, env) == ("split" in name), f"{name}: the launch rule picks another kernel for V = {V}"
    p, w, h, adjs = rgcn_case(V, D, H, L, agg, act, seed=V + H)
    ref = mo.message_passing_forward("rgcn", p, w, h, adjs, dtype=np.float64)
    bound = b64.forward_bound("rgcn", p, w, h, adjs)
    deg = in_degree(V, adjs)
    got = rgcn_abi(p, w, h, adjs, path)
    tiles = path == "fused_tc"
    report(name, b64.assert_within_bound(got, ref, bound, REL, what=name, row_sizes=deg, tiles=tiles))
    lo, hi = shard_range(V)
    if path == "atomic":
        with pytest.raises(NotImplementedError):          # the atomic path has no shard form
            rgcn_abi(p, w, h, adjs, path, target_range=(lo, hi))
        return
    got = rgcn_abi(p, w, h, adjs, path, target_range=(lo, hi))
    report(name + "/shard", b64.assert_within_bound(got, ref[lo:hi], bound[lo:hi], REL, what=name + " shard",
                                                    row_sizes=deg[lo:hi], tiles=tiles))


@pytest.mark.parametrize("V,act", LAYERNORM_CASES)
def test_rgcn_layernorm_entry_within_bound(V, act):
    """tfgnn_b200_rgcn_ln_fwd (H = 64: LayerNorm in the fused kernel's epilogue) against LayerNorm of the float64 layer,
    with the bound of elementwise_cases.layernorm_reference."""
    _need_gpu()
    p, w, h, adjs, ln = layernorm_case(V, act)
    ref, bound = layernorm_reference(p, w, h, adjs, ln)
    got = rgcn_abi(p, w, h, adjs, "fused_tc", ln=ln)
    report(f"layernorm_{act}", b64.assert_within_bound(got, ref, bound, REL, what="rgcn_ln_fwd",
                                                       row_sizes=in_degree(V, adjs), tiles=True))


# ------------------------------------------------------------------------------------------------------------------
# Edge-MLP family and RGAT through the layers
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,kind,extra", FAMILY_CASES, ids=[c[0] for c in FAMILY_CASES])
def test_message_passing_family_within_bound(name, kind, extra):
    _need_gpu()
    from tf2_gnn_b200.layers import MessagePassingInput
    p, w, h, adjs = family_case(kind, extra)
    V, D = h.shape
    L = len(adjs)
    layer = make_layer(kind, p, D, L, w)
    with torch.no_grad():
        out = layer(MessagePassingInput(torch.from_numpy(h).cuda(), tuple(torch.from_numpy(a).cuda() for a in adjs)))
    torch.cuda.synchronize()
    ref = mo.message_passing_forward(kind, p, w, h, adjs, dtype=np.float64)
    bound = b64.forward_bound(kind, p, w, h, adjs)
    report(name, b64.assert_within_bound(out.cpu().numpy(), ref, bound, REL, what=name, row_sizes=in_degree(V, adjs)))


# ------------------------------------------------------------------------------------------------------------------
# Graph reductions
# ------------------------------------------------------------------------------------------------------------------
def test_reduction_layout_has_every_edge_case():
    ptr = reduction_layout()
    sizes = np.diff(ptr)
    assert sizes[0] == 0 and sizes[-1] == 0 and np.any(sizes[1:-1] == 0)
    assert np.any(sizes == 1) and sizes.max() == 100_000
    assert len(straddles(ptr, SEG_ROWS)) and len(straddles(ptr, PART_ROWS))


def _graph_sizes(ptr):
    return np.diff(ptr.astype(np.int64))


def test_segment_sum_rows_within_bound():
    _need_gpu()
    from tf2_gnn_b200 import _ffi
    from tf2_gnn_b200.runtime import stream_ptr
    ptr, x, _ = reduction_inputs()
    G, C = len(ptr) - 1, x.shape[1]
    ids = b64.graph_ids(ptr).astype(np.int32)
    out = nan_out(G, C)
    xt, idt, pt = (torch.from_numpy(a).cuda() for a in (x, ids, ptr))
    _ffi.check(_ffi.lib().tfgnn_b200_segment_sum_rows(xt.data_ptr(), idt.data_ptr(), pt.data_ptr(), len(x), G, C,
                                                      out.data_ptr(), stream_ptr()))
    ref = mo.unsorted_segment_sum(x.astype(np.float64), ids, G)
    report("segment_sum_rows", b64.assert_within_bound(out.cpu().numpy(), ref, b64.segment_bound(x, ptr), REL,
                                                       what="segment_sum_rows", row_sizes=_graph_sizes(ptr),
                                                       row_label="graph size"))


@pytest.mark.parametrize("weighting", ["none", "average", "sigmoid", "softmax"])
def test_weighted_segment_sum_within_bound(weighting):
    """tfgnn_b200_weighted_segment_sum under the readout's four weightings; softmax takes its weights from
    tfgnn_b200_segment_softmax."""
    _need_gpu()
    from tf2_gnn_b200 import _ffi
    from tf2_gnn_b200.runtime import stream_ptr
    K = 4
    ptr, x, scores = reduction_inputs(K=K)
    G, C = len(ptr) - 1, x.shape[1]
    ids = b64.graph_ids(ptr)
    x64 = x.astype(np.float64)
    xt, pt = torch.from_numpy(x).cuda(), torch.from_numpy(ptr).cuda()
    wt = None
    if weighting == "sigmoid":
        w = (1.0 / (1.0 + np.exp(-scores.astype(np.float64)))).astype(np.float32)
        wt = torch.from_numpy(w).cuda()
        ref = mo.unsorted_segment_sum((x64.reshape(-1, K, C // K) * w[:, :, None]).reshape(-1, C), ids, G)
        bound = b64.segment_bound(x, ptr, weights=w, num_heads=K)
    elif weighting == "softmax":
        st = torch.from_numpy(scores).cuda()
        wt = nan_out(len(x), K)
        _ffi.check(_ffi.lib().tfgnn_b200_segment_softmax(st.data_ptr(), pt.data_ptr(), G, K, wt.data_ptr(), stream_ptr()))
        alpha = np.stack([mo.unsorted_segment_softmax(scores[:, k].astype(np.float64), ids, G) for k in range(K)], 1)
        ref = mo.unsorted_segment_sum((x64.reshape(-1, K, C // K) * alpha[:, :, None]).reshape(-1, C), ids, G)
        bound = b64.softmax_segment_bound(x, scores, ptr, K)
    else:
        mean = weighting == "average"
        ref = (mo.unsorted_segment_mean if mean else mo.unsorted_segment_sum)(x64, ids, G)
        bound = b64.segment_bound(x, ptr, agg="mean" if mean else "sum")
    out = nan_out(G, C)
    _ffi.check(_ffi.lib().tfgnn_b200_weighted_segment_sum(xt.data_ptr(), 0 if wt is None else wt.data_ptr(), pt.data_ptr(),
                                                          G, C, K, 1 if weighting == "average" else 0, out.data_ptr(),
                                                          stream_ptr()))
    report(f"weighted_segment_sum_{weighting}",
           b64.assert_within_bound(out.cpu().numpy(), ref, bound, REL, what=f"weighted_segment_sum {weighting}",
                                   row_sizes=_graph_sizes(ptr), row_label="graph size"))


@pytest.mark.parametrize("world", [1, 2, 4])
@pytest.mark.parametrize("weighting", ["softmax", "sigmoid", "none"])
def test_readout_partial_merge_within_bound(world, weighting):
    """tfgnn_b200_readout_partial on each of `world` contiguous row ranges (cut inside graphs), tfgnn_b200_readout_merge
    over the stacked partials."""
    _need_gpu()
    from tf2_gnn_b200 import _ffi
    from tf2_gnn_b200.runtime import stream_ptr
    ptr, x, scores = reduction_inputs()
    G, GD = len(ptr) - 1, x.shape[1]
    K = 1 if weighting == "none" else scores.shape[1]
    mode = _ffi.READOUT_MODE[weighting]
    ids = b64.graph_ids(ptr)
    x64 = x.astype(np.float64)
    if weighting == "softmax":
        w_in = scores
        alpha = np.stack([mo.unsorted_segment_softmax(scores[:, k].astype(np.float64), ids, G) for k in range(K)], 1)
        bound = b64.softmax_segment_bound(x, scores, ptr, K)
    elif weighting == "sigmoid":
        w_in = alpha = (1.0 / (1.0 + np.exp(-scores.astype(np.float64)))).astype(np.float32)
        bound = b64.segment_bound(x, ptr, weights=alpha, num_heads=K)
    else:
        w_in, alpha = None, np.ones((len(x), 1))
        bound = b64.segment_bound(x, ptr)
    ref = mo.unsorted_segment_sum((x64.reshape(-1, K, GD // K) * alpha[:, :, None]).reshape(-1, GD), ids, G)
    cuts = np.linspace(0, len(x), world + 1).astype(np.int64)
    cuts[1:-1] += 17                                      # off any chunk border
    P = 2 * K + GD
    parts = nan_out(world, G, P)
    keep = []
    for r in range(world):
        lo, hi = int(cuts[r]), int(cuts[r + 1])
        local = ids[lo:hi].astype(np.int32)
        lptr = np.searchsorted(local, np.arange(G + 1), side="left").astype(np.int32)
        xt, nt, pt = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x[lo:hi], local, lptr))
        st = None if w_in is None else torch.from_numpy(np.ascontiguousarray(w_in[lo:hi])).cuda()
        keep += [xt, nt, pt, st]
        _ffi.check(_ffi.lib().tfgnn_b200_readout_partial(0 if st is None else st.data_ptr(), xt.data_ptr(), nt.data_ptr(),
                                                         pt.data_ptr(), hi - lo, G, GD, K, mode, parts[r].data_ptr(),
                                                         stream_ptr()))
    out = nan_out(G, GD)
    gmax = nan_out(G, K) if weighting == "softmax" else None
    gsum = nan_out(G, K) if weighting == "softmax" else None
    _ffi.check(_ffi.lib().tfgnn_b200_readout_merge(parts.data_ptr(), world, G, GD, K, mode, out.data_ptr(),
                                                   0 if gmax is None else gmax.data_ptr(),
                                                   0 if gsum is None else gsum.data_ptr(), stream_ptr()))
    torch.cuda.synchronize()
    name = f"readout_{weighting}_world{world}"
    report(name, b64.assert_within_bound(out.cpu().numpy(), ref, bound, REL, what=name, row_sizes=_graph_sizes(ptr),
                                         row_label="graph size"))


@pytest.mark.parametrize("agg", ["sum", "mean", "sqrt_n", "max"])
def test_unsorted_segment_reduce_within_bound(agg):
    """tfgnn_b200_unsorted_segment_reduce over the same layout with the rows shuffled (the ids are not sorted)."""
    _need_gpu()
    from tf2_gnn_b200 import _ffi
    from tf2_gnn_b200.runtime import stream_ptr
    ptr, x, _ = reduction_inputs()
    G, C = len(ptr) - 1, x.shape[1]
    perm = np.random.default_rng(5).permutation(len(x))
    xs, ids = np.ascontiguousarray(x[perm]), b64.graph_ids(ptr)[perm].astype(np.int32)
    out = nan_out(G, C)
    xt, it = torch.from_numpy(xs).cuda(), torch.from_numpy(ids).cuda()
    _ffi.check(_ffi.lib().tfgnn_b200_unsorted_segment_reduce(xt.data_ptr(), it.data_ptr(), 1, len(xs), C, G, _ffi.AGG[agg],
                                                             out.data_ptr(), stream_ptr()))
    ref = mo.get_aggregation_function(agg)(xs.astype(np.float64), ids, G)
    report(f"unsorted_segment_{agg}", b64.assert_within_bound(out.cpu().numpy(), ref, b64.segment_bound(x, ptr, agg=agg),
                                                              REL, what=f"unsorted_segment_reduce {agg}",
                                                              row_sizes=_graph_sizes(ptr), row_label="graph size"))


# ------------------------------------------------------------------------------------------------------------------
# Backward
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("act", ["tanh", "gelu"])
@pytest.mark.parametrize("V,K,N,bias", DENSE_BWD_CASES)
def test_dense_bwd_within_bound(act, V, K, N, bias):
    _need_gpu()
    from tf2_gnn_b200 import _ffi
    from tf2_gnn_b200.layers import node_ops
    from tf2_gnn_b200.runtime import stream_ptr
    from tf2_gnn_b200.utils.param_helpers import get_activation_function
    x, W, b, g = dense_bwd_inputs(V, K, N, bias)
    xt, Wt, gt = (torch.from_numpy(a).cuda() for a in (x, W, g))
    bt = torch.from_numpy(b).cuda() if bias else None
    out = node_ops.dense(xt, Wt, bt, get_activation_function(act))
    gx, gW, gb = nan_out(V, K), nan_out(K, N), nan_out(N) if bias else None
    _ffi.check(_ffi.lib().tfgnn_b200_dense_bwd(xt.data_ptr(), Wt.data_ptr(), 0 if bt is None else bt.data_ptr(),
                                               out.data_ptr(), gt.data_ptr(), V, K, N, _ffi.ACT[act], gx.data_ptr(),
                                               gW.data_ptr(), 0 if gb is None else gb.data_ptr(), stream_ptr()))
    torch.cuda.synchronize()
    x64, W64 = (torch.from_numpy(a).double().requires_grad_() for a in (x, W))
    b64_ = torch.from_numpy(b).double().requires_grad_() if bias else None
    z = x64 @ W64 + (b64_ if bias else 0.0)
    y, _ = r64.act_and_grad(z, act)
    y.backward(torch.from_numpy(g).double())
    bd = b64.dense_backward_bound(x, W, b, g, act)
    name = f"dense_bwd_{act}_{V}x{K}x{N}"
    ratios = [b64.assert_within_bound(out.cpu().numpy(), y.detach().numpy(), bd["out"], REL, what=name + " out"),
              b64.assert_within_bound(gx.cpu().numpy(), x64.grad.numpy(), bd["grad_x"], REL, what=name + " grad_x"),
              b64.assert_within_bound(gW.cpu().numpy(), W64.grad.numpy(), bd["grad_W"], REL, what=name + " grad_W")]
    if bias:
        ratios.append(b64.assert_within_bound(gb.cpu().numpy(), b64_.grad.numpy(), bd["grad_bias"], REL,
                                              what=name + " grad_bias"))
    report(name, max(ratios))


def _layer_bwd_abi(entry, h, adjs, weights, grad_out, flags, agg, act, n_hidden=None):
    """Forward (auto path) then the fused backward `entry` (rgcn_bwd or edge_mlp_bwd) into NaN-filled gradients:
    (out, grad_h, [grad of each weight])."""
    from tf2_gnn_b200 import _ffi
    from tf2_gnn_b200.runtime import PreparedBatch, stream_ptr
    V, D = h.shape
    lib = _ffi.lib()
    adj_dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in adjs]
    pb = PreparedBatch(adj_dev, V)
    ht = torch.from_numpy(h).cuda()
    wt = [torch.from_numpy(x).cuda() for x in weights]
    H = grad_out.shape[1]
    g = torch.from_numpy(grad_out).cuda()
    out = nan_out(V, H)
    grad_h = nan_out(V, D)
    grad_w = [torch.full_like(x, NAN) for x in wt]
    a, c = _ffi.AGG[agg], _ffi.ACT[act]
    if entry == "rgcn":
        _ffi.check(lib.tfgnn_b200_rgcn_fwd(pb.handle, ht.data_ptr(), D, _ffi.ptr_array(wt), H, flags, a, c, 0,
                                           out.data_ptr(), stream_ptr()))
        _ffi.check(lib.tfgnn_b200_rgcn_bwd(pb.handle, pb.transposed().handle, ht.data_ptr(), D, _ffi.ptr_array(wt), H,
                                           flags, a, c, out.data_ptr(), g.data_ptr(), grad_h.data_ptr(),
                                           _ffi.ptr_array(grad_w), stream_ptr()))
    else:
        _ffi.check(lib.tfgnn_b200_edge_mlp_fwd(pb.handle, ht.data_ptr(), D, _ffi.ptr_array(wt), n_hidden, H, flags, a, c,
                                               0, out.data_ptr(), stream_ptr()))
        _ffi.check(lib.tfgnn_b200_edge_mlp_bwd(pb.handle, pb.transposed().handle, ht.data_ptr(), D, _ffi.ptr_array(wt),
                                               n_hidden, H, flags, a, c, out.data_ptr(), g.data_ptr(), grad_h.data_ptr(),
                                               _ffi.ptr_array(grad_w), stream_ptr()))
    torch.cuda.synchronize()
    return out.cpu().numpy(), grad_h.cpu().numpy(), [x.cpu().numpy() for x in grad_w]


@pytest.mark.parametrize("act", ["tanh", "gelu"])
@pytest.mark.parametrize("V,D,H,agg,normalize", RGCN_BWD_CASES)
def test_rgcn_backward_within_bound(act, V, D, H, agg, normalize):
    """tfgnn_b200_rgcn_bwd on a graph with Zipf source hubs (segments of thousands of edges in the dh reduce)."""
    _need_gpu()
    from tf2_gnn_b200 import _ffi
    h, adjs, Ws, g = rgcn_bwd_inputs(V, D, H)
    L = len(Ws)
    out, gh, gW = _layer_bwd_abi("rgcn", h, adjs, Ws, g, _ffi.FLAG_NORMALIZE if normalize else 0, agg, act)
    ref = r64.rgcn_layer(h, adjs, Ws, g, agg=agg, act=act, normalize=normalize)
    bd = b64.rgcn_backward_bound(h, adjs, Ws, g, agg=agg, act=act, normalize=normalize)
    name = f"rgcn_bwd_{act}_{V}"
    ratios = [b64.assert_within_bound(out, ref["out"].numpy(), bd["out"], REL, what=name + " out",
                                      row_sizes=in_degree(V, adjs), tiles=True),
              b64.assert_within_bound(gh, ref["grad_h"].numpy(), bd["grad_h"], REL, what=name + " grad_h",
                                      row_sizes=out_degree(V, adjs), row_label="out-degree")]
    ratios += [b64.assert_within_bound(gW[l], ref["grad_W"][l].numpy(), bd["grad_W"][l], REL, what=f"{name} grad_W[{l}]")
               for l in range(L)]
    report(name, max(ratios))


@pytest.mark.parametrize("act,agg,use_target", EDGE_MLP_BWD_CASES)
def test_edge_mlp_backward_within_bound(act, agg, use_target):
    """tfgnn_b200_edge_mlp_bwd (one hidden layer) on an unnormalised source-hub graph.  h and the first kernels sit on the
    1/64 grid, so every hidden pre-activation is exact in fp32 and in 3xTF32 and the GPU's relu mask is the float64 one."""
    _need_gpu()
    from tf2_gnn_b200 import _ffi
    h, adjs, Us, W2s, g = edge_mlp_bwd_inputs(use_target)
    V, L = len(h), len(Us)
    flags = _ffi.FLAG_USE_TARGET if use_target else 0
    out, gh, gw = _layer_bwd_abi("edge_mlp", h, adjs, [x for pair in zip(Us, W2s) for x in pair], g, flags, agg, act,
                                 n_hidden=1)
    ref = rm.edge_mlp_layer(h, adjs, Us, W2s, g, agg=agg, act=act, normalize=False, use_target=use_target)
    bd = b64.edge_mlp_backward_bound(h, adjs, Us, W2s, g, agg=agg, act=act, normalize=False, use_target=use_target)
    name = f"edge_mlp_bwd_{act}_{agg}"
    ratios = [b64.assert_within_bound(out, ref["out"].numpy(), bd["out"], REL, what=name + " out",
                                      row_sizes=in_degree(V, adjs)),
              b64.assert_within_bound(gh, ref["grad_h"].numpy(), bd["grad_h"], REL, what=name + " grad_h",
                                      row_sizes=out_degree(V, adjs), row_label="out-degree")]
    for l in range(L):
        ratios.append(b64.assert_within_bound(gw[2 * l], ref["grad_U"][l].numpy(), bd["grad_U"][l], REL,
                                              what=f"{name} grad_U[{l}]"))
        ratios.append(b64.assert_within_bound(gw[2 * l + 1], ref["grad_W2"][l].numpy(), bd["grad_W2"][l], REL,
                                              what=f"{name} grad_W2[{l}]"))
    report(name, max(ratios))
