"""GPU parity of the round-2 additions: graph readout + global exchange (SURVEY.md §8f-4), the GNN stack with the
reference's DEFAULT hyper-parameters (global exchange every 2 layers), training-time glue (Dense / LayerNorm / residual /
dropout backward), one full training step of a PPI_RGCN-shaped stack, and the round-1 ADVICE regressions."""
import os
import sys

import numpy as np
import pytest

torch = pytest.importorskip("torch")

from oracle import message_passing_oracle as mo

pytestmark = pytest.mark.gpu
TOL = 1e-5


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def close(got, ref64, tol=TOL, what=""):
    got = np.asarray(got, np.float64)
    ref64 = np.asarray(ref64, np.float64)
    assert got.shape == ref64.shape, f"{what}: shape {got.shape} vs {ref64.shape}"
    scale = max(np.abs(ref64).max(), 1e-30)
    err = np.abs(got - ref64).max()
    assert err <= tol * scale, f"{what}: max abs err {err:.3e} > {tol:g} * {scale:.3e}"


def random_n2g(rng, V, G, empty_graph=None):
    ids = np.sort(rng.integers(0, G, size=V)).astype(np.int32)
    if empty_graph is not None:
        ids[ids == empty_graph] = empty_graph + 1 if empty_graph + 1 < G else empty_graph - 1
        ids = np.sort(ids)
    return ids


# ------------------------------------------------------------------------------------------------------------------
# readout
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("weighting", ["softmax", "sigmoid", "average", "none"])
@pytest.mark.parametrize("V,G,D,GD,K", [(500, 7, 32, 24, 3), (4000, 300, 64, 64, 4), (9000, 3, 320, 320, 4)])
def test_weighted_sum_graph_representation(weighting, V, G, D, GD, K):
    """nodes_to_graph_representation.py:170-229; QM9-like (many tiny graphs) and PPI-like (3 graphs of thousands of nodes)."""
    _need_gpu()
    from tf2_gnn_b200.layers import NodesToGraphRepresentationInput, WeightedSumGraphRepresentation
    rng = np.random.default_rng(V + G)
    x = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    n2g = random_n2g(rng, V, G, empty_graph=2 if G > 5 else None)
    layer = WeightedSumGraphRepresentation(graph_representation_size=GD, num_heads=K, weighting_fun=weighting,
                                           scoring_mlp_layers=[D], transformation_mlp_layers=[48])
    layer.build(NodesToGraphRepresentationInput((None, D), None, None))
    w = {"transformation_mlp": [mo.glorot_uniform(rng, (D, 48)), mo.glorot_uniform(rng, (48, GD))]}
    for var, m in zip(layer._transformation_mlp.kernels, w["transformation_mlp"]):
        var.assign(m)
    if weighting in ("softmax", "sigmoid"):
        w["scoring_mlp"] = [mo.glorot_uniform(rng, (D, D)) * 3, mo.glorot_uniform(rng, (D, K)) * 3]
        for var, m in zip(layer._scoring_mlp.kernels, w["scoring_mlp"]):
            var.assign(m)
    out = layer(NodesToGraphRepresentationInput(torch.from_numpy(x).cuda(), torch.from_numpy(n2g).cuda(), G))
    ref = mo.weighted_sum_graph_representation(x, n2g, G, w, GD, K, weighting, dtype=np.float64)
    close(out.cpu().numpy(), ref, what=f"readout {weighting}")


def test_readout_with_biases_bounds_and_elu():
    """The graph_regression_task.py configuration: biases, non-ReLU activation, clipped transformation results."""
    _need_gpu()
    from tf2_gnn_b200.layers import NodesToGraphRepresentationInput, WeightedSumGraphRepresentation
    rng = np.random.default_rng(5)
    V, G, D, GD, K = 700, 40, 32, 16, 4
    x = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    n2g = random_n2g(rng, V, G)
    layer = WeightedSumGraphRepresentation(GD, K, "sigmoid", scoring_mlp_layers=[20], scoring_mlp_activation_fun="elu",
                                           scoring_mlp_use_biases=True, transformation_mlp_layers=[24],
                                           transformation_mlp_activation_fun="tanh", transformation_mlp_use_biases=True,
                                           transformation_mlp_result_lower_bound=-0.3,
                                           transformation_mlp_result_upper_bound=0.4)
    layer.build(NodesToGraphRepresentationInput((None, D), None, None))
    w = {"scoring_mlp": [mo.glorot_uniform(rng, (D, 20)), mo.glorot_uniform(rng, (20, K))],
         "scoring_biases": [rng.uniform(-.2, .2, 20).astype(np.float32), rng.uniform(-.2, .2, K).astype(np.float32)],
         "transformation_mlp": [mo.glorot_uniform(rng, (D, 24)), mo.glorot_uniform(rng, (24, GD))],
         "transformation_biases": [rng.uniform(-.2, .2, 24).astype(np.float32), rng.uniform(-.2, .2, GD).astype(np.float32)]}
    for mlp, key in ((layer._scoring_mlp, "scoring"), (layer._transformation_mlp, "transformation")):
        for var, m in zip(mlp.kernels, w[f"{key}_mlp"]):
            var.assign(m)
        for var, m in zip(mlp.biases, w[f"{key}_biases"]):
            var.assign(m)
    out = layer(NodesToGraphRepresentationInput(torch.from_numpy(x).cuda(), torch.from_numpy(n2g).cuda(), G))
    ref = mo.weighted_sum_graph_representation(x, n2g, G, w, GD, K, "sigmoid", scoring_activation="elu",
                                               transformation_activation="tanh", lower_bound=-0.3, upper_bound=0.4,
                                               dtype=np.float64)
    close(out.cpu().numpy(), ref, what="readout with biases")


def test_node_to_graph_map_validation():
    _need_gpu()
    from tf2_gnn_b200.layers import node_ops
    bad = torch.tensor([0, 1, 1, 0, 2], dtype=torch.int32).cuda()
    with pytest.raises(ValueError):
        node_ops.graph_offsets(bad, 3, validate=True)
    ok = torch.tensor([0, 0, 2, 2, 2, 4], dtype=torch.int32).cuda()
    ptr = node_ops.graph_offsets(ok, 6, validate=True).cpu().numpy()
    assert ptr.tolist() == [0, 2, 2, 5, 5, 6, 6]      # empty graphs 1, 3, 5 (trailing) are zero-length ranges


# ------------------------------------------------------------------------------------------------------------------
# global exchange
# ------------------------------------------------------------------------------------------------------------------
def _load_exchange(ex, w):
    rep = ex._node_to_graph_representation_layer
    for var, m in zip(rep._transformation_mlp.kernels, w["transformation_mlp"]):
        var.assign(m)
    if "scoring_mlp" in w:
        for var, m in zip(rep._scoring_mlp.kernels, w["scoring_mlp"]):
            var.assign(m)
    if "gru_kernel" in w:
        ex._gru_kernel.assign(w["gru_kernel"])
        ex._gru_recurrent_kernel.assign(w["gru_recurrent_kernel"])
        ex._gru_bias.assign(w["gru_bias"])
    if "mlp" in w:
        for var, m in zip(ex._mlp.kernels, w["mlp"]):
            var.assign(m)


@pytest.mark.parametrize("mode", ["mean", "gru", "mlp"])
@pytest.mark.parametrize("weighting,V,G,H", [("softmax", 900, 50, 32), ("softmax", 6000, 4, 128),
                                             ("sigmoid", 900, 50, 32), ("sigmoid", 6000, 400, 128)])
def test_graph_global_exchange(mode, weighting, V, G, H):
    """graph_global_exchange.py:106-183, inference mode.  Softmax weights sum to 1 per graph, so PPI-sized graphs (1500
    nodes) stay O(1); sigmoid weights sum ~0.5 per NODE (the reference uses them on molecule-sized graphs: with 1500-node
    graphs the graph representation reaches ~1e2 and saturates the GRU / MLP that follow, where 1e-5 of the OUTPUT scale is
    below what float32 itself delivers), hence QM9-sized graphs (15 nodes) for that weighting."""
    _need_gpu()
    from tf2_gnn_b200.layers import (GraphGlobalExchangeInput, GraphGlobalGRUExchange, GraphGlobalMeanExchange,
                                     GraphGlobalMLPExchange)
    rng = np.random.default_rng(V + H)
    x = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    n2g = random_n2g(rng, V, G)
    cls = {"mean": GraphGlobalMeanExchange, "gru": GraphGlobalGRUExchange, "mlp": GraphGlobalMLPExchange}[mode]
    ex = cls(hidden_dim=H, weighting_fun=weighting, num_heads=4, dropout_rate=0.2)
    ex.build(GraphGlobalExchangeInput((None, H), (None,), ()))
    w = mo.make_exchange_weights(mode, H, 4, rng, weighting)
    _load_exchange(ex, w)
    out = ex(GraphGlobalExchangeInput(torch.from_numpy(x).cuda(), torch.from_numpy(n2g).cuda(), G), training=False)
    ref = mo.graph_global_exchange(mode, x, n2g, G, w, H, 4, weighting, dtype=np.float64)
    close(out.cpu().numpy(), ref, what=f"exchange {mode}/{weighting}")


def _build_gnn(params, F, L, rng, with_exchange):
    from tf2_gnn_b200.layers import GNN, GNNInput
    kind, H = params["message_calculation_class"], params["hidden_dim"]
    gnn = GNN(params)
    gnn.build(GNNInput((None, F), tuple((None, 2) for _ in range(L)), (None,), ()))
    w = {"initial_projection": mo.glorot_uniform(rng, (F, H)), "mp": [], "dense": {}, "layernorm": [], "exchange": {}}
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
        if str(i) in gnn._global_exchange_layers:
            we = mo.make_exchange_weights(params["global_exchange_mode"], H, params["global_exchange_num_heads"], rng,
                                          params["global_exchange_weighting_fun"])
            _load_exchange(gnn._global_exchange_layers[str(i)], we)
            w["exchange"][i] = we
    return gnn, w


def teacher_forced_stack_check(gnn, params, w, feats, adjs, n2g, G):
    """Replays GNN._internal_call (gnn.py:276-329) stage by stage on the GPU.  Every stage is compared with the float64
    oracle of THAT stage applied to the GPU's own input of the stage, at the north_star's 1e-5: errors of earlier stages
    do not hide in (or get blamed on) later ones, so no loosened end-to-end tolerance is needed.  The replay is then
    shown to be the same computation as the real call (bitwise equal result)."""
    from tf2_gnn_b200.layers import GraphGlobalExchangeInput, MessagePassingInput, node_ops
    from tf2_gnn_b200.runtime import PreparedBatch
    kind = params["message_calculation_class"]
    f = torch.from_numpy(feats).cuda()
    adj_dev = tuple(torch.from_numpy(a).cuda() for a in adjs)
    n2g_dev = torch.from_numpy(n2g).cuda()
    prepared = PreparedBatch(adj_dev, feats.shape[0])
    act_init = mo.get_activation_function(params["initial_node_representation_activation"])
    act_dense = mo.get_activation_function(params["dense_intermediate_layer_activation"])
    f64 = lambda t: t.cpu().numpy().astype(np.float64)
    cur = gnn._initial_projection_layer(f)
    close(f64(cur), act_init(feats.astype(np.float64) @ w["initial_projection"].astype(np.float64)), what="projection")
    last = cur
    for i, mp in enumerate(gnn._mp_layers):
        if i % params["residual_every_num_layers"] == 0:
            tmp = cur
            if i > 0:
                new = node_ops.residual_average(cur, last)
                close(f64(new), (f64(cur) + f64(last)) / 2, what=f"residual {i}")
                cur = new
            last = tmp
        out = mp(MessagePassingInput(cur, adj_dev), prepared=prepared)
        close(f64(out), mo.message_passing_forward(kind, params, w["mp"][i], f64(cur), adjs, dtype=np.float64),
              what=f"message passing {i}")
        cur = out
        if i and i % params["global_exchange_every_num_layers"] == 0:
            out = gnn._global_exchange_layers[str(i)](GraphGlobalExchangeInput(cur, n2g_dev, G))
            close(f64(out), mo.graph_global_exchange(params["global_exchange_mode"], f64(cur), n2g, G, w["exchange"][i],
                                                     params["hidden_dim"], params["global_exchange_num_heads"],
                                                     params["global_exchange_weighting_fun"], dtype=np.float64),
                  what=f"exchange {i}")
            cur = out
        if params["use_inter_layer_layernorm"]:
            g, b = w["layernorm"][i]
            out = gnn._inter_layer_layernorms[i](cur)
            close(f64(out), mo.layer_norm(f64(cur), g.astype(np.float64), b.astype(np.float64)), what=f"layernorm {i}")
            cur = out
        if i % params["dense_every_num_layers"] == 0:
            out = gnn._dense_layers[str(i)](cur)
            close(f64(out), act_dense(f64(cur) @ w["dense"][i].astype(np.float64)), what=f"dense {i}")
            cur = out
    return cur


@pytest.mark.parametrize("mode,weighting", [("gru", "softmax"), ("mlp", "sigmoid"), ("mean", "softmax")])
def test_gnn_default_hyperparameters_run_with_global_exchange(mode, weighting):
    """GNN.get_default_hyperparameters() has global_exchange_every_num_layers = 2 (gnn.py:66): the default-configured GNN
    (and QM9_RGCN.json, 8 layers) must run.  Stage-wise parity at 1e-5 + the replay equals the real call bitwise."""
    _need_gpu()
    from tf2_gnn_b200.layers import GNN, GNNInput
    rng = np.random.default_rng(3)
    V, F, L, G = 800, 20, 3, 30
    params = GNN.get_default_hyperparameters()       # rgcn, 4 layers, exchange every 2, hidden 16
    params.update(hidden_dim=32, global_exchange_mode=mode, global_exchange_weighting_fun=weighting,
                  use_inter_layer_layernorm=True)
    adjs = [rng.integers(0, V, size=(3000, 2)).astype(np.int32) for _ in range(L)]
    feats = rng.uniform(-1, 1, (V, F)).astype(np.float32)
    n2g = random_n2g(rng, V, G)
    gnn, w = _build_gnn(params, F, L, rng, True)
    assert sorted(gnn._global_exchange_layers) == ["2"]
    final = teacher_forced_stack_check(gnn, params, w, feats, adjs, n2g, G)
    inp = GNNInput(torch.from_numpy(feats).cuda(), tuple(torch.from_numpy(a).cuda() for a in adjs),
                   torch.from_numpy(n2g).cuda(), G)
    out, reps = gnn(inp, training=False, return_all_representations=True)
    assert torch.equal(out, final)
    assert len(reps) == params["num_layers"] + 1
    # end to end against the float64 oracle: 4 message-passing layers + exchange + layernorm + dense in sequence; the
    # stage-wise bound above is the parity statement, this is a sanity bound on the accumulated drift
    ref, _ = mo.gnn_forward(params, w, feats, adjs, dtype=np.float64, node_to_graph_map=n2g, num_graphs=G)
    close(out.cpu().numpy(), ref, tol=1e-4, what="whole stack (accumulated over 12 stages)")


def test_integration_md_snippet_runs():
    """INTEGRATION.md §3: defaults + hidden_dim=320 (ADVICE r1: this used to raise NotImplementedError)."""
    _need_gpu()
    from tf2_gnn_b200.layers import GNN, GNNInput
    rng = np.random.default_rng(0)
    V = 500
    params = GNN.get_default_hyperparameters("rgcn")
    params["hidden_dim"] = 320
    gnn = GNN(params)
    node_features = torch.from_numpy(rng.uniform(-1, 1, (V, 50)).astype(np.float32)).cuda()
    adjacency_lists = tuple(torch.from_numpy(rng.integers(0, V, size=(2000, 2)).astype(np.int32)).cuda() for _ in range(3))
    node_to_graph_map = torch.from_numpy(np.sort(rng.integers(0, 4, size=V)).astype(np.int32)).cuda()
    out = gnn(GNNInput(node_features, adjacency_lists, node_to_graph_map, 4), training=False)
    assert tuple(out.shape) == (V, 320) and torch.isfinite(out).all()


# ------------------------------------------------------------------------------------------------------------------
# training-time glue
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("act", [None, "relu", "tanh", "gelu", "elu"])
@pytest.mark.parametrize("V,K,N,bias", [(300, 50, 64, False), (9000, 64, 96, True), (1000, 33, 7, True)])
def test_dense_backward(act, V, K, N, bias):
    _need_gpu()
    from tf2_gnn_b200.layers import node_ops
    from tf2_gnn_b200.utils.param_helpers import get_activation_function
    rng = np.random.default_rng(V + N)
    x = rng.uniform(-1, 1, (V, K)).astype(np.float32)
    W = mo.glorot_uniform(rng, (K, N))
    b = rng.uniform(-.3, .3, N).astype(np.float32) if bias else None
    R = rng.uniform(-1, 1, (V, N)).astype(np.float32)
    xt = torch.from_numpy(x).cuda().requires_grad_()
    Wt = torch.from_numpy(W).cuda().requires_grad_()
    bt = torch.from_numpy(b).cuda().requires_grad_() if bias else None
    y = node_ops.dense(xt, Wt, bt, get_activation_function(act) if act else None)
    (y * torch.from_numpy(R).cuda()).sum().backward()
    x64 = torch.from_numpy(x).double().requires_grad_()
    W64 = torch.from_numpy(W).double().requires_grad_()
    b64 = torch.from_numpy(b).double().requires_grad_() if bias else None
    z = x64 @ W64 + (b64 if bias else 0)
    fn = {None: lambda t: t, "relu": torch.relu, "tanh": torch.tanh, "elu": torch.nn.functional.elu,
          "gelu": lambda t: torch.nn.functional.gelu(t, approximate="tanh")}[act]
    (fn(z) * torch.from_numpy(R).double()).sum().backward()
    close(y.detach().cpu().numpy(), fn(z).detach().numpy(), what="dense fwd")
    close(xt.grad.cpu().numpy(), x64.grad.numpy(), what="dense grad_x")
    close(Wt.grad.cpu().numpy(), W64.grad.numpy(), what="dense grad_W")
    if bias:
        close(bt.grad.cpu().numpy(), b64.grad.numpy(), what="dense grad_bias")


@pytest.mark.parametrize("V,H", [(500, 64), (20000, 320), (77, 7)])
def test_layer_norm_backward(V, H):
    _need_gpu()
    from tf2_gnn_b200.layers import node_ops
    rng = np.random.default_rng(V)
    x = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    g = rng.uniform(0.5, 1.5, H).astype(np.float32)
    b = rng.uniform(-.2, .2, H).astype(np.float32)
    R = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    xt, gt, bt = (torch.from_numpy(a).cuda().requires_grad_() for a in (x, g, b))
    y = node_ops.layer_norm(xt, gt, bt, 1e-3)
    (y * torch.from_numpy(R).cuda()).sum().backward()
    x64, g64, b64 = (torch.from_numpy(a).double().requires_grad_() for a in (x, g, b))
    y64 = torch.nn.functional.layer_norm(x64, (H,), g64, b64, eps=1e-3)
    (y64 * torch.from_numpy(R).double()).sum().backward()
    close(y.detach().cpu().numpy(), y64.detach().numpy(), what="ln fwd")
    close(xt.grad.cpu().numpy(), x64.grad.numpy(), what="ln grad_x")
    close(gt.grad.cpu().numpy(), g64.grad.numpy(), what="ln grad_gamma")
    close(bt.grad.cpu().numpy(), b64.grad.numpy(), what="ln grad_beta")


def test_dropout_statistics_determinism_and_backward():
    """tf.nn.dropout semantics (gnn.py:285-289): keep prob 1-rate, kept values scaled by 1/(1-rate); mask is a function of
    (seed, offset, index) so the backward pass regenerates it."""
    _need_gpu()
    from tf2_gnn_b200.layers import node_ops
    n, rate = 4_000_003, 0.2
    x = torch.ones(n, device="cuda").requires_grad_()
    st = node_ops.DropoutState(seed=42)
    y = node_ops.dropout(x, rate, st)
    kept = (y != 0)
    frac = kept.float().mean().item()
    assert abs(frac - (1 - rate)) < 5 * np.sqrt(rate * (1 - rate) / n)
    assert torch.allclose(y[kept], torch.full_like(y[kept], 1 / (1 - rate)))
    y.sum().backward()
    assert torch.equal(x.grad, y.detach())            # d/dx = mask / (1 - rate): the same mask
    y_again = node_ops.dropout(torch.ones(n, device="cuda"), rate, node_ops.DropoutState(seed=42))
    assert torch.equal(y_again, y.detach())           # reproducible from the seed
    y_next = node_ops.dropout(torch.ones(n, device="cuda"), rate, st)
    assert not torch.equal(y_next, y.detach())        # the stream advances between calls
    y_other = node_ops.dropout(torch.ones(n, device="cuda"), rate, node_ops.DropoutState(seed=43))
    assert not torch.equal(y_other, y.detach())
    # chi-square over 4-bit windows of the keep pattern: no lane / word bias
    bits = kept[: n // 4 * 4].view(-1, 4).int()
    hist = torch.bincount((bits * torch.tensor([1, 2, 4, 8], device="cuda")).sum(1), minlength=16).double().cpu().numpy()
    p = np.array([(1 - rate) ** bin(i).count("1") * rate ** (4 - bin(i).count("1")) for i in range(16)])
    chi2 = ((hist - p * hist.sum()) ** 2 / (p * hist.sum())).sum()
    assert chi2 < 60.0, chi2                           # 15 dof: P(chi2 > 60) ~ 2e-7
    assert node_ops.dropout(x, 0.0, st) is x


def _torch_stack_reference(params, w, feats, adjs):
    """float64 torch restatement of gnn.py:276-329 for an RGCN stack without exchange (differentiable)."""
    t = lambda a: torch.from_numpy(np.asarray(a)).double().requires_grad_()
    leaves = {"proj": t(w["initial_projection"]), "mp": [[t(m[0]) for m in wi["edge_mlps"]] for wi in w["mp"]],
              "dense": {i: t(d) for i, d in w["dense"].items()}, "ln": [(t(g), t(b)) for g, b in w["layernorm"]]}
    act = {"tanh": torch.tanh, "relu": torch.relu}
    V = feats.shape[0]
    cur = act[params["initial_node_representation_activation"]](torch.from_numpy(feats).double() @ leaves["proj"])
    last = cur
    for i in range(params["num_layers"]):
        if i % params["residual_every_num_layers"] == 0:
            tmp = cur
            if i > 0:
                cur = (cur + last) / 2
            last = tmp
        agg = torch.zeros((V, params["hidden_dim"]), dtype=torch.float64)
        for a, W in zip(adjs, leaves["mp"][i]):
            src, tgt = torch.from_numpy(a[:, 0]).long(), torch.from_numpy(a[:, 1]).long()
            c = torch.bincount(tgt, minlength=V).double()
            m = (cur[src] @ W) / (c[tgt] + 1e-7)[:, None]
            agg = agg.index_add(0, tgt, m)
        cur = act[params["message_activation_function"]](agg)
        if params["use_inter_layer_layernorm"]:
            g, b = leaves["ln"][i]
            cur = torch.nn.functional.layer_norm(cur, (params["hidden_dim"],), g, b, eps=1e-3)
        if i % params["dense_every_num_layers"] == 0:
            cur = act[params["dense_intermediate_layer_activation"]](cur @ leaves["dense"][i])
    return cur, leaves


@pytest.mark.parametrize("variant", ["ppi_rgcn", "qm9_like"])
def test_training_step_of_an_rgcn_stack_matches_float64_autograd(variant):
    """One optimizer step (SGD) of a PPI_RGCN.json-shaped stack (4 RGCN layers, tanh projection, no dense / residual) and of
    a stack with residuals + LayerNorm + Dense: every variable's gradient vs float64 autograd of the reference op order
    (models/graph_task_model.py:338-365 computes them with tf.GradientTape)."""
    _need_gpu()
    from tf2_gnn_b200.layers import GNN, GNNInput
    rng = np.random.default_rng(11)
    V, F, H, L = 700, 50, 64, 3
    params = GNN.get_default_hyperparameters("rgcn")
    params.update(hidden_dim=H, num_layers=4, global_exchange_every_num_layers=10000, layer_input_dropout_rate=0.0)
    if variant == "ppi_rgcn":
        params.update(dense_every_num_layers=10000, residual_every_num_layers=10000)
    else:
        params.update(dense_every_num_layers=2, residual_every_num_layers=2, use_inter_layer_layernorm=True)
    adjs = [rng.integers(0, V, size=(4000, 2)).astype(np.int32) for _ in range(L)]
    feats = rng.uniform(-1, 1, (V, F)).astype(np.float32)
    R = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    gnn, w = _build_gnn(params, F, L, rng, False)
    for v in gnn.variables:
        v.requires_grad_(True)
    inp = GNNInput(torch.from_numpy(feats).cuda(), tuple(torch.from_numpy(a).cuda() for a in adjs),
                   torch.zeros(V, dtype=torch.int32).cuda(), 1)
    out = gnn(inp, training=True)          # dropout rate 0: identity, so the step is comparable
    loss = (out * torch.from_numpy(R).cuda()).sum()
    loss.backward()
    ref_out, leaves = _torch_stack_reference(params, w, feats, adjs)
    (ref_out * torch.from_numpy(R).double()).sum().backward()
    close(out.detach().cpu().numpy(), ref_out.detach().numpy(), tol=5e-5, what="stack output (4 layers accumulated)")
    # Gradients flow back through up to 4 message-passing layers + glue: each stage meets 1e-5 on its own (tested above and
    # in test_gpu_parity), the chain is given the number of stages it passes through.
    tol = 1e-5 * (2 * params["num_layers"] + 2)
    named = {v.name: v for v in gnn.variables}
    got_proj = gnn._initial_projection_layer.kernel.grad
    assert got_proj is not None, "gradient did not reach the initial projection (truncated autograd chain)"
    close(got_proj.cpu().numpy(), leaves["proj"].grad.numpy(), tol=tol, what="grad initial projection")
    for i, mp in enumerate(gnn._mp_layers):
        for l, mlp in enumerate(mp._edge_type_mlps):
            g = mlp.layers[0].grad
            assert g is not None
            close(g.cpu().numpy(), leaves["mp"][i][l].grad.numpy(), tol=tol, what=f"grad W layer {i} type {l}")
    for i, d in gnn._dense_layers.items():
        close(d.kernel.grad.cpu().numpy(), leaves["dense"][int(i)].grad.numpy(), tol=tol, what=f"grad dense {i}")
    for i, ln in enumerate(gnn._inter_layer_layernorms):
        close(ln.gamma.grad.cpu().numpy(), leaves["ln"][i][0].grad.numpy(), tol=tol, what=f"grad gamma {i}")
        close(ln.beta.grad.cpu().numpy(), leaves["ln"][i][1].grad.numpy(), tol=tol, what=f"grad beta {i}")
    # the SGD step itself: w <- w - lr * g on device tensors, loss must go down for a small step
    lr = 1e-3
    with torch.no_grad():
        for v in gnn.variables:
            if v.grad is not None:
                v.value -= lr * v.grad
    out2 = gnn(inp, training=False)
    assert (out2 * torch.from_numpy(R).cuda()).sum().item() < loss.item()
    assert len(named) == len(gnn.variables)


def test_training_with_dropout_runs_and_is_reproducible():
    """Every PPI_*.json sets gnn_layer_input_dropout_rate 0.1-0.2: a training step must run (round 1 raised)."""
    _need_gpu()
    from tf2_gnn_b200.layers import GNN, GNNInput
    rng = np.random.default_rng(2)
    V, F, L = 400, 30, 3
    params = GNN.get_default_hyperparameters("rgcn")
    params.update(hidden_dim=32, global_exchange_every_num_layers=10000, layer_input_dropout_rate=0.1,
                  b200_dropout_seed=7)
    adjs = tuple(torch.from_numpy(rng.integers(0, V, size=(2000, 2)).astype(np.int32)).cuda() for _ in range(L))
    feats = torch.from_numpy(rng.uniform(-1, 1, (V, F)).astype(np.float32)).cuda()
    outs = []
    for _ in range(2):
        torch.manual_seed(0)
        gnn = GNN(params)
        inp = GNNInput(feats, adjs, torch.zeros(V, dtype=torch.int32).cuda(), 1)
        gnn.build(GNNInput((None, F), tuple((None, 2) for _ in range(L)), (None,), ()))
        for v in gnn.variables:
            v.requires_grad_(True)
        o = gnn(inp, training=True)
        o.sum().backward()
        assert all(v.grad is not None and torch.isfinite(v.grad).all() for v in gnn.variables)
        outs.append(o.detach().clone())
        o_eval = gnn(inp, training=False)
        assert not torch.equal(o_eval, o.detach())     # dropout really dropped something
    assert torch.equal(outs[0], outs[1])               # same seed, same weights -> same masks


@pytest.mark.parametrize("K,act", [(4, "relu"), (3, "tanh")])
def test_rgat_training_matches_float64_autograd(K, act):
    """RGAT trains through the reference's op order (layers/differentiable.py: gather -> scores -> segment softmax over all
    types -> weighted sum), every op with its adjoint kernel: output and gradients vs float64 autograd of rgat.py:91-163."""
    _need_gpu()
    from tf2_gnn_b200.layers import MessagePassingInput, get_message_passing_class
    rng = np.random.default_rng(K)
    V, D, H, L = 250, 20, 24, 3
    d = H // K
    adjs = [rng.integers(0, V, size=(1200, 2)).astype(np.int32) for _ in range(L - 1)] + [np.zeros((0, 2), np.int32)]
    cls = get_message_passing_class("rgat")
    p = cls.get_default_hyperparameters()
    p.update(hidden_dim=H, num_heads=K, message_activation_function=act)
    w = mo.make_weights("rgat", p, D, L, rng)
    layer = cls(p)
    layer.build(MessagePassingInput((None, D), tuple((None, 2) for _ in range(L))))
    layer.set_weights_from_oracle_dict(w)
    for v in layer.variables:
        v.requires_grad_(True)
    h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    R = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    ht = torch.from_numpy(h).cuda().requires_grad_()
    out = layer(MessagePassingInput(ht, tuple(torch.from_numpy(a).cuda() for a in adjs)))
    (out * torch.from_numpy(R).cuda()).sum().backward()
    # float64 reference
    t = lambda a: torch.from_numpy(np.asarray(a)).double().requires_grad_()
    h64 = t(h)
    Ws, As = [t(x) for x in w["edge_kernels"]], [t(x) for x in w["edge_attention"]]
    msgs, scs, ids = [], [], []
    for l, a in enumerate(adjs):
        src, tgt = torch.from_numpy(a[:, 0]).long(), torch.from_numpy(a[:, 1]).long()
        ps = (h64[src] @ Ws[l]).reshape(-1, K, d)
        pt = (h64[tgt] @ Ws[l]).reshape(-1, K, d)
        sc = torch.nn.functional.leaky_relu(torch.einsum("vki,ki->vk", torch.cat([ps, pt], -1), As[l]), 0.2)
        msgs.append(ps); scs.append(sc); ids.append(tgt)
    M, S, T = torch.cat(msgs), torch.cat(scs), torch.cat(ids)
    mx = torch.full((V, K), -1e300, dtype=torch.float64).scatter_reduce(0, T[:, None].expand(-1, K), S, reduce="amax")
    e = torch.exp(S - mx[T])
    Z = torch.zeros((V, K), dtype=torch.float64).index_add(0, T, e)
    alpha = e / Z[T]
    agg = torch.zeros((V, K, d), dtype=torch.float64).index_add(0, T, alpha[:, :, None] * M).reshape(V, H)
    ref = {"relu": torch.relu, "tanh": torch.tanh}[act](agg)
    (ref * torch.from_numpy(R).double()).sum().backward()
    close(out.detach().cpu().numpy(), ref.detach().numpy(), what="rgat forward")
    tol = 3e-5
    close(ht.grad.cpu().numpy(), h64.grad.numpy(), tol=tol, what="rgat grad_h")
    for l in range(L):
        gW = Ws[l].grad.numpy() if Ws[l].grad is not None else np.zeros_like(w["edge_kernels"][l])
        gA = As[l].grad.numpy() if As[l].grad is not None else np.zeros_like(w["edge_attention"][l])
        close(layer._edge_type_to_message_computation_layer[l].grad.cpu().numpy(), gW, tol=tol, what=f"rgat grad W {l}")
        close(layer._edge_type_to_attention_parameters[l].grad.cpu().numpy(), gA, tol=tol, what=f"rgat grad a {l}")


@pytest.mark.parametrize("mode,weighting", [("gru", "softmax"), ("mlp", "sigmoid"), ("mean", "softmax")])
def test_global_exchange_training_matches_float64_autograd(mode, weighting):
    """GraphGlobal{GRU,MLP,Mean}Exchange differentiable (graph_global_exchange.py:83-183): gradients of the node states and of
    every exchange weight (scoring / transformation MLPs, GRU cell, MLP) vs float64 autograd."""
    _need_gpu()
    from tf2_gnn_b200.layers import (GraphGlobalExchangeInput, GraphGlobalGRUExchange, GraphGlobalMeanExchange,
                                     GraphGlobalMLPExchange)
    rng = np.random.default_rng(len(mode))
    V, G, H, K = 400, 25, 32, 4
    x = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    n2g = random_n2g(rng, V, G)
    R = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    cls = {"mean": GraphGlobalMeanExchange, "gru": GraphGlobalGRUExchange, "mlp": GraphGlobalMLPExchange}[mode]
    ex = cls(hidden_dim=H, weighting_fun=weighting, num_heads=K, dropout_rate=0.0)
    ex.build(GraphGlobalExchangeInput((None, H), (None,), ()))
    w = mo.make_exchange_weights(mode, H, K, rng, weighting)
    _load_exchange(ex, w)
    for v in ex.variables:
        v.requires_grad_(True)
    xt = torch.from_numpy(x).cuda().requires_grad_()
    # training=False: no dropout inside the readout MLPs (their class default rate is 0.2), gradients still recorded
    out = ex(GraphGlobalExchangeInput(xt, torch.from_numpy(n2g).cuda(), G), training=False)
    (out * torch.from_numpy(R).cuda()).sum().backward()
    # float64 reference
    t = lambda a: torch.from_numpy(np.asarray(a)).double().requires_grad_()
    x64 = t(x)
    ids = torch.from_numpy(n2g).long()
    sm, tm = [t(m) for m in w["scoring_mlp"]], [t(m) for m in w["transformation_mlp"]]
    scores = torch.relu(x64 @ sm[0]) @ sm[1]
    if weighting == "sigmoid":
        wts = torch.sigmoid(scores)
    else:
        mx = torch.full((G, K), -1e300, dtype=torch.float64).scatter_reduce(0, ids[:, None].expand(-1, K), scores, reduce="amax")
        e = torch.exp(scores - mx[ids])
        wts = e / torch.zeros((G, K), dtype=torch.float64).index_add(0, ids, e)[ids]
    reprs = torch.relu(torch.relu(x64 @ tm[0]) @ tm[1]).reshape(V, K, H // K)
    g = torch.zeros((G, K, H // K), dtype=torch.float64).index_add(0, ids, wts[:, :, None] * reprs).reshape(G, H)
    per_node = g[ids]
    leaves = {"scoring": sm, "transformation": tm}
    if mode == "mean":
        ref = (x64 + per_node) / 2
    elif mode == "gru":
        Kk, U, b = t(w["gru_kernel"]), t(w["gru_recurrent_kernel"]), t(w["gru_bias"])
        leaves["gru"] = [Kk, U, b]
        gx, gh = per_node @ Kk + b[0], x64 @ U + b[1]
        z = torch.sigmoid(gx[:, :H] + gh[:, :H])
        r = torch.sigmoid(gx[:, H:2 * H] + gh[:, H:2 * H])
        hh = torch.tanh(gx[:, 2 * H:] + r * gh[:, 2 * H:])
        ref = z * x64 + (1 - z) * hh
    else:
        mm = [t(m) for m in w["mlp"]]
        leaves["mlp"] = mm
        ref = torch.relu(torch.cat([per_node, x64], -1) @ mm[0]) @ mm[1]
    (ref * torch.from_numpy(R).double()).sum().backward()
    close(out.detach().cpu().numpy(), ref.detach().numpy(), what=f"exchange {mode} forward")
    tol = 3e-5
    close(xt.grad.cpu().numpy(), x64.grad.numpy(), tol=tol, what=f"exchange {mode} grad_x")
    rep = ex._node_to_graph_representation_layer
    for var, leaf in zip(rep._scoring_mlp.kernels, sm):
        close(var.grad.cpu().numpy(), leaf.grad.numpy(), tol=tol, what="grad scoring MLP")
    for var, leaf in zip(rep._transformation_mlp.kernels, tm):
        close(var.grad.cpu().numpy(), leaf.grad.numpy(), tol=tol, what="grad transformation MLP")
    if mode == "gru":
        for var, leaf in zip((ex._gru_kernel, ex._gru_recurrent_kernel, ex._gru_bias), leaves["gru"]):
            close(var.grad.cpu().numpy(), leaf.grad.numpy(), tol=tol, what="grad GRU")
    if mode == "mlp":
        for var, leaf in zip(ex._mlp.kernels, leaves["mlp"]):
            close(var.grad.cpu().numpy(), leaf.grad.numpy(), tol=tol, what="grad exchange MLP")


def test_default_gnn_trains_end_to_end():
    """GNN.get_default_hyperparameters() (RGCN + GRU global exchange every 2 layers, exchange dropout 0.2) takes a training
    step: every variable receives a finite gradient (round 1: forward raised; earlier this round: exchange had no backward)."""
    _need_gpu()
    from tf2_gnn_b200.layers import GNN, GNNInput
    rng = np.random.default_rng(0)
    V, F, L, G = 300, 12, 2, 10
    params = GNN.get_default_hyperparameters()
    params.update(hidden_dim=32, layer_input_dropout_rate=0.1)
    gnn = GNN(params)
    gnn.build(GNNInput((None, F), tuple((None, 2) for _ in range(L)), (None,), ()))
    for v in gnn.variables:
        v.requires_grad_(True)
    inp = GNNInput(torch.from_numpy(rng.uniform(-1, 1, (V, F)).astype(np.float32)).cuda(),
                   tuple(torch.from_numpy(rng.integers(0, V, size=(1500, 2)).astype(np.int32)).cuda() for _ in range(L)),
                   torch.from_numpy(random_n2g(rng, V, G)).cuda(), G)
    out = gnn(inp, training=True)
    out.sum().backward()
    missing = [v.name for v in gnn.variables if v.grad is None or not torch.isfinite(v.grad).all()]
    assert not missing, missing


def _torch_literal_reference(kind, p, w, h, adjs):
    """float64 torch restatement of message_passing.py:95-218 + gnn_edge_mlp.py:84-107 / gnn_film.py:83-108 /
    rgin.py:88-106 (differentiable)."""
    t = lambda a: torch.from_numpy(np.asarray(a)).double().requires_grad_()
    V, H = h.shape[0], p["hidden_dim"]
    leaves = {"h": t(h), "edge": [[t(m) for m in mats] for mats in w["edge_mlps"]]}
    if kind == "gnn_film":
        leaves["film"] = [[t(m) for m in mats] for mats in w["film_mlps"]]
    if kind == "rgin" and w.get("aggr_mlp") is not None:
        leaves["aggr"] = [t(m) for m in w["aggr_mlp"]]
    acts = {"relu": torch.relu, "tanh": torch.tanh, "leaky_relu": lambda x: torch.nn.functional.leaky_relu(x, 0.2),
            "elu": torch.nn.functional.elu, "gelu": lambda x: torch.nn.functional.gelu(x, approximate="tanh")}
    act = acts[p["message_activation_function"]]

    def mlp(x, ws):
        for W in ws[:-1]:
            x = torch.relu(x @ W)
        return x @ ws[-1]

    msgs, ids = [], []
    for l, a in enumerate(adjs):
        src, tgt = torch.from_numpy(a[:, 0]).long(), torch.from_numpy(a[:, 1]).long()
        hs, ht = leaves["h"][src], leaves["h"][tgt]
        x = torch.cat([hs, ht], 1) if p["use_target_state_as_input"] else hs
        m = mlp(x, leaves["edge"][l])
        if p["normalize_by_num_incoming"]:
            c = torch.bincount(tgt, minlength=V).double()
            m = m / (c[tgt] + 1e-7)[:, None]
        if kind == "gnn_film":
            f = mlp(ht, leaves["film"][l])
            m = f[:, :H] * m + f[:, H:]
        msgs.append(m)
        ids.append(tgt)
    M, T = torch.cat(msgs, 0), torch.cat(ids, 0)
    before = bool(p.get("message_activation_before_aggregation", False)) and kind != "rgin"
    if before:
        M = act(M)
    agg_name = p["aggregation_function"]
    if agg_name == "max":
        out = torch.full((V, H), float(np.finfo(np.float32).min), dtype=torch.float64)
        out = out.scatter_reduce(0, T[:, None].expand(-1, H), M, reduce="amax", include_self=True)
    else:
        out = torch.zeros((V, H), dtype=torch.float64).index_add(0, T, M)
        cnt = torch.bincount(T, minlength=V).double().clamp(min=1)
        if agg_name == "mean":
            out = out / cnt[:, None]
        elif agg_name == "sqrt_n":
            out = out / cnt.sqrt()[:, None]
    if "aggr" in leaves:
        out = mlp(out, leaves["aggr"])
    if not before:
        out = act(out)
    return out, leaves


@pytest.mark.parametrize("kind,extra", [
    ("gnn_edge_mlp", {}),                                                              # defaults: 1 hidden layer, target input
    ("gnn_edge_mlp", dict(num_edge_MLP_hidden_layers=2, normalize_by_num_incoming=True, aggregation_function="mean",
                          message_activation_function="gelu")),
    ("rgcn", dict(aggregation_function="max")),
    ("rgcn", dict(message_activation_before_aggregation=True, message_activation_function="tanh",
                  aggregation_function="sqrt_n")),
    ("rgin", dict(num_aggr_MLP_hidden_layers=1, normalize_by_num_incoming=True)),     # PPI_RGIN.json shape
    ("rgin", {}),
    ("gnn_film", {}),
    ("gnn_film", dict(use_target_state_as_input=True, normalize_by_num_incoming=True)),  # PPI_GNN_FiLM.json shape
])
def test_training_through_the_differentiable_generic_path(kind, extra):
    """Variants without a fused backward train through the reference's literal op order (layers/differentiable.py):
    output and every gradient (node states, edge MLPs, FiLM MLPs, aggregation MLP) against float64 autograd."""
    _need_gpu()
    from tf2_gnn_b200.layers import MessagePassingInput, get_message_passing_class
    rng = np.random.default_rng(4)
    V, D, H, L = 300, 24, 32, 3
    adjs = [rng.integers(0, V, size=(1500, 2)).astype(np.int32) for _ in range(L - 1)] + [np.zeros((0, 2), np.int32)]
    cls = get_message_passing_class(kind)
    p = cls.get_default_hyperparameters()
    p["hidden_dim"] = H
    p.update(extra)
    w = mo.make_weights(kind, p, D, L, rng)
    layer = cls(p)
    layer.build(MessagePassingInput((None, D), tuple((None, 2) for _ in range(L))))
    layer.set_weights_from_oracle_dict(w)
    for v in layer.variables:
        v.requires_grad_(True)
    h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    R = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    ht = torch.from_numpy(h).cuda().requires_grad_()
    out = layer(MessagePassingInput(ht, tuple(torch.from_numpy(a).cuda() for a in adjs)))
    ref, leaves = _torch_literal_reference(kind, p, w, h, adjs)
    sentinel = ref.detach() < -1e38              # empty segments of the max aggregation (no gradient flows there)
    Rt = torch.from_numpy(R).double()
    (torch.where(sentinel, torch.zeros_like(ref), ref) * Rt).sum().backward()
    o = out.detach().cpu().double()
    assert torch.equal(o < -1e38, sentinel)
    (torch.where(sentinel.cuda(), torch.zeros_like(out), out) * torch.from_numpy(R).cuda()).sum().backward()
    close(torch.where(sentinel, torch.zeros_like(o), o).numpy(), torch.where(sentinel, torch.zeros_like(ref), ref).detach().numpy(),
          what=f"{kind} forward")
    tol = 3e-5   # gradients pass through 3-5 chained contractions / reductions, each at 1e-5 of its own scale
    close(ht.grad.cpu().numpy(), leaves["h"].grad.numpy(), tol=tol, what=f"{kind} grad_h")
    for l, mlp in enumerate(layer._edge_type_mlps):
        for j, var in enumerate(mlp.layers):
            close(var.grad.cpu().numpy(), leaves["edge"][l][j].grad.numpy() if leaves["edge"][l][j].grad is not None
                  else np.zeros_like(w["edge_mlps"][l][j]), tol=tol, what=f"{kind} grad edge MLP {l}/{j}")
    if kind == "gnn_film":
        for l, mlp in enumerate(layer._edge_type_film_layer_computations):
            g = leaves["film"][l][0].grad
            close(mlp.layers[0].grad.cpu().numpy(), g.numpy() if g is not None else np.zeros_like(w["film_mlps"][l][0]),
                  tol=tol, what=f"{kind} grad FiLM {l}")
    if "aggr" in leaves:
        for j, var in enumerate(layer._aggregation_mlp):
            close(var.grad.cpu().numpy(), leaves["aggr"][j].grad.numpy(), tol=tol, what=f"{kind} grad aggregation MLP {j}")


# ------------------------------------------------------------------------------------------------------------------
# round-1 ADVICE regressions
# ------------------------------------------------------------------------------------------------------------------
def test_segment_max_of_negative_zero():
    """atomic max on floats: a segment whose only message is -0.0 must give (-)0, not the -FLT_MAX identity."""
    _need_gpu()
    from tf2_gnn_b200.utils.param_helpers import get_aggregation_function
    data = torch.tensor([[-0.0, 1.0], [-0.0, -2.0], [3.0, -0.0]], device="cuda")
    ids = torch.tensor([0, 0, 2], dtype=torch.int32, device="cuda")
    out = get_aggregation_function("max")(data, ids, 3).cpu().numpy()
    assert out[0, 0] == 0.0 and out[0, 1] == 1.0
    assert out[2, 0] == 3.0 and out[2, 1] == 0.0
    assert (out[1] < -3e38).all()                      # empty segment keeps TF's identity


def test_gelu_backward_survives_scratch_regrowth_in_the_nested_forward(monkeypatch):
    """rgcn_bwd + gelu recomputes the pre-activation through the forward entry point, which on the pipelined path takes
    and frees its own large chunk buffer; the backward must not hold a pointer into memory that nested call frees."""
    _need_gpu()
    monkeypatch.setenv("TFGNN_B200_PIPE_CHUNK_ROWS", "128")     # forces the pipelined path with a large chunk buffer
    monkeypatch.setenv("TFGNN_B200_FUSED", "0")
    from tf2_gnn_b200.layers import MessagePassingInput, get_message_passing_class
    rng = np.random.default_rng(9)
    V, D, H, L = 1000, 36, 48, 3                                 # D % 32 != 0: not the fused kernel
    adjs = [rng.integers(0, V, size=(5000, 2)).astype(np.int32) for _ in range(L)]
    cls = get_message_passing_class("rgcn")
    p = cls.get_default_hyperparameters()
    p.update(hidden_dim=H, message_activation_function="gelu")
    w = mo.make_weights("rgcn", p, D, L, rng)
    layer = cls(p)
    layer.build(MessagePassingInput((None, D), tuple((None, 2) for _ in range(L))))
    layer.set_weights_from_oracle_dict(w)
    for v in layer.variables:
        v.requires_grad_(True)
    h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    R = rng.uniform(-1, 1, (V, H)).astype(np.float32)
    ht = torch.from_numpy(h).cuda().requires_grad_()
    out = layer(MessagePassingInput(ht, tuple(torch.from_numpy(a).cuda() for a in adjs)))
    (out * torch.from_numpy(R).cuda()).sum().backward()
    h64 = torch.from_numpy(h).double().requires_grad_()
    Ws = [torch.from_numpy(m[0]).double().requires_grad_() for m in w["edge_mlps"]]
    agg = torch.zeros((V, H), dtype=torch.float64)
    for a, W in zip(adjs, Ws):
        src, tgt = torch.from_numpy(a[:, 0]).long(), torch.from_numpy(a[:, 1]).long()
        c = torch.bincount(tgt, minlength=V).double()
        agg = agg.index_add(0, tgt, (h64[src] @ W) / (c[tgt] + 1e-7)[:, None])
    ref = torch.nn.functional.gelu(agg, approximate="tanh")
    (ref * torch.from_numpy(R).double()).sum().backward()
    close(out.detach().cpu().numpy(), ref.detach().numpy(), what="gelu fwd")
    close(ht.grad.cpu().numpy(), h64.grad.numpy(), tol=2e-5, what="gelu grad_h (two chained contractions)")
    for l, mlp in enumerate(layer._edge_type_mlps):
        close(mlp.layers[0].grad.cpu().numpy(), Ws[l].grad.numpy(), tol=2e-5, what=f"gelu grad_W {l}")


def test_per_batch_path_makes_no_synchronising_allocations_after_warmup():
    """VERDICT r1 weak #5: every host-input call used to pay cudaMalloc/cudaFree + device syncs (26 ms for a PPI batch).
    With the library's stream-ordered pool, preparing + running a PPI-sized batch from device tensors must cost about its
    kernels: well under 2 ms wall (it was 29-50 ms)."""
    _need_gpu()
    import time
    from tf2_gnn_b200.layers import MessagePassingInput, get_message_passing_class
    from tf2_gnn_b200.runtime import PreparedBatch
    rng = np.random.default_rng(1)
    V, H, L = 8000, 320, 3
    adjs = tuple(torch.from_numpy(rng.integers(0, V, size=(80_000, 2)).astype(np.int32)).cuda() for _ in range(L))
    h = torch.rand((V, H), device="cuda")
    cls = get_message_passing_class("rgcn")
    p = cls.get_default_hyperparameters()
    p["hidden_dim"] = H
    layer = cls(p)
    for _ in range(3):
        pb = PreparedBatch(adjs, V)
        layer(MessagePassingInput(h, adjs), prepared=pb)
        del pb
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = 20
    for _ in range(n):
        pb = PreparedBatch(adjs, V)
        layer(MessagePassingInput(h, adjs), prepared=pb)
        del pb
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) / n * 1e3
    print(f"prepare + layer on a PPI-sized batch: {ms:.3f} ms per batch")
    assert ms < 2.0, ms


@pytest.mark.parametrize("V,H,act,agg", [(50_000, 128, "leaky_relu", "sum"),     # QM9_RGCN.json shape: pairs, 391 tiles
                                         (3000, 256, "relu", "mean"),            # small batch: LayerNorm keeps one CTA per tile
                                         (20_000, 64, "tanh", "sqrt_n"),
                                         (6000, 320, "relu", "sum")])            # H > 256: composed fallback, same result
def test_layernorm_fused_into_the_layer_kernel(V, H, act, agg):
    """tfgnn_b200_rgcn_ln_fwd: LayerNorm in the fused kernel's epilogue (gnn.py:299-321 with use_inter_layer_layernorm) against
    the float64 oracle and against the composed layer + LayerNorm kernels."""
    _need_gpu()
    from tf2_gnn_b200.layers import MessagePassingInput, get_message_passing_class, node_ops
    rng = np.random.default_rng(V + H)
    D, L = H, 3
    adjs = [rng.integers(0, V, size=(3 * V, 2)).astype(np.int32) for _ in range(L)]
    cls = get_message_passing_class("rgcn")
    p = cls.get_default_hyperparameters()
    p.update(hidden_dim=H, message_activation_function=act, aggregation_function=agg)
    w = mo.make_weights("rgcn", p, D, L, rng)
    layer = cls(p)
    layer.build(MessagePassingInput((None, D), tuple((None, 2) for _ in range(L))))
    layer.set_weights_from_oracle_dict(w)
    h = rng.uniform(-1, 1, (V, D)).astype(np.float32)
    g = rng.uniform(0.5, 1.5, H).astype(np.float32)
    b = rng.uniform(-0.2, 0.2, H).astype(np.float32)
    inp = MessagePassingInput(torch.from_numpy(h).cuda(), tuple(torch.from_numpy(a).cuda() for a in adjs))
    gt, bt = torch.from_numpy(g).cuda(), torch.from_numpy(b).cuda()
    fused = layer.call_with_layernorm(inp, gt, bt, 1e-3)
    mp = layer(inp)
    composed = node_ops.layer_norm(mp, gt, bt, 1e-3)
    ref = mo.layer_norm(mp.cpu().numpy().astype(np.float64), g.astype(np.float64), b.astype(np.float64))   # teacher forced
    close(fused.cpu().numpy(), ref, what="fused LayerNorm epilogue")
    close(composed.cpu().numpy(), ref, what="composed LayerNorm")
    fused2 = layer.call_with_layernorm(inp, gt, bt, 1e-3)
    assert torch.equal(fused, fused2)


def test_gnn_stack_uses_the_fused_layernorm_and_matches_the_unfused_stack():
    """QM9_RGCN-shaped stack (LayerNorm after every layer): the call that does not ask for all representations takes the fused
    layer + LayerNorm kernel; its result must agree with the call that does (which composes the ops) to fp32 rounding."""
    _need_gpu()
    from tf2_gnn_b200.layers import GNN, GNNInput
    rng = np.random.default_rng(5)
    V, F, L = 20_000, 15, 3
    params = GNN.get_default_hyperparameters("rgcn")
    params.update(hidden_dim=128, num_layers=4, use_inter_layer_layernorm=True, residual_every_num_layers=2,
                  dense_every_num_layers=32, global_exchange_every_num_layers=10000,
                  message_activation_function="leaky_relu")
    gnn = GNN(params)
    inp = GNNInput(torch.from_numpy(rng.uniform(-1, 1, (V, F)).astype(np.float32)).cuda(),
                   tuple(torch.from_numpy(rng.integers(0, V, size=(60_000, 2)).astype(np.int32)).cuda() for _ in range(L)),
                   torch.zeros(V, dtype=torch.int32).cuda(), 1)
    fused = gnn(inp, training=False)
    composed, reps = gnn(inp, training=False, return_all_representations=True)
    assert all(r is not None for r in reps)
    close(fused.cpu().numpy(), composed.cpu().numpy().astype(np.float64), tol=5e-6, what="fused vs composed stack")


def test_ops_without_a_backward_raise_instead_of_truncating_gradients():
    """ADVICE r1 (medium): an op without a backward must not hand back a tensor without grad_fn.  What is left without one:
    the generic user-plugin MessagePassing.call and the forward-only graph primitives."""
    _need_gpu()
    from tf2_gnn_b200.layers import MessagePassing, MessagePassingInput, node_ops

    class PassSourceStates(MessagePassing):
        def __init__(self):
            super().__init__(super().get_default_hyperparameters())

        def _message_function(self, edge_source_states, edge_target_states, num_incoming_to_node_per_message,
                              edge_type_idx, training):
            return edge_source_states

    rng = np.random.default_rng(0)
    V = 40
    adjs = (torch.from_numpy(rng.integers(0, V, size=(90, 2)).astype(np.int32)).cuda(),)
    h = torch.rand((V, 7), device="cuda", requires_grad=True)
    layer = PassSourceStates()
    with pytest.raises(NotImplementedError):
        layer(MessagePassingInput(h, adjs))
    with torch.no_grad():
        assert tuple(layer(MessagePassingInput(h, adjs)).shape) == (V, 7)
    ptr = node_ops.graph_offsets(torch.zeros(V, dtype=torch.int32, device="cuda"), 1)
    with pytest.raises(NotImplementedError):
        node_ops.segment_softmax(torch.rand((V, 2), device="cuda", requires_grad=True), ptr)
