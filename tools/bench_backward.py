"""Measurement of the backward pass (SURVEY.md §8f-1) at bench.py's workloads: forward and backward device time of one
RGCN, GGNN or GNN-FiLM layer through the autograd hook, CUDA events, inputs resident in HBM.
  python tools/bench_backward.py [--workload cfg2] [--steps 10] [--warmup 3] [--shards N] [--film-literal]
                                 [--film-hidden WIDTHS]
                                 [--kind rgin|gnn_edge_mlp|ggnn] [--literal]
                                 [--aggregation sum|mean|sqrt_n|max] [--act-before] [--activation NAME]
  python tools/bench_backward.py --kind rgat --literal [--steps 5] [--warmup 2]
With --aggregation / --act-before / --activation: the layer's hyper-parameters changed accordingly (e.g. the RGCN layer of
cfg2 with max aggregation, which trains through the transform-then-aggregate backward); --literal then times that
configuration (RGCN unless --kind) against the literal path on the reduced graph below.
For GNN-FiLM the line also carries the device memory in use after the steps (the library's pool and torch's allocator keep
their high-water marks, so this is the peak of the run, inputs included).
With --film-literal: a reduced FiLM graph on which the literal per-edge path (layers/differentiable.py) fits, 250k nodes /
6 x 666,667 edges / D = H = 320, with the fused and the literal training step alternated in one process.
With --film-hidden WIDTHS (e.g. 320 or 320,160): hidden FiLM-MLP layers of those widths (film_parameter_MLP_hidden_layers) in
the GNN-FiLM layer of --film-literal or of a GNN-FiLM workload (--workload cfg5_shard): the fused path is then the hidden
chain at node level feeding tfgnn_b200_film_in_fwd / _bwd; the line names the autograd function that trained the layer.
--workload cfg3 is RGAT (tfgnn_b200_rgat_bwd); with --kind rgat --literal: cfg3's graph and layer shape reduced to 250k
nodes / 3 x 1M edges, where the literal per-edge path fits, with the fused and the literal step alternated in one process.
With --kind rgin|gnn_edge_mlp|ggnn: that layer (class defaults, one hidden layer in the edge MLPs; RGIN normalised as in
PPI_RGIN.json; GGNN trains through the fused edge-MLP backward and the GRU update pair) on the workload's graph, with D = H = the workload's hidden_dim; the line carries the device memory in use and
the literal path's saved activations computed from shapes.  Adding --literal runs the fused and the literal path alternated
on a reduced graph (250k nodes / 4 x 1M edges / D = H = 256).
With --shards N: the per-rank compute of training on N target-range shards (DESIGN.md §6), on ONE GPU and without
communication: for each shard, the build of its owned-transpose batch (TFGNN_PREPARE_TRANSPOSE_OWNED) and the backward of
the layer on the shard from the full [V, D] table; one JSON line per workload.
Algorithmic bytes of the backward: gather of h rows for A (recomputed) + scatter-side gather of dA rows + dOut/out reads +
dh write + weights, i.e. about twice the forward's (see DESIGN.md)."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from tf2_gnn_b200 import _ffi  # noqa: E402
from tf2_gnn_b200.layers import MessagePassingInput, get_message_passing_class  # noqa: E402
from tf2_gnn_b200.runtime import PreparedBatch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--shards", type=int, default=0, help="time the backward of each of N target-range shards")
    ap.add_argument("--film-literal", action="store_true",
                    help="fused vs literal GNN-FiLM training step on a reduced graph the literal path fits")
    ap.add_argument("--film-hidden", type=lambda s: [int(x) for x in s.split(",")], default=None, metavar="WIDTHS",
                    help="comma-separated widths of hidden FiLM-MLP layers for the GNN-FiLM layer (--film-literal or a "
                         "gnn_film workload)")
    ap.add_argument("--kind", choices=sorted(EDGE_MLP_KINDS) + ["rgat"],
                    help="time this layer kind (class defaults, one hidden layer of width H) on the workload's graph "
                         "instead of the workload's own layer; rgat only with --literal (--workload cfg3 is RGAT)")
    ap.add_argument("--literal", action="store_true",
                    help="with --kind, --aggregation or --act-before: fused vs literal training step on a reduced graph the "
                         "literal path fits")
    ap.add_argument("--aggregation", choices=["sum", "mean", "sqrt_n", "max"],
                    help="aggregation_function of the timed layer (default: the layer's)")
    ap.add_argument("--act-before", action="store_true",
                    help="message_activation_before_aggregation=True for the timed layer")
    ap.add_argument("--activation", help="message_activation_function of the timed layer (default: the layer's)")
    args = ap.parse_args()
    if args.film_literal:
        return bench_film_literal(args)
    if args.kind == "rgat":
        if not args.literal:
            ap.error("--kind rgat goes with --literal (--workload cfg3 times the RGAT workload)")
        return bench_rgat_literal(args)
    if args.literal:
        if not args.kind and not config_overrides(args):
            ap.error("--literal needs --kind, --aggregation or --act-before")
        if args.kind == "ggnn":
            ap.error("--kind ggnn has no --literal comparison")
        return bench_edge_mlp_literal(args)
    wl = bench.WORKLOADS[args.workload]
    if args.film_hidden and (args.kind or wl["kind"]) != "gnn_film":
        ap.error("--film-hidden goes with --film-literal or a gnn_film workload (cfg5, cfg5_shard)")
    V, H, L = wl["V"], wl["H"], len(wl["E"])
    h_np, adjs_np, w_np = bench.make_inputs(wl, seed=0)
    kind = args.kind or wl["kind"]
    wl = dict(wl, kind=kind)
    cls = get_message_passing_class(kind)
    params = cls.get_default_hyperparameters()
    params.update(EDGE_MLP_KINDS[kind] if args.kind else wl.get("params", {}))
    params.update(hidden_dim=H, **config_overrides(args))
    if args.film_hidden:
        params["film_parameter_MLP_hidden_layers"] = args.film_hidden
    layer = cls(params)
    torch.manual_seed(1)
    layer.build(MessagePassingInput((None, H), tuple((None, 2) for _ in range(L))))
    for v in layer.variables:
        v.requires_grad_()
    dev = torch.device("cuda", 0)
    h = torch.from_numpy(h_np).to(dev).requires_grad_()
    adj = tuple(torch.from_numpy(a).to(dev) for a in adjs_np)
    g = torch.rand((V, H), device=dev) * 2 - 1
    inp = MessagePassingInput(h, adj)
    if args.shards:
        return bench_shards(args, wl, layer, h, adj, g)
    prepared = PreparedBatch(adj, V)
    prepared.transposed()
    fwd_ms, bwd_ms = [], []
    for i in range(args.warmup + args.steps):
        e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        h.grad = None
        for v in layer.variables:
            v.value.grad = None
        e0.record()
        out = layer(inp, prepared=prepared)
        e1.record()
        out.backward(g)
        e2.record()
        torch.cuda.synchronize()
        if i >= args.warmup:
            fwd_ms.append(e0.elapsed_time(e1))
            bwd_ms.append(e1.elapsed_time(e2))
    trained_by = type(out.grad_fn).__name__
    del out
    M = sum(wl["E"])
    rec = {
        "workload": wl["desc"], "kind": kind, "forward_ms": float(np.median(fwd_ms)), "backward_ms": float(np.median(bwd_ms)),
        "edges_per_s_fwd_bwd": M / ((np.median(fwd_ms) + np.median(bwd_ms)) * 1e-3), "steps": args.steps,
        "card": card(), "note": NOTES.get(kind, NOTES["rgcn"])}
    if args.kind:
        rec["params"] = EDGE_MLP_KINDS[kind]
        if kind == "ggnn":
            rec["note"] = NOTES["ggnn_mlp"]
        rec["literal_saved_activations_GB_from_shapes"] = literal_footprint_gb(M, H, H, params)
    else:
        rec["forward_algorithmic_bytes"] = bench.algorithmic_bytes(kind, V, wl["E"], H, H, params)
    if config_overrides(args):
        rec["overrides"] = config_overrides(args)
        rec["note"] = NOTES["transform_aggregate"]
    if args.film_hidden:
        rec["film_parameter_MLP_hidden_layers"] = args.film_hidden
        rec["trained_by"] = trained_by
        rec["note"] = NOTES["gnn_film_mlp"]
    if kind in ("gnn_film", "rgat") + tuple(EDGE_MLP_KINDS) or config_overrides(args):
        rec["device_memory_used_GB"] = device_used_gb()
    print(json.dumps(rec), flush=True)


# --kind: class defaults (one hidden layer in the edge MLPs); RGIN with PPI_RGIN.json's normalisation
EDGE_MLP_KINDS = {"rgin": {"normalize_by_num_incoming": True}, "gnn_edge_mlp": {}, "ggnn": {"num_edge_MLP_hidden_layers": 1}}


def config_overrides(args):
    """Hyper-parameters set by --aggregation / --act-before / --activation."""
    o = {}
    if args.aggregation:
        o["aggregation_function"] = args.aggregation
    if args.act_before:
        o["message_activation_before_aggregation"] = True
    if args.activation:
        o["message_activation_function"] = args.activation
    return o


def literal_footprint_gb(M, D, H, params):
    """Saved activations of the literal per-edge path (layers/differentiable.py, edge_mlp_family_forward) for one
    one-hidden-layer edge-MLP layer over M edges, from the shapes of its op sequence (not measured): the gathered source
    rows [E, D] (with target-state input also the target rows and their [E, 2D] concat), the hidden layer's output
    [E, H], the output layer's [E, H], the normalised messages [E, H] and the [M, H] concat of all types."""
    target = params.get("use_target_state_as_input", False)
    per_edge = (4 * D if target else D) + 2 * H + (H if params.get("normalize_by_num_incoming") else 0) + H
    return 4.0 * M * per_edge / 1e9


NOTES = {
    "rgcn": "backward = recompute A (CSR reduce) + TN GEMM dW (fp32 FFMA) + tensor-core GEMM dA + source-keyed CSR reduce dh; "
            "autograd hook overhead included; not tuned (two-kernel form, SIMT dW)",
    "ggnn": "backward = recomputed GRU inputs + gate backward + TN GEMMs for the GRU kernels + the RGCN-style message backward; "
            "autograd hook overhead included",
    "ggnn_mlp": "one hidden layer in the message MLPs: the messages through the rgin-style fused backward, then the GRU update "
                "pair (recomputed gx / gh, gate backward, TN GEMMs for the GRU kernels, tensor-core GEMMs for dagg and dh); "
                "autograd hook overhead included",
    "rgin": "one hidden layer: backward = recompute Xs (= h U^s) and A_l (hidden_relu CSR reduce), dW2 (TN, fp32 FFMA), "
            "dA (tensor-core GEMM), dXs over the source-keyed CSR (one warp per (type, source)), dU (TN), grad_h "
            "(tensor-core GEMM, K = L*H); autograd hook overhead included",
    "gnn_edge_mlp": "as rgin, plus Xt = h_v U^t, the per-column count of active edges in the recompute pass, "
                    "dXt = dA * count, dU^t (TN) and the target rows of grad_h (accumulating GEMM)",
    "transform_aggregate": "no hidden layer, max aggregation or activation before aggregation: backward = recompute P = h W "
                           "(node GEMM) and, for max, the maximum and its tie count (one pass of the forward's edge "
                           "reduce), dZ, dP over the source-keyed CSR (one warp per (type, source)), dW (TN), grad_h "
                           "(tensor-core GEMM, K = L*H); autograd hook overhead included",
    "gnn_film": "backward = per type: recompute [A_l | T_l] (CSR reduce), dQ_l and dgamma_l (tensor-core GEMMs with the dZ "
                "multiply in the epilogue), dW_l and dF_l (TN GEMMs, fp32 FFMA), dA_l and the target-side terms "
                "(tensor-core GEMMs); then one source-keyed CSR reduce for dh; autograd hook overhead included",
    "gnn_film_mlp": "hidden FiLM-MLP layers: forward = the hidden chain (Dense + ReLU per layer and type, node level), its "
                    "last activations concatenated to [V, L*S], then the FiLM layer fed them (tfgnn_b200_film_in_fwd); "
                    "backward = the FiLM layer's (tfgnn_b200_film_in_bwd, as gnn_film with z_l for h_v) and the chain's "
                    "Dense backward; autograd hook overhead included",
    "rgat": "backward = recompute P = h W and the score halves (the forward's GEMM), target pass (one online-softmax walk "
            "per target, hubs in chunk-ordered partials), source pass over the source-keyed CSR (dP, ds_src), attention "
            "gradients (fixed row chunks), dW (TN), grad_h (tensor-core GEMM, K = L*H); no float atomics; autograd hook "
            "overhead included",
}


def card():
    """Name of device 0 and its power limit (read-only query)."""
    import subprocess
    rec = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        rec["power_limit_W"] = float(q.stdout.strip().splitlines()[0])
    except Exception as e:   # the number is then reported without its power limit
        rec["power_limit_W"] = f"unavailable: {type(e).__name__}"
    return rec


def device_used_gb():
    torch.cuda.synchronize()
    free, total = torch.cuda.mem_get_info()
    return (total - free) / 1e9


def release_memory():
    import gc
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    _ffi.lib().tfgnn_b200_release_device_state()


def bench_film_literal(args):
    """Fused (tfgnn_b200_film_bwd, or with --film-hidden the node-level chain and tfgnn_b200_film_in_bwd) vs literal
    (layers/differentiable.py) GNN-FiLM training step, alternated step by step."""
    from tf2_gnn_b200.layers.differentiable import edge_mlp_family_forward
    wl = dict(V=250_000, E=[666_667] * 6, H=320, kind="gnn_film", graph="er",
              desc="GNN-FiLM reduced graph: 250k nodes / 4M edges / 6 edge types, D = H = 320 (class defaults)")
    V, H, L = wl["V"], wl["H"], len(wl["E"])
    h_np, adjs_np, _ = bench.make_inputs(wl, seed=0)
    hidden = args.film_hidden or []
    if hidden:
        wl["desc"] += f", hidden FiLM-MLP layers {hidden}"
    layer = get_message_passing_class("gnn_film")(dict(get_message_passing_class("gnn_film").get_default_hyperparameters(),
                                                       hidden_dim=H, film_parameter_MLP_hidden_layers=hidden))
    torch.manual_seed(1)
    layer.build(MessagePassingInput((None, H), tuple((None, 2) for _ in range(L))))
    for v in layer.variables:
        v.requires_grad_()
    dev = torch.device("cuda", 0)
    h = torch.from_numpy(h_np).to(dev).requires_grad_()
    adj = tuple(torch.from_numpy(a).to(dev) for a in adjs_np)
    g = torch.rand((V, H), device=dev) * 2 - 1
    prepared = PreparedBatch(adj, V)
    prepared.transposed()
    film = [[v.value for v in m.layers] for m in layer._edge_type_film_layer_computations]
    paths = {"fused": lambda: layer(MessagePassingInput(h, adj), prepared=prepared),
             "literal": lambda: edge_mlp_family_forward(layer, h, prepared, film_kernels=film)}
    ms = {k: ([], []) for k in paths}
    mem = {k: 0.0 for k in paths}
    trained_by = {}
    for i in range(args.warmup + args.steps):
        for name, fwd in paths.items():
            release_memory()
            e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            h.grad = None
            for v in layer.variables:
                v.value.grad = None
            e0.record()
            out = fwd()
            e1.record()
            out.backward(g)
            e2.record()
            torch.cuda.synchronize()
            mem[name] = max(mem[name], device_used_gb())
            trained_by[name] = type(out.grad_fn).__name__
            del out
            if i >= args.warmup:
                ms[name][0].append(e0.elapsed_time(e1))
                ms[name][1].append(e1.elapsed_time(e2))
    print(json.dumps({
        "workload": wl["desc"], "kind": "gnn_film", "steps": args.steps, "card": card(),
        "paths": {k: {"forward_ms": float(np.median(f)), "backward_ms": float(np.median(b)),
                      "device_memory_used_GB": mem[k], "trained_by": trained_by[k]} for k, (f, b) in ms.items()},
        "note": "alternated step by step in one process; memory = device memory in use after the step with the library's "
                "pool and torch's allocator cache emptied before it (their high-water mark for that path, inputs included)"}),
        flush=True)


def bench_rgat_literal(args):
    """Fused (tfgnn_b200_rgat_bwd) vs literal (layers/differentiable.py: rgat_forward) RGAT training step, alternated step
    by step, on cfg3's graph and layer shape reduced to a size the literal path fits."""
    from tf2_gnn_b200.layers.differentiable import rgat_forward
    wl = dict(bench.WORKLOADS["cfg3"], V=250_000, E=[1_000_000] * 3,
              desc="RGAT reduced cfg3: power-law 250k nodes / 3M edges / 3 edge types, D = H = 128, 4 heads")
    V, H, L = wl["V"], wl["H"], len(wl["E"])
    h_np, adjs_np, _ = bench.make_inputs(wl, seed=0)
    cls = get_message_passing_class("rgat")
    layer = cls(dict(cls.get_default_hyperparameters(), hidden_dim=H, **wl["params"]))
    torch.manual_seed(1)
    layer.build(MessagePassingInput((None, H), tuple((None, 2) for _ in range(L))))
    for v in layer.variables:
        v.requires_grad_()
    dev = torch.device("cuda", 0)
    h = torch.from_numpy(h_np).to(dev).requires_grad_()
    adj = tuple(torch.from_numpy(a).to(dev) for a in adjs_np)
    g = torch.rand((V, H), device=dev) * 2 - 1
    prepared = PreparedBatch(adj, V)
    prepared.transposed()
    paths = {"fused": lambda: layer(MessagePassingInput(h, adj), prepared=prepared),
             "literal": lambda: rgat_forward(layer, h, prepared)}
    ms = {k: ([], []) for k in paths}
    mem = {k: 0.0 for k in paths}
    for i in range(args.warmup + args.steps):
        for name, fwd in paths.items():
            release_memory()
            e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            h.grad = None
            for v in layer.variables:
                v.value.grad = None
            e0.record()
            out = fwd()
            e1.record()
            out.backward(g)
            e2.record()
            torch.cuda.synchronize()
            mem[name] = max(mem[name], device_used_gb())
            del out
            if i >= args.warmup:
                ms[name][0].append(e0.elapsed_time(e1))
                ms[name][1].append(e1.elapsed_time(e2))
    print(json.dumps({
        "workload": wl["desc"], "kind": "rgat", "steps": args.steps, "card": card(),
        "paths": {k: {"forward_ms": float(np.median(f)), "backward_ms": float(np.median(b)),
                      "device_memory_used_GB": mem[k]} for k, (f, b) in ms.items()},
        "note": "alternated step by step in one process; memory = device memory in use after the step with the library's "
                "pool and torch's allocator cache emptied before it (their high-water mark for that path, inputs included)"}),
        flush=True)


def bench_edge_mlp_literal(args):
    """Fused (tfgnn_b200_edge_mlp_bwd / tfgnn_b200_rgcn_bwd) vs literal (layers/differentiable.py) training step of an RGIN
    or GNN_Edge_MLP layer (class defaults) or of an RGCN layer, with --aggregation / --act-before / --activation applied,
    alternated step by step, on a reduced graph the literal path fits."""
    from tf2_gnn_b200.layers.differentiable import edge_mlp_family_forward
    kind = args.kind or "rgcn"
    changed = dict(EDGE_MLP_KINDS.get(kind, {}), **config_overrides(args))
    wl = dict(V=250_000, E=[1_000_000] * 4, H=256, kind=kind, graph="er",
              desc=f"{kind} reduced graph: 250k nodes / 4M edges / 4 edge types, D = H = 256 (class defaults, "
                   f"{changed or 'nothing'} changed)")
    V, H, L = wl["V"], wl["H"], len(wl["E"])
    h_np, adjs_np, _ = bench.make_inputs(wl, seed=0)
    cls = get_message_passing_class(kind)
    layer = cls(dict(cls.get_default_hyperparameters(), hidden_dim=H, **changed))
    torch.manual_seed(1)
    layer.build(MessagePassingInput((None, H), tuple((None, 2) for _ in range(L))))
    for v in layer.variables:
        v.requires_grad_()
    dev = torch.device("cuda", 0)
    h = torch.from_numpy(h_np).to(dev).requires_grad_()
    adj = tuple(torch.from_numpy(a).to(dev) for a in adjs_np)
    g = torch.rand((V, H), device=dev) * 2 - 1
    prepared = PreparedBatch(adj, V)
    prepared.transposed()
    literal_kw = dict(activation_before=False, aggr_kernels=None) if kind == "rgin" else {}
    paths = {"fused": lambda: layer(MessagePassingInput(h, adj), prepared=prepared),
             "literal": lambda: edge_mlp_family_forward(layer, h, prepared, **literal_kw)}
    ms = {k: ([], []) for k in paths}
    mem = {k: 0.0 for k in paths}
    for i in range(args.warmup + args.steps):
        for name, fwd in paths.items():
            release_memory()
            e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            h.grad = None
            for v in layer.variables:
                v.value.grad = None
            e0.record()
            out = fwd()
            e1.record()
            out.backward(g)
            e2.record()
            torch.cuda.synchronize()
            mem[name] = max(mem[name], device_used_gb())
            del out
            if i >= args.warmup:
                ms[name][0].append(e0.elapsed_time(e1))
                ms[name][1].append(e1.elapsed_time(e2))
    print(json.dumps({
        "workload": wl["desc"], "kind": kind, "steps": args.steps, "card": card(),
        "paths": {k: {"forward_ms": float(np.median(f)), "backward_ms": float(np.median(b)),
                      "device_memory_used_GB": mem[k]} for k, (f, b) in ms.items()},
        "note": "alternated step by step in one process; memory = device memory in use after the step with the library's "
                "pool and torch's allocator cache emptied before it (their high-water mark for that path, inputs included)"}),
        flush=True)


def _median_ms(fn, steps, warmup):
    ms = []
    for i in range(warmup + steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        if i >= warmup:
            ms.append(e0.elapsed_time(e1))
    return float(np.median(ms))


def bench_shards(args, wl, layer, h, adj, g):
    from tf2_gnn_b200 import sharding
    V = wl["V"]
    deg = sum(np.bincount(a[:, 1].cpu().numpy(), minlength=V) for a in adj)
    bounds = sharding.partition_target_range(V, args.shards, deg)
    prep_ms, bwd_ms = [], []
    for lo, hi in bounds:
        shard = PreparedBatch(adj, V, target_range=(lo, hi))
        prep_ms.append(_median_ms(lambda: PreparedBatch(adj, V, target_range=(lo, hi), transpose_owned=True), args.steps,
                                  args.warmup))
        shard.transposed()
        out = None

        def forward():
            nonlocal out
            h.grad = None
            for v in layer.variables:
                v.value.grad = None
            out = layer(MessagePassingInput(h, adj), prepared=shard)

        def backward():
            out.backward(g[lo:hi])

        ms = []
        for i in range(args.warmup + args.steps):
            forward()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            backward()
            e1.record()
            torch.cuda.synchronize()
            if i >= args.warmup:
                ms.append(e0.elapsed_time(e1))
        bwd_ms.append(float(np.median(ms)))
        del shard, out
    print(json.dumps({
        "workload": wl["desc"], "kind": wl["kind"], "shards": args.shards, "bounds": bounds,
        "owned_transpose_prepare_ms": prep_ms, "backward_ms": bwd_ms, "backward_ms_max": max(bwd_ms),
        "backward_ms_sum": sum(bwd_ms), "prepare_ms_max": max(prep_ms), "card": card(),
        "note": "one GPU, per-rank compute only: no all-gather / reduce-scatter / all-reduce; grad_h is the full [V, D] "
                "table per shard"}), flush=True)


if __name__ == "__main__":
    main()
