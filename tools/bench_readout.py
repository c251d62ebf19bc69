"""Forward + backward of the graph readout and the three global exchanges: the row-range training path
(layers/graph_autograd.py) against the literal op order (layers/differentiable.py), on an H100.

    python tools/bench_readout.py [--steps 50] [--warmup 5] [--shapes ppi,qm9,one_graph] [--out result.json]

Shapes: PPI (8000 nodes, 3 graphs, H = 320), QM9-like (500k nodes in 27.8k graphs of 9-29 nodes, H = 128) and one graph of
1M nodes (H = 256); softmax weighting, 4 heads, no dropout.  The two paths are alternated step by step, timed with CUDA
events around forward + backward, and their outputs and node-state gradients are compared at the timed size.  Also reported:
peak torch-allocated memory of one step per path, and the forward-only time of the untouched segment kernels
(segment_softmax, weighted_segment_sum).  Fails without a GPU; the card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = {
    "ppi": dict(desc="PPI: 8000 nodes, 3 graphs, H=320", H=320, sizes=lambda rng: np.array([2400, 3500, 2100])),
    "qm9": dict(desc="QM9-like: 500k nodes, 27.8k graphs of 9-29 nodes, H=128", H=128,
                sizes=lambda rng: rng.integers(9, 30, size=27800)),
    "one_graph": dict(desc="one graph of 1M nodes, H=256", H=256, sizes=lambda rng: np.array([1_000_000])),
}
K = 4


def card():
    rec = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        rec["power_limit_W"] = float(q.stdout.strip().splitlines()[0])
    except Exception as e:   # the numbers are then reported without the power limit
        rec["power_limit_W"] = f"unavailable: {type(e).__name__}"
    return rec


def build(kind, H):
    from tf2_gnn_b200.layers import (GraphGlobalExchangeInput, GraphGlobalGRUExchange, GraphGlobalMeanExchange,
                                     GraphGlobalMLPExchange, NodesToGraphRepresentationInput,
                                     WeightedSumGraphRepresentation)
    torch.manual_seed(1)
    if kind == "readout":
        layer = WeightedSumGraphRepresentation(H, K, "softmax", scoring_mlp_layers=[H])
        layer.build(NodesToGraphRepresentationInput((None, H), None, None))
    else:
        cls = {"mean": GraphGlobalMeanExchange, "gru": GraphGlobalGRUExchange, "mlp": GraphGlobalMLPExchange}[kind]
        layer = cls(hidden_dim=H, weighting_fun="softmax", num_heads=K, dropout_rate=0.0)
        layer.build(GraphGlobalExchangeInput((None, H), (None,), ()))
    for v in layer.variables:
        v.requires_grad_(True)
    return layer


def literal_forward(kind, layer, x, n2g, G):
    from tf2_gnn_b200.layers import differentiable as lit
    if kind == "readout":
        return lit.weighted_sum_graph_representation(layer, x, n2g, G, False)
    per_node = lit.per_node_graph_representations(layer, x, n2g, G, False)
    if kind == "mean":
        return lit._AddFunction.apply(x, per_node, 0.5, 0.5)
    if kind == "gru":
        return lit.gru_cell(per_node, x, layer._gru_kernel.value, layer._gru_recurrent_kernel.value, layer._gru_bias.value)
    return layer._mlp(torch.cat([per_node, x], dim=-1), False, None)


def new_forward(kind, layer, x, n2g, G):
    from tf2_gnn_b200.layers import GraphGlobalExchangeInput, NodesToGraphRepresentationInput
    inp = (NodesToGraphRepresentationInput if kind == "readout" else GraphGlobalExchangeInput)(x, n2g, G)
    return layer(inp, training=False)


def step(fwd, kind, layer, x_data, n2g, G, R):
    for v in layer.variables:
        v.value.grad = None
    x = x_data.clone().requires_grad_()
    out = fwd(kind, layer, x, n2g, G)
    (out * R[:out.shape[0]]).sum().backward()
    return out.detach(), x.grad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--shapes", default="ppi,qm9,one_graph")
    ap.add_argument("--kinds", default="readout,mean,gru,mlp")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_readout.py needs a CUDA device: a time taken anywhere else says nothing about the H100")
    from tf2_gnn_b200.layers import node_ops
    result = {"card": card(), "steps": args.steps, "warmup": args.warmup, "rows": []}
    for shape in args.shapes.split(","):
        cfg = SHAPES[shape]
        rng = np.random.default_rng(0)
        sizes = cfg["sizes"](rng)
        H, G = cfg["H"], len(sizes)
        n2g = torch.from_numpy(np.repeat(np.arange(G), sizes).astype(np.int32)).cuda()
        V = int(n2g.shape[0])
        x_data = torch.rand((V, H), device="cuda") * 2 - 1
        R = torch.rand((V, H), device="cuda") * 2 - 1
        # forward-only time of the untouched segment kernels
        ptr = node_ops.graph_offsets(n2g, G)
        scores = torch.rand((V, K), device="cuda")
        fwd_ms = {}
        for name, call in (("segment_softmax", lambda: node_ops.segment_softmax(scores, ptr)),
                           ("weighted_segment_sum", lambda: node_ops.weighted_segment_sum(x_data, scores, ptr, K))):
            for _ in range(args.warmup):
                call()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.steps):
                call()
            b.record()
            torch.cuda.synchronize()
            fwd_ms[name] = a.elapsed_time(b) / args.steps
        for kind in args.kinds.split(","):
            layer = build(kind, H)
            paths = {"row_ranges": new_forward, "literal": literal_forward}
            outs, peaks = {}, {}
            for name, fwd in paths.items():
                for _ in range(args.warmup):
                    step(fwd, kind, layer, x_data, n2g, G, R)
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                outs[name] = step(fwd, kind, layer, x_data, n2g, G, R)
                torch.cuda.synchronize()
                peaks[name] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
            diffs = [float((a.double() - b.double()).norm() / b.double().norm().clamp(min=1e-30))
                     for a, b in zip(outs["row_ranges"], outs["literal"])]
            events = {name: [] for name in paths}
            for _ in range(args.steps):                       # the two paths alternated step by step
                for name, fwd in paths.items():
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    step(fwd, kind, layer, x_data, n2g, G, R)
                    b.record()
                    events[name].append((a, b))
            torch.cuda.synchronize()
            row = {"shape": shape, "desc": cfg["desc"], "kind": kind, "V": V, "G": G, "H": H,
                   "rel_diff_output": diffs[0], "rel_diff_grad_x": diffs[1], "forward_only_ms": fwd_ms}
            for name in paths:
                ms = sorted(a.elapsed_time(b) for a, b in events[name])
                row[name] = {"fwd_bwd_ms_median": ms[len(ms) // 2], "fwd_bwd_ms_min": ms[0], "fwd_bwd_ms_max": ms[-1],
                             "peak_step_MiB": peaks[name]}
            result["rows"].append(row)
            print(json.dumps(row), flush=True)
            del layer, outs
            torch.cuda.empty_cache()
    print(json.dumps({"card": result["card"]}))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
