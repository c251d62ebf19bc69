"""float64 restatement of QM9RegressionTask's head (qm9_regression.py:83-114) in numpy, forward and closed-form backward,
and a generator of seeded synthetic records in the QM9 file format (the reference ships no QM9 data).

Head: t = X W_t + b_t ([V, 1]), s = Z W_g + b_g with Z = [X0 ‖ X] ([V, 1]), out[g] = Σ_{v in g} σ(s_v) t_v."""
import gzip
import json
import os

import numpy as np

NUM_TARGETS = 13
NUM_FEATURES = 15
NUM_FWD_TYPES = 4

# QM9_RGCN.json's model parameters (the reference's default_hypers/QM9_RGCN.json)
QM9_RGCN = dict(gnn_residual_every_num_layers=2, gnn_num_layers=8, gnn_initial_node_representation_activation="tanh",
                gnn_dense_intermediate_layer_activation="tanh", gnn_layer_input_dropout_rate=0.0,
                gnn_message_activation_function="leaky_relu", rmsprop_rho=0.98, momentum=0.85,
                gnn_aggregation_function="sum", gnn_dense_every_num_layers=32, learning_rate=0.0005720408870458782,
                gnn_use_inter_layer_layernorm=True, gnn_hidden_dim=128, gradient_clip_value=1.0, optimizer="RMSProp")


def head_forward(x0, x, n2g, num_graphs, w):
    """out [G]; w: dict of gate_kernel [F + H, 1], gate_bias [1], transform_kernel [H, 1], transform_bias [1]."""
    x0, x = np.asarray(x0, np.float64), np.asarray(x, np.float64)
    t = x @ np.asarray(w["transform_kernel"], np.float64) + np.asarray(w["transform_bias"], np.float64)
    z = np.concatenate([x0, x], axis=1)
    s = z @ np.asarray(w["gate_kernel"], np.float64) + np.asarray(w["gate_bias"], np.float64)
    sig = 1.0 / (1.0 + np.exp(-s))
    out = np.zeros(num_graphs)
    np.add.at(out, np.asarray(n2g, np.int64), (sig * t)[:, 0])
    return out


def head_backward(x0, x, n2g, w, grad_out):
    """Gradients for the upstream gradient grad_out [G]: dict of gate_input [V, F + H], transform_input [V, H] and the four
    variables."""
    x0, x = np.asarray(x0, np.float64), np.asarray(x, np.float64)
    Wt, Wg = np.asarray(w["transform_kernel"], np.float64), np.asarray(w["gate_kernel"], np.float64)
    t = x @ Wt + np.asarray(w["transform_bias"], np.float64)
    z = np.concatenate([x0, x], axis=1)
    sig = 1.0 / (1.0 + np.exp(-(z @ Wg + np.asarray(w["gate_bias"], np.float64))))
    g_rows = np.asarray(grad_out, np.float64)[np.asarray(n2g, np.int64)][:, None]   # [V, 1]
    dt = g_rows * sig
    ds = g_rows * t * sig * (1.0 - sig)
    return {"gate_input": ds @ Wg.T, "transform_input": dt @ Wt.T,
            "gate_kernel": z.T @ ds, "gate_bias": ds.sum(axis=0),
            "transform_kernel": x.T @ dt, "transform_bias": dt.sum(axis=0)}


# ---- synthetic QM9-format records --------------------------------------------------------------------------------------
def molecule(rng, num_atoms=None):
    """One record as in the QM9 fold files: 9-29 atoms, a random spanning tree plus a few ring bonds, bond types 1..4,
    15-wide one-hot atom features, 13 targets of one value each."""
    n = int(rng.integers(9, 30)) if num_atoms is None else int(num_atoms)
    bonds = [(int(rng.integers(0, v)), v) for v in range(1, n)]
    for _ in range(int(rng.integers(0, 4)) if n > 2 else 0):
        a, b = rng.choice(n, 2, replace=False)
        bonds.append((int(a), int(b)))
    graph = [[a, int(rng.integers(1, NUM_FWD_TYPES + 1)), b] for a, b in bonds]
    feats = np.zeros((n, NUM_FEATURES), dtype=np.int64)
    feats[np.arange(n), rng.integers(0, NUM_FEATURES, n)] = 1
    # targets that depend on the molecule, so a model can learn them: atom-type counts and bond counts, plus noise
    counts = feats.sum(axis=0)
    targets = [[float(counts[k % NUM_FEATURES] * 0.1 + len(bonds) * 0.01 * (k + 1) + rng.normal(0, 0.01))]
               for k in range(NUM_TARGETS)]
    return {"graph": graph, "node_features": feats.tolist(), "targets": targets}


def write_fold(path, records):
    with gzip.open(path, "wt") as f:
        for r in records:
            f.write(json.dumps(r) + "\n")


def write_dataset(directory, rng, sizes=(200, 50, 50)):
    """train / valid / test fold files of synthetic molecules in `directory`; returns the records per file name."""
    out = {}
    for name, k in zip(("train.jsonl.gz", "valid.jsonl.gz", "test.jsonl.gz"), sizes):
        recs = [molecule(rng) for _ in range(k)]
        write_fold(os.path.join(directory, name), recs)
        out[name] = recs
    return out
