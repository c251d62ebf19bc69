"""The float64 restatement of GNN-FiLM with hidden FiLM-MLP layers (reference64_film_mlp.py) against the numpy oracle's
inference forward, on small graphs with empty types, isolated nodes, duplicate edges and self-loops.  CPU only."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

import reference64_film_mlp as rfm  # noqa: E402
from oracle import message_passing_oracle as mo  # noqa: E402
from test_reference64_cpu import close, small_graph  # noqa: E402


@pytest.mark.parametrize("film_hidden", [[5], [9, 6], [16]])
@pytest.mark.parametrize("agg,act,normalize,use_target,act_before,edge_hidden", [
    ("sum", "relu", False, False, False, 0),
    ("mean", "tanh", True, False, False, 0),
    ("sqrt_n", "elu", False, True, False, 0),
    ("sum", "gelu", True, True, False, 1),
    ("mean", "tanh", False, False, True, 2),
])
def test_film_mlp_restatement_matches_oracle(film_hidden, agg, act, normalize, use_target, act_before, edge_hidden):
    rng = np.random.default_rng(len(film_hidden) + 3 * edge_hidden + 5 * normalize + len(agg))
    V, D, H, L = 60, 12, 8, 3
    adjs = small_graph(rng, V, L)
    p = mo.default_hyperparameters("gnn_film")
    p.update(hidden_dim=H, aggregation_function=agg, message_activation_function=act, normalize_by_num_incoming=normalize,
             use_target_state_as_input=use_target, message_activation_before_aggregation=act_before,
             num_edge_MLP_hidden_layers=edge_hidden, film_parameter_MLP_hidden_layers=film_hidden)
    w = mo.make_weights("gnn_film", p, D, L, rng, dtype=np.float64)
    assert [f.shape for f in w["film_mlps"][0]] == [(a, b) for a, b in zip([D] + film_hidden, film_hidden + [2 * H])]
    h = rng.uniform(-1, 1, (V, D))
    ref = mo.message_passing_forward("gnn_film", p, w, h, adjs, dtype=np.float64)
    t = lambda mats: [torch.from_numpy(m) for m in mats]
    got = rfm.film_mlp_autograd(torch.from_numpy(h), adjs, [t(m) for m in w["edge_mlps"]], [t(m) for m in w["film_mlps"]],
                                agg=agg, act=act, normalize=normalize, use_target=use_target, act_before=act_before)
    close(got, torch.from_numpy(ref))
    pre = rfm.hidden_preactivations(torch.from_numpy(h), [t(m) for m in w["film_mlps"]])
    assert pre[0].shape == (V, sum(film_hidden))
