"""The readout / exchange backward entries without a GPU: exported and bound, arguments validated before any CUDA call, and
the float64 reference the GPU tests compare against checked against autograd, the oracle and itself."""
import ctypes

import numpy as np
import pytest

torch = pytest.importorskip("torch")

import reference64_readout as r64  # noqa: E402
from oracle import message_passing_oracle as mo  # noqa: E402
from tf2_gnn_b200 import _ffi  # noqa: E402

NEW = ("tfgnn_b200_segment_sum_rows", "tfgnn_b200_readout_bwd", "tfgnn_b200_gru_gate_bwd_indexed")


def test_new_entries_are_exported_and_bound():
    raw = ctypes.CDLL(_ffi.library_path())
    lib = _ffi.lib()
    for name in NEW:
        assert hasattr(raw, name) and name in _ffi.EXPORTED_SYMBOLS
        assert getattr(lib, name).argtypes, f"{name} has no argtypes in _ffi.py"
    assert lib.tfgnn_b200_abi_version() == 1


def test_invalid_arguments_are_reported_before_any_cuda_call():
    lib = _ffi.lib()
    p = 64     # never dereferenced: validation fails first
    bad = _ffi.ERR_INVALID_ARGUMENT
    assert lib.tfgnn_b200_segment_sum_rows(p, p, p, -1, 3, 8, p, None) == bad
    assert b"segment_sum_rows" in lib.tfgnn_b200_last_error()
    assert lib.tfgnn_b200_segment_sum_rows(p, p, p, 10, 3, 0, p, None) == bad
    assert lib.tfgnn_b200_segment_sum_rows(None, p, p, 10, 3, 8, p, None) == bad
    assert lib.tfgnn_b200_segment_sum_rows(p, p, None, 10, 3, 8, p, None) == bad
    assert lib.tfgnn_b200_segment_sum_rows(p, p, p, 10, 0, 8, None, None) == 0          # no graphs: nothing to do

    def readout(reprs=p, weights=p, n2g=p, ptr=p, out=p, go=p, V=10, G=3, GD=8, K=4, mode=0, gr=p, gs=p):
        return lib.tfgnn_b200_readout_bwd(reprs, weights, n2g, ptr, out, go, V, G, GD, K, mode, 0.0, 0.0, 0, 0, gr, gs, None)

    assert readout(GD=10, K=4) == bad
    assert b"num_heads must divide" in lib.tfgnn_b200_last_error()
    assert readout(V=-1) == bad
    assert readout(mode=4) == bad
    assert b"mode" in lib.tfgnn_b200_last_error()
    assert readout(mode=-1) == bad
    assert readout(reprs=None) == bad
    assert readout(weights=None, mode=1) == bad
    assert readout(gs=None, mode=0) == bad
    assert readout(out=None, mode=0) == bad
    assert readout(V=0) == 0
    with pytest.raises(ValueError):
        _ffi.check(readout(gr=None, mode=2, weights=None, gs=None))

    def gru(gx=p, n2g=p, ptr=p, V=10, G=3, H=4, dgx=p):
        return lib.tfgnn_b200_gru_gate_bwd_indexed(gx, n2g, ptr, p, p, p, V, G, H, dgx, p, p, None)

    assert gru(H=0) == bad
    assert gru(V=-2) == bad
    assert gru(gx=None) == bad
    assert gru(dgx=None) == bad
    assert gru(G=0) == 0


def _case(rng, V=60, G=7, D=6, GD=12, K=3, biases=False):
    n2g = np.sort(rng.integers(0, G, size=V)).astype(np.int32)
    n2g[n2g == 2] = 3                                         # an empty graph in the middle
    x = rng.uniform(-1, 1, (V, D))
    w = {"scoring_mlp": [rng.uniform(-1, 1, (D, 5)), rng.uniform(-1, 1, (5, K))],
         "transformation_mlp": [rng.uniform(-1, 1, (D, 5)), rng.uniform(-1, 1, (5, GD))]}
    if biases:
        w["scoring_biases"] = [rng.uniform(-.2, .2, 5), rng.uniform(-.2, .2, K)]
        w["transformation_biases"] = [rng.uniform(-.2, .2, 5), rng.uniform(-.2, .2, GD)]
    return x, n2g, w


@pytest.mark.parametrize("mode", ["softmax", "sigmoid", "none", "average"])
@pytest.mark.parametrize("bounds", [(None, None), (-0.2, 0.3), (None, 0.1), (0.0, None)])
def test_closed_form_readout_backward_is_autograd_of_the_literal_formulas(mode, bounds):
    rng = np.random.default_rng(3)
    V, G, GD, K = 80, 6, 12, 3
    n2g = np.sort(rng.integers(0, G - 1, size=V)).astype(np.int32)          # last graph empty
    scores, reprs = r64.leaf(rng.uniform(-2, 2, (V, K))), r64.leaf(rng.uniform(-1, 1, (V, GD)))
    with torch.no_grad():
        reprs[:5, :4] = 0.3 if bounds[1] == 0.3 else (0.0 if bounds[0] == 0.0 else reprs[:5, :4])   # ties with a bound
    R = rng.uniform(-1, 1, (G, GD))
    out = r64.readout_from_scores(scores, reprs, n2g, G, K, mode, *bounds)
    (out * torch.from_numpy(R)).sum().backward()
    gs, gr = r64.readout_backward_closed_form(scores.detach().numpy(), reprs.detach().numpy(), n2g, G, K, mode, R, *bounds)
    np.testing.assert_allclose(gr, reprs.grad.numpy(), rtol=1e-12, atol=1e-13)
    if gs is not None:
        np.testing.assert_allclose(gs, scores.grad.numpy(), rtol=1e-10, atol=1e-13)
    else:
        assert scores.grad is None


@pytest.mark.parametrize("mode", ["softmax", "sigmoid", "none", "average"])
def test_reference_forward_agrees_with_the_readout_oracle(mode):
    rng = np.random.default_rng(4)
    x, n2g, w = _case(rng, biases=True)
    G, GD, K = 7, 12, 3
    ref = mo.weighted_sum_graph_representation(x, n2g, G, w, GD, K, mode, scoring_activation="elu",
                                               transformation_activation="tanh", lower_bound=-0.3, upper_bound=0.4,
                                               dtype=np.float64)
    got = r64.readout_layer(torch.from_numpy(x), r64.leaves_of(w), n2g, G, K, mode, "elu", "tanh", -0.3, 0.4)
    np.testing.assert_allclose(got.detach().numpy(), ref, rtol=1e-12, atol=1e-13)


@pytest.mark.parametrize("mode", ["mean", "gru", "mlp"])
@pytest.mark.parametrize("weighting", ["softmax", "sigmoid"])
def test_reference_exchange_agrees_with_the_exchange_oracle(mode, weighting):
    rng = np.random.default_rng(5)
    V, G, H, K = 70, 6, 8, 2
    n2g = np.sort(rng.integers(0, G, size=V)).astype(np.int32)
    x = rng.uniform(-1, 1, (V, H))
    w = mo.make_exchange_weights(mode, H, K, rng, weighting, dtype=np.float64)
    ref = mo.graph_global_exchange(mode, x, n2g, G, w, H, K, weighting, dtype=np.float64)
    got = r64.exchange(mode, torch.from_numpy(x), r64.leaves_of(w), n2g, G, K, weighting)
    np.testing.assert_allclose(got.detach().numpy(), ref, rtol=1e-12, atol=1e-13)


def test_reference_was_is_two_readouts_and_a_projection():
    rng = np.random.default_rng(6)
    x, n2g, w_avg = _case(rng, biases=True)
    _, _, w_sum = _case(rng, biases=True)
    P = rng.uniform(-1, 1, (24, 12))
    got = r64.was(torch.from_numpy(x), r64.leaves_of(w_avg), r64.leaves_of(w_sum), torch.from_numpy(P), n2g, 7, 3)
    parts = [mo.weighted_sum_graph_representation(x, n2g, 7, w, 12, 3, fun, scoring_activation="elu",
                                                  transformation_activation="elu", dtype=np.float64)
             for w, fun in ((w_avg, "softmax"), (w_sum, "sigmoid"))]
    np.testing.assert_allclose(got.detach().numpy(), np.concatenate(parts, -1) @ P, rtol=1e-12, atol=1e-13)


@pytest.mark.parametrize("seed", range(6))
def test_chunked_segment_sum_gives_the_same_sums_for_any_chunk_cut(seed):
    """Integer data: every order of additions is exact, so every chunk size and lane count must give the plain sums; graphs
    are empty at the front, in the middle and at the end."""
    rng = np.random.default_rng(seed)
    G, C = int(rng.integers(1, 12)), int(rng.integers(1, 7))
    sizes = rng.integers(0, 40, size=G)
    sizes[rng.integers(0, G)] = 0
    if seed % 2:
        sizes[0] = sizes[-1] = 0
    ptr = np.concatenate([[0], np.cumsum(sizes)])
    data = rng.integers(-8, 9, size=(int(ptr[-1]), C)).astype(np.float32)
    plain = np.stack([data[ptr[g]:ptr[g + 1]].sum(0) for g in range(G)]) if G else np.zeros((0, C), np.float32)
    for chunk_rows in (1, 3, 7, 64, 1000):
        for lanes in (1, 8):
            got = r64.segment_sum_rows_chunked(data, ptr, chunk_rows, lanes)
            assert np.array_equal(got, plain), (chunk_rows, lanes)
    assert np.array_equal(r64.graph_ptr_of(np.repeat(np.arange(G), sizes), G), ptr)
