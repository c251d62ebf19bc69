"""reference64_rgat.forward_backward (chunked, one edge type at a time) against float64 torch autograd of the reference's
literal RGAT op order."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

import reference64_rgat as r64  # noqa: E402


def _case(seed, V, D, K, d, L, act, E=400):
    rng = np.random.default_rng(seed)
    H = K * d
    t = lambda a: torch.from_numpy(np.asarray(a, np.float64))
    adjs = [torch.from_numpy(rng.integers(0, V, size=(E, 2)).astype(np.int32)) for _ in range(L - 1)]
    adjs.append(torch.zeros((0, 2), dtype=torch.int32))   # an empty type
    adjs[0][:40, 1] = 3                                    # a target with many incoming edges
    adjs[0][41] = adjs[0][40]                              # a duplicate
    h = t(rng.uniform(-1, 1, (V, D)))
    Ws = [t(rng.uniform(-0.5, 0.5, (D, H))) for _ in range(L)]
    As = [t(rng.uniform(-0.5, 0.5, (K, 2 * d))) for _ in range(L)]
    g = t(rng.uniform(-1, 1, (V, H)))
    return adjs, h, Ws, As, g


@pytest.mark.parametrize("K,d,D,L,act,chunk", [(1, 4, 6, 2, "none", 7), (3, 8, 20, 3, "tanh", 50), (4, 6, 5, 4, "relu", 1 << 20),
                                               (2, 10, 8, 3, "gelu", 33)])
def test_chunked_reference_matches_literal_autograd(K, d, D, L, act, chunk):
    adjs, h, Ws, As, g = _case(K + d, 60, D, K, d, L, act)
    out, grad_h, dWs, das, margin = r64.forward_backward(h, adjs, Ws, As, g, act, chunk=chunk)
    assert margin > 0
    leaves = [x.clone().requires_grad_() for x in [h] + Ws + As]
    ref = r64.literal_autograd(leaves[0], adjs, leaves[1:1 + L], leaves[1 + L:], act)
    ref.backward(g)
    np.testing.assert_allclose(out.numpy(), ref.detach().numpy(), rtol=0, atol=1e-12)
    np.testing.assert_allclose(grad_h.numpy(), leaves[0].grad.numpy(), rtol=0, atol=1e-12)
    for l in range(L):
        gW = leaves[1 + l].grad
        gA = leaves[1 + L + l].grad
        np.testing.assert_allclose(dWs[l].numpy(), np.zeros_like(dWs[l]) if gW is None else gW.numpy(), rtol=0, atol=1e-12)
        np.testing.assert_allclose(das[l].numpy(), np.zeros_like(das[l]) if gA is None else gA.numpy(), rtol=0, atol=1e-12)


def test_chunked_reference_grad_h_rows():
    adjs, h, Ws, As, g = _case(1, 50, 8, 2, 4, 2, "tanh")
    full = r64.forward_backward(h, adjs, Ws, As, g, "tanh")[1]
    rows = torch.tensor([3, 0, 17])
    np.testing.assert_allclose(r64.forward_backward(h, adjs, Ws, As, g, "tanh", grad_h_rows=rows)[1].numpy(),
                               full[rows].numpy(), rtol=0, atol=1e-14)
