"""A numpy float64 restatement of the steps of tfgnn_b200_rgat_bwd (rgat.cu, backward.cu) against torch autograd of the
reference's literal RGAT op order: the target pass's one online walk (running maximum, per-type sums flushed and brought to
the final maximum), hub chunks combined in chunk order, the source-keyed formulas, and target ranges whose contributions sum
to the whole."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

import reference64_rgat as r64  # noqa: E402

LEAKY = 0.2


def _leaky(x):
    return x if x > 0 else LEAKY * x


def _walk(edges, P, s_src, s_tgt_v, dz_v, L, K, d):
    """One walk over `edges` [(l, u)] (type-major) of one target: per head the running maximum m, den, G and per type A1, A2
    flushed at the end of the type with the maximum they refer to, then brought to the final maximum."""
    m = np.full(K, -np.inf)
    den, G = np.zeros(K), np.zeros(K)
    flushed = {}
    for l in range(L):
        A1, A2 = np.zeros(K), np.zeros(K)
        for ll, u in edges:
            if ll != l:
                continue
            for k in range(K):
                xs = s_src[u, l, k] + s_tgt_v[l, k]
                score, lp = _leaky(xs), (1.0 if xs > 0 else LEAKY)
                da = dz_v[k * d:(k + 1) * d] @ P[l][u, k * d:(k + 1) * d]
                if score > m[k]:
                    r = np.exp(m[k] - score) if np.isfinite(m[k]) else 0.0
                    m[k] = score
                    den[k], G[k], A1[k], A2[k] = den[k] * r + 1, G[k] * r + da, A1[k] * r + lp * da, A2[k] * r + lp
                else:
                    w = np.exp(score - m[k])
                    den[k] += w
                    G[k] += w * da
                    A1[k] += w * lp * da
                    A2[k] += w * lp
        flushed[l] = (A1, A2, m.copy())
    # a type walked before the first edge flushed zeros at m = -inf: its factor is 0
    scale = lambda ml: np.exp(np.where(np.isfinite(ml), ml, 0.0) - np.where(np.isfinite(ml), m, 0.0)) * np.isfinite(ml)
    A1 = np.stack([flushed[l][0] * scale(flushed[l][2]) for l in range(L)])
    A2 = np.stack([flushed[l][1] * scale(flushed[l][2]) for l in range(L)])
    return m, den, G, A1, A2


def _fused(h, adjs, Ws, As, g, act, lo, hi, chunk):
    """grad_h, [dW], [da] of the targets [lo, hi): target pass (hubs: targets with more than `chunk` edges, cut into chunks),
    source pass, attention and weight gradients."""
    V, H = h.shape[0], Ws[0].shape[1]
    K, L = As[0].shape[0], len(adjs)
    d = H // K
    P = [h @ W for W in Ws]
    s_src = np.stack([(Pl.reshape(V, K, d) * a[:, :d]).sum(-1) for Pl, a in zip(P, As)], 1)   # [V, L, K]
    s_tgt = np.stack([(Pl.reshape(V, K, d) * a[:, d:]).sum(-1) for Pl, a in zip(P, As)], 1)
    into = {v: [(l, int(u)) for l, a in enumerate(adjs) for u, t in a if t == v] for v in range(V)}
    # the pre-activation o (only its derivative is needed) and dZ
    o = np.zeros((V, H))
    for v in range(V):
        for k in range(K):
            sc = np.array([_leaky(s_src[u, l, k] + s_tgt[v, l, k]) for l, u in into[v]])
            if sc.size:
                w = np.exp(sc - sc.max()) / np.exp(sc - sc.max()).sum()
                o[v, k * d:(k + 1) * d] = sum(wi * P[l][u, k * d:(k + 1) * d] for wi, (l, u) in zip(w, into[v]))
    _, dact = r64._act(act, torch.from_numpy(o))
    dz = g * dact.numpy()
    # target pass over the owned rows
    stat = np.zeros((V, 3, K))
    ds_tgt = np.zeros((V, L, K))
    for v in range(lo, hi):
        e = into[v]
        parts = [e[c:c + chunk] for c in range(0, len(e), chunk)] if len(e) > chunk else [e]
        res = [_walk(pc, P, s_src, s_tgt[v], dz[v], L, K, d) for pc in parts]
        m = np.max([r[0] for r in res], 0)
        sc = [np.exp(r[0] - m) if np.isfinite(m).all() else np.ones(K) for r in res]
        den = sum(s * r[1] for s, r in zip(sc, res))          # chunk order
        G = sum(s * r[2] for s, r in zip(sc, res))
        A1 = sum(s * r[3] for s, r in zip(sc, res))
        A2 = sum(s * r[4] for s, r in zip(sc, res))
        gk = np.where(den > 0, G / np.where(den > 0, den, 1), 0)
        assert np.allclose(gk, [dz[v, k * d:(k + 1) * d] @ o[v, k * d:(k + 1) * d] for k in range(K)], atol=1e-12)
        stat[v] = m, den, gk
        ds_tgt[v] = np.where(den > 0, (A1 - gk * A2) / np.where(den > 0, den, 1), 0)
    # source pass: the edges into owned targets, keyed by source
    dP = [np.zeros((V, H)) for _ in range(L)]
    ds_src = np.zeros((V, L, K))
    for l, a in enumerate(adjs):
        for u, v in a:
            if not lo <= v < hi:
                continue
            for k in range(K):
                cols = slice(k * d, (k + 1) * d)
                xs = s_src[u, l, k] + s_tgt[v, l, k]
                alpha = np.exp(_leaky(xs) - stat[v, 0, k]) / stat[v, 1, k]
                da = dz[v, cols] @ P[l][u, cols]
                ds_src[u, l, k] += alpha * (da - stat[v, 2, k]) * (1.0 if xs > 0 else LEAKY)
                dP[l][u, cols] += alpha * dz[v, cols]
    das, dWs = [], []
    own = np.zeros((V, 1))
    own[lo:hi] = 1
    grad_h = np.zeros_like(h)
    for l in range(L):
        for k in range(K):
            cols = slice(k * d, (k + 1) * d)
            dP[l][:, cols] += ds_src[:, l, k:k + 1] * As[l][k, :d] + own * ds_tgt[:, l, k:k + 1] * As[l][k, d:]
        Pl = P[l].reshape(V, K, d)
        das.append(np.concatenate([(ds_src[:, l, :, None] * Pl).sum(0), (ds_tgt[:, l, :, None] * Pl).sum(0)], -1))
        dWs.append(h.T @ dP[l])
        grad_h += dP[l] @ Ws[l].T
    return grad_h, dWs, das


def _case(seed, V=24, D=6, K=2, d=3, L=3, E=60):
    rng = np.random.default_rng(seed)
    H = K * d
    adjs = [rng.integers(0, V, size=(E, 2)) for _ in range(L - 1)] + [np.zeros((0, 2), np.int64)]
    adjs[0][:14, 1] = 5          # target 5: a hub for chunk = 4
    adjs[1][:6, 1] = 5
    adjs[0][15] = adjs[0][14]    # duplicate
    adjs[1][7] = (9, 9)          # self-loop
    h = rng.uniform(-1, 1, (V, D))
    Ws = [rng.uniform(-0.7, 0.7, (D, H)) for _ in range(L)]
    As = [rng.uniform(-0.7, 0.7, (K, 2 * d)) for _ in range(L)]
    g = rng.uniform(-1, 1, (V, H))
    return adjs, h, Ws, As, g


def _autograd(adjs, h, Ws, As, g, act):
    L = len(adjs)
    leaves = [torch.from_numpy(x).requires_grad_() for x in [h] + Ws + As]
    out = r64.literal_autograd(leaves[0], [torch.from_numpy(a) for a in adjs], leaves[1:1 + L], leaves[1 + L:], act)
    out.backward(torch.from_numpy(g))
    z = lambda x, ref: x.grad.numpy() if x.grad is not None else np.zeros_like(ref)
    return leaves[0].grad.numpy(), [z(leaves[1 + l], Ws[l]) for l in range(L)], [z(leaves[1 + L + l], As[l]) for l in range(L)]


@pytest.mark.parametrize("act,chunk", [("tanh", 4), ("gelu", 7), ("relu", 1000), ("none", 3)])
def test_fused_steps_match_autograd(act, chunk):
    """Online walk with rescaling, hubs (more than `chunk` edges) combined in chunk order, source-keyed formulas."""
    adjs, h, Ws, As, g = _case(len(act) + chunk)
    ref_h, ref_W, ref_a = _autograd(adjs, h, Ws, As, g, act)
    grad_h, dWs, das = _fused(h, adjs, Ws, As, g, act, 0, h.shape[0], chunk)
    np.testing.assert_allclose(grad_h, ref_h, rtol=0, atol=1e-12)
    for a, b in zip(dWs + das, ref_W + ref_a):
        np.testing.assert_allclose(a, b, rtol=0, atol=1e-12)


def test_online_walk_rescales_when_the_maximum_grows():
    """Edges in increasing score order make the maximum grow at every edge: the walk still gives the exact softmax sums."""
    rng = np.random.default_rng(3)
    K, d, L = 1, 2, 2
    P = [rng.uniform(-1, 1, (6, 2)) for _ in range(L)]
    s_src = np.arange(6, dtype=np.float64).reshape(6, 1, 1).repeat(L, 1) * 0.9
    s_tgt_v = np.zeros((L, 1))
    dz_v = rng.uniform(-1, 1, 2)
    edges = [(0, 0), (0, 2), (1, 1), (1, 4), (1, 5)]
    m, den, G, A1, A2 = _walk(edges, P, s_src, s_tgt_v, dz_v, L, K, d)
    sc = np.array([_leaky(s_src[u, l, 0]) for l, u in edges])
    w = np.exp(sc - sc.max())
    da = np.array([dz_v @ P[l][u] for l, u in edges])
    lp = np.array([1.0 if s_src[u, l, 0] > 0 else LEAKY for l, u in edges])
    assert m[0] == sc.max() and np.isclose(den[0], w.sum(), rtol=1e-15) and np.isclose(G[0], (w * da).sum(), rtol=1e-15)
    for l in range(L):
        sel = np.array([e[0] == l for e in edges])
        assert np.isclose(A1[l, 0], (w * lp * da)[sel].sum(), rtol=1e-14)
        assert np.isclose(A2[l, 0], (w * lp)[sel].sum(), rtol=1e-14)


@pytest.mark.parametrize("bounds", [[(0, 10), (10, 24)], [(0, 5), (5, 6), (6, 24)], [(0, 8), (8, 8), (8, 24)]])
def test_target_range_contributions_sum_to_the_whole(bounds):
    adjs, h, Ws, As, g = _case(11)
    whole = _fused(h, adjs, Ws, As, g, "tanh", 0, 24, 4)
    parts = [_fused(h, adjs, Ws, As, g, "tanh", lo, hi, 4) for lo, hi in bounds]
    np.testing.assert_allclose(sum(p[0] for p in parts), whole[0], rtol=0, atol=1e-12)
    for i in (1, 2):
        for l in range(len(adjs)):
            np.testing.assert_allclose(sum(p[i][l] for p in parts), whole[i][l], rtol=0, atol=1e-12)
