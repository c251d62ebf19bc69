"""Float64 reference of the RGAT layer (rgat.py:91-163) and of its gradients, for tests at any size.

The math is the backward's (DESIGN.md §6): with P_l = h W_l, x_e = s_src[u,l,k] + s_tgt[v,l,k], sigma_e = leaky(x_e),
alpha_e = softmax over all edges into v (all types jointly) per head, o[v]_k = sum_e alpha_e P_l[u]_k, out = act(o), and
dZ = dOut * act'(o):
    g[v,k] = dZ[v]_k . o[v]_k,   dx_e = alpha_e (dZ[v]_k . P_l[u]_k - g[v,k]) leaky'(x_e)
    dP_l[u] = sum_{e leaving u} alpha_e dZ[v] + ds_src[u,l] a_l[:, :d] + ds_tgt[u,l] a_l[:, d:]
    da_l = [sum_u ds_src[u,l,k] P_l[u]_k | sum_v ds_tgt[v,l,k] P_l[v]_k],  dW_l = h^T dP_l,  grad_h = sum_l dP_l W_l^T
It works one edge type at a time and holds the per-edge terms of at most `chunk` edges at once: no [E, H] array is built,
so it runs on the device at bench.py's cfg3 size.  `literal_autograd` is the reference's literal op order for autograd."""
import torch

LEAKY = 0.2


def _act(name, z):
    """(act(z), act'(z)) in float64 (tf2_gnn/utils/param_helpers.py; gelu: the tanh approximation)."""
    if name in (None, "none", "linear"):
        return z, torch.ones_like(z)
    if name == "relu":
        return torch.relu(z), (z > 0).to(z.dtype)
    if name == "tanh":
        y = torch.tanh(z)
        return y, 1 - y * y
    if name == "gelu":
        c = 0.7978845608028654
        t = torch.tanh(c * (z + 0.044715 * z ** 3))
        return 0.5 * z * (1 + t), 0.5 * (1 + t) + 0.5 * z * (1 - t * t) * c * (1 + 3 * 0.044715 * z * z)
    raise ValueError(name)


def act_autograd(name, z):
    return _act(name, z)[0]


def _chunks(a, chunk):
    for c0 in range(0, a.shape[0], chunk):
        yield a[c0:c0 + chunk, 0].long(), a[c0:c0 + chunk, 1].long()


def forward_backward(h, adjs, Ws, As, g, act, chunk=1 << 20, grad_h_rows=None):
    """float64 (out, grad_h, [dW_l], [da_l], min |x_e|) of the layer for dOut = g.  h [V, D], adjs: [E_l, 2] int tensors
    (source, target), Ws [D, H], As [K, 2d], g [V, H], all on one device.  grad_h_rows: only these rows of grad_h."""
    h = h.double()
    V, H = h.shape[0], Ws[0].shape[1]
    K = As[0].shape[0]
    d = H // K
    P = [h @ W.double() for W in Ws]
    A = [a.double() for a in As]
    s_src = [(Pl.view(V, K, d) * a[:, :d]).sum(-1) for Pl, a in zip(P, A)]
    s_tgt = [(Pl.view(V, K, d) * a[:, d:]).sum(-1) for Pl, a in zip(P, A)]
    m = torch.full((V, K), -torch.inf, dtype=torch.float64, device=h.device)
    margin = torch.inf
    for l, adj in enumerate(adjs):
        for s, t in _chunks(adj, chunk):
            x = s_src[l][s] + s_tgt[l][t]
            margin = min(margin, float(x.abs().min()))
            m.scatter_reduce_(0, t[:, None].expand(-1, K), torch.where(x > 0, x, LEAKY * x), reduce="amax")
    den = torch.zeros((V, K), dtype=torch.float64, device=h.device)
    o = torch.zeros((V, K, d), dtype=torch.float64, device=h.device)
    for l, adj in enumerate(adjs):
        for s, t in _chunks(adj, chunk):
            x = s_src[l][s] + s_tgt[l][t]
            w = torch.exp(torch.where(x > 0, x, LEAKY * x) - m[t])
            den.index_add_(0, t, w)
            o.index_add_(0, t, w[:, :, None] * P[l][s].view(-1, K, d))
    inv = torch.where(den > 0, 1.0 / den.clamp(min=1e-300), torch.zeros_like(den))
    o = o * inv[:, :, None]
    out, dact = _act(act, o.reshape(V, H))
    dz = (g.double() * dact).view(V, K, d)
    gk = (dz * o).sum(-1)
    rows = torch.arange(V, device=h.device) if grad_h_rows is None else grad_h_rows
    grad_h = torch.zeros((rows.numel(), h.shape[1]), dtype=torch.float64, device=h.device)
    dWs, das = [], []
    for l, adj in enumerate(adjs):
        dP = torch.zeros((V, K, d), dtype=torch.float64, device=h.device)
        ds_src = torch.zeros((V, K), dtype=torch.float64, device=h.device)
        ds_tgt = torch.zeros((V, K), dtype=torch.float64, device=h.device)
        for s, t in _chunks(adj, chunk):
            x = s_src[l][s] + s_tgt[l][t]
            alpha = torch.exp(torch.where(x > 0, x, LEAKY * x) - m[t]) * inv[t]
            da = (dz[t] * P[l][s].view(-1, K, d)).sum(-1)
            dx = alpha * (da - gk[t]) * torch.where(x > 0, torch.ones_like(x), torch.full_like(x, LEAKY))
            dP.index_add_(0, s, alpha[:, :, None] * dz[t])
            ds_src.index_add_(0, s, dx)
            ds_tgt.index_add_(0, t, dx)
        dP += ds_src[:, :, None] * A[l][:, :d] + ds_tgt[:, :, None] * A[l][:, d:]
        Pl = P[l].view(V, K, d)
        das.append(torch.cat([(ds_src[:, :, None] * Pl).sum(0), (ds_tgt[:, :, None] * Pl).sum(0)], -1))
        dP = dP.reshape(V, H)
        dWs.append(h.T @ dP)
        grad_h += dP[rows] @ Ws[l].double().T
        del dP
    return out, grad_h, dWs, das, margin


def literal_autograd(h, adjs, Ws, As, act):
    """The reference's literal op order (rgat.py:91-163) on float64 leaves, for torch autograd: per-edge gathers, the
    concatenated messages, the einsum scores, the segment softmax over all types jointly, the weighted sum."""
    V, H = h.shape[0], Ws[0].shape[1]
    K = As[0].shape[0]
    d = H // K
    msgs, scs, ids = [], [], []
    for l, a in enumerate(adjs):
        src, tgt = a[:, 0].long(), a[:, 1].long()
        ps = (h[src] @ Ws[l]).reshape(-1, K, d)
        pt = (h[tgt] @ Ws[l]).reshape(-1, K, d)
        x = torch.einsum("vki,ki->vk", torch.cat([ps, pt], -1), As[l])
        sc = torch.where(x > 0, x, LEAKY * x)   # F.leaky_relu would round the slope to float32
        msgs.append(ps)
        scs.append(sc)
        ids.append(tgt)
    M, S, T = torch.cat(msgs), torch.cat(scs), torch.cat(ids)
    mx = torch.full((V, K), -1e300, dtype=torch.float64).scatter_reduce(0, T[:, None].expand(-1, K), S, reduce="amax")
    e = torch.exp(S - mx[T])
    Z = torch.zeros((V, K), dtype=torch.float64).index_add(0, T, e)
    alpha = e / Z[T]
    agg = torch.zeros((V, K, d), dtype=torch.float64).index_add(0, T, alpha[:, :, None] * M).reshape(V, H)
    return act_autograd(act, agg)
