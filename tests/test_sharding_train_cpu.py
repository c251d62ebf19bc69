"""Training on target-range shards, host side (world_size 2, gloo, float64 torch layers standing in for the CUDA ones):
reduce_scatter_node_grads is the adjoint of all_gather_node_states, gradients through gather_node_states equal
single-process autograd, and regather_saved_tables() gives the same gradients while saving only the rank's own rows.
The GPU tests of the same flow with the CUDA backward are in tests/test_gpu_shard_backward.py."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tf2_gnn_b200 import sharding


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _reference_layer(h, adjs, Ws, agg):
    """float64 RGCN layer on the whole graph (index_select / index_add_ form): normalised messages, tanh."""
    V = h.shape[0]
    out = torch.zeros((V, Ws[0].shape[1]), dtype=h.dtype)
    n = torch.zeros(V, dtype=h.dtype)
    for adj, W in zip(adjs, Ws):
        src, tgt = adj[:, 0].long(), adj[:, 1].long()
        c = torch.zeros(V, dtype=h.dtype).index_add_(0, tgt, torch.ones(len(tgt), dtype=h.dtype))
        m = (1.0 / (c.index_select(0, tgt) + 1e-7)).unsqueeze(-1) * (h.index_select(0, src) @ W)
        out = out.index_add(0, tgt, m)
        n = n.index_add(0, tgt, torch.ones(len(tgt), dtype=h.dtype))
    if agg == "mean":
        out = out / n.clamp(min=1).unsqueeze(-1)
    return torch.tanh(out)


def _shard_layer(h_full, adjs, Ws, lo, hi, agg):
    """The same layer for the owned targets [lo, hi) only, from the full source table: dense [hi-lo, V] per-type
    operators, so every saved tensor but the table has at most hi-lo rows (or a weight's rows)."""
    V = h_full.shape[0]
    out = torch.zeros((hi - lo, Ws[0].shape[1]), dtype=h_full.dtype)
    n = torch.zeros(hi - lo, dtype=h_full.dtype)
    for adj, W in zip(adjs, Ws):
        keep = (adj[:, 1] >= lo) & (adj[:, 1] < hi)
        src, tgt = adj[keep, 0].long(), adj[keep, 1].long() - lo
        A = torch.zeros((hi - lo, V), dtype=h_full.dtype).index_put_((tgt, src), torch.ones(len(src), dtype=h_full.dtype),
                                                                    accumulate=True)
        c = A.sum(dim=1, keepdim=True)
        out = out + ((A / (c + 1e-7)) @ h_full) @ W
        n = n + c[:, 0]
    if agg == "mean":
        out = out / n.clamp(min=1).unsqueeze(-1)
    return torch.tanh(out)


class _SavingShardLayer(torch.autograd.Function):
    """_shard_layer with the saving pattern of the CUDA layer hooks (_EdgeMLPLayerFunction, _GGNNFunction): the input
    table and the weights are saved, everything else is recomputed in backward."""

    @staticmethod
    def forward(ctx, h_full, lo, hi, agg, adjs, *Ws):
        ctx.args = (lo, hi, agg, adjs)
        ctx.save_for_backward(h_full, *Ws)
        return _shard_layer(h_full, adjs, Ws, lo, hi, agg)

    @staticmethod
    def backward(ctx, g):
        h_full, *Ws = ctx.saved_tensors
        lo, hi, agg, adjs = ctx.args
        with torch.enable_grad():
            leaves = [h_full.detach().requires_grad_()] + [w.detach().requires_grad_() for w in Ws]
            out = _shard_layer(leaves[0], adjs, leaves[1:], lo, hi, agg)
            grads = torch.autograd.grad(out, leaves, g)
        return (grads[0], None, None, None, None, *grads[1:])


class _RecordingRegather(sharding.regather_saved_tables):
    def __init__(self):
        super().__init__()
        self.saved_rows, self.regathered = [], 0

    def _pack(self, t):
        s = super()._pack(t)
        if isinstance(s, torch.Tensor):
            self.saved_rows.append(int(s.shape[0]) if s.dim() else 0)
        else:
            self.regathered += 1
        return s


def _check_adjoint(rank, world, rng):
    ok = []
    for V, bounds in [(7, [(0, 3), (3, 7)]), (9, [(0, 9), (9, 9)]), (8, [(0, 4), (4, 8)]), (5, [(0, 0), (0, 5)])]:
        D = 3
        lo, hi = bounds[rank]
        x = torch.from_numpy(rng.standard_normal((hi - lo, D)))     # rank-specific (rng advanced per rank below)
        y = torch.from_numpy(rng.standard_normal((V, D)))
        lhs = (sharding.all_gather_node_states(x, bounds) * y).sum()
        rs = sharding.reduce_scatter_node_grads(y, bounds)
        assert tuple(rs.shape) == (hi - lo, D)
        rhs = (x * rs).sum()
        t = torch.stack([lhs, rhs])
        dist.all_reduce(t)
        ok.append(bool(abs(float(t[0] - t[1])) <= 1e-12 * max(1.0, abs(float(t[0])))))
    return ok


def _worker(rank, world, port, tmp):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        ok = _check_adjoint(rank, world, np.random.default_rng(100 + rank))
        rng = np.random.default_rng(5)       # same graph and weights on every rank
        V, D, H, L = 12, 4, 4, 2
        adjs = [torch.from_numpy(rng.integers(0, V, (30, 2)).astype(np.int64)) for _ in range(L)]
        X = rng.uniform(-1, 1, (V, D))
        Ws = [[rng.uniform(-0.8, 0.8, (D if k == 0 else H, H)) for _ in range(L)] for k in range(2)]
        G = rng.uniform(-1, 1, (V, H))
        bounds = [(0, 5), (5, 12)]
        lo, hi = bounds[rank]
        for agg in ("sum", "mean"):
            # single-process autograd
            Xr = torch.from_numpy(X).requires_grad_()
            Wr = [[torch.from_numpy(w).requires_grad_() for w in ws] for ws in Ws]
            h = Xr
            for k in range(2):
                h = _reference_layer(h, adjs, Wr[k], agg)
            (h * torch.from_numpy(G)).sum().backward()
            results = []
            for regather in (False, True):
                x_local = torch.from_numpy(X[lo:hi].copy()).requires_grad_()
                Wl = [[torch.from_numpy(w).requires_grad_() for w in ws] for ws in Ws]
                rec = _RecordingRegather() if regather else None
                h_local = x_local
                if rec:
                    rec.__enter__()
                for k in range(2):
                    h_local = _SavingShardLayer.apply(sharding.gather_node_states(h_local, bounds), lo, hi, agg, adjs,
                                                      *Wl[k])
                if rec:
                    rec.__exit__(None, None, None)
                    ok.append(rec.regathered >= 2 and max(rec.saved_rows) <= hi - lo)
                (h_local * torch.from_numpy(G[lo:hi])).sum().backward()
                grads = [w.grad.clone() for ws in Wl for w in ws]
                for g in grads:
                    dist.all_reduce(g)           # weight gradients are partial per rank
                results.append((x_local.grad.clone(), grads))
                ok.append(bool(torch.allclose(x_local.grad, Xr.grad[lo:hi], rtol=0, atol=1e-12)))
                ok.append(all(torch.allclose(g, w.grad, rtol=0, atol=1e-12)
                              for g, w in zip(grads, [w for ws in Wr for w in ws])))
            # the re-gather changes what is saved, not what is computed
            ok.append(torch.equal(results[0][0], results[1][0]) and
                      all(torch.equal(a, b) for a, b in zip(results[0][1], results[1][1])))
        np.save(os.path.join(tmp, f"ok{rank}.npy"), np.array(ok))
    finally:
        dist.destroy_process_group()


def test_shard_training_gloo_world_size_2(tmp_path):
    port = _free_port()
    mp.spawn(_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    for r in range(2):
        ok = np.load(os.path.join(str(tmp_path), f"ok{r}.npy"))
        assert ok.size >= 10 and ok.all(), ok
