"""Device plumbing between the tf2_gnn-shaped Python API and the C ABI.

PyTorch is used here only as the carrier of device memory and CUDA streams (the reference's
carrier, TensorFlow, is not installed in this image; see tf_adapter.py for the DLPack bridge).
No arithmetic of the message-passing path is done with torch ops.
"""
from __future__ import annotations

import weakref
from ctypes import byref, c_int32, c_int64, c_void_p
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _ffi


def require_cuda() -> torch.device:
    if not torch.cuda.is_available():
        raise RuntimeError(
            "tf2_gnn_b200 needs a CUDA device (sm_90a): the message-passing path has no CPU fallback")
    return torch.device("cuda", torch.cuda.current_device())


def stream_ptr() -> int:
    return int(torch.cuda.current_stream().cuda_stream)


def to_device_f32(x, device: Optional[torch.device] = None) -> torch.Tensor:
    """float32, contiguous, on the GPU (host inputs are copied: that copy is part of e2e timing)."""
    device = device or require_cuda()
    if isinstance(x, torch.Tensor):
        t = x
    elif hasattr(x, "__dlpack__") and not isinstance(x, np.ndarray):
        t = torch.from_dlpack(x)
    else:
        t = torch.from_numpy(np.ascontiguousarray(np.asarray(x, dtype=np.float32)))
    if t.dtype != torch.float32:
        t = t.to(torch.float32)
    if t.device != device:
        t = t.to(device, non_blocking=True)
    return t.contiguous()


def to_device_adj(a, device: Optional[torch.device] = None) -> torch.Tensor:
    """int32 [E,2] contiguous on the GPU (graph_dataset.py:244 gives int32[0,2] for empty types)."""
    device = device or require_cuda()
    if isinstance(a, torch.Tensor):
        t = a
    elif hasattr(a, "__dlpack__") and not isinstance(a, np.ndarray):
        t = torch.from_dlpack(a)
    else:
        t = torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.int32).reshape(-1, 2)))
    if (isinstance(a, torch.Tensor) and a.dtype == torch.int32 and a.device == device and a.dim() == 2
            and a.shape[1] == 2 and a.is_contiguous()):
        return a  # same object: lets prepared_batch_for() recognise the tensor across layers / calls
    if t.dtype != torch.int32:
        t = t.to(torch.int32)
    if t.device != device:
        t = t.to(device, non_blocking=True)
    t = t.reshape(-1, 2) if t.numel() else t.reshape(0, 2)
    return t.contiguous()


class PreparedBatch:
    """Owner of a tfgnn_batch_t: the per-batch CSR (sorted by type,target) + in-degree, built once
    and shared by all layers (the adjacency is layer-invariant, gnn.py:278,301)."""

    def __init__(self, adjacency_lists: Sequence[torch.Tensor], num_nodes: int, validate: bool = False,
                 target_range: Optional[Tuple[int, int]] = None, transpose: bool = False,
                 transpose_owned: bool = False):
        """target_range=(lo, hi): this batch is one rank's target-range shard of a graph with `num_nodes`
        nodes (sharding.py case 2); layer outputs then have hi-lo rows and `node_embeddings` passed to the
        layers must be the full [num_nodes, D] table.
        transpose / transpose_owned: the backward CSR (TFGNN_PREPARE_TRANSPOSE / TFGNN_PREPARE_TRANSPOSE_OWNED); use
        transposed() rather than building one directly."""
        self.adjacency_lists = tuple(adjacency_lists)  # keep caller memory alive (atomic path reads it)
        self.num_source_nodes = int(num_nodes)
        self.target_range = (0, int(num_nodes)) if target_range is None else (int(target_range[0]), int(target_range[1]))
        self.num_nodes = self.target_range[1] - self.target_range[0]
        self.num_edge_types = len(self.adjacency_lists)
        if self.num_edge_types > _ffi.MAX_EDGE_TYPES:
            raise ValueError(f"at most {_ffi.MAX_EDGE_TYPES} edge types are supported")
        self.num_edges = [int(a.shape[0]) for a in self.adjacency_lists]
        self._handle = c_void_p()
        ptrs = _ffi.ptr_array(self.adjacency_lists)
        counts = (c_int64 * max(self.num_edge_types, 1))(*self.num_edges)
        _ffi.check(_ffi.lib().tfgnn_b200_prepare_sharded(
            ptrs, counts, self.num_edge_types, self.num_source_nodes, self.target_range[0], self.num_nodes,
            (_ffi.PREPARE_VALIDATE if validate else 0) | (_ffi.PREPARE_TRANSPOSE if transpose else 0)
            | (_ffi.PREPARE_TRANSPOSE_OWNED if transpose_owned else 0),
            byref(self._handle), stream_ptr()))
        self._transposed: Optional["PreparedBatch"] = None
        self._finalizer = weakref.finalize(self, PreparedBatch._free, self._handle.value)

    @staticmethod
    def _free(handle):
        try:
            if handle:
                _ffi.lib().tfgnn_b200_free_batch(c_void_p(handle))
        except Exception:
            pass

    @property
    def handle(self) -> c_void_p:
        return self._handle

    def transposed(self) -> "PreparedBatch":
        """The same edges keyed by SOURCE (built lazily, once): the CSR of the backward pass.  On a target-range shard it
        holds the edges into the owned targets, keyed by global source, with local target ids
        (TFGNN_PREPARE_TRANSPOSE_OWNED); its csr() then has L * num_source_nodes segments."""
        if self._transposed is None:
            if self.target_range != (0, self.num_source_nodes):
                self._transposed = PreparedBatch(self.adjacency_lists, self.num_source_nodes,
                                                 target_range=self.target_range, transpose_owned=True)
            else:
                self._transposed = PreparedBatch(self.adjacency_lists, self.num_source_nodes, transpose=True)
        return self._transposed

    def in_degree(self) -> torch.Tensor:
        """float32 [L, V] — calculate_type_to_num_incoming_edges (message_passing.py:230-263)."""
        out = torch.empty((self.num_edge_types, self.num_nodes), dtype=torch.float32, device=require_cuda())
        _ffi.check(_ffi.lib().tfgnn_b200_in_degree(self._handle, out.data_ptr(), stream_ptr()))
        return out

    def csr(self) -> Tuple[torch.Tensor, torch.Tensor]:
        """Copies of (row_ptr int32[L*V+1], src_sorted int32[M]) for inspection/tests."""
        V, L, M = c_int64(), c_int32(), c_int64()
        rp, ss = c_void_p(), c_void_p()
        _ffi.check(_ffi.lib().tfgnn_b200_batch_info(self._handle, byref(V), byref(L), byref(M), byref(rp), byref(ss)))
        n_seg = V.value * L.value
        dev = require_cuda()
        row_ptr = torch.empty(n_seg + 1, dtype=torch.int32, device=dev)
        src = torch.empty(M.value, dtype=torch.int32, device=dev)
        _ffi.check(_ffi.lib().tfgnn_b200_batch_export_csr(self._handle, row_ptr.data_ptr(), src.data_ptr(),
                                                          stream_ptr()))
        return row_ptr, src


class HostPipeline:
    """Software pipeline for callers whose batches live in (pinned) HOST memory.

    One step = H2D of the step's inputs, per-batch prepare, the layer call(s) and the D2H of the result.  Steps are
    issued round-robin on `depth` CUDA streams, so the D2H of step i overlaps the H2D of step i+1 (PCIe is full
    duplex) and both overlap the kernels; every step still performs all of its own copies.  The reference overlaps
    host batch construction with the step in the same spirit (DoubleBufferedIterator, graph_dataset.py:292-295).

        pipe = HostPipeline(lambda batch: layer(batch), depth=2)
        for batch, out_host in work:            # out_host: pinned torch tensor the result is copied into
            pipe.submit(batch, out_host)        # returns immediately; at most `depth` steps are in flight
        pipe.drain()                            # all results have landed in their out_host buffers
    """

    def __init__(self, step_fn, depth: int = 2):
        require_cuda()
        self.step_fn = step_fn
        self.depth = max(1, int(depth))
        self.streams = [torch.cuda.Stream() for _ in range(self.depth)]
        self.done: List[Optional[torch.cuda.Event]] = [None] * self.depth
        self._keep: List[Optional[object]] = [None] * self.depth
        self._i = 0

    def submit(self, batch, out_host: torch.Tensor) -> None:
        slot = self._i % self.depth
        self._i += 1
        if self.done[slot] is not None:
            self.done[slot].synchronize()       # the slot's previous result has landed: its buffers may be reused
        s = self.streams[slot]
        with torch.cuda.stream(s):
            out = self.step_fn(batch)
            out_host.copy_(out, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(s)
        self.done[slot] = ev
        self._keep[slot] = out                  # keeps the device result alive until its D2H copy has completed

    def drain(self) -> None:
        for ev in self.done:
            if ev is not None:
                ev.synchronize()
        self._keep = [None] * self.depth


_cache: List[Tuple[tuple, "weakref.ref", PreparedBatch]] = []
_CACHE_SIZE = 2


def prepared_batch_for(adjacency_lists: Sequence[torch.Tensor], num_nodes: int) -> PreparedBatch:
    """Prepared batch for these adjacency tensors, reused while the SAME tensor objects (same
    python identity and in-place version) are passed again — e.g. by each layer of a GNN stack."""
    key = tuple((id(a), a._version, a.data_ptr(), int(a.shape[0])) for a in adjacency_lists) + (int(num_nodes),)
    for k, refs, pb in _cache:
        if k == key and all(r() is a for r, a in zip(refs, adjacency_lists)):
            return pb
    pb = PreparedBatch(adjacency_lists, num_nodes)
    refs = tuple(weakref.ref(a) for a in adjacency_lists)
    _cache.insert(0, (key, refs, pb))
    del _cache[_CACHE_SIZE:]
    return pb


def clear_prepared_batch_cache() -> None:
    del _cache[:]
