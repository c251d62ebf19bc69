"""Task losses, the optimizer step and the learning-rate schedule of tf2_gnn.models on the library's kernels
(csrc/task_ops.cu, csrc/optimizer.cu).

Each loss is a torch.autograd.Function over a forward and a backward C-ABI entry; its scalars stay on the device and the
backward reads the upstream gradient from there, so a training step does not wait on the host.  torch is the autograd
tape and allocates the outputs; it does no arithmetic here.
"""
from __future__ import annotations

import ctypes
from typing import List, Optional, Sequence, Tuple

import torch

from .. import _ffi
from ..runtime import stream_ptr


def _scalar(like: torch.Tensor, dtype=torch.float32, n: Tuple[int, ...] = ()) -> torch.Tensor:
    return torch.empty(n, dtype=dtype, device=like.device)


class _NodeMulticlassLoss(torch.autograd.Function):
    """tf.reduce_mean(tf.reduce_sum(sigmoid_cross_entropy_with_logits(logits, labels), -1)) and micro_f1
    (node_multiclass_task.py:10-23, 60-68).  Returns (loss, f1_score, int64 counts (tp, fp, fn))."""

    @staticmethod
    def forward(ctx, logits, labels):
        logits, labels = logits.contiguous(), labels.contiguous()
        V, C = int(logits.shape[0]), int(logits.shape[1])
        loss, f1, counts = _scalar(logits), _scalar(logits), _scalar(logits, torch.int64, (3,))
        _ffi.check(_ffi.lib().tfgnn_b200_node_multiclass_loss_fwd(logits.data_ptr(), labels.data_ptr(), V, C, loss.data_ptr(),
                                                                  f1.data_ptr(), counts.data_ptr(), stream_ptr()))
        ctx.save_for_backward(logits, labels)
        ctx.mark_non_differentiable(f1, counts)
        return loss, f1, counts

    @staticmethod
    def backward(ctx, g, _g_f1, _g_counts):
        logits, labels = ctx.saved_tensors
        grad = torch.empty_like(logits)
        _ffi.check(_ffi.lib().tfgnn_b200_node_multiclass_loss_bwd(logits.data_ptr(), labels.data_ptr(), int(logits.shape[0]),
                                                                  int(logits.shape[1]), g.contiguous().data_ptr(),
                                                                  grad.data_ptr(), stream_ptr()))
        return grad, None


class _ShardNodeMulticlassLoss(torch.autograd.Function):
    """_NodeMulticlassLoss over a batch cut by target range: the rank's raw sum and counts (…_loss_partial), all-gathered and
    merged in rank order over the batch's row count (…_loss_merge), so every rank gets the same (loss, f1_score, counts).
    The backward needs no collective: a rank's logits enter its own partial only (…_loss_bwd_rows with 1 / total rows)."""

    @staticmethod
    def forward(ctx, logits, labels, shard):
        from .. import sharding
        logits, labels = logits.contiguous(), labels.contiguous()
        V, C = int(logits.shape[0]), int(logits.shape[1])
        lib = _ffi.lib()
        part_sum, part_counts = _scalar(logits, n=(1,)), _scalar(logits, torch.int64, (3,))
        _ffi.check(lib.tfgnn_b200_node_multiclass_loss_partial(logits.data_ptr(), labels.data_ptr(), V, C,
                                                               part_sum.data_ptr(), part_counts.data_ptr(), stream_ptr()))
        sums = sharding.all_gather_stacked(part_sum, shard.group).contiguous()
        counts_all = sharding.all_gather_stacked(part_counts, shard.group).contiguous()
        loss, f1, counts = _scalar(logits), _scalar(logits), _scalar(logits, torch.int64, (3,))
        _ffi.check(lib.tfgnn_b200_node_multiclass_loss_merge(sums.data_ptr(), counts_all.data_ptr(), int(sums.shape[0]),
                                                             shard.num_nodes, loss.data_ptr(), f1.data_ptr(),
                                                             counts.data_ptr(), stream_ptr()))
        ctx.save_for_backward(logits, labels)
        ctx.total_rows = shard.num_nodes
        ctx.mark_non_differentiable(f1, counts)
        return loss, f1, counts

    @staticmethod
    def backward(ctx, g, _g_f1, _g_counts):
        logits, labels = ctx.saved_tensors
        grad = torch.empty_like(logits)
        _ffi.check(_ffi.lib().tfgnn_b200_node_multiclass_loss_bwd_rows(
            logits.data_ptr(), labels.data_ptr(), int(logits.shape[0]), int(logits.shape[1]), ctx.total_rows,
            g.contiguous().data_ptr(), grad.data_ptr(), stream_ptr()))
        return grad, None, None


class _CountOnce(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, rank):
        ctx.rank = rank
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return (g if ctx.rank == 0 else torch.zeros_like(g)), None


def count_once(x: torch.Tensor, shard) -> torch.Tensor:
    """The identity, whose backward passes the gradient on rank 0 and exact zeros on every other rank.  For a value that is
    the same on every rank of a target-range shard (a merged per-graph row and what a replicated head computes from it): its
    loss is then counted once when the readout's backward sums the ranks' gradients, and the head's weight gradients are
    rank 0's after sharding.sum_gradient_list_over_ranks.  shard None: the identity."""
    if shard is None:
        return x
    return _CountOnce.apply(x, shard.rank)


class _GraphRegressionLoss(torch.autograd.Function):
    """tf.losses.mean_squared_error / mean_absolute_error over the batch's graphs (graph_regression_task.py:152-166).
    Returns (mse, mae)."""

    @staticmethod
    def forward(ctx, pred, target):
        pred, target = pred.contiguous(), target.contiguous()
        mse, mae = _scalar(pred), _scalar(pred)
        _ffi.check(_ffi.lib().tfgnn_b200_graph_regression_loss_fwd(pred.data_ptr(), target.data_ptr(), int(pred.shape[0]),
                                                                   mse.data_ptr(), mae.data_ptr(), stream_ptr()))
        ctx.save_for_backward(pred, target)
        ctx.mark_non_differentiable(mae)
        return mse, mae

    @staticmethod
    def backward(ctx, g, _g_mae):
        pred, target = ctx.saved_tensors
        grad = torch.empty_like(pred)
        _ffi.check(_ffi.lib().tfgnn_b200_graph_regression_loss_bwd(pred.data_ptr(), target.data_ptr(), int(pred.shape[0]),
                                                                   g.contiguous().data_ptr(), grad.data_ptr(), stream_ptr()))
        return grad, None


class _GraphBinaryLoss(torch.autograd.Function):
    """reduce_mean(keras binary_crossentropy(target, prob, from_logits=False)) and the number of graphs whose rounded
    probability equals the target (graph_binary_classification_task.py:33-58).  Returns (loss, int64 num_correct)."""

    @staticmethod
    def forward(ctx, prob, target):
        prob, target = prob.contiguous(), target.contiguous()
        loss, correct = _scalar(prob), _scalar(prob, torch.int64)
        _ffi.check(_ffi.lib().tfgnn_b200_graph_binary_loss_fwd(prob.data_ptr(), target.data_ptr(), int(prob.shape[0]),
                                                               loss.data_ptr(), correct.data_ptr(), stream_ptr()))
        ctx.save_for_backward(prob, target)
        ctx.mark_non_differentiable(correct)
        return loss, correct

    @staticmethod
    def backward(ctx, g, _g_correct):
        prob, target = ctx.saved_tensors
        grad = torch.empty_like(prob)
        _ffi.check(_ffi.lib().tfgnn_b200_graph_binary_loss_bwd(prob.data_ptr(), target.data_ptr(), int(prob.shape[0]),
                                                               g.contiguous().data_ptr(), grad.data_ptr(), stream_ptr()))
        return grad, None


def node_multiclass_loss(logits: torch.Tensor, labels: torch.Tensor, shard=None):
    """(loss, f1_score, counts (tp, fp, fn)) as 0-d / [3] CUDA tensors.  shard (sharding.TargetRangeShard): logits and labels
    are the rank's rows of the batch; the results are those of the whole batch, the same bits on every rank (collective in
    the forward only)."""
    if shard is not None:
        return _ShardNodeMulticlassLoss.apply(logits, labels.to(torch.float32), shard)
    return _NodeMulticlassLoss.apply(logits, labels.to(torch.float32))


def graph_regression_loss(pred: torch.Tensor, target: torch.Tensor):
    """(mse, mae) as 0-d CUDA tensors."""
    return _GraphRegressionLoss.apply(pred, target.to(torch.float32))


def graph_binary_loss(prob: torch.Tensor, target: torch.Tensor):
    """(loss, num_correct) as 0-d CUDA tensors."""
    return _GraphBinaryLoss.apply(prob, target.to(torch.float32))


def sigmoid(x: torch.Tensor) -> torch.Tensor:
    """tf.nn.sigmoid, differentiable (tfgnn_b200_activation / _activation_bwd)."""
    from ..layers.differentiable import _ActivationFunction
    return _ActivationFunction.apply(x, _ffi.ACT_SIGMOID)


# ---- learning rate ----------------------------------------------------------------------------------------------
class PolynomialWarmupAndDecaySchedule:
    """tf2_gnn/utils/polynomial_warmup_and_decay_schedule.py, evaluated on the host at the optimizer's step counter."""

    def __init__(self, learning_rate: float, warmup_steps: int, decay_steps: int, initial_learning_rate: float,
                 final_learning_rate: float, power: float = 1.0, name: Optional[str] = None):
        self.learning_rate = learning_rate
        self.initial_learning_rate = initial_learning_rate
        self.final_learning_rate = final_learning_rate
        self.warmup_steps = warmup_steps
        self.decay_steps = decay_steps
        self.power = power
        self.name = name

    def __call__(self, step: int) -> float:
        if step <= self.warmup_steps:
            return ((self.learning_rate - self.initial_learning_rate) * (step / self.warmup_steps) ** self.power
                    + self.initial_learning_rate)
        effective_step = min(step - self.warmup_steps, self.decay_steps)
        return ((self.learning_rate - self.final_learning_rate) * (1 - effective_step / self.decay_steps) ** self.power
                + self.final_learning_rate)


# ---- optimizer --------------------------------------------------------------------------------------------------
class Optimizer:
    """tf.keras.optimizers.{SGD, RMSprop, Adam} (graph_task_model.py:262-276) with Keras' defaults (epsilon 1e-7,
    beta_1 0.9, beta_2 0.999), plus the gradient clipping of _apply_gradients (:296-322).  One apply_gradients call is one
    tfgnn_b200_optimizer_step: a single launch over all variables (two with norm clipping).  `learning_rate` is a float
    or a callable of the 0-based step counter (`iterations`, as Keras evaluates its schedules)."""

    def __init__(self, name: str, learning_rate, momentum: float = 0.0, rho: float = 0.9, clip_value: Optional[float] = None,
                 clip_norm: Optional[float] = None, clip_global_norm: Optional[float] = None):
        name = name.lower()
        if name not in _ffi.OPTIMIZER:
            raise Exception('Unknown optimizer "%s".' % name)
        self.kind = _ffi.OPTIMIZER[name]
        self.learning_rate = learning_rate
        self.momentum = float(momentum) if name != "adam" else 0.0
        self.rho = float(rho)
        self.clip_mode, self.clip = _ffi.CLIP_NONE, 0.0
        if clip_value is not None:
            self.clip_mode, self.clip = _ffi.CLIP_VALUE, float(clip_value)
        elif clip_norm is not None:
            self.clip_mode, self.clip = _ffi.CLIP_NORM, float(clip_norm)
        elif clip_global_norm is not None:
            self.clip_mode, self.clip = _ffi.CLIP_GLOBAL_NORM, float(clip_global_norm)
        self.iterations = 0
        self._slots = {}   # id(variable tensor) -> (variable tensor, slot_a, slot_b); the tensor pins the id

    def _lr(self) -> float:
        lr = self.learning_rate
        return float(lr(self.iterations) if callable(lr) else lr)

    def _needs_slots(self) -> Tuple[bool, bool]:
        if self.kind == _ffi.OPTIMIZER["adam"]:
            return True, True
        if self.kind == _ffi.OPTIMIZER["rmsprop"]:
            return True, self.momentum > 0.0
        return self.momentum > 0.0, False

    def slots(self, var: torch.Tensor) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
        """The variable's slots (zeros, created on the first step that updates it, as Keras' _create_slots)."""
        key = id(var)
        if key not in self._slots:
            need_a, need_b = self._needs_slots()
            self._slots[key] = (var, torch.zeros_like(var, memory_format=torch.contiguous_format) if need_a else None,
                                torch.zeros_like(var, memory_format=torch.contiguous_format) if need_b else None)
        return self._slots[key][1:]

    def apply_gradients(self, grads_and_vars: Sequence[Tuple[Optional[torch.Tensor], torch.Tensor]]) -> None:
        """w <- update(w, clip(g)) for every pair whose gradient is not None; then iterations += 1."""
        pairs = [(g, v) for g, v in grads_and_vars if g is not None]
        if pairs:
            grads = [g.detach().contiguous() for g, _ in pairs]
            for _, v in pairs:
                if not v.is_contiguous():
                    raise ValueError("optimizer: variables must be contiguous")
            slots = [self.slots(v) for _, v in pairs]
            params = [v.detach() for _, v in pairs]
            n = len(pairs)
            sizes = (ctypes.c_int64 * n)(*[p.numel() for p in params])
            _ffi.check(_ffi.lib().tfgnn_b200_optimizer_step(
                self.kind, n, _ffi.ptr_array(params), _ffi.ptr_array(grads), _ffi.ptr_array([s[0] for s in slots]),
                _ffi.ptr_array([s[1] for s in slots]), sizes, self._lr(), self.momentum, self.rho, self.iterations,
                self.clip_mode, self.clip, stream_ptr()))
        self.iterations += 1
