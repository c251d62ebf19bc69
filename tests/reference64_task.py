"""float64 restatement of the task losses, their gradients and metrics, the Keras optimizers, the gradient clipping and the
learning-rate schedule of tf2_gnn.models (node_multiclass_task.py, graph_regression_task.py,
graph_binary_classification_task.py, graph_task_model.py:224-324, utils/polynomial_warmup_and_decay_schedule.py), in
numpy.  The kernels of csrc/task_ops.cu and csrc/optimizer.cu are checked against it."""
import math

import numpy as np

# Keras hands its hyper-parameters to the training ops as float32 tensors: the rules run on those values (1 - 0.999f is
# 1.3e-5 away from 0.001, which moves an Adam step of a zero-initialised bias by as much)
F32 = lambda v: float(np.float32(v))   # noqa: E731
EPS = F32(1e-7)       # Keras backend.epsilon() / optimizer epsilon
BETA_1, BETA_2 = F32(0.9), F32(0.999)


def _sigmoid32(x):
    x = np.asarray(x, np.float32)
    with np.errstate(over="ignore"):
        return (np.float32(1) / (np.float32(1) + np.exp(-x))).astype(np.float32)


# ---- losses -------------------------------------------------------------------------------------------------------
def node_multiclass_loss(logits, labels):
    """(loss, grad_logits for an upstream gradient of 1, (tp, fp, fn), f1).  loss = mean over nodes of the summed
    tf.nn.sigmoid_cross_entropy_with_logits; the prediction is rint(sigmoid_f32(x)) (a logit of 0 predicts 0)."""
    x = np.asarray(logits, np.float64)
    y = np.asarray(labels, np.float64)
    V = x.shape[0]
    with np.errstate(invalid="ignore", divide="ignore"):
        per = np.maximum(x, 0) - x * y + np.log1p(np.exp(-np.abs(x)))
        loss = per.sum(axis=-1).mean() if V else float("nan")
        grad = (1.0 / (1.0 + np.exp(-x)) - y) / V if V else np.zeros_like(x)
    p = np.rint(_sigmoid32(logits)).astype(np.int64)
    l = np.asarray(labels).astype(np.int64)
    counts = (int(np.count_nonzero(p * l)), int(np.count_nonzero(p * (l - 1))), int(np.count_nonzero((p - 1) * l)))
    return loss, grad, counts, micro_f1(counts)


def micro_f1(counts):
    """node_multiclass_task.py:10-23 from (tp, fp, fn): NaN whenever tp == 0 (0 / 0)."""
    tp, fp, fn = (np.float64(c) for c in counts)
    with np.errstate(invalid="ignore", divide="ignore"):
        precision = tp / (tp + fp)
        recall = tp / (tp + fn)
        return float((2 * precision * recall) / (precision + recall))


def graph_regression_loss(pred, target):
    """(mse, mae, grad_pred of the mse)."""
    p = np.asarray(pred, np.float64)
    t = np.asarray(target, np.float64)
    G = p.shape[0]
    if G == 0:
        return float("nan"), float("nan"), np.zeros(0)
    d = p - t
    return float((d * d).mean()), float(np.abs(d).mean()), 2.0 * d / G


def graph_binary_loss(prob, target):
    """Keras binary_crossentropy(from_logits=False), TF >= 2.2: (loss, grad_prob, num_correct).  The gradient is zero
    where the clip to [eps, 1 - eps] cut (tf.clip_by_value passes it where lo <= p <= hi)."""
    p = np.asarray(prob, np.float64)
    t = np.asarray(target, np.float64)
    G = p.shape[0]
    lo, hi = float(np.float32(EPS)), float(np.float32(1) - np.float32(EPS))
    q = np.clip(p, lo, hi)
    if G == 0:
        return float("nan"), np.zeros(0), 0
    loss = -np.mean(t * np.log(q + EPS) + (1 - t) * np.log(1 - q + EPS))
    grad = -(t / (q + EPS) - (1 - t) / (1 - q + EPS)) / G
    grad = np.where((p >= lo) & (p <= hi), grad, 0.0)
    correct = int(np.sum(np.asarray(target, np.float32) == np.rint(np.asarray(prob, np.float32))))
    return float(loss), grad, correct


# ---- clipping -----------------------------------------------------------------------------------------------------
def clip_gradients(grads, mode, c):
    """mode None / "value" / "norm" / "global_norm" (graph_task_model.py:296-322)."""
    grads = [np.asarray(g, np.float64) for g in grads]
    if mode is None:
        return grads
    if mode == "value":
        return [np.clip(g, -c, c) for g in grads]
    if mode == "norm":
        return [g * c / max(math.sqrt(float((g * g).sum())), c) for g in grads]
    if mode == "global_norm":
        gn = math.sqrt(sum(float((g * g).sum()) for g in grads))
        scale = c * min(1.0 / gn if gn else math.inf, 1.0 / c) + (gn - gn)
        return [g * scale for g in grads]
    raise ValueError(mode)


# ---- optimizers ---------------------------------------------------------------------------------------------------
class Optimizer64:
    """Keras optimizer_v2 SGD / RMSprop / Adam, one step per apply(); slots start at zero."""

    def __init__(self, kind, lr, momentum=0.0, rho=0.9, clip_mode=None, clip=0.0):
        self.kind, self.lr, self.momentum, self.rho = kind, lr, F32(momentum), F32(rho)
        self.clip_mode, self.clip = clip_mode, F32(clip)
        self.iterations = 0
        self.slots = {}

    def apply(self, weights, grads):
        """weights: list of float64 arrays (updated in place); grads: list, None entries skipped."""
        idx = [i for i, g in enumerate(grads) if g is not None]
        clipped = clip_gradients([grads[i] for i in idx], self.clip_mode, self.clip)
        lr = F32(self.lr(self.iterations) if callable(self.lr) else self.lr)
        t = self.iterations + 1
        for i, g in zip(idx, clipped):
            w = weights[i]
            a, b = self.slots.setdefault(i, (np.zeros_like(w), np.zeros_like(w)))
            if self.kind == "sgd":
                if self.momentum > 0:
                    a[...] = a * self.momentum - lr * g
                    w += a
                else:
                    w -= lr * g
            elif self.kind == "rmsprop":
                a += (g * g - a) * (1 - self.rho)
                if self.momentum > 0:
                    b[...] = self.momentum * b + lr * g / np.sqrt(a + EPS)
                    w -= b
                else:
                    w -= lr * g / (np.sqrt(a) + EPS)
            elif self.kind == "adam":
                alpha = lr * math.sqrt(1 - BETA_2 ** t) / (1 - BETA_1 ** t)
                a += (g - a) * (1 - BETA_1)
                b += (g * g - b) * (1 - BETA_2)
                w -= alpha * a / (np.sqrt(b) + EPS)
            else:
                raise ValueError(self.kind)
        self.iterations += 1


# ---- schedule -----------------------------------------------------------------------------------------------------
def polynomial_warmup_and_decay(step, learning_rate, warmup_steps, decay_steps, initial_learning_rate,
                                final_learning_rate, power=1.0):
    if step <= warmup_steps:
        return (learning_rate - initial_learning_rate) * (step / warmup_steps) ** power + initial_learning_rate
    step = min(step - warmup_steps, decay_steps)
    return (learning_rate - final_learning_rate) * (1 - step / decay_steps) ** power + final_learning_rate
