"""The float64 restatement of the task losses, optimizers, clipping and schedule (tests/reference64_task.py) against torch
autograd in float64 and against closed forms."""
import math

import numpy as np
import pytest

torch = pytest.importorskip("torch")

import reference64_task as rt


def _grad(fn, x):
    t = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    out = fn(t)
    out.backward()
    return float(out), t.grad.numpy()


def test_node_multiclass_loss_and_gradient_match_autograd():
    rng = np.random.default_rng(0)
    x = rng.normal(0, 3, (50, 7))
    y = (rng.uniform(size=(50, 7)) < 0.3).astype(np.float64)
    loss, grad, _, _ = rt.node_multiclass_loss(x, y)
    yt = torch.tensor(y)
    ref_loss, ref_grad = _grad(lambda t: torch.nn.functional.binary_cross_entropy_with_logits(t, yt, reduction="none")
                               .sum(-1).mean(), x)
    assert loss == pytest.approx(ref_loss, rel=1e-12)
    np.testing.assert_allclose(grad, ref_grad, rtol=1e-10, atol=1e-15)


def test_node_multiclass_counts_and_f1():
    x = np.array([[0.0, 1.0, -1.0, 2.0], [-3.0, 0.0, 5.0, -0.5]])
    y = np.array([[1.0, 1.0, 1.0, 0.0], [0.0, 0.0, 1.0, 1.0]])
    _, _, counts, f1 = rt.node_multiclass_loss(x, y)
    # predictions: [[0, 1, 0, 1], [0, 0, 1, 0]] (a logit of exactly 0 predicts 0)
    assert counts == (2, 1, 3)
    p, r = 2 / 3, 2 / 5
    assert f1 == pytest.approx(2 * p * r / (p + r))


def test_micro_f1_is_nan_without_true_positives():
    assert math.isnan(rt.micro_f1((0, 5, 3)))
    assert math.isnan(rt.micro_f1((0, 0, 0)))
    _, _, counts, f1 = rt.node_multiclass_loss(np.full((3, 2), -4.0), np.ones((3, 2)))
    assert counts == (0, 0, 6) and math.isnan(f1)


def test_graph_regression_loss_matches_autograd():
    rng = np.random.default_rng(1)
    p, t = rng.normal(size=33), rng.normal(size=33)
    mse, mae, grad = rt.graph_regression_loss(p, t)
    tt = torch.tensor(t)
    ref, ref_grad = _grad(lambda q: ((q - tt) ** 2).mean(), p)
    assert mse == pytest.approx(ref, rel=1e-12)
    assert mae == pytest.approx(np.abs(p - t).mean(), rel=1e-12)
    np.testing.assert_allclose(grad, ref_grad, rtol=1e-12)


def test_graph_binary_loss_matches_autograd_and_zeroes_clipped_gradients():
    rng = np.random.default_rng(2)
    p = np.concatenate([rng.uniform(0.01, 0.99, 20), [0.0, 1.0, 1e-9, 0.5]])
    t = (rng.uniform(size=p.size) < 0.5).astype(np.float64)
    loss, grad, correct = rt.graph_binary_loss(p, t)
    lo, hi = float(np.float32(1e-7)), float(np.float32(1) - np.float32(1e-7))
    tt = torch.tensor(t)

    def bce(q):
        qc = torch.clamp(q, lo, hi)
        return -(tt * torch.log(qc + rt.EPS) + (1 - tt) * torch.log(1 - qc + rt.EPS)).mean()

    ref, ref_grad = _grad(bce, p)
    assert loss == pytest.approx(ref, rel=1e-12)
    np.testing.assert_allclose(grad, ref_grad, rtol=1e-10, atol=1e-15)
    assert grad[20] == 0.0 and grad[21] == 0.0 and grad[22] == 0.0   # cut by the clip
    assert correct == int(np.sum(t == np.rint(p)))


def _torch_opt_step(kind, weights, grads, steps, **kw):
    """The same rules written with torch float64 ops (Keras epsilon placement), as a second statement."""
    ws = [torch.tensor(w) for w in weights]
    a = [torch.zeros_like(w) for w in ws]
    b = [torch.zeros_like(w) for w in ws]
    lr, b1, b2, eps = rt.F32(kw["lr"]), rt.BETA_1, rt.BETA_2, rt.EPS
    mom, rho = rt.F32(kw["momentum"]), rt.F32(kw["rho"])
    for s in range(steps):
        for i, (w, g) in enumerate(zip(ws, grads)):
            g = torch.tensor(g)
            if kind == "sgd":
                a[i] = a[i] * mom - lr * g
                w += a[i]
            elif kind == "rmsprop":
                a[i] = a[i] + (g * g - a[i]) * (1 - rho)
                b[i] = mom * b[i] + lr * g / torch.sqrt(a[i] + eps)
                w -= b[i]
            else:
                t = s + 1
                alpha = lr * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)
                a[i] = a[i] + (g - a[i]) * (1 - b1)
                b[i] = b[i] + (g * g - b[i]) * (1 - b2)
                w -= alpha * a[i] / (torch.sqrt(b[i]) + eps)
    return [w.numpy() for w in ws]


@pytest.mark.parametrize("kind", ["sgd", "rmsprop", "adam"])
def test_optimizers_match_a_torch_statement(kind):
    rng = np.random.default_rng(3)
    weights = [rng.normal(size=(5, 3)), rng.normal(size=7)]
    grads = [rng.normal(size=(5, 3)), rng.normal(size=7)]
    opt = rt.Optimizer64(kind, 0.01, momentum=0.85, rho=0.98)
    ws = [w.copy() for w in weights]
    for _ in range(4):
        opt.apply(ws, grads)
    ref = _torch_opt_step(kind, weights, grads, 4, lr=0.01, momentum=0.85, rho=0.98)
    for got, want in zip(ws, ref):
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-15)


def test_adam_first_step_closed_form():
    rng = np.random.default_rng(4)
    w0, g = rng.normal(size=20), rng.normal(size=20)
    w = [w0.copy()]
    rt.Optimizer64("adam", 0.003).apply(w, [g])
    lr = rt.F32(0.003)
    np.testing.assert_allclose(w0 - w[0], lr * g / (np.abs(g) + rt.EPS / math.sqrt(1 - rt.BETA_2)), rtol=1e-12)


def test_momentum_free_rules_and_skipped_variables():
    w = [np.ones(3), np.ones(2)]
    g = [np.full(3, 2.0), None]
    rt.Optimizer64("sgd", 0.5, momentum=0.0).apply(w, g)
    np.testing.assert_array_equal(w[0], np.zeros(3))
    np.testing.assert_array_equal(w[1], np.ones(2))
    w = [np.ones(3)]
    rt.Optimizer64("rmsprop", 0.1, momentum=0.0, rho=0.9).apply(w, [np.full(3, 2.0)])
    rho = rt.F32(0.9)
    np.testing.assert_allclose(w[0], 1 - rt.F32(0.1) * 2.0 / (math.sqrt((1 - rho) * 4.0) + rt.EPS))


def test_clip_rules():
    g = [np.array([3.0, -4.0]), np.array([12.0])]
    np.testing.assert_array_equal(rt.clip_gradients(g, "value", 2.0)[0], [2.0, -2.0])
    by_norm = rt.clip_gradients(g, "norm", 1.0)
    np.testing.assert_allclose(by_norm[0], [0.6, -0.8])
    np.testing.assert_allclose(by_norm[1], [1.0])
    np.testing.assert_allclose(rt.clip_gradients(g, "norm", 100.0)[0], g[0])
    by_global = rt.clip_gradients(g, "global_norm", 6.5)   # global norm 13
    np.testing.assert_allclose(by_global[0], [1.5, -2.0])
    np.testing.assert_allclose(rt.clip_gradients(g, "global_norm", 100.0)[1], g[1])
    assert np.isnan(rt.clip_gradients([np.array([np.inf, 1.0])], "global_norm", 1.0)[0]).all()
    np.testing.assert_allclose(by_global[1], [6.0])


def test_schedule_boundaries():
    kw = dict(learning_rate=1e-3, warmup_steps=10, decay_steps=100, initial_learning_rate=1e-5, final_learning_rate=1e-5)
    assert rt.polynomial_warmup_and_decay(0, **kw) == pytest.approx(1e-5)
    assert rt.polynomial_warmup_and_decay(5, **kw) == pytest.approx(1e-5 + 0.5 * (1e-3 - 1e-5))
    assert rt.polynomial_warmup_and_decay(10, **kw) == pytest.approx(1e-3)
    assert rt.polynomial_warmup_and_decay(60, **kw) == pytest.approx(1e-5 + 0.5 * (1e-3 - 1e-5))
    assert rt.polynomial_warmup_and_decay(110, **kw) == pytest.approx(1e-5)
    assert rt.polynomial_warmup_and_decay(1000, **kw) == pytest.approx(1e-5)
    # no warmup (graph_task_model.py:245-247): warmup_steps = -1, initial = learning_rate
    nw = dict(kw, warmup_steps=-1, initial_learning_rate=1e-3)
    assert rt.polynomial_warmup_and_decay(0, **nw) == pytest.approx(1e-3 - (1e-3 - 1e-5) / 100)


def test_host_schedule_matches_the_restatement():
    from tf2_gnn_b200.models import PolynomialWarmupAndDecaySchedule
    kw = dict(learning_rate=1e-3, warmup_steps=10, decay_steps=100, initial_learning_rate=1e-5, final_learning_rate=1e-5)
    sched = PolynomialWarmupAndDecaySchedule(**kw)
    for step in (0, 1, 9, 10, 11, 50, 110, 111, 500):
        assert sched(step) == pytest.approx(rt.polynomial_warmup_and_decay(step, **kw), rel=1e-15)
