"""GPU tests of the GP posterior's reverse mode: ``slb_gp_vjp`` against float64 autograd through
``GPRCached.torch_predict`` and central differences of ``slb_gp_predict``, and ``GaussianProcess.torch`` /
``FunctionStack.torch`` as one autograd node, up to five SGD steps of inverted_pendulum.ipynb cell 17."""
import os
import sys

import numpy as np
import pytest
import torch

import safe_learning_b200 as sl
from safe_learning_b200 import functions as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench_workloads as W  # noqa: E402

pytestmark = pytest.mark.gpu

MS = [0, 1, 7, 8, 9, 255, 256, 257, 500]
NS = [0, 1, 15, 16, 17, 63, 64, 65, 4099]


def _kernel(kind, din, rng):
    """Covariance expressions on `din` inputs; primitives alone act on a subset of the columns."""
    sub = sorted(rng.choice(din, size=max(1, din - 1), replace=False).tolist()) if din > 1 else [0]
    ls = lambda k: rng.uniform(0.6, 1.6, k)
    if kind == "rbf":
        return sl.RBF(din, variance=0.7, lengthscales=ls(din))          # the plain fast path
    if kind == "rbf_sub":
        return sl.RBF(len(sub), variance=0.7, lengthscales=ls(len(sub)), active_dims=sub)
    if kind in ("matern12", "matern32", "matern52"):
        cls = {"matern12": sl.Matern12, "matern32": sl.Matern32, "matern52": sl.Matern52}[kind]
        return cls(len(sub), variance=0.6, lengthscales=ls(len(sub)), active_dims=sub)
    if kind == "linear":
        return sl.Linear(len(sub), variance=rng.uniform(0.2, 1.0, len(sub)), active_dims=sub, ARD=True)
    if kind == "constant":
        return sl.Constant(len(sub), variance=0.8, active_dims=sub) + sl.RBF(din, variance=0.3)
    if kind == "white":
        return sl.White(len(sub), variance=0.2, active_dims=sub) + sl.Matern32(din, variance=0.5)
    if kind == "notebook":
        # cell 6: Linear(3, ARD) + Matern32(1, active_dims=[0]) * Linear(1), on the first min(din, 3) inputs
        k = min(din, 3)
        return (sl.Linear(k, variance=rng.uniform(0.05, 0.2, k), ARD=True)
                + sl.Matern32(1, lengthscales=1.0, active_dims=[0]) * sl.Linear(1, variance=0.1))
    if kind == "six":
        return (sl.RBF(din, variance=0.5, lengthscales=ls(din)) * sl.Matern32(len(sub), lengthscales=ls(len(sub)),
                                                                             active_dims=sub)
                + sl.Linear(din, variance=0.3) * sl.Matern12(1, variance=0.4, active_dims=[din - 1])
                + sl.Matern52(din, variance=0.3, lengthscales=ls(din)) + sl.Constant(din, variance=0.2))
    raise KeyError(kind)


def _stack(din, M, kinds, prior=True, shared=False, seed=0, beta=2.0, scale=1.0):
    """FunctionStack of len(kinds) GPs on one data set; shared=True: identical kernels -> one factor."""
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1, 1, (M, din))
    gps = []
    for o, kind in enumerate(kinds):
        krng = np.random.default_rng(seed + (0 if shared else 100 + o))
        kern = _kernel(kind, din, krng)
        Y = np.sin(X @ rng.normal(size=din) + o)[:, None] + 0.05 * rng.normal(size=(M, 1))
        mean = sl.LinearSystem(rng.normal(size=(1, din))) if prior else None
        gp = sl.GPRCached(X, Y, kern, mean_function=mean, noise_variance=0.01, scale=scale)
        gps.append(sl.GaussianProcess(gp, beta=beta if o % 2 == 0 else 1.5))
    return sl.FunctionStack(gps)


def _points(n, din, seed=1):
    return torch.tensor(np.random.default_rng(seed).uniform(-1.2, 1.2, (n, din)), device="cuda")


def _reference(stack, x, gm, ge):
    """Float64 autograd through torch_predict: (mean part, err part) of the points' gradient."""
    xg = x.clone().requires_grad_(True)
    mean, err = stack._torch_expression(xg)
    out = []
    for y, g in ((mean, gm), (err, ge)):
        # a prior-only stationary variance does not depend on the points
        grad = torch.autograd.grad(y, xg, g, retain_graph=True)[0] if y.requires_grad and x.shape[0] else None
        out.append(torch.zeros_like(x) if grad is None else grad)
    return tuple(out)


def _assert_close(got, want, tol=1e-9, what=""):
    """Per column, relative to the column's max |grad| over the batch."""
    assert got.shape == want.shape
    if got.numel() == 0:
        return
    scale = want.abs().max(dim=0).values
    floor = 1e-12 * float(scale.max())
    err = (got - want).abs().max(dim=0).values
    bad = err > tol * torch.clamp(scale, min=floor)
    assert not bool(bad.any()), "%s: error %s against column scale %s" % (what, err.tolist(), scale.tolist())


def _away_from_matern12_kinks(stack, x, rmin=3e-3):
    """The rows of x at scaled distance >= rmin from every training input in each Matern12 primitive's
    active dimensions.  Matern12 has a kink at r = 0, and near it the reference's expanded square distance
    (-2 z.x + |z|^2 + |x|^2, gpflow's) loses the digits a 1e-9 comparison needs."""
    keep = torch.ones(x.shape[0], dtype=torch.bool, device=x.device)
    for f in stack.functions:
        X = torch.tensor(f.gaussian_process.X, device=x.device)
        for term in f.gaussian_process.kern.terms():
            for p in term:
                if isinstance(p, sl.Matern12) and X.shape[0] and x.shape[0]:
                    ls = torch.tensor(p.lengthscales, device=x.device)
                    d = torch.cdist(x[:, p.active_dims] / ls, X[:, p.active_dims] / ls)
                    keep &= d.min(dim=1).values >= rmin
    return x[keep]


def _check_all_modes(stack, x, seed=2):
    x = _away_from_matern12_kinks(stack, x)
    n, D = x.shape[0], stack.num_fun
    rng = np.random.default_rng(seed)
    gm = torch.tensor(rng.normal(size=(n, D)), device="cuda")
    ge = torch.tensor(rng.normal(size=(n, D)), device="cuda")
    gmr, ger = _reference(stack, x, gm, ge)
    _assert_close(stack.vjp_device(x, gm, None), gmr, what="mean only")
    _assert_close(stack.vjp_device(x, None, ge), ger, what="err only")
    _assert_close(stack.vjp_device(x, gm, ge), gmr + ger, what="both")


# ---------------------------------------------------------------- agreement with float64 autograd
@pytest.mark.parametrize("din", range(1, 7))
@pytest.mark.parametrize("kind", ["rbf", "rbf_sub", "matern12", "matern32", "matern52", "linear", "constant",
                                  "white", "notebook", "six"])
def test_each_kernel_and_input_dim(din, kind):
    """Every primitive alone (on an active_dims subset), the plain RBF, the notebook kernel and a six-primitive
    sum of products, at two data-set sizes and two batch sizes, with a prior mean and two distinct factors."""
    i = din * 7 + len(kind)
    for M in (MS[i % 4], MS[4 + i % 5]):
        stack = _stack(din, M, [kind, kind], prior=True, seed=i)
        _check_all_modes(stack, _points(NS[i % 9] + 40, din, seed=i))


@pytest.mark.parametrize("M", MS)
def test_row_block_and_panel_boundaries(M):
    """M at the 8-row-block and 256-row-panel boundaries, every batch size (tile boundaries of both kernels)."""
    for kinds in (["rbf", "rbf"], ["notebook", "notebook"]):
        stack = _stack(3, M, kinds, prior=M % 2 == 0, seed=M)
        for n in NS:
            _check_all_modes(stack, _points(n, 3, seed=n))


@pytest.mark.parametrize("D", range(1, 7))
@pytest.mark.parametrize("shared", [True, False])
def test_outputs_and_factor_sharing(D, shared):
    kinds = ["rbf", "six", "matern32", "notebook", "rbf", "linear"][:D] if not shared else ["six"] * D
    stack = _stack(4, 57, kinds, prior=D % 2 == 1, shared=shared, seed=D, beta=3.0, scale=1.7)
    assert stack.gp_stack().num_factors == (1 if shared else D)
    _check_all_modes(stack, _points(301, 4, seed=D))


def test_single_gaussian_process_without_prior_mean():
    gp = _stack(2, 33, ["matern52"], prior=False, beta=0.7).functions[0]
    x = _points(129, 2)
    g = torch.tensor(np.random.default_rng(0).normal(size=(129, 1)), device="cuda")
    gmr, ger = _reference(gp, x, g, g)
    _assert_close(gp.vjp_device(x, g, g), gmr + ger)


# ---------------------------------------------------------------- central differences, v = 0, determinism
@pytest.mark.parametrize("kind, M", [("rbf", 500), ("notebook", 50), ("six", 9), ("notebook", 0)])
def test_central_differences_of_the_forward(kind, M):
    stack = _stack(3, M, [kind, kind], seed=5)
    x = _points(5, 3, seed=6)
    rng = np.random.default_rng(7)
    gm, ge = (torch.tensor(rng.normal(size=(5, 2)), device="cuda") for _ in range(2))

    def objective(p):
        mean, err = stack.predict_device(p)
        return (gm * mean + ge * err).sum(dim=1)

    got = stack.vjp_device(x, gm, ge)
    for c in range(3):
        h = 1e-5 * max(1.0, float(x[:, c].abs().max()))
        e = torch.zeros_like(x)
        e[:, c] = h
        fd = (objective(x + e) - objective(x - e)) / (2 * h)
        assert torch.allclose(got[:, c], fd, rtol=1e-5, atol=1e-5 * float(got.abs().max())), (c, got[:, c], fd)


@pytest.mark.parametrize("M", [0, 5])
def test_zero_variance_follows_torch(M):
    """A Linear-only kernel has zero variance at z = 0: torch's sqrt backward divides by 2 sqrt(0), so the
    err gradient there is NaN (inf * 0), and the mean gradient is finite."""
    rng = np.random.default_rng(8)
    X = rng.uniform(-1, 1, (M, 2))
    gp = sl.GaussianProcess(sl.GPRCached(X, rng.normal(size=(M, 1)), sl.Linear(2, variance=[0.5, 0.2], ARD=True),
                                         noise_variance=0.01))
    x = _points(20, 2)
    x[3] = 0.0
    g = torch.tensor(rng.normal(size=(20, 1)), device="cuda")
    gmr, ger = _reference(gp, x, g, g)
    got_e, got_m = gp.vjp_device(x, None, g), gp.vjp_device(x, g, None)
    assert torch.equal(torch.isnan(got_e), torch.isnan(ger)) and bool(torch.isnan(got_e[3]).all())
    assert bool(torch.isfinite(got_m).all())
    keep = torch.ones(20, dtype=torch.bool, device="cuda")
    keep[3] = False
    _assert_close(got_e[keep], ger[keep])
    _assert_close(got_m, gmr)


def test_two_calls_are_bit_identical():
    stack = _stack(3, 500, ["rbf", "notebook"], seed=9)
    x = _points(4099, 3)
    g = torch.tensor(np.random.default_rng(1).normal(size=(4099, 2)), device="cuda")
    assert torch.equal(stack.vjp_device(x, g, g), stack.vjp_device(x, g, g))
    assert torch.equal(stack.vjp_device(x, g, None), stack.vjp_device(x, g, None))


# ---------------------------------------------------------------- the autograd node
def test_node_forward_is_predict_device_and_backward_one_vjp(monkeypatch):
    stack = _stack(3, 200, ["rbf", "notebook"], seed=10)
    x = _points(777, 3)
    calls = []
    real = F._gp_vjp

    def spy(st, p, gm, ge):
        calls.append((gm is not None, ge is not None))
        return real(st, p, gm, ge)

    monkeypatch.setattr(F, "_gp_vjp", spy)
    xg = x.clone().requires_grad_(True)
    mean, err = stack.torch(xg)
    want_m, want_e = stack.predict_device(x)
    assert torch.equal(mean.detach(), want_m) and torch.equal(err.detach(), want_e)
    g = torch.tensor(np.random.default_rng(2).normal(size=(777, 2)), device="cuda")
    (mean * g).sum().backward()                                  # a mean-only objective (cell 9)
    assert calls == [(True, False)]
    gmr, ger = _reference(stack, x, g, g)
    assert torch.equal(xg.grad, real(stack.gp_stack(), x, g, None))
    _assert_close(xg.grad, gmr)
    xg.grad = None
    mean, err = stack.torch(xg)
    ((mean * g).sum() + (err * g).sum()).backward()
    assert calls[-1] == (True, True)
    _assert_close(xg.grad, gmr + ger)
    gp = stack.functions[1]
    xg.grad = None
    m1, e1 = gp.torch(xg)
    assert torch.equal(m1.detach(), gp.predict_device(x)[0]) and m1.shape == (777, 1)
    (e1 * g[:, 1:]).sum().backward()
    assert calls[-1] == (False, True)


def test_second_derivative_equals_torch_predicts():
    stack = _stack(3, 60, ["notebook", "rbf"], seed=11)
    x = _points(50, 3)
    rng = np.random.default_rng(3)
    gm, ge, v = (torch.tensor(rng.normal(size=s), device="cuda") for s in ((50, 2), (50, 2), (50, 3)))
    out = []
    for fn in (stack.torch, stack._torch_expression):
        xg = x.clone().requires_grad_(True)
        mean, err = fn(xg)
        (gx,) = torch.autograd.grad((gm * mean).sum() + (ge * err).sum(), xg, create_graph=True)
        (hv,) = torch.autograd.grad((gx * v).sum(), xg)
        out.append((gx.detach(), hv))
    assert torch.allclose(out[0][0], out[1][0], rtol=1e-12, atol=0)
    assert torch.allclose(out[0][1], out[1][1], rtol=1e-12, atol=1e-14)
    # every other node still refuses a second derivative
    lin = sl.LinearSystem(np.ones((1, 3)))
    xg = x.clone().requires_grad_(True)
    (gx,) = torch.autograd.grad((lin.torch(xg) ** 2).sum(), xg, create_graph=True)
    with pytest.raises(RuntimeError, match="once_differentiable"):
        gx.sum().backward()


# ---------------------------------------------------------------- inverted_pendulum.ipynb cell 17
@pytest.mark.parametrize("M", [0, 50])
def test_cell17_policy_steps_match_torch_predict(M):
    """Five SGD steps on -mean(future_values(states, lyapunov=...)) with the notebook's L_V (which used to
    raise in the backward): the node and torch_predict as the dynamics give the same weights, and the fused
    update_safe_set then follows the trained policy."""
    runs = []
    for torch_dynamics in (False, True):
        case = W.notebook_policy_case(sl, M, torch_dynamics=torch_dynamics)
        net = case["policy"]
        net._build(2)
        opt = torch.optim.SGD(net.parameters, lr=0.05)
        losses = [float(case["step"](opt)) for _ in range(5)]
        runs.append((case, [p.detach().clone() for p in net.parameters], losses))
    (case, w_node, l_node), (_, w_ref, l_ref) = runs
    assert np.allclose(l_node, l_ref, rtol=1e-12, atol=0)
    for a, b in zip(w_node, w_ref):
        assert torch.allclose(a, b, rtol=0, atol=1e-9), float((a - b).abs().max())
    w0 = W.notebook_policy_case(sl, M)["policy"]
    w0._build(2)
    assert any(not torch.equal(a, b.detach()) for a, b in zip(w_node, w0.parameters))
    # the fused sweep sees the trained weights: same result as a Lyapunov object built after training
    lyap = case["lyapunov"]
    lyap.update_safe_set()
    fresh = sl.Lyapunov(case["grid"], -case["value"], case["dynamics"], case["l_dyn"],
                        sl.MaxAbsFunction(case["value"].gradient_function()), case["tau"], case["policy"],
                        initial_set=case["initial"])
    fresh.update_safe_set()
    assert np.array_equal(lyap.safe_set, fresh.safe_set)
