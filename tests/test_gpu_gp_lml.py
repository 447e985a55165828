"""GPU tests of the GP marginal likelihood and hyper-parameter fit: GPRCached.compute_log_likelihood /
log_likelihood_and_gradient (the fused gradient slb_gp_lml_grad, csrc/gp_hyper.cu) against the numpy
reference of tests/gp_lml_reference.py at every compiled d_in and across tile boundaries, its
determinism, torch autograd, optimize against scipy on the reference objective, and a safe-set update
after a fit against the oracle built with the fitted values."""
import json

import numpy as np
import pytest
import torch
from numpy.testing import assert_allclose, assert_array_equal

import bench_workloads as W
import gp_lml_reference as R

pytestmark = pytest.mark.gpu

NOISE = 0.01
TILE = 64          # SLB_GP_HYPER_TILE


@pytest.fixture(scope="module")
def sl():
    import __graft_entry__
    __graft_entry__.build()
    import safe_learning_b200 as sl
    return sl


def _models(sl, din, builder, M, prior, seed):
    X, Y = R.data(din, M, seed=seed)
    row = np.linspace(0.3, -0.2, din)[None, :]
    gp = sl.GPR(X, Y, builder(sl.kernels), noise_variance=NOISE,
                mean_function=sl.LinearSystem(row) if prior else None, scale=1.7)
    ref = dict(kern=builder(R.ORACLE_KERNELS), noise=R.Noise(NOISE), X=X, Y=Y,
               mean=R.O.LinearMean(row) if prior else None)
    return gp, ref


def _reference(ref, **kw):
    return R.log_likelihood_and_gradient(ref["kern"], ref["noise"], ref["X"], ref["Y"], ref["mean"], **kw)


def _check_against_reference(gp, ref, M, rtol=1e-7):
    lml, grads = gp.log_likelihood_and_gradient()
    lml_ref, grads_ref, mags = _reference(ref, with_magnitude=True)
    assert_allclose(lml, lml_ref, rtol=1e-9, atol=1e-9 * max(M, 1))
    assert_allclose(gp.compute_log_likelihood(), lml, rtol=0, atol=0)
    assert list(grads) == list(grads_ref)
    for path, g in grads.items():
        want, mag = grads_ref[path], mags[path]
        if np.ndim(g) == 0:                      # non-ARD: the sum over its columns
            want, mag = want.sum(), mag.sum()
        # W = alpha alpha^T - K^-1 cancels: the bound is the size of what is summed, not of the sum
        assert np.all(np.abs(np.asarray(g) - want) <= rtol * mag + 1e-300), (path, g, want, mag)


@pytest.mark.parametrize("M", [1, 2, TILE - 1, TILE, TILE + 1, 500, 2000])
@pytest.mark.parametrize("din", range(1, 7))
def test_value_and_gradient_match_the_reference(sl, din, M):
    for k, (name, builder) in enumerate(R.kernel_set(din)):
        gp, ref = _models(sl, din, builder, M, prior=k % 2 == 1, seed=100 * din + M + k)
        _check_against_reference(gp, ref, M)


def test_two_calls_are_bit_identical(sl):
    for din in (3, 6):
        for name, builder in R.kernel_set(din):
            gp, _ = _models(sl, din, builder, 777, prior=True, seed=din)
            a = gp._log_likelihood(True)[1]
            b = gp._log_likelihood(True)[1]
            assert_array_equal(a, b)
            assert np.any(a != 0.0)


def test_gradient_matches_torch_autograd(sl):
    """M = 500: the notebook kernel and an ARD RBF as torch expressions of K, differentiated by autograd."""
    M, din = 500, 3
    X, Y = R.data(din, M, seed=11)
    Xd = torch.tensor(X, dtype=torch.float64, device="cuda")
    Yd = torch.tensor(Y[:, 0], dtype=torch.float64, device="cuda")
    k = sl.kernels

    def lml_of(K, noise):
        L = torch.linalg.cholesky(K + noise * torch.eye(M, dtype=torch.float64, device="cuda"))
        a = torch.linalg.solve_triangular(L, Yd[:, None], upper=False)
        return -0.5 * M * np.log(2 * np.pi) - torch.log(torch.diagonal(L)).sum() - 0.5 * (a * a).sum()

    # Linear(3, ARD) + Matern32(1, active_dims=[0]) * Linear(1)
    lin3 = k.Linear(3, variance=[0.2, 0.5, 0.3], ARD=True)
    m32 = k.Matern32(1, variance=0.8, lengthscales=0.7, active_dims=[0])
    lin1 = k.Linear(1, variance=0.6)
    gp = sl.GPR(X, Y, lin3 + m32 * lin1, noise_variance=NOISE)
    t = {n: torch.tensor(np.asarray(v, dtype=np.float64), device="cuda", requires_grad=True)
         for n, v in gp.hyperparameters().items()}
    v3, var32, ls32 = t["kern.kern_list[0].variance"], t["kern.kern_list[1].kern_list[0].variance"], \
        t["kern.kern_list[1].kern_list[0].lengthscales"]
    v1, noise = t["kern.kern_list[1].kern_list[1].variance"], t["likelihood.variance"]
    x0 = Xd[:, :1] / ls32
    r = torch.sqrt(torch.clamp(-2 * x0 @ x0.T + (x0 * x0).sum(1)[:, None] + (x0 * x0).sum(1)[None, :], min=0) + 1e-12)
    K = (Xd * v3) @ Xd.T + var32 * (1 + np.sqrt(3) * r) * torch.exp(-np.sqrt(3) * r) * (v1 * Xd[:, :1] @ Xd[:, :1].T)
    lml_t = lml_of(K, noise)
    lml_t.backward()
    lml, grads = gp.log_likelihood_and_gradient()
    assert_allclose(lml, lml_t.item(), rtol=1e-10)
    for n, g in grads.items():
        assert_allclose(g, t[n].grad.cpu().numpy(), rtol=1e-7, atol=1e-9 * np.abs(t[n].grad.cpu().numpy()).max(),
                        err_msg=n)

    ls = np.array([0.7, 1.2, 0.9])
    gp = sl.GPR(X, Y, k.RBF(3, variance=1.3, lengthscales=ls, ARD=True), noise_variance=NOISE)
    var = torch.tensor(1.3, dtype=torch.float64, device="cuda", requires_grad=True)
    lsd = torch.tensor(ls, device="cuda", requires_grad=True)
    noise = torch.tensor(NOISE, dtype=torch.float64, device="cuda", requires_grad=True)
    xs = Xd / lsd
    sq = (xs * xs).sum(1)
    lml_t = lml_of(var * torch.exp(-0.5 * (-2 * xs @ xs.T + sq[:, None] + sq[None, :])), noise)
    lml_t.backward()
    lml, grads = gp.log_likelihood_and_gradient()
    assert_allclose(lml, lml_t.item(), rtol=1e-10)
    assert_allclose(grads["kern.variance"], var.grad.item(), rtol=1e-7)
    assert_allclose(grads["kern.lengthscales"], lsd.grad.cpu().numpy(), rtol=1e-7)
    assert_allclose(grads["likelihood.variance"], noise.grad.item(), rtol=1e-7)


def _notebook(ns, v=(0.3, 0.4, 0.2), mvar=0.5, ls=0.6, v1=0.4):
    return ns.Linear(3, variance=np.asarray(v), ARD=True) + \
        ns.Matern32(1, variance=mvar, lengthscales=ls, active_dims=[0]) * ns.Linear(1, variance=v1)


def test_optimize_matches_scipy_on_the_reference(sl, monkeypatch):
    """Data sampled from a known GP (notebook kernel, seeded), noise fixed: optimize reaches the LML of
    scipy L-BFGS-B on the reference objective from the same start, its gradient is small at the end, the
    values are written back, and a Cholesky failure during the search restores the start."""
    M = 300
    rng = np.random.default_rng(7)
    X = rng.uniform(-1, 1, (M, 3))
    truth = _notebook(R.ORACLE_KERNELS, v=(0.8, 0.2, 0.5), mvar=1.5, ls=0.4, v1=1.2)
    C = truth.K(X) + NOISE * np.eye(M)
    Y = np.linalg.cholesky(C).dot(rng.standard_normal(M))[:, None]
    gp = sl.GPR(X, Y, _notebook(sl.kernels), noise_variance=NOISE)
    start = gp.hyperparameters()
    res = gp.optimize(fixed=("likelihood.variance",))
    kern_ref, noise_ref = _notebook(R.ORACLE_KERNELS), R.Noise(NOISE)
    res_ref = R.fit(kern_ref, noise_ref, X, Y, fixed=("likelihood.variance",))
    lml = gp.compute_log_likelihood()
    lml_ref = R.log_likelihood(kern_ref, noise_ref, X, Y)
    assert lml >= lml_ref - 1e-6 * abs(lml_ref), (lml, lml_ref, res.message, res_ref.message)
    assert_allclose(lml, -res.fun, rtol=1e-12)
    # the gradient in the free space of the positive transform
    lml2, grads = gp.log_likelihood_and_gradient()
    hp = gp.hyperparameters()
    free = [p for p in hp if p != "likelihood.variance"]
    for p in free:
        y = np.asarray(hp[p]) - 1e-6
        dfree = np.asarray(grads[p]) * -np.expm1(-y)           # d softplus(x) / dx at softplus(x) = y
        assert np.all(np.abs(dfree) <= 1e-4 * abs(lml)), (p, dfree)
    assert hp["likelihood.variance"] == NOISE
    assert any(np.any(np.asarray(hp[p]) != np.asarray(start[p])) for p in free)
    assert np.all(gp.kern.kern_list[0].variance == hp["kern.kern_list[0].variance"])   # written back

    # a Cholesky failure during the search: the error propagates and the start values come back
    gp2 = sl.GPR(X, Y, _notebook(sl.kernels), noise_variance=NOISE)
    calls = []
    real = torch.linalg.cholesky

    def failing(A, *args, **kwargs):
        calls.append(1)
        if len(calls) == 4:
            raise torch.linalg.LinAlgError("linalg.cholesky: The factorization could not be completed")
        return real(A, *args, **kwargs)

    monkeypatch.setattr(torch.linalg, "cholesky", failing)
    with pytest.raises(torch.linalg.LinAlgError):
        gp2.optimize(fixed=("likelihood.variance",))
    monkeypatch.setattr(torch.linalg, "cholesky", real)
    for p, v in gp2.hyperparameters().items():
        assert_array_equal(v, start[p])


def _fitted_spec(kern):
    lin3, prod = kern.kern_list
    m32, lin1 = prod.kern_list
    return json.dumps(["add", ["linear", 3, {"variance": lin3.variance.tolist(), "ARD": True}],
                       ["prod", ["matern32", 1, {"variance": m32.variance, "lengthscales": m32.lengthscales.tolist(),
                                                 "active_dims": [0]}],
                        ["linear", 1, {"variance": float(lin1.variance[0])}]]])


def test_safe_set_after_a_fit_matches_the_oracle(sl):
    """optimize() between sweeps: the next update_safe_set (decision filter on) refits the factor and the
    filter tables, and gives the oracle's safe set and c_max built with the fitted values."""
    par = W.make_pendulum(num_points=41, M=200, with_prior_mean=True, noise_std=1e-2)
    par["kernel_specs"] = W.notebook_pendulum_kernels([[2e-3, 6e-3, 1.5e-3], [2.5e-2, 8e-3, 1.2e-2]])
    gpu = W.build_product(par)
    gpu.filter = True
    gpu.update_safe_set()
    before = gpu.safe_set.copy()
    gps = [f.gaussian_process for f in gpu.dynamics.functions]
    for gp in gps:
        gp.optimize(maxiter=50, fixed=("likelihood.variance",))
    gpu.update_safe_set()
    par["kernel_specs"] = [_fitted_spec(gp.kern) for gp in gps]
    cpu = W.build_oracle(par)
    cpu.update_safe_set()
    assert_array_equal(gpu.safe_set, cpu.safe_set)
    assert gpu.feed_dict[gpu.c_max] == cpu.c_max
    assert gpu.safe_set.sum() > 0
    print("safe points before / after the fit: %d / %d" % (before.sum(), gpu.safe_set.sum()))
