"""GPU tests of multi-output GPs: one ``GPRCached`` whose ``Y`` has k columns, under one kernel and noise.

A k-column ``GaussianProcess`` must be, bit for bit, the ``FunctionStack`` of k one-column GPs with the same X,
kernel, noise, scale, beta and prior-mean rows: its outputs are k outputs on one factor, and every table
row is what the one-column GP computes on that factor.  Compared here: ``predict_device``, the torch node
forward and backward, the mean model's rollouts, value iteration and the greedy policy, ``update_safe_set``
(filtered, unfiltered, adaptive, ``can_shrink=False``), ``get_safe_sample``, and ``add_data_point`` past a
refit.  Also: the joint log marginal likelihood and its fused gradient (``slb_gp_lml_grad_cols``), and
``optimize`` on two columns against torch autograd of the same expression."""
import os
import sys

import numpy as np
import pytest
import torch
from numpy.testing import assert_array_equal

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import bench_workloads as W  # noqa: E402
import gp_lml_cols_reference as LC  # noqa: E402
import gp_lml_reference as LR  # noqa: E402
import safe_learning_b200 as sl  # noqa: E402
from safe_learning_b200 import _device as dev  # noqa: E402
from safe_learning_b200 import _native as nat  # noqa: E402

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------- models
def _kernel(kind, din):
    if kind == "rbf":
        return sl.RBF(din, variance=0.6, lengthscales=[0.9 + 0.15 * c for c in range(din)], ARD=True)
    # the notebooks' expression, on d_in inputs
    return (sl.Linear(din, variance=np.linspace(0.2, 0.5, din), ARD=True)
            + sl.Matern32(1, lengthscales=1.0, active_dims=[0]) * sl.Linear(1, variance=0.3))


def _data(M, k, din, seed):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1, 1, (M, din))
    mix = rng.uniform(-0.4, 0.4, (din, k))
    if k <= din:
        mix[:k, :k] += 0.7 * np.eye(k)
    Y = np.sin(X @ mix) + 0.3 * X @ mix + 1e-2 * rng.standard_normal((M, k))
    rows = rng.uniform(-0.5, 0.5, (k, din))
    if k < din:
        rows[:, :k] += 0.6 * np.eye(k)
    return X, Y, rows


def _pair(M, k, kind="rbf", prior=True, din=3, scale=1.0, beta=2.0, seed=0):
    """(k-column GaussianProcess, FunctionStack of its k columns as one-column GPs)."""
    X, Y, rows = _data(M, k, din, seed)
    multi = sl.GaussianProcess(sl.GPRCached(X, Y, _kernel(kind, din),
                                            mean_function=sl.LinearSystem(rows) if prior else None,
                                            scale=scale, noise_variance=1e-2), beta=beta)
    single = sl.FunctionStack([sl.GaussianProcess(sl.GPRCached(
        X, Y[:, [c]], _kernel(kind, din), mean_function=sl.LinearSystem(rows[[c]]) if prior else None,
        scale=scale, noise_variance=1e-2), beta=beta) for c in range(k)])
    return multi, single


def _lyapunov(dyn, d, num, adaptive=False):
    grid = sl.GridWorld(np.array([[-1., 1.]] * d), num)
    policy = sl.Saturation(sl.LinearSystem(-0.4 * np.ones((1, d))), -1., 1.)
    P = np.diag(np.linspace(1.0, 1.5, d))
    pts = grid.all_points
    initial = np.linalg.norm(pts, axis=1) <= 0.35
    return sl.Lyapunov(grid, sl.QuadraticFunction(P), dyn, 1.2, sl.AbsFunction(sl.LinearSystem((2 * P,))),
                       float(np.sum(grid.unit_maxes) / 2), policy, initial_set=initial, adaptive=adaptive)


def _num(d):
    return {1: 301, 2: 41, 3: 13, 4: 7}[d]


Q = np.random.default_rng(11).uniform(-1.3, 1.3, (333, 6))
MS = [0, 1, 7, 257, 500]
KS = [1, 2, 3, 4, 6]


# ---------------------------------------------------------------- posterior, torch node, mean model
@pytest.mark.parametrize("prior", [True, False])
@pytest.mark.parametrize("kind", ["rbf", "expr"])
@pytest.mark.parametrize("M", MS)
@pytest.mark.parametrize("k", KS)
def test_posterior_equals_the_stack_of_columns(k, M, kind, prior):
    multi, single = _pair(M, k, kind, prior, din=3, scale=1.7 if prior else 1.0, seed=k * 10 + M)
    assert multi.output_dim == single.output_dim == k
    z = Q[:, :3]
    ma, ea = multi.predict_device(z)
    mb, eb = single.predict_device(z)
    assert ma.shape == (333, k)
    assert_array_equal(ma.cpu().numpy(), mb.cpu().numpy())
    assert_array_equal(ea.cpu().numpy(), eb.cpu().numpy())
    e = ea.cpu().numpy()
    assert_array_equal(e, np.repeat(e[:, :1], k, axis=1))          # one sigma in every column
    m2, e2 = multi(z[:, :2], z[:, 2:])
    assert_array_equal(m2, ma.cpu().numpy())
    assert_array_equal(e2, e)
    # variances too
    _, va = multi.predict_device(z, want_var=True)
    _, vb = single.predict_device(z, want_var=True)
    assert_array_equal(va.cpu().numpy(), vb.cpu().numpy())
    # alpha [M, k]
    alpha = multi.gaussian_process.alpha
    assert alpha.shape == (M, k)
    for c in range(k):
        assert_array_equal(alpha[:, c], single.functions[c].gaussian_process.alpha[:, 0])
    # the torch node: forward and backward
    rng = np.random.default_rng(M + k)
    gm, ge = (dev.to_device(rng.standard_normal((333, k))) for _ in range(2))
    grads = []
    for f in (multi, single):
        x = dev.to_device(z).requires_grad_(True)
        mean, err = f.torch(x)
        ((mean * gm).sum() + (err * ge).sum()).backward()
        grads.append((mean.detach().cpu().numpy(), err.detach().cpu().numpy(), x.grad.cpu().numpy()))
    for a, b in zip(*grads):
        assert_array_equal(a, b)
    assert_array_equal(multi.vjp_device(z, gm, ge).cpu().numpy(), grads[1][2])
    # the mean model
    pa, pb = multi.to_mean_function(), single.to_mean_function()
    assert pa.output_dim == k
    assert_array_equal(pa(z), pb(z))
    assert_array_equal(pa.jacobian_device(z).cpu().numpy(), pb.jacobian_device(z).cpu().numpy())


@pytest.mark.parametrize("k", [1, 2, 3])
def test_create_graph_expression_tiles_sigma(k):
    multi, single = _pair(40, k, "expr", True, seed=5)
    z = dev.to_device(Q[:20, :3])
    for f in (multi, single):
        ma, ea = f._torch_expression(z)
        assert ma.shape == ea.shape == (20, k)
    ma, ea = multi._torch_expression(z)
    mb, eb = single._torch_expression(z)
    np.testing.assert_allclose(ma.cpu().numpy(), mb.cpu().numpy(), rtol=1e-12, atol=1e-12)
    assert_array_equal(ea.cpu().numpy(), eb.cpu().numpy())
    m0, e0 = multi.predict_device(z)
    np.testing.assert_allclose(ma.cpu().numpy(), m0.cpu().numpy(), rtol=1e-9, atol=1e-10)
    np.testing.assert_allclose(ea.cpu().numpy(), e0.cpu().numpy(), rtol=1e-9, atol=1e-10)
    # second derivatives exist
    x = z.clone().requires_grad_(True)
    mean, err = multi.torch(x)
    (g,) = torch.autograd.grad((mean.sum() + err.sum()), x, create_graph=True)
    (h,) = torch.autograd.grad(g.sum(), x)
    assert torch.isfinite(h).all()


# ---------------------------------------------------------------- closed loops and policy iteration
@pytest.mark.parametrize("prior", [True, False])
@pytest.mark.parametrize("kind", ["rbf", "expr"])
@pytest.mark.parametrize("M", [0, 7, 257])
@pytest.mark.parametrize("k", [1, 2, 3])
def test_rollouts_and_policy_iteration_equal_the_stack(k, M, kind, prior):
    din = k + 1
    multi, single = _pair(M, k, kind, prior, din=din, seed=100 + k * 10 + M)
    policy = sl.Saturation(sl.LinearSystem(-0.4 * np.ones((1, k))), -1., 1.)
    grid = sl.GridWorld(np.array([[-1., 1.]] * k), _num(k))
    x = np.random.default_rng(3).uniform(-1, 1, (200, k))
    reward = sl.QuadraticFunction(-np.diag(np.linspace(1.0, 2.0, din)))
    out = []
    for f in (multi, single):
        cl = sl.ClosedLoop(f.to_mean_function(), policy)
        roa, traj = sl.compute_roa(x, cl, 30, 0.05, no_traj=False)
        roa_grid = sl.compute_roa(grid, cl, 30, 0.05)
        sums = sl.reward_rollout(x, cl, sl.ClosedLoop(reward, policy), 0.9, 40, 1e-3)
        states, actions = sl.compute_trajectory(f.to_mean_function(), policy, x[:1], 12)
        v0 = -np.random.default_rng(2).random((grid.nindex, 1))
        rl = sl.PolicyIteration(policy, f, reward, sl.Triangulation(grid, v0.copy(), project=True), gamma=0.9)
        vi = [rl.value_iteration() for _ in range(2)]
        table = rl.value_function.parameters[0].copy()
        rl = sl.PolicyIteration(sl.Triangulation(grid, np.zeros((grid.nindex, 1))), f, reward,
                                sl.Triangulation(grid, v0.copy(), project=True), gamma=0.9)
        greedy = rl.discrete_policy_optimization(np.linspace(-1, 1, 5)[:, None]).cpu().numpy()
        out.append((roa, traj, roa_grid, sums, states, actions, np.array(vi), table, greedy))
    for a, b in zip(*out):
        assert_array_equal(a, b)


# ---------------------------------------------------------------- Lyapunov
@pytest.mark.parametrize("prior", [True, False])
@pytest.mark.parametrize("kind", ["rbf", "expr"])
@pytest.mark.parametrize("M", [0, 1, 7, 257, 500])
@pytest.mark.parametrize("k", [1, 2, 3, 4])
def test_update_safe_set_equals_the_stack(k, M, kind, prior):
    din = k + 1
    multi, single = _pair(M, k, kind, prior, din=din, seed=200 + k * 10 + M)
    results = []
    for f in (multi, single):
        got = []
        for filt in ("auto", False):
            ly = _lyapunov(f, k, _num(k))
            ly.filter = filt
            ly.update_safe_set()
            got += [ly.safe_set.copy(), ly.feed_dict[ly.c_max], ly.filter_stats]
            ly.update_safe_set(can_shrink=False)
            got += [ly.safe_set.copy(), ly.feed_dict[ly.c_max]]
        ly = _lyapunov(f, k, _num(k), adaptive=True)
        ly.update_safe_set(True, 4, 1.0)
        got += [ly.safe_set.copy(), ly.feed_dict[ly.c_max]]
        ly.update_safe_set(False, 4, 1.0)
        got += [ly.safe_set.copy(), ly.feed_dict[ly.c_max]]
        np.random.seed(7)
        sample, bound = sl.get_safe_sample(ly, perturbations=np.linspace(-0.2, 0.2, 3)[:, None],
                                           limits=np.array([[-1., 1.]]), num_samples=20)
        got += [np.asarray(sample), np.asarray(bound)]
        results.append(got)
    for a, b in zip(*results):
        if isinstance(a, dict):
            assert a == b
        else:
            assert_array_equal(a, b)


def test_grid_mean_scheme_on_two_columns():
    """C2's pendulum with one kernel for both state columns as ONE k = 2 GP: stage 1 takes the factored
    grid mean, and the flags, values, c_max and filter statistics equal the two-member stack's."""
    par = W.make_pendulum(num_points=64, M=300, shared_hypers=True, seed=3)
    gpu_stack = W.build_product(par)
    kern = sl.RBF(3, variance=par["variances"][0], lengthscales=par["lengthscales"][0])
    gp = sl.GaussianProcess(sl.GPRCached(par["X"], par["Y"], kern, mean_function=sl.LinearSystem(par["prior_rows"]),
                                         noise_variance=par["noise_variance"], scale=par["scale"]), beta=par["beta"])
    gpu_multi = sl.Lyapunov(sl.GridWorld(par["limits"], par["num_points"]), sl.QuadraticFunction(par["P"]), gp,
                            par["L_dyn"], sl.AbsFunction(sl.LinearSystem((2 * par["P"],))), par["tau"],
                            sl.Saturation(sl.LinearSystem(-par["K"]), -1., 1.), initial_set=par["initial"])
    lib = nat.load()
    for ly in (gpu_stack, gpu_multi):
        assert lib.slb_filter_mean_scheme(ly.sweep_descriptor()) == nat.MEAN_GRID_FACTORED
        ly.update_safe_set()
    assert_array_equal(gpu_multi.values, gpu_stack.values)
    assert_array_equal(gpu_multi.safe_set, gpu_stack.safe_set)
    assert gpu_multi.feed_dict[gpu_multi.c_max] == gpu_stack.feed_dict[gpu_stack.c_max]
    assert gpu_multi.filter_stats == gpu_stack.filter_stats


# ---------------------------------------------------------------- data updates
@pytest.mark.parametrize("M", [0, 7, 257])
@pytest.mark.parametrize("k", [2, 3])
def test_add_data_point_sequence(k, M):
    multi, single = _pair(M, k, "rbf", True, seed=300 + M)
    rng = np.random.default_rng(M)
    z = Q[:50, :3]
    for step in range(270):                            # past 256 appends: a refit
        x = rng.uniform(-1, 1, (1, 3))
        y = rng.standard_normal((1, k))
        multi.add_data_point(x, y)
        single.add_data_point(x, y)
        if step % 45 == 0 or step == 269:
            for a, b in zip(multi.predict_device(z), single.predict_device(z)):
                assert_array_equal(a.cpu().numpy(), b.cpu().numpy())
    assert multi.gaussian_process.Y.shape == (M + 270, k)
    assert_array_equal(multi.gaussian_process.Y, np.hstack([f.Y for f in single.functions]))


def test_mixed_stack_and_its_split():
    """A FunctionStack of a two-column and a one-column GP is the stack of its three columns, and
    add_data_point hands each member its columns."""
    two, two_single = _pair(60, 2, "rbf", True, seed=1)
    one, _ = _pair(45, 1, "expr", False, seed=2)
    mixed = sl.FunctionStack([two, one])
    flat = sl.FunctionStack(two_single.functions + [one])
    assert mixed.output_dim == 3
    z = Q[:, :3]
    for a, b in zip(mixed.predict_device(z), flat.predict_device(z)):
        assert_array_equal(a.cpu().numpy(), b.cpu().numpy())
    x = np.array([[0.1, -0.2, 0.3]])
    y = np.array([[1.0, 2.0, 3.0]])
    before = [f.gaussian_process.Y.shape[0] for f in (two, one)]
    mixed.add_data_point(x, y)
    assert_array_equal(two.gaussian_process.Y[-1], [1.0, 2.0])
    assert_array_equal(one.gaussian_process.Y[-1], [3.0])
    assert [f.gaussian_process.Y.shape[0] for f in (two, one)] == [b + 1 for b in before]
    mixed.add_data_point(x, y.ravel())                 # a flat row is one observation
    assert two.gaussian_process.Y.shape[0] == before[0] + 2


def test_packed_cache_round_trip():
    multi, single = _pair(100, 3, "rbf", True, seed=4)
    z = Q[:64, :3]
    m0, e0 = multi.predict_device(z)
    packed = multi.export_cache()
    gp = multi.gaussian_process
    gp._alpha_dev.zero_()
    packed.restore()
    torch.cuda.synchronize()
    m1, e1 = multi.predict_device(z)
    assert_array_equal(m0.cpu().numpy(), m1.cpu().numpy())
    tables = gp.export_cache(pinned=False)
    assert tuple(tables["alpha"].shape) == (3, 104)
    gp._gamma_f_dev.zero_()
    gp.import_cache(tables)
    torch.cuda.synchronize()
    assert_array_equal(single.to_mean_function()(z), multi.to_mean_function()(z))


# ---------------------------------------------------------------- joint log marginal likelihood
@pytest.mark.parametrize("M", [1, 63, 64, 65, 500, 1000])
@pytest.mark.parametrize("k", [1, 2, 3, 6])
def test_joint_lml_matches_the_reference_and_the_column_sum(k, M):
    din = 3
    X, Y, rows = _data(M, k, din, seed=M + k)
    for idx, (name, builder) in enumerate(LR.kernel_set(din)):
        noise = 0.05
        gp = sl.GPR(X, Y, builder(sl.kernels), noise_variance=noise, mean_function=sl.LinearSystem(rows),
                    scale=1.7)
        lml, grads = gp.log_likelihood_and_gradient()
        assert gp.compute_log_likelihood() == lml
        ref_lml, ref_grads, mags = LC.log_likelihood_and_gradient_cols(builder(LR.ORACLE_KERNELS),
                                                                       LR.Noise(noise), X, Y, rows)
        assert abs(lml - ref_lml) <= 1e-9 * (abs(ref_lml) + M * k), name
        assert list(grads) == list(ref_grads)
        for path, g in grads.items():
            want, mag = ref_grads[path], mags[path]
            if np.ndim(g) == 0:
                want, mag = want.sum(), mag.sum()
            assert np.all(np.abs(np.asarray(g) - want) <= 1e-7 * mag + 1e-300), (name, path, g, want, mag)
        # the sum of the k one-column fits (same kernel objects, so the same kernel matrix)
        parts = [sl.GPR(X, Y[:, [c]], gp.kern, noise_variance=noise, mean_function=sl.LinearSystem(rows[[c]]),
                        scale=1.7).log_likelihood_and_gradient() for c in range(k)]
        assert abs(lml - sum(p[0] for p in parts)) <= 1e-10 * (abs(ref_lml) + M * k), name
        for path, g in grads.items():
            mag = mags[path].sum() if np.ndim(g) == 0 else mags[path]
            want = sum(np.asarray(p[1][path]) for p in parts)
            assert np.all(np.abs(np.asarray(g) - want) <= 1e-7 * mag + 1e-300), (name, path)
        if k == 1:
            assert_array_equal(np.asarray(grads[path]), np.asarray(parts[0][1][path]))


def _lml_model(M, k, seed):
    X, Y, rows = _data(M, k, 3, seed)
    return sl.GPRCached(X, Y, _kernel("expr", 3), mean_function=sl.LinearSystem(rows), noise_variance=0.05), X, Y, rows


@pytest.mark.parametrize("M", [1, 64, 300])
def test_cols_entry_point_k1_is_the_one_column_call(M):
    gp, X, Y, rows = _lml_model(M, 1, seed=M)
    lib = nat.load()
    kstruct = nat.SlbKernel()
    gp.kern.fill(kstruct, 3)
    Xd = dev.to_device(X)
    K = gp.kern.K_device(Xd) + torch.eye(M, dtype=torch.float64, device=Xd.device) * gp.likelihood.variance
    L = torch.linalg.cholesky(K)
    kinv = torch.cholesky_inverse(L).contiguous()
    alpha = dev.to_device(np.random.default_rng(M).standard_normal((M, 1)))
    work = dev.empty((int(lib.slb_gp_lml_grad_workspace(M)) // 8,))
    outs = []
    for call in range(3):
        grad = dev.empty((nat.SLB_GP_HYPER_SLOTS,))
        if call == 0:
            rc = lib.slb_gp_lml_grad(dev.stream(), Xd.data_ptr(), M, 3, kstruct, kinv.data_ptr(), alpha.data_ptr(),
                                     grad.data_ptr(), work.data_ptr())
        else:
            rc = lib.slb_gp_lml_grad_cols(dev.stream(), Xd.data_ptr(), M, 3, kstruct, kinv.data_ptr(),
                                          alpha.data_ptr(), 1, grad.data_ptr(), work.data_ptr())
        assert rc == 0
        outs.append(grad.cpu().numpy())
    assert_array_equal(outs[0], outs[1])
    assert_array_equal(outs[1], outs[2])
    # two k = 4 calls are bit-identical too
    alpha4 = dev.to_device(np.random.default_rng(M + 1).standard_normal((M, 4)))
    runs = []
    for _ in range(2):
        grad = dev.empty((nat.SLB_GP_HYPER_SLOTS,))
        assert lib.slb_gp_lml_grad_cols(dev.stream(), Xd.data_ptr(), M, 3, kstruct, kinv.data_ptr(),
                                        alpha4.data_ptr(), 4, grad.data_ptr(), work.data_ptr()) == 0
        runs.append(grad.cpu().numpy())
    assert_array_equal(runs[0], runs[1])


def test_optimize_two_columns_agrees_with_autograd():
    """optimize() on k = 2 data: the fused gradient at the start and at the optimum agrees with torch
    autograd of the joint LML (the sum of both columns' log densities), and the fit converges."""
    _, X, Y, rows = _lml_model(120, 2, seed=9)
    kern = sl.RBF(3, variance=0.6, lengthscales=[0.9, 1.05, 1.2], ARD=True)
    gp = sl.GPRCached(X, Y, kern, mean_function=sl.LinearSystem(rows), noise_variance=0.05)

    def autograd_lml():
        var = torch.tensor(float(kern.variance), dtype=torch.float64, requires_grad=True)
        ls = torch.tensor(np.asarray(kern.lengthscales, dtype=np.float64), requires_grad=True)
        noise = torch.tensor(gp.likelihood.variance, dtype=torch.float64, requires_grad=True)
        x = torch.from_numpy(X) / ls
        r2 = ((x[:, None, :] - x[None, :, :]) ** 2).sum(-1)
        K = var * torch.exp(-0.5 * r2) + noise * torch.eye(X.shape[0], dtype=torch.float64)
        L = torch.linalg.cholesky(K)
        d = torch.from_numpy(Y - X @ rows.T)
        a = torch.linalg.solve_triangular(L, d, upper=False)
        n, k = d.shape
        lml = -0.5 * n * k * np.log(2 * np.pi) - k * torch.log(torch.diagonal(L)).sum() - 0.5 * (a * a).sum()
        lml.backward()
        return float(lml), {"kern.variance": float(var.grad), "kern.lengthscales": ls.grad.numpy(),
                            "likelihood.variance": float(noise.grad)}

    for stage in range(2):
        lml, grads = gp.log_likelihood_and_gradient()
        ref, ref_grads = autograd_lml()
        assert abs(lml - ref) <= 1e-9 * abs(ref)
        for path, g in ref_grads.items():
            np.testing.assert_allclose(grads[path], g, rtol=1e-7, atol=1e-8 * abs(ref))
        if stage == 0:
            start = lml
            res = gp.optimize(maxiter=200)
            assert res.success or "ABNORMAL" in str(res.message)
    assert lml > start


# ---------------------------------------------------------------- the reference's multi-output GP (fixture)
GOLDEN = np.load(os.path.join(HERE, "golden", "multi_output_gp.npz"))


def _golden_gp(kind, k, M):
    g = GOLDEN
    tag = "%s_k%d_M%d" % (kind, k, M)
    kern = W.build_kernel(sl, str(g["kernel_" + kind]))
    gp = sl.GPRCached(g[tag + "_X"], g[tag + "_Y"], kern, mean_function=sl.LinearSystem(g[tag + "_rows"]),
                      scale=float(g["scale"]), noise_variance=float(g["noise"]))
    return tag, sl.GaussianProcess(gp, beta=float(g["beta"]))


@pytest.mark.parametrize("kind", ["rbf", "expr"])
@pytest.mark.parametrize("k, M", [(2, 40), (3, 33), (2, 0)])
def test_posterior_matches_the_reference(kind, k, M):
    g = GOLDEN
    tag, fun = _golden_gp(kind, k, M)
    for suffix in ("", "_after"):
        mean, err = fun(g["points"])
        assert mean.shape == err.shape == (g["points"].shape[0], k)
        np.testing.assert_allclose(mean, g[tag + "_mean" + suffix], rtol=1e-5, atol=1e-12)
        np.testing.assert_allclose(err, g[tag + "_err" + suffix], rtol=1e-5, atol=1e-12)
        if not suffix:
            fun.add_data_point(g[tag + "_xnew"], g[tag + "_ynew"])


def test_safe_set_matches_the_reference():
    g = GOLDEN
    p = {key[len("lyap_par_"):]: g[key] for key in g.files if key.startswith("lyap_par_")}
    kern = sl.RBF(3, variance=float(p["variances"][0]), lengthscales=p["lengthscales"][0])
    gp = sl.GPRCached(p["X"], p["Y"], kern, mean_function=sl.LinearSystem(p["prior_rows"]),
                      noise_variance=float(p["noise_variance"]), scale=float(p["scale"]))
    dynamics = sl.GaussianProcess(gp, beta=float(p["beta"]))
    grid = sl.GridWorld(p["limits"], p["num_points"])
    policy = sl.Saturation(sl.LinearSystem(-p["K"]), -1., 1.)
    lyap = sl.Lyapunov(grid, sl.QuadraticFunction(p["P"]), dynamics, float(p["L_dyn"]),
                       sl.AbsFunction(sl.LinearSystem((2 * p["P"],))), float(p["tau"]), policy,
                       initial_set=p["initial"].copy())
    # V agrees to the last ulp or two (the shim's matmul is a BLAS dot, the kernels sum left to right);
    # adopt the fixture's V so that the V-sorted prefix rule is compared on identical keys
    np.testing.assert_allclose(lyap.values, g["lyap_values"], rtol=4e-15, atol=1e-15)
    lyap.values = g["lyap_values"]
    lyap.update_safe_set()
    assert_array_equal(lyap.safe_set, g["lyap_safe_set"])
    assert lyap.feed_dict[lyap.c_max] == float(g["lyap_c_max"])
