"""GPU tests of the reverse-time Van der Pol plant (``VanDerPol``, ``SLB_FN_VANDERPOL``) in every path that
takes plants: one-step evaluation, the VJP and ``Function.torch``, the fused rollouts, the Lyapunov sweep
behind ``update_safe_set`` and the Bellman sweep of ``value_iteration``; against the numpy oracle and the
reference-generated fixture."""
import os
import sys

import numpy as np
import pytest
import scipy.linalg
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import oracle as O  # noqa: E402
import rollout_oracle as R  # noqa: E402
import safe_learning_b200 as sl  # noqa: E402
from vanderpol_oracle import VanDerPol  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(HERE, "golden", "vanderpol.npz"))


def _tx(name):
    return GOLDEN["Tx"] if name == "norm" else None


def _pair(name="norm"):
    g = GOLDEN
    args = (float(g["damping"]), float(g["dt"]), _tx(name))
    return sl.VanDerPol(*args), VanDerPol(*args)


def _stop_of(capsys):
    out = capsys.readouterr().out.strip().splitlines()[-1]
    if "did not converge" in out:
        return -1
    return int(out.split("after ")[1].split(" ")[0]) - 1


# ---------------------------------------------------------------- one step
@pytest.mark.parametrize("name", ["plain", "norm"])
def test_evaluate_device_bit_identical(name):
    vdp, ovdp = _pair(name)
    sa = GOLDEN["step_inputs"]
    got = vdp.evaluate_device(sa).cpu().numpy()
    assert np.array_equal(got, GOLDEN["step_" + name], equal_nan=True)
    assert not np.isfinite(got).all()
    # seeded states over the region of interest, and the numpy call path
    x = np.random.default_rng(7).uniform(-2., 2., (4096, 3))
    assert np.array_equal(vdp(x[:, :2], x[:, 2:]), ovdp(x[:, :2], x[:, 2:]), equal_nan=True)


def _torch_step(z, damping, dt, tx):
    """The plant as a torch-CPU recurrence (the normalisation as matrix products)."""
    s = z[:, :2]
    if tx is not None:
        s = s @ torch.diag(torch.tensor(tx, dtype=torch.float64))
    for _ in range(10):
        x, y = s[:, 0:1], s[:, 1:2]
        s = s + (dt / 10) * torch.cat((-y, x + damping * (x ** 2 - 1) * y), dim=1)
    if tx is not None:
        s = s @ torch.diag(torch.tensor(tx, dtype=torch.float64) ** -1)
    return s


@pytest.mark.parametrize("name", ["plain", "norm"])
def test_jacobian_and_backward_match_autograd(name):
    vdp, _ = _pair(name)
    g = GOLDEN
    z = np.random.default_rng(8).uniform(-1.5, 1.5, (500, 3))
    zc = torch.tensor(z, requires_grad=True)
    out = _torch_step(zc, float(g["damping"]), float(g["dt"]), _tx(name))
    want = torch.stack([torch.autograd.grad(out[:, o].sum(), zc, retain_graph=True)[0] for o in range(2)],
                       dim=1).numpy()
    assert np.all(want[:, :, 2] == 0.0)
    J = vdp.jacobian_device(torch.tensor(z, device="cuda")).cpu().numpy()
    assert J.shape == (500, 2, 3)
    assert np.all(J[:, :, 2] == 0.0)
    np.testing.assert_allclose(J, want, rtol=1e-12, atol=1e-12 * np.abs(want).max())
    # Function.torch: one autograd node whose backward is the fused VJP
    cot = np.random.default_rng(9).standard_normal((500, 2))
    zg = torch.tensor(z, device="cuda", requires_grad=True)
    y = vdp.torch(zg)
    np.testing.assert_array_equal(y.detach().cpu().numpy(), vdp.evaluate_device(z).cpu().numpy())
    (y * torch.tensor(cot, device="cuda")).sum().backward()
    (gin,) = torch.autograd.grad(out, zc, torch.tensor(cot))
    np.testing.assert_allclose(zg.grad.cpu().numpy(), gin.numpy(), rtol=1e-12,
                               atol=1e-12 * np.abs(gin.numpy()).max())


# ---------------------------------------------------------------- rollouts
def _loops():
    vdp, _ = _pair("norm")
    policy = sl.LinearSystem(np.zeros((1, 2)))
    return sl.ClosedLoop(vdp, policy), sl.ClosedLoop(sl.QuadraticFunction(GOLDEN["reward"]), policy)


@pytest.mark.parametrize("case", ["grid", "states"])
def test_compute_roa_matches_fixture(case):
    g = GOLDEN
    cl, _ = _loops()
    horizon, tol = int(g[case + "_horizon"]), float(g[case + "_tol"])
    if case == "grid":
        grid = sl.GridWorld(g["grid_limits"], g["grid_num_points"])
        sources = (grid, grid.all_points)
    else:
        sources = (g["states"],)
    for source in sources:
        roa = sl.compute_roa(source, cl, horizon, tol)
        assert np.array_equal(roa, g[case + "_roa"])
        roa, traj = sl.compute_roa(source, cl, horizon, tol, no_traj=False)
        assert np.array_equal(roa, g[case + "_roa"])
        picked = traj[g[case + "_traj_index"]]
        assert np.array_equal(picked, g[case + "_traj"], equal_nan=True)
        assert not np.isfinite(picked).all()


@pytest.mark.parametrize("case", ["grid", "inner"])
def test_reward_rollout_matches_fixture(case, capsys):
    g = GOLDEN
    cl, rw = _loops()
    if case == "grid":
        grid = sl.GridWorld(g["grid_limits"], g["grid_num_points"])
        sources = (grid, grid.all_points)
    else:
        sources = (g["inner_states"],)
    for source in sources:
        sums = sl.reward_rollout(source, cl, rw, float(g[case + "_discount"]), int(g[case + "_reward_horizon"]),
                                 float(g[case + "_reward_tol"]))
        assert _stop_of(capsys) == int(g[case + "_stop"])
        assert np.array_equal(sums, g[case + "_sums"], equal_nan=True)


# ---------------------------------------------------------------- Lyapunov sweep
def _lyapunov_args(ns, vdp, V):
    g = GOLDEN
    return (ns.GridWorld(g["lyap_limits"], g["lyap_num_points"]), V, vdp, float(g["lyap_L_f"]),
            float(g["lyap_L_v"]), float(g["lyap_tau"]), ns.LinearSystem((np.zeros((1, 2)),)),
            g["lyap_initial"].copy())


def test_update_safe_set_quadratic_matches_fixture():
    g = GOLDEN
    vdp, ovdp = _pair("norm")
    gpu = sl.Lyapunov(*_lyapunov_args(sl, vdp, sl.QuadraticFunction(g["lyap_P"])))
    cpu = O.Lyapunov(*_lyapunov_args(O, ovdp, O.QuadraticFunction(g["lyap_P"])))
    gpu.update_values()
    assert np.array_equal(gpu.values, cpu.values)
    # the reference sums x^T P x in its matmul's order: a few ulp apart; decide on its values
    np.testing.assert_allclose(gpu.values, g["lyap_values"], rtol=4e-15, atol=1e-15)
    gpu.values = cpu.values = g["lyap_values"]
    gpu.update_safe_set()
    cpu.update_safe_set()
    assert np.array_equal(gpu.safe_set, g["lyap_safe_set"])
    assert np.array_equal(cpu.safe_set, g["lyap_safe_set"])
    assert gpu.feed_dict[gpu.c_max] == float(g["lyap_c_max"]) == cpu.c_max
    assert 0 < g["lyap_safe_set"].sum() < g["lyap_safe_set"].size


def test_update_safe_set_lyapunov_network_matches_oracle():
    vdp, ovdp = _pair("norm")
    net = sl.LyapunovNetwork(2, [16, 16], ["tanh", "tanh"], seed=5)
    onet = O.LyapunovNetwork(2, net.output_dims, [np.tanh] * 2, net.weights, eps=net.eps)
    gpu = sl.Lyapunov(*_lyapunov_args(sl, vdp, net))
    cpu = O.Lyapunov(*_lyapunov_args(O, ovdp, onet))
    gpu.update_values()
    np.testing.assert_allclose(gpu.values, cpu.values, rtol=1e-12, atol=1e-15)
    gpu.values = cpu.values                       # identical sort keys (tanh differs by an ulp)
    gpu.update_safe_set()
    cpu.update_safe_set()
    assert np.array_equal(gpu.safe_set, cpu.safe_set)
    assert gpu.feed_dict[gpu.c_max] == cpu.c_max
    assert np.all(gpu.safe_set[GOLDEN["lyap_initial"]])


# ---------------------------------------------------------------- Bellman sweep
def test_value_iteration_matches_oracle():
    vdp, ovdp = _pair("norm")
    limits = [[-1., 1.], [-1., 1.]]
    reward = GOLDEN["reward"]
    grid, ogrid = sl.GridWorld(limits, 31), O.GridWorld(limits, 31)
    v0 = -np.sum(ogrid.all_points ** 2, axis=1, keepdims=True)
    rl_g = sl.PolicyIteration(sl.LinearSystem((np.zeros((1, 2)),)), vdp, sl.QuadraticFunction(reward),
                              sl.Triangulation(grid, v0, project=True))
    rl_c = O.PolicyIteration(O.LinearSystem((np.zeros((1, 2)),)), ovdp, O.QuadraticFunction(reward),
                             O.Triangulation(ogrid, v0, project=True))
    res = rl_g.value_iteration()
    new = rl_c.value_iteration()
    np.testing.assert_allclose(rl_g.value_function.parameters[0], new, rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(res, np.max(np.abs(new - v0)), rtol=1e-12)
