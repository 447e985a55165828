"""GPU tests of the fused closed-loop rollouts (``compute_roa`` / ``reward_rollout``,
``csrc/rollout.cu``) against the CPU oracle, the library's own one-step evaluations and the
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
from safe_learning_b200 import rollout as rollout_mod  # noqa: E402
from safe_learning_b200.rollout import discount_table  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(HERE, "golden", "rollout.npz")


def _pendulum_setup():
    """reinforcement_learning_pendulum.ipynb cells 7-14: normalised plant, saturated LQR."""
    theta_max, omega_max = np.deg2rad(30), np.sqrt(9.81 / 0.5)
    u_max = 9.81 * 0.15 * 0.5 * np.sin(theta_max)
    norm = [np.array([theta_max, omega_max]), np.array([u_max])]
    args = (0.15, 0.5, 0.1, 0.01)
    pend = sl.InvertedPendulum(*args, normalization=norm)
    opend = O.InvertedPendulum(*args, normalization=norm)
    A, B = pend.linearize()
    Q, Rm = 0.1 * np.eye(2), 0.1 * np.eye(1)
    K, _ = O.dlqr(A, B, Q, Rm)
    return pend, opend, A, B, K, scipy.linalg.block_diag(-Q, -Rm)


def _cartpole_setup():
    m, M, L, b, dt = 0.175, 1.732, 0.28, 0.01, 0.01
    tx = np.array([0.5, np.deg2rad(30), 2., np.deg2rad(30)])
    tu = np.array([(m + M) * 4 / 0.5])
    cp, ocp = sl.CartPole(m, M, L, b, dt, [tx, tu]), O.CartPole(m, M, L, b, dt, [tx, tu])
    A, B = cp.linearize()
    Q, Rm = 0.1 * np.eye(4), 0.1 * np.eye(1)
    K, _ = O.dlqr(A, B, Q, Rm)
    return cp, ocp, K, scipy.linalg.block_diag(-Q, -Rm)


def _linear_loops(A, B, K, rew):
    policy = sl.Saturation(sl.LinearSystem((-K,)), -1., 1.)
    cl = sl.ClosedLoop(sl.LinearSystem((A, B)), policy)
    rw = sl.ClosedLoop(sl.QuadraticFunction(rew), policy)
    opol = O.Saturation(O.LinearSystem((-K,)), -1., 1.)
    ocl = R.closed_loop(O.LinearSystem((A, B)), opol)
    orw = R.closed_loop(O.QuadraticFunction(rew), opol)
    return cl, rw, ocl, orw


def _stop_of(capsys):
    out = capsys.readouterr().out.strip().splitlines()[-1]
    if "did not converge" in out:
        return -1
    return int(out.split("after ")[1].split(" ")[0]) - 1


# ---------------------------------------------------------------- linear closed loop: bit for bit
@pytest.mark.parametrize("num_points, horizon", [([67, 53], 77), ([29, 31], 33), ([41, 37], 100)])
def test_linear_closed_loop_bit_exact(num_points, horizon, capsys):
    _, _, A, B, K, rew = _pendulum_setup()
    cl, rw, ocl, orw = _linear_loops(A, B, K, rew)
    limits = [[-5., 5.], [-5., 5.]]
    grid, ogrid = sl.GridWorld(limits, num_points), O.GridWorld(limits, num_points)
    want_roa, want_traj = R.compute_roa(ogrid, ocl, horizon, 0.5, no_traj=False)
    assert 0 < want_roa.sum() < want_roa.size
    for source in (grid, ogrid.all_points):
        roa = sl.compute_roa(source, cl, horizon, 0.5)
        assert np.array_equal(roa, want_roa)
        roa, traj = sl.compute_roa(source, cl, horizon, 0.5, no_traj=False)
        assert np.array_equal(roa, want_roa)
        assert traj.dtype == np.float64 and traj.shape == want_traj.shape
        assert np.array_equal(traj, want_traj)
    for disc, tol, rh in ((0.98, 1e-2, 400), (0.9, 1e-3, 1000), (0.95, 1e-30, 70)):
        want, want_stop = R.reward_rollout(ogrid, ocl, orw, disc, rh, tol)
        for source in (grid, ogrid.all_points):
            got = sl.reward_rollout(source, cl, rw, disc, rh, tol)
            assert _stop_of(capsys) == want_stop
            assert np.array_equal(got, want)


def test_linear_stop_at_every_position_of_a_chunk(capsys):
    """T* at many offsets inside and at the edges of the 32-step chunks: tol swept over the
    reference's own per-step maxima."""
    _, _, A, B, K, rew = _pendulum_setup()
    cl, rw, ocl, orw = _linear_loops(A, B, K, rew)
    states = np.random.default_rng(3).uniform(-0.8, 0.8, (1000, 2))
    cur, maxima = states, []
    for t in range(120):
        maxima.append(np.max(np.abs((0.97 ** t) * orw(cur).ravel())))
        cur = ocl(cur)
    for target in (0, 1, 30, 31, 32, 33, 63, 64, 65, 95, 110):
        tol = np.nextafter(maxima[target], np.inf)
        want, want_stop = R.reward_rollout(states, ocl, orw, 0.97, 120, tol)
        got = sl.reward_rollout(states, cl, rw, 0.97, 120, tol)
        assert _stop_of(capsys) == want_stop
        assert np.array_equal(got, want)


# ---------------------------------------------------------------- plants: against the one-step path
def _compose(policy, dynamics, reward, states, horizon, disc, tol):
    """h compositions of the library's one-step device evaluations."""
    x = torch.as_tensor(states, dtype=torch.float64, device="cuda").contiguous()
    traj = [x]
    for _ in range(1, horizon):
        u = policy.evaluate_device(x)
        x = dynamics.evaluate_device(torch.cat((x, u), dim=1))
        traj.append(x)
    traj = torch.stack(traj, dim=2).cpu().numpy()
    x = torch.as_tensor(states, dtype=torch.float64, device="cuda").contiguous()
    sums, stop = torch.zeros(x.shape[0], dtype=torch.float64, device="cuda"), -1
    table = discount_table(disc, horizon)
    for t in range(horizon):
        z = torch.cat((x, policy.evaluate_device(x)), dim=1)
        temp = table[t] * reward.evaluate_device(z)[:, 0]
        sums = sums + temp
        if float(torch.max(torch.abs(temp)).item()) < tol:
            stop = t
            break
        x = dynamics.evaluate_device(z)
    return traj, sums.cpu().numpy(), stop


def _plant_cases():
    pend, opend, A, B, K, rew = _pendulum_setup()
    cp, ocp, Kc, rewc = _cartpole_setup()
    # tanh hidden layer whose linearisation at the origin is the LQR gain
    w1 = 0.05 * np.random.default_rng(4).standard_normal((2, 16))
    w2 = np.linalg.pinv(w1).dot(-K.T)
    nn = sl.NeuralNetwork([2, 16, 1], ["tanh", None], weights=[w1, w2], biases=[np.zeros(16)])
    onn = O.NeuralNetwork([2, 16, 1], [np.tanh, None], [w1, w2], [np.zeros(16)])
    return {
        "pendulum": (sl.Saturation(sl.LinearSystem((-K,)), -1., 1.), pend, sl.QuadraticFunction(rew),
                     O.Saturation(O.LinearSystem((-K,)), -1., 1.), opend, O.QuadraticFunction(rew),
                     sl.GridWorld([[-3., 3.], [-3., 3.]], [53, 47]), 300, 1e-2),
        "cartpole": (sl.Saturation(sl.LinearSystem((-Kc,)), -1., 1.), cp, sl.QuadraticFunction(rewc),
                     O.Saturation(O.LinearSystem((-Kc,)), -1., 1.), ocp, O.QuadraticFunction(rewc),
                     sl.GridWorld([[-2., 2.]] * 4, [7, 9, 7, 9]), 400, 0.1),
        "pendulum_nn": (sl.Saturation(nn, -1., 1.), pend, sl.QuadraticFunction(rew),
                        O.Saturation(onn, -1., 1.), opend, O.QuadraticFunction(rew),
                        sl.GridWorld([[-2., 2.], [-2., 2.]], [37, 41]), 200, 1e-2),
    }


def _boundary(ocl, start, horizon, tol, flag):
    """The oracle's own flag flips when the start state moves by a few ulp."""
    for k in (1, 2, 4, 8, 16):
        for c in range(start.size):
            for direction in (np.inf, -np.inf):
                x = start.copy()
                for _ in range(k):
                    x[c] = np.nextafter(x[c], direction)
                if R.compute_roa(x[None, :], ocl, horizon, tol)[0] != flag:
                    return True
    return False


@pytest.mark.parametrize("case", ["pendulum", "cartpole", "pendulum_nn"])
def test_plant_closed_loops(case, capsys):
    pol, dyn, rew, opol, odyn, orew, grid, horizon, tol = _plant_cases()[case]
    cl, rw = sl.ClosedLoop(dyn, pol), sl.ClosedLoop(rew, pol)
    states = grid.index_to_state(np.arange(grid.nindex))
    # fused == the library's one-step evaluations composed h times (bit for bit)
    roa, traj = sl.compute_roa(grid, cl, horizon, tol, no_traj=False)
    ref_traj, ref_sums, ref_stop = _compose(pol, dyn, rew, states, horizon, 0.98, 1e-2)
    assert np.array_equal(traj, ref_traj)
    assert np.array_equal(roa, R.row_norm_sequential(ref_traj[:, :, -1]) <= tol)
    sums = sl.reward_rollout(grid, cl, rw, 0.98, horizon, 1e-2)
    assert _stop_of(capsys) == ref_stop
    assert np.array_equal(sums, ref_sums)
    # against the oracle: flags and T* equal (a differing flag sits on a basin boundary);
    # trajectories inside the ROA within 1e-9 (device sin/cos/tanh differ from numpy's in the last bit)
    ocl, orw = R.closed_loop(odyn, opol), R.closed_loop(orew, opol)
    o_roa, o_traj = R.compute_roa(states, ocl, horizon, tol, no_traj=False)
    assert 0 < o_roa.sum() < o_roa.size
    differ = np.flatnonzero(roa != o_roa)
    assert differ.size <= max(2, roa.size // 1000)
    for i in differ:
        assert _boundary(ocl, states[i], horizon, tol, o_roa[i]), "flag of start state %d" % i
    both = roa & o_roa
    np.testing.assert_allclose(traj[both], o_traj[both], rtol=0, atol=1e-9)
    o_sums, o_stop = R.reward_rollout(states, ocl, orw, 0.98, horizon, 1e-2)
    assert o_stop == ref_stop
    np.testing.assert_allclose(sums[both], o_sums[both], rtol=1e-9, atol=1e-12)


def test_closed_loop_call_is_one_step():
    pol, dyn, _, opol, odyn, _, grid, _, _ = _plant_cases()["pendulum"]
    x = grid.index_to_state(np.arange(0, grid.nindex, 7))
    want = dyn(x, pol(x))
    assert np.array_equal(sl.ClosedLoop(dyn, pol)(x), want)


# ---------------------------------------------------------------- against the reference's fixture
@pytest.mark.parametrize("name", ["linear", "pendulum", "cartpole"])
def test_against_reference_fixture(name, capsys):
    z = np.load(GOLDEN)
    K, rew = z[name + "_K"], z[name + "_reward"]
    pol = sl.Saturation(sl.LinearSystem((-K,)), -1., 1.)
    opol = O.Saturation(O.LinearSystem((-K,)), -1., 1.)
    if name == "linear":
        dyn, odyn = sl.LinearSystem((z["linear_A"], z["linear_B"])), O.LinearSystem((z["linear_A"], z["linear_B"]))
    elif name == "pendulum":
        p, norm = z["pendulum_plant"], [z["pendulum_Tx"], z["pendulum_Tu"]]
        dyn, odyn = sl.InvertedPendulum(*p, normalization=norm), O.InvertedPendulum(*p, normalization=norm)
    else:
        p, norm = z["cartpole_plant"], [z["cartpole_Tx"], z["cartpole_Tu"]]
        dyn, odyn = sl.CartPole(*p, normalization=norm), O.CartPole(*p, normalization=norm)
    if name + "_states" in z.files:
        source = states = z[name + "_states"]
    else:
        source = sl.GridWorld(z[name + "_limits"], z[name + "_num_points"])
        states = source.index_to_state(np.arange(source.nindex))
    cl, rw = sl.ClosedLoop(dyn, pol), sl.ClosedLoop(sl.QuadraticFunction(rew), pol)
    H, tol = int(z[name + "_horizon"]), float(z[name + "_tol"])
    roa, traj = sl.compute_roa(source, cl, H, tol, no_traj=False)
    ocl = R.closed_loop(odyn, opol)
    for i in np.flatnonzero(roa != z[name + "_roa"]):
        assert _boundary(ocl, states[i], H, tol, z[name + "_roa"][i]), "flag of start state %d" % i
    sub = z[name + "_traj_index"]
    inside = z[name + "_roa"][sub] & roa[sub]
    np.testing.assert_allclose(traj[sub][inside], z[name + "_traj"][inside], rtol=0, atol=1e-9)
    if name == "linear":                 # no transcendental functions: only matmul's summation order
        np.testing.assert_allclose(traj[sub], z[name + "_traj"], rtol=1e-12, atol=1e-12)
    sums = sl.reward_rollout(source, cl, rw, float(z[name + "_discount"]),
                             int(z[name + "_reward_horizon"]), float(z[name + "_reward_tol"]))
    assert _stop_of(capsys) == int(z[name + "_stop"])
    fin = np.isfinite(z[name + "_sums"])
    assert np.array_equal(np.isfinite(sums), fin)
    keep = fin & roa
    np.testing.assert_allclose(sums[keep], z[name + "_sums"][keep], rtol=1e-9, atol=1e-12)


# ---------------------------------------------------------------- edge cases
def test_short_horizons(capsys):
    _, _, A, B, K, rew = _pendulum_setup()
    cl, rw, ocl, orw = _linear_loops(A, B, K, rew)
    grid = sl.GridWorld([[-1., 1.], [-2., 2.]], [13, 11])
    ogrid = O.GridWorld([[-1., 1.], [-2., 2.]], [13, 11])
    for h in (0, 1, 2):
        assert np.array_equal(sl.compute_roa(grid, cl, h, 0.5), R.compute_roa(ogrid, ocl, h, 0.5))
        if h >= 1:
            roa, traj = sl.compute_roa(grid, cl, h, 0.5, no_traj=False)
            want_roa, want_traj = R.compute_roa(ogrid, ocl, h, 0.5, no_traj=False)
            assert np.array_equal(roa, want_roa) and np.array_equal(traj, want_traj)
        got = sl.reward_rollout(grid, cl, rw, 0.9, h, 1e-3)
        want, stop = R.reward_rollout(ogrid, ocl, orw, 0.9, h, 1e-3)
        assert _stop_of(capsys) == stop
        assert np.array_equal(got, want)
    with pytest.raises(IndexError):
        sl.compute_roa(grid, cl, 0, 0.5, no_traj=False)
    # T* = 0: the first rewards are already below tol
    got = sl.reward_rollout(grid, cl, rw, 0.9, 50, 1e3)
    assert _stop_of(capsys) == 0
    assert np.array_equal(got, R.reward_rollout(ogrid, ocl, orw, 0.9, 50, 1e3)[0])


def test_diverging_closed_loop(capsys):
    """States overflow to inf / NaN: outside the ROA, sums non-finite where the oracle's are."""
    A, B = 3.0 * np.eye(2), np.zeros((2, 1))
    K = np.zeros((1, 2))
    cl, rw, ocl, orw = _linear_loops(A, B, K, -np.eye(3))
    states = np.random.default_rng(0).uniform(-1, 1, (777, 2))
    states[5] = 0.0
    roa = sl.compute_roa(states, cl, 800, 1e-3)
    assert np.array_equal(roa, R.compute_roa(states, ocl, 800, 1e-3))
    assert roa.sum() == 1 and roa[5]
    got = sl.reward_rollout(states, cl, rw, 0.99, 900, 1e-3)
    want, stop = R.reward_rollout(states, ocl, orw, 0.99, 900, 1e-3)
    assert stop == -1 and _stop_of(capsys) == -1
    assert np.array_equal(np.isfinite(got), np.isfinite(want))
    assert not np.isfinite(got).all()


def test_trajectories_over_several_slabs(monkeypatch):
    _, _, A, B, K, rew = _pendulum_setup()
    cl, _, ocl, _ = _linear_loops(A, B, K, rew)
    grid, ogrid = sl.GridWorld([[-4., 4.], [-4., 4.]], [39, 27]), O.GridWorld([[-4., 4.], [-4., 4.]], [39, 27])
    monkeypatch.setattr(rollout_mod, "TRAJECTORY_SLAB_BYTES", 100 * 2 * 45 * 8 + 8)   # 100 points
    roa, traj = sl.compute_roa(grid, cl, 45, 0.05, no_traj=False)
    want_roa, want_traj = R.compute_roa(ogrid, ocl, 45, 0.05, no_traj=False)
    assert np.array_equal(roa, want_roa) and np.array_equal(traj, want_traj)


def test_empty_state_array():
    _, _, A, B, K, rew = _pendulum_setup()
    cl, rw, _, _ = _linear_loops(A, B, K, rew)
    empty = np.zeros((0, 2))
    assert sl.compute_roa(empty, cl, 50, 1e-2).shape == (0,)
    roa, traj = sl.compute_roa(empty, cl, 50, 1e-2, no_traj=False)
    assert roa.shape == (0,) and traj.shape == (0, 2, 50)
    with pytest.raises(ValueError):                 # the reference's np.max over no states
        sl.reward_rollout(empty, cl, rw, 0.9, 10, 1e-3)
    assert sl.reward_rollout(empty, cl, rw, 0.9, 0, 1e-3).shape == (0,)
