"""CPU tests of the closed-loop rollouts (``safe_learning_b200.rollout``, ``csrc/rollout.cu``):
the restated reference helpers against the reference-generated fixture, the arithmetic the kernels
restate (row norm, discount table, chunked early stop), the host path for callables the kernels
cannot fuse, and the host-side checks of the C entry points."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import scipy.linalg

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import oracle as O  # noqa: E402
import rollout_oracle as R  # noqa: E402
import safe_learning_b200 as sl  # noqa: E402
from safe_learning_b200 import _native as nat  # noqa: E402
from safe_learning_b200.rollout import discount_table  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "rollout.npz")


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:  # pragma: no cover
        return False


# ---------------------------------------------------------------- arithmetic the kernels restate
@pytest.mark.parametrize("d", range(1, 7))
def test_row_norm_is_sequential_sum_of_squares(d):
    """np.linalg.norm(x, 2, axis=1) == sqrt(x0^2 + x1^2 + ...) summed left to right, on magnitudes
    spread over 60 binades (where other summation orders round differently)."""
    rng = np.random.default_rng(d)
    x = rng.standard_normal((200000, d)) * np.exp(rng.uniform(-30, 30, (200000, d)))
    ref = np.linalg.norm(x, ord=2, axis=1, keepdims=True).ravel()
    assert np.array_equal(R.row_norm_sequential(x), ref)


@pytest.mark.parametrize("discount", [0.95, 0.99, 0.9, 1.0, 0.5, 1.0 / 3.0])
def test_discount_table_is_python_pow(discount):
    table = discount_table(discount, 1000)
    expect = [discount ** t for t in range(1000)]
    assert table.dtype == np.float64
    assert [float(v) for v in table] == expect
    assert discount_table(discount, 0).shape == (0,)


def _reference_loop(rewards, table, tol):
    sums = np.zeros(rewards.shape[1])
    for t in range(rewards.shape[0]):
        temp = table[t] * rewards[t]
        sums += temp
        if np.max(np.abs(temp)) < tol:
            return sums, t
    return sums, -1


def _decaying(rng, horizon, n, stop):
    """Rewards whose discounted maximum first drops below 1e-3 at step `stop` (never if -1)."""
    r = rng.uniform(-1, 1, (horizon, n))
    for t in range(horizon):
        if stop >= 0 and t >= stop:
            r[t] *= 1e-6
        else:
            r[t, rng.integers(n)] = 5.0
    return r


@pytest.mark.parametrize("chunk", [32, 4, 1])
def test_chunked_early_stop_equals_reference_loop(chunk):
    rng = np.random.default_rng(chunk)
    cases = []
    for horizon in (0, 1, 2, 3, 31, 32, 33, 64, 65, 100):
        for stop in sorted({-1, 0, 1, chunk - 1, chunk, chunk + 1, 2 * chunk, horizon - 1, horizon // 2}):
            if stop < horizon:
                cases.append((horizon, stop))
    for horizon, stop in cases:
        for n in (1, 7, 300):
            r = _decaying(rng, horizon, n, stop)
            table = discount_table(0.97, horizon)
            got = R.chunked_reward_rollout(r, table, 1e-3, chunk)
            want = _reference_loop(r, table, 1e-3)
            assert got[1] == want[1] == (stop if stop >= 0 else -1), (horizon, stop, n)
            assert np.array_equal(got[0], want[0])


@pytest.mark.parametrize("chunk", [32, 3])
def test_chunked_early_stop_non_finite(chunk):
    """NaN anywhere keeps a step from converging (np.max propagates NaN); inf never passes."""
    rng = np.random.default_rng(7)
    for horizon in (1, 2, 10, 40, 70):
        for poison in ("nan", "inf", "-inf"):
            r = rng.uniform(-1e-5, 1e-5, (horizon, 50))          # every step would converge ...
            bad = rng.integers(horizon, size=max(1, horizon // 3))
            r[bad, rng.integers(50)] = float(poison)              # ... except the poisoned ones
            table = discount_table(0.9, horizon)
            for tol in (1e-3, 0.0, -1.0, np.inf, np.nan):
                got = R.chunked_reward_rollout(r, table, tol, chunk)
                with np.errstate(invalid="ignore"):
                    want = _reference_loop(r, table, tol)
                assert got[1] == want[1], (horizon, poison, tol)
                assert np.array_equal(got[0], want[0], equal_nan=True)


# ---------------------------------------------------------------- oracle against the fixture
def _golden():
    return np.load(GOLDEN, allow_pickle=False)


def _oracle_case(z, name):
    """The closed loop of a fixture case rebuilt from oracle objects."""
    kind = str(z[name + "_kind"])
    policy = O.Saturation(O.LinearSystem((-z[name + "_K"],)), -1.0, 1.0)
    if kind == "linear":
        dyn = O.LinearSystem((z[name + "_A"], z[name + "_B"]))
    elif kind == "pendulum":
        p = z[name + "_plant"]
        dyn = O.InvertedPendulum(p[0], p[1], p[2], p[3],
                                 normalization=[z[name + "_Tx"], z[name + "_Tu"]])
    else:
        p = z[name + "_plant"]
        dyn = O.CartPole(p[0], p[1], p[2], p[3], p[4],
                         normalization=[z[name + "_Tx"], z[name + "_Tu"]])
    reward = O.QuadraticFunction(z[name + "_reward"])
    return policy, dyn, reward


def _states(z, name):
    if name + "_states" in z.files:
        return z[name + "_states"]
    return O.GridWorld(z[name + "_limits"], z[name + "_num_points"])


@pytest.mark.parametrize("name", ["linear", "pendulum", "cartpole"])
def test_oracle_matches_reference_fixture(name):
    """Flags and T* equal; trajectories and sums within 1e-12 relative.  The reference ran on the
    fixture shim, whose tf.matmul is numpy's matmul: a different summation order than the oracle's
    left-to-right dot products, so the last bits differ."""
    z = _golden()
    policy, dyn, reward = _oracle_case(z, name)
    grid = _states(z, name)
    cl, rw = R.closed_loop(dyn, policy), R.closed_loop(reward, policy)
    H, tol = int(z[name + "_horizon"]), float(z[name + "_tol"])
    roa, traj = R.compute_roa(grid, cl, H, tol, no_traj=False)
    assert np.array_equal(roa, z[name + "_roa"])
    sub = z[name + "_traj_index"]
    np.testing.assert_allclose(traj[sub], z[name + "_traj"], rtol=1e-12, atol=1e-12)
    sums, stop = R.reward_rollout(grid, cl, rw, float(z[name + "_discount"]),
                                  int(z[name + "_reward_horizon"]), float(z[name + "_reward_tol"]))
    assert stop == int(z[name + "_stop"])
    np.testing.assert_allclose(sums, z[name + "_sums"], rtol=1e-12, atol=1e-12)


# ---------------------------------------------------------------- host path of the product
def _pendulum_parts():
    pend = sl.InvertedPendulum(0.15, 0.5, 0.1, 0.01, normalization=[np.deg2rad([180., 360.]), [0.6]])
    A, B = pend.linearize()
    K, _ = O.dlqr(A, B, np.diag([1., 1.]), np.eye(1))
    return pend, A, B, K


def test_unfused_callables_take_the_host_path():
    """Plain callables (no descriptors) run the reference's loop on the host -- no device is
    touched -- and match the oracle exactly (same numpy operations)."""
    _, A, B, K = _pendulum_parts()
    o_pol = O.Saturation(O.LinearSystem((-K,)), -1., 1.)
    o_dyn = O.LinearSystem((A, B))
    o_rew = O.QuadraticFunction(-scipy.linalg.block_diag(np.eye(2), 0.1 * np.eye(1)))
    cl, rw = R.closed_loop(o_dyn, o_pol), R.closed_loop(o_rew, o_pol)
    limits = [[-1., 1.], [-1., 1.]]
    grid, ogrid = sl.GridWorld(limits, [23, 19]), O.GridWorld(limits, [23, 19])
    for horizon in (0, 1, 2, 40):
        assert np.array_equal(sl.compute_roa(grid, cl, horizon, 0.05),
                              R.compute_roa(ogrid, cl, horizon, 0.05))
    roa, traj = sl.compute_roa(ogrid.all_points, cl, 25, 0.05, equilibrium=[0., 0.], no_traj=False)
    want_roa, want_traj = R.compute_roa(ogrid, cl, 25, 0.05, no_traj=False)
    assert np.array_equal(roa, want_roa) and np.array_equal(traj, want_traj)
    sums = sl.reward_rollout(grid, cl, rw, 0.95, 300, 1e-4)
    want, _ = R.reward_rollout(ogrid, cl, rw, 0.95, 300, 1e-4)
    assert np.array_equal(sums, want)
    # a ClosedLoop around plain callables is not fused either
    loop = sl.ClosedLoop(o_dyn, o_pol)
    assert not loop.fused
    assert np.array_equal(sl.compute_roa(grid, loop, 30, 0.05), R.compute_roa(ogrid, cl, 30, 0.05))


def test_reward_rollout_messages(capsys):
    cl = lambda x: 0.5 * x            # noqa: E731
    rw = lambda x: -np.sum(x * x, axis=1, keepdims=True)  # noqa: E731
    states = np.linspace(-1, 1, 20).reshape(10, 2)
    sums = sl.reward_rollout(states, cl, rw, 0.9, 0, 1e-3)
    assert np.array_equal(sums, np.zeros(10))
    assert capsys.readouterr().out == "Reward sums did not converge!\n"
    sl.reward_rollout(states, cl, rw, 0.9, 100, 1e-3)
    _, stop = R.reward_rollout(states, cl, rw, 0.9, 100, 1e-3)
    assert capsys.readouterr().out == "Reward sums converged after {} steps!\n".format(stop + 1)


def test_roa_argument_checks_follow_the_reference():
    cl = lambda x: 0.5 * x            # noqa: E731
    states = np.zeros((4, 2))
    with pytest.raises(IndexError):
        sl.compute_roa(states, cl, 0, no_traj=False)
    with pytest.raises(ValueError):
        sl.compute_roa(states, cl, -1, no_traj=False)
    assert sl.compute_roa(states, cl, 0).all() and sl.compute_roa(states, cl, -3).all()
    assert np.array_equal(sl.compute_roa(states + 1, cl, 1, 1e-3, equilibrium=np.ones((1, 2))),
                          np.ones(4, bool))


def test_gp_dynamics_cannot_form_a_closed_loop():
    gp = sl.GaussianProcess.__new__(sl.GaussianProcess)
    with pytest.raises(TypeError):
        sl.ClosedLoop(gp, sl.LinearSystem(np.ones((1, 2))))


@pytest.mark.skipif(_has_gpu(), reason="checks the behaviour without a CUDA device")
def test_fused_rollouts_need_a_device():
    """No CPU fallback: a fused closed loop without a device raises NativeLibraryError."""
    _, A, B, K = _pendulum_parts()
    policy = sl.Saturation(sl.LinearSystem((-K,)), -1., 1.)
    cl = sl.ClosedLoop(sl.LinearSystem((A, B)), policy)
    rw = sl.ClosedLoop(sl.QuadraticFunction(-np.eye(3)), policy)
    assert cl.fused and rw.fused
    grid = sl.GridWorld([[-1., 1.], [-1., 1.]], 11)
    with pytest.raises(nat.NativeLibraryError):
        sl.compute_roa(grid, cl, 10, 1e-3)
    with pytest.raises(nat.NativeLibraryError):
        sl.reward_rollout(grid, cl, rw, 0.9, 10, 1e-3)
    with pytest.raises(nat.NativeLibraryError):
        cl(np.zeros((3, 2)))


# ---------------------------------------------------------------- C entry points
def test_rollout_symbols_exported():
    lib = nat.load()
    for name in ("slb_rollout", "slb_reward_rollout", "slb_rollout_workspace"):
        assert name in nat.SIGNATURES
        assert getattr(lib, name) is not None


def _linear_cfg(d=2):
    """A closed-loop descriptor with fake (never dereferenced) device pointers."""
    cfg = nat.SlbBellman()
    cfg.grid.ndim, cfg.grid.nindex = d, 9 ** d
    for c in range(d):
        cfg.grid.num_points[c], cfg.grid.unit_maxes[c] = 9, 0.25
    cfg.policy.kind, cfg.policy.in_dim, cfg.policy.out_dim = nat.FN_LINEAR, d, 1
    cfg.policy.matrix = 0x1000
    cfg.dynamics.kind, cfg.dynamics.in_dim, cfg.dynamics.out_dim = nat.FN_LINEAR, d + 1, d
    cfg.dynamics.matrix = 0x2000
    cfg.reward.kind, cfg.reward.in_dim, cfg.reward.out_dim = nat.FN_QUADRATIC, d + 1, 1
    cfg.reward.matrix = 0x3000
    return cfg


@pytest.mark.parametrize("mutate, message", [
    (lambda c: setattr(c.gp, "num_outputs", 2), "GP dynamics"),
    (lambda c: setattr(c.grid, "ndim", 7), "state dimension"),
    (lambda c: setattr(c.policy, "kind", nat.FN_NONE), "policy is required"),
    (lambda c: setattr(c.policy, "kind", 42), "not implemented"),
    (lambda c: setattr(c.dynamics, "in_dim", 2), "expects 3 inputs"),
    (lambda c: setattr(c.dynamics, "out_dim", 3), "columns"),
    (lambda c: setattr(c.reward, "out_dim", 1) or setattr(c.reward, "kind", nat.FN_LINEAR)
     or setattr(c.reward, "out_dim", 2), "one column"),
    (lambda c: setattr(c, "fixed_action", 1), "fixed_action"),
])
def test_host_checks_precede_any_launch(mutate, message):
    """Malformed descriptors are rejected by host-side checks (no device needed), with the reason in
    slb_last_error like every other entry point."""
    lib = nat.load()
    cfg = _linear_cfg()
    mutate(cfg)
    rc = lib.slb_reward_rollout(None, cfg, None, 0, 81, 10, C.c_void_p(0x4000), 1e-3,
                                C.c_void_p(0x5000), C.c_void_p(0x6000), C.c_void_p(0x7000))
    assert rc == 1 and message in nat.last_error(), nat.last_error()


def test_host_checks_of_sizes_and_pointers():
    lib = nat.load()
    cfg = _linear_cfg()
    eq = (C.c_double * 2)()
    rc = lib.slb_rollout(None, cfg, None, 0, 81, -1, eq, 1e-3, C.c_void_p(0x10), None, None, None)
    assert rc == 1 and "negative horizon" in nat.last_error()
    rc = lib.slb_rollout(None, cfg, None, 0, 82, 5, eq, 1e-3, C.c_void_p(0x10), None, None, None)
    assert rc == 1 and "outside the grid" in nat.last_error()
    rc = lib.slb_rollout(None, cfg, None, 0, 81, 0, eq, 1e-3, C.c_void_p(0x10), None,
                         C.c_void_p(0x20), None)
    assert rc == 1 and "horizon >= 1" in nat.last_error()
    rc = lib.slb_rollout(None, cfg, None, 0, 81, 5, eq, 1e-3, None, None, None, None)
    assert rc == 1 and "null flag output" in nat.last_error()
    rc = lib.slb_rollout(None, cfg, None, 0, 81, 100, eq, 1e-3, C.c_void_p(0x10), None, None, None)
    assert rc == 1 and "workspace" in nat.last_error()
    assert lib.slb_rollout(None, cfg, None, 0, 0, 5, eq, 1e-3, None, None, None, None) == 0   # n = 0
    assert lib.slb_rollout_workspace(cfg, 1000, 0) >= 2 * 1000 * 2 * 8
    assert lib.slb_rollout_workspace(cfg, 1000, 1) >= 2 * 1000 * 3 * 8 + 32 * 8
    assert lib.slb_rollout_workspace(cfg, 0, 1) == 0
