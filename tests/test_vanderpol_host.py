"""Host tests of the reverse-time Van der Pol plant (``VanDerPol``, ``SLB_FN_VANDERPOL``): the numpy oracle
against the reference-generated fixture, the descriptor the Python object writes, and the library's host
checks of the new kind (shape validation, column count, VJP workspace and parameter rejection)."""
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
from vanderpol_oracle import VanDerPol  # noqa: E402

GOLDEN = np.load(os.path.join(HERE, "golden", "vanderpol.npz"))


def _lib():
    return nat.load()


def _oracle(name):
    g = GOLDEN
    return VanDerPol(float(g["damping"]), float(g["dt"]), g["Tx"] if name == "norm" else None)


def _closed_loop():
    return R.closed_loop(_oracle("norm"), O.LinearSystem((np.zeros((1, 2)),)))


# ---------------------------------------------------------------- the oracle against the reference
@pytest.mark.parametrize("name", ["plain", "norm"])
def test_oracle_one_step_and_linearize_match_reference(name):
    sa = GOLDEN["step_inputs"]
    want = GOLDEN["step_" + name]
    got = _oracle(name)(sa[:, :2], sa[:, 2:])
    assert np.array_equal(got, want, equal_nan=True)
    assert not np.isfinite(want).all()                   # the fixture has overflowing rows
    assert np.array_equal(_oracle(name).linearize(), GOLDEN["linearize_" + name])


def test_oracle_normalisation_is_a_matrix_product():
    vdp = _oracle("norm")
    np.testing.assert_array_equal(vdp.denormalize(np.array([[np.inf, 1.]])), [[np.inf, np.nan]])
    np.testing.assert_array_equal(vdp.normalize(np.array([[2., np.nan]])), [[np.nan, np.nan]])


@pytest.mark.parametrize("case", ["grid", "states"])
def test_oracle_compute_roa_matches_reference(case):
    g = GOLDEN
    start = (O.GridWorld(g["grid_limits"], g["grid_num_points"]) if case == "grid" else g["states"])
    roa, traj = R.compute_roa(start, _closed_loop(), int(g[case + "_horizon"]), float(g[case + "_tol"]),
                              no_traj=False)
    assert np.array_equal(roa, g[case + "_roa"])
    assert np.array_equal(traj[g[case + "_traj_index"]], g[case + "_traj"], equal_nan=True)
    assert not np.isfinite(g[case + "_traj"]).all()      # trajectories that escape are in the fixture


@pytest.mark.parametrize("case", ["grid", "inner"])
def test_oracle_reward_rollout_matches_reference(case):
    g = GOLDEN
    start = (O.GridWorld(g["grid_limits"], g["grid_num_points"]) if case == "grid" else g["inner_states"])
    reward = R.closed_loop(O.QuadraticFunction(g["reward"]), O.LinearSystem((np.zeros((1, 2)),)))
    with np.errstate(over="ignore", invalid="ignore"):
        sums, stop = R.reward_rollout(start, _closed_loop(), reward, float(g[case + "_discount"]),
                                      int(g[case + "_reward_horizon"]), float(g[case + "_reward_tol"]))
    assert np.array_equal(sums, g[case + "_sums"], equal_nan=True)
    assert stop == int(g[case + "_stop"])


def test_oracle_safe_set_matches_reference():
    g = GOLDEN
    vdp = _oracle("norm")
    P = scipy.linalg.solve_discrete_lyapunov(vdp.linearize().T, 0.1 * np.eye(2))
    assert np.array_equal(P, g["lyap_P"])
    lyap = O.Lyapunov(O.GridWorld(g["lyap_limits"], g["lyap_num_points"]), O.QuadraticFunction(P), vdp,
                      float(g["lyap_L_f"]), float(g["lyap_L_v"]), float(g["lyap_tau"]),
                      O.LinearSystem((np.zeros((1, 2)),)), g["lyap_initial"].copy())
    # V = x^T P x summed in another order than the reference's matmul: equal to a few ulp; the safe set
    # and c_max are then decided on the reference's values
    np.testing.assert_allclose(lyap.values, g["lyap_values"], rtol=4e-15, atol=1e-15)
    lyap.values = g["lyap_values"]
    lyap.update_safe_set()
    assert np.array_equal(lyap.safe_set, g["lyap_safe_set"])
    assert lyap.c_max == float(g["lyap_c_max"])


# ---------------------------------------------------------------- the Python object and its descriptor
def test_descriptor_layout():
    vdp = sl.VanDerPol(damping=1.5, dt=0.02, normalization=(2.5, 3.0))
    assert (vdp.state_dim, vdp.action_dim, vdp.input_dim, vdp.output_dim) == (2, 0, 3, 2)
    assert vdp.name == "VanDerPol"
    d = vdp.descriptor()
    assert (d.kind, d.in_dim, d.out_dim, d.flags) == (nat.FN_VANDERPOL, 3, 2, 0)
    assert list(d.cparams[:7]) == [1.5, 0.02 / 10, 1.0, 2.5, 3.0, 2.5 ** -1, 3.0 ** -1]
    assert all(c == 0.0 for c in d.cparams[7:])
    plain = sl.VanDerPol().descriptor()
    assert list(plain.cparams[:3]) == [1.0, 0.01 / 10, 0.0]
    assert all(c == 0.0 for c in plain.cparams[3:])


@pytest.mark.parametrize("name", ["plain", "norm"])
def test_linearize_and_normalize_match_oracle(name):
    tx = GOLDEN["Tx"] if name == "norm" else None
    vdp, ovdp = sl.VanDerPol(1, 0.01, tx), _oracle(name)
    assert np.array_equal(vdp.linearize(), GOLDEN["linearize_" + name])
    x = np.array([[np.inf, 1.], [0.5, -0.25], [1., np.nan]])
    assert np.array_equal(vdp.normalize(x), ovdp.normalize(x), equal_nan=True)
    assert np.array_equal(vdp.denormalize(x), ovdp.denormalize(x), equal_nan=True)


# ---------------------------------------------------------------- host checks of the library
def _desc(in_dim=3, out_dim=2, flags=0):
    d = sl.VanDerPol(normalization=(2.5, 3.0)).descriptor()
    d.in_dim, d.out_dim, d.flags = in_dim, out_dim, flags
    return d


def test_columns_and_validation():
    lib = _lib()
    assert lib.slb_function_columns(_desc()) == 2
    assert lib.slb_function_columns(_desc(flags=nat.FLAG_NORM1)) == 1
    # slb_eval_function validates before it needs a device or the points
    for in_dim, out_dim in ((2, 2), (3, 3), (4, 2), (3, 1)):
        assert lib.slb_eval_function(None, _desc(in_dim, out_dim), 0x1000, 4, 0x2000) != 0
        assert "Van der Pol must map 3 -> 2" in nat.last_error()


def test_validation_accepts_three_to_two_as_dynamics():
    lib = _lib()
    cfg = nat.SlbBellman()
    cfg.grid = sl.GridWorld([[-1., 1.], [-1., 1.]], 5).descriptor()
    cfg.policy.kind, cfg.policy.in_dim, cfg.policy.out_dim = nat.FN_LINEAR, 2, 1
    cfg.policy.matrix = 0x1000               # never read: nothing is launched
    eq = np.zeros(2)

    def rollout():           # an empty range: validated, nothing launched
        return lib.slb_rollout(None, cfg, None, 0, 0, 10, eq.ctypes.data, 0.1, None, None, None, None)

    cfg.dynamics = _desc()
    assert rollout() == 0, nat.last_error()
    cfg.dynamics = _desc(4, 2)
    assert rollout() != 0
    assert "Van der Pol must map 3 -> 2" in nat.last_error()


def test_vjp_workspace_and_parameters():
    lib = _lib()
    assert lib.slb_function_vjp_workspace(_desc(), 10 ** 6) == 0
    assert lib.slb_function_vjp(None, _desc(), 0x1000, 10, 0x2000, 0x3000, 0x4000, None, None) != 0
    assert "grad_params must be NULL" in nat.last_error()
    assert lib.slb_function_vjp_workspace(_desc(flags=nat.FLAG_SCALE), 10) == -1
    assert "flags" in nat.last_error()
