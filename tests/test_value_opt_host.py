"""CPU tests of exact policy evaluation (``PolicyIteration.optimize_value_function``,
``csrc/value_opt.cu``): the numpy restatement against the fixture made by the unmodified reference
(LP solved by HiGHS), the grid-line (Q6) repair, and the host-side checks of the C entry points."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import oracle as O  # noqa: E402
import value_opt_oracle as V  # noqa: E402
import safe_learning_b200 as sl  # noqa: E402
from safe_learning_b200 import _native as nat  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "value_optimization.npz")
EPS = np.finfo(np.float64).eps


def _golden():
    return np.load(GOLDEN, allow_pickle=False)


def lqr_setup(z, name):
    """The fixture's saturated linear closed loop on the case's grid, as oracle objects."""
    grid = O.GridWorld([[-1., 1.], [-1., 1.]], z[name + "_num_points"])
    tri = O.Triangulation(grid, np.zeros(grid.nindex), project=True)
    states = grid.all_points
    actions = O.Saturation(O.LinearSystem((-z["K"],)), -1., 1.)(states)
    next_states = O.LinearSystem((z["A"], z["B"]))(states, actions)
    rewards = O.QuadraticFunction(z["reward"])(states, actions).ravel()
    return grid, tri, next_states, rewards


def _ref_rows(z, name, n):
    T = sp.coo_matrix((z[name + "_T_data"], (z[name + "_T_rows"], z[name + "_T_cols"])), shape=(n, n))
    return T


@pytest.mark.parametrize("name", ["lqr24", "lqr25"])
def test_restated_operator_equals_reference_outside_q6(name):
    z = _golden()
    grid, tri, nxt, rewards = lqr_setup(z, name)
    np.testing.assert_allclose(nxt, z[name + "_next_states"], rtol=1e-15, atol=1e-15)
    np.testing.assert_allclose(rewards, z[name + "_rewards"].ravel(), rtol=1e-14, atol=1e-15)
    cols, w, q6 = V.operator(tri, z[name + "_next_states"])
    n = grid.nindex
    rows = z[name + "_T_rows"].reshape(n, -1)
    assert np.array_equal(rows, np.repeat(np.arange(n), 3).reshape(n, 3))
    ref_cols = z[name + "_T_cols"].reshape(n, 3)
    ref_w = z[name + "_T_data"].reshape(n, 3)
    assert np.array_equal(cols[~q6], ref_cols[~q6])
    assert np.array_equal(w[~q6], ref_w[~q6])                 # bit for bit
    # the repaired rows are exactly the reference's rows with a negative weight
    assert np.array_equal(q6, np.min(ref_w, axis=1) < -1e-12)
    assert q6.sum() == (9 if name == "lqr25" else 0)


@pytest.mark.parametrize("num_points", [[24, 20], [25, 21], [512, 512]])
def test_library_lookup_differs_from_qhull_only_on_ties(num_points):
    """Where the library's simplex search and Qhull pick different simplices, both rows are valid
    (after the Q6 repair) and interpolate the point: the pick is a tie on a shared face."""
    z = _golden()
    zz = dict(z)
    zz["x_num_points"] = np.array(num_points)
    grid, tri, nxt, _ = lqr_setup(zz, "x")
    c1, w1, _ = V.operator(tri, nxt)
    c2, w2, _ = V.operator(tri, nxt, lookup="library")
    differ = np.any(c1 != c2, axis=1)
    assert differ.sum() <= 4
    for cols, w in ((c1, w1), (c2, w2)):
        assert np.min(w) >= -1e-12
        pts = np.einsum("qk,qkc->qc", w[differ], grid.all_points[cols[differ]])
        np.testing.assert_allclose(pts, nxt[differ], rtol=0, atol=1e-12)


def test_repaired_rows_interpolate_the_point():
    z = _golden()
    grid, tri, _, _ = lqr_setup(z, "lqr25")
    nxt = z["lqr25_next_states"]
    cols, w, q6 = V.operator(tri, nxt)
    assert q6.any()
    wr = w[q6]
    assert np.all(wr >= -1e-12) and np.all(wr <= 1 + 1e-12)
    assert np.all(np.abs(wr.sum(axis=1) - 1.0) <= 4 * EPS)
    verts = grid.all_points[cols[q6]]                          # [q, 3, 2]
    np.testing.assert_allclose(np.einsum("qk,qkc->qc", wr, verts), nxt[q6], rtol=0, atol=1e-12)


def test_reference_lp_matches_spsolve_and_the_restated_iteration():
    z = _golden()
    grid, tri, nxt, rewards = lqr_setup(z, "lqr24")
    n = grid.nindex
    lp = z["lqr24_values"].ravel()
    assert str(z["lqr24_status"]) == "optimal"
    T = _ref_rows(z, "lqr24", n).tocsr()
    exact = spla.spsolve((sp.identity(n) - z["lqr24_gamma"] * T).tocsc(), rewards)
    assert np.max(np.abs(exact - lp)) <= 1e-9 * np.max(np.abs(exact))
    cols, w, _ = V.operator(tri, nxt)
    v, iters, _, bound = V.solve(cols, w, rewards, float(z["lqr24_gamma"]), np.zeros(n))
    assert iters > 10
    err = np.max(np.abs(v - exact))
    assert err <= bound + 10 * EPS * np.max(np.abs(exact)) / (1 - z["lqr24_gamma"])
    assert np.max(np.abs(v - lp)) <= 1e-8 * np.max(np.abs(lp))


def test_reference_lp_is_unbounded_on_grid_line_rows():
    """The reference's 25 x 21 operator has weight -1 rows; its LP is unbounded.  The restated
    operator repairs them and then has a fixed point that agrees with spsolve."""
    z = _golden()
    assert "unbounded" in str(z["lqr25_status"])
    grid, tri, nxt, rewards = lqr_setup(z, "lqr25")
    cols, w, q6 = V.operator(tri, nxt)
    with pytest.raises(ValueError):
        V.solve(z["lqr25_T_cols"].reshape(-1, 3), z["lqr25_T_data"].reshape(-1, 3), rewards, 0.98,
                np.zeros(grid.nindex))
    v, _, _, bound = V.solve(cols, w, rewards, 0.98, np.zeros(grid.nindex))
    exact = np.linalg.solve(np.eye(grid.nindex) - 0.98 * V.dense(cols, w, grid.nindex), rewards)
    assert np.max(np.abs(v - exact)) <= bound + 10 * EPS * np.max(np.abs(exact)) / 0.02


def test_transition_matrix_case():
    """The reference's own test: LP optimum == solve(I - gamma T, r).  Its second row sums to 1.1,
    so gamma rho = 1.078: the certified iteration refuses it (a Triangulation's rows sum to 1), and
    with the discount lowered until gamma rho < 1 it agrees with the direct solve."""
    z = _golden()
    T, r, g = z["matrix_T"], z["matrix_rewards"].ravel(), float(z["matrix_gamma"])
    exact = np.linalg.solve(np.eye(4) - g * T, r)
    np.testing.assert_allclose(z["matrix_values"].ravel(), exact, rtol=1e-9)
    cols = np.tile(np.arange(4), (4, 1))
    assert V.rho(T) == 1.1 + 2 * EPS or abs(V.rho(T) - 1.1) < 1e-15
    with pytest.raises(ValueError, match="contraction"):
        V.solve(cols, T, r, g, np.zeros(4))
    g = 0.9
    exact = np.linalg.solve(np.eye(4) - g * T, r)
    v, _, _, bound = V.solve(cols, T, r, g, np.zeros(4), tol=1e-12)
    assert np.max(np.abs(v - exact)) <= bound + 1e-12 * np.max(np.abs(exact))


# ---------------------------------------------------------------- Python API without a device
def test_policy_iteration_has_optimize_value_function():
    assert callable(getattr(sl.PolicyIteration, "optimize_value_function", None))


def test_unknown_solver_options_raise_type_error():
    """cvxpy's solver / verbose / eps / warm_start are accepted; anything else is a TypeError,
    raised before any device work."""
    grid = sl.GridWorld([[-1., 1.], [-1., 1.]], [5, 4])
    value = sl.Triangulation(grid, None, project=True)
    rl = sl.PolicyIteration(lambda x: x[:, :1], lambda x, u: x, lambda x, u: x[:, :1], value)
    with pytest.raises(TypeError, match="max_iter"):
        rl.optimize_value_function(max_iter=10)
    with pytest.raises(TypeError):
        rl.optimize_value_function(solver="ECOS", abstol=1e-3)


# ---------------------------------------------------------------- C entry points
def test_value_opt_symbols_exported():
    lib = nat.load()
    for name in ("slb_value_operator", "slb_value_operator_points", "slb_value_solve",
                 "slb_value_solve_workspace"):
        assert name in nat.SIGNATURES
        assert getattr(lib, name) is not None
    assert lib.slb_abi_version() == 6


def _solve(lib, **kw):
    args = dict(n=100, ncols=3, cols=C.c_void_p(0x1000), w=C.c_void_p(0x2000), r=C.c_void_p(0x3000),
                gamma=0.9, tol=1e-10, max_iters=100, v=C.c_void_p(0x4000), work=C.c_void_p(0x5000),
                stats=C.c_void_p(0x6000))
    args.update(kw)
    return lib.slb_value_solve(None, args["n"], args["ncols"], args["cols"], args["w"], args["r"],
                               args["gamma"], args["tol"], args["max_iters"], args["v"], args["work"],
                               args["stats"])


@pytest.mark.parametrize("kw, message", [
    (dict(gamma=1.0), "gamma"),
    (dict(gamma=-0.1), "gamma"),
    (dict(gamma=float("nan")), "gamma"),
    (dict(tol=0.0), "tol"),
    (dict(tol=float("nan")), "tol"),
    (dict(ncols=1), "ncols"),
    (dict(ncols=8), "ncols"),
    (dict(n=0), "n >= 1"),
    (dict(max_iters=0), "max_iters"),
    (dict(cols=None), "null"),
    (dict(stats=None), "null"),
    (dict(v=None), "null"),
    (dict(n=20000, work=None), "workspace"),
])
def test_solve_host_checks(kw, message):
    lib = nat.load()
    assert _solve(lib, **kw) == 1
    assert message in nat.last_error(), nat.last_error()


def test_solve_workspace_size():
    lib = nat.load()
    assert lib.slb_value_solve_workspace(262144, 3) >= 262144 * 8
    assert lib.slb_value_solve_workspace(12288, 3) == 0          # one-CTA tier: no workspace
    assert lib.slb_value_solve_workspace(12289, 3) >= 12289 * 8
    assert lib.slb_value_solve_workspace(0, 3) == 0
    assert lib.slb_value_solve_workspace(10, 9) == 0


def _tri_function(d=2):
    f = nat.SlbFunction()
    f.kind, f.in_dim, f.out_dim = nat.FN_TRIANGULATION, d, 1
    f.matrix, f.hyperplanes, f.unit_simplices, f.nsimplex = 0x1000, 0x2000, 0x3000, 2
    f.grid.ndim, f.grid.nindex = d, 5 ** d
    f.grid.discrete_points = 0x4000
    for c in range(d):
        f.grid.num_points[c], f.grid.unit_maxes[c] = 5, 0.5
    return f


@pytest.mark.parametrize("mutate, message", [
    (lambda f: setattr(f.grid, "ndim", 7), "ndim"),
    (lambda f: setattr(f, "kind", nat.FN_LINEAR), "Triangulation"),
    (lambda f: setattr(f, "out_dim", 2), "one-output"),
    (lambda f: setattr(f, "flags", nat.FLAG_SCALE), "plain"),
])
def test_operator_points_host_checks(mutate, message):
    lib = nat.load()
    f = _tri_function()
    mutate(f)
    rc = lib.slb_value_operator_points(None, f, C.c_void_p(0x10), 25, C.c_void_p(0x20),
                                       C.c_void_p(0x30), C.c_void_p(0x40))
    assert rc == 1 and message in nat.last_error(), nat.last_error()


def test_operator_points_null_stats():
    lib = nat.load()
    rc = lib.slb_value_operator_points(None, _tri_function(), C.c_void_p(0x10), 25, C.c_void_p(0x20),
                                       C.c_void_p(0x30), None)
    assert rc == 1 and "null stats" in nat.last_error()


def _bellman_cfg(d=2):
    cfg = nat.SlbBellman()
    cfg.grid.ndim, cfg.grid.nindex = d, 5 ** d
    for c in range(d):
        cfg.grid.num_points[c], cfg.grid.unit_maxes[c] = 5, 0.5
    cfg.policy.kind, cfg.policy.in_dim, cfg.policy.out_dim = nat.FN_LINEAR, d, 1
    cfg.policy.matrix = 0x1000
    cfg.dynamics.kind, cfg.dynamics.in_dim, cfg.dynamics.out_dim = nat.FN_LINEAR, d + 1, d
    cfg.dynamics.matrix = 0x2000
    cfg.reward.kind, cfg.reward.in_dim, cfg.reward.out_dim = nat.FN_QUADRATIC, d + 1, 1
    cfg.reward.matrix = 0x3000
    cfg.value = _tri_function(d)
    cfg.gamma = 0.9
    return cfg


@pytest.mark.parametrize("mutate, message", [
    (lambda c: setattr(c.grid, "ndim", 7), "ndim"),
    (lambda c: setattr(c, "fixed_action", 1), "fixed_action"),
    (lambda c: setattr(c.value, "kind", nat.FN_QUADRATIC), "Triangulation"),
    (lambda c: setattr(c.value, "flags", nat.FLAG_SCALE), "plain"),
    (lambda c: setattr(c.policy, "kind", nat.FN_NONE), "policy is required"),
    (lambda c: setattr(c.reward, "kind", nat.FN_NONE), "reward function is required"),
])
def test_operator_host_checks(mutate, message):
    lib = nat.load()
    cfg = _bellman_cfg()
    mutate(cfg)
    rc = lib.slb_value_operator(None, cfg, 0, 25, C.c_void_p(0x10), C.c_void_p(0x20),
                                C.c_void_p(0x30), C.c_void_p(0x40))
    assert rc == 1 and message in nat.last_error(), nat.last_error()


def test_operator_range_check():
    lib = nat.load()
    rc = lib.slb_value_operator(None, _bellman_cfg(), 0, 26, C.c_void_p(0x10), C.c_void_p(0x20),
                                C.c_void_p(0x30), C.c_void_p(0x40))
    assert rc == 1 and "outside the grid" in nat.last_error()


# ---------------------------------------------------------------- GP dynamics (notebook shapes)
def test_gp55_restatement_matches_reference():
    """Notebook-kernel GP pendulum on 55 x 55: the oracle's GP mean next states and the restated
    operator agree with the reference's (its GP mean is numpy matmul / TF-shim arithmetic, so to
    rounding), and the certified iteration reproduces the reference's LP optimum."""
    z = _golden()
    rl, grid = V.gp55_objects(O, "oracle")
    n = grid.nindex
    states = grid.all_points
    mean = rl.dynamics(states, rl.policy(states))[0]
    np.testing.assert_allclose(mean, z["gp55_next_states"], rtol=0, atol=1e-11)
    cols, w, q6 = V.operator(rl.value_function, z["gp55_next_states"])
    assert not q6.any()
    assert np.array_equal(cols.ravel(), z["gp55_T_cols"])
    assert np.array_equal(w.ravel(), z["gp55_T_data"])
    v, _, _, _ = V.evaluate(rl, lookup="qhull")
    lp = z["gp55_values"].ravel()
    assert np.max(np.abs(v - lp)) <= 1e-8 * np.max(np.abs(lp))


def test_gp1d_policy_iteration_loop_matches_reference():
    """1d_example cell 15 shape: three rounds of optimize_value_function ->
    discrete_policy_optimization with a GP model; values within the LP's tolerance, identical
    greedy policies."""
    z = _golden()
    rl, _ = V.gp1d_objects(O, z, "oracle")
    for k in range(3):
        v, _, _, _ = V.evaluate(rl, lookup="qhull")
        ref = z["gp1d_values"][k].ravel()
        assert np.max(np.abs(v - ref)) <= 1e-8 * max(1.0, np.max(np.abs(ref)))
        rl.value_function.parameters = v
        best = rl.discrete_policy_optimization(V.GP1D_ACTIONS)
        assert np.array_equal(best, z["gp1d_policies"][k])
