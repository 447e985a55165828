"""The Triangulation lookup (``tri_lookup``, csrc/common.cuh) at every dimension it is compiled for,
d = 1..6, with and without projection and with 1, 2 and 6 output columns, against the exact reference
``tests/triangulation_reference.py``: evaluation, the gradient flag (``Triangulation.gradient`` and
``MaxAbsFunction(gradient_function())``), the value operator's rows with the grid-line repair
(``slb_value_operator_points``, csrc/value_opt.cu), and the certified solve of
``PolicyIteration.optimize_value_function`` on both tiers.  Every tolerance is the bound derived in the
reference; ``tests/test_triangulation_reference_host.py`` shows each check rejects a subtly wrong result."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import oracle as O  # noqa: E402
import triangulation_reference as R  # noqa: E402
import value_opt_oracle as V  # noqa: E402

pytestmark = pytest.mark.gpu
DIMS = range(1, 7)
OUTS = [1, 2, 6]


@pytest.fixture(scope="module")
def sl():
    import __graft_entry__
    __graft_entry__.build()
    import safe_learning_b200 as mod
    return mod


def _lookup(grid, project):
    return R.Lookup.of(O.Triangulation(grid, None, project=project))


def _rows(sl, tri, x):
    """slb_value_operator_points: (cols, weights, repaired rows, smallest weight, rho)."""
    import torch
    from safe_learning_b200 import _device as dev, _native as nat
    from safe_learning_b200.reinforcement_learning import min_weight_of_stats
    lib = nat.load()
    n, d = x.shape
    xs = dev.to_device(np.ascontiguousarray(x))
    cols = dev.empty((n, d + 1), torch.int32)
    w = dev.empty((n, d + 1))
    stats = dev.zeros((nat.VALUE_STATS,), torch.int64)
    nat.check(lib.slb_value_operator_points(dev.stream(), tri.descriptor(), xs.data_ptr(), n, cols.data_ptr(),
                                            w.data_ptr(), stats.data_ptr()), "slb_value_operator_points")
    raw = stats.cpu().numpy().view(np.uint64)
    return (cols.cpu().numpy(), w.cpu().numpy(), int(raw[2]), min_weight_of_stats(raw[0]),
            float(raw[1:2].view(np.float64)[0]))


# ---------------------------------------------------------------- a. affine vertex values
@pytest.mark.parametrize("out", OUTS)
@pytest.mark.parametrize("project", [False, True])
@pytest.mark.parametrize("d", DIMS)
def test_affine_values_and_gradient(sl, d, project, out):
    """v_j = a . x_j + b: every simplex, the wrong-side one of a grid line and an extrapolating one
    included, interpolates the same affine function, so the value is a . x + b (a . clip(x) + b under
    projection) and the gradient is a, within the rounding bound."""
    rng = np.random.default_rng(100 * d + 10 * out + project)
    grid = R.shape_grid(O, d)
    x = R.point_classes(grid, rng)
    a = rng.normal(size=(d, out))
    b = rng.normal(size=out)
    vals = grid.all_points @ a + b
    tri = sl.Triangulation(sl.GridWorld(grid.limits, grid.num_points), vals, project=project)
    got = tri(x)
    grad = tri.gradient(x) if out == 1 else None
    R.check_affine(_lookup(grid, project), x, got, grad, a, b, vals)


# ---------------------------------------------------------------- b. random vertex values
@pytest.mark.parametrize("out", OUTS)
@pytest.mark.parametrize("project", [False, True])
@pytest.mark.parametrize("d", DIMS)
def test_random_values_and_gradient(sl, d, project, out):
    """The value within the bound of the exact value of a simplex first-fit can pick; for one column the
    gradient (SLB_FLAG_GRADIENT) and its max-abs taken exactly, likewise."""
    rng = np.random.default_rng(200 * d + 10 * out + project)
    grid = R.shape_grid(O, d)
    x = R.point_classes(grid, rng)
    vals = rng.normal(size=(grid.nindex, out))
    tri = sl.Triangulation(sl.GridWorld(grid.limits, grid.num_points), vals, project=project)
    lk = _lookup(grid, project)
    R.check_values(lk, x, tri(x), vals)
    if out == 1:
        # finite coordinates near the top of the double range: the weights overflow, the gradient (a
        # constant of the simplex) does not
        huge = np.vstack([np.full((1, d), 1.5e308), np.full((1, d), -1.5e308)])
        xg = np.vstack([x, huge])
        R.check_gradients(lk, xg, tri.gradient(xg), vals)
        R.check_gradients(lk, xg, sl.MaxAbsFunction(tri.gradient_function())(xg), vals, maxabs=True)


# ---------------------------------------------------------------- c. value-operator rows
@pytest.mark.parametrize("project", [False, True])
@pytest.mark.parametrize("d", DIMS)
def test_value_operator_rows(sl, d, project):
    """Rows at next states that include exact grid-line points (the wrong-side lookup that the repair
    re-searches) and points projected onto the boundary: admissible simplex, exact weights, exact
    reconstruction, no negative weight inside, and the repaired-row count, smallest weight and rho of
    the restatement (value_opt_oracle)."""
    rng = np.random.default_rng(300 * d + project)
    grid = R.shape_grid(O, d)
    x = R.operator_points(grid, rng)
    tri = sl.Triangulation(sl.GridWorld(grid.limits, grid.num_points), np.zeros((grid.nindex, 1)),
                           project=project)
    cols, w, repaired, minw, rho = _rows(sl, tri, x)
    lk = _lookup(grid, project)
    only_repair = R.check_rows(lk, x, cols, w)
    ocols, ow, q6 = V.operator(O.Triangulation(grid, np.zeros(grid.nindex), project=project), x,
                               lookup="library")
    assert repaired == int(q6.sum()) >= only_repair
    assert minw == float(ow.min())
    assert rho == V.rho(ow)
    if d >= 2:
        assert repaired > 0, "no grid-line row was repaired"


# ---------------------------------------------------------------- d. the certified solve
SOLVE_GRIDS = [(1, [12288]), (1, [12289]), (2, [111, 111]), (3, [24] * 3), (4, [11] * 4), (5, [7] * 5),
               (6, [5] * 6), (1, [40]), (2, [21, 19]), (3, [9, 8, 7]), (4, [6, 5, 5, 4]), (5, [4] * 5),
               (6, [3, 4, 3, 3, 4, 3])]


def _ids(case):
    d, num = case
    n = int(np.prod(num))
    return "d%d-n%d-tier%d" % (d, n, 2 if n > 12288 else 1)


@pytest.mark.parametrize("case", SOLVE_GRIDS, ids=[_ids(c) for c in SOLVE_GRIDS])
def test_certified_solve(sl, case):
    """optimize_value_function on the composed path (numpy callables): values and iteration count bit
    for bit with the restatement, the tier from the size (one CTA up to 12288 vertices), and the values
    within the certified bound plus the derived slack of an extended-precision fixed point."""
    d, num = case
    gamma = 0.9
    limits = [[-1.0 - 0.1 * c, 1.0 + 0.2 * c] for c in range(d)]
    grid = sl.GridWorld(limits, num)
    n = grid.nindex
    value = sl.Triangulation(grid, np.zeros((n, 1)), project=True)
    rot = np.roll(np.eye(d), 1, axis=1)

    def policy(x):
        return -0.5 * x[:, :1]

    def dynamics(x, u):                 # leaves the grid on both sides: projected rows
        return 0.7 * x @ rot + 0.4 * x + 0.3 * u

    def reward(x, u):
        return -np.sum(x * x, axis=1, keepdims=True) - 0.1 * u * u

    rl = sl.PolicyIteration(policy, dynamics, reward, value, gamma=gamma)
    got = rl.optimize_value_function().ravel()
    info = rl.last_solve
    assert info["tier"] == (2 if n > 12288 else 1)
    ogrid = O.GridWorld(limits, num)
    states = ogrid.all_points
    u = policy(states)
    nxt = dynamics(states, u)
    rewards = reward(states, u).ravel()
    cols, w, q6 = V.operator(O.Triangulation(ogrid, np.zeros(n), project=True), nxt, lookup="library")
    v, iters, delta, bound = V.solve(cols, w, rewards, gamma, np.zeros(n))
    # the certificate users get: rho, the last delta and the bound equal the restatement's bit for bit
    assert info["iterations"] == iters
    assert info["repaired_rows"] == int(q6.sum())
    assert info["rho"] == V.rho(w) and info["min_weight"] == float(w.min())
    assert info["delta"] == delta and info["bound"] == bound
    assert np.array_equal(got, v)
    # and it holds: the values within bound + slack of the exact fixed point
    slack = R.solve_slack(w, rewards, gamma, got, d, info["bound"])
    vstar, err = R.fixed_point(cols, w, rewards, gamma, 1e-3 * (info["bound"] + slack))
    dev, lim = R.check_fixed_point(got, vstar, err, info["bound"], slack)
    print("d=%d n=%d tier %d: %d iterations, |v - v*| = %.3g <= bound %.3g + slack %.3g"
          % (d, n, info["tier"], iters, dev, info["bound"], slack))
