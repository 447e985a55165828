"""CPU tests of the exact Triangulation reference (``tests/triangulation_reference.py``): it reproduces the
unmodified reference's fixtures at d = 1..6 -- every group, vertex queries and outside queries included --
and every check the GPU tests use rejects a result that is wrong in one way at a time."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import oracle as O  # noqa: E402
import triangulation_reference as R  # noqa: E402
import value_opt_oracle as V  # noqa: E402

GOLDEN = os.path.join(HERE, "golden")


def load(name):
    return np.load(os.path.join(GOLDEN, name))


def _lookup(grid, project):
    return R.Lookup.of(O.Triangulation(grid, None, project=project))


# ---------------------------------------------------------------- the fixtures, d = 1..6
def test_reproduces_grid_triangulation_fixture():
    fix = load("grid_triangulation.npz")
    for tag in ("g1", "g2", "g3"):
        grid = O.GridWorld(fix[tag + "_limits"], fix[tag + "_num"])
        for project in (False, True):
            lk = _lookup(grid, project)
            key = tag + ("_proj" if project else "_noproj")
            for group, pts in (("inside", fix[tag + "_inside"]), ("vertices", grid.all_points),
                               ("outside", fix[tag + "_outside"])):
                R.check_values(lk, pts, fix[key + "_" + group], fix[tag + "_vals"], fixture=True)


def test_reproduces_triangulation_gradient_fixture():
    fix = load("triangulation_gradient.npz")
    for tag in ("g1", "g2", "g3"):
        grid = O.GridWorld(fix[tag + "_limits"], fix[tag + "_num"])
        R.check_gradients(_lookup(grid, False), fix[tag + "_inside"], fix[tag + "_gradient"], fix[tag + "_vals"],
                          fixture=True)


def test_reproduces_parameter_derivative_fixture():
    fix = load("triangulation_param_derivative.npz")
    for key in sorted(k[:-len("_points")] for k in fix.files if k.endswith("_points")):
        tag, proj, _ = key.split("_", 2)
        grid = O.GridWorld(fix[tag + "_limits"], fix[tag + "_num"])
        R.check_fixture_rows(_lookup(grid, proj == "proj"), fix[key + "_points"], fix[key + "_cols"],
                             fix[key + "_weights"])


@pytest.mark.parametrize("tag", ["h4", "h5", "h6"])
def test_reproduces_high_dim_fixture(tag):
    """Values, gradients and rows of every group; the corner group pins corner_simplex (Qhull's pick of
    each of the 2^d patterns) and the reference's unit_simplices / hyperplanes."""
    fix = load("triangulation_high_dim.npz")
    grid = O.GridWorld(fix[tag + "_limits"], fix[tag + "_num"])
    groups = ("inside", "faces", "vertices", "outside", "corners")
    for project in (False, True):
        otri = O.Triangulation(grid, None, project=project)
        np.testing.assert_array_equal(otri.unit_simplices, fix[tag + "_unit_simplices"])
        np.testing.assert_array_equal(otri.hyperplanes, fix[tag + "_hyperplanes"])
        lk = R.Lookup.of(otri)
        key = tag + ("_proj" if project else "_noproj")
        for group in groups:
            pts = fix[tag + "_" + group]
            R.check_values(lk, pts, fix[key + "_" + group + "_value"], fix[tag + "_vals"], fixture=True)
            R.check_fixture_rows(lk, pts, fix[key + "_" + group + "_cols"], fix[key + "_" + group + "_weights"])
            if not project:
                R.check_gradients(lk, pts, fix[tag + "_" + group + "_gradient"], fix[tag + "_gvals"],
                                  fixture=True)
        # the corner table is Qhull's pick: the library's row of each corner pattern is the reference's
        for i, p in enumerate(fix[tag + "_corners"]):
            corner, sims = lk.lookup_set(p)
            assert sims == [lk.corner_table[lk.cell(p)[3]]]
            assert np.array_equal(lk.simp[sims[0]] + corner, fix[key + "_corners_cols"][i])


def test_admissible_set_and_bound_are_small():
    """delta stays below W_TOL at d = 6, so a simplex that contains the unit point exactly always passes
    first-fit's test and the largest-smallest-weight fallback never applies to a finite point; the
    hyperplanes' rounding is a few ulps."""
    grid = R.shape_grid(O, 6)
    lk = _lookup(grid, False)
    assert lk.S == 652 and lk.D_unit.max() < 1e-14
    rng = np.random.default_rng(0)
    for p in R.point_classes(grid, rng)[:-1]:
        _, unit, _, _ = lk.cell(p)
        _, delta = lk.screen(unit)
        assert delta.max() < R.W_TOL


# ---------------------------------------------------------------- every check rejects a wrong result
def _library_values(lk, otri, x, V_):
    """What a correct kernel computes (fp64, first-fit simplex): value_opt_oracle's restatement."""
    corners = otri.discretization.rectangle_corner_index(otri.discretization.state_to_rectangle(x))
    sims = V.library_simplices(otri, x)
    out = []
    for p, c, s in zip(x, corners, sims):
        w = V._barycentric(otri, p, c, s)
        out.append(w @ V_[otri.unit_simplices[s] + c])
    return np.array(out)


@pytest.mark.parametrize("d,project", [(2, False), (3, True), (6, False), (6, True)])
def test_value_check_rejects_wrong_results(d, project):
    grid = R.shape_grid(O, d)
    rng = np.random.default_rng(d)
    vals = rng.normal(size=(grid.nindex, 2))
    otri = O.Triangulation(grid, vals, project=project)
    lk = R.Lookup.of(otri)
    x = rng.uniform(grid.limits[:, 0], grid.limits[:, 1], (6, d))
    if project:
        x[:, 0] = grid.limits[0, 1] + 0.3                   # outside in one coordinate: projected
    good = _library_values(lk, otri, x, vals)
    R.check_values(lk, x, good, vals)
    for i, p in enumerate(x):
        corner, sims = lk.lookup_set(p)
        s = sims[0]
        # the neighbouring cell's corner in one axis
        k = np.array(np.unravel_index(corner, grid.num_points))
        k[0] += 1 if k[0] + 1 <= grid.num_points[0] - 2 else -1
        wrong_corner = int(np.ravel_multi_index(k, grid.num_points))
        # a simplex outside the admissible set, whose plane differs at the point
        others = [t for t in range(lk.S) if t not in sims
                  and np.max(np.abs(lk.exact(p, corner, t, vals)["value"] - good[i])) > 1e-6]
        wrongs = [lk.exact(p, wrong_corner, s, vals)["value"], lk.exact(p, corner, others[0], vals)["value"]]
        if project:                                         # project ignored
            plain = R.Lookup(grid, lk.simp, lk.H, lk.corner_table, False)
            wrongs.append(plain.exact(p, corner, s, vals)["value"])
        for wrong in wrongs:
            bad = good.copy()
            bad[i] = wrong
            with pytest.raises(AssertionError):
                R.check_values(lk, x, bad, vals)


@pytest.mark.parametrize("d", [2, 4, 6])
def test_gradient_check_rejects_the_wrong_simplex(d):
    grid = R.shape_grid(O, d)
    rng = np.random.default_rng(10 + d)
    vals = rng.normal(size=(grid.nindex, 1))
    lk = _lookup(grid, False)
    x = rng.uniform(grid.limits[:, 0], grid.limits[:, 1], (4, d))
    good = np.array([lk.candidates(p, vals)[0]["gradient"] for p in x])
    R.check_gradients(lk, x, good, vals)
    R.check_gradients(lk, x, np.max(np.abs(good), axis=1, keepdims=True), vals, maxabs=True)
    for i, p in enumerate(x):
        corner, sims = lk.lookup_set(p)
        t = next(t for t in range(lk.S) if t not in sims and np.max(np.abs(
            lk.exact(p, corner, t, vals)["gradient"] - good[i])) > 1e-6)
        bad = good.copy()
        bad[i] = lk.exact(p, corner, t, vals)["gradient"]
        with pytest.raises(AssertionError):
            R.check_gradients(lk, x, bad, vals)


@pytest.mark.parametrize("d", [1, 3, 6])
def test_affine_check_rejects_wrong_results(d):
    grid = R.shape_grid(O, d)
    rng = np.random.default_rng(20 + d)
    a = rng.normal(size=(d, 1))
    b = rng.normal(size=1)
    vals = grid.all_points @ a + b
    for project in (False, True):
        otri = O.Triangulation(grid, vals, project=project)
        lk = R.Lookup.of(otri)
        x = rng.uniform(grid.limits[:, 0] - 0.5, grid.limits[:, 1] + 0.5, (5, d))
        x[0] = grid.limits[:, 1] + 0.25                       # outside in every coordinate
        good = _library_values(lk, otri, x, vals)
        grad = np.tile(a[:, 0], (len(x), 1))
        R.check_affine(lk, x, good, grad, a, b, vals)
        with pytest.raises(AssertionError):                   # project ignored / applied wrongly
            R.check_affine(lk, x, x @ a + b if project else np.clip(x, grid.limits[:, 0], grid.limits[:, 1]) @ a + b,
                           grad, a, b, vals)
        bad = grad.copy()
        bad[1, 0] *= 1 + 1e-9
        with pytest.raises(AssertionError):
            R.check_affine(lk, x, good, bad, a, b, vals)


@pytest.mark.parametrize("d,project", [(2, True), (4, False), (6, True)])
def test_row_check_rejects_wrong_rows(d, project):
    grid = R.shape_grid(O, d)
    rng = np.random.default_rng(30 + d)
    x = R.operator_points(grid, rng)[:60]
    otri = O.Triangulation(grid, np.zeros(grid.nindex), project=project)
    cols, w, _ = V.operator(otri, x, lookup="library")
    lk = R.Lookup.of(otri)
    R.check_rows(lk, x, cols, w)
    i = int(np.argmax(np.abs(w[:, 1] - w[:, 2])))            # two vertex columns swapped in a row
    bad = cols.copy()
    bad[i, [1, 2]] = bad[i, [2, 1]]
    with pytest.raises(AssertionError):
        R.check_rows(lk, x, bad, w)
    bad = w.copy()                                           # the weights of the neighbouring row's point
    bad[i] = V._barycentric(otri, x[i] + 1e-7, lk.cell(x[i])[0], lk.lookup_set(x[i])[1][0])
    with pytest.raises(AssertionError):
        R.check_rows(lk, x, cols, bad)


def test_fixed_point_check_rejects_twice_the_bound():
    grid = R.shape_grid(O, 3)
    rng = np.random.default_rng(4)
    otri = O.Triangulation(grid, np.zeros(grid.nindex), project=True)
    nxt = 0.9 * grid.all_points[:, ::-1] + 0.2
    cols, w, _ = V.operator(otri, nxt, lookup="library")
    rewards = -np.sum(grid.all_points ** 2, axis=1) + rng.normal(size=grid.nindex)
    v, _, delta, bound = V.solve(cols, w, rewards, 0.9, np.zeros(grid.nindex))
    slack = R.solve_slack(w, rewards, 0.9, v, 3, bound)
    vstar, err = R.fixed_point(cols, w, rewards, 0.9, 1e-3 * (bound + slack))
    R.check_fixed_point(v, vstar, err, bound, slack)
    bad = v.copy()
    bad[rng.integers(grid.nindex)] += 2 * (bound + slack)
    with pytest.raises(AssertionError):
        R.check_fixed_point(bad, vstar, err, bound, slack)
    with pytest.raises(AssertionError):                      # a certificate that is too small
        R.check_fixed_point(v, vstar, err, 0.25 * bound, R.solve_slack(w, rewards, 0.9, v, 3, 0.25 * bound))
