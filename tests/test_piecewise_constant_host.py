"""Host tests of ``PiecewiseConstant`` (``SLB_FN_PIECEWISE_CONSTANT``): the numpy restatement against the
reference-generated fixture and the reference's own test vectors, the descriptor the Python object writes,
the library's host checks of the new kind, and tabular dynamic programming in the numpy oracle."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import piecewise_constant_oracle as P  # noqa: E402
import safe_learning_b200 as sl  # noqa: E402
from safe_learning_b200 import _native as nat  # noqa: E402

GOLDEN = np.load(os.path.join(HERE, "golden", "piecewise_constant.npz"))
GRIDS = ("g1", "g2", "g2m", "g3")
GROUPS = ("inside", "vertices", "ties", "outside", "inf")


def _grid(tag):
    return GOLDEN[tag + "_limits"], GOLDEN[tag + "_num"]


# ---------------------------------------------------------------- the restatement against the reference
@pytest.mark.parametrize("tag", GRIDS)
@pytest.mark.parametrize("ncol", [1, 2])
@pytest.mark.parametrize("group", GROUPS)
def test_oracle_matches_reference(tag, ncol, group):
    limits, num = _grid(tag)
    key = "%s_c%d" % (tag, ncol)
    pts = GOLDEN["%s_%s_points" % (key, group)]
    got = P.evaluate(limits, num, GOLDEN[key + "_table"], pts)
    assert np.array_equal(got, GOLDEN["%s_%s_values" % (key, group)])
    if ncol == 1:
        k = "%s_%s" % (key, group)
        idx = P.nearest_index(limits, num, pts)
        assert np.array_equal(idx, GOLDEN[k + "_index"])
        assert np.array_equal(GOLDEN[k + "_pd_row"], np.arange(len(pts)))
        assert np.array_equal(GOLDEN[k + "_pd_col"], idx)
        assert np.all(GOLDEN[k + "_pd_data"] == 1)
        assert np.array_equal(GOLDEN[k + "_gradient"], np.zeros((len(pts), len(num))))


def test_fixture_has_exact_half_cell_ties():
    """The tie group sits exactly half a cell from a vertex, and rint rounds those to even."""
    limits, num = _grid("g2")
    unit = (limits[:, 1] - limits[:, 0]) / (num - 1)
    pts = GOLDEN["g2_c1_ties_points"]
    frac = (np.clip(pts, limits[:, 0], limits[:, 1]) - limits[:, 0]) / unit
    half = np.abs(frac - np.floor(frac) - 0.5) == 0
    assert half.any()
    ijk = np.stack(np.unravel_index(GOLDEN["g2_c1_ties_index"], num), axis=1)
    assert np.all(ijk[half] % 2 == 0)
    assert np.isinf(GOLDEN["g3_c2_inf_points"]).any()


def test_nan_rows_are_nan_in_every_column():
    limits, num = _grid("g2")
    pts = np.array([[np.nan, 1.0], [0.2, np.nan], [0.2, 1.0]])
    out = P.evaluate(limits, num, GOLDEN["g2_c2_table"], pts)
    assert np.isnan(out[:2]).all() and np.isfinite(out[2]).all()
    assert list(P.nearest_index(limits, num, pts)[:2]) == [-1, -1]


def test_reference_test_vectors():
    """tests/test_functions.py:408-451 on the restatement."""
    g = GOLDEN
    assert np.array_equal(g["t_init_parameters"], np.arange(16, dtype=np.float64)[:, None])
    limits, num = [[-1, 1], [-1, 1]], [3, 3]
    assert np.array_equal(P.evaluate(limits, num, g["t_eval_values"], g["t_eval_points"]), g["t_eval_result"])
    np.testing.assert_allclose(g["t_eval_result"], g["t_eval_values"])
    assert np.array_equal(P.evaluate(limits, num, g["t_eval_values"], [[-1.5, -1.5]]), g["t_eval_outside"])
    np.testing.assert_allclose(g["t_eval_outside"], [[-2]])
    np.testing.assert_allclose(g["t_eval_constraint"], g["t_eval_values"])
    np.testing.assert_allclose(g["t_gradient"], 0)


# ---------------------------------------------------------------- the Python object without a device
def test_surface_without_values():
    grid = sl.GridWorld([[-1, 1], [-1, 1]], 3)
    pwc = sl.PiecewiseConstant(grid)
    assert pwc.parameters is None and pwc.output_dim is None
    assert pwc.input_dim == 2 and pwc.nindex == 9 and pwc.discretization is grid
    assert np.array_equal(pwc.limits, grid.limits)
    grad = pwc.gradient(np.zeros((4, 2)))
    assert grad.shape == (4, 2) and not grad.any()
    with pytest.raises(ValueError):
        pwc.descriptor()
    gf = pwc.gradient_function()
    assert isinstance(gf, sl.ConstantFunction) and gf.input_dim == gf.output_dim == 2
    assert not gf.constant.any()
    assert "PiecewiseConstant" in sl.__dict__


@pytest.fixture
def host_tables(monkeypatch):
    """Vertex tables in host memory: the descriptor only records their address."""
    from safe_learning_b200 import functions
    monkeypatch.setattr(functions.dev, "to_device",
                        lambda a, dtype=torch.float64: torch.as_tensor(np.asarray(a), dtype=dtype).contiguous())


@pytest.mark.parametrize("tag", GRIDS)
def test_descriptor_fields(tag, host_tables):
    limits, num = _grid(tag)
    grid = sl.GridWorld(limits, num)
    pwc = sl.PiecewiseConstant(grid, np.arange(grid.nindex * 2.0))
    assert pwc.parameters.shape == (grid.nindex, 2) and pwc.output_dim == 2
    d = pwc.descriptor()
    assert (d.kind, d.in_dim, d.out_dim, d.flags) == (nat.FN_PIECEWISE_CONSTANT, grid.ndim, 2, 0)
    assert d.matrix == pwc._param_dev.data_ptr()
    inv = np.array([d.cparams[c] for c in range(grid.ndim)])
    assert np.array_equal(inv.view(np.uint64), (1. / grid.unit_maxes).view(np.uint64))
    assert d.grid.ndim == grid.ndim and d.grid.nindex == grid.nindex
    assert [d.grid.num_points[c] for c in range(grid.ndim)] == list(grid.num_points)
    v0 = pwc.version
    pwc.parameters = np.zeros(grid.nindex)
    assert pwc.version != v0 and pwc.output_dim == 1


# ---------------------------------------------------------------- the C ABI's host checks
def _function(d=2, out=1):
    f = nat.SlbFunction()
    f.kind, f.in_dim, f.out_dim = nat.FN_PIECEWISE_CONSTANT, d, out
    f.matrix = 0x1000
    f.grid.ndim, f.grid.nindex = d, 5 ** d
    for c in range(d):
        f.grid.num_points[c], f.grid.unit_maxes[c], f.grid.offset[c], f.grid.upper[c] = 5, 0.5, -1.0, 1.0
        f.cparams[c] = 2.0
    return f


def _eval_rc(f, n=4):
    lib = nat.load()
    return lib.slb_eval_function(None, f, C.c_void_p(0x2000), n, C.c_void_p(0x3000))


def test_columns_follow_the_post_ops():
    lib = nat.load()
    f = _function(out=3)
    assert lib.slb_function_columns(f) == 3
    f.flags = nat.FLAG_NORM1
    assert lib.slb_function_columns(f) == 1
    f.flags = nat.FLAG_MAXABS
    assert lib.slb_function_columns(f) == 1


@pytest.mark.parametrize("case, message", [
    ("in_dim", "in_dim 3 != grid ndim 2"),
    ("null table", "without vertex values"),
    ("out_dim", "out_dim 7"),
    ("gradient", "gradient flag"),
    ("project", "no projection flag"),
    ("inv", "cparams[1]"),
    ("grid", "grid nindex"),
])
def test_validation(case, message):
    f = _function()
    if case == "in_dim":
        f.in_dim = 3
    elif case == "null table":
        f.matrix = None
    elif case == "out_dim":
        f.out_dim = 7
    elif case == "gradient":
        f.flags = nat.FLAG_GRADIENT
    elif case == "project":
        f.flags = nat.FLAG_PROJECT
    elif case == "inv":
        f.cparams[1] = float("inf")
    elif case == "grid":
        f.grid.nindex = 24
    assert _eval_rc(f) == 1
    assert message in nat.last_error(), nat.last_error()


def test_vjp_host_checks():
    lib = nat.load()
    f = _function()
    rc = lib.slb_function_vjp(None, f, C.c_void_p(0x2000), 4, C.c_void_p(0x3000), C.c_void_p(0x4000),
                              None, None, None)
    assert rc == 1 and "point gradient is 0" in nat.last_error()
    f.flags = nat.FLAG_SATURATE
    assert lib.slb_function_vjp_workspace(f, 4) == -1
    assert "post-op flags" in nat.last_error()


def test_nearest_index_host_checks():
    lib = nat.load()
    g = _function().grid
    assert lib.slb_grid_nearest_index(None, g, C.c_void_p(0x2000), -1, C.c_void_p(0x3000)) == 1
    assert "negative n" in nat.last_error()
    assert lib.slb_grid_nearest_index(None, g, None, 0, None) == 0        # n = 0: nothing to do
    g.unit_maxes[0] = 0.0
    assert lib.slb_grid_nearest_index(None, g, C.c_void_p(0x2000), 1, C.c_void_p(0x3000)) == 1
    assert "unit_maxes[0]" in nat.last_error()


def test_value_operator_points_rejects_a_table_with_post_ops():
    lib = nat.load()
    for flags, out in ((nat.FLAG_SCALE, 1), (0, 2)):
        f = _function(out=out)
        f.flags = flags
        rc = lib.slb_value_operator_points(None, f, C.c_void_p(0x2000), 4, C.c_void_p(0x3000),
                                           C.c_void_p(0x4000), C.c_void_p(0x5000))
        assert rc == 1 and "plain one-output Triangulation or PiecewiseConstant" in nat.last_error()


# ---------------------------------------------------------------- tabular DP in the numpy oracle
def _chain(n=41, gamma=0.9):
    """A 1-D chain: action a in {-1, 0, 1} moves a cell; reward -|x|."""
    limits, num = [[-1.0, 1.0]], [n]
    x = np.linspace(-1, 1, n)[:, None]
    unit = 2.0 / (n - 1)
    actions = np.array([-1.0, 0.0, 1.0])
    nxt = [x + a * unit for a in actions]
    rew = [-np.abs(x[:, 0]) for _ in actions]
    return limits, num, x, actions, nxt, rew, gamma


def test_oracle_value_iteration_reaches_the_policy_evaluation():
    limits, num, x, actions, nxt, rew, gamma = _chain()
    v = np.zeros(len(x))
    for _ in range(400):
        best, q = P.greedy(limits, num, v, nxt, rew, gamma)
        v_new = q[best, np.arange(len(x))]
        if np.max(np.abs(v_new - v)) < 1e-13:
            break
        v = v_new
    best, _ = P.greedy(limits, num, v, nxt, rew, gamma)
    # greedy moves towards the origin, and stays there
    assert np.all(actions[best][x[:, 0] < -1e-9] == 1) and np.all(actions[best][x[:, 0] > 1e-9] == -1)
    chosen = np.stack([nxt[b][i] for i, b in enumerate(best)])
    exact = P.evaluate_policy(limits, num, chosen, rew[0], gamma)
    np.testing.assert_allclose(v, exact, rtol=0, atol=1e-11)
    sweep = P.bellman_sweep(limits, num, exact, chosen, rew[0], gamma)
    np.testing.assert_allclose(sweep, exact, rtol=0, atol=1e-12)


def test_oracle_argmax_takes_the_first_maximum_and_nan():
    limits, num = [[0.0, 1.0]], [3]
    nxt = [np.array([[0.0], [0.5], [1.0]])] * 3
    rew = [np.zeros(3), np.array([0.0, np.nan, 0.0]), np.zeros(3)]
    best, _ = P.greedy(limits, num, np.zeros(3), nxt, rew, 0.5)
    assert list(best) == [0, 1, 0]
