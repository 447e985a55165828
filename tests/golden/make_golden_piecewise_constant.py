"""Generate ``tests/golden/piecewise_constant.npz`` by running the UNMODIFIED reference's
``PiecewiseConstant`` (``functions.py:820-932``) and ``GridWorld.state_to_index`` (``:733-752``) on the
numpy-backed TF1 shim.

    SAFE_LEARNING_REFERENCE=<checkout> python tests/golden/make_golden_piecewise_constant.py

Grids with d = 1, 2, 3 (power-of-two spacings, so that half-cell points are exact ties of ``np.rint``)
and one 2-D grid with the mountain-car limits (inexact spacings), each with a one- and a two-column
table.  Per grid the groups ``inside`` (random interior points), ``vertices`` (every vertex), ``ties``
(every coordinate half a cell from a vertex), ``outside`` (beyond the limits) and ``inf`` (a +-inf
coordinate), each stored with the reference's evaluation, ``state_to_index``, ``parameter_derivative``
(rows, columns, data) and ``gradient``.  Then the three reference tests (``tests/test_functions.py:
408-451``): their parameters, evaluations and ``parameter_derivative`` products.  NaN is not in the
fixture: the reference raises from ``ravel_multi_index`` (DESIGN.md §3.15).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from reference_loader import load_reference  # noqa: E402

sl = load_reference()

GRIDS = (("g1", [[-1.0, 1.0]], [9]),
         ("g2", [[-1.0, 1.0], [0.0, 4.0]], [5, 9]),
         ("g2m", [[-1.2, 0.6], [-0.07, 0.07]], [20, 20]),
         ("g3", [[-1.0, 1.0], [0.0, 2.0], [-0.5, 0.5]], [5, 3, 9]))


def point_groups(grid, rng):
    lo, hi = grid.limits[:, 0], grid.limits[:, 1]
    d = grid.ndim
    ties = grid.all_points + 0.5 * grid.unit_maxes
    ties = ties[np.all(ties <= hi, axis=1)]
    ties = np.concatenate([ties, grid.all_points - 0.5 * grid.unit_maxes])
    inf = rng.uniform(lo, hi, (4 * d, d))
    for i in range(len(inf)):
        inf[i, i % d] = np.inf if i % 2 == 0 else -np.inf
    return {"inside": rng.uniform(lo, hi, (200, d)),
            "vertices": grid.all_points.copy(),
            "ties": ties,
            "outside": rng.uniform(lo - 0.5 * (hi - lo), hi + 0.5 * (hi - lo), (100, d)),
            "inf": inf}


def reference_tests():
    """The three tests of tests/test_functions.py:408-451, their quantities."""
    out = {}
    disc = sl.GridWorld([[-1, 1], [-1, 1]], 4)
    pwc = sl.PiecewiseConstant(disc, np.arange(16))
    out["t_init_parameters"] = np.asarray(pwc.parameters, dtype=np.float64)
    disc = sl.GridWorld([[-1, 1], [-1, 1]], 3)
    pwc = sl.PiecewiseConstant(disc)
    vertex_points = pwc.discretization.index_to_state(np.arange(pwc.nindex))
    vertex_values = np.sum(vertex_points, axis=1, keepdims=True)
    pwc.parameters = vertex_values
    out["t_eval_points"] = vertex_points
    out["t_eval_values"] = vertex_values
    out["t_eval_result"] = np.asarray(pwc.build_evaluation(vertex_points))
    out["t_eval_outside"] = np.asarray(pwc.build_evaluation(np.array([[-1.5, -1.5]])))
    out["t_eval_constraint"] = pwc.parameter_derivative(vertex_points).toarray().dot(vertex_values)
    out["t_gradient"] = np.asarray(pwc.gradient(vertex_points), dtype=np.float64)
    return out


def main(out):
    rng = np.random.default_rng(31)
    res = {}
    for tag, limits, num in GRIDS:
        grid = sl.GridWorld(limits, num)
        res[tag + "_limits"], res[tag + "_num"] = grid.limits, grid.num_points
        groups = point_groups(grid, rng)
        for ncol in (1, 2):
            values = rng.standard_normal((grid.nindex, ncol))
            pwc = sl.PiecewiseConstant(grid, values)
            key = "%s_c%d" % (tag, ncol)
            res[key + "_table"] = values
            for group, pts in groups.items():
                k = "%s_%s" % (key, group)
                res[k + "_points"] = pts
                res[k + "_values"] = np.asarray(pwc.build_evaluation(pts))
                if ncol == 1:
                    res[k + "_index"] = grid.state_to_index(pts).astype(np.int64)
                    m = pwc.parameter_derivative(pts)
                    res[k + "_pd_row"] = m.row.astype(np.int64)
                    res[k + "_pd_col"] = m.col.astype(np.int64)
                    res[k + "_pd_data"] = m.data
                    res[k + "_gradient"] = np.asarray(pwc.gradient(pts))
    res.update(reference_tests())
    np.savez_compressed(os.path.join(out, "piecewise_constant.npz"), **res)
    print("PiecewiseConstant fixtures written:", len(res), "arrays")


if __name__ == "__main__":
    main(HERE)
