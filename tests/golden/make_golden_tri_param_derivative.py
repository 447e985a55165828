"""Generate ``tests/golden/triangulation_param_derivative.npz`` by running the UNMODIFIED reference's
``_Triangulation.parameter_derivative`` (``functions.py:1228-1259``) on the numpy-backed TF1 shim.

    SAFE_LEARNING_REFERENCE=<checkout> python tests/golden/make_golden_tri_param_derivative.py

Grids with d = 1, 2, 3, each with and without projection; per grid the groups ``inside``, ``faces``
(one coordinate on an interior grid line), ``outside`` and ``vertices`` (exact vertex queries, whose
simplex is order dependent upstream, DESIGN.md §3.2 Q6, so they are a group of their own), and the
seven points of ``tests/test_functions.py:674-680`` (``test_gradient_param``) on its 3 x 3 grid.  Each
query is made alone: scipy's find_simplex walks from the previous query's simplex.  Stored per case:
the points, the vertex columns [n, d + 1] and the weights [n, d + 1] of the reference's rows.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from reference_loader import load_reference  # noqa: E402

sl = load_reference()

GRIDS = (("g1", [[-1.0, 1.5]], [6]), ("g2", [[-1.0, 1.5], [0.0, 2.0]], [5, 4]),
         ("g3", [[-1, 1], [0, 2], [-0.5, 0.5]], [4, 3, 5]), ("tp", [[0, 1], [0, 1]], [3, 3]))


def point_groups(grid, tag, rng):
    if tag == "tp":
        return {"points": np.array([[-10, -10], [0.2, 0.7], [0, 0], [0, 1], [1, 1], [-0.2, 0.5],
                                    [0.43, 0.21]], dtype=np.float64)}
    lo, hi = grid.limits[:, 0], grid.limits[:, 1]
    inside = rng.uniform(lo, hi, (60, grid.ndim))
    faces = rng.uniform(lo, hi, (60, grid.ndim))
    for i in range(len(faces)):
        c = i % grid.ndim
        pts = grid.discrete_points[c]
        faces[i, c] = pts[1 + i % (len(pts) - 2)] if len(pts) > 2 else pts[0]
    return {"inside": inside, "faces": faces,
            "outside": rng.uniform(lo - 0.4 * (hi - lo), hi + 0.4 * (hi - lo), (60, grid.ndim)),
            "vertices": grid.all_points.copy()}


def main(out):
    rng = np.random.default_rng(23)
    res = {}
    for tag, limits, num in GRIDS:
        grid = sl.GridWorld(limits, num)
        groups = point_groups(grid, tag, rng)
        res[tag + "_limits"], res[tag + "_num"] = grid.limits, grid.num_points
        for project in (False, True):
            trinp = sl.functions._Triangulation(grid, np.zeros((grid.nindex, 1)), project=project)
            for group, pts in groups.items():
                key = "%s_%s_%s" % (tag, "proj" if project else "noproj", group)
                cols, data = [], []
                for p in pts:
                    m = trinp.parameter_derivative(p[None, :])
                    assert np.array_equal(m.row, np.zeros(grid.ndim + 1))
                    cols.append(m.col)
                    data.append(m.data)
                res[key + "_points"] = pts
                res[key + "_cols"] = np.stack(cols).astype(np.int64)
                res[key + "_weights"] = np.stack(data)
    np.savez_compressed(os.path.join(out, "triangulation_param_derivative.npz"), **res)
    print("triangulation parameter_derivative fixtures written:", len(res), "arrays")


if __name__ == "__main__":
    main(HERE)
