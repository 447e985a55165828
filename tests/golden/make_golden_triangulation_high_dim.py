"""Generate ``tests/golden/triangulation_high_dim.npz`` by running the UNMODIFIED reference's
``Triangulation`` (evaluation ``functions.py:1473-1499``, gradient ``:1502-1510``) and
``_Triangulation.parameter_derivative`` (``:1228-1259``) on the numpy-backed TF1 shim.

    SAFE_LEARNING_REFERENCE=<checkout> python tests/golden/make_golden_triangulation_high_dim.py

Grids with d = 4, 5, 6 on ``[-1 - 0.1 c, 1 + 0.2 c]`` (the grids of ``test_gpu_triangulation_grad.GRIDS``).
Per grid the point groups ``inside``, ``faces`` (one coordinate on an interior grid line), ``vertices``
(every vertex), ``outside`` and ``corners`` (one point beyond every combination of lower and upper
faces: all 2^d corner patterns).  Each query is made alone: scipy's find_simplex walks from the
previous query's simplex within one call.  Stored per grid: limits, num_points, unit_simplices,
hyperplanes, a two-column table ``vals`` and a one-column table ``gvals``; per grid and group the
points; per grid, ``project`` and group the values of ``vals`` and the rows (vertex columns and
weights of ``parameter_derivative``); per grid and group the gradient of ``gvals`` (the reference's
gradient does not project).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from reference_loader import load_reference  # noqa: E402

sl = load_reference()
import tensorflow as tf  # noqa: E402  (shim)

NUM = {4: [3, 4, 3, 3], 5: [3] * 5, 6: [3, 2, 3, 2, 3, 2]}


def point_groups(grid, rng):
    d = grid.ndim
    lo, hi = grid.limits[:, 0], grid.limits[:, 1]
    span = hi - lo
    inside = rng.uniform(lo, hi, (40, d))
    faces = rng.uniform(lo, hi, (40, d))
    for i in range(len(faces)):
        c = i % d
        pts = grid.discrete_points[c]
        faces[i, c] = pts[1 + i % (len(pts) - 2)] if len(pts) > 2 else pts[0]
    outside = rng.uniform(lo - 0.4 * span, hi + 0.4 * span, (40, d))
    bits = (np.arange(2 ** d)[:, None] >> np.arange(d)[None, :]) & 1
    corners = np.where(bits == 1, hi + rng.uniform(0.05, 0.5, (2 ** d, d)) * span,
                       lo - rng.uniform(0.05, 0.5, (2 ** d, d)) * span)
    return {"inside": inside, "faces": faces, "vertices": grid.all_points.copy(), "outside": outside,
            "corners": corners}


def main(out):
    rng = np.random.default_rng(29)
    res = {}
    with tf.Session():
        for d, num in NUM.items():
            tag = "h%d" % d
            grid = sl.GridWorld([[-1.0 - 0.1 * c, 1.0 + 0.2 * c] for c in range(d)], num)
            groups = point_groups(grid, rng)
            vals = rng.normal(size=(grid.nindex, 2))
            gvals = rng.normal(size=(grid.nindex, 1))
            res[tag + "_limits"], res[tag + "_num"] = grid.limits, grid.num_points
            res[tag + "_vals"], res[tag + "_gvals"] = vals, gvals
            for group, pts in groups.items():
                res["%s_%s" % (tag, group)] = pts
            gtri = sl.Triangulation(grid, gvals, name="tri_hd_grad_%d" % d)
            for group, pts in groups.items():
                res["%s_%s_gradient" % (tag, group)] = np.vstack(
                    [gtri.gradient(p[None, :]).eval() for p in pts])
            for project in (False, True):
                tri = sl.Triangulation(grid, vals, project=project, name="tri_hd_%d_%d" % (d, project))
                for group, pts in groups.items():
                    key = "%s_%s_%s" % (tag, "proj" if project else "noproj", group)
                    res[key + "_value"] = np.vstack([tri(p[None, :]).eval() for p in pts])
                    cols, data = [], []
                    for p in pts:
                        m = tri.tri.parameter_derivative(p[None, :])
                        assert np.array_equal(m.row, np.zeros(d + 1))
                        cols.append(m.col)
                        data.append(m.data)
                    res[key + "_cols"] = np.stack(cols).astype(np.int64)
                    res[key + "_weights"] = np.stack(data)
            res[tag + "_unit_simplices"] = tri.tri.unit_simplices
            res[tag + "_hyperplanes"] = tri.tri.hyperplanes
            print("d = %d: %d unit simplices" % (d, len(tri.tri.unit_simplices)), flush=True)
    np.savez_compressed(os.path.join(out, "triangulation_high_dim.npz"), **res)
    print("triangulation high-dimension fixtures written:", len(res), "arrays")


if __name__ == "__main__":
    main(HERE)
