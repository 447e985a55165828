"""Generate ``tests/golden/lyapunov_adaptive.npz`` by running the UNMODIFIED reference's adaptive branch
of ``Lyapunov.update_safe_set`` (``lyapunov.py:445-487, 497-606``) on the numpy-backed TF1 shim.

    SAFE_LEARNING_REFERENCE=<checkout> python tests/golden/make_golden_adaptive.py

The branch needs ``tf.map_fn``, ``tf.linspace`` and ``tf.meshgrid``, which this script adds to the shim.
Its refined check compares the outer ``decrease`` tensor of every fed state (``:474-478``), so the fixture
pins the as-written reading, ``refinement_mode="reference"``.

Cases: the GP pendulum of ``bench_workloads.make_pendulum`` and the same pendulum with the deterministic
linear plant ``LinearSystem((A_true, B_true))``, each at three tau, (max_refinement, safety_factor) in
{(4, 1), (16, 2)} and batch sizes 64 and 37.  Per case: ``update_safe_set(True, R, s)``; then
``add_data_point`` (GP) or a seeded earlier safe set and refinement (deterministic plant); then
``update_safe_set(False, R, s)`` twice.  The reference builds its graph, tau and the safety factor
included, on the first call, so every case gets a fresh ``Lyapunov``.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden  # noqa: E402  (loads the reference on the shim)

sl, tf, W = make_golden.sl, make_golden.tf, make_golden.W


# The adaptive branch's `refined_safety_check` (lyapunov.py:457-481) needs three ops the shim lacks.
def _linspace(start, stop, num, name=None):
    """TF's LinSpace kernel: ``start + i (stop - start) / (num - 1)``, ``[start]`` for num = 1."""
    def run(f, c):
        a, b, n = float(tf._val(start, f, c)), float(tf._val(stop, f, c)), int(tf._val(num, f, c))
        if n == 1:
            return np.array([a])
        return a + np.arange(n) * ((b - a) / (n - 1))
    return tf.Tensor(run, name)


def _meshgrid(*args, **kwargs):
    indexing = kwargs.get("indexing", "xy")
    return [tf.Tensor(lambda f, c, i=i: np.meshgrid(*[tf._val(a, f, c) for a in args], indexing=indexing)[i])
            for i in range(len(args))]


def _map_fn(fn, elems, dtype=None, parallel_iterations=10, back_prop=True, swap_memory=False,
            infer_shape=True, name=None):
    """``fn`` on each row of ``elems``, stacked.  Each row builds its own graph from a constant and is
    evaluated with a copy of the cache: the cache is keyed on ``id()``, and the ids of a previous row's
    tensors come back once they are garbage-collected."""
    def run(f, c):
        rows = tf._val(elems, f, c)
        out = [np.asarray(tf._val(fn(tf.constant(row)), f, dict(c))) for row in rows]
        return np.array(out, dtype=tf._np_dtype(dtype) if dtype is not None else None)
    return tf.Tensor(run, name)


for _name, _op in (("linspace", _linspace), ("meshgrid", _meshgrid), ("map_fn", _map_fn)):
    if not hasattr(tf, _name):
        setattr(tf, _name, _op)


TAUS = (0.03, 0.01, 0.004)
REFINE = ((4, 1.0), (16, 2.0))
BATCHES = (64, 37)
XNEW = np.array([[0.3, -0.2, 0.1]])     # the reference stack adds one point per call


def case_params():
    par = W.make_pendulum(num_points=[31, 27], M=60, tau_scale=1.0)
    ynew = W._pendulum_step(XNEW, state_norm=par["plant"]["state_norm"],
                            action_norm=par["plant"]["action_norm"], **par["plant"]["true"])
    return par, ynew


def ref_lyapunov(par, plant):
    grid = sl.GridWorld(par["limits"], par["num_points"])
    if plant == "gp":
        dynamics = make_golden.ref_gp_stack(par)
    else:
        dynamics = sl.LinearSystem((par["A_true"], par["B_true"]), name="true_dynamics")
    policy = sl.Saturation(sl.LinearSystem((-par["K"],), name="policy"), -1., 1.)
    grad = sl.LinearSystem((2 * par["P"],), name="grad_v")
    l_v = lambda x: tf.abs(grad(x))  # noqa: E731  (notebook cell 17)
    return sl.Lyapunov(grid, sl.QuadraticFunction(par["P"]), dynamics, par["L_dyn"], l_v,
                       par["tau"], policy, par["initial"].copy(), adaptive=True)


def seeded_previous(safe_set, max_refinement, seed):
    """An earlier safe set: the current one plus seeded extra states, with refinement in [1, R]."""
    rng = np.random.default_rng(seed)
    safe = safe_set | (rng.random(safe_set.size) < 0.15)
    refinement = np.where(safe, rng.integers(1, max_refinement + 1, safe.size), 0)
    return safe, refinement


def record(res, key, lyap):
    res[key + "_safe_set"] = lyap.safe_set.copy()
    res[key + "_refinement"] = np.asarray(lyap._refinement).copy()
    res[key + "_c_max"] = np.array(lyap.feed_dict[lyap.c_max], dtype=np.float64)


def main():
    par, ynew = case_params()
    res = make_golden.flat_par(par)
    res["xnew"], res["ynew"] = XNEW, ynew
    res["taus"], res["refine"], res["batches"] = np.array(TAUS), np.array(REFINE), np.array(BATCHES)
    for plant in ("gp", "linear"):
        for ti, tau in enumerate(TAUS):
            for ri, (R, s) in enumerate(REFINE):
                for batch in BATCHES:
                    key = "%s_t%d_r%d_b%d" % (plant, ti, ri, batch)
                    with tf.Session():
                        sl.config.gp_batch_size = batch
                        lyap = ref_lyapunov(dict(par, tau=tau), plant)
                        res["values"] = lyap.values.copy()
                        lyap.update_safe_set(True, R, s)
                        record(res, key + "_1", lyap)
                        if plant == "gp":
                            lyap.dynamics.add_data_point(XNEW, ynew)
                        else:
                            safe, refinement = seeded_previous(lyap.safe_set, R, 100 * ti + 10 * ri + batch)
                            res[key + "_prev_safe_set"], res[key + "_prev_refinement"] = safe, refinement
                            lyap.safe_set = safe.copy()
                            lyap._refinement = refinement.copy()
                        lyap.update_safe_set(False, R, s)
                        record(res, key + "_2", lyap)
                        lyap.update_safe_set(False, R, s)
                        record(res, key + "_3", lyap)
                    print(key, [int(res[key + "_%d_safe_set" % k].sum()) for k in (1, 2, 3)],
                          "refined", int((res[key + "_3_refinement"] > 1).sum()))
    sl.config.gp_batch_size = 10000
    np.savez_compressed(os.path.join(HERE, "lyapunov_adaptive.npz"), **res)


if __name__ == "__main__":
    main()
