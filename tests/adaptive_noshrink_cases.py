"""Shared builders of the adaptive ``update_safe_set(can_shrink=False)`` tests: the pendulum of
``bench_workloads.make_pendulum`` with GP dynamics or the deterministic linear plant, as the oracle
(``oracle``) or the product (``safe_learning_b200``) builds it, and the replay of the reference-generated
``tests/golden/lyapunov_adaptive.npz`` (``tests/golden/make_golden_adaptive.py``)."""
import os

import numpy as np
from numpy.testing import assert_array_equal

import bench_workloads as W

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def build(ns, par, plant, kind, lipschitz_lyapunov=None):
    """Adaptive ``Lyapunov`` on ``par``: ``plant`` "gp" (the stacked GPs) or "linear"
    (``LinearSystem((A_true, B_true))``); L_V = |2 P x| unless given."""
    grid, dynamics = W._build(ns, par, kind)
    if plant == "linear":
        dynamics = ns.LinearSystem((par["A_true"], par["B_true"]))
    policy = ns.Saturation(ns.LinearSystem(-par["K"]), -1., 1.)
    l_v = lipschitz_lyapunov or ns.AbsFunction(ns.LinearSystem((2 * par["P"],)))
    return ns.Lyapunov(grid, ns.QuadraticFunction(par["P"]), dynamics, par["L_dyn"], l_v, par["tau"],
                       policy, initial_set=par["initial"], adaptive=True)


def load_fixture():
    fix = np.load(os.path.join(GOLDEN, "lyapunov_adaptive.npz"))
    par = {k[4:]: fix[k] for k in fix.files if k.startswith("par_")}
    for k in ("tau", "beta", "scale", "noise_variance", "L_dyn"):
        par[k] = float(par[k])
    par["variances"] = [float(v) for v in par["variances"]]
    par["lengthscales"] = [list(map(float, ls)) for ls in par["lengthscales"]]
    par["num_points"] = par["num_points"].astype(int)
    par["kernel_specs"] = None
    return fix, par


def fixture_cases(fix):
    """(key, plant, tau, max_refinement, safety_factor, batch) of every recorded sequence."""
    out = []
    for plant in ("gp", "linear"):
        for ti, tau in enumerate(fix["taus"]):
            for ri, (R, s) in enumerate(fix["refine"]):
                for batch in fix["batches"]:
                    out.append(("%s_t%d_r%d_b%d" % (plant, ti, ri, batch), plant, float(tau), int(R),
                                float(s), int(batch)))
    return out


def replay_fixture(ns, kind, fix, par, case, update):
    """Run one recorded sequence on `ns` and compare every step with the fixture.  ``update(lyap,
    can_shrink, R, s)`` calls ``update_safe_set`` in the reference reading of the backend."""
    key, plant, tau, R, s, batch = case
    old = ns.config.gp_batch_size
    try:
        ns.config.gp_batch_size = batch
        lyap = build(ns, dict(par, tau=tau), plant, kind)
        lyap.values = fix["values"]      # V of the reference itself: the sort keys are identical
        for step, can_shrink in ((1, True), (2, False), (3, False)):
            if step == 2:
                if plant == "gp":
                    lyap.dynamics.add_data_point(fix["xnew"], fix["ynew"])
                else:
                    lyap.safe_set = fix[key + "_prev_safe_set"].copy()
                    lyap._refinement = fix[key + "_prev_refinement"].copy()
            update(lyap, can_shrink, R, s)
            tag = "%s_%d" % (key, step)
            assert_array_equal(lyap.safe_set, fix[tag + "_safe_set"], err_msg=tag)
            assert_array_equal(lyap._refinement, fix[tag + "_refinement"], err_msg=tag)
            c_max = lyap.c_max if kind == "oracle" else lyap.feed_dict[lyap.c_max]
            assert float(c_max) == float(fix[tag + "_c_max"]), tag
    finally:
        ns.config.gp_batch_size = old
