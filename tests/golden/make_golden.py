"""Generate golden fixtures by executing the UNMODIFIED reference (a befelix/safe_learning @ f1aad5a
checkout named by $SAFE_LEARNING_REFERENCE) on the numpy-backed TF1 / gpflow API shims in
``tf1_shim/``.

    SAFE_LEARNING_REFERENCE=<checkout> python tests/golden/make_golden.py [grid|gp|gp_kernels|lyapunov|policy|tri_gradient ...]   # rewrites tests/golden/*.npz

Each fixture stores the raw inputs and the reference's outputs; tests/test_golden_fixtures.py
rebuilds the numpy oracle (CPU tests) and the CUDA product (GPU tests) from the same inputs
and compares.  What runs from the reference's own source: GridWorld, _Triangulation /
Triangulation, LinearSystem, QuadraticFunction, Saturation, GPRCached (cache + predict),
GaussianProcess, FunctionStack, Lyapunov (threshold, v_decrease_*, update_values,
update_safe_set incl. the batch loop and c_max), PolicyIteration (future_values,
value_iteration, discrete_policy_optimization), utilities (batchify, dlqr, concatenate_inputs).
What is restated in the shim (third-party, not part of the reference): tf ops -> numpy,
gpflow 0.4.0 RBF kernel arithmetic.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)

from reference_loader import load_reference  # noqa: E402

sl = load_reference()
import gpflow  # noqa: E402  (shim)
import tensorflow as tf  # noqa: E402  (shim)

import bench_workloads as W  # noqa: E402


def ref_gp_stack(par):
    gps = []
    for j in range(par["Y"].shape[1]):
        din = par["X"].shape[1]
        if par.get("kernel_specs") is not None:
            kern = W.build_kernel(gpflow.kernels, par["kernel_specs"][j])
        else:
            kern = gpflow.kernels.RBF(din, variance=par["variances"][j],
                                      lengthscales=np.asarray(par["lengthscales"][j]), ARD=True)
        mean = gpflow.mean_functions.Zero() if par["prior_rows"] is None else \
            sl.LinearSystem((par["prior_rows"][j][None, :],), name="prior_%d" % j)
        gp = sl.GPRCached(par["X"], par["Y"][:, [j]], kern, mean, par["scale"])
        gp.likelihood.variance = par["noise_variance"]
        gp.update_cache()
        gps.append(sl.GaussianProcess(gp, beta=par["beta"]))
    return sl.FunctionStack(gps)


def ref_pendulum_lyapunov(par):
    grid = sl.GridWorld(par["limits"], par["num_points"])
    dynamics = ref_gp_stack(par)
    policy = sl.Saturation(sl.LinearSystem((-par["K"],), name="policy"), -1., 1.)
    lyap_fun = sl.QuadraticFunction(par["P"])
    grad = sl.LinearSystem((2 * par["P"],), name="grad_v")
    l_v = lambda x: tf.abs(grad(x))  # noqa: E731  (notebook cell 17)
    return sl.Lyapunov(grid, lyap_fun, dynamics, par["L_dyn"], l_v, par["tau"], policy,
                       par["initial"].copy())


def ref_toy_lyapunov(par):
    grid = sl.GridWorld(par["limits"], par["num_points"])
    dynamics = ref_gp_stack(par)
    policy = sl.LinearSystem((np.array([[0.0]]),), name="zero_policy")
    vgrid = sl.GridWorld(par["limits"], 3)
    lyap_fun = sl.Triangulation(vgrid, np.array([[1.0], [0.0], [1.0]]), name="v_tri")
    return sl.Lyapunov(grid, lyap_fun, dynamics, par["L_dyn"], par["L_v"], par["tau"], policy,
                       par["initial"].copy())


def flat_par(par, prefix="par_"):
    out = {}
    for k, v in par.items():
        if k in ("name", "plant"):
            continue
        if v is None:
            continue
        out[prefix + k] = np.asarray(v)
    return out


def sweep_outputs(lyap, feed=None):
    """decrease / threshold / negative on every grid point, plus GP mean and error."""
    states = lyap.discretization.all_points
    tf_states = tf.placeholder(tf.float64, [None, lyap.discretization.ndim])
    actions = lyap.policy(tf_states)
    nxt = lyap.dynamics(tf_states, actions)
    decrease = lyap.v_decrease_bound(tf_states, nxt)
    threshold = lyap.threshold(tf_states, lyap.tau)
    fd = dict(lyap.feed_dict)
    fd[tf_states] = states
    mean, err = nxt
    thr = threshold.eval(fd) if isinstance(threshold, tf.Tensor) else np.asarray(threshold)
    return dict(decrease=decrease.eval(fd), threshold=np.broadcast_to(thr, (len(states), 1)).copy(),
                mean=mean.eval(fd), err=err.eval(fd))


def gen_lyapunov(out, only=None):
    cases = {}
    # C2-like pendulum, multi-batch (batch 64), growing safe set
    par = W.make_pendulum(num_points=[26, 21], M=90, tau_scale=1 / 150.)
    cases["pendulum"] = (par, ref_pendulum_lyapunov, 64)
    par = W.make_pendulum(num_points=[17, 19], M=30, tau_scale=0.0, scale=1.7, shared_hypers=True)
    cases["pendulum_allsafe"] = (par, ref_pendulum_lyapunov, 50)
    par = W.make_toy_1d(num_points=101, M=25)
    par["tau"] = 0.02
    cases["toy1d"] = (par, ref_toy_lyapunov, 40)
    # the kernels of the reference's own experiments (inverted_pendulum.ipynb cell 6): linear ARD +
    # Matern32 x linear, one expression per output, linear prior mean
    par = W.make_pendulum(num_points=[24, 19], M=90, tau_scale=1 / 150., with_prior_mean=True, seed=3)
    par["kernel_specs"] = W.notebook_pendulum_kernels([[2e-3, 6e-3, 1.5e-3], [2.5e-2, 8e-3, 1.2e-2]])
    cases["pendulum_nbkernel"] = (par, ref_pendulum_lyapunov, 64)
    # 1d_region_of_attraction_estimate.ipynb cell 5: Matern32 x Linear on the state column
    par = W.make_toy_1d(num_points=91, M=20)
    par["tau"] = 0.02
    par["kernel_specs"] = [json.dumps(
        ["prod", ["matern32", 1, {"lengthscales": 1.0, "variance": 0.16, "active_dims": [0]}],
         ["linear", 1, {"active_dims": [0]}]])]
    cases["toy1d_nbkernel"] = (par, ref_toy_lyapunov, 40)
    for name, (par, builder, batch) in cases.items():
        if only and name not in only:
            continue
        with tf.Session():
            sl.config.gp_batch_size = batch
            lyap = builder(par)
            res = flat_par(par)
            res["batch"] = np.array(batch)
            res["values"] = lyap.values.copy()
            res.update({"sweep_" + k: v for k, v in sweep_outputs(lyap).items()})
            lyap.update_safe_set()
            res["safe_set"] = lyap.safe_set.copy()
            res["c_max"] = np.array(lyap.feed_dict[lyap.c_max])
            res["refinement"] = lyap._refinement.copy()
            if name == "pendulum":       # lyapunov.py:657-797 on the fresh safe set
                pert = np.array([[-0.2], [-0.05], [0.0], [0.05], [0.2]])
                lim = np.array([[-1., 1.]])
                res["gss_perturbations"], res["gss_limits"] = pert, lim
                for positive in (True, False):
                    sa, bound = sl.get_safe_sample(lyap, pert, lim, positive=positive)
                    res["gss_state_action_%d" % positive] = sa
                    res["gss_bound_%d" % positive] = np.array(bound)
            # second phase: add a data point (Cholesky update path) then can_shrink=False
            xnew = np.array([[0.3, -0.2, 0.1]])[:, :par["X"].shape[1]]
            ynew = np.array([[0.05, -0.02]])[:, :par["Y"].shape[1]]
            if par["Y"].shape[1] == 1:      # FunctionStack.add_data_point iterates y.squeeze()
                lyap.dynamics.functions[0].add_data_point(xnew, ynew)
            else:
                lyap.dynamics.add_data_point(xnew, ynew)
            res["xnew"], res["ynew"] = xnew, ynew
            lyap.update_safe_set(can_shrink=False)
            res["safe_set_noshrink"] = lyap.safe_set.copy()
            res["c_max_noshrink"] = np.array(lyap.feed_dict[lyap.c_max])
            res["refinement_noshrink"] = lyap._refinement.copy()
            lyap.update_safe_set(can_shrink=True)
            res["safe_set_after_add"] = lyap.safe_set.copy()
            res["c_max_after_add"] = np.array(lyap.feed_dict[lyap.c_max])
            np.savez_compressed(os.path.join(out, "lyapunov_%s.npz" % name), **res)
            print(name, "safe", res["safe_set"].sum(), "/", res["safe_set"].size, "c_max",
                  res["c_max"], "| no-shrink", res["safe_set_noshrink"].sum(), "| after add",
                  res["safe_set_after_add"].sum())
    sl.config.gp_batch_size = 10000


def gen_gp(out):
    rng = np.random.default_rng(42)
    res = {}
    with tf.Session():
        for tag, scale, with_mean in (("plain", 1.0, False), ("scaled_mean", 2.5, True)):
            par = W.make_pendulum(num_points=8, M=60, scale=scale, with_prior_mean=with_mean,
                                  seed=5)
            stack = ref_gp_stack(par)
            pts = rng.uniform(-1.2, 1.2, (80, 3))
            mean, err = stack(pts)
            res.update({tag + "_" + k: v for k, v in flat_par(par).items()})
            res[tag + "_points"] = pts
            res[tag + "_mean"] = mean.eval(stack.feed_dict)
            res[tag + "_err"] = err.eval(stack.feed_dict)
            gp0 = stack.functions[0].gaussian_process
            m0, v0 = gp0.build_predict(pts)
            res[tag + "_var0"] = v0.eval()
            res[tag + "_cholesky0"] = gp0.cholesky.value.copy()
            res[tag + "_alpha0"] = gp0.alpha.value.copy()
    np.savez_compressed(os.path.join(out, "gp_predict.npz"), **res)
    print("gp fixtures:", sorted(k for k in res if k.endswith("_mean")))


def gen_gp_kernels(out):
    """GP posterior through the reference's GPRCached / GaussianProcess / FunctionStack for the
    covariance expressions of SURVEY.md 8(f) item 3 (every primitive, active_dims, sums of
    products, shared and distinct factors, empty data set)."""
    rng = np.random.default_rng(7)
    nb = W.notebook_pendulum_kernels([[0.02, 0.06, 0.015], [0.25, 0.08, 0.12]])
    mix = json.dumps(
        ["add",
         ["prod", ["rbf", 2, {"variance": 0.7, "lengthscales": [0.8, 1.3], "active_dims": [0, 2],
                              "ARD": True}],
          ["matern52", 1, {"variance": 1.4, "lengthscales": 0.6, "active_dims": [1]}]],
         ["matern12", 3, {"variance": 0.3, "lengthscales": 1.7}],
         ["prod", ["constant", 3, {"variance": 0.05}], ["linear", 1, {"variance": 0.9, "active_dims": [2]}]],
         ["white", 3, {"variance": 0.01}]])
    m32 = json.dumps(["matern32", 3, {"variance": 0.9, "lengthscales": [0.5, 1.1, 0.9], "ARD": True}])
    rbf_sub = json.dumps(["rbf", 2, {"variance": 1.2, "lengthscales": [0.7, 0.4], "active_dims": [1, 0],
                                     "ARD": True}])
    cases = {"notebook": (nb, 45, True, 1.0), "mix": ([mix, mix], 33, False, 2.0),
             "matern32": ([m32, rbf_sub], 70, True, 1.0), "empty": (nb, 0, True, 1.0)}
    res = {}
    with tf.Session():
        for tag, (specs, M, with_mean, scale) in cases.items():
            par = W.make_pendulum(num_points=8, M=max(M, 1), scale=scale, with_prior_mean=with_mean,
                                  seed=11)
            if M == 0:
                par["X"], par["Y"] = par["X"][:0], par["Y"][:0]
            par["kernel_specs"] = specs
            stack = ref_gp_stack(par)
            pts = rng.uniform(-1.2, 1.2, (70, 3))
            pts[:min(M, 5)] = par["X"][:min(M, 5)]           # a few queries on training inputs
            mean, err = stack(pts)
            res.update({tag + "_" + k: v for k, v in flat_par(par).items()})
            res[tag + "_points"] = pts
            res[tag + "_mean"] = mean.eval(stack.feed_dict)
            res[tag + "_err"] = err.eval(stack.feed_dict)
            gp0 = stack.functions[0].gaussian_process
            _, v0 = gp0.build_predict(pts)
            res[tag + "_var0"] = v0.eval()
            if M:
                res[tag + "_cholesky0"] = gp0.cholesky.value.copy()
    np.savez_compressed(os.path.join(out, "gp_kernels.npz"), **res)
    print("gp kernel fixtures:", sorted(k for k in res if k.endswith("_mean")))


def gen_grid_triangulation(out):
    rng = np.random.default_rng(7)
    res = {}
    for tag, limits, num in (("g1", [[-1.0, 1.5]], [6]), ("g2", [[-1.0, 1.5], [0.0, 2.0]], [5, 4]),
                             ("g3", [[-1, 1], [0, 2], [-0.5, 0.5]], [4, 3, 5])):
        grid = sl.GridWorld(limits, num)
        lo, hi = grid.limits[:, 0], grid.limits[:, 1]
        inside = rng.uniform(lo, hi, (300, grid.ndim))
        outside = rng.uniform(lo - 0.4 * (hi - lo), hi + 0.4 * (hi - lo), (300, grid.ndim))
        vals = rng.normal(size=(grid.nindex, 2))
        res[tag + "_limits"], res[tag + "_num"] = grid.limits, grid.num_points
        res[tag + "_inside"], res[tag + "_outside"], res[tag + "_vals"] = inside, outside, vals
        res[tag + "_all_points"] = grid.all_points
        res[tag + "_idx_of_outside"] = grid.state_to_index(outside)
        res[tag + "_rect_of_outside"] = grid.state_to_rectangle(outside)
        with tf.Session():
            for project in (False, True):
                tri = sl.Triangulation(grid, vals, project=project, name="tri_%s_%d" % (tag, project))
                key = tag + ("_proj" if project else "_noproj")
                res[key + "_inside"] = tri(inside).eval()
                res[key + "_vertices"] = tri(grid.all_points).eval()
                # one query at a time: scipy's find_simplex walks from the previous query's
                # simplex, which makes corner-clipped extrapolation batch-order dependent
                res[key + "_outside"] = np.vstack([tri(p[None, :]).eval() for p in outside])
            res[tag + "_unit_simplices"] = tri.tri.unit_simplices
            res[tag + "_hyperplanes"] = tri.tri.hyperplanes
    np.savez_compressed(os.path.join(out, "grid_triangulation.npz"), **res)
    print("grid/triangulation fixtures written")


def gen_triangulation_gradient(out):
    """Triangulation.gradient (functions.py:1260-1326, 1506-1510) on 1-D / 2-D / 3-D grids, and a
    Lyapunov sweep with V = -value table and L_V = max |gradient| as in
    examples/inverted_pendulum.ipynb cell 14."""
    rng = np.random.default_rng(17)
    res = {}
    with tf.Session():
        for tag, limits, num in (("g1", [[-1.0, 1.5]], [6]), ("g2", [[-1.0, 1.5], [0.0, 2.0]], [5, 4]),
                                 ("g3", [[-1, 1], [0, 2], [-0.5, 0.5]], [4, 3, 5])):
            grid = sl.GridWorld(limits, num)
            lo, hi = grid.limits[:, 0], grid.limits[:, 1]
            inside = rng.uniform(lo, hi, (200, grid.ndim))
            vals = rng.normal(size=(grid.nindex, 1))
            tri = sl.Triangulation(grid, vals, name="tri_grad_%s" % tag)
            res[tag + "_limits"], res[tag + "_num"] = grid.limits, grid.num_points
            res[tag + "_inside"], res[tag + "_vals"] = inside, vals
            res[tag + "_gradient"] = tri.gradient(inside).eval()
        # Lyapunov sweep: V = -(value table) on a coarse triangulation, L_V(x) = max_k |dV/dx_k|
        # upstream quirk: a query exactly ON a vertex can land in a simplex of the cell that does not
        # contain that vertex ((x - offset) % unit_maxes rounds to ~unit_maxes instead of 0), and the
        # value is then extrapolated from the wrong plane -- the interpolant does not reproduce its
        # own vertex values on e.g. a 25 x 21 grid.  Pinned as is.
        qgrid = sl.GridWorld([[-1, 1], [-1, 1]], [25, 21])
        qvals = rng.normal(size=(qgrid.nindex, 1))
        qtri = sl.Triangulation(qgrid, qvals, name="tri_quirk")
        res["quirk_vals"] = qvals
        res["quirk_at_vertices"] = qtri(qgrid.all_points).eval()
        par = W.make_pendulum(num_points=[25, 21], M=90, tau_scale=1 / 400.)
        # the value table lives on a slightly larger, non-commensurate grid so that no state of the
        # sweep sits on a simplex face (the gradient is discontinuous there and upstream's pick is
        # scipy's order-dependent walk)
        vgrid = sl.GridWorld(par["limits"] * np.array([[1.05, 1.08], [1.03, 1.06]]), [30, 26])
        table = -np.sum(vgrid.all_points.dot(par["P"]) * vgrid.all_points, axis=1, keepdims=True)
        value = sl.Triangulation(vgrid, table, name="value_table")
        l_v = lambda x: tf.reduce_max(tf.abs(value.gradient(x)), axis=1, keepdims=True)  # noqa: E731
        grid = sl.GridWorld(par["limits"], par["num_points"])
        policy = sl.Saturation(sl.LinearSystem((-par["K"],), name="policy_g"), -1., 1.)
        lyap = sl.Lyapunov(grid, -value, ref_gp_stack(par), par["L_dyn"], l_v, par["tau"], policy,
                           par["initial"].copy())
        res.update(flat_par(par, "lyap_par_"))
        res["lyap_vgrid_num"], res["lyap_table"] = np.array([30, 26]), table
        res["lyap_vgrid_limits"] = vgrid.limits
        res["lyap_values"] = lyap.values.copy()
        res.update({"lyap_sweep_" + k: v for k, v in sweep_outputs(lyap).items()})
        lyap.update_safe_set()
        res["lyap_safe_set"] = lyap.safe_set.copy()
        res["lyap_c_max"] = np.array(lyap.feed_dict[lyap.c_max])
    np.savez_compressed(os.path.join(out, "triangulation_gradient.npz"), **res)
    print("triangulation gradient fixtures written; lyapunov safe", res["lyap_safe_set"].sum(), "/",
          res["lyap_safe_set"].size)


def gen_policy_iteration(out):
    res = {}
    par = W.make_pendulum(num_points=8, M=40, seed=9)
    rng = np.random.default_rng(3)
    with tf.Session():
        grid = sl.GridWorld(par["limits"], [13, 11])
        dynamics = ref_gp_stack(par)
        policy = sl.Saturation(sl.LinearSystem((-par["K"],), name="rl_policy"), -1., 1.)
        import scipy.linalg
        rew = -scipy.linalg.block_diag(np.diag([1., 2.]), 1.2 * np.eye(1))
        reward = sl.QuadraticFunction(rew)
        v0 = -rng.random((grid.nindex, 1))
        value = sl.Triangulation(grid, v0, project=True, name="value_fn")
        rl = sl.PolicyIteration(policy, dynamics, reward, value, gamma=0.98)
        states = rng.uniform(-1, 1, (60, 2))
        fv = rl.future_values(tf.constant(states))
        res["future_values"] = fv.eval(rl.feed_dict)
        op = rl.value_iteration()
        tables = []
        for _ in range(3):
            op.eval(rl.feed_dict)
            tables.append(value.parameters[0].eval().copy())
        res["value_tables"] = np.stack(tables)
        # greedy policy over a discrete action set (deterministic dynamics variant as well)
        pol_tri = sl.Triangulation(grid, np.zeros((grid.nindex, 1)), name="policy_tri")
        rl2 = sl.PolicyIteration(pol_tri, dynamics, reward, value, gamma=0.98)
        actions = np.linspace(-1, 1, 9)[:, None]
        constraint = lambda arr: np.where(np.abs(arr[:, 0]) > 0.8, -1.0, 1.0)  # noqa: E731
        rl2.discrete_policy_optimization(actions, constraint)
        res["greedy_policy"] = pol_tri.parameters[0].eval().copy()
    res.update(flat_par(par))
    res["grid_num"], res["reward"], res["v0"] = np.array([13, 11]), rew, v0
    res["states"], res["actions"] = states, actions
    np.savez_compressed(os.path.join(out, "policy_iteration.npz"), **res)
    print("policy iteration fixtures written; greedy actions used:",
          np.unique(res["greedy_policy"]).size)


if __name__ == "__main__":
    generators = {"grid": gen_grid_triangulation, "gp": gen_gp, "gp_kernels": gen_gp_kernels,
                  "lyapunov": gen_lyapunov, "policy": gen_policy_iteration,
                  "tri_gradient": gen_triangulation_gradient}
    for name in (sys.argv[1:] or list(generators)):     # "lyapunov:case1,case2" limits the cases
        name, _, only = name.partition(":")
        if only:
            generators[name](HERE, only.split(","))
        else:
            generators[name](HERE)
