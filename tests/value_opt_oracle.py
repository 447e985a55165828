"""numpy restatement of ``PolicyIteration.optimize_value_function`` as this build computes it
(``csrc/value_opt.cu``): the operator rows of the value Triangulation at the next states, with the
grid-line rows (DESIGN.md §3.2 Q6) re-searched, and the certified fixed-point iteration.  Elementwise
numpy operations are never contracted, so the restatement is bit-exact where the kernels use
non-contracted fp64 in the same order."""
import numpy as np

W_TOL = 1e-12
EPS = np.finfo(np.float64).eps


def _search(tri, unit):
    """First simplex of the unit cell whose barycentric weights at `unit` are all >= -W_TOL, else the
    one whose smallest weight is largest (common.cuh tri_lookup)."""
    disc = tri.discretization
    d = tri.input_dim
    best, best_min = 0, -np.inf
    for s in range(tri.nsimplex_unit):
        ijk = np.array(np.unravel_index(tri.unit_simplices[s, 0], disc.num_points), dtype=np.float64)
        o = ijk * disc.unit_maxes
        H = tri.hyperplanes[s]
        w = np.array([np.sum((unit - o) * H[:, c]) for c in range(d)])
        wmin = min(np.min(w), 1.0 - np.sum(w))
        if wmin > best_min:
            best, best_min = s, wmin
        if wmin >= -W_TOL:
            break
    return best


def _barycentric(tri, x, corner, s):
    disc = tri.discretization
    d = tri.input_dim
    origin = disc.index_to_state(tri.unit_simplices[s, 0] + corner)[0]
    if tri.project:
        x = np.minimum(np.maximum(x, disc.limits[:, 0]), disc.limits[:, 1])
    off = x - origin
    H = tri.hyperplanes[s]
    w = np.empty(d + 1)
    for c in range(d):
        acc = off[0] * H[0, c]
        for k in range(1, d):
            acc = acc + off[k] * H[k, c]
        w[c + 1] = acc
    acc = w[1]
    for c in range(2, d + 1):
        acc = acc + w[c]
    w[0] = 1.0 - acc
    return w


def library_simplices(tri, x):
    """The simplex of the unit cell the library's lookup picks (common.cuh): the first simplex whose
    weights at the `% unit_maxes` coordinates are >= -W_TOL (else the largest smallest weight); a
    point clipped in every dimension takes Qhull's simplex of that corner.  It differs from Qhull's
    pick only where both simplices contain the point (a shared face) or both miss it."""
    disc = tri.discretization
    d = tri.input_dim
    centered = x - disc.offset
    lo = disc.offset_limits[:, 0] + 2 * EPS
    hi = disc.offset_limits[:, 1] - 2 * EPS
    unit = np.clip(centered, lo, hi) % disc.unit_maxes
    all_clipped = np.all((centered < lo) | (centered > hi), axis=1)
    best = np.zeros(len(x), dtype=np.int64)
    best_min = np.full(len(x), -np.inf)
    done = np.zeros(len(x), dtype=bool)
    for s in range(tri.nsimplex_unit):
        ijk = np.array(np.unravel_index(tri.unit_simplices[s, 0], disc.num_points), dtype=np.float64)
        ws = (unit - ijk * disc.unit_maxes) @ tri.hyperplanes[s]
        wmin = np.minimum(np.min(ws, axis=1), 1.0 - np.sum(ws, axis=1))
        take = ~done & (wmin > best_min)
        best[take], best_min[take] = s, wmin[take]
        done |= wmin >= -W_TOL
    # Qhull's simplex of an isolated query (the library's corner_simplex table): within one call scipy's
    # walk starts from the previous query's simplex, so the points are asked one at a time
    for i in np.flatnonzero(all_clipped) if d > 1 else ():
        best[i] = tri.find_simplex(x[i:i + 1])[0] % tri.nsimplex_unit
    return best



def operator(tri, next_states, lookup="qhull"):
    """Rows of T for an ``oracle.Triangulation`` at next_states [N, d]: (cols [N, d+1] int64,
    weights [N, d+1], repaired [N] bool).  ``lookup="qhull"``: rows outside Q6 are the reference's
    (``parameter_derivative``); ``lookup="library"``: the first lookup picks the library's simplex
    (``library_simplices``), which is what the kernels compute."""
    x = np.atleast_2d(np.asarray(next_states, dtype=np.float64))
    disc = tri.discretization
    w, cols = tri.weights(x)
    w, cols = w.copy(), cols.astype(np.int64)
    if lookup == "library":
        corners = disc.rectangle_corner_index(disc.state_to_rectangle(x))
        ids = tri.find_simplex(x) % tri.nsimplex_unit
        mine = library_simplices(tri, x)
        for i in np.flatnonzero(mine != ids):
            w[i] = _barycentric(tri, x[i], corners[i], mine[i])
            cols[i] = tri.unit_simplices[mine[i]] + corners[i]
    inside = np.all((x >= disc.limits[:, 0]) & (x <= disc.limits[:, 1]), axis=1)
    q6 = (np.min(w, axis=1) < -W_TOL) & (tri.project | inside)
    corners = disc.rectangle_corner_index(disc.state_to_rectangle(x))
    for i in np.flatnonzero(q6):
        lo = disc.index_to_state(corners[i])[0]
        unit = np.minimum(np.maximum(x[i], disc.limits[:, 0]), disc.limits[:, 1]) - lo
        s = _search(tri, unit)
        w[i] = _barycentric(tri, x[i], corners[i], s)
        cols[i] = tri.unit_simplices[s] + corners[i]
    return cols, w, q6


def rho(weights):
    a = np.abs(weights[:, 0])
    for k in range(1, weights.shape[1]):
        a = a + np.abs(weights[:, k])
    return float(np.max(a))


def apply(cols, weights, rewards, gamma, v):
    """r + gamma (w_0 v[c_0] + w_1 v[c_1] + ...), left to right."""
    s = weights[:, 0] * v[cols[:, 0]]
    for k in range(1, cols.shape[1]):
        s = s + weights[:, k] * v[cols[:, k]]
    return rewards + gamma * s


def solve(cols, weights, rewards, gamma, v0, tol=1e-10, max_iters=200000):
    """The certified iteration: returns (values, iterations, last delta, bound) or raises
    ValueError when the operator is not a nonnegative contraction or the iteration does not
    converge."""
    rewards = np.asarray(rewards, dtype=np.float64).reshape(-1)
    v = np.asarray(v0, dtype=np.float64).reshape(-1).copy()
    if np.min(weights) < -W_TOL:
        raise ValueError("negative weight")
    gr = gamma * rho(weights)
    if not gr < 1.0:
        raise ValueError("not a contraction")
    q = gr / (1.0 - gr)
    for k in range(1, max_iters + 1):
        nv = apply(cols, weights, rewards, gamma, v)
        delta = float(np.max(np.abs(nv - v)))
        vmax = float(np.max(np.abs(nv)))
        v = nv
        bound = q * delta
        if bound <= tol * max(1.0, vmax):
            return v, k, delta, bound
    raise ValueError("not converged")


def dense(cols, weights, n):
    T = np.zeros((cols.shape[0], n))
    for k in range(cols.shape[1]):
        np.add.at(T, (np.arange(cols.shape[0]), cols[:, k]), weights[:, k])
    return T


# ------------------------------------------------------------------ the fixture's GP cases
GP1D_KERNEL = ["prod", ["matern32", 1, {"lengthscales": 0.5, "variance": 0.04, "active_dims": [0]}],
               ["linear", 1, {"active_dims": [0]}]]
GP1D_PRIOR = np.array([[1.0, 0.1]])
GP1D_REWARD = np.diag([-1.0, -0.2])
GP1D_ACTIONS = np.linspace(-0.5, 0.5, 11)[:, None]
GP55_VARIANCES = [[2e-3, 6e-3, 1.5e-3], [2.5e-2, 8e-3, 1.2e-2]]


def gp1d_objects(ns, z, kind):
    """``make_golden_value_opt.py``'s 1-D case built from `ns` (the oracle or the product):
    (policy iteration, grid).  kind: "oracle" or "product" (how the prior mean is given)."""
    import bench_workloads as W
    grid = ns.GridWorld([[-1., 1.]], 51)
    kern = W.build_kernel(ns, GP1D_KERNEL)
    mean = ns.LinearMean(GP1D_PRIOR[0]) if kind == "oracle" else ns.LinearSystem(GP1D_PRIOR)
    gp = ns.GaussianProcess(ns.GPRCached(z["gp1d_X"], z["gp1d_Y"], kern, mean_function=mean,
                                         noise_variance=1e-6), beta=2.0)
    policy = ns.Triangulation(grid, -0.3 * grid.all_points)
    value = ns.Triangulation(grid, np.zeros((grid.nindex, 1)), project=True)
    return ns.PolicyIteration(policy, gp, ns.QuadraticFunction(GP1D_REWARD), value, gamma=0.98), grid


def gp55_objects(ns, kind):
    """The 55 x 55 notebook-kernel pendulum case: (policy iteration, grid)."""
    import bench_workloads as W
    from scipy.linalg import block_diag
    par = W.make_pendulum(num_points=55, M=12, with_prior_mean=True, seed=3)
    par["kernel_specs"] = W.notebook_pendulum_kernels(GP55_VARIANCES)
    grid, dynamics = W._build(ns, par, kind)
    policy = ns.Saturation(ns.LinearSystem((-par["K"],)), -1., 1.)
    reward = ns.QuadraticFunction(block_diag(-np.diag([1., 2.]), -1.2 * np.eye(1)))
    value = ns.Triangulation(grid, np.zeros((grid.nindex, 1)), project=True)
    return ns.PolicyIteration(policy, dynamics, reward, value, gamma=0.98), grid


def evaluate(rl, lookup="library", tol=1e-10):
    """optimize_value_function restated on oracle objects: (values, cols, weights, rewards)."""
    states = rl.state_space
    actions = rl.policy(states)
    nxt = rl.dynamics(states, actions)
    if isinstance(nxt, tuple):
        nxt = nxt[0]
    rewards = np.asarray(rl.reward_function(states, actions), dtype=np.float64).ravel()
    cols, w, _ = operator(rl.value_function, nxt, lookup=lookup)
    v, _, _, _ = solve(cols, w, rewards, rl.gamma, np.asarray(rl.value_function.parameters).ravel(),
                       tol=tol)
    return v, cols, w, rewards
