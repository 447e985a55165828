"""Synthetic workloads (SURVEY.md section 8d) shared by tests/, bench.py and __graft_entry__.smoke().

Raw parameters are plain numpy (``make_*``); ``build_product`` instantiates the CUDA-backed
``safe_learning_b200`` objects and ``build_oracle`` the numpy oracle from the SAME parameters,
so parity tests compare like with like.  This module is not part of the product package.

Workloads follow the reference's pendulum experiment
(upstream examples/adaptive_safety_verification.ipynb cells 7-17) with the RBF kernel
BASELINE.json names: true pendulum (m=0.15, l=0.5, b=0.1), "wrong" prior model (m=0.1, l=0.4,
b=0) as linear GP prior mean, LQR policy saturated to [-1, 1], V = x^T P x, per-dimension
Lipschitz |2 P x|, tau = sum(unit_maxes)/2, initial safe set |x|_2 <= 0.2, beta = 2,
noise variance 0.001^2.
"""

from __future__ import annotations

import numpy as np
import scipy.linalg
import scipy.signal


# --------------------------------------------------------------------------- pendulum helpers
def _pendulum_linearize(mass, length, friction, dt, state_norm, action_norm):
    g = 9.81
    inertia = mass * length ** 2
    A = np.array([[0, 1], [g / length, -friction / inertia]], dtype=np.float64)
    B = np.array([[0], [1 / inertia]], dtype=np.float64)
    Tx, Tu = np.diag(state_norm), np.diag(action_norm)
    A = np.linalg.multi_dot((np.linalg.inv(Tx), A, Tx))
    B = np.linalg.multi_dot((np.linalg.inv(Tx), B, Tu))
    sysd = scipy.signal.StateSpace(A, B, np.eye(2), np.zeros((2, 1))).to_discrete(dt)
    return sysd.A, sysd.B


def _pendulum_step(sa, mass, length, friction, dt, state_norm, action_norm):
    """True dynamics used to label the GP training set (numpy, fixture generation only)."""
    g = 9.81
    inertia = mass * length ** 2
    state = sa[:, :2] * np.asarray(state_norm)
    action = sa[:, 2:3] * np.asarray(action_norm)
    h = dt / 10
    for _ in range(10):
        acc = g / length * np.sin(state[:, 0:1]) + action / inertia
        if friction > 0:
            acc = acc - friction / inertia * state[:, 1:2]
        state = state + h * np.concatenate((state[:, 1:2], acc), axis=1)
    return state / np.asarray(state_norm)


def _dlqr(a, b, q, r):
    p = scipy.linalg.solve_discrete_are(a, b, q, r)
    btp = b.T.dot(p)
    return np.linalg.solve(btp.dot(b) + r, btp.dot(a)), p


def make_pendulum(num_points=256, M=500, shared_hypers=False, seed=1, noise_std=1e-3,
                  with_prior_mean=True, tau_scale=1.0, scale=1.0):
    """Config C2 (and C5 members): 2-D inverted pendulum, two stacked RBF GPs on [x, u]."""
    dt = 0.01
    theta_max = np.deg2rad(30)
    omega_max = np.sqrt(9.81 / 0.5)
    u_max = 9.81 * 0.15 * 0.5 * np.sin(theta_max)
    state_norm, action_norm = (theta_max, omega_max), (u_max,)
    true_par = dict(mass=0.15, length=0.5, friction=0.1, dt=dt)
    wrong_par = dict(mass=0.1, length=0.4, friction=0.0, dt=dt)
    A_true, B_true = _pendulum_linearize(state_norm=state_norm, action_norm=action_norm, **true_par)
    A, B = _pendulum_linearize(state_norm=state_norm, action_norm=action_norm, **wrong_par)

    K, P = _dlqr(A_true, B_true, np.diag([1., 2.]), 1.2 * np.eye(1))
    P = P / np.abs(P).max()
    L_pol = np.linalg.norm(-K, 1)
    L_dyn = np.linalg.norm(A_true, 1) + np.linalg.norm(B_true, 1) * L_pol

    rng = np.random.default_rng(seed)
    X = rng.uniform(-1, 1, size=(M, 3))
    Y = _pendulum_step(X, state_norm=state_norm, action_norm=action_norm, **true_par)
    Y = Y + noise_std * rng.standard_normal(Y.shape)
    prior_rows = np.hstack((A, B))                        # row j: linear prior mean of output j
    resid = Y - X.dot(prior_rows.T) if with_prior_mean else Y
    if shared_hypers:
        variances = [float(np.mean(resid.var(axis=0)))] * 2
        lengthscales = [[1.5, 1.5, 2.0]] * 2
    else:
        variances = [float(v) for v in resid.var(axis=0)]
        lengthscales = [[1.5, 1.5, 2.0], [1.2, 1.5, 1.8]]

    limits = np.array([[-1., 1.], [-1., 1.]])
    num = np.broadcast_to(num_points, 2).astype(int)
    unit = (limits[:, 1] - limits[:, 0]) / (num - 1)
    # initial safe set from grid coordinates (ijk * unit + offset), cell 11
    axes = [np.arange(n) * u + lo for n, u, lo in zip(num, unit, limits[:, 0])]
    mesh = np.meshgrid(*axes, indexing="ij")
    pts = np.column_stack([m.ravel() for m in mesh])
    initial = np.linalg.norm(pts, ord=2, axis=1) <= 0.2

    return dict(
        name="pendulum%dx%d_M%d_%s" % (num[0], num[1], M, "shared" if shared_hypers else "distinct"),
        limits=limits, num_points=num, tau=float(np.sum(unit) / 2) * tau_scale,
        X=X, Y=Y, variances=variances, lengthscales=lengthscales, noise_variance=noise_std ** 2,
        beta=2.0, scale=scale, prior_rows=prior_rows if with_prior_mean else None,
        K=K, P=P, L_dyn=float(L_dyn), initial=initial,
        plant=dict(state_norm=state_norm, action_norm=action_norm, true=true_par, wrong=wrong_par),
        A_true=A_true, B_true=B_true,
    )


def make_toy_1d(num_points=101, M=50, seed=0):
    """Config C1: 1-D toy dynamics x+ = 0.25 x + 0.1 sin(3 x) (+GP), V = |x| as a 3-vertex
    Triangulation on a separate grid, policy u = 0 (1d_region_of_attraction_estimate.ipynb)."""
    rng = np.random.default_rng(seed)
    X = np.column_stack((rng.uniform(-1, 1, M), np.zeros(M)))
    g = 0.25 * X[:, 0] + 0.1 * np.sin(3 * X[:, 0])
    Y = (g + 0.01 * rng.standard_normal(M))[:, None]
    limits = np.array([[-1., 1.]])
    unit = 2.0 / (num_points - 1)
    pts = np.arange(num_points) * unit - 1.0
    return dict(name="toy1d_%d_M%d" % (num_points, M), limits=limits,
                num_points=np.array([num_points]), tau=1.0 / num_points,
                X=X, Y=Y, variances=[0.4 ** 2], lengthscales=[[1.0, 1.0]],
                noise_variance=0.01 ** 2, beta=2.0, scale=1.0,
                prior_rows=np.array([[0.25, 0.0]]), initial=np.abs(pts) < 0.2,
                L_dyn=0.25, L_v=1.0)


def _cartpole_step(sa, m, M, L, b, dt, state_norm, action_norm):
    g = 9.81
    s = sa[:, :4] * np.asarray(state_norm)
    u = sa[:, 4:5] * np.asarray(action_norm)
    h = dt / 10
    for _ in range(10):
        th, v, om = s[:, 1:2], s[:, 2:3], s[:, 3:4]
        det = L * (M + m * np.square(np.sin(th)))
        v_dot = (u - m * L * np.square(om) * np.sin(th) - b * om * np.cos(th)
                 + 0.5 * m * g * L * np.sin(2 * th)) * L / det
        om_dot = (u * np.cos(th) - 0.5 * m * L * np.square(om) * np.sin(2 * th)
                  - b * (m + M) * om / (m * L) + (m + M) * g * np.sin(th)) / det
        s = s + h * np.concatenate((v, om, v_dot, om_dot), axis=1)
    return s / np.asarray(state_norm)


def make_cartpole(num_points=16, M=200, seed=4, tau_scale=1.0, with_initial=True):
    """Config C4: 4-D cart-pole (reinforcement_learning_cartpole.ipynb cell 7 constants), four
    stacked RBF GPs on [x, u], V = LyapunovNetwork(4, [64, 64, 64], tanh) with fixed-seed
    weights, saturated LQR policy, scalar Lipschitz constants."""
    m, Mc, L, b, dt = 0.175, 1.732, 0.28, 0.01, 0.01
    g = 9.81
    x_max, theta_max, v_max, omega_max = 0.5, np.deg2rad(20), 2.0, np.sqrt(g / L)
    u_max = (m + Mc) * (x_max * 10)
    state_norm, action_norm = (x_max, theta_max, v_max, omega_max), (u_max,)
    A = np.array([[0, 0, 1, 0], [0, 0, 0, 1], [0, g * m / Mc, 0, -b / (Mc * L)],
                  [0, g * (m + Mc) / (L * Mc), 0, -b * (m + Mc) / (m * Mc * L ** 2)]])
    B = np.array([0, 0, 1 / Mc, 1 / (Mc * L)]).reshape((-1, 1))
    Tx, Tu = np.diag(state_norm), np.diag(action_norm)
    A = np.linalg.multi_dot((np.linalg.inv(Tx), A, Tx))
    B = np.linalg.multi_dot((np.linalg.inv(Tx), B, Tu))
    Ad, Bd, _, _, _ = scipy.signal.cont2discrete((A, B, 0, 0), dt, method="zoh")
    K, P = _dlqr(Ad, Bd, np.diag([0.1, 0.1, 0.1, 0.1]), 0.1 * np.eye(1))
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1, 1, size=(M, 5))
    Y = _cartpole_step(X, m, Mc, L, b, dt, state_norm, action_norm)
    Y = Y + 1e-3 * rng.standard_normal(Y.shape)
    prior_rows = np.hstack((Ad, Bd))
    resid = Y - X.dot(prior_rows.T)
    variances = [float(max(v, 1e-6)) for v in resid.var(axis=0)]
    lengthscales = [[1.5, 1.2, 1.5, 1.3, 2.0], [1.4, 1.0, 1.5, 1.2, 1.8],
                    [1.5, 1.1, 1.4, 1.3, 1.9], [1.3, 1.0, 1.5, 1.1, 1.7]]
    limits = np.array([[-1., 1.]] * 4)
    num = np.broadcast_to(num_points, 4).astype(int)
    unit = (limits[:, 1] - limits[:, 0]) / (num - 1)
    initial = None
    if with_initial:        # (skipped for the 64^4 descriptor tests: 16.7 M x 4 coordinates)
        axes = [np.arange(n) * u + lo for n, u, lo in zip(num, unit, limits[:, 0])]
        mesh = np.meshgrid(*axes, indexing="ij")
        pts = np.column_stack([mm.ravel() for mm in mesh])
        initial = np.linalg.norm(pts, ord=2, axis=1) <= 0.3
    wrng = np.random.default_rng(123)
    weights, din = [], 4
    for width in (64, 64, 64):
        hid = int(np.ceil((din + 1) / 2))
        lim0, lim1 = np.sqrt(6.0 / (hid + din)), np.sqrt(6.0 / (max(width - din, 1) + din))
        w0 = wrng.uniform(-lim0, lim0, (hid, din))
        w1 = wrng.uniform(-lim1, lim1, (width - din, din)) if width > din else None
        weights.append((w0, w1))
        din = width
    return dict(name="cartpole%d^4_M%d" % (num[0], M), limits=limits, num_points=num,
                tau=float(np.sum(unit) / 2) * tau_scale, X=X, Y=Y, variances=variances,
                lengthscales=lengthscales, noise_variance=1e-6, beta=2.0, scale=1.0,
                prior_rows=prior_rows, K=K, P=P, initial=initial, nn_weights=weights,
                L_dyn=float(np.linalg.norm(Ad, 1) + np.linalg.norm(Bd, 1) * np.linalg.norm(K, 1)),
                L_v=1.0)


# --------------------------------------------------------------------------- builders
def build_kernel(ns, spec):
    """Kernel from a portable nested-list spec (JSON string or list):
    ["add", k1, k2, ...] | ["prod", k1, k2, ...] | [kind, input_dim, {constructor kwargs}] with kind in
    rbf / matern12 / matern32 / matern52 / linear / constant / white.  `ns` provides classes with
    gpflow 0.4.0's constructor signatures (the oracle, the product, or the fixture shim's
    ``gpflow.kernels``)."""
    import json
    if isinstance(spec, (str, bytes, np.str_)):
        spec = json.loads(str(spec))
    head = spec[0]
    if head in ("add", "prod"):
        parts = [build_kernel(ns, sub) for sub in spec[1:]]
        out = parts[0]
        for k in parts[1:]:
            out = out + k if head == "add" else out * k
        return out
    cls = {"rbf": "RBF", "matern12": "Matern12", "matern32": "Matern32", "matern52": "Matern52",
           "linear": "Linear", "constant": "Constant", "white": "White"}[head]
    kwargs = dict(spec[2]) if len(spec) > 2 else {}
    for key in ("variance", "lengthscales"):
        if isinstance(kwargs.get(key), list):
            kwargs[key] = np.asarray(kwargs[key], dtype=np.float64)
    return getattr(ns, cls)(int(spec[1]), **kwargs)


def notebook_pendulum_kernels(variances):
    """Kernel specs of examples/inverted_pendulum.ipynb cell 6 / adaptive_safety_verification.ipynb
    cell 9: Linear(3, ARD) + Matern32(1, active_dims=[0]) * Linear(1), one per output row of
    `variances` ((m_true - m)^2 clipped)."""
    import json
    specs = []
    for row in np.asarray(variances, dtype=np.float64):
        specs.append(json.dumps(
            ["add", ["linear", 3, {"variance": row.tolist(), "ARD": True}],
             ["prod", ["matern32", 1, {"lengthscales": 1.0, "active_dims": [0]}],
              ["linear", 1, {"variance": float(row[1])}]]]))
    return specs


def _build(ns, par, kind):
    """ns: module namespace providing GridWorld, RBF, GPRCached, ... (product or oracle)."""
    grid = ns.GridWorld(par["limits"], par["num_points"])
    gps = []
    for j in range(par["Y"].shape[1]):
        din = par["X"].shape[1]
        if par.get("kernel_specs") is not None:
            kern = build_kernel(ns, par["kernel_specs"][j])
        else:
            kern = ns.RBF(din, variance=par["variances"][j], lengthscales=par["lengthscales"][j])
        if par["prior_rows"] is None:
            mean = None
        elif kind == "oracle":
            mean = ns.LinearMean(par["prior_rows"][j])
        else:
            mean = ns.LinearSystem(par["prior_rows"][j][None, :])
        gp = ns.GPRCached(par["X"], par["Y"][:, [j]], kern, mean_function=mean,
                          noise_variance=par["noise_variance"], scale=par["scale"])
        gps.append(ns.GaussianProcess(gp, beta=par["beta"]))
    dynamics = ns.FunctionStack(gps)
    return grid, dynamics


def _pendulum_objects(ns, par, kind, deterministic=False):
    grid, dynamics = _build(ns, par, kind)
    policy = ns.Saturation(ns.LinearSystem(-par["K"]), -1., 1.)
    lyap_fun = ns.QuadraticFunction(par["P"])
    l_v = ns.AbsFunction(ns.LinearSystem((2 * par["P"],)))
    if deterministic:
        pl = par["plant"]
        dynamics = ns.InvertedPendulum(normalization=[pl["state_norm"], pl["action_norm"]],
                                       **pl["true"])
    lyap = ns.Lyapunov(grid, lyap_fun, dynamics, par["L_dyn"], l_v, par["tau"], policy,
                       initial_set=par["initial"])
    return lyap


def _toy_objects(ns, par, kind):
    grid, dynamics = _build(ns, par, kind)
    policy = ns.LinearSystem(np.array([[0.0]]))
    vgrid = ns.GridWorld(par["limits"], 3)
    lyap_fun = ns.Triangulation(vgrid, np.array([[1.0], [0.0], [1.0]]))
    return ns.Lyapunov(grid, lyap_fun, dynamics, par["L_dyn"], par["L_v"], par["tau"], policy,
                       initial_set=par["initial"])


def _cartpole_objects(ns, par, kind):
    grid, dynamics = _build(ns, par, kind)
    policy = ns.Saturation(ns.LinearSystem(-par["K"]), -1., 1.)
    if kind == "oracle":
        lyap_fun = ns.LyapunovNetwork(4, [64, 64, 64], [np.tanh] * 3, par["nn_weights"])
    else:
        lyap_fun = ns.LyapunovNetwork(4, [64, 64, 64], ["tanh"] * 3, weights=par["nn_weights"])
    return ns.Lyapunov(grid, lyap_fun, dynamics, par["L_dyn"], par["L_v"], par["tau"], policy,
                       initial_set=par["initial"])


def build_product(par, deterministic=False):
    import safe_learning_b200 as ns
    if par["name"].startswith("toy1d"):
        return _toy_objects(ns, par, "product")
    if par["name"].startswith("cartpole"):
        return _cartpole_objects(ns, par, "product")
    return _pendulum_objects(ns, par, "product", deterministic)


def build_oracle(par, deterministic=False):
    import oracle as ns
    if par["name"].startswith("toy1d"):
        return _toy_objects(ns, par, "oracle")
    if par["name"].startswith("cartpole"):
        return _cartpole_objects(ns, par, "oracle")
    return _pendulum_objects(ns, par, "oracle", deterministic)


def notebook_policy_case(ns, M, batch=1000, seed=0, torch_dynamics=False):
    """examples/inverted_pendulum.ipynb cell 17 at batch size `batch`: a NeuralNetwork([32, 32, 1], relu,
    relu, tanh) policy trained by SGD on -mean(future_values(states, lyapunov=...)) against a FunctionStack
    of two GPs with the notebook's kernel (cell 6) and the wrong model as linear prior mean, M of
    make_pendulum's training points (M = 0: the prior-only stack the notebook starts from), a 55x55
    Triangulation(project=True) value function V = -x^T P x, the Lyapunov function -V and the Lipschitz term
    of cell 14, L_V = MaxAbsFunction(V.gradient_function()).  With `torch_dynamics` the PolicyIteration
    gets the stack's torch_predict expression as a plain callable instead of the stack itself.
    Returns a dict with rl, lyapunov, policy, dynamics, states (device tensor) and step(optimizer)."""
    import torch
    par = make_pendulum(num_points=55, M=max(M, 1), seed=seed)
    X, Y = par["X"][:M], par["Y"][:M]
    specs = notebook_pendulum_kernels([[0.05, 0.1, 0.02], [0.08, 0.12, 0.05]])
    gps = []
    for j in range(2):
        gp = ns.GPRCached(X, Y[:, [j]], build_kernel(ns, specs[j]),
                          mean_function=ns.LinearSystem(par["prior_rows"][j][None, :]),
                          noise_variance=par["noise_variance"])
        gps.append(ns.GaussianProcess(gp, beta=2.0))
    dynamics = ns.FunctionStack(gps)
    grid = ns.GridWorld(par["limits"], par["num_points"])
    pts = grid.all_points
    value = ns.Triangulation(grid, -np.sum(pts.dot(par["P"]) * pts, axis=1, keepdims=True), project=True)
    policy = ns.NeuralNetwork([32, 32, 1], ["relu", "relu", "tanh"], seed=seed + 7)
    reward = -ns.QuadraticFunction(np.diag([1.0, 1.0, 0.1]))
    l_v = ns.MaxAbsFunction(value.gradient_function())
    lyapunov = ns.Lyapunov(grid, -value, dynamics, par["L_dyn"], l_v, par["tau"], policy,
                           initial_set=par["initial"])
    if torch_dynamics:
        def dyn(states, actions):
            return dynamics._torch_expression(torch.cat((states, actions), dim=1))
    else:
        dyn = dynamics
    rl = ns.PolicyIteration(policy, dyn, reward, value, gamma=0.98)
    states = torch.tensor(np.random.default_rng(seed + 11).uniform(-1, 1, (batch, 2)), device="cuda")

    def step(opt, lagrange_multiplier=1.0):
        opt.zero_grad()
        loss = -torch.mean(rl.future_values(states, lyapunov=lyapunov, lagrange_multiplier=lagrange_multiplier))
        loss.backward()
        opt.step()
        return loss.detach()

    return dict(rl=rl, lyapunov=lyapunov, policy=policy, dynamics=dynamics, value=value, states=states,
                step=step, grid=grid, l_dyn=par["L_dyn"], tau=par["tau"], initial=par["initial"])
