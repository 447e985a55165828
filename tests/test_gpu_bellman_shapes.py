"""The policy-iteration kernels at the shapes they are compiled for, against the numpy oracle.

``value_iteration`` (``bellman_kernel``), ``discrete_policy_optimization`` (the per-action
``bellman_argmax_kernel`` and the factored ``bellman_argmax_tile_kernel`` of ``csrc/bellman_tile.cu``)
and the value-operator assembly of ``optimize_value_function`` all run the staged GP mean of
``csrc/gp_mean_staged.cuh``, compiled for d_in = d + m = 1..6.  Here they run at every (d, m) from
(1, 1) to (5, 1), with M on the boundaries of the staged slice (``mean_chunk_rows``: C - 1, C, C + 1)
and of the factored path's 128-row chunk (127, 128, 129), distinct and shared factors, with and
without a linear prior mean, scale 1.7, and a stack whose first GP has no data.

The greedy action is checked against the oracle's Q matrix ``Q[s, i] = future_values(s, a_i)``
(constraint -> -inf) with np.argmax's rules: first maximum, NaN counts as the maximum.  A state is
decisive when its best value beats the runner-up by more than 1e-8 max(1, |Q|); there the index must
be the oracle's, elsewhere the chosen action's value must be within that margin of the maximum."""
import numpy as np
import pytest
from numpy.testing import assert_allclose, assert_array_equal

import bench_workloads as W
import oracle as O
from test_bellman_shapes_host import mean_chunk_rows

pytestmark = pytest.mark.gpu

SCALE = 1.7
GAMMA = 0.9
# about 1.5 k vertices at every state dimension, different counts per axis
NUM = {1: [1501], 2: [41, 37], 3: [13, 12, 11], 4: [7, 6, 6, 7], 5: [5, 4, 4, 5, 4]}


@pytest.fixture(scope="module")
def sl():
    import safe_learning_b200 as mod
    return mod


# ------------------------------------------------------------------------------------ workloads
def make_par(d, m, M, seed, shared=False, prior=True, empty=None):
    """A `bench_workloads._build`-style parameter dict: d state and m action dimensions, M samples of
    a smooth contracting map on [-1, 1]^(d + m) (next states stay inside the grid), ARD RBF
    lengthscales that differ per output (or one factor for all outputs when `shared`), an optional
    linear prior mean, scale 1.7.  `empty`: index of a GP that gets no data."""
    rng = np.random.default_rng(seed)
    A = 0.6 * np.eye(d) + 0.1 / d * rng.uniform(-1, 1, (d, d))
    B = 0.15 / m * rng.uniform(-1, 1, (d, m))
    X = rng.uniform(-1, 1, size=(M, d + m))
    Y = X[:, :d] @ A.T + X[:, d:] @ B.T + 0.05 * np.sin(3 * X[:, :d] + X[:, d:d + 1])
    prior_rows = np.hstack((0.9 * A, 1.1 * B)) if prior else None
    resid = Y - X @ prior_rows.T if prior else Y
    variances = [float(max(v, 1e-3)) for v in resid.var(axis=0)]
    lengthscales = [list(0.8 + 0.6 * rng.random(d + m)) for _ in range(d)]
    if shared:
        variances, lengthscales = [float(np.mean(variances))] * d, [lengthscales[0]] * d
    num = np.array(NUM[d])
    n = int(np.prod(num))
    grid_pts = O.GridWorld(np.array([[-1., 1.]] * d), num).all_points
    # the policy Triangulation's vertex values lie on one linear map u = K x (|u| <= 0.9): the sweeps
    # query it exactly at its vertices, where the reference's lookup may extrapolate from a plane
    # of a neighbouring simplex and the choice among them is not defined (DESIGN.md §3.2 Q6); every
    # plane of a linear map gives the same value
    K = rng.uniform(-1, 1, (m, d))
    K *= 0.9 / np.abs(K).sum(axis=1, keepdims=True)
    policy = grid_pts @ K.T
    # V < 0 everywhere (so every Q < 0 and a best value of 0 is never right), smooth plus noise
    v0 = -(1.0 + 0.5 * np.sum(grid_pts ** 2, axis=1, keepdims=True) + 0.3 * rng.random((n, 1)))
    reward = -scipy_block_diag(np.diag(0.5 + rng.random(d)), np.diag(0.2 + 0.3 * rng.random(m)))
    return dict(name="bellman%dd%da_M%d" % (d, m, M), d=d, m=m, limits=np.array([[-1., 1.]] * d),
                num_points=num, X=X, Y=Y, variances=variances, lengthscales=lengthscales,
                noise_variance=1e-3, beta=2.0, scale=SCALE, prior_rows=prior_rows, empty=empty,
                policy=policy, v0=v0, reward=reward)


def scipy_block_diag(a, b):
    import scipy.linalg
    return scipy.linalg.block_diag(a, b)


def build(ns, par, kind):
    """PolicyIteration with a FunctionStack of one-output GPs (the GP `par["empty"]` without data),
    a policy Triangulation and a projected value Triangulation on one grid, a quadratic reward."""
    grid = ns.GridWorld(par["limits"], par["num_points"])
    gps = []
    for j in range(par["d"]):
        X, Y = par["X"], par["Y"][:, [j]]
        if par["empty"] == j:
            X, Y = X[:0], Y[:0]
        kern = ns.RBF(X.shape[1], variance=par["variances"][j], lengthscales=par["lengthscales"][j])
        if par["prior_rows"] is None:
            mean = None
        elif kind == "oracle":
            mean = ns.LinearMean(par["prior_rows"][j])
        else:
            mean = ns.LinearSystem(par["prior_rows"][j][None, :])
        gp = ns.GPRCached(X, Y, kern, mean_function=mean, noise_variance=par["noise_variance"],
                          scale=par["scale"])
        gps.append(ns.GaussianProcess(gp, beta=par["beta"]))
    policy = ns.Triangulation(grid, par["policy"].copy())
    value = ns.Triangulation(grid, par["v0"].copy(), project=True)
    return ns.PolicyIteration(policy, ns.FunctionStack(gps), ns.QuadraticFunction(par["reward"]),
                              value, gamma=GAMMA)


def nomax(par, shared):
    return par["d"] if shared else 1


# (d, m): layout, prior mean, and M on the staged slice's boundaries C - 1, C, C + 1 plus one M that
# is not a multiple of 8; C = mean_chunk_rows(d + m, outputs on the largest factor)
SWEEP_CONFIGS = [
    (1, 1, False, True, 61),
    (1, 2, False, False, 99),
    (2, 1, True, True, 45),
    (2, 2, True, False, 101),
    (3, 1, True, False, 75),
    (3, 2, False, True, 53),
    (4, 1, True, True, 83),
    (4, 2, False, False, 67),
    (5, 1, True, False, 93),
]


def _sweep_cases():
    out = []
    for d, m, shared, prior, odd in SWEEP_CONFIGS:
        C = mean_chunk_rows(d + m, d if shared else 1)
        for M in (C - 1, C, C + 1, odd):
            out.append(pytest.param(d, m, M, shared, prior,
                                    id="d%dm%d-%s-%s-M%d-C%d" % (d, m, "shared" if shared else "distinct",
                                                                "prior" if prior else "noprior", M, C)))
    return out


def test_sweep_cases_sit_on_the_slice_boundaries():
    """The slice sizes the cases are built around (4 and 5 outputs on one factor included)."""
    sizes = sorted({mean_chunk_rows(d + m, d if shared else 1) for d, m, shared, _, _ in SWEEP_CONFIGS})
    assert sizes == [128, 152, 192, 216, 256]
    assert mean_chunk_rows(6, 1) == 192 and mean_chunk_rows(5, 4) == 152


# ------------------------------------------------------------------------------ a. Bellman sweep
def _sweeps_vs_oracle(sl, par):
    rl_g, rl_c = build(sl, par, "product"), build(O, par, "oracle")
    for _ in range(3):
        res = rl_g.value_iteration()
        old = rl_c.value_function.parameters.copy()
        new = rl_c.value_iteration()
        assert_allclose(rl_g.value_function.parameters[0], new, rtol=1e-9, atol=1e-12)
        assert_allclose(res, np.max(np.abs(new - old)), rtol=1e-9)
    return rl_g


@pytest.mark.parametrize("d,m,M,shared,prior", _sweep_cases())
def test_bellman_sweep_vs_oracle(sl, d, m, M, shared, prior):
    par = make_par(d, m, M, seed=100 * d + 10 * m + M % 10, shared=shared, prior=prior)
    rl = _sweeps_vs_oracle(sl, par)
    st = rl.dynamics.gp_stack()
    assert st.num_factors == (1 if shared else d)
    assert [st.factors[f].M for f in range(st.num_factors)] == [M] * st.num_factors


@pytest.mark.parametrize("empty", [0, 1])
def test_bellman_sweep_with_an_empty_factor(sl, empty):
    """Two GPs, one without data: its factor has M = 0 next to one with 100 rows, and the staged
    mean's producer skips it (first_factor_with_data); its mean is the prior mean."""
    par = make_par(2, 1, 100, seed=7, prior=True, empty=empty)
    rl = _sweeps_vs_oracle(sl, par)
    st = rl.dynamics.gp_stack()
    assert st.num_factors == 2
    assert sorted(st.factors[f].M for f in range(2)) == [0, 100]
    assert st.factors[st.outputs[empty].factor].M == 0
    # the factored path needs data on every factor: the per-action kernel, against the oracle
    actions = np.linspace(-1, 1, 9)[:, None]
    Q, _ = _oracle_q(build(O, par, "oracle"), actions)
    rl.value_function.parameters = par["v0"]
    best, bv, need = _argmax(sl, rl, actions, factored=True)
    assert need == 0
    _check_greedy(Q, best, bv)


# ---------------------------------------------------------------------- b. greedy policy, both paths
def _argmax(sl, rl, actions, constraint=None, begin=0, end=None, factored=True):
    """slb_bellman_argmax through the C ABI with a best_value buffer; the factored path when
    `factored` and the library offers a workspace.  Returns (best, best_value, workspace bytes)."""
    import torch
    from safe_learning_b200 import _device as dev, _native as nat
    lib = nat.load()
    end = rl.value_function.nindex if end is None else end
    n, n_actions = end - begin, len(actions)
    cfg = rl.bellman_descriptor(fixed_action=actions[0])
    need = int(lib.slb_bellman_argmax_workspace(cfg, n_actions))
    ws = dev.empty((need // 8 + 1,)) if factored and need else None
    actions_dev = dev.to_device(np.ascontiguousarray(actions, dtype=np.float64))
    cons_dev = None if constraint is None else dev.to_device(np.ascontiguousarray(constraint))
    best = dev.empty((n,), torch.int32)
    best_value = dev.empty((n,))
    nat.check(lib.slb_bellman_argmax(dev.stream(), cfg, begin, end, actions_dev.data_ptr(), n_actions,
                                     dev.ptr(cons_dev), best.data_ptr(), best_value.data_ptr(),
                                     dev.ptr(ws)), "slb_bellman_argmax")
    return best.cpu().numpy(), best_value.cpu().numpy(), need


def _oracle_q(rl_c, actions, states=None):
    """The oracle's future_values(states, a_i) for every action, split as the oracle computes it
    (rewards + gamma * V(mean next state)) so that other value tables reuse the GP means.
    Returns (Q, q_of) with q_of(table) giving Q for another value table."""
    states = rl_c.state_space if states is None else states
    parts = []
    for a in actions:
        arr = np.broadcast_to(a, (len(states), len(a)))
        mean, _ = rl_c.dynamics(states, arr)
        parts.append((rl_c.reward_function(states, arr)[:, 0], mean))

    def q_of(table):
        rl_c.value_function.parameters = table
        return np.stack([r + rl_c.gamma * rl_c.value_function(mean)[:, 0] for r, mean in parts], axis=1)

    q = q_of(rl_c.value_function.parameters.copy())
    assert_allclose(q[:, 0], rl_c.future_values(states, actions=np.broadcast_to(
        actions[0], (len(states), actions.shape[1])))[:, 0], rtol=0, atol=0)
    return q, q_of


def _masked(Q, constraint):
    Q = Q.copy()
    if constraint is not None:
        Q[constraint.T < 0] = -np.inf
    return Q


def _check_greedy(Q, best, bv, min_decisive=0.95):
    """np.argmax's rules against the oracle's Q [n, n_actions]; returns the decisive fraction."""
    n = Q.shape[0]
    want = np.argmax(Q, axis=1)
    nan_row = np.isnan(Q).any(axis=1)
    assert_array_equal(best[nan_row], want[nan_row])                  # the first NaN
    assert np.isnan(bv[nan_row]).all()
    dead = ~nan_row & np.all(Q == -np.inf, axis=1)                    # every action constrained
    assert_array_equal(best[dead], 0)
    assert (bv[dead] == -np.inf).all()
    rest = ~nan_row & ~dead
    Qr, br, vr = Q[rest], best[rest], bv[rest]
    chosen = Qr[np.arange(len(Qr)), br]
    assert_allclose(vr, chosen, rtol=1e-9, atol=0)
    top = np.sort(Qr, axis=1)
    first, second = top[:, -1], (top[:, -2] if Q.shape[1] > 1 else np.full(len(Qr), -np.inf))
    margin = 1e-8 * np.maximum(1.0, np.abs(first))
    decisive = first - second > margin
    assert_array_equal(br[decisive], want[rest][decisive])
    assert np.all(first - chosen <= margin)                           # near ties: within the margin
    frac = decisive.sum() / max(1, len(Qr))
    assert frac >= min_decisive, "only %.3f of the states are decisive" % frac
    return frac


def _actions(m, count, seed):
    if m == 1:
        return np.linspace(-1, 1, count)[:, None]
    return np.random.default_rng(seed).uniform(-1, 1, (count, m))


# (d, m, M, shared, prior, n_actions): d <= 2 takes the factored path (DS = 1, 2) as well as the
# per-action kernel; M = 127 / 128 / 129 sit on the tile's 128-row chunk, the others on the staged
# slice; 2 / 7 / 8 actions keep only warp 0 busy, 129 leaves one row block for the second pass, 202
# makes two passes of 16 and 10 row blocks
GREEDY_CASES = [
    (1, 1, 127, False, True, 202),
    (1, 2, 128, False, False, 129),
    (1, 1, 129, False, False, 2),
    (1, 1, 61, False, True, 128),
    (2, 1, 127, True, False, 7),
    (2, 1, 128, False, True, 101),
    (2, 2, 129, True, True, 8),
    (2, 2, 257, False, False, 9),
    (3, 1, 255, False, True, 9),
    (3, 2, 169, True, True, 9),
    (4, 1, 152, True, False, 7),
    (4, 2, 193, False, True, 9),
    (5, 1, 127, True, True, 7),
]


def _greedy_id(c):
    return "d%dm%d-M%d-%s-%s-A%d" % (c[0], c[1], c[2], "shared" if c[3] else "distinct",
                                     "prior" if c[4] else "noprior", c[5])


@pytest.mark.parametrize("d,m,M,shared,prior,n_actions", GREEDY_CASES, ids=[_greedy_id(c) for c in GREEDY_CASES])
def test_greedy_policy_both_paths_vs_oracle(sl, d, m, M, shared, prior, n_actions):
    par = make_par(d, m, M, seed=1000 + 100 * d + 10 * m + n_actions, shared=shared, prior=prior)
    rl = build(sl, par, "product")
    rl_c = build(O, par, "oracle")
    actions = _actions(m, n_actions, seed=d)
    Q, q_of = _oracle_q(rl_c, actions)
    n = Q.shape[0]
    rng = np.random.default_rng(d + m)
    some = np.where(rng.random((n_actions, n)) < 0.3, -1.0, 1.0)     # ~30% of the actions per state
    dead = some.copy()
    dead[:, ::11] = -1.0                                              # every action at every 11th state
    v_nan = par["v0"].copy()
    v_nan[n // 3:n // 3 + n // 10] = np.nan
    Q_nan = q_of(v_nan)
    assert np.isnan(Q_nan).any(axis=1).mean() > 0.02 and not np.isnan(Q_nan).all()
    begin, end = 37, 37 + 64 * ((n - 100) // 64) + 23
    factorable = d <= 2
    paths = (True, False) if factorable else (False,)
    for factored in paths:
        rl.value_function.parameters = par["v0"]
        best, bv, need = _argmax(sl, rl, actions, factored=factored)
        assert (need > 0) == factorable
        if need:
            nrb, total = -(-n_actions // 8), 0
            st = rl.dynamics.gp_stack()
            for o in range(d):
                total += nrb * -(-st.factors[st.outputs[o].factor].M // 8) * 64 * 8
            assert need == total
        _check_greedy(Q, best, bv)
        for cons in (some, dead):
            best, bv, _ = _argmax(sl, rl, actions, constraint=cons, factored=factored)
            _check_greedy(_masked(Q, cons), best, bv, min_decisive=0.0)
        assert (np.all(dead.T < 0, axis=1)).sum() >= n // 11
        # an index range that starts at 37 and is not a multiple of 64 long: the constraint slab
        # [n_actions, end - begin] is indexed relative to the range
        best, bv, _ = _argmax(sl, rl, actions, constraint=some[:, begin:end], begin=begin, end=end,
                              factored=factored)
        _check_greedy(_masked(Q, some)[begin:end], best, bv, min_decisive=0.0)
        best, bv, _ = _argmax(sl, rl, actions, begin=begin, end=end, factored=factored)
        _check_greedy(Q[begin:end], best, bv)
        # NaN in the value table: the first NaN of the oracle's row wins
        rl.value_function.parameters = v_nan
        best, bv, _ = _argmax(sl, rl, actions, factored=factored)
        _check_greedy(Q_nan, best, bv, min_decisive=0.0)


@pytest.mark.parametrize("d,m,M,shared", [(1, 1, 129, False), (2, 1, 128, False), (2, 2, 127, True),
                                          (3, 1, 100, False)])
def test_greedy_exact_ties(sl, d, m, M, shared):
    """Duplicate actions give bit-identical values on each path, so np.argmax must pick the first
    copy: the 101-action list repeated ([A; A], two passes of the tile) and interleaved
    (a0, a0, a1, a1, ...: the copies fall into different i mod 4 groups of a thread)."""
    par = make_par(d, m, M, seed=77 + d, shared=shared, prior=True)
    rl = build(sl, par, "product")
    A = _actions(m, 101, seed=5)
    for factored in ((True, False) if d <= 2 else (False,)):
        best, bv, need = _argmax(sl, rl, A, factored=factored)
        assert (need > 0) == (d <= 2)
        b2, v2, _ = _argmax(sl, rl, np.concatenate((A, A)), factored=factored)
        assert_array_equal(b2, best)
        assert_array_equal(v2.view(np.int64), bv.view(np.int64))
        b3, v3, _ = _argmax(sl, rl, np.repeat(A, 2, axis=0), factored=factored)
        assert_array_equal(b3, 2 * best)
        assert_array_equal(v3.view(np.int64), bv.view(np.int64))
    rl_c = build(O, par, "oracle")
    idx = np.random.default_rng(3).choice(rl.value_function.nindex, 300, replace=False)
    Q, _ = _oracle_q(rl_c, A, states=rl_c.state_space[idx])
    _check_greedy(Q, best[idx], bv[idx])


# ------------------------------------------------------------------------------------------- c. C3
def test_c3_factored_equals_per_action(sl):
    """C3: 512 x 512 states, 101 actions, two RBF factors of M = 500 rows.  The factored path and
    the per-action kernel agree on every state; both against the oracle on 4096 seeded states."""
    par = W.make_pendulum(num_points=8, M=500)
    out = {}
    for ns, kind in ((sl, "product"), (O, "oracle")):
        grid = ns.GridWorld(par["limits"], 512)
        _, dyn = W._build(ns, par, kind)
        reward = ns.QuadraticFunction(-scipy_block_diag(np.diag([1., 2.]), 1.2 * np.eye(1)))
        pts = O.GridWorld(par["limits"], 512).all_points
        noise = np.random.default_rng(0).random((grid.nindex, 1))
        v0 = -(1.0 + np.sum(pts ** 2, axis=1, keepdims=True) + 0.01 * noise)
        value = ns.Triangulation(grid, v0, project=True)
        policy = ns.Triangulation(grid, np.zeros((grid.nindex, 1)), project=True)
        out[kind] = ns.PolicyIteration(policy, dyn, reward, value, gamma=0.98)
    rl = out["product"]
    actions = np.linspace(-1, 1, 101)[:, None]
    b_f, v_f, need = _argmax(sl, rl, actions, factored=True)
    b_p, v_p, _ = _argmax(sl, rl, actions, factored=False)
    assert need == 2 * 13 * 63 * 64 * 8
    assert_allclose(v_f, v_p, rtol=1e-12, atol=0)
    # the choices may differ only where the per-action values of both choices are within 1e-12
    # (one fixed-action sweep per action involved: the per-action kernel's own values)
    differ = np.flatnonzero(b_f != b_p)
    q_at = {}
    for i in np.unique(np.concatenate((b_f[differ], b_p[differ]))):
        q_at[i] = _fixed_action_sweep(sl, rl, actions[i])
    for s in differ:
        qf, qp = q_at[b_f[s]][s], q_at[b_p[s]][s]
        assert abs(qf - qp) <= 1e-12 * abs(qp), (s, b_f[s], b_p[s], qf, qp)
    rl_c = out["oracle"]
    idx = np.random.default_rng(11).choice(rl.value_function.nindex, 4096, replace=False)
    Q, _ = _oracle_q(rl_c, actions, states=rl_c.state_space[idx])
    _check_greedy(Q, b_f[idx], v_f[idx])
    _check_greedy(Q, b_p[idx], v_p[idx])


def _fixed_action_sweep(sl, rl, action):
    """r(x, a) + gamma V(mean f(x, a)) at every vertex for one action (slb_bellman_sweep)."""
    from safe_learning_b200 import _device as dev, _native as nat
    n = rl.value_function.nindex
    out = dev.empty((n,))
    nat.check(nat.load().slb_bellman_sweep(dev.stream(), rl.bellman_descriptor(fixed_action=action), 0, n,
                                           out.data_ptr()), "slb_bellman_sweep")
    return out.cpu().numpy()


# -------------------------------------------------------------------------- d. value operator
@pytest.mark.parametrize("d,m,shared,prior,M", [(c[0], c[1], c[2], c[3], c[4]) for c in SWEEP_CONFIGS],
                         ids=["d%dm%d" % (c[0], c[1]) for c in SWEEP_CONFIGS])
def test_value_operator_is_one_sweep(sl, d, m, shared, prior, M):
    """One iteration of optimize_value_function's solve from a random table is one value_iteration
    sweep bit for bit: the fused assembly runs the same staged GP mean at every d_in.  The GP-mean
    next states stay inside the grid, so no row needs the grid-line repair (stats slot 2)."""
    par = make_par(d, m, M, seed=300 + d + m, shared=shared, prior=prior)
    rl = build(sl, par, "product")
    values, info = rl._evaluate_policy(1e-10, 1)
    assert info["iterations"] == 1
    assert info["repaired_rows"] == 0
    rl.value_iteration()
    assert_array_equal(values, rl.value_function.parameters[0])
