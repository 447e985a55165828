"""GPU tests of the Triangulation vertex gradient (``csrc/triangulation_grad.cu``), ``vertex_values``,
``parameter_derivative``, parameter gradients through post-op wrappers, and the reference's training
loops that use them (``tests/test_functions.py:740-761``, ``tests/test_rl.py:29-77``,
``examples/basic_dynamic_programming.ipynb`` cells 2-5)."""
import os

import numpy as np
import pytest
import scipy.linalg
import scipy.sparse
import scipy.sparse.linalg
import torch

import network_grad_oracle as G
import oracle as O
import safe_learning_b200 as sl
from safe_learning_b200 import functions as F

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                      "triangulation_param_derivative.npz")
GOLDEN_HIGH_DIM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                               "triangulation_high_dim.npz")
T64 = torch.float64
CUDA = "cuda"

GRIDS = {1: [7], 2: [6, 5], 3: [4, 3, 5], 4: [3, 4, 3, 3], 5: [3] * 5, 6: [3, 2, 3, 2, 3, 2]}


def _grid(d):
    return sl.GridWorld([[-1.0 - 0.1 * c, 1.0 + 0.2 * c] for c in range(d)], GRIDS[d])


def _points(grid, rng):
    """33 points: inside, on cell faces, outside, one NaN and two vertices."""
    lo, hi = grid.limits[:, 0], grid.limits[:, 1]
    inside = rng.uniform(lo, hi, (12, grid.ndim))
    faces = rng.uniform(lo, hi, (8, grid.ndim))
    for i in range(len(faces)):
        c = i % grid.ndim
        faces[i, c] = grid.discrete_points[c][i % grid.num_points[c]]
    outside = rng.uniform(lo - 0.5 * (hi - lo), hi + 0.5 * (hi - lo), (10, grid.ndim))
    nan = np.full((1, grid.ndim), np.nan)
    verts = grid.all_points[[0, grid.nindex // 2]]
    return np.vstack([inside, faces, outside, nan, verts])


def _add_at(pd, g, nindex):
    """np.add.at over parameter_derivative's rows: the determinism contract of the kernel."""
    n = pd.shape[0]
    nsimp = pd.nnz // max(n, 1)
    c = pd.col.reshape(n, nsimp)
    w = pd.data.reshape(n, nsimp)
    out = np.zeros((nindex, g.shape[1]))
    np.add.at(out, c.ravel(), (w[..., None] * g[:, None, :]).reshape(-1, g.shape[1]))
    return out


def _vertex_grad(tri, x, g):
    return tri._param_vjp(torch.tensor(x, device=CUDA), torch.tensor(g, device=CUDA))[0].cpu().numpy()


# ---------------------------------------------------------------- 1. the determinism contract
@pytest.mark.parametrize("d", range(1, 7))
@pytest.mark.parametrize("out", [1, 2])
@pytest.mark.parametrize("project", [False, True])
def test_vertex_gradient_is_add_at_of_the_rows(d, out, project):
    rng = np.random.default_rng(10 * d + out)
    grid = _grid(d)
    tri = sl.Triangulation(grid, rng.normal(size=(grid.nindex, out)), project=project)
    pts = _points(grid, rng)
    for n in (0, 1, 33):
        x, g = pts[:n], rng.normal(size=(n, out))
        got = _vertex_grad(tri, x, g)
        pd = tri.tri.parameter_derivative(x) if n else scipy.sparse.coo_matrix((0, grid.nindex))
        want = _add_at(pd, g, grid.nindex) if n else np.zeros((grid.nindex, out))
        np.testing.assert_array_equal(got, want)
        assert np.array_equal(got.view(np.uint64), _vertex_grad(tri, x, g).view(np.uint64))
    if d in (2, 4) and out == 1:
        lo, hi = grid.limits[:, 0], grid.limits[:, 1]
        x = rng.uniform(lo - 0.2 * (hi - lo), hi + 0.2 * (hi - lo), (10 ** 6, d))
        g = rng.normal(size=(10 ** 6, out))
        got = _vertex_grad(tri, x, g)
        np.testing.assert_array_equal(got, _add_at(tri.tri.parameter_derivative(x), g, grid.nindex))
        assert np.array_equal(got.view(np.uint64), _vertex_grad(tri, x, g).view(np.uint64))


def test_all_points_on_one_vertex():
    grid = _grid(2)
    tri = sl.Triangulation(grid, np.arange(grid.nindex, dtype=np.float64), project=True)
    x = np.full((10 ** 5, 2), -100.0)
    g = np.random.default_rng(0).normal(size=(10 ** 5, 1))
    got = _vertex_grad(tri, x, g)
    pd = tri.tri.parameter_derivative(x)
    np.testing.assert_array_equal(got, _add_at(pd, g, grid.nindex))
    # the clipped corner is the first vertex; the others of its simplex carry rounding-size weights
    assert np.abs(got[1:]).max() < 1e-12 * np.abs(got[0, 0])


# ---------------------------------------------------------------- 2. parameter_derivative vs the reference
def _fixture_cases():
    """(fixture, key, points) of triangulation_param_derivative.npz (d = 1..3) and of
    triangulation_high_dim.npz (d = 4..6, whose points are stored once per grid and group)."""
    fix = np.load(GOLDEN)
    for key in sorted(k[:-len("_points")] for k in fix.files if k.endswith("_points")):
        yield fix, key, fix[key + "_points"]
    high = np.load(GOLDEN_HIGH_DIM)
    for key in sorted(k[:-len("_cols")] for k in high.files if k.endswith("_cols")):
        tag, _, group = key.split("_", 2)
        yield high, key, high[tag + "_" + group]


def test_parameter_derivative_matches_reference_fixture():
    report = {}
    for fix, key, pts in _fixture_cases():
        tag, proj, group = key.split("_", 2)
        grid = sl.GridWorld(fix[tag + "_limits"], fix[tag + "_num"])
        rng = np.random.default_rng(1)
        v = rng.normal(size=(grid.nindex, 1))
        tri = sl.Triangulation(grid, v, project=proj == "proj")
        pd = tri.tri.parameter_derivative(pts)
        n, nsimp = fix[key + "_cols"].shape
        assert pd.shape == (n, grid.nindex)
        np.testing.assert_array_equal(pd.row, np.repeat(np.arange(n), nsimp))
        cols, w = pd.col.reshape(n, nsimp), pd.data.reshape(n, nsimp)
        same = np.all(cols == fix[key + "_cols"], axis=1)
        np.testing.assert_array_equal(w[same], fix[key + "_weights"][same])
        other = np.flatnonzero(~same)
        report[key] = len(other)
        # rows whose simplex differs lie on a face shared by both simplices: same linear form, except
        # for exact vertex queries (DESIGN.md §3.2 Q6) and unprojected queries clipped in some but not
        # all dimensions (an extrapolation across a shared edge), where the reference's choice depends
        # on scipy's walk
        if other.size and group != "vertices" and not (proj == "noproj" and group == "outside"):
            ref = scipy.sparse.coo_matrix((fix[key + "_weights"].ravel(),
                                           (np.repeat(np.arange(n), nsimp), fix[key + "_cols"].ravel())),
                                          shape=(n, grid.nindex)).toarray()
            np.testing.assert_allclose(pd.toarray()[other], ref[other], rtol=0, atol=1e-12)
        val = tri(pts)
        np.testing.assert_allclose(pd @ v, val, rtol=1e-14, atol=1e-14 * np.abs(v).max())
    print("rows with a different simplex than Qhull's:", {k: c for k, c in report.items() if c})


# ---------------------------------------------------------------- 3. exactness, point gradient unchanged
@pytest.mark.parametrize("d", [1, 2, 3])
def test_vertex_gradient_is_exact(d):
    rng = np.random.default_rng(d)
    grid = _grid(d)
    v = rng.normal(size=(grid.nindex, 1))
    tri = sl.Triangulation(grid, v, project=True)
    x = _points(grid, rng)[:30]
    g = np.ones((len(x), 1))
    for _ in range(5):
        e = rng.normal(size=(grid.nindex, 1))
        t = 1e-3
        f0 = tri(x)
        tri.parameters = v + t * e
        f1 = tri(x)
        tri.parameters = v
        rows = tri.tri.parameter_derivative(x)
        np.testing.assert_allclose(f1 - f0, t * (rows @ e), rtol=1e-9, atol=1e-13)
        # per point (unit cotangent on one point), the vertex gradient is that point's row
        for p in range(0, len(x), 7):
            gp = np.zeros_like(g)
            gp[p] = 1.0
            np.testing.assert_array_equal(_vertex_grad(tri, x, gp)[:, 0], rows.toarray()[p])


@pytest.mark.parametrize("project", [False, True])
def test_point_gradient_is_the_previous_path(project):
    rng = np.random.default_rng(5)
    grid = _grid(2)
    tri = sl.Triangulation(grid, rng.normal(size=(grid.nindex, 1)), project=project)
    x = torch.tensor(rng.uniform(-1.5, 1.5, (500, 2)), device=CUDA)
    g = torch.tensor(rng.normal(size=(500, 1)), device=CUDA)
    x1 = x.clone().requires_grad_(True)
    F._FusedApply.apply(x1, tri).backward(g)
    leaf = tri.vertex_values
    x2 = x.clone().requires_grad_(True)
    tri.torch(x2).backward(g)
    assert torch.equal(x1.grad, x2.grad)
    assert leaf.grad is not None and torch.equal(
        leaf.grad, tri._param_vjp(x, g)[0])


# ---------------------------------------------------------------- 4. transcribed reference tests
def test_gradient_param():
    """tests/test_functions.py:740-761."""
    disc = sl.GridWorld([[0, 1], [0, 1]], 3)
    params = np.sum(disc.all_points ** 2, axis=1, keepdims=True)
    tri = sl.Triangulation(disc, params, project=True)
    test_points = np.array([[-10, -10], [0.2, 0.7], [0, 0], [0, 1], [1, 1], [-0.2, 0.5], [0.43, 0.21]],
                           dtype=np.float64)
    true_gradient = np.array(tri.tri.parameter_derivative(test_points).todense())
    leaf = tri.vertex_values
    for i, test in enumerate(test_points):
        leaf.grad = None
        tri.torch(torch.tensor(test[None, :], device=CUDA)).sum().backward()
        np.testing.assert_allclose(leaf.grad.cpu().numpy()[:, 0], true_gradient[i])


def test_integration():
    """tests/test_rl.py:29-77 with torch.optim.SGD(lr=0.01) on [policy.vertex_values]."""
    a, b, q, r = np.array([[1.2]]), np.array([[0.9]]), np.array([[1]]), np.array([[0.1]])
    k, p = O.dlqr(a, b, q, r)
    discretization = sl.GridWorld([[-1, 1]], 19)
    value_function = sl.Triangulation(discretization, 0. * discretization.all_points, project=True)
    dynamics = sl.LinearSystem((a, b))
    policy_discretization = sl.GridWorld([-1, 1], 5)
    policy = sl.Triangulation(policy_discretization, -k / 2 * policy_discretization.all_points)
    reward_function = sl.QuadraticFunction(-scipy.linalg.block_diag(q, r))
    rl = sl.PolicyIteration(policy, dynamics, reward_function, value_function)
    opt = torch.optim.SGD([rl.policy.vertex_values], lr=0.01)
    states = torch.tensor(rl.state_space, device=CUDA)
    for _ in range(10):
        rl.value_iteration()
        for _ in range(5):
            loss = -torch.sum(rl.future_values(states))
            opt.zero_grad()
            loss.backward()
            opt.step()
    values = rl.value_function.parameters[0]
    true_values = O.QuadraticFunction(-p)(rl.state_space)
    np.testing.assert_allclose(values, true_values, atol=0.1)
    np.testing.assert_allclose(rl.policy.parameters[0], -k * policy_discretization.all_points, atol=0.1)


# ---------------------------------------------------------------- torch-CPU restatement
def tri_torch(x, v, otri):
    """Triangulation(x) on CPU tensors, differentiable in x and v: the oracle's simplices and origins,
    w = (clip(x) - origin) H, the reference's weights (functions.py:1473-1499)."""
    xn = x.detach().numpy()
    ids = otri.find_simplex(xn)
    simp = otri.simplices(ids)
    origins = torch.tensor(otri.discretization.index_to_state(simp[:, 0]))
    planes = torch.tensor(otri.hyperplanes[ids % otri.nsimplex_unit])
    if otri.project:
        lim = torch.tensor(otri.discretization.limits)
        x = torch.minimum(torch.maximum(x, lim[:, 0]), lim[:, 1])
    w1 = torch.einsum("nk,nkc->nc", x - origins, planes)
    w = torch.cat([1 - w1.sum(dim=1, keepdim=True), w1], dim=1)
    return torch.einsum("nk,nko->no", w, v[torch.tensor(simp)])


def saturate(u, lo, hi):
    """clip with the library's gradient rule: zero at equality with a bound (DESIGN.md §3.11)."""
    return torch.where((u > lo) & (u < hi), u, u.detach().clamp(lo, hi))


def _mountain_car(xp):
    gamma = 0.99

    def dynamics(states, actions):
        x0 = states[:, 0] + states[:, 1]
        x1 = states[:, 1] + 0.001 * actions[:, 0] - 0.0025 * xp.cos(3 * states[:, 0])
        return xp.stack((x0, x1), 1)

    def reward(states, actions):
        hit = states[:, :1] > 0.6
        return xp.where(hit, (1 - gamma) * xp.ones_like(states[:, :1]), xp.zeros_like(states[:, :1]))
    return gamma, dynamics, reward


class _XP:
    """numpy or torch, by the argument type (the notebook's callables are TF; these run on both)."""

    def __getattr__(self, name):
        def call(*args, **kw):
            arr = args[0][0] if isinstance(args[0], tuple) else args[0]
            mod = torch if isinstance(arr, torch.Tensor) else np
            if name == "stack" and mod is torch:
                return torch.stack(args[0], dim=args[1])
            if name == "stack":
                return np.stack(args[0], axis=args[1])
            return getattr(mod, name)(*args, **kw)
        return call


def test_basic_dynamic_programming_matches_torch_cpu():
    """examples/basic_dynamic_programming.ipynb cells 2-5 (20 x 20 mountain car), 3 outer x 20 inner
    steps, against a float64 torch-CPU restatement step by step.  The policy is queried exactly at its
    vertices, where the simplex choice is undefined upstream (DESIGN.md §3.2 Q6), so the restatement
    takes the policy's rows at the state space from parameter_derivative; everything else (value
    lookups at the next states, the exact policy evaluation, gradients, SGD) is restated on the CPU."""
    domain, n_points = [[-1.2, 0.7], [-.07, .07]], [20, 20]
    disc = sl.GridWorld(domain, n_points)
    value_function = sl.Triangulation(disc, np.zeros(disc.nindex), project=True)
    policy_tri = sl.Triangulation(disc, np.zeros(disc.nindex), project=True)
    policy = sl.Saturation(policy_tri, -1., 1.)
    gamma, dynamics, reward = _mountain_car(_XP())
    rl = sl.PolicyIteration(policy, dynamics, reward, value_function, gamma=gamma)
    opt = torch.optim.SGD([policy_tri.vertex_values], lr=1.)
    states = torch.tensor(rl.state_space, device=CUDA)

    odisc = O.GridWorld(domain, n_points)
    otri = O.Triangulation(odisc, np.zeros((odisc.nindex, 1)), project=True)
    pv = torch.zeros((disc.nindex, 1), dtype=T64, requires_grad=True)
    copt = torch.optim.SGD([pv], lr=1.)
    cstates = torch.tensor(rl.state_space)
    prows = torch.tensor(policy_tri.tri.parameter_derivative(rl.state_space).toarray())
    for _ in range(3):
        rl.optimize_value_function()
        # CPU: exact policy evaluation v = r + gamma T v on the oracle's rows
        with torch.no_grad():
            u = saturate(prows @ pv, -1., 1.)
            nxt = dynamics(cstates, u).numpy()
            r = reward(cstates, u).numpy()[:, 0]
        w, c = otri.weights(nxt)
        n = disc.nindex
        T = scipy.sparse.csr_matrix((w.ravel(), (np.repeat(np.arange(n), w.shape[1]), c.ravel())), shape=(n, n))
        cv = torch.tensor(scipy.sparse.linalg.spsolve((scipy.sparse.identity(n) - gamma * T).tocsc(), r)[:, None])
        gv = value_function.parameters[0]
        np.testing.assert_allclose(gv, cv.numpy(), rtol=0, atol=1e-9 * max(1.0, np.abs(cv.numpy()).max()))
        for _ in range(20):
            loss = -1 / (1 - gamma) * torch.mean(rl.future_values(states))
            opt.zero_grad()
            loss.backward()
            opt.step()
            ua = saturate(prows @ pv, -1., 1.)
            closs = -1 / (1 - gamma) * torch.mean(reward(cstates, ua) + gamma * tri_torch(
                dynamics(cstates, ua), torch.tensor(gv), otri))
            copt.zero_grad()
            closs.backward()
            copt.step()
            got, want = policy_tri.parameters[0], pv.detach().numpy()
            np.testing.assert_allclose(got, want, rtol=0, atol=1e-9 * max(1e-3, np.abs(want).max()))
    assert np.abs(policy_tri.parameters[0]).max() > 0          # the policy did move


# ---------------------------------------------------------------- 6. Saturation(NeuralNetwork) in future_values
def test_saturated_network_policy_gets_parameter_gradients():
    rng = np.random.default_rng(7)
    net = sl.NeuralNetwork([2, 16, 1], ["tanh", None], seed=4)
    policy = sl.Saturation(net, -0.3, 0.3)
    disc = sl.GridWorld([[-1, 1], [-1, 1]], [9, 8])
    vals = rng.normal(size=(disc.nindex, 1))
    value = sl.Triangulation(disc, vals, project=True)
    A = np.array([[1.0, 0.1], [0.0, 1.0]])
    B = np.array([[0.0], [0.1]])
    dynamics = sl.LinearSystem((A, B))
    Q = -np.diag([1.0, 0.5, 0.2])
    reward = sl.QuadraticFunction(Q)
    rl = sl.PolicyIteration(policy, dynamics, reward, value, gamma=0.9)
    x = rng.uniform(-1, 1, (200, 2))
    loss = -rl.future_values(torch.tensor(x, device=CUDA)).sum()
    loss.backward()
    grads = [p.grad.cpu() for p in net.parameters]
    assert all(g is not None and torch.any(g != 0) for g in grads)

    cp = [p.detach().cpu().clone().requires_grad_(True) for p in net.parameters]
    xs = torch.tensor(x)
    u = saturate(G.mlp(xs, [cp[0], cp[2]], [cp[1]], ["tanh", "linear"], 1.0), -0.3, 0.3)
    z = torch.cat([xs, u], dim=1)
    nxt = z @ torch.tensor(np.hstack([A, B])).T
    otri = O.Triangulation(O.GridWorld([[-1, 1], [-1, 1]], [9, 8]), vals, project=True)
    closs = -(torch.sum((z @ torch.tensor(Q)) * z, dim=1, keepdim=True)
              + 0.9 * tri_torch(nxt, torch.tensor(vals), otri)).sum()
    closs.backward()
    for g, c in zip(grads, cp):
        np.testing.assert_allclose(g.numpy(), c.grad.numpy(), rtol=1e-10, atol=1e-12)


# ---------------------------------------------------------------- 7. in-place steps are seen; stale backward raises
def _rl(disc, value_table, policy_table):
    value = sl.Triangulation(disc, value_table, project=True)
    policy = sl.Triangulation(disc, policy_table, project=True)
    dyn = sl.LinearSystem((np.array([[1.0, 0.1], [0.0, 1.0]]), np.array([[0.0], [0.1]])))
    return sl.PolicyIteration(policy, dyn, sl.QuadraticFunction(-np.eye(3)), value, gamma=0.9)


def test_in_place_steps_reach_the_fused_sweeps():
    disc = sl.GridWorld([[-1, 1], [-1, 1]], [11, 9])
    rl = _rl(disc, np.zeros((disc.nindex, 1)), np.zeros((disc.nindex, 1)))
    value, policy = rl.value_function, rl.policy
    rl.value_iteration()
    leaf, ptr, v0 = value.vertex_values, value.vertex_values.data_ptr(), value.version
    pleaf = policy.vertex_values
    with torch.no_grad():                      # optimizer-style steps on both tables
        leaf.add_(1.0)
        pleaf.fill_(0.5)
    assert value.version != v0
    stepped = value.parameters[0].copy()
    ref = _rl(disc, stepped, np.full((disc.nindex, 1), 0.5))
    for _ in range(2):
        assert rl.value_iteration() == ref.value_iteration()
        np.testing.assert_array_equal(value.parameters[0], ref.value_function.parameters[0])
    assert value.vertex_values is leaf and leaf.data_ptr() == ptr and leaf.is_leaf
    rl.optimize_value_function()
    ref.optimize_value_function()
    np.testing.assert_array_equal(value.parameters[0], ref.value_function.parameters[0])
    rl.discrete_policy_optimization(np.linspace(-1, 1, 5)[:, None])
    ref.discrete_policy_optimization(np.linspace(-1, 1, 5)[:, None])
    assert policy.vertex_values is pleaf
    np.testing.assert_array_equal(policy.parameters[0], ref.policy.parameters[0])


def test_lyapunov_safe_set_follows_vertex_steps():
    grid = sl.GridWorld([[-1, 1], [-1, 1]], [21, 21])
    vtri = sl.Triangulation(grid, np.sum(grid.all_points ** 2, axis=1, keepdims=True), project=True)
    dyn = sl.LinearSystem((0.5 * np.eye(2), np.zeros((2, 1))))
    policy = sl.LinearSystem((np.zeros((1, 2)),))
    initial = np.zeros(grid.nindex, dtype=bool)
    initial[grid.nindex // 2] = True
    lyap = sl.Lyapunov(grid, vtri, dyn, 1.0, 1.0, 1e-4, policy, initial)
    lyap.update_safe_set()
    first = lyap.safe_set.copy()
    leaf = vtri.vertex_values
    with torch.no_grad():                     # V -> -V: nothing decreases any more
        leaf.mul_(-1.0)
    lyap.update_values()
    lyap.update_safe_set()
    assert first.sum() > 1 and lyap.safe_set.sum() < first.sum()
    np.testing.assert_array_equal(np.ravel(lyap.values), vtri(grid.all_points).ravel())
    assert np.ravel(lyap.values).max() < 1e-12              # -V: the origin up to rounding


def test_write_between_forward_and_backward_raises():
    disc = sl.GridWorld([[-1, 1], [-1, 1]], [5, 5])
    tri = sl.Triangulation(disc, np.ones((disc.nindex, 1)), project=True)
    leaf = tri.vertex_values
    y = tri.torch(torch.zeros((3, 2), dtype=T64, device=CUDA)).sum()
    tri.parameters = np.zeros((disc.nindex, 1))              # in place: the leaf is handed out
    assert tri.vertex_values is leaf and not leaf.detach().any()
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        y.backward()
    y = sl.Saturation(tri, -1, 1).torch(torch.zeros((3, 2), dtype=T64, device=CUDA)).sum()
    with torch.no_grad():
        leaf.add_(0.1)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        y.backward()
    y = tri.torch(torch.zeros((3, 2), dtype=T64, device=CUDA)).sum()
    with pytest.raises(RuntimeError):
        torch.autograd.grad(torch.autograd.grad(y, leaf, create_graph=True)[0].sum(), leaf)
