"""The oracle against the reference's OWN known-answer tests (SURVEY.md section 8c).

Each test names the reference test it transcribes (paths relative to
the upstream safe_learning/tests).  These pin the numpy restatement before it
is trusted as the checker for the CUDA path.
"""
import numpy as np
import pytest
from numpy.testing import assert_allclose, assert_equal

import oracle as O


def test_gp_golden_vector():
    """test_functions.py:237-261 (Testgpflow.test_new_data): RBF(2) defaults, noise 1, beta 2."""
    x = np.array([[1, 0], [0, 1]], dtype=float)
    y = np.array([[0], [1]], dtype=float)
    gp = O.GPRCached(x, y, O.RBF(2), noise_variance=1.0)
    ufun = O.GaussianProcess(gp)
    ufun.add_data_point(np.array([[1.2, 2.3]]), np.array([[2.4]]))
    assert_allclose(ufun.X, np.array([[1, 0], [0, 1], [1.2, 2.3]]))
    assert_allclose(ufun.Y, np.array([[0], [1], [2.4]]))
    a1, b1 = ufun(np.array([[0.9, 0.1], [3., 2]]))
    assert_allclose(a1, np.array([[0.16371139], [0.22048311]]))
    assert_allclose(b1, np.array([[1.37678679], [1.98183191]]))


def test_gp_input_concatenation():
    """test_functions.py:216-235: GaussianProcess(x) == GaussianProcess(x[:, 0], x[:, 1])."""
    gp = O.GPRCached(np.array([[1, 0], [0, 1.]]), np.array([[0], [1.]]), O.RBF(2))
    ufun = O.GaussianProcess(gp, beta=3.0)
    pts = np.array([[0.9, 0.1], [3., 2]])
    m1, e1 = ufun(pts)
    m2, e2 = ufun(pts[:, [0]], pts[:, [1]])
    assert_allclose(m1, m2)
    assert_allclose(e1, e2)


def test_gp_cached_equals_uncached_algebra():
    """test_functions.py:164-199: cached predict == textbook (uncached gpflow GPR) posterior,
    including scale != 1 (functions.py:399-405, :438-456)."""
    rng = np.random.default_rng(0)
    X = rng.uniform(-1, 1, (12, 3))
    Y = rng.normal(size=(12, 1))
    kern = O.RBF(3, variance=0.7, lengthscales=[0.8, 1.1, 1.4])
    xs = rng.uniform(-1, 1, (5, 3))
    K = kern.K(X) + 0.01 * np.eye(12)
    mean_ref = kern.K(xs, X) @ np.linalg.solve(K, Y)
    var_ref = kern.Kdiag(xs) - np.einsum('ij,ji->i', kern.K(xs, X), np.linalg.solve(K, kern.K(X, xs)))
    for scale in (1.0, 3.5):
        gp = O.GPRCached(X, Y, kern, noise_variance=0.01, scale=scale)
        m, v = gp.build_predict(xs)
        assert_allclose(m, mean_ref, rtol=1e-9)
        assert_allclose(v[:, 0], var_ref, rtol=1e-7)


def test_quadratic_function():
    """test_functions.py:264-282."""
    points = np.array([[0, 0], [0, 1], [1, 0], [1, 1]], dtype=float)
    quad = O.QuadraticFunction(np.array([[1., 0.1], [0.2, 2.]]))
    assert_allclose(quad(points), np.array([[0., 2., 1., 3.3]]).T)


def test_gridworld_round_trips():
    """test_functions.py:313-367 (TestGridworld)."""
    grid = O.GridWorld([[-1.1, 1.5], [2.2, 2.4]], [7, 8])
    with pytest.raises(O.DimensionError):
        grid._check_dimensions(np.array([[1, 2, 3]]))
    with pytest.raises(O.DimensionError):
        grid._check_dimensions(np.array([[1]]))
    idx = np.arange(grid.nindex)
    states = grid.index_to_state(idx)
    assert_equal(idx, grid.state_to_index(states))
    assert_equal(states, grid.all_points)           # linspace grid == ijk*unit+offset bitwise here
    rect = np.arange(grid.nrectangles)
    rstates = grid.rectangle_to_state(rect)
    assert_equal(rect, grid.state_to_rectangle(rstates + grid.unit_maxes / 2))
    assert_equal(grid.state_to_rectangle(100 * np.ones((1, 2))), grid.nrectangles - 1)
    assert_equal(grid.state_to_rectangle(-100 * np.ones((1, 2))), 0)
    assert_equal(grid.rectangle_corner_index(rect), grid.state_to_index(rstates))
    assert_equal(grid.state_to_index(np.array([[-1.2, 2.]])), 0)
    assert_equal(O.GridWorld([[1, 2], [3, 4]], 2).num_points, np.array([2, 2]))
    g1 = O.GridWorld([[0, 1]], 3)
    test = np.array([[0.1, 0.4, 0.9]]).T
    assert_allclose(g1.state_to_index(test), np.array([0, 1, 2]))
    assert_allclose(g1.state_to_rectangle(test), np.array([0, 0, 1]))
    assert_allclose(g1.rectangle_to_state(np.array([0, 0, 1])), np.array([0, 0, 1])[:, None] * 0.5)
    with pytest.raises(O.DimensionError):
        O.GridWorld([[0, 1]], 1)


def _lyap_1d(eps):
    grid = O.GridWorld([[-1, 1]], 3)
    lyap_fun = O.QuadraticFunction(np.array([[1.0]]))        # sum(x^2, keep_dims)
    policy = O.LinearSystem(np.array([[-.1]]))                # lambda x: -.1 * x
    dynamics = O.LinearSystem(np.array([[1, 1.]]))
    return O.Lyapunov(grid, lyap_fun, dynamics, 0.4, 0.3, eps, policy, initial_set=[1])


def test_update_safe_set_known_answers():
    """test_lyapunov.py:48-74 (TestLyapunov.test_update)."""
    lyap = _lyap_1d(0.5)
    lyap.update_safe_set()
    assert_equal(lyap.safe_set, np.array([False, True, False]))
    assert lyap.c_max == 0.0
    lyap = _lyap_1d(0.0)
    lyap.update_safe_set()
    assert_equal(lyap.safe_set, np.ones(3, dtype=bool))
    assert lyap.c_max == 1.0        # the -1 index quirk (SURVEY Q4)


def test_safe_set_init():
    """test_lyapunov.py:24-46."""
    grid = O.GridWorld([[0, 1], [0, 1]], 3)
    lyap_fun = O.QuadraticFunction(np.eye(2))
    dynamics = O.LinearSystem(np.array([[1, 0.01], [0., 1.]]))
    policy = O.LinearSystem(np.zeros((2, 2)))
    O.Lyapunov(grid, lyap_fun, lambda x, u: dynamics(x), 0.4, 0.3, 0.5, policy)
    lyap = O.Lyapunov(grid, lyap_fun, lambda x, u: dynamics(x), 0.4, 0.3, 0.5, policy,
                      initial_set=[1, 3])
    assert_equal(lyap.safe_set,
                 np.array([False, True, False, True, False, False, False, False, False]))


def test_dlqr_golden():
    """test_utilities.py:17-28: scalar system, k = 0.618..., p = 1.618... (golden ratio)."""
    k, p = O.dlqr(1., 1., 1., 1.)
    assert_allclose(k, 0.5 * (np.sqrt(5) - 1), rtol=1e-10)
    assert_allclose(p, 0.5 * (np.sqrt(5) + 1), rtol=1e-10)


def test_future_values_r_plus_gamma_v():
    """test_rl.py:145-172 (mock plumbing): future_values == rewards + gamma * V(dynamics)."""
    grid = O.GridWorld([[-1, 1]], 5)
    vf = O.Triangulation(grid, np.arange(5.0)[:, None] ** 2, project=True)
    dynamics = O.LinearSystem(np.array([[0.9, 0.1]]))
    reward = O.QuadraticFunction(-np.eye(2))
    policy = O.LinearSystem(np.array([[-0.5]]))
    rl = O.PolicyIteration(policy, dynamics, reward, vf, gamma=0.9)
    states = grid.all_points
    u = policy(states)
    expect = reward(states, u) + 0.9 * vf(dynamics(states, u))
    assert_allclose(rl.future_values(states), expect, rtol=0, atol=0)


def test_prefix_rule_matches_batch_loop():
    """SURVEY Q1/Q4: the sort-free closed form == the batch loop as written (random ties,
    random batch sizes, random initial sets)."""
    rng = np.random.default_rng(7)
    old = O.config.gp_batch_size
    try:
        for _ in range(300):
            n = int(rng.integers(2, 40))
            grid = O.GridWorld([[-1, 1]], n)
            values = rng.integers(0, 6, n).astype(float)
            neg = rng.random(n) < 0.8
            init = rng.random(n) < 0.2
            lyap = O.Lyapunov(grid, lambda x: np.zeros((len(x), 1)), None, 0., 0., 0.,
                              None, initial_set=init)
            lyap.values = values
            lyap.negative = lambda states, g=grid, nn=neg: nn[g.state_to_index(states)]
            O.config.gp_batch_size = int(rng.integers(1, 24))
            lyap.update_safe_set()
            safe, p = O.prefix_rule(values, neg | init, init)
            assert_equal(lyap.safe_set, safe)
    finally:
        O.config.gp_batch_size = old


def test_adaptive_closed_form_matches_batch_loop():
    """The adaptive branch (lyapunov.py:540-582) of the oracle's batch loop, with the refined check
    evaluated on the mesh and known-safe cells skipped, equals the closed form the CUDA path uses:
    ok = negative | initial | (2 <= n_req <= R and refined check) followed by the prefix rule, with
    N(x) = 1 / n_req / 0.  Random labels, refinement demands, ties and batch sizes."""
    rng = np.random.default_rng(11)
    old = O.config.gp_batch_size
    try:
        for _ in range(300):
            n = int(rng.integers(2, 40))
            R = int(rng.integers(2, 6))
            grid = O.GridWorld([[-1, 1]], n)
            values = rng.integers(0, 6, n).astype(float)
            neg = rng.random(n) < 0.6
            init = rng.random(n) < 0.15
            n_req = np.where(neg, 1, rng.integers(0, 8, n))
            fine = rng.random(n) < 0.7                      # outcome of the refined mesh check
            lyap = O.Lyapunov(grid, lambda x: np.zeros((len(x), 1)), None, 0., 0., 0.,
                              None, initial_set=init, adaptive=True)
            lyap.values = values
            index = grid.state_to_index
            lyap.negative = lambda states: neg[index(states)]
            lyap.required_refinement = lambda states, sf=1.: n_req[index(states)].astype(float)
            lyap.refined_negative = lambda states, refinement, mode="mesh", known_safe=None: \
                np.where(known_safe, True, fine[index(states)] & (refinement >= 2))   # n = 1: plain check
            O.config.gp_batch_size = int(rng.integers(1, 24))
            lyap.update_safe_set(max_refinement=R)
            ok = neg | init | ((n_req >= 2) & (n_req <= R) & fine)
            safe, p = O.prefix_rule(values, ok, init)
            assert_equal(lyap.safe_set, safe)
            expect = np.where(safe, np.where(neg | init, 1, n_req), 0)
            assert_equal(lyap._refinement, expect)
            # c_max index arithmetic (lyapunov.py:586-590): when nothing fails it depends on
            # whether the LAST batch holds a cell that only the refinement verified
            order = O.stable_value_order(values)
            if p < n:
                position = p - 1
            else:
                batch = O.config.gp_batch_size
                start = ((n - 1) // batch) * batch
                rescued = ~(neg | init)[order[start:]]
                position = n - 1 if rescued.any() else start - 1
            assert lyap.c_max == values[order[position]]
    finally:
        O.config.gp_batch_size = old


def test_triangulation_known_answers():
    """Upstream safe_learning/tests/test_functions.py:457-655 (find_simplex, values,
    projection, three dimensions, gradient, 1-D) restated against the oracle's Triangulation."""
    # find_simplex :457-499
    limits, num = [[-1, 1], [-1, 2]], [3, 7]
    tri = O.Triangulation(O.GridWorld(limits, num))
    assert tri.discretization.nrectangles == 12 and tri.input_dim == 2
    assert tri.nsimplex_unit * tri.discretization.nrectangles == 24
    assert_equal(tri.discretization.offset, np.array([-1, -1]))
    assert_equal(tri.discretization.unit_maxes, np.array([2, 3]) / (np.array(num) - 1))
    lower = int(np.squeeze(tri.triangulation.find_simplex(np.array([0, 0]))))
    upper = 1 - lower
    pts = np.array([[0, 0], [0.9, 0.45], [1.1, 0], [1.9, 2.9]]) + np.array(limits)[:, 0]
    ids = tri.find_simplex(pts)
    assert_equal(ids, np.array([lower, upper, 6 * 2 + lower, 11 * 2 + upper]))
    assert_equal(np.sort(tri.simplices(ids), axis=1),
                 np.array([[0, 1, 7], [1, 7, 8], [7, 8, 14], [13, 19, 20]]))
    assert_equal(tri.find_simplex(np.array([[-100., -100.]])), lower)
    assert_equal(tri.find_simplex(np.array([[100., 100.]])), 24 - 1 - lower)

    # values and projection :501-546
    eps = 1e-10
    tri = O.Triangulation(O.GridWorld([[0, 1], [0, 1]], [2, 2]))
    nodes = tri.discretization.state_to_index(np.array([[0, 0], [1, 0], [0, 1]]))
    pts = np.array([[0, 0], [1 - eps, 0], [0, 1 - eps], [0.5 - eps, 0.5 - eps], [0, 0.5], [0.5, 0]])
    vals = np.random.default_rng(0).random(tri.nindex)
    tri.parameters = vals
    want = np.array([vals[nodes[0]], vals[nodes[1]], vals[nodes[2]],
                     0.5 * (vals[nodes[1]] + vals[nodes[2]]), 0.5 * (vals[nodes[0]] + vals[nodes[2]]),
                     0.5 * (vals[nodes[0]] + vals[nodes[1]])])[:, None]
    assert_allclose(tri(pts), want, atol=1e-7)
    tri.parameters = np.array([0, 1, 1, 1])
    assert_allclose(tri(np.array([[-0.5, -0.5]])), np.array([[-1]]))
    tri.project = True
    assert_allclose(tri(np.array([[-0.5, -0.5]])), np.array([[0]]))

    # three dimensions :548-580
    tri = O.Triangulation(O.GridWorld([[0, 1]] * 3, [2] * 3))
    assert tri.input_dim == 3 and tri.discretization.nrectangles == 1 and tri.nsimplex_unit == 6
    corners = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [0, 1, 1], [1, 1, 0], [1, 0, 1],
                        [1, 1, 1]], dtype=float)
    tri.parameters = np.sum(tri.discretization.index_to_state(np.arange(8)), axis=1) / 3
    pts = np.vstack((corners, np.array([[0, 0, 0.5], [0.5, 0, 0], [0, 0.5, 0], [0.5, 0.5, 0.5]])))
    want = np.hstack((np.sum(corners, axis=1) / 3, np.array([1 / 6, 1 / 6, 1 / 6, 1 / 2])))
    assert_allclose(tri(pts), want[:, None], atol=1e-5)

    # gradient :582-624
    tri = O.Triangulation(O.GridWorld([[0, 1], [0, 1]], [2, 2]))
    nodes = tri.discretization.state_to_index(np.array([[0, 0], [1, 0], [0, 1], [1, 1]]))
    vals = np.zeros(tri.nindex)
    vals[nodes] = [1, 2, 3, 1]
    tri.parameters = vals
    assert_allclose(tri.gradient(np.array([[0.01, 0.01], [0.99, 0.99]])), np.array([[1, 2], [-2, -1]]))

    # 1-D :626-655
    tri = O.Triangulation(O.GridWorld([[0, 1]], 3), [0, 0.5, 0])
    pts = np.array([[0, 0.2, 0.5, 0.6, 0.9, 1.]]).T
    assert_equal(tri.find_simplex(pts), np.array([0, 0, 1, 1, 1, 1]))
    assert_allclose(tri(pts), np.array([0, 0.2, 0.5, 0.4, 0.1, 0])[:, None])
    assert_allclose(tri.gradient(pts), np.array([1, 1, -1, -1, -1, -1])[:, None])


def test_unique_rows_and_perturb_actions():
    """tests/test_utilities.py:86-91 (unique_rows) and the action perturbation grid of
    lyapunov.py:609-651."""
    a = np.array([[1, 1], [1, 2], [1, 3], [1, 2], [1, 3], [1, 4], [2, 3]])
    assert_equal(O.unique_rows(a), np.array([[1, 1], [1, 2], [1, 3], [1, 4], [2, 3]]))
    states = np.array([[0., 1.], [2., 3.]])
    actions = np.array([[0.5], [-0.5]])
    out = O.perturb_actions(states, actions, np.array([[-1.], [0.], [1.]]), limits=np.array([[-1., 1.]]))
    want = np.array([[0., 1., -0.5], [0., 1., 0.5], [0., 1., 1.],
                     [2., 3., -1.], [2., 3., -0.5], [2., 3., 0.5]])
    # row order is np.unique's on the raw bytes (utilities.py:509-516), compare as a set of rows
    assert_equal(out[np.lexsort(out.T[::-1])], want)
    dup = O.perturb_actions(states, actions, np.array([[2.], [3.]]), limits=np.array([[-1., 1.]]))
    assert_equal(dup[np.lexsort(dup.T[::-1])], np.array([[0., 1., 1.], [2., 3., 1.]]))


def test_smallest_boundary_value():
    """tests/test_lyapunov.py:77-84."""
    fun = lambda x: 2 * np.sum(np.abs(x), axis=1)  # noqa: E731
    assert O.smallest_boundary_value(fun, O.GridWorld([[-1.5, 1], [-1, 1.5]], [3, 3])) == 2.5
