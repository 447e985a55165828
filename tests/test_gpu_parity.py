"""GPU parity tests: the CUDA path (through the Python API -> ctypes -> C ABI) against the
CPU oracle on the same seeded inputs.  Bar (BASELINE.json north_star): safe-set membership
bit-exact, GP posterior and V within 1e-5 relative; the cheap element-wise pieces (grid
coordinates, linear / quadratic / triangulation values, thresholds) are bit-exact.
"""
import numpy as np
import pytest
from numpy.testing import assert_allclose, assert_array_equal

import bench_workloads as W
import oracle as O

pytestmark = pytest.mark.gpu

RTOL = 1e-5   # GP posterior / V tolerance stated by north_star


@pytest.fixture(scope="module")
def sl():
    import __graft_entry__
    __graft_entry__.build()
    import safe_learning_b200 as sl
    return sl


def _assert_negative_parity(gpu, cpu, details):
    """`negative` must agree everywhere except (reported, expected none) points whose margin
    |decrease - threshold| is below rounding noise of the GP contraction."""
    neg_gpu = details["negative"]
    states = cpu.discretization.all_points
    actions = cpu.policy(states)
    nxt = cpu.dynamics(states, actions)
    dec = cpu.v_decrease_bound(states, nxt).ravel()
    thr = np.broadcast_to(cpu.threshold(states), (len(states), 1)).ravel()
    with np.errstate(invalid="ignore"):
        neg_cpu = dec < thr
    margin = np.abs(dec - thr)
    scale = np.maximum(np.abs(dec), np.abs(thr))
    mismatch = neg_gpu != neg_cpu
    outside = mismatch & ~(margin <= 1e-9 * np.maximum(scale, 1e-300))
    assert not outside.any(), "negative differs at %d points outside the rounding margin" \
        % outside.sum()
    assert mismatch.sum() == 0, "%d borderline points flipped" % mismatch.sum()
    assert_allclose(details["decrease"], dec, rtol=RTOL, atol=1e-12)
    assert_array_equal(details["threshold"], thr)


def _sweep_details(lyap):
    neg, det = lyap.compute_negative(want_details=True)
    out = {k: v.cpu().numpy() for k, v in det.items()}
    out["negative"] = neg.cpu().numpy().astype(bool)
    return out


# ------------------------------------------------------------------ reference known answers
def test_reference_update_known_answers(sl):
    """Upstream safe_learning/tests/test_lyapunov.py:48-74 through the product API."""
    def make(eps):
        grid = sl.GridWorld([[-1, 1]], 3)
        return sl.Lyapunov(grid, sl.QuadraticFunction(np.array([[1.0]])),
                           sl.LinearSystem(np.array([[1, 1.]])), 0.4, 0.3, eps,
                           sl.LinearSystem(np.array([[-.1]])), initial_set=[1])
    lyap = make(0.5)
    lyap.update_safe_set()
    assert_array_equal(lyap.safe_set, np.array([False, True, False]))
    assert lyap.feed_dict[lyap.c_max] == 0.0
    lyap = make(0.0)
    lyap.update_safe_set()
    assert_array_equal(lyap.safe_set, np.ones(3, dtype=bool))
    assert lyap.feed_dict[lyap.c_max] == 1.0


def test_reference_safe_set_init(sl):
    """test_lyapunov.py:24-46."""
    grid = sl.GridWorld([[0, 1], [0, 1]], 3)
    dyn = sl.LinearSystem(np.array([[1, 0.01, 0, 0], [0., 1., 0, 0]]))
    lyap = sl.Lyapunov(grid, sl.QuadraticFunction(np.eye(2)), dyn, 0.4, 0.3, 0.5,
                       sl.LinearSystem(np.zeros((2, 2))), initial_set=[1, 3])
    assert_array_equal(lyap.safe_set, np.array([False, True, False, True, False, False, False,
                                                False, False]))


def test_reference_gp_golden_vector(sl):
    """test_functions.py:237-261 on the GPU."""
    gp = sl.GPRCached(np.array([[1, 0], [0, 1.]]), np.array([[0], [1.]]), sl.RBF(2))
    ufun = sl.GaussianProcess(gp)
    ufun.add_data_point(np.array([[1.2, 2.3]]), np.array([[2.4]]))
    a1, b1 = ufun(np.array([[0.9, 0.1], [3., 2]]))
    assert_allclose(a1, np.array([[0.16371139], [0.22048311]]))
    assert_allclose(b1, np.array([[1.37678679], [1.98183191]]))
    m2, e2 = ufun(np.array([[0.9], [3.]]), np.array([[0.1], [2.]]))     # :216-235
    assert_array_equal(a1, m2)
    assert_array_equal(b1, e2)


def test_reference_quadratic_and_grid(sl):
    """test_functions.py:264-282 and :313-367."""
    quad = sl.QuadraticFunction(np.array([[1., 0.1], [0.2, 2.]]))
    pts = np.array([[0, 0], [0, 1], [1, 0], [1, 1]], dtype=float)
    assert_allclose(quad(pts), np.array([[0., 2., 1., 3.3]]).T)
    grid = sl.GridWorld([[-1.1, 1.5], [2.2, 2.4]], [7, 8])
    idx = np.arange(grid.nindex)
    assert_array_equal(idx, grid.state_to_index(grid.index_to_state(idx)))
    rect = np.arange(grid.nrectangles)
    assert_array_equal(rect, grid.state_to_rectangle(grid.rectangle_to_state(rect)
                                                     + grid.unit_maxes / 2))
    with pytest.raises(sl.DimensionError):
        sl.GridWorld([[0, 1]], 1)


# ------------------------------------------------------------------ element-wise pieces, bit-exact
def test_index_to_state_bit_exact(sl):
    import torch
    from safe_learning_b200 import _device as dev, _native as nat
    lib = nat.load()
    for limits, num in ([[[-1.1, 1.5], [2.2, 2.4]], [7, 8]], [[[-1, 1]] * 3, [5, 9, 4]],
                        [[[-0.3, 0.7]], [101]]):
        g_gpu, g_cpu = sl.GridWorld(limits, num), O.GridWorld(limits, num)
        out = dev.empty((g_gpu.nindex, g_gpu.ndim))
        nat.check(lib.slb_index_to_state(dev.stream(), g_gpu.descriptor(), 0, g_gpu.nindex,
                                         out.data_ptr()), "index_to_state")
        assert_array_equal(out.cpu().numpy(), g_cpu.index_to_state(np.arange(g_cpu.nindex)))
        assert_array_equal(out.cpu().numpy(), g_cpu.all_points)


def test_small_functions_bit_exact(sl):
    rng = np.random.default_rng(3)
    x = rng.uniform(-2, 2, (257, 3))
    A = rng.normal(size=(2, 3))
    P = rng.normal(size=(3, 3))
    assert_array_equal(sl.LinearSystem(A)(x), O.LinearSystem(A)(x))
    assert_array_equal(sl.QuadraticFunction(P)(x), O.QuadraticFunction(P)(x))
    assert_array_equal(sl.Saturation(sl.LinearSystem(A), -0.5, 0.7)(x),
                       O.Saturation(O.LinearSystem(A), -0.5, 0.7)(x))
    assert_array_equal(abs(sl.LinearSystem(A))(x), O.AbsFunction(O.LinearSystem(A))(x))
    assert_array_equal(sl.Norm1Function(sl.LinearSystem(A))(x),
                       O.Norm1Function(O.LinearSystem(A))(x))
    assert_array_equal((-sl.QuadraticFunction(P))(x), O.ScaledFunction(O.QuadraticFunction(P), -1)(x))
    assert_array_equal(sl.LinearSystem((A[:, :2], A[:, 2:]))(x[:, :2], x[:, 2:]),
                       O.LinearSystem(A)(x))


TRI_LIMITS = [[-1.0, 1.5], [0.0, 2.0], [-0.5, 0.5], [-1.2, 0.8], [0.3, 1.1], [-2.0, -0.5]]


@pytest.mark.parametrize("dims,project", [(1, False), (2, False), (2, True), (3, True), (4, True), (5, True),
                                          (6, True)])
def test_triangulation_vs_oracle(sl, dims, project):
    """functions.py:1103-1158, 1473-1499; reference tests test_functions.py:457-701."""
    rng = np.random.default_rng(dims)
    limits = TRI_LIMITS[:dims]
    num = [5, 4, 3, 3, 3, 2][:dims]
    g_gpu, g_cpu = sl.GridWorld(limits, num), O.GridWorld(limits, num)
    vals = rng.normal(size=(g_cpu.nindex, 2))
    t_gpu = sl.Triangulation(g_gpu, vals, project=project)
    t_cpu = O.Triangulation(g_cpu, vals, project=project)
    lo, hi = np.array(limits)[:, 0], np.array(limits)[:, 1]
    span = 0.3 * (hi - lo)
    pts = rng.uniform(lo - span, hi + span, size=(2000, dims))
    # vertices: shared-face lookups.  From d = 5 on, exact-vertex queries hit the Q6 rounding (DESIGN.md
    # §3.2) where the oracle's batch walk and the library's first fit pick different extrapolating
    # simplices; tests/test_gpu_triangulation_shapes.py holds them to the exact reference instead
    if dims <= 4:
        pts = np.vstack((pts, g_cpu.all_points))
    got = t_gpu(pts)
    # A non-projected query outside the grid in EVERY coordinate is clipped onto a unit-cell
    # corner where several simplices meet; scipy's find_simplex walks from the previous query's
    # simplex, so the reference's (discontinuous) extrapolation there depends on batch order.
    # The build pins Qhull's answer for an isolated query: compare those one point at a time.
    corner = np.all((pts < lo) | (pts > hi), axis=1) & (dims > 1) & (not project)
    assert_allclose(got[~corner], t_cpu(pts)[~corner], rtol=1e-12, atol=1e-12)
    for i in np.nonzero(corner)[0][:60]:
        assert_allclose(got[i], t_cpu(pts[i:i + 1])[0], rtol=1e-12, atol=1e-12)
    inside = rng.uniform(lo, hi, size=(500, dims))
    assert_allclose(t_gpu(inside), t_cpu(inside), rtol=1e-13, atol=1e-13)


@pytest.mark.parametrize("dims", [1, 2, 3, 4, 5, 6])
def test_triangulation_gradient_vs_oracle(sl, dims):
    """Triangulation.gradient (functions.py:1260-1326) and max |.| over it -- the Lipschitz lambda
    of examples/inverted_pendulum.ipynb cell 14 -- incl. queries on vertices and outside."""
    rng = np.random.default_rng(dims)
    limits = TRI_LIMITS[:dims]
    num = [7, 5, 4, 3, 3, 2][:dims]
    g_gpu, g_cpu = sl.GridWorld(limits, num), O.GridWorld(limits, num)
    vals = rng.normal(size=(g_cpu.nindex, 1))
    lo, hi = g_cpu.limits[:, 0], g_cpu.limits[:, 1]
    pts = rng.uniform(lo, hi, (400, dims))
    for project in (False, True):
        t_gpu = sl.Triangulation(g_gpu, vals, project=project)
        t_cpu = O.Triangulation(g_cpu, vals, project=project)
        assert_allclose(t_gpu.gradient(pts), t_cpu.gradient(pts), rtol=1e-12, atol=1e-13)
        lv_gpu = sl.MaxAbsFunction(t_gpu.gradient_function())
        lv_cpu = O.MaxAbsFunction(t_cpu.gradient_function())
        assert_array_equal(lv_gpu(pts), np.max(np.abs(t_gpu.gradient(pts)), axis=1, keepdims=True))
        assert_allclose(lv_gpu(pts), lv_cpu(pts), rtol=1e-12, atol=1e-13)
    with pytest.raises(sl.DimensionError):
        sl.Triangulation(g_gpu, rng.normal(size=(g_cpu.nindex, 2))).gradient(pts)


def test_constant_callable_lipschitz_dynamics(sl):
    """The notebooks pass L_f as `lambda x: const` (lyapunov_function_learning.ipynb cell 13)."""
    par = W.make_pendulum(num_points=[13, 11], M=40)
    a, b = W.build_product(par), W.build_product(par)
    const = float(par["L_dyn"])
    b._lipschitz_dynamics = lambda x: const
    a.update_safe_set()
    b.update_safe_set()
    assert_array_equal(a.safe_set, b.safe_set)


def test_state_dependent_lipschitz_dynamics_vs_oracle(sl):
    """lyapunov.py:227-244, 287: L_f(x) as an arbitrary Python callable (tabulated per grid index,
    ADVICE r01: a callable that merely coincides at a few probe points must not pass as constant)
    and as a fused Function object; threshold bit-exact, safe set identical to the oracle."""
    par = W.make_pendulum(num_points=[29, 23], M=60, tau_scale=1 / 40.)
    lf = lambda x: 0.5 + np.abs(x[:, [1]]) * (np.abs(x[:, [0]]) < 0.5)   # noqa: E731  even, flat at the corners
    gpu, cpu = W.build_product(par), W.build_oracle(par)
    gpu._lipschitz_dynamics = lf
    cpu._lipschitz_dynamics = lf
    det = _sweep_details(gpu)
    states = cpu.discretization.all_points
    assert_array_equal(det["threshold"], cpu.threshold(states).ravel())
    _assert_negative_parity(gpu, cpu, det)
    gpu.update_safe_set()
    cpu.update_safe_set()
    assert_array_equal(gpu.safe_set, cpu.safe_set)
    assert gpu.feed_dict[gpu.c_max] == cpu.c_max
    # the same dependence as a fused function object: L_f(x) = |x A^T| 1-norm
    A = np.array([[0.3, -0.2], [0.1, 0.4]])
    gpu2, cpu2 = W.build_product(par), W.build_oracle(par)
    gpu2._lipschitz_dynamics = sl.Norm1Function(sl.LinearSystem(A))
    cpu2._lipschitz_dynamics = O.Norm1Function(O.LinearSystem(A))
    det2 = _sweep_details(gpu2)
    assert_array_equal(det2["threshold"], cpu2.threshold(states).ravel())
    gpu2.update_safe_set()
    cpu2.update_safe_set()
    assert_array_equal(gpu2.safe_set, cpu2.safe_set)


def test_arbitrary_python_callables_vs_oracle(sl):
    """lyapunov.py:227-263 and lyapunov_function_learning.ipynb cells 13-19: V, policy, L_V and
    L_f given as plain Python callables on numpy arrays (the composed path: GP posterior on the
    GPU, the callables on the host), against the oracle running the same lambdas and against the
    fused path running the equivalent Function objects."""
    par = W.make_pendulum(num_points=[41, 37], M=90, tau_scale=1 / 40.)
    P, K = par["P"], par["K"]
    v_fn = lambda x: np.sum(x.dot(P) * x, axis=1, keepdims=True)              # noqa: E731
    pi_fn = lambda x: np.clip(x.dot(-K.T), -1., 1.)                            # noqa: E731
    lv_fn = lambda x: np.abs(x.dot((2 * P).T))                                 # noqa: E731  two columns -> 1-norm in threshold
    lf_fn = lambda x: np.full((len(x), 1), par["L_dyn"])                       # noqa: E731
    fused, cpu = W.build_product(par), W.build_oracle(par)
    gpu = sl.Lyapunov(fused.discretization, v_fn, fused.dynamics, lf_fn, lv_fn, par["tau"], pi_fn,
                      initial_set=par["initial"])
    ref = O.Lyapunov(cpu.discretization, v_fn, cpu.dynamics, lf_fn, lv_fn, par["tau"], pi_fn,
                     initial_set=par["initial"])
    assert gpu._is_composed() and not fused._is_composed()
    assert_array_equal(gpu.values, ref.values)
    det = _sweep_details(gpu)
    _assert_negative_parity(gpu, ref, det)
    for lyap in (gpu, ref, fused, cpu):
        lyap.update_safe_set()
    assert par["initial"].sum() < ref.safe_set.sum() < ref.safe_set.size
    assert_array_equal(gpu.safe_set, ref.safe_set)
    assert gpu.feed_dict[gpu.c_max] == ref.c_max
    # the lambdas restate the Function objects: same safe set as the fused sweep
    assert_array_equal(gpu.safe_set, fused.safe_set)
    assert_array_equal(gpu.safe_set, cpu.safe_set)
    # only some members are callables: a lambda policy with fused V / L_V
    mixed = sl.Lyapunov(fused.discretization, fused.lyapunov_function, fused.dynamics,
                        par["L_dyn"], fused._lipschitz_lyapunov, par["tau"], pi_fn,
                        initial_set=par["initial"])
    mixed.update_safe_set()
    assert_array_equal(mixed.safe_set, cpu.safe_set)


def test_gp_cache_export_import_round_trip(sl):
    """FunctionStack.export_cache / import_cache (the host-buffer side of bench.py's end-to-end arm):
    the tables move into one device arena with a page-locked host mirror; wiping the arena and
    restoring it with one H2D copy reproduces the sweep; a refit invalidates the checkpoint."""
    import torch
    par = W.make_pendulum(num_points=[33, 31], M=70, tau_scale=1 / 40.)
    gpu, cpu = W.build_product(par), W.build_oracle(par)
    gpu.update_safe_set()
    cpu.update_safe_set()
    before = gpu.safe_set.copy()
    assert_array_equal(before, cpu.safe_set)
    cache = gpu.dynamics.export_cache(pinned=True)
    assert cache.valid() and cache.nbytes > 70 * 70 * 8
    gpu.update_safe_set()                       # descriptors rebuilt on the re-homed tables
    assert_array_equal(gpu.safe_set, before)
    cache.arena.zero_()
    copied = gpu.dynamics.import_cache(cache)
    assert copied == cache.nbytes
    gpu.update_safe_set()
    assert_array_equal(gpu.safe_set, before)
    assert gpu.feed_dict[gpu.c_max] == cpu.c_max
    gpu.dynamics.add_data_point(np.array([[0.1, -0.2, 0.3]]), np.array([[0.05, -0.02]]))
    gpu.update_safe_set()
    with pytest.raises(sl.functions.DimensionError):
        gpu.dynamics.import_cache(cache)


def test_initial_safe_set_edited_in_place(sl):
    """ADVICE r01: the reference re-reads ``initial_safe_set`` on every update_safe_set
    (lyapunov.py:504-506); an in-place edit of the same array must reach the device."""
    par = W.make_pendulum(num_points=[21, 17], M=40, tau_scale=0.0)
    gpu, cpu = W.build_product(par), W.build_oracle(par)
    for lyap in (gpu, cpu):
        lyap.initial_safe_set = par["initial"].copy()
    gpu.update_safe_set()
    cpu.update_safe_set()
    assert_array_equal(gpu.safe_set, cpu.safe_set)
    for lyap in (gpu, cpu):
        lyap.initial_safe_set[:5] = True          # same object, new content
        lyap.update_safe_set()
    assert_array_equal(gpu.safe_set, cpu.safe_set)
    assert gpu.safe_set[:5].all()
    for lyap in (gpu, cpu):
        lyap.initial_safe_set = None
        lyap.update_safe_set()
    assert_array_equal(gpu.safe_set, cpu.safe_set)


@pytest.fixture(params=["fp32 screening", "fp64 mean stage"])
def mean_stage(request):
    """Stage 1 of the decision filter: the fp32 screening kernel (default where V is quadratic) or
    the fp64 mean kernel (bit 2 of slb_debug_filter_stages forces it)."""
    from safe_learning_b200 import _native as nat
    lib = nat.load()
    lib.slb_debug_filter_stages(3 if request.param == "fp32 screening" else 7)
    yield request.param
    lib.slb_debug_filter_stages(3)


@pytest.mark.parametrize("tau_scale", [1.0, 1 / 8., 1 / 48., 0.0])
@pytest.mark.parametrize("M", [0, 1, 8, 40, 64, 65, 100, 200, 256])
def test_filtered_flags_equal_full_posterior(sl, M, tau_scale, mean_stage):
    """The decision filter (csrc/filter.cu) must reproduce the full posterior's flags bit for bit
    at every training-set size (M <= 64: the head bound is the whole posterior; M = 0: the prior)
    and in every regime of tau (all fail ... most pass), incl. the guard-band hand-over; with
    either first stage."""
    par = W.make_pendulum(num_points=[45, 37], M=max(M, 1), tau_scale=tau_scale, seed=M + 3)
    if M == 0:
        par["X"], par["Y"] = par["X"][:0], par["Y"][:0]
    gpu = W.build_product(par)
    assert gpu._filter_enabled(gpu.sweep_descriptor())
    gpu.reset_filter_stats()
    fast = gpu.compute_negative().cpu().numpy().copy()
    stats = gpu.filter_stats
    assert stats["points"] == gpu.discretization.nindex
    assert stats["prior"] + stats["head"] + stats["refined"] == stats["points"]
    gpu.filter = False
    full = gpu.compute_negative().cpu().numpy()
    assert_array_equal(fast, full)
    if M and tau_scale > 0:
        cpu = W.build_oracle(par)
        assert_array_equal(full.astype(bool), cpu.full_grid_negative())


@pytest.mark.parametrize("case", ["pendulum", "short lengthscales", "shared factor", "scaled targets",
                                  "large noise-free gammas"])
def test_screening_mean_error_is_within_its_certified_bound(sl, case):
    """The fp32 screening stage decides points from a mean it only knows to within a bound it
    computes (gp_mean_staged.cuh); slb_debug_screening_probe exposes mean and bound: the fp64
    posterior mean must lie inside the bound at every point, and the flags must equal the full
    posterior's in regimes where the bound is large."""
    import torch
    from safe_learning_b200 import _native as nat, _device as dev
    lib = nat.load()
    kw = dict(num_points=[61, 53], M=300, tau_scale=1 / 16., seed=7)
    if case == "shared factor":
        kw["shared_hypers"] = True
    if case == "scaled targets":
        kw["scale"] = 7.5
    if case == "large noise-free gammas":
        kw["noise_std"] = 2e-4
    par = W.make_pendulum(**kw)
    if case == "short lengthscales":
        # |z - centre| / lengthscale reaches ~7 inside a CTA: large exponents of the split-off factor
        # 2^(|zc|^2 / 2), argument errors of several thousand ulps -- all inside the computed bound
        par["lengthscales"] = [[0.2, 0.15, 0.4], [0.25, 0.12, 0.3]]
    gpu = W.build_product(par)
    cpu = W.build_oracle(par)
    desc = gpu.sweep_descriptor()
    if not gpu._filter_enabled(desc):
        pytest.skip("variance floor below the filter's limit for this case")
    n, D = gpu.discretization.nindex, 2
    mu = torch.zeros((n, D), dtype=torch.float64, device=dev.device())
    dm = torch.full((n, D), -1.0, dtype=torch.float64, device=dev.device())
    try:
        lib.slb_debug_screening_probe(mu.data_ptr(), dm.data_ptr())
        fast = gpu.compute_negative().cpu().numpy().copy()
        torch.cuda.synchronize()
    finally:
        lib.slb_debug_screening_probe(None, None)
    mu, dm = mu.cpu().numpy(), dm.cpu().numpy()
    assert (dm >= 0).all(), "the screening stage did not run"
    states = cpu.discretization.all_points
    mean64, _ = gpu.dynamics(states, cpu.policy(states))
    finite = np.isfinite(dm)
    assert finite.mean() > 0.25, "most points left to the fp64 stages: %g" % finite.mean()
    err = np.abs(mu - mean64)
    assert (err[finite] <= dm[finite]).all(), "fp32 mean outside its certified bound: max ratio %g" % (
        (err[finite] / dm[finite]).max())
    gpu.filter = False
    assert_array_equal(fast, gpu.compute_negative().cpu().numpy())


@pytest.mark.parametrize("split,label", [((0,), "64-point tiles"), ((1 << 40,), "32-point tiles")])
def test_refine_pass_tile_sizes(sl, split, label):
    """The refine pass of the filtered sweep picks its tile size from the list length; every tile
    size (forced through slb_debug_refine_split) must reproduce the full posterior's flags, with
    M across a panel boundary and a ragged list length."""
    from safe_learning_b200 import _native as nat
    lib = nat.load()
    try:
        lib.slb_debug_refine_split(*split)
        for M, num in ((300, [67, 59]), (40, [45, 37])):
            par = W.make_pendulum(num_points=num, M=M, tau_scale=1 / 64., seed=11)
            gpu = W.build_product(par)
            gpu.reset_filter_stats()
            fast = gpu.compute_negative().cpu().numpy().copy()
            assert gpu.filter_stats["refined"] > 20, label
            gpu.filter = False
            assert_array_equal(fast, gpu.compute_negative().cpu().numpy(), err_msg=label)
    finally:
        lib.slb_debug_refine_split(32 * 132)           # the library's default split


def test_pivoted_head_subset_matches_greedy_selection(sl):
    """slb_pivoted_subset (the head subset of the decision filter) against a numpy restatement of the
    pivoted Cholesky factorisation: same pivots in the same order; and the subset's variance bound
    is an upper bound of the full posterior variance at random points (what the filter relies on)."""
    import torch
    from safe_learning_b200 import _device as dev
    from safe_learning_b200.functions import GPRCached
    rng = np.random.default_rng(5)
    X = rng.uniform(-1, 1, (137, 3))
    K = np.exp(-0.5 * ((X[:, None, :] - X[None, :, :]) ** 2 / np.array([1.5, 1.2, 2.0]) ** 2).sum(-1))
    r = 64
    diag, low, ref = np.diag(K).copy(), np.zeros((len(X), r)), []
    for t in range(r):
        i = int(np.argmax(diag))
        ref.append(i)
        col = (K[i] - low[:, :t] @ low[i, :t]) / np.sqrt(diag[i])
        low[:, t] = col
        diag = diag - col * col
        diag[ref] = -np.inf
    picks = GPRCached._pivoted_subset(dev.to_device(K), r).cpu().numpy()
    assert sorted(set(picks.tolist())) == sorted(picks.tolist()) and len(picks) == r
    assert_array_equal(picks, np.array(ref))
    par = W.make_pendulum(num_points=[9, 9], M=137)
    gpu = W.build_product(par)
    gp = gpu.dynamics.functions[0].gaussian_process
    gp._ensure()
    fac = gp._factor
    assert fac.head_rows == 64
    z = rng.uniform(-1, 1, (200, 3))
    _, var = gpu.dynamics.functions[0].predict_device(z, want_var=True)
    Xh = fac.Xhead.cpu().numpy()
    zs = z / np.asarray(gp.kern.lengthscales)
    kz = gp.kern.variance * np.exp(-0.5 * ((Xh[:, None, :] - zs[None, :, :]) ** 2).sum(-1))
    a = fac.Whead.cpu().numpy().T[:64, :64] @ kz           # Whead[j, i] = L_S^-1[i, j]
    bound = gp.kern.variance - (a * a).sum(axis=0)
    assert (bound >= var.cpu().numpy()[:, 0] * (1 - 1e-9)).all()


def test_filter_is_not_used_below_the_variance_floor(sl):
    """With (almost) noise-free data the reference's negative-variance -> NaN -> unsafe corner is
    reachable; "auto" then keeps the full posterior."""
    par = W.make_pendulum(num_points=[9, 9], M=30)
    par["noise_variance"] = 1e-14
    gpu = W.build_product(par)
    assert gpu.dynamics.variance_floor() < 1e-9
    assert not gpu._filter_enabled(gpu.sweep_descriptor())
    gpu.filter = True
    assert gpu._filter_enabled(gpu.sweep_descriptor())


def test_adaptive_refinement_as_written_vs_oracle(sl):
    """refinement_mode="reference": the adaptive branch exactly as upstream evaluates it
    (lyapunov.py:457-481, 540-582), against the oracle's reference mode."""
    old = (sl.config.gp_batch_size, O.config.gp_batch_size)
    try:
        sl.config.gp_batch_size = O.config.gp_batch_size = 64
        for tau_scale, kwargs in ((1 / 30., dict(max_refinement=4, safety_factor=2.0)),
                                  (1 / 60., dict(max_refinement=12, safety_factor=4.0))):
            par = W.make_pendulum(num_points=[26, 21], M=90, tau_scale=tau_scale)
            pair = []
            for ns, kind in ((sl, "product"), (O, "oracle")):
                grid, dyn = W._build(ns, par, kind)
                policy = ns.Saturation(ns.LinearSystem(-par["K"]), -1., 1.)
                pair.append(ns.Lyapunov(grid, ns.QuadraticFunction(par["P"]), dyn, par["L_dyn"],
                                        ns.AbsFunction(ns.LinearSystem((2 * par["P"],))),
                                        par["tau"], policy, initial_set=par["initial"],
                                        adaptive=True))
            gpu, cpu = pair
            gpu.refinement_mode = "reference"
            gpu.update_safe_set(**kwargs)
            cpu.update_safe_set(refinement_mode="reference", **kwargs)
            assert_array_equal(gpu.safe_set, cpu.safe_set)
            assert_array_equal(gpu._refinement, cpu._refinement)
            assert gpu.feed_dict[gpu.c_max] == cpu.c_max
    finally:
        sl.config.gp_batch_size, O.config.gp_batch_size = old


def test_smallest_boundary_value(sl):
    """lyapunov.py:22-56, known answer of tests/test_lyapunov.py:77-84 and a fused V."""
    grid = sl.GridWorld([[-1.5, 1], [-1, 1.5]], [3, 3])
    assert sl.smallest_boundary_value(lambda x: 2 * np.sum(np.abs(x), axis=1), grid) == 2.5
    P = np.array([[1.3, 0.2], [0.2, 0.7]])
    got = sl.smallest_boundary_value(sl.QuadraticFunction(P), sl.GridWorld([[-1, 2], [-1, 1]], [7, 9]))
    want = O.smallest_boundary_value(O.QuadraticFunction(P), O.GridWorld([[-1, 2], [-1, 1]], [7, 9]))
    assert got == want


def test_neural_network_policy_vs_oracle(sl):
    """functions.py:1702-1729 inference (the 2-32-32-1 policy of inverted_pendulum.ipynb cell 9)
    and its use as the policy of a Lyapunov sweep."""
    rng = np.random.default_rng(8)
    net_g = sl.NeuralNetwork([2, 32, 32, 1], ["relu", "relu", "tanh"], output_scale=0.8, seed=4)
    net_g.biases = [rng.normal(scale=0.1, size=32), rng.normal(scale=0.1, size=32)]
    net_c = O.NeuralNetwork([2, 32, 32, 1], [lambda v: np.maximum(v, 0.0)] * 2 + [np.tanh],
                            net_g.weights, net_g.biases, output_scale=0.8)
    x = rng.uniform(-1, 1, (500, 2))
    assert_allclose(net_g(x), net_c(x), rtol=1e-13, atol=1e-15)
    par = W.make_pendulum(num_points=24, M=50, tau_scale=1 / 64.)
    gpu, cpu = W.build_product(par), W.build_oracle(par)
    gpu.policy, cpu.policy = net_g, net_c
    det = _sweep_details(gpu)
    _assert_negative_parity(gpu, cpu, det)
    gpu.update_safe_set()
    cpu.update_safe_set()
    assert_array_equal(gpu.safe_set, cpu.safe_set)


def test_learning_loop_vs_oracle(sl):
    """The loop of adaptive_safety_verification.ipynb cells 23-25: update_safe_set ->
    get_safe_sample -> measure the true plant -> add_data_point -> update_safe_set ..."""
    par = W.make_pendulum(num_points=32, M=20, tau_scale=1 / 64., seed=11)
    gpu, cpu = W.build_product(par), W.build_oracle(par)
    pl = par["plant"]
    true_dyn = O.InvertedPendulum(normalization=[pl["state_norm"], pl["action_norm"]], **pl["true"])
    perturbations = np.array([[0.0]])
    limits = np.array([[-1., 1.]])
    gpu.update_safe_set()
    cpu.update_safe_set()
    for it in range(6):
        assert_array_equal(gpu.safe_set, cpu.safe_set)
        assert gpu.feed_dict[gpu.c_max] == cpu.c_max
        sa_g, b_g = sl.get_safe_sample(gpu, perturbations, limits, positive=True)
        sa_c, b_c = O.get_safe_sample(cpu, perturbations, limits, positive=True)
        assert_array_equal(sa_g, sa_c)
        assert_allclose(b_g, b_c, rtol=RTOL)
        measurement = true_dyn(sa_c)
        gpu.dynamics.add_data_point(sa_g, measurement)
        cpu.dynamics.add_data_point(sa_c, measurement)
        gpu.update_safe_set(can_shrink=bool(it % 2))
        cpu.update_safe_set(can_shrink=bool(it % 2))
    assert_array_equal(gpu.safe_set, cpu.safe_set)
    assert gpu.dynamics.functions[0].gaussian_process._factor.appends == 6


def test_plants_vs_oracle(sl):
    rng = np.random.default_rng(5)
    norm = [(0.5, 4.4), (0.37,)]
    sa = rng.uniform(-1, 1, (300, 3))
    for fr in (0.0, 0.1):
        assert_allclose(sl.InvertedPendulum(0.15, 0.5, fr, 0.01, norm)(sa),
                        O.InvertedPendulum(0.15, 0.5, fr, 0.01, norm)(sa), rtol=1e-12)
    sa5 = rng.uniform(-1, 1, (300, 5))
    cn = [(1.0, 0.5, 2.0, 3.0), (20.0,)]
    assert_allclose(sl.CartPole(0.175, 1.732, 0.28, 0.01, 0.01, cn)(sa5),
                    O.CartPole(0.175, 1.732, 0.28, 0.01, 0.01, cn)(sa5), rtol=1e-11)


# ------------------------------------------------------------------ GP posterior
@pytest.mark.parametrize("M", [1, 7, 64, 255, 256, 257, 500, 513, 777])
def test_gp_posterior_vs_oracle(sl, M):
    """functions.py:417-458, 507-515, 278-291 at panel-boundary sizes; distinct hypers, prior
    mean, scale != 1."""
    par = W.make_pendulum(num_points=8, M=M, scale=1.7, seed=M)
    _, dyn_gpu = W._build(sl, par, "product")
    _, dyn_cpu = W._build(O, par, "oracle")
    rng = np.random.default_rng(M + 1)
    pts = rng.uniform(-1, 1, (333, 3))
    m_gpu, e_gpu = dyn_gpu(pts[:, :2], pts[:, 2:])
    m_cpu, e_cpu = dyn_cpu(pts[:, :2], pts[:, 2:])
    assert_allclose(m_gpu, m_cpu, rtol=RTOL, atol=1e-12)
    assert_allclose(e_gpu, e_cpu, rtol=RTOL, atol=1e-12)
    gp_gpu = dyn_gpu.functions[1].gaussian_process
    gp_cpu = dyn_cpu.functions[1].gaussian_process
    assert_allclose(gp_gpu.cholesky, gp_cpu.cholesky, rtol=1e-7, atol=1e-12)
    assert_allclose(gp_gpu.alpha, gp_cpu.alpha, rtol=1e-6, atol=1e-10)


@pytest.mark.parametrize("M", [5, 257, 600])
def test_gp_kernel_expressions_vs_oracle(sl, M):
    """Sums of products of gpflow primitives with active_dims (SURVEY.md 8f item 3; the kernels of
    examples/inverted_pendulum.ipynb cell 6) through the sweep kernel's generation phase, across
    panel boundaries; one output keeps the plain RBF fast path in the same launch."""
    par = W.make_pendulum(num_points=8, M=M, scale=1.3, seed=M, with_prior_mean=True)
    nb = W.notebook_pendulum_kernels([[2e-3, 6e-3, 1.5e-3], [2.5e-2, 8e-3, 1.2e-2]])
    plain = '["rbf", 3, {"variance": 0.8, "lengthscales": [0.9, 1.4, 0.7], "ARD": true}]'
    m52 = ('["add", ["matern52", 2, {"variance": 0.5, "lengthscales": [0.8, 1.1], "active_dims": [0, 2], '
           '"ARD": true}], ["prod", ["matern12", 1, {"lengthscales": 2.0, "active_dims": [1]}], '
           '["constant", 3, {"variance": 0.3}]], ["white", 3, {"variance": 0.02}]]')
    for specs in ([nb[0], nb[1]], [m52, plain]):
        par["kernel_specs"] = specs
        _, dyn_gpu = W._build(sl, par, "product")
        _, dyn_cpu = W._build(O, par, "oracle")
        pts = np.random.default_rng(M + 1).uniform(-1, 1, (333, 3))
        m_gpu, e_gpu = dyn_gpu(pts)
        m_cpu, e_cpu = dyn_cpu(pts)
        assert_allclose(m_gpu, m_cpu, rtol=RTOL, atol=1e-10)
        assert_allclose(e_gpu, e_cpu, rtol=RTOL, atol=1e-7)
        gp_gpu, gp_cpu = (d.functions[0].gaussian_process for d in (dyn_gpu, dyn_cpu))
        assert_allclose(gp_gpu.cholesky, gp_cpu.cholesky, rtol=1e-7, atol=1e-12)
    # the mean-only Bellman path evaluates the same expressions (reinforcement_learning.py:98-99)
    par["kernel_specs"] = [nb[0], m52]
    rl_gpu, _ = _rl_objects(sl, par, "product")
    rl_cpu, _ = _rl_objects(O, par, "oracle")
    states = np.random.default_rng(3).uniform(-1, 1, (150, 2))
    assert_allclose(rl_gpu.future_values(states), rl_cpu.future_values(states), rtol=1e-8,
                    atol=1e-10)


def test_gp_empty_data_is_the_prior(sl):
    """The notebooks start from np.empty((0, d)) data (inverted_pendulum.ipynb cell 6): the
    posterior is the prior mean and kern.Kdiag, and the first add_data_point refits."""
    par = W.make_pendulum(num_points=[15, 13], M=1, with_prior_mean=True, tau_scale=1 / 150.)
    par["X"], par["Y"] = par["X"][:0], par["Y"][:0]
    for specs in (None, W.notebook_pendulum_kernels([[2e-3, 6e-3, 1.5e-3], [2.5e-2, 8e-3, 1.2e-2]])):
        par["kernel_specs"] = specs
        gpu, cpu = W.build_product(par), W.build_oracle(par)
        pts = np.random.default_rng(1).uniform(-1, 1, (70, 3))
        for a, b in zip(gpu.dynamics(pts), cpu.dynamics(pts)):
            assert_allclose(a, b, rtol=1e-12, atol=1e-15)
        gpu.update_safe_set()
        cpu.update_safe_set()
        assert_array_equal(gpu.safe_set, cpu.safe_set)
        x, y = np.array([[0.1, -0.2, 0.05]]), np.array([[0.02, -0.01]])
        gpu.dynamics.add_data_point(x, y)
        cpu.dynamics.add_data_point(x, y)
        for a, b in zip(gpu.dynamics(pts), cpu.dynamics(pts)):
            assert_allclose(a, b, rtol=RTOL, atol=1e-10)
        gpu.update_safe_set()
        cpu.update_safe_set()
        assert_array_equal(gpu.safe_set, cpu.safe_set)


def test_gp_shared_factor_equals_distinct_path(sl):
    """Outputs sharing X/kernel/noise use one Cholesky factor (D'=1); results must equal the
    oracle, which factorises per output like the reference (functions.py:283-286)."""
    par = W.make_pendulum(num_points=8, M=300, shared_hypers=True)
    _, dyn_gpu = W._build(sl, par, "product")
    _, dyn_cpu = W._build(O, par, "oracle")
    assert dyn_gpu.gp_stack().num_factors == 1
    pts = np.random.default_rng(0).uniform(-1, 1, (200, 3))
    m_gpu, e_gpu = dyn_gpu(pts)
    m_cpu, e_cpu = dyn_cpu(pts)
    assert_allclose(m_gpu, m_cpu, rtol=RTOL, atol=1e-12)
    assert_allclose(e_gpu, e_cpu, rtol=RTOL, atol=1e-12)


def test_incremental_factor_growth_equals_refit(sl):
    """add_data_point grows the cached factor by rank-one appends (O(M^2)); the result must equal
    a fresh factorisation (functions.py:395-415, 525-546) and the oracle's predictions."""
    import time
    import torch
    par = W.make_pendulum(num_points=8, M=200, seed=3)
    _, dyn_gpu = W._build(sl, par, "product")
    _, dyn_cpu = W._build(O, par, "oracle")
    dyn_gpu(np.zeros((1, 3)))                                  # build the initial factors
    rng = np.random.default_rng(0)
    for i in range(5):
        x = rng.uniform(-1, 1, (1, 3))
        y = rng.normal(scale=0.01, size=(1, 2))
        dyn_gpu.add_data_point(x, y)
        dyn_cpu.add_data_point(x, y)
    gp = dyn_gpu.functions[1].gaussian_process
    assert gp._factor.appends == 5 and gp._factor.M == 205
    fresh = sl.GPRCached(gp.X, gp.Y, gp.kern, mean_function=gp.mean_function,
                         noise_variance=gp.likelihood.variance, scale=gp._scale)
    import safe_learning_b200.functions as F
    F._FACTOR_CACHE.clear()
    fresh.update_cache()
    assert fresh._factor.appends == 0
    assert_allclose(gp.cholesky, fresh.cholesky, rtol=1e-9, atol=1e-13)
    assert_allclose(gp.alpha, fresh.alpha, rtol=1e-7, atol=1e-11)
    pts = rng.uniform(-1, 1, (100, 3))
    m_gpu, e_gpu = dyn_gpu(pts)
    m_cpu, e_cpu = dyn_cpu(pts)
    assert_allclose(m_gpu, m_cpu, rtol=RTOL, atol=1e-12)
    assert_allclose(e_gpu, e_cpu, rtol=RTOL, atol=1e-12)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    dyn_gpu.add_data_point(rng.uniform(-1, 1, (1, 3)), rng.normal(scale=0.01, size=(1, 2)))
    torch.cuda.synchronize()
    print("incremental add_data_point (2 GPs, M=205): %.3f ms" % (1e3 * (time.perf_counter() - t0)))


def test_gp_negative_variance_is_nan_not_clamped(sl):
    """functions.py:451, 514: var < 0 -> sqrt -> NaN -> unsafe.  Query AT training points of a
    noise-free-ish GP, where cancellation can push var below zero: wherever the oracle's var is
    NaN-producing or tiny the GPU must not clamp silently; finite stds must agree loosely."""
    rng = np.random.default_rng(2)
    X = rng.uniform(-1, 1, (40, 2))
    Y = np.sin(X[:, :1])
    gp = sl.GPRCached(X, Y, sl.RBF(2, lengthscales=2.0), noise_variance=1e-10)
    mean, var = sl.GaussianProcess(gp).predict_device(X, want_var=True)
    var = var.cpu().numpy()
    assert np.all(np.abs(var) < 1e-3)
    _, err = sl.GaussianProcess(gp)(X)
    assert np.array_equal(np.isnan(err), var < 0)


# ------------------------------------------------------------------ the sweep
@pytest.mark.parametrize("shared", [False, True])
def test_pendulum_sweep_vs_oracle(sl, shared):
    """C2 at test size (48x48, M=150): negative / decrease / threshold / values / safe set /
    c_max / _refinement against the oracle running the reference loop."""
    par = W.make_pendulum(num_points=48, M=150, shared_hypers=shared, tau_scale=1 / 48.)
    gpu, cpu = W.build_product(par), W.build_oracle(par)
    assert_array_equal(gpu.values, cpu.values)
    det = _sweep_details(gpu)
    assert_array_equal(det["values"], cpu.values)
    _assert_negative_parity(gpu, cpu, det)
    states = cpu.discretization.all_points
    m_cpu, e_cpu = cpu.dynamics(states, cpu.policy(states))
    assert_allclose(det["mean"], m_cpu, rtol=RTOL, atol=1e-12)
    assert_allclose(det["err"], e_cpu, rtol=RTOL, atol=1e-12)
    gpu.update_safe_set()
    cpu.update_safe_set()
    assert cpu.safe_set.sum() > par["initial"].sum(), "test config should grow the safe set"
    assert cpu.safe_set.sum() < cpu.safe_set.size
    assert_array_equal(gpu.safe_set, cpu.safe_set)
    assert gpu.feed_dict[gpu.c_max] == cpu.c_max
    assert_array_equal(gpu._refinement, cpu._refinement)


@pytest.mark.parametrize("lv_kind", ["abs2", "const", "norm1", "abs1"])
@pytest.mark.parametrize("num", [[48, 48], [37, 29], [5, 3]])
def test_deterministic_linear_sweep_specialised_kernel(sl, lv_kind, num):
    """The register-resident kernel of the LQR composition with deterministic LinearSystem dynamics
    (det_sweep_fast_kernel, light.cu): flags and V bit-identical to the generic interpreter and
    to the oracle's arithmetic, ragged sizes (not multiples of 8 points per thread) included."""
    from safe_learning_b200 import _native as nat
    lib = nat.load()
    par = W.make_pendulum(num_points=num, M=8, tau_scale=1 / 20.)
    P = par["P"]
    objs = []
    for ns in (sl, O):
        grid = ns.GridWorld(par["limits"], par["num_points"])
        policy = ns.Saturation(ns.LinearSystem(-par["K"]), -1., 1.)
        dyn = ns.LinearSystem((par["A_true"], par["B_true"]))
        l_v = {"abs2": lambda: ns.AbsFunction(ns.LinearSystem((2 * P,))), "const": lambda: 0.7,
               "norm1": lambda: ns.Norm1Function(ns.LinearSystem((2 * P,))),
               "abs1": lambda: ns.AbsFunction(ns.LinearSystem((2 * P[[0]],)))}[lv_kind]()
        objs.append(ns.Lyapunov(grid, ns.QuadraticFunction(P), dyn, par["L_dyn"], l_v, par["tau"],
                                policy, initial_set=par["initial"]))
    gpu, cpu = objs
    fast = gpu.compute_negative().cpu().numpy().astype(bool)
    nat.check(lib.slb_debug_det_fast(0), "slb_debug_det_fast")
    try:
        generic = gpu.compute_negative().cpu().numpy().astype(bool)
    finally:
        nat.check(lib.slb_debug_det_fast(1), "slb_debug_det_fast")
    assert_array_equal(fast, generic)
    states = cpu.discretization.all_points
    nxt = cpu.dynamics(states, cpu.policy(states))
    dec = cpu.v_decrease_bound(states, nxt).ravel()
    thr = np.broadcast_to(cpu.threshold(states), (len(states), 1)).ravel()
    assert_array_equal(fast, dec < thr)
    assert 0 < fast.sum() < fast.size or min(num) < 8
    gpu.update_safe_set()
    cpu.update_safe_set()
    assert_array_equal(gpu.values, cpu.values)
    assert_array_equal(gpu.safe_set, cpu.safe_set)
    assert gpu.feed_dict[gpu.c_max] == cpu.c_max


def test_toy_1d_sweep_vs_oracle(sl):
    """C1: 101-point grid, M=50, V = |x| as a Triangulation on its own 3-point grid."""
    for tau in (1.0 / 101, 0.02, 0.2):
        par = W.make_toy_1d()
        par["tau"] = tau
        gpu, cpu = W.build_product(par), W.build_oracle(par)
        assert_allclose(gpu.values, cpu.values, rtol=1e-14, atol=1e-15)
        gpu.values = cpu.values          # identical keys -> identical prefix decisions
        det = _sweep_details(gpu)
        _assert_negative_parity(gpu, cpu, det)
        gpu.update_safe_set()
        cpu.update_safe_set()
        assert_array_equal(gpu.safe_set, cpu.safe_set)
        assert gpu.feed_dict[gpu.c_max] == cpu.c_max


def test_deterministic_sweep_vs_oracle(sl):
    """Deterministic dynamics (true pendulum plant + LinearSystem), the HBM-side variant."""
    par = W.make_pendulum(num_points=40, M=8, tau_scale=1 / 64.)
    gpu, cpu = W.build_product(par, deterministic=True), W.build_oracle(par, deterministic=True)
    det = _sweep_details(gpu)
    assert "err" not in det
    _assert_negative_parity(gpu, cpu, det)
    gpu.update_safe_set()
    cpu.update_safe_set()
    assert_array_equal(gpu.safe_set, cpu.safe_set)
    assert gpu.feed_dict[gpu.c_max] == cpu.c_max


def test_cartpole_4d_lyapunov_network_vs_oracle(sl):
    """C4 at test size: 4-D grid (7^4), four GPs on 5-D inputs (4 Cholesky factors), V = fixed-weight
    LyapunovNetwork(4, [64, 64, 64], tanh) (examples/utilities.py:48-104)."""
    par = W.make_cartpole(num_points=7, M=150, tau_scale=0.01)
    gpu, cpu = W.build_product(par), W.build_oracle(par)
    pts = np.random.default_rng(1).uniform(-1, 1, (300, 4))
    assert_allclose(gpu.lyapunov_function(pts), cpu.lyapunov_function(pts), rtol=1e-12, atol=1e-14)
    assert_allclose(gpu.values, cpu.values, rtol=1e-12, atol=1e-14)
    gpu.values = cpu.values                      # identical sort keys (tanh differs by an ulp)
    det = _sweep_details(gpu)
    _assert_negative_parity(gpu, cpu, det)
    states = cpu.discretization.all_points
    m_cpu, e_cpu = cpu.dynamics(states, cpu.policy(states))
    assert_allclose(det["mean"], m_cpu, rtol=RTOL, atol=1e-12)
    assert_allclose(det["err"], e_cpu, rtol=RTOL, atol=1e-12)
    gpu.update_safe_set()
    cpu.update_safe_set()
    assert_array_equal(gpu.safe_set, cpu.safe_set)
    assert gpu.feed_dict[gpu.c_max] == cpu.c_max


def test_get_safe_sample_vs_oracle(sl):
    """lyapunov.py:609-651, 657-797: most uncertain safe state-action pair (SURVEY 8f item 1)."""
    par = W.make_pendulum(num_points=40, M=60, tau_scale=1 / 100.)
    gpu, cpu = W.build_product(par), W.build_oracle(par)
    gpu.update_safe_set()
    cpu.update_safe_set()
    assert_array_equal(gpu.safe_set, cpu.safe_set)
    assert cpu.safe_set.sum() > 30
    perturbations = np.array([[-0.2], [-0.05], [0.0], [0.05], [0.2]])
    limits = np.array([[-1., 1.]])
    for positive in (True, False):
        sa_g, b_g = sl.get_safe_sample(gpu, perturbations, limits, positive=positive)
        sa_c, b_c = O.get_safe_sample(cpu, perturbations, limits, positive=positive)
        assert_array_equal(sa_g, sa_c)
        assert_allclose(b_g, b_c, rtol=RTOL)
    states = cpu.discretization.index_to_state(np.where(cpu.safe_set)[0])
    assert_array_equal(sl.perturb_actions(states, cpu.policy(states), perturbations, limits),
                       O.perturb_actions(states, cpu.policy(states), perturbations, limits))


def test_multi_batch_quirks_and_ragged_sizes(sl):
    """N not a multiple of the 64-point tile, N > gp_batch_size, all-safe c_max quirk
    (lyapunov.py:590-595, SURVEY Q4)."""
    old = (sl.config.gp_batch_size, O.config.gp_batch_size)
    try:
        sl.config.gp_batch_size = O.config.gp_batch_size = 100
        for num, tau_scale in (([37, 23], 1 / 48.), ([13, 5], 0.0), ([50, 11], 1 / 16.)):
            par = W.make_pendulum(num_points=num, M=70, tau_scale=tau_scale)
            gpu, cpu = W.build_product(par), W.build_oracle(par)
            gpu.update_safe_set()
            cpu.update_safe_set()
            assert_array_equal(gpu.safe_set, cpu.safe_set)
            assert gpu.feed_dict[gpu.c_max] == cpu.c_max
    finally:
        sl.config.gp_batch_size, O.config.gp_batch_size = old


@pytest.mark.parametrize("tau_scale,max_refinement,safety_factor",
                         [(1 / 60., 4, 2.0), (1 / 30., 8, 2.0), (1 / 30., 4, 2.0), (1 / 60., 12, 4.0)])
def test_adaptive_refinement_vs_oracle(sl, tau_scale, max_refinement, safety_factor):
    """Adaptive discretisation (lyapunov.py:445-487, 540-582) with the decrease evaluated on the
    refined mesh: the closed form on the GPU against the oracle's batch loop (several batches)."""
    par = W.make_pendulum(num_points=[26, 21], M=90, tau_scale=tau_scale)
    old = (sl.config.gp_batch_size, O.config.gp_batch_size)
    try:
        sl.config.gp_batch_size = O.config.gp_batch_size = 64
        lyaps = []
        for ns, kind in ((sl, "product"), (O, "oracle")):
            grid, dyn = W._build(ns, par, kind)
            policy = ns.Saturation(ns.LinearSystem(-par["K"]), -1., 1.)
            lyaps.append(ns.Lyapunov(grid, ns.QuadraticFunction(par["P"]), dyn, par["L_dyn"],
                                     ns.AbsFunction(ns.LinearSystem((2 * par["P"],))), par["tau"],
                                     policy, initial_set=par["initial"], adaptive=True))
        gpu, cpu = lyaps
        gpu.update_safe_set(max_refinement=max_refinement, safety_factor=safety_factor)
        cpu.update_safe_set(max_refinement=max_refinement, safety_factor=safety_factor,
                            refinement_mode="mesh")
        assert_array_equal(gpu.safe_set, cpu.safe_set)
        assert_array_equal(gpu._refinement, cpu._refinement)
        assert gpu.feed_dict[gpu.c_max] == cpu.c_max
        # max_refinement = 1 is the plain sweep
        gpu.update_safe_set(max_refinement=1)
        cpu.update_safe_set(max_refinement=1)
        assert_array_equal(gpu.safe_set, cpu.safe_set)
        assert_array_equal(gpu._refinement, cpu._refinement)
    finally:
        sl.config.gp_batch_size, O.config.gp_batch_size = old


def test_future_values_lyapunov_penalty_vs_oracle(sl):
    """reinforcement_learning.py:107-112: values - lambda (v_decrease_bound - threshold)."""
    par = W.make_pendulum(num_points=[15, 13], M=60)
    rl_gpu, _ = _rl_objects(sl, par, "product")
    rl_cpu, _ = _rl_objects(O, par, "oracle")
    gpu, cpu = W.build_product(par), W.build_oracle(par)
    states = np.random.default_rng(5).uniform(-1, 1, (120, 2))
    for lam in (1.0, 3.5):
        assert_allclose(rl_gpu.future_values(states, lyapunov=gpu, lagrange_multiplier=lam),
                        rl_cpu.future_values(states, lyapunov=cpu, lagrange_multiplier=lam),
                        rtol=1e-8, atol=1e-10)


def test_future_values_is_differentiable(sl):
    """reinforcement_learning.py:65-114 under autodiff (inverted_pendulum.ipynb cell 17): the torch
    form of future_values equals the numpy form, and its gradient with respect to the actions --
    through the reward, the GP mean, the Triangulation value function and the Lyapunov penalty
    with its beta * sigma term -- equals central differences of the numpy form."""
    import torch
    par = W.make_pendulum(num_points=[31, 29], M=60, tau_scale=1 / 30.)
    rl, grid = _rl_objects(sl, par, "product", num=24)
    rng = np.random.default_rng(2)
    rl.value_function.parameters = rng.normal(size=(grid.nindex, 1))
    lyap = W.build_product(par)
    states = rng.uniform(-0.9, 0.9, (40, 2))
    actions = rng.uniform(-0.6, 0.6, (40, 1))
    for kwargs in (dict(), dict(lyapunov=lyap, lagrange_multiplier=0.7)):
        a_t = torch.tensor(actions, dtype=torch.float64, device="cuda", requires_grad=True)
        out = rl.future_values(torch.tensor(states, dtype=torch.float64, device="cuda"),
                               actions=a_t, **kwargs)
        ref = rl.future_values(states, actions=actions, **kwargs)
        assert_allclose(out.detach().cpu().numpy(), ref, rtol=1e-9, atol=1e-12)
        out.sum().backward()
        h = 1e-6
        fd = (rl.future_values(states, actions=actions + h, **kwargs)
              - rl.future_values(states, actions=actions - h, **kwargs)) / (2 * h)
        assert_allclose(a_t.grad.cpu().numpy(), fd, rtol=2e-4, atol=1e-6)
    # a parametric torch policy: the gradient reaches its weights
    net = torch.nn.Linear(2, 1, dtype=torch.float64, device="cuda")
    s_t = torch.tensor(states, dtype=torch.float64, device="cuda")
    loss = -rl.future_values(s_t, policy=lambda x: torch.tanh(net(x)), lyapunov=lyap).sum()
    loss.backward()
    assert net.weight.grad is not None and torch.isfinite(net.weight.grad).all()
    assert float(net.weight.grad.abs().sum()) > 0


def test_can_shrink_false_vs_oracle(sl):
    """lyapunov.py:507-510, 583-587 (SURVEY Q3): previous safe set seeds, batch-dependent."""
    old = (sl.config.gp_batch_size, O.config.gp_batch_size)
    try:
        sl.config.gp_batch_size = O.config.gp_batch_size = 64
        par = W.make_pendulum(num_points=[30, 21], M=60, tau_scale=1 / 32.)
        gpu, cpu = W.build_product(par), W.build_oracle(par)
        rng = np.random.default_rng(9)
        prev = rng.random(cpu.safe_set.size) < 0.3
        gpu.safe_set = prev | par["initial"]
        cpu.safe_set = (prev | par["initial"]).copy()
        gpu._refinement = (prev | par["initial"]).astype(int)
        cpu._refinement = (prev | par["initial"]).astype(int)
        gpu.update_safe_set(can_shrink=False)
        cpu.update_safe_set(can_shrink=False)
        assert_array_equal(gpu.safe_set, cpu.safe_set)
        assert gpu.feed_dict[gpu.c_max] == cpu.c_max
        assert_array_equal(gpu._refinement, cpu._refinement)
    finally:
        sl.config.gp_batch_size, O.config.gp_batch_size = old


def test_prefix_rule_random_ties(sl):
    """slb_first_fail / slb_apply_prefix against the oracle's closed form on heavily tied V
    (SURVEY Q1/Q2), including no-failure and first-point-fails cases."""
    import torch
    from safe_learning_b200 import _device as dev, _native as nat
    lib = nat.load()
    rng = np.random.default_rng(11)
    for trial in range(40):
        n = int(rng.integers(1, 5000))
        values = rng.integers(-3, 4, n).astype(float)
        values[rng.random(n) < 0.05] = -0.0
        neg = rng.random(n) < (0.999 if trial % 3 else 0.5)
        init = rng.random(n) < 0.1
        if trial == 0:
            neg[:] = True
        if trial == 1:
            neg[:] = False
            init[:] = False
        safe_cpu, p = O.prefix_rule(values, neg | init, init)
        v, ng, it = dev.to_device(values), dev.to_device(neg.astype(np.uint8), torch.uint8), \
            dev.to_device(init.astype(np.uint8), torch.uint8)
        ws = dev.empty((int(lib.slb_first_fail_workspace(n)) // 8,))
        key, stats = dev.zeros((4,), torch.int64), dev.zeros((4,), torch.int64)
        safe = dev.empty((n,), torch.uint8)
        nat.check(lib.slb_first_fail(dev.stream(), v.data_ptr(), ng.data_ptr(), it.data_ptr(), n, 0,
                                     ws.data_ptr(), key.data_ptr()), "first_fail")
        nat.check(lib.slb_apply_prefix(dev.stream(), v.data_ptr(), it.data_ptr(), n, 0,
                                       key.data_ptr(), safe.data_ptr(), ws.data_ptr(),
                                       stats.data_ptr()), "apply_prefix")
        assert_array_equal(safe.cpu().numpy().astype(bool), safe_cpu)
        st = stats.cpu().numpy()
        assert st[1] == p and st[0] == safe_cpu.sum()
        assert key.cpu().numpy()[2] == (neg | init).sum()


# ------------------------------------------------------------------ Bellman sweep
def _rl_objects(ns, par, kind, num=24):
    grid = ns.GridWorld(par["limits"], num)
    _, dynamics = W._build(ns, par, kind)
    policy = ns.Saturation(ns.LinearSystem(-par["K"]), -1., 1.)
    reward = ns.QuadraticFunction(-scipy_block(np.diag([1., 2.]), 1.2 * np.eye(1)))
    value = ns.Triangulation(grid, np.zeros((grid.nindex, 1)), project=True)
    return ns.PolicyIteration(policy, dynamics, reward, value, gamma=0.98), grid


def scipy_block(a, b):
    import scipy.linalg
    return scipy.linalg.block_diag(a, b)


def test_value_iteration_vs_oracle(sl):
    """reinforcement_learning.py:65-114, 135-140 with GP-mean dynamics (C3 at test size)."""
    par = W.make_pendulum(num_points=8, M=120)
    rl_gpu, _ = _rl_objects(sl, par, "product")
    rl_cpu, _ = _rl_objects(O, par, "oracle")
    for sweep in range(4):
        res = rl_gpu.value_iteration()
        old = rl_cpu.value_function.parameters.copy()
        new = rl_cpu.value_iteration()
        assert_allclose(rl_gpu.value_function.parameters[0], new, rtol=1e-9, atol=1e-12)
        assert_allclose(res, np.max(np.abs(new - old)), rtol=1e-9)
    states = np.random.default_rng(0).uniform(-1, 1, (100, 2))
    assert_allclose(rl_gpu.future_values(states), rl_cpu.future_values(states), rtol=1e-9,
                    atol=1e-12)


def test_discrete_policy_optimization_vs_oracle(sl):
    """reinforcement_learning.py:213-279: first argmax over a discrete action set, with a
    constraint mask."""
    par = W.make_pendulum(num_points=8, M=60)
    grid_g, grid_c = sl.GridWorld(par["limits"], 15), O.GridWorld(par["limits"], 15)
    dyn_g = sl.LinearSystem((par["A_true"], par["B_true"]))
    dyn_c = O.LinearSystem((par["A_true"], par["B_true"]))
    rew = -scipy_block(np.diag([1., 2.]), 1.2 * np.eye(1))
    rng = np.random.default_rng(4)
    v0 = -rng.random((grid_c.nindex, 1))
    rl_g = sl.PolicyIteration(sl.Triangulation(grid_g, np.zeros((grid_c.nindex, 1))), dyn_g,
                              sl.QuadraticFunction(rew), sl.Triangulation(grid_g, v0, project=True))
    rl_c = O.PolicyIteration(O.Triangulation(grid_c, np.zeros((grid_c.nindex, 1))), dyn_c,
                             O.QuadraticFunction(rew), O.Triangulation(grid_c, v0, project=True))
    actions = np.linspace(-1, 1, 21)[:, None]
    constraint = lambda arr: np.where(np.abs(arr[:, 0]) > 0.8, -1.0, 1.0)  # noqa: E731
    best_g = rl_g.discrete_policy_optimization(actions, constraint)
    best_c = rl_c.discrete_policy_optimization(actions, constraint)
    assert_array_equal(best_g.cpu().numpy(), best_c)
    assert_array_equal(rl_g.policy.parameters[0], best_c)


# ------------------------------------------------------------------ C-ABI error behaviour
def test_errors_are_loud(sl):
    from safe_learning_b200 import _native as nat
    grid = sl.GridWorld([[-1, 1]], 3)
    with pytest.raises(TypeError):      # neither a Function object nor a callable
        sl.Lyapunov(grid, "x^2", sl.LinearSystem(np.array([[1, 1.]])), 0.4, 0.3, 0.5,
                    sl.LinearSystem(np.array([[-.1]])))
    lyap = sl.Lyapunov(grid, sl.QuadraticFunction(np.array([[1.0]])),
                       sl.LinearSystem(np.array([[1, 1., 1.]])), 0.4, 0.3, 0.5,
                       sl.LinearSystem(np.array([[-.1]])))
    with pytest.raises(nat.NativeLibraryError):
        lyap.update_safe_set()          # dynamics expect 3 inputs, state+action give 2
    with pytest.raises(NotImplementedError):
        sl.Lyapunov(grid, sl.QuadraticFunction(np.array([[1.0]])),
                    sl.LinearSystem(np.array([[1, 1.]])), 0.4, 0.3, 0.5,
                    sl.LinearSystem(np.array([[-.1]])), adaptive=True).update_safe_set(
                        can_shrink=False, max_refinement=4)
    with pytest.raises(TypeError):
        sl.GPRCached(np.zeros((2, 2)), np.zeros((2, 1)), kern="rbf")
    with pytest.raises(NotImplementedError):      # expands to 8 primitives, the descriptor holds 6
        k = sl.RBF(2) + sl.Matern32(2)
        sl.GaussianProcess(sl.GPRCached(np.zeros((2, 2)), np.zeros((2, 1)), (k * k) * k))(np.zeros((1, 2)))


@pytest.mark.parametrize("filtered", [True, False])
def test_packed_restore_orders_the_factor_copy_behind_the_sweep(sl, filtered):
    """PackedCache.restore sends the packed factors on a second stream and registers an event the
    library waits for before any launch that reads them (slb_record_factor_dependency).  The copy is
    held back by ~10 ms of busy-waiting on that stream while the device copy of the factors is
    zeroed: the sweep (direct launches, then CUDA-graph replays) must still see the restored
    factors."""
    import torch
    par = W.make_pendulum(num_points=[61, 53], M=200, tau_scale=1 / 16., seed=3)
    gpu = W.build_product(par)
    if not filtered:
        gpu.filter = False
    gpu.update_safe_set()
    want = gpu.safe_set.copy()
    if filtered:
        gpu.reset_filter_stats()
        gpu.compute_negative()
        assert gpu.filter_stats["refined"] > 0
    tables = gpu.dynamics.export_cache(pinned=True)
    assert 0 < tables.split < tables.arena.numel()
    gpu.dynamics.import_cache(tables)                 # creates the second stream
    gpu.update_safe_set()
    assert_array_equal(gpu.safe_set, want)
    for trial in range(4):                            # trial >= 2: graph replays
        tables.arena[tables.split:].zero_()
        with torch.cuda.stream(tables._side):
            torch.cuda._sleep(20000000)
        gpu.dynamics.import_cache(tables)
        gpu.update_safe_set()
        assert_array_equal(gpu.safe_set, want, err_msg="trial %d" % trial)
    cpu = W.build_oracle(par)
    cpu.update_safe_set()
    assert_array_equal(want, cpu.safe_set)


@pytest.mark.parametrize("form", ["constant L_V", "1-norm L_V", "scaled abs L_V", "scaled V"])
def test_screening_stage_other_lipschitz_forms(sl, form, mean_stage):
    """The closed-form slack of the fp32 screening stage (filter.cu: screening_slack) has one branch per
    accepted form of V / L_V: constant L_V, 1-norm of a linear map (one column for all outputs), scaled
    abs-linear map, scaled quadratic V.  Flags must equal the full posterior's and the oracle's with
    either first stage."""
    import safe_learning_b200 as ns
    import oracle as O
    from safe_learning_b200 import _native as nat
    par = W.make_pendulum(num_points=[53, 47], M=150, tau_scale=1 / 12., seed=21)
    out = []
    for mod, kind in ((ns, "product"), (O, "oracle")):
        grid, dynamics = W._build(mod, par, kind)
        policy = mod.Saturation(mod.LinearSystem(-par["K"]), -1., 1.)
        lyap_fun = mod.QuadraticFunction(par["P"])
        lin = mod.LinearSystem((2 * par["P"],))
        if form == "constant L_V":
            l_v = 0.25         # small enough that the decision depends on the GP (not a valid bound of V)
        elif form == "1-norm L_V":
            l_v = mod.Norm1Function(lin)
        elif form == "scaled abs L_V":
            l_v = mod.ScaledFunction(mod.AbsFunction(lin), 1.25)
        else:
            lyap_fun = mod.ScaledFunction(lyap_fun, 0.5)
            l_v = mod.ScaledFunction(mod.AbsFunction(lin), 0.5)
        out.append(mod.Lyapunov(grid, lyap_fun, dynamics, par["L_dyn"], l_v, par["tau"], policy,
                                initial_set=par["initial"]))
    gpu, cpu = out
    desc = gpu.sweep_descriptor()
    assert gpu._filter_enabled(desc)
    lib = nat.load()
    assert lib.slb_filter_stage1(desc) == (32 if mean_stage == "fp32 screening" else 64)
    gpu.reset_filter_stats()
    fast = gpu.compute_negative().cpu().numpy().copy()
    st = gpu.filter_stats
    assert st["prior"] > 0 and st["prior"] + st["head"] + st["refined"] == st["points"]
    gpu.filter = False
    full = gpu.compute_negative().cpu().numpy()
    assert_array_equal(fast, full)
    assert 0 < full.sum() < full.size, "trivial case: every point has the same flag"
    assert_array_equal(full.astype(bool), cpu.full_grid_negative())


def _linear_workload(d, num, M, seed, shared=False):
    """Synthetic d-dimensional counterpart of the pendulum configuration (one action): noisy samples of a
    stable linear map with a mild nonlinearity, a "wrong" linear prior mean, quadratic V."""
    rng = np.random.default_rng(seed)
    A = 0.85 * np.eye(d) + 0.05 * rng.standard_normal((d, d))
    B = 0.1 * rng.standard_normal((d, 1))
    X = rng.uniform(-1, 1, size=(M, d + 1))
    Y = X[:, :d] @ A.T + X[:, d:] @ B.T + 0.02 * np.sin(3 * X[:, :d]) + 1e-3 * rng.standard_normal((M, d))
    prior = np.hstack((A * 0.95, B * 1.1))
    resid = Y - X @ prior.T
    Q = rng.standard_normal((d, d))
    P = Q @ Q.T + d * np.eye(d)
    P = P / np.abs(P).max()
    K = 0.3 * rng.standard_normal((1, d))
    limits = np.array([[-1., 1.]] * d)
    nump = np.asarray(num, dtype=int)
    unit = (limits[:, 1] - limits[:, 0]) / (nump - 1)
    axes = [np.arange(n) * u + lo for n, u, lo in zip(nump, unit, limits[:, 0])]
    pts = np.column_stack([m.ravel() for m in np.meshgrid(*axes, indexing="ij")])
    variances = [float(v) for v in resid.var(axis=0)]
    lengthscales = [list(1.2 + 0.3 * rng.random(d + 1)) for _ in range(d)]
    if shared:                                    # one Cholesky factor for all outputs
        variances, lengthscales = [float(np.mean(variances))] * d, [lengthscales[0]] * d
    return dict(name="linear%dd" % d, limits=limits, num_points=nump, tau=float(np.sum(unit) / 2) / 8,
                X=X, Y=Y, variances=variances, lengthscales=lengthscales,
                noise_variance=1e-6, beta=2.0, scale=1.0, prior_rows=prior, K=K, P=P,
                L_dyn=float(np.linalg.norm(A, 1) + np.linalg.norm(B, 1) * np.linalg.norm(K, 1)),
                initial=np.linalg.norm(pts, axis=1) <= 0.25)


@pytest.mark.parametrize("d,num,M,tau_mult", [(1, [211], 60, 64.0), (3, [13, 11, 12], 90, 1.0),
                                              (4, [7, 6, 7, 6], 70, 0.125)])
def test_screening_stage_other_dimensions(sl, d, num, M, tau_mult, mean_stage):
    """The fp32 screening kernel stores its centred rows as 2, 4 or 8 floats (d_in + 1 <= 2 / 4 / 8) and
    unrolls the slack for up to four outputs: state dimensions 1, 3 and 4 with one action (d_in = 2, 4, 5)
    next to the pendulum's d_in = 3, every first stage against the full posterior and the oracle."""
    import safe_learning_b200 as ns
    import oracle as O
    from safe_learning_b200 import _native as nat
    # d = 4: one shared factor (four 64 x 64 head factors + the screened tables do not fit the head
    # stage's shared memory; such stacks keep the fp64 mean stage)
    par = _linear_workload(d, num, M, seed=40 + d, shared=(d == 4))
    par["tau"] *= tau_mult                        # mixed flags in every case (checked with the oracle)
    out = []
    for mod, kind in ((ns, "product"), (O, "oracle")):
        grid, dynamics = W._build(mod, par, kind)
        policy = mod.Saturation(mod.LinearSystem(-par["K"]), -1., 1.)
        lyap_fun = mod.QuadraticFunction(par["P"])
        l_v = mod.AbsFunction(mod.LinearSystem((2 * par["P"],)))
        out.append(mod.Lyapunov(grid, lyap_fun, dynamics, par["L_dyn"], l_v, par["tau"], policy,
                                initial_set=par["initial"]))
    gpu, cpu = out
    desc = gpu.sweep_descriptor()
    assert gpu._filter_enabled(desc)
    assert nat.load().slb_filter_stage1(desc) == (32 if mean_stage == "fp32 screening" else 64)
    gpu.reset_filter_stats()
    fast = gpu.compute_negative().cpu().numpy().copy()
    st = gpu.filter_stats
    assert st["prior"] > 0 and st["prior"] + st["head"] + st["refined"] == st["points"]
    gpu.filter = False
    full = gpu.compute_negative().cpu().numpy()
    assert_array_equal(fast, full)
    assert_array_equal(full.astype(bool), cpu.full_grid_negative())
    gpu.filter = "auto"
    gpu.update_safe_set()
    cpu.update_safe_set()
    assert_array_equal(gpu.safe_set, cpu.safe_set)
