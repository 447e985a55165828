"""The GP posterior kernel (``gp_tile_kernel``, csrc/gp_tile.cuh) and the decision filter in front of it at
every shape they are compiled or launched for, against the long-double reference and the per-point error
bound of tests/gp_posterior_reference.py.

Coverage (compiled shape or run-time path -> test):

=============================================================  ================================================
gp_tile_kernel<DIN, KEXPR, TP=64>, DIN 1..6, RBF / expression   test_predict_every_input_dimension (want_var 0/1,
                                                                M across k-pair / 8-row / 256-row / i-panel
                                                                boundaries, n across the 64-point tile)
stacks: 1..6 outputs, shared / distinct / mixed factors,        test_predict_stacks
empty-data output, scale, prior mean
MODE_SWEEP_GRID / MODE_SWEEP_STATES (mean, err, decrease)       test_sweep_grid_and_points, (d, m) = (1..5, 1),
                                                                (2, 2), (4, 2)
refine pass, TP = 32 split over G = 1..8 CTAs, FS > 1,          test_refine_pass (slb_debug_refine; DIN 2..6 --
unsplit 32-point tiles, persistent 64-point tiles               DIN 1 needs m = 0, which a sweep cannot have),
(> 132 tiles), RBF / expression, 1 / 2 / 5 factors              test_split_plan_covers_every_shape
filter_mean_kernel<DIN>, DIN 2..6; filter_mean32_kernel<DIN,    test_filter_every_input_dimension (both first
D> and filter_head_kernel<DIN, D>, D = DIN - m, m = 1, 2         stages, m = 1, 2), RBF and expressions
filter_head_kernel<6>, head tables in global memory (5 factors) test_filter_five_factors_head_tables_in_global
stack with an empty factor                                      test_filter_empty_factor
=============================================================  ================================================

A module-scope fixture prints the largest observed-error / bound ratio of each section and the smallest
mutation / bound ratio (``pytest -s``).
"""
import numpy as np
import pytest
import torch

import gp_posterior_reference as R
import oracle as O
import safe_learning_b200 as sl
from safe_learning_b200 import _device as dev
from safe_learning_b200 import _native as nat
from test_gpu_gp_vjp import _kernel

pytestmark = pytest.mark.gpu

MS = [0, 1, 3, 4, 5, 7, 8, 9, 255, 256, 257, 513]
NS = [1, 63, 64, 65, 200]
EXPRESSIONS = ["matern12", "matern32", "matern52", "linear", "constant", "white", "notebook", "six", "rbf_sub"]
SMS = 132
DEFAULT_SPLIT = 32 * SMS
LENGTHS = [1, 7, 32, 33, 100, 550, 600, 800, 1000, 2000, 4224, 4225, 9000]

_REPORT = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for key in sorted(_REPORT):
        print("%-28s %.3g" % (key, _REPORT[key]))


def _note(section, value, smallest=False):
    old = _REPORT.get(section)
    if old is None or (value < old if smallest else value > old):
        _REPORT[section] = value


def _hold(section, tables, z, mean=None, var=None, err=None, mutations=True):
    """Observed values within the bound; every applicable mutation exceeds it 10x somewhere."""
    ref = R.reference(tables, z)
    r = R.ratios(ref, mean=mean, var=var, err=err)
    _note("%s: error / bound" % section, R.worst(r))
    assert R.worst(r) <= 1.0, r
    if mutations:
        zm = z[:256]
        mut = R.mutation_ratios(tables, zm)
        if mut:
            _note("mutation / bound (min)", min(mut.values()), smallest=True)
            assert min(mut.values()) >= 10.0, mut
    return ref


def _gp(X, Y, kern, prior=None, scale=1.0, beta=2.0, noise=0.01):
    mean = sl.LinearSystem(prior[None, :]) if prior is not None else None
    return sl.GaussianProcess(sl.GPRCached(X, Y, kern, mean_function=mean, noise_variance=noise, scale=scale),
                              beta=beta)


def _stack(din, M, kinds, seed, shared=False, prior=True, scale=1.0, empty=None):
    """FunctionStack of len(kinds) GPs on one data set (output `empty`: no data); "rbf" is the plain path."""
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1, 1, (M, din))
    gps = []
    for o, kind in enumerate(kinds):
        krng = np.random.default_rng(seed + (0 if shared else 100 + o))
        Xo = X[:0] if o == empty else X
        Y = np.sin(Xo @ rng.normal(size=din) + o)[:, None] + 0.05 * rng.normal(size=(Xo.shape[0], 1))
        p = rng.normal(size=din) if prior else None
        gps.append(_gp(Xo, Y, _kernel(kind, din, krng), p, scale, beta=2.0 if o % 2 == 0 else 1.5))
    return sl.FunctionStack(gps)


def _predict(stack, z, want_var):
    mean, err = stack.predict_device(torch.tensor(z, device=dev.device()), want_var=want_var)
    return mean.cpu().numpy(), err.cpu().numpy()


# ------------------------------------------------------------------------ slb_gp_predict (64-point tiles)
@pytest.mark.parametrize("din", range(1, 7))
@pytest.mark.parametrize("M", MS)
def test_predict_every_input_dimension(din, M):
    """Plain RBF and one covariance expression (rotating through the kinds) per (d_in, M); every d_in meets
    every M class; n rotates through the tile boundaries; mean, var (want_var = 1) and err (want_var = 0)."""
    i = MS.index(M)
    for j, kinds in enumerate((["rbf", "rbf"], [EXPRESSIONS[(din + i) % len(EXPRESSIONS)]] * 2)):
        stack = _stack(din, M, kinds, seed=1000 * din + 10 * i + j, shared=j == 1, prior=M == 0 or (i + j) % 2 == 0,
                       scale=1.7 if i % 3 == 0 else 1.0)
        tables = R.stack_tables(stack)
        n = NS[(din + i + j) % len(NS)]
        if M >= 500:
            n = min(n, 65)
        z = R.query_points(tables, n, np.random.default_rng(i))
        mean, var = _predict(stack, z, True)
        mean2, err = _predict(stack, z, False)
        assert np.array_equal(mean, mean2)
        _hold("predict", tables, z, mean=mean, var=var, err=err, mutations=M > 0 or n > 1)


@pytest.mark.parametrize("D", range(1, 7))
@pytest.mark.parametrize("layout", ["shared", "distinct", "mixed", "empty output"])
def test_predict_stacks(D, layout):
    """Stacks of 1..6 outputs: one shared factor, one factor each, plain and expression factors mixed in one
    stack, one empty-data output among non-empty ones; scale 1.7 and a prior mean throughout."""
    kinds = {"shared": ["six"] * D, "distinct": ["rbf"] * D,
             "mixed": (["rbf", "notebook", "matern32", "rbf", "six", "linear"] * 2)[:D],
             "empty output": ["rbf", "matern52", "rbf", "six", "rbf", "notebook"][:D]}[layout]
    empty = D // 2 if layout == "empty output" and D > 1 else None
    stack = _stack(4, 137, kinds, seed=D * 7 + len(layout), shared=layout == "shared", scale=1.7, empty=empty)
    desc = stack.gp_stack()
    if layout == "shared":
        assert desc.num_factors == 1
    elif layout == "distinct":
        assert desc.num_factors == D
    tables = R.stack_tables(stack)
    z = R.query_points(tables, 150, np.random.default_rng(D))
    mean, var = _predict(stack, z, True)
    _, err = _predict(stack, z, False)
    _hold("predict stacks", tables, z, mean=mean, var=var, err=err)


# ------------------------------------------------------------------------ sweeps
def _workload(d, m, M, num, seed, kinds=None, shared=False, empty=None, noise=1e-4, tau_mult=1.0):
    """Product and oracle Lyapunov objects for a d-state, m-action linear plant with GP dynamics: training
    inputs next to grid points [x, policy(x)] (so dropping a row moves the posterior there), quadratic V,
    L_V = |2 P mu|, saturated linear policy."""
    rng = np.random.default_rng(seed)
    din = d + m
    limits = [[-1.0, 1.0]] * d
    ogrid = O.GridWorld(limits, num)
    K = 0.3 * rng.standard_normal((m, d))
    opolicy = O.Saturation(O.LinearSystem(-K), -1., 1.)
    idx = rng.choice(ogrid.nindex, size=M, replace=M > ogrid.nindex)
    xs = ogrid.index_to_state(idx)
    X = np.hstack((xs, opolicy(xs))) + 1e-3 * rng.standard_normal((M, din))
    A = 0.85 * np.eye(d) + 0.05 * rng.standard_normal((d, d))
    B = 0.1 * rng.standard_normal((d, m))
    Y = X[:, :d] @ A.T + X[:, d:] @ B.T + 0.02 * np.sin(3 * X[:, :d]) + 1e-3 * rng.standard_normal((M, d))
    prior = np.hstack((A * 0.95, B * 1.1))
    Q = rng.standard_normal((d, d))
    P = Q @ Q.T + d * np.eye(d)
    P /= np.abs(P).max()
    kinds = kinds or ["rbf"] * d
    gps = []
    for j in range(d):
        krng = np.random.default_rng(seed + (0 if shared else 100 + j))
        if kinds[j] == "rbf":
            kern = sl.RBF(din, variance=0.01, lengthscales=1.2 + 0.3 * krng.random(din))
        else:
            kern = _kernel(kinds[j], din, krng)
        Xj = X[:0] if j == empty else X
        gps.append(_gp(Xj, Y[:Xj.shape[0], [j]], kern, prior[j], noise=noise))
    unit = 2.0 / (np.asarray(num) - 1)
    tau = tau_mult * float(np.sum(unit) / 2) / 8
    L_dyn = float(np.linalg.norm(A, 1) + np.linalg.norm(B, 1) * np.linalg.norm(K, 1))
    lyap = sl.Lyapunov(sl.GridWorld(limits, num), sl.QuadraticFunction(P), sl.FunctionStack(gps), L_dyn,
                       sl.AbsFunction(sl.LinearSystem((2 * P,))), tau, sl.Saturation(sl.LinearSystem(-K), -1., 1.))
    return dict(lyap=lyap, ogrid=ogrid, opolicy=opolicy, P=P, idx=idx, din=din, d=d)


def _decrease_bound(wl, x, ref, dec):
    """|decrease - reference| / bound, decrease = V(mu) - V(x) + sum_j |2 P mu|_j err_j, from the mean and err
    bounds (first and second order) plus the decision's own fp64 rounding, (2 d + 4) u times its magnitudes."""
    LD, u = np.longdouble, R.U
    P = wl["P"].astype(LD)
    mu, err = ref["mean"], ref["err"]
    x = x.astype(LD)
    dmu = ref["mean_bound"].astype(LD)
    v, dv, beta = ref["var"], ref["var_bound"].astype(LD), ref["beta"]
    with np.errstate(invalid="ignore", divide="ignore"):
        derr = np.minimum(beta * dv / (np.sqrt(np.maximum(v, 0)) + np.sqrt(np.maximum(v - dv, 0))),
                          beta * np.sqrt(dv)) + 2 * u * err
    g = np.abs(mu @ (2 * P).T)
    want = (mu @ P * mu).sum(axis=1) - (x @ P * x).sum(axis=1) + (g * err).sum(axis=1)
    aP = np.abs(P)
    bound = ((g * dmu).sum(axis=1) + (dmu @ aP * dmu).sum(axis=1)
             + ((dmu @ (2 * aP).T) * (err + derr)).sum(axis=1) + (g * derr).sum(axis=1)
             + (2 * wl["d"] + 4) * u * 1.01 * ((np.abs(x) @ aP * np.abs(x)).sum(axis=1)
                                               + (np.abs(mu) @ aP * np.abs(mu)).sum(axis=1)
                                               + ((np.abs(mu) @ (2 * aP).T) * err).sum(axis=1)))
    return float(np.max(np.abs(np.asarray(dec, dtype=LD) - want) / bound))


@pytest.mark.parametrize("d,m", [(1, 1), (2, 1), (3, 1), (4, 1), (5, 1), (2, 2), (4, 2)])
def test_sweep_grid_and_points(d, m):
    num = {1: [1000], 2: [32, 31], 3: [10, 10, 10], 4: [6, 6, 5, 6], 5: [4, 4, 4, 4, 4]}[d]
    wl = _workload(d, m, 150, num, seed=10 * d + m)
    lyap = wl["lyap"]
    tables = R.stack_tables(lyap.dynamics)
    # grid mode: z = [x, policy(x)] exactly as the kernel forms it (index_to_state and the policy are
    # bit-exact with the oracle, test_gpu_parity)
    n = lyap.discretization.nindex
    x = wl["ogrid"].index_to_state(np.arange(n))
    z = np.hstack((x, wl["opolicy"](x)))
    _, det = lyap.compute_negative(want_details=True)
    mean, err, dec = (det[k].cpu().numpy() for k in ("mean", "err", "decrease"))
    near = np.concatenate((wl["idx"][-8:], wl["idx"][:120]))
    ref = _hold("sweep (grid)", tables, z, mean=mean, err=err, mutations=False)
    assert min(R.mutation_ratios(tables, z[near]).values()) >= 10.0
    r = _decrease_bound(wl, x, ref, dec)
    _note("sweep decrease: error / bound", r)
    assert r <= 1.0
    # state-list mode: states next to the training inputs and anywhere in the box
    rng = np.random.default_rng(d)
    states = np.vstack((x[wl["idx"][:100]] + 1e-3 * rng.standard_normal((100, d)), rng.uniform(-1, 1, (101, d))))
    zs = np.hstack((states, wl["opolicy"](states)))
    D = d
    lib = nat.load()
    sdev = torch.tensor(states, device=dev.device())
    neg = dev.empty((len(states),), torch.uint8)
    out = {k: dev.empty((len(states),) + ((D,) if k in ("mean", "err") else ())) for k in
           ("values", "decrease", "threshold", "mean", "err")}
    nat.check(lib.slb_lyapunov_points(dev.stream(), lyap.sweep_descriptor(), sdev.data_ptr(), len(states),
                                      neg.data_ptr(), *(out[k].data_ptr() for k in
                                                        ("values", "decrease", "threshold", "mean", "err"))),
              "slb_lyapunov_points")
    torch.cuda.synchronize()
    pm, pe, pd = (out[k].cpu().numpy() for k in ("mean", "err", "decrease"))
    ref = _hold("sweep (states)", tables, zs, mean=pm, err=pe)
    r = _decrease_bound(wl, states, ref, pd)
    _note("sweep decrease: error / bound", r)
    assert r <= 1.0


# ------------------------------------------------------------------------ the refine pass
def split_plan(length, n_max, upto32, nfac):
    """The refine pass's choice for a list of `length` points, restated from gp_sweep.cu / gp_tile.cuh:
    (points per tile, G row groups, FS factor slots, persistent CTAs walking several tiles)."""
    if length <= upto32:
        an = max(min(n_max, upto32), SMS * 32)
        grid = -(-an // 32)
        if grid > 512:                       # SLB_SPLIT_ITEMS: no split workspace for this grid
            return 32, 1, 1, -(-length // 32) > SMS
        spare = grid // -(-length // 32)
        FS = 1
        if nfac > 1 and spare >= 2 * nfac:
            FS, spare = nfac, spare // nfac
        return 32, min(8, max(1, spare)), FS, False
    return 64, 1, 1, -(-length // 64) > SMS


def _refine_grid(din):
    d = din - 1
    return d, {1: [22500], 2: [150, 150], 3: [29, 29, 29], 4: [13, 13, 13, 13], 5: [8, 8, 8, 8, 8]}[d]


def test_split_plan_covers_every_shape():
    """The lengths and split settings of test_refine_pass reach every G from 1 to 8, FS > 1, unsplit 32-point
    tiles and persistent 64-point tiles with several tiles per CTA."""
    seen = set()
    for din in range(2, 7):
        n_max = int(np.prod(_refine_grid(din)[1]))
        assert n_max > 512 * 32
        for nfac in (1, 2, 5):
            for split in (DEFAULT_SPLIT, 0, 1 << 40):
                for length in LENGTHS:
                    seen.add(split_plan(length, n_max, split, nfac))
    assert {g for tp, g, fs, _ in seen if tp == 32} == set(range(1, 9))
    assert any(fs > 1 for _, _, fs, _ in seen)
    assert (32, 1, 1, True) in seen and (32, 1, 1, False) in seen
    assert (64, 1, 1, True) in seen


def _refine_run(lyap, lst, n_max, D, sentinel):
    lib = nat.load()
    cfg = lyap.sweep_descriptor()
    ldev = torch.tensor(lst, dtype=torch.int64, device=dev.device())
    count = torch.tensor([len(lst)], dtype=torch.int64, device=dev.device())
    neg = torch.full((n_max,), 0xA5, dtype=torch.uint8, device=dev.device())
    vals = torch.full((n_max,), sentinel, dtype=torch.float64, device=dev.device())
    mean = torch.full((n_max, D), sentinel, dtype=torch.float64, device=dev.device())
    err = torch.full((n_max, D), sentinel, dtype=torch.float64, device=dev.device())
    ws = dev.empty((int(lib.slb_filter_workspace(n_max)) // 8 + 1,), torch.int64)
    nat.check(lib.slb_debug_refine(dev.stream(), cfg, 0, n_max, ldev.data_ptr(), count.data_ptr(), neg.data_ptr(),
                                   vals.data_ptr(), mean.data_ptr(), err.data_ptr(), ws.data_ptr()),
              "slb_debug_refine")
    torch.cuda.synchronize()
    return neg.cpu().numpy(), vals.cpu().numpy(), mean.cpu().numpy(), err.cpu().numpy()


@pytest.mark.parametrize("din", range(2, 7))
@pytest.mark.parametrize("kind", ["rbf", "expression"])
@pytest.mark.parametrize("nfac", [1, 2, 5])
def test_refine_pass(din, kind, nfac):
    """slb_debug_refine on unsorted, non-contiguous lists of every length under the default split, 0 (64-point
    tiles only) and 1 << 40 (32-point tiles only, unsplit beyond 512 CTAs).  Mean and err within the bound;
    negative and values equal slb_lyapunov_sweep's at the listed points; sentinels untouched elsewhere; two
    runs bit-identical; an unsplit tile (32 or 64 points) equal to the sweep's 64-point tile bit for bit."""
    d, num = _refine_grid(din)
    nf = min(nfac, d)
    kinds = ["rbf"] * d if kind == "rbf" else [["six", "notebook", "matern32", "linear", "matern52"][j % 5]
                                                if nf > 1 else "six" for j in range(d)]
    M = [70, 150, 300][(din + nfac) % 3]
    wl = _workload(d, 1, M, num, seed=din * 31 + nfac, kinds=kinds, shared=nf == 1)
    lyap = wl["lyap"]
    gp = lyap.dynamics
    if nf > 1 and nf < d:                    # nf distinct factors: outputs beyond nf share the last one
        for j in range(nf, d):
            gp.functions[j].gaussian_process.kern = gp.functions[nf - 1].gaussian_process.kern
            gp.functions[j].gaussian_process._stale = True
    desc = lyap.sweep_descriptor()
    assert desc.gp.num_factors == nf
    D = d
    n_max = lyap.discretization.nindex
    neg_full, det = lyap.compute_negative(want_details=True)
    neg_full = neg_full.cpu().numpy()
    vals_full, mean_full, err_full = (det[k].cpu().numpy() for k in ("values", "mean", "err"))
    # the list: a random permutation, so unsorted and non-contiguous; the reference on a sample of it
    perm = np.random.default_rng(din + nfac).permutation(n_max)
    sample = np.unique(np.concatenate((perm[:600], perm[600:max(LENGTHS)][::40])))
    x = wl["ogrid"].index_to_state(sample)
    tables = R.stack_tables(gp)
    ref = R.reference(tables, np.hstack((x, wl["opolicy"](x))))
    pos = {int(i): k for k, i in enumerate(sample)}
    lib = nat.load()
    sentinel = -7.25
    try:
        for split in (DEFAULT_SPLIT, 0, 1 << 40):
            lib.slb_debug_refine_split(split)
            for length in LENGTHS:
                lst = perm[:length]
                tp, G, FS, _ = split_plan(length, n_max, split, nf)
                neg, vals, mean, err = _refine_run(lyap, lst, n_max, D, sentinel)
                other = np.ones(n_max, dtype=bool)
                other[lst] = False
                assert (neg[other] == 0xA5).all() and (vals[other] == sentinel).all()
                assert (mean[other] == sentinel).all() and (err[other] == sentinel).all()
                assert np.array_equal(neg[lst], neg_full[lst]), (split, length)
                assert np.array_equal(vals[lst], vals_full[lst])
                again = _refine_run(lyap, lst, n_max, D, sentinel)
                for a, b in zip((neg, vals, mean, err), again):
                    assert np.array_equal(a, b), ("not deterministic", split, length, tp, G, FS)
                if G * FS == 1:
                    # an unsplit tile of either size equals the sweep's 64-point tile bit for bit
                    assert np.array_equal(mean[lst], mean_full[lst]), ("32/64 bit identity", split, length, tp)
                    assert np.array_equal(err[lst], err_full[lst]), ("32/64 bit identity", split, length, tp)
                rows = [pos[int(i)] for i in lst if int(i) in pos]
                sub = {k: (v[rows] if np.ndim(v) and k not in ("beta",) else v) for k, v in ref.items()}
                r = R.ratios(sub, mean=mean[[sample[k] for k in rows]], err=err[[sample[k] for k in rows]])
                _note("refine: error / bound", R.worst(r))
                assert R.worst(r) <= 1.0, (split, length, tp, G, FS, r)
    finally:
        lib.slb_debug_refine_split(DEFAULT_SPLIT)
    mut = R.mutation_ratios(tables, np.hstack((x, wl["opolicy"](x)))[:256])
    _note("mutation / bound (min)", min(mut.values()), smallest=True)
    assert min(mut.values()) >= 10.0, mut


# ------------------------------------------------------------------------ the filter
@pytest.fixture(params=["fp32 screening", "fp64 mean stage"])
def mean_stage(request):
    lib = nat.load()
    lib.slb_debug_filter_stages(3 if request.param == "fp32 screening" else 7)
    yield request.param
    lib.slb_debug_filter_stages(3)


def _filter_check(wl, want_stage1=None, require_all_stages=True):
    """Flags of the filtered sweep equal slb_lyapunov_sweep's bit for bit at a tau where all three stages
    decide points, and the oracle's wherever the full sweep's margin |decrease - threshold| is clear of its
    rounding (1e-9 relative)."""
    lyap = wl["lyap"]
    lib = nat.load()
    if want_stage1 is not None:
        assert lib.slb_filter_stage1(lyap.sweep_descriptor()) == want_stage1
    tau0 = lyap.tau
    found = None
    for mult in (1.0, 0.5, 2.0, 0.25, 4.0, 0.125, 8.0, 1 / 16., 16.0, 1 / 32., 32.0):
        lyap.tau = tau0 * mult
        lyap.filter = "auto"
        assert lyap._filter_enabled(lyap.sweep_descriptor())
        lyap.reset_filter_stats()
        fast = lyap.compute_negative().cpu().numpy().copy()
        st = lyap.filter_stats
        assert st["prior"] + st["head"] + st["refined"] == st["points"] == lyap.discretization.nindex
        lyap.filter = False
        full, det = lyap.compute_negative(want_details=True)
        full = full.cpu().numpy()
        assert np.array_equal(fast, full), mult
        if st["prior"] > 0 and st["head"] > 0 and st["refined"] > 0:
            found = (mult, full, det)
            break
    assert found is not None or not require_all_stages, "no tau lets all three stages decide points"
    if found is None:
        return
    _, full, det = found
    dec, thr = det["decrease"].cpu().numpy(), det["threshold"].cpu().numpy()
    clear = np.abs(dec - thr) > 1e-9 * (np.abs(dec) + np.abs(thr)) + 1e-300
    states = wl["ogrid"].index_to_state(np.arange(lyap.discretization.nindex))
    want = _oracle_negative(wl, states, lyap.tau)
    assert np.array_equal(full.astype(bool)[clear], want[clear])


def _oracle_negative(wl, states, tau):
    """decrease < threshold in fp64 numpy from the product's own GP posterior at [x, policy(x)]."""
    lyap = wl["lyap"]
    P = wl["P"]
    z = np.hstack((states, wl["opolicy"](states)))
    mean, err = _predict(lyap.dynamics, z, False)
    vx = (states @ P * states).sum(axis=1)
    vm = (mean @ P * mean).sum(axis=1)
    dec = vm - vx + (np.abs(mean @ (2 * P).T) * err).sum(axis=1)
    lv = np.abs(states @ (2 * P).T).sum(axis=1)
    thr = -lv * (1 + lyap._lipschitz_dynamics) * tau
    return dec < thr


# (d_in, m): every d_in with one action, and two actions wherever the fp32 screening kernel then runs (D = d_in - 2
# outputs, 1..4) -- with the m = 1 cases every (d_in, D) the screened kernels are compiled for
FILTER_SHAPES = ([pytest.param(din, 1, id=str(din)) for din in range(2, 7)] +
                 [pytest.param(din, 2, id="%d-m2" % din) for din in range(3, 7)])


@pytest.mark.parametrize("din,m", FILTER_SHAPES)
def test_filter_every_input_dimension(din, m, mean_stage):
    """Plain RBF factors (fp32 screening where D <= 4), with either first stage."""
    d = din - m
    num = {1: [401], 2: [45, 37], 3: [13, 11, 12], 4: [7, 6, 7, 6], 5: [5, 5, 5, 5, 5]}[d]
    wl = _workload(d, m, 120, num, seed=50 + din + 10 * (m - 1), shared=d == 4)
    stage = 32 if mean_stage == "fp32 screening" and d <= 4 else 64
    _filter_check(wl, want_stage1=stage)


@pytest.mark.parametrize("din", range(2, 7))
def test_filter_covariance_expressions(din):
    d = din - 1
    num = {1: [401], 2: [45, 37], 3: [13, 11, 12], 4: [7, 6, 7, 6], 5: [5, 5, 5, 5, 5]}[d]
    kinds = [["notebook", "matern32", "six", "linear", "matern52"][j % 5] for j in range(d)]
    wl = _workload(d, 1, 90, num, seed=60 + din, kinds=kinds)
    _filter_check(wl, want_stage1=64, require_all_stages=False)


def test_filter_five_factors_head_tables_in_global():
    """d = 5, m = 1, five distinct factors: the head stage stages four factors' tables in shared memory and
    reads the fifth from global memory (filter_head_kernel<6>, head_group_bound<6, false>)."""
    wl = _workload(5, 1, 200, [6, 6, 6, 6, 6], seed=77)
    assert wl["lyap"].sweep_descriptor().gp.num_factors == 5
    _filter_check(wl, want_stage1=64)


def test_filter_empty_factor():
    wl = _workload(3, 1, 120, [13, 11, 12], seed=78, empty=1)
    desc = wl["lyap"].sweep_descriptor()
    assert any(desc.gp.factors[f].M == 0 for f in range(desc.gp.num_factors))
    _filter_check(wl, require_all_stages=False)
