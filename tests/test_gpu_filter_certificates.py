"""The decision filter's certificates at every point it decides (csrc/filter.cu, slb_lyapunov_sweep_filtered).

One sweep gives every grid point its own threshold through a tabulated L_f (lyapunov_state_terms reads
``cfg.lf_values`` per flat index in all three stage-1 kernels and in the full sweep): each point sits next to
one edge of one stage (tests/filter_certificate_reference.py, ``PLACEMENTS``) -- a hair on the wrong side
(E - 1e-6 G), inside the guard (E + 0.5 G), clear of it (E + 10 x the stage's restated slack), or at the true
edge D(sigma_full) +- 10 B, 2 B, 0.01 B.  slb_debug_filter_lists tells which stage decided every point; the
audit then holds, against the long-double restatement from the product's own tables:
soundness (a decided negative point has D_hi(s) < thr, a non-negative one D_lo(s) >= thr, s the stage's
sigma bound), the guard (no decision with an exact margin below 0.5 G), liveness, the exact outcome outside
B, and the full sweep's flags bit for bit (except at +-0.01 B, recorded).

Coverage (compiled shape or run-time path -> test; every case under the stage-1 schemes that apply x both
head schedules, split 3|8 and round loop 3|16):

===========================================================  =================================================
filter_grid_mean_kernel<2> (default), filter_mean32_kernel<3,   test_pendulum (M = 500; 0, 1, 8, 64, 65, 200),
2> (3|32), filter_mean_kernel<3> (7); filter_head_kernel<3, 2>  test_lv_forms, test_shared_factor_short_scales
(both screened schemes), filter_head_kernel<3, 0> (fp64)
stage 1 / head edges D_hi, D_lo (D_lo with c_j < 0)            test_lv_forms["linear"] (LINEAR without abs)
variance floor (floor_rel in [1.05e-9, 2e-9]), M = 8, 64       test_variance_floor
filter_mean_kernel<DIN>, filter_head_kernel<DIN, 0>, DIN 2..6;  test_input_dimensions (d_in = 2..6 with m = 1;
filter_mean32_kernel<DIN, D>, filter_head_kernel<DIN, D>,       d_in = 3..6 with m = 2)
D = DIN - m <= 4, m = 1, 2 (screening_slack at D = 1..4)
kernel_expr_diag (prior sigma, head kss), Linear / White        test_expressions (d_in = 2..6, fp64 scheme)
filter_head_kernel<6, 0>, head tables in global memory; empty  test_five_factors, test_empty_factor
factor
screening_slack branches: const, abs-linear, 1-norm, scaled,  test_lv_forms
signed LINEAR, scaled quadratic V
===========================================================  =================================================

A module fixture prints, per case, scheme and stage, the smallest exact margin / G, the decided counts and
the class counts, and the run time of the long-double reference (``pytest -s``).
"""
import ctypes as C
import time

import numpy as np
import pytest
import torch

import bench_workloads as W
import filter_certificate_reference as F
import gp_posterior_reference as R
import oracle as O
import safe_learning_b200 as sl
from safe_learning_b200 import _native as nat
from test_gpu_gp_shapes import FILTER_SHAPES, _workload

pytestmark = pytest.mark.gpu

SCHEMES = {"grid": 3, "fp32": 3 | 32, "fp64": 7}
SCHEDULES = {"split": 8, "rounds": 16}
SCHEME_ID = {"grid": nat.MEAN_GRID_FACTORED, "fp32": nat.MEAN_FP32_SCREENED, "fp64": nat.MEAN_FP64}
_REPORT = []
_KEEP = []                     # every placement's L_f callable stays alive (the caches key on its id)
_CPU = {"reference seconds": 0.0}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for line in _REPORT:
        print(line)
    print("long-double reference: %.1f s" % _CPU["reference seconds"])


class _LfTable:
    """L_f per grid point of a 'num'-point grid on 'limits', looked up from the states it is called with."""

    def __init__(self, limits, num, values):
        self.lo = np.asarray(limits, dtype=np.float64)[:, 0]
        self.unit = (np.asarray(limits, dtype=np.float64)[:, 1] - self.lo) / (np.asarray(num) - 1)
        self.num = np.asarray(num)
        self.values = np.asarray(values, dtype=np.float64)

    def __call__(self, states):
        ijk = np.rint((np.asarray(states) - self.lo) / self.unit).astype(np.int64)
        flat = np.ravel_multi_index(tuple(ijk.T), tuple(self.num))
        return self.values[flat]


def _beta(tables):
    return np.array([o["beta"] for o in tables["outputs"]])


def _probe(lyap, mask, n, D):
    from safe_learning_b200 import _device as dev
    lib = nat.load()
    mu = torch.zeros((n, D), dtype=torch.float64, device=dev.device())
    dm = torch.full((n, D), np.inf, dtype=torch.float64, device=dev.device())
    lib.slb_debug_filter_stages(mask)
    try:
        lib.slb_debug_screening_probe(mu.data_ptr(), dm.data_ptr())
        lyap.compute_negative()
        torch.cuda.synchronize()
    finally:
        lib.slb_debug_screening_probe(None, None)
        lib.slb_debug_filter_stages(3)
    return dm.cpu().numpy()


def _lists(lyap, n):
    lib = nat.load()
    off = (C.c_int64 * 3)()
    nat.check(lib.slb_debug_filter_lists(n, off), "slb_debug_filter_lists")
    ws = lyap._filter_ws
    counts = ws[off[0] // 8: off[0] // 8 + 3].cpu().numpy().view(np.uint64)
    la = ws[off[1] // 8: off[1] // 8 + int(counts[0])].cpu().numpy()
    lb = ws[off[2] // 8: off[2] // 8 + int(counts[1])].cpu().numpy()
    return la, lb


def _factor_checks(name, tables):
    """Every factor's head table L_S^-1 against the long-double Cholesky of scale^2 (K_SS + noise I): within
    max(1e-10, |S| u cond) relative, and so its residual |W A W^T - I|; the full factor's residual too.
    Returns factor index -> (head residual, full residual): the rounding allowance of sigma_S >= sigma_full."""
    out = {}
    for o in tables["outputs"]:
        fac = o["factor"]
        if fac["index"] in out:
            continue
        rel, res_s, cond = F.check_head_factor(fac)
        res_f = F.full_factor_residual(fac)
        if rel is not None:
            allowed = max(1e-10, fac["Whead"].shape[0] * F.U * cond)
            assert rel <= allowed and res_s <= allowed, (name, fac["index"], rel, res_s, cond)
            _REPORT.append("%-34s factor %d: |S| %d, Whead vs long double %.2g, residual %.2g (cond %.2g); "
                           "full factor residual %.2g" % (name, fac["index"], fac["Whead"].shape[0], rel, res_s,
                                                          cond, res_f))
        out[fac["index"]] = (res_s or 0.0, res_f)
    return out


def _check_subset_bound(name, tables, terms, sfull, rows, resid):
    """sigma_S^2 >= sigma_full^2 at `rows`, within the two factors' residuals times the prior variance.
    Returns the largest allowance / sigma_full^2 (how tight the check is)."""
    if len(rows) == 0:
        return 0.0
    worst = 0.0
    for j, o in enumerate(tables["outputs"]):
        rs, rf = resid[o["factor"]["index"]]
        if o["factor"]["M"] == 0:
            continue
        tol = (rs + rf) * terms["sigma_prior"][rows, j] ** 2 + 1e-300
        ss2 = terms["sigma_S"][rows, j] ** 2
        sf2 = np.asarray(sfull[rows, j], dtype=F.LD) ** 2
        bad = ss2 < sf2 - tol
        assert not bad.any(), (name, "sigma_S below sigma_full", j, rows[bad][:8].tolist(),
                               (ss2[bad] / sf2[bad])[:8].astype(float).tolist())
        worst = max(worst, float(np.max(tol / np.maximum(sf2, 1e-300))))
    return worst


def _run(name, lyap, spec, z, d, schemes, limits, num, lf_neutral, lo_head=False, head=True, seed=0,
         focus=None, all_head=False):
    """Place, sweep under every scheme x schedule, audit.  focus: where placements go (default: anywhere);
    all_head: check sigma_S >= sigma_full at every head-decided point (else at a sample of 200)."""
    lib = nat.load()
    stack = lyap.dynamics
    n = lyap.discretization.nindex
    assert n == len(z) and n <= 1 << 22
    t0 = time.time()
    tables = F.head_tables(stack, R.stack_tables(stack))
    resid = _factor_checks(name, tables)
    terms = F.point_terms(tables, z)
    x = z[:, :d]
    meanerr = F.mean_error_term(tables, spec, terms, x)
    extra1 = meanerr.copy()
    extra2 = meanerr.copy()
    beta = _beta(tables)
    mu64 = terms["mu"].astype(np.float64)
    sfull = np.full(terms["mu"].shape, np.nan, dtype=F.LD)
    tight = 0.0
    for s in schemes:
        if s == "fp64":
            continue
        dm = _probe(lyap, SCHEMES[s], n, len(beta))
        with np.errstate(invalid="ignore"):
            extra1 = np.maximum(extra1, np.where(np.isfinite(dm).all(axis=1),
                                                 F.screening_slack(spec, beta, mu64, dm, terms["sigma_prior"]), np.inf))
            if s == "grid":
                ok = np.isfinite(dm).all(axis=1)
                extra2 = np.maximum(extra2, np.where(ok, F.screening_slack(spec, beta, mu64, np.where(ok[:, None], dm, 0),
                                                                          terms["sigma_S"]), 0.0))
    pl = F.plan(tables, spec, z, d, lyap.tau, lf_neutral, extra1, extra2, seed=seed, head_classes=head,
                lo_head=lo_head, terms=terms, true_weight=0.3, gap_extra=meanerr, focus=focus,
                sfull=sfull)
    _CPU["reference seconds"] += time.time() - t0
    fn = _LfTable(limits, num, pl["lf"])
    _KEEP.append(fn)
    lyap._lipschitz_dynamics = fn
    neg_full, det = lyap.compute_negative(want_details=True)
    neg_full = neg_full.cpu().numpy().astype(bool)
    thr = det["threshold"].cpu().numpy()
    # the read-back thresholds are this placement's (a stale table would put them elsewhere)
    placed = pl["place"] != "neutral"
    t = pl["target"].astype(np.float64)
    assert (np.abs(thr[placed] - t[placed]) <= 1e-12 * (np.abs(t[placed])
                                                       + np.abs(pl["lvx"][placed] * lyap.tau))).all(), name
    dt, e1, e2 = F.certify(tables, spec, x, terms, thr)
    counts = {p: int((pl["place"] == p).sum()) for p in F.PLACEMENTS}
    for p in F.PLACEMENTS[1:]:
        if p.startswith("hd") and not head or p.startswith("hd_lo") and not lo_head:
            continue
        assert counts[p] >= 20, (name, p, counts)
    assert lyap._filter_enabled(lyap.sweep_descriptor()), name
    for s in schemes:
        for h in SCHEDULES:
            mask = SCHEMES[s] | SCHEDULES[h]
            lib.slb_debug_filter_stages(mask)
            try:
                assert lib.slb_filter_mean_scheme(lyap.sweep_descriptor()) == SCHEME_ID[s], (name, s)
                lyap.reset_filter_stats()
                flags = lyap.compute_negative().cpu().numpy().astype(bool)
                st = lyap.filter_stats
                la, lb = _lists(lyap, n)
            finally:
                lib.slb_debug_filter_stages(3)
            stage = F.stages_from_lists(n, la, lb)
            assert len(np.unique(la)) == len(la) and set(lb.tolist()) <= set(la.tolist())
            assert (st["prior"], st["head"], st["refined"], st["points"]) == (
                int((stage == 1).sum()), int((stage == 2).sum()), int((stage == 3).sum()), n), (name, s, h)
            t0 = time.time()
            # sigma_full at every refined point and at the head-decided ones (all, or every k-th of them)
            hd = np.flatnonzero(stage == 2)
            if not all_head and len(hd) > 200:
                hd = hd[::-(-len(hd) // 200)]
            rows = np.union1d(np.flatnonzero(stage == 3), hd)
            F.exact_decrease(tables, spec, z, d, terms, rows[np.isnan(sfull[rows, 0].astype(np.float64))],
                             pl["dfull"], pl["B"], sfull)
            # the head subset's sigma bounds the full posterior's, to the two factors' rounding
            tight = max(tight, _check_subset_bound(name, tables, terms, sfull, rows, resid))
            _CPU["reference seconds"] += time.time() - t0
            fails, rep = F.audit(pl["place"], stage, flags, thr, e1, e2, pl["dfull"], pl["B"], neg_full, dt["mag"])
            _REPORT.append("%-34s %-4s %-6s stage 1: %6d decided, min margin/G %8.3g | head: %6d decided, min "
                           "margin/G %8.3g | refined %5d | +-0.01B disagreements %d"
                           % (name, s, h, rep["stage 1 decided"], rep["stage 1 min margin / G"],
                              rep["stage 2 decided"], rep["stage 2 min margin / G"], int((stage == 3).sum()),
                              rep["+-0.01B disagreements"]))
            if fails:
                bad = np.flatnonzero(flags != neg_full)[:6]
                sp, ss = terms["sigma_prior"], terms["sigma_S"]
                diag = [(int(i), pl["place"][i], int(stage[i]), bool(flags[i]), bool(neg_full[i]), float(thr[i]),
                         float(pl["dfull"][i]), float(pl["B"][i]), float(e1[0][i]), float(e2[0][i]),
                         sp[i].astype(float).tolist(), ss[i].astype(float).tolist(),
                         float(det["decrease"][i]), det["err"][i].cpu().numpy().tolist()) for i in bad]
                raise AssertionError((name, s, h, fails, "idx place stage flag full thr Dfull B Dhi1 Dhi2 "
                                      "sp sS dec_full err_full", diag))
    _REPORT.append("%-34s classes %s" % (name, {k: v for k, v in counts.items() if v}))
    _REPORT.append("%-34s sigma_S >= sigma_full: largest rounding allowance / sigma_full^2 %.2g" % (name, tight))
    # the +-0.01 B placements under 32-point refine tiles only (the split refine pass sums in another order)
    try:
        lib.slb_debug_refine_split(1 << 40)
        flags = lyap.compute_negative().cpu().numpy().astype(bool)
    finally:
        lib.slb_debug_refine_split(32 * 132)
    # (split tiles sum a^2 in another order than the full sweep's 64-point tile: there the flags are the exact
    # outcome wherever the decrease is more than B from the threshold, and may differ from the full sweep's
    # only within B)
    rec = np.isin(pl["place"], F.RECORDED)
    diff = np.flatnonzero(~rec & (flags != neg_full))
    F.exact_decrease(tables, spec, z, d, terms, diff[np.isnan(sfull[diff, 0].astype(np.float64))],
                     pl["dfull"], pl["B"], sfull)
    within = np.abs(pl["dfull"][diff] - thr[diff]) <= pl["B"][diff]
    _REPORT.append("%-34s refine split 1<<40: +-0.01B disagreements %d of %d, elsewhere %d (all within B: %s)"
                   % (name, int((rec & (flags != neg_full)).sum()), int(rec.sum()), len(diff), bool(within.all())))
    assert within.all(), (name, diff[~within][:8].tolist())
    known = ~np.isnan(pl["dfull"].astype(np.float64))
    clear = known & (np.abs(pl["dfull"] - thr) > pl["B"])
    assert (flags[clear] == (pl["dfull"][clear] < thr[clear])).all(), name


def _pendulum_spec(par, **kw):
    return F.fn_spec(par["P"], A=2 * par["P"], **kw)


def _pendulum(par, lyap=None):
    gpu = W.build_product(par) if lyap is None else lyap
    cpu = W.build_oracle(par)
    states = cpu.discretization.all_points
    z = np.hstack((states, cpu.policy(states)))
    return gpu, z


# ------------------------------------------------------------------------ cases
@pytest.mark.parametrize("M", [500, 0, 1, 8, 64, 65, 200])
def test_pendulum(M):
    """bench_workloads.make_pendulum at 61 x 53 points, two factors; M <= 64: the head subset is the whole
    data set (sigma_S = sigma_full); M = 0: the prior alone (no head subset: its classes are empty)."""
    par = W.make_pendulum(num_points=[61, 53], M=max(M, 1), tau_scale=1 / 16., seed=M + 3)
    if M == 0:
        par["X"], par["Y"] = par["X"][:0], par["Y"][:0]
    gpu, z = _pendulum(par)
    _run("pendulum M=%d" % M, gpu, _pendulum_spec(par), z, 2, ("grid", "fp32", "fp64"), par["limits"],
         par["num_points"], par["L_dyn"], head=M >= 8)


@pytest.mark.parametrize("form", ["const", "norm1", "scaled abs-linear", "linear", "scaled V"])
def test_lv_forms(form):
    """The L_V and V forms screening_applicable accepts, on the pendulum (abs-linear: test_pendulum)."""
    par = W.make_pendulum(num_points=[61, 53], M=300, tau_scale=1 / 16., seed=21)
    base, z = _pendulum(par)
    P = par["P"]
    V, LVf, spec = sl.QuadraticFunction(P), sl.AbsFunction(sl.LinearSystem((2 * P,))), None
    if form == "const":
        LVf, spec = 2.0, F.fn_spec(P, lv="const", lv_const=2.0)
    elif form == "norm1":
        LVf, spec = sl.Norm1Function(sl.LinearSystem((2 * P,))), _pendulum_spec(par, lv="norm1")
    elif form == "scaled abs-linear":
        LVf, spec = sl.AbsFunction(sl.LinearSystem((2 * P,))) * 1.7, _pendulum_spec(par, lv_scale=1.7)
    elif form == "linear":
        LVf, spec = sl.LinearSystem((2 * P,)), _pendulum_spec(par, lv="linear")
    else:
        V, LVf, spec = sl.QuadraticFunction(P) * 0.5, sl.AbsFunction(sl.LinearSystem((P,))), \
            F.fn_spec(P, v_scale=0.5, A=P)
    lyap = sl.Lyapunov(base.discretization, V, base.dynamics, par["L_dyn"], LVf, base.tau, base.policy)
    _run("pendulum L_V %s" % form, lyap, spec, z, 2, ("grid", "fp32", "fp64"), par["limits"], par["num_points"],
         par["L_dyn"], lo_head=form == "linear")


@pytest.mark.parametrize("k_scale", [0.01, 30.0], ids=["unsaturated", "saturated"])
def test_shared_factor_short_scales(k_scale):
    """One shared factor, scale 7.5, no prior mean, short lengthscales (tiles the grid mean leaves to fp64)."""
    par = W.make_pendulum(num_points=[61, 53], M=300, tau_scale=1 / 16., seed=5, shared_hypers=True,
                          with_prior_mean=False, scale=7.5)
    par["lengthscales"] = [[0.2, 0.15, 0.4]] * 2
    par["K"] = np.asarray(par["K"]) * k_scale
    gpu, z = _pendulum(par)
    assert gpu.sweep_descriptor().gp.num_factors == 1
    if not gpu._filter_enabled(gpu.sweep_descriptor()):
        pytest.skip("variance floor below the filter's limit for this case")
    _run("shared, scale 7.5, k x %g" % k_scale, gpu, _pendulum_spec(par), z, 2, ("grid", "fp32", "fp64"),
         par["limits"], par["num_points"], par["L_dyn"])


def _gp_workload_case(name, wl, num, schemes, seed, **kw):
    lyap = wl["lyap"]
    n = lyap.discretization.nindex
    x = wl["ogrid"].index_to_state(np.arange(n))
    z = np.hstack((x, wl["opolicy"](x)))
    d = wl["d"]
    spec = F.fn_spec(wl["P"], A=2 * wl["P"])
    limits = np.array([[-1.0, 1.0]] * d)
    focus = kw.pop("focus", None)
    _run(name, lyap, spec, z, d, schemes, limits, num, lyap._lipschitz_dynamics, seed=seed,
         focus=focus(lyap, z) if focus is not None else None, **kw)


def _near_subset_or_origin(share):
    """The grid points nearest (in length scales) to a head-subset input -- the `share` of them closest -- and
    those within 0.15 of the origin: where the sigma terms dominate G."""
    def focus(lyap, z):
        dist = np.full(len(z), np.inf)
        for f in lyap.dynamics.functions:
            gp = f.gaussian_process
            gp._ensure()
            fac = gp._factor
            ls = np.asarray(gp.kern.lengthscales, dtype=np.float64)
            Xh = fac.Xhead.cpu().numpy()[:fac.head_rows]
            zs = z / ls
            dist = np.minimum(dist, np.sqrt(((zs[:, None, :] - Xh[None, :, :]) ** 2).sum(axis=2)).min(axis=1))
        near = dist <= np.quantile(dist, share)
        return near | (np.linalg.norm(z[:, :-1], axis=1) < 0.15)
    return focus


@pytest.mark.parametrize("M", [8, 64])
def test_variance_floor(M):
    """noise chosen so that the certified variance floor noise / (M k_max + noise) is 1.5e-9 (the filter
    stays on just above its 1e-9 limit): the entries of L_S^-1 grow like noise^-1/2 and sum a^2 cancels
    against k** next to the training inputs.  Placements only next to head-subset inputs and near the origin
    (a 91 x 75 grid, the quarter of it nearest the subset); sigma_S >= sigma_full at every head-decided point."""
    noise = 1.5e-9 * M * 0.01 / (1 - 1.5e-9)
    wl = _workload(2, 1, M, [91, 75], seed=90 + M, noise=noise)
    floor = wl["lyap"].dynamics.variance_floor()
    assert 1.05e-9 <= floor <= 2e-9, floor
    _gp_workload_case("variance floor M=%d" % M, wl, [91, 75], ("grid", "fp32", "fp64"), M,
                      focus=_near_subset_or_origin(0.25), all_head=True)


DIMS = {1: [1201], 2: [45, 37], 3: [13, 11, 12], 4: [7, 6, 7, 6], 5: [5, 5, 5, 5, 5]}


@pytest.mark.parametrize("din,m", FILTER_SHAPES)
def test_input_dimensions(din, m):
    d = din - m
    wl = _workload(d, m, 120, DIMS[d], seed=50 + din + 10 * (m - 1), shared=d == 4)
    schemes = ("grid", "fp32", "fp64") if (din, m) == (3, 1) else ("fp32", "fp64") if d <= 4 else ("fp64",)
    _gp_workload_case("d_in=%d m=%d rbf" % (din, m), wl, DIMS[d], schemes, din)


@pytest.mark.parametrize("din", range(2, 7))
def test_expressions(din):
    """Covariance expressions with Linear and White primitives: the prior sigma and the head's k** depend on z."""
    d = din - 1
    kinds = [["linear", "white", "notebook", "six", "matern32"][j % 5] for j in range(d)]
    if d == 1:
        kinds = ["white"]
    wl = _workload(d, 1, 90, DIMS[d], seed=60 + din, kinds=kinds)
    _gp_workload_case("d_in=%d expressions" % din, wl, DIMS[d], ("fp64",), din)


def test_head_subset_of_a_rank_deficient_kernel_is_a_subset():
    """A Linear kernel on two inputs has rank 2: after two pivots the remaining diagonal is rounding noise.
    The 64 picks must still be 64 distinct training points -- a repeated pick counts one observation twice,
    and the head stage's sigma then falls below the full posterior's (seen at d_in = 3 with a Linear
    factor: sigma_S 0.0016 against sigma_full 0.0026, points decided negative that are not)."""
    from safe_learning_b200 import _device as dev
    from safe_learning_b200.functions import GPRCached
    rng = np.random.default_rng(11)
    X = rng.uniform(-1, 1, (90, 2)) * np.array([0.7, 0.9])
    picks = GPRCached._pivoted_subset(dev.to_device(X @ X.T), 64).cpu().numpy()
    assert len(set(picks.tolist())) == 64 and picks.min() >= 0 and picks.max() < 90


def test_two_passes():
    """2049 x 2049 > 2^22 points, M = 100: one filtered call sweeps them in two passes (per-pass idx_begin,
    flag offset, tabulated L_f at the pass's flat indices, counters reset per pass, lists of capacity 2^22).
    Placements on the 4096 points either side of index 2^22; the stages of the last pass from that call's
    lists, those of the 4096 points before the boundary from a one-pass call on exactly that range.  Flags of
    the two-pass call equal the full sweep's at all 4 198 401 points (except the +-0.01 B placements)."""
    lib = nat.load()
    chunk = 1 << 22
    par = W.make_pendulum(num_points=[2049, 2049], M=100, tau_scale=1 / 16., seed=8)
    gpu = W.build_product(par)
    n = gpu.discretization.nindex
    assert n > chunk and n - chunk < 8192
    name = "2049 x 2049, two passes"
    rows = np.arange(chunk - 4096, n)
    x = O.GridWorld(par["limits"], par["num_points"]).index_to_state(rows)
    z = np.hstack((x, O.Saturation(O.LinearSystem(-par["K"]), -1., 1.)(x)))
    spec = _pendulum_spec(par)
    t0 = time.time()
    tables = F.head_tables(gpu.dynamics, R.stack_tables(gpu.dynamics))
    resid = _factor_checks(name, tables)
    terms = F.point_terms(tables, z)
    meanerr = F.mean_error_term(tables, spec, terms, x)
    extra1, extra2 = meanerr.copy(), meanerr.copy()
    beta, mu64 = _beta(tables), terms["mu"].astype(np.float64)
    for s in ("grid", "fp32"):
        dm = _probe(gpu, SCHEMES[s], n, 2)[rows]
        ok = np.isfinite(dm).all(axis=1)
        with np.errstate(invalid="ignore"):
            extra1 = np.maximum(extra1, np.where(ok, F.screening_slack(spec, beta, mu64, np.where(ok[:, None], dm, 0),
                                                                       terms["sigma_prior"]), np.inf))
            if s == "grid":
                extra2 = np.maximum(extra2, np.where(ok, F.screening_slack(
                    spec, beta, mu64, np.where(ok[:, None], dm, 0), terms["sigma_S"]), 0.0))
    sfull = np.full(terms["mu"].shape, np.nan, dtype=F.LD)
    pl = F.plan(tables, spec, z, 2, gpu.tau, par["L_dyn"], extra1, extra2, seed=8, terms=terms, true_weight=0.3,
                gap_extra=meanerr, sfull=sfull)
    _CPU["reference seconds"] += time.time() - t0
    lf = np.full(n, par["L_dyn"])
    lf[rows] = pl["lf"]
    fn = _LfTable(par["limits"], par["num_points"], lf)
    _KEEP.append(fn)
    gpu._lipschitz_dynamics = fn
    neg_full, det = gpu.compute_negative(want_details=True)
    neg_full = neg_full.cpu().numpy().astype(bool)
    thr = det["threshold"].cpu().numpy()[rows]
    placed = pl["place"] != "neutral"
    t = pl["target"].astype(np.float64)
    assert (np.abs(thr[placed] - t[placed]) <= 1e-12 * (np.abs(t[placed])
                                                       + np.abs(pl["lvx"][placed] * gpu.tau))).all()
    counts = {p: int((pl["place"] == p).sum()) for p in F.PLACEMENTS}
    assert all(counts[p] >= 20 for p in F.PLACEMENTS[1:] if not p.startswith("hd_lo")), counts
    dt, e1, e2 = F.certify(tables, spec, x, terms, thr)
    rec = np.zeros(n, dtype=bool)
    rec[rows[np.isin(pl["place"], F.RECORDED)]] = True
    tight = 0.0
    for s in SCHEMES:
        for h in SCHEDULES:
            lib.slb_debug_filter_stages(SCHEMES[s] | SCHEDULES[h])
            try:
                assert lib.slb_filter_mean_scheme(gpu.sweep_descriptor()) == SCHEME_ID[s]
                gpu.reset_filter_stats()
                flags = gpu.compute_negative().cpu().numpy().astype(bool)
                st = gpu.filter_stats
                la, lb = _lists(gpu, chunk)                  # the last pass: [2^22, n)
                gpu.reset_filter_stats()
                part = gpu.compute_negative_range(chunk - 4096, chunk).cpu().numpy().astype(bool)
                st_part = gpu.filter_stats
                pa, pb = _lists(gpu, 4096)
            finally:
                lib.slb_debug_filter_stages(3)
            assert st["points"] == n and st["prior"] + st["head"] + st["refined"] == n
            assert not (~rec & (flags != neg_full)).any(), (s, h, int((~rec & (flags != neg_full)).sum()))
            assert not (~rec[chunk - 4096:chunk] & (part != neg_full[chunk - 4096:chunk])).any(), (s, h)
            last = F.stages_from_lists(n - chunk, la, lb)
            first = F.stages_from_lists(4096, pa, pb)
            assert (st_part["prior"], st_part["head"], st_part["refined"]) == (
                int((first == 1).sum()), int((first == 2).sum()), int((first == 3).sum()))
            stage = np.concatenate((first, last))
            fl = np.concatenate((part, flags[chunk:]))
            t0 = time.time()
            hd = np.flatnonzero(stage == 2)
            sel = np.union1d(np.flatnonzero(stage == 3), hd[::max(1, len(hd) // 200)])
            F.exact_decrease(tables, spec, z, 2, terms, sel[np.isnan(sfull[sel, 0].astype(np.float64))],
                             pl["dfull"], pl["B"], sfull)
            tight = max(tight, _check_subset_bound(name, tables, terms, sfull, sel, resid))
            _CPU["reference seconds"] += time.time() - t0
            fails, rep = F.audit(pl["place"], stage, fl, thr, e1, e2, pl["dfull"], pl["B"], neg_full[rows], dt["mag"])
            _REPORT.append("%-34s %-4s %-6s stage 1: %6d decided, min margin/G %8.3g | head: %6d decided, min "
                           "margin/G %8.3g | refined %5d | +-0.01B disagreements %d"
                           % (name, s, h, rep["stage 1 decided"], rep["stage 1 min margin / G"],
                              rep["stage 2 decided"], rep["stage 2 min margin / G"], int((stage == 3).sum()),
                              rep["+-0.01B disagreements"]))
            assert not fails, (s, h, fails)
    _REPORT.append("%-34s classes %s" % (name, {k: v for k, v in counts.items() if v}))
    _REPORT.append("%-34s sigma_S >= sigma_full: largest rounding allowance / sigma_full^2 %.2g" % (name, tight))


def test_five_factors():
    """Five distinct factors: four factors' head tables in shared memory, the fifth read from global memory."""
    wl = _workload(5, 1, 200, [6, 6, 6, 6, 6], seed=77)
    assert wl["lyap"].sweep_descriptor().gp.num_factors == 5
    _gp_workload_case("five factors", wl, [6, 6, 6, 6, 6], ("fp64",), 77)


def test_empty_factor():
    wl = _workload(3, 1, 120, [13, 11, 12], seed=78, empty=1)
    desc = wl["lyap"].sweep_descriptor()
    assert any(desc.gp.factors[f].M == 0 for f in range(desc.gp.num_factors))
    _gp_workload_case("empty factor", wl, [13, 11, 12], ("fp32", "fp64"), 78)
