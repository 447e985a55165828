"""Without a GPU: the long-double certificates of tests/filter_certificate_reference.py and the sharpness of
the audit that tests/test_gpu_filter_certificates.py holds the filter to.

* The reference: sigma given a subset of the training set is never below the full posterior's (equal for
  the whole set), the long-double Cholesky against numpy's fp64 one, and the tabulated L_f that places a
  threshold lands within a few ulps of its target.
* Sharpness: a simulated filter on a numpy-built pendulum-like workload decides exactly from the restated
  certificates (stage 1 with the prior sigma, the head stage with sigma given the head subset, the rest from
  the full posterior).  It passes the audit; each of seven mutants of it -- the kinds of error a kernel could
  make: a head sigma 1e-5 too small, a guard band of 1e-7, the prior sigma without the scale, the prior sigma
  of the other factor, L_V's abs dropped from c_j, a head stage that decides nothing, a stage 1 that decides
  at 0.4 G -- fails it.
* slb_debug_filter_lists: its offsets against slb_filter_workspace, and its rejections.
"""
import ctypes as C

import numpy as np
import pytest
import scipy.linalg as sla

import filter_certificate_reference as F
import gp_posterior_reference as R

LD = np.longdouble


# ------------------------------------------------------------------------ a numpy-built workload
def _rbf(Xs, variance):
    t = ((Xs[:, None, :] - Xs[None, :, :]) ** 2).sum(axis=2)
    return variance * np.exp(-t / 2)


def _pivoted(K, r):
    """First r pivots of the pivoted Cholesky factorisation of K (greedy largest remaining variance)."""
    M = K.shape[0]
    d = np.diag(K).copy()
    L = np.zeros((M, r))
    picks = []
    for k in range(r):
        p = int(np.argmax(d))
        picks.append(p)
        L[:, k] = (K[:, p] - L[:, :k] @ L[p, :k]) / np.sqrt(d[p])
        d = d - L[:, k] ** 2
        d[picks] = -np.inf
    return np.array(picks)


def _factor(X, variance, lengthscales, scale, noise, index, head=64):
    M = X.shape[0]
    Xs = X / lengthscales
    K = _rbf(Xs, variance)
    A = scale ** 2 * (K + noise * np.eye(M))
    Linv = sla.solve_triangular(np.linalg.cholesky(A), np.eye(M), lower=True)
    r = min(M, head)
    S = _pivoted(K, r) if r else np.zeros(0, dtype=int)
    AS = scale ** 2 * (K[np.ix_(S, S)] + noise * np.eye(r))
    Whead = sla.solve_triangular(np.linalg.cholesky(AS), np.eye(r), lower=True) if r else np.zeros((0, 0))
    return dict(M=M, Xs=Xs, Linv=Linv, lengthscales=np.asarray(lengthscales, dtype=np.float64),
                variance=float(variance), scale=float(scale), kss=float(scale ** 2 * variance), prims=[],
                index=index, Whead=Whead, Xhead=Xs[S], noise=noise, hmax=float((Xs * Xs).sum(axis=1).max() / 2))


def _workload(M=120, scale=0.8, num=(41, 37), seed=3, noise=1e-4):
    """Two outputs on distinct RBF factors over z = [x0, x1, clip(-K x)], training inputs next to grid
    points, a linear prior mean, scale < 1; V = x^T P x, L_V = |2 P mu|."""
    rng = np.random.default_rng(seed)
    axes = [np.linspace(-1, 1, k) for k in num]
    x = np.column_stack([m.ravel() for m in np.meshgrid(*axes, indexing="ij")])
    Kp = np.array([[0.6, 0.9]])
    z = np.hstack((x, np.clip(-x @ Kp.T, -1, 1)))
    idx = rng.choice(len(z), M, replace=False)
    X = z[idx] + 1e-3 * rng.standard_normal((M, 3))
    prior = np.array([[0.98, 0.05, 0.01], [-0.1, 0.95, 0.1]])
    Y = X @ prior.T + 0.05 * np.sin(3 * X[:, :2]) + 1e-3 * rng.standard_normal((M, 2))
    outs = []
    for j, (v, ls) in enumerate(((0.004, [1.2, 1.4, 1.6]), (0.0025, [0.9, 1.1, 1.3]))):
        fac = _factor(X, v, np.array(ls), scale, noise, j)
        alpha = fac["Linv"] @ (scale * (Y[:, j] - X @ prior[j]))
        l1 = scale ** 2 * v * float((np.abs(fac["Linv"]).T @ np.abs(alpha)).sum())
        outs.append(dict(factor=fac, beta=2.0, alpha=alpha, prior=prior[j], gamma_l1=l1))
    Q = rng.standard_normal((2, 2))
    P = Q @ Q.T + 2 * np.eye(2)
    P /= np.abs(P).max()
    spec = F.fn_spec(P, lv="abs-linear", A=2 * P)
    tau = 0.5 * float(np.sum(2.0 / (np.asarray(num) - 1))) / 8
    return dict(tables=dict(din=3, outputs=outs), spec=spec, z=z, d=2, tau=tau, lf=1.3, scale=scale)


@pytest.fixture(scope="module")
def case():
    wl = _workload()
    tables, spec, z, d = wl["tables"], wl["spec"], wl["z"], wl["d"]
    n = len(z)
    zero = np.zeros(n)
    pl = F.plan(tables, spec, z, d, wl["tau"], wl["lf"], zero, zero, seed=1)
    thr = F.threshold_fp64(pl["lvx"], pl["lf"], wl["tau"])
    # the simulated refine pass needs the full posterior everywhere (small here)
    F.exact_decrease(tables, spec, z, d, pl["terms"], np.arange(n), pl["dfull"], pl["B"])
    return dict(wl, pl=pl, thr=thr)


# ------------------------------------------------------------------------ the reference
def test_subset_sigma_bounds_the_full_posterior():
    """sigma given a random subset >= sigma_full (to the factors' rounding), = when S is every point."""
    wl = _workload(M=80)
    tables = wl["tables"]
    rng = np.random.default_rng(5)
    z = np.vstack((wl["z"][rng.choice(len(wl["z"]), 150, replace=False)],
                   tables["outputs"][0]["factor"]["Xs"][:20] * tables["outputs"][0]["factor"]["lengthscales"]))
    full = R.reference(tables, z)["var"]
    for r in (0, 5, 31, 64, 80):
        for o in tables["outputs"]:
            fac = o["factor"]
            S = np.sort(rng.choice(fac["M"], r, replace=False)) if r < fac["M"] else np.arange(fac["M"])
            AS = fac["scale"] ** 2 * (_rbf(fac["Xs"][S], fac["variance"]) + fac["noise"] * np.eye(r))
            fac["Whead"] = (sla.solve_triangular(np.linalg.cholesky(AS), np.eye(r), lower=True) if r
                            else np.zeros((0, 0)))
            fac["Xhead"] = fac["Xs"][S]
        terms = F.point_terms(tables, z)
        for j, o in enumerate(tables["outputs"]):
            fac = o["factor"]
            res = F.check_head_factor(fac)[1] or 0.0
            slack = (res + F.full_factor_residual(fac, fac["noise"]) + 1e-15) * fac["variance"]
            vs = terms["sigma_S"][:, j] ** 2
            assert (vs >= full[:, j] - slack).all(), (r, j)
            assert (terms["sigma_S"][:, j] <= terms["sigma_prior"][:, j] * (1 + 1e-15)).all()
            if r == fac["M"]:
                assert np.max(np.abs(vs - full[:, j])) <= 1e-9 * fac["variance"], r


def test_long_double_cholesky_against_numpy():
    rng = np.random.default_rng(2)
    for n in (1, 2, 7, 64):
        B = rng.standard_normal((n, n))
        A = B @ B.T + n * np.eye(n)
        L = F.cholesky_ld(A)
        assert np.max(np.abs(L.astype(np.float64) - np.linalg.cholesky(A))) <= 1e-13 * np.abs(L).max()
        W = F.lower_inverse_ld(L)
        assert np.max(np.abs((W @ A.astype(LD) @ W.T).astype(np.float64) - np.eye(n))) <= 1e-16 * n * n
    fac = _workload()["tables"]["outputs"][0]["factor"]
    rel, res, cond = F.check_head_factor(fac)
    assert rel <= 1e-10 and res <= 1e-10, (rel, res, cond)


def test_placed_threshold_lands_on_its_target(case):
    pl, thr = case["pl"], case["thr"]
    placed = pl["place"] != "neutral"
    t = pl["target"].astype(np.float64)
    # a few ulps of the target, plus those of -L_V(x) tau that 1 + L_f loses when the target is far below it
    # (L_f near -1); the audit uses the thresholds as they land in any case
    scale = np.abs(pl["lvx"] * case["tau"])[placed]
    err = np.abs(thr[placed] - t[placed])
    assert (err <= 4 * np.spacing(np.abs(t[placed])) + 2 * np.spacing(scale)).all()
    assert np.median(err / np.spacing(np.abs(t[placed]))) <= 1.0


def test_every_class_is_populated(case):
    counts = {p: int((case["pl"]["place"] == p).sum()) for p in F.PLACEMENTS}
    for p in F.PLACEMENTS[1:]:
        if p.startswith("hd_lo"):          # c >= 0 (|2 P mu|): the head's lower edge is stage 1's, excluded
            assert counts[p] == 0
        else:
            assert counts[p] >= 20, counts


# ------------------------------------------------------------------------ the simulated filter
def simulate(dt, s_prior, s_S, dfull, thr, guard=F.GUARD, c=None, head=True, s1_frac=1.0):
    """Decide from the restated certificates: stage 1 with s_prior, the head with s_S, the rest exactly."""
    n = len(thr)
    stage = np.full(n, 3)
    flag = np.asarray(dfull < thr)
    open_ = np.ones(n, dtype=bool)
    for s, sig, frac in ((1, s_prior, s1_frac), (2, s_S, 1.0)):
        if s == 2 and not head:
            break
        hi, lo, G = F.edges(dt, sig, guard=guard, c=c)
        neg = open_ & (thr - hi > frac * G)
        pos = open_ & ~neg & (lo - thr >= frac * G)
        stage[neg | pos] = s
        flag[neg], flag[pos] = True, False
        open_ &= ~(neg | pos)
    return stage, flag


def _audit(case, **mut):
    pl, tables, spec = case["pl"], case["tables"], case["spec"]
    thr = case["thr"].astype(LD)
    terms = pl["terms"]
    dt, e1, e2 = F.certify(tables, spec, pl["x"], terms, thr)
    s_prior = mut.pop("s_prior", terms["sigma_prior"])
    s_S = terms["sigma_S"] * mut.pop("s_S_factor", 1.0)
    c = mut.pop("c", None)
    stage, flag = simulate(dt, s_prior, s_S, pl["dfull"], thr, c=c, **mut)
    full = np.asarray(pl["dfull"] < thr)
    return F.audit(pl["place"], stage, flag, thr, e1, e2, pl["dfull"], pl["B"], full, dt["mag"])


def test_simulated_filter_passes(case):
    fails, rep = _audit(case)
    assert not fails, fails
    assert rep["stage 1 decided"] > 0 and rep["stage 2 decided"] > 0


def _mutants(case):
    terms, tables, spec = case["pl"]["terms"], case["tables"], case["spec"]
    mu = terms["mu"]
    beta = np.array([o["beta"] for o in tables["outputs"]], dtype=LD)
    signed = (mu @ (2 * spec["P"]).astype(LD).T) * beta          # L_V = 2 P mu without the abs
    return {
        "sigma_S x (1 - 1e-5)": dict(s_S_factor=1 - 1e-5),
        "guard 1e-7": dict(guard=1e-7),
        "prior sigma without the scale": dict(s_prior=terms["sigma_prior"] * case["scale"]),
        "prior sigma of the other factor": dict(s_prior=terms["sigma_prior"][:, ::-1]),
        "c_j without the abs": dict(c=signed),
        "head decides nothing": dict(head=False),
        "stage 1 decides at 0.4 G": dict(s1_frac=0.4),
    }


@pytest.mark.parametrize("name", ["sigma_S x (1 - 1e-5)", "guard 1e-7", "prior sigma without the scale",
                                  "prior sigma of the other factor", "c_j without the abs",
                                  "head decides nothing", "stage 1 decides at 0.4 G"])
def test_every_mutant_fails_the_audit(case, name):
    fails, _ = _audit(case, **_mutants(case)[name])
    assert fails, "the audit does not notice: %s" % name


# ------------------------------------------------------------------------ slb_debug_filter_lists
@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from safe_learning_b200 import _native
    return _native.load()


@pytest.mark.parametrize("n", [0, 1, 7, 64, 65536, 1 << 22])
def test_filter_list_offsets(lib, n):
    off = (C.c_int64 * 3)(-1, -1, -1)
    assert lib.slb_debug_filter_lists(n, off) == 0
    o = list(off)
    ws = int(lib.slb_filter_workspace(n))
    assert o[0] == 0 and o[1] >= 3 * 8 and o[1] % 8 == 0
    assert o[2] == o[1] + 8 * n                       # list A: int64 [n]
    assert o[2] + 8 * n <= ws                         # list B: int64 [n], inside the workspace
    # the rest of the workspace is the entries' terms: the same per-point size at every n
    if n:
        per = (ws - o[1]) // n
        assert (ws - o[1]) == per * n and per > 16


def test_filter_list_offsets_rejected(lib):
    off = (C.c_int64 * 3)(-1, -1, -1)
    for n in (-1, (1 << 22) + 1, 1 << 40):
        assert lib.slb_debug_filter_lists(n, off) != 0
        assert list(off) == [-1, -1, -1]
    assert lib.slb_debug_filter_lists(10, None) != 0
    from safe_learning_b200 import _native
    assert "slb_debug_filter_lists" in _native.last_error()
