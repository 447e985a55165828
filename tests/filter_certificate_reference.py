"""The certificates of the decision filter (csrc/filter.cu, ``slb_lyapunov_sweep_filtered``) restated in long
double, and the audit that holds a filtered sweep to them.

The filter decides a point in stage 1 or in the head stage only when the comparison

    D(sigma) = V(mu) - V(x) + sum_j L_V(mu)_j beta_j sigma_j  <  thr = -L_V(x) (1 + L_f) tau

has the same outcome for every sigma_j in [0, s_j], with s = the prior sigma (stage 1) or the sigma given the
head subset S (head stage), and a guard band.  With c_j = L_V(mu*)_j beta_j and D0 = V(mu*) - V(x):

    D_hi(s) = D0 + sum_j max(c_j s_j, 0),   D_lo(s) = D0 + sum_j min(c_j s_j, 0)
    G(s)    = 1e-6 (|V(mu*)| + |V(x)| + |thr| + sum_j |L_V(mu*)_j mu*_j| + sum_j |c_j s_j|)

(``mean_decision_terms`` and ``decide``).  A decided negative point must have D_hi(s) < thr, a decided
non-negative one D_lo(s) >= thr, for the EXACT posterior mean mu* and the stage's own sigma bound.  Everything
here starts from the product's tables (tests/gp_posterior_reference.py ``stack_tables``, plus the head
tables of ``head_tables``) and runs in ``np.longdouble``:

* mu*: k . (L^-T alpha) + the prior mean, with L^-1 and alpha of the product (O(M) per point);
* sigma_prior: sqrt(variance) for the plain RBF, sqrt(Kdiag(z)) for a covariance expression;
* sigma_S: from ``Whead`` = L_S^-1 and ``Xhead`` (O(|S|^2) per point); checked against a long-double
  Cholesky of scale^2 (K_SS + noise I) written below (numpy has none) by ``check_head_factor``;
* sigma_full: the posterior of gp_posterior_reference.py, O(M^2) per point -- only where it is needed.

The audit (``audit``) is a pure function of the certificate arrays, the placement of every point (which
edge its threshold sits next to, ``PLACEMENTS``) and what the filter did (the stage that decided each point,
its flag).  tests/test_filter_certificate_host.py drives it with a simulated filter and its mutants;
tests/test_gpu_filter_certificates.py with the kernels.
"""
import numpy as np

import gp_posterior_reference as R

LD = np.longdouble
U = 2.0 ** -53
GUARD = 1e-6                      # the relative guard band of mean_decision_terms / decide
EPS_K = 1e-13                     # gp_mean_staged.cuh: certified relative error of a kernel value
TOL = 1e-15                       # "exactly": long-double tolerance relative to the magnitudes

# one placement per point: (stage of the edge, edge, kind) -- see edge_targets
PLACEMENTS = ("neutral",
              "s1_hi_hair", "s1_hi_guard", "s1_hi_live", "s1_lo_hair", "s1_lo_guard", "s1_lo_live",
              "hd_hi_hair", "hd_hi_guard", "hd_hi_live", "hd_lo_hair", "hd_lo_guard", "hd_lo_live",
              "true_p10", "true_m10", "true_p2", "true_m2", "true_p001", "true_m001")
TRUE_K = {"true_p10": 10.0, "true_m10": -10.0, "true_p2": 2.0, "true_m2": -2.0,
          "true_p001": 0.01, "true_m001": -0.01}
RECORDED = ("true_p001", "true_m001")          # flags there are recorded, not asserted


# ------------------------------------------------------------------------ tables
def head_tables(stack, tables):
    """Attach the filter's tables of every factor (device read-back, needs the GPU): Whead as L_S^-1
    [r, r] (lower triangular), Xhead [r, d_in], noise, hmax; gamma_l1 of every output."""
    desc = stack.gp_stack()
    members = getattr(stack, "functions", [stack])
    for o, member in enumerate(members):
        gp = member.gaussian_process
        fac = tables["outputs"][o]["factor"]
        if "Whead" not in fac:
            F = gp._factor
            r = int(F.head_rows)
            W = F.Whead.cpu().numpy()
            fac.update(Whead=np.ascontiguousarray(W[:r, :r].T), Xhead=F.Xhead.cpu().numpy()[:r].copy(),
                       noise=float(gp.likelihood.variance), hmax=float(desc.factors[fac["index"]].hmax))
        tables["outputs"][o]["gamma_l1"] = float(desc.outputs[o].gamma_l1)
    return tables


def cholesky_ld(A):
    """Lower Cholesky factor of a symmetric positive definite matrix in long double."""
    A = np.asarray(A, dtype=LD)
    n = A.shape[0]
    L = np.zeros((n, n), dtype=LD)
    for j in range(n):
        d = A[j, j] - L[j, :j] @ L[j, :j]
        L[j, j] = np.sqrt(d)
        L[j + 1:, j] = (A[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return L


def lower_inverse_ld(L):
    n = L.shape[0]
    X = np.zeros((n, n), dtype=LD)
    eye = np.eye(n, dtype=LD)
    for i in range(n):
        X[i] = (eye[i] - L[i, :i] @ X[:i]) / L[i, i]
    return X


def train_gram(fac, X):
    """scale^2 (K(X, X) + noise I) in long double, K as gpflow forms it for training inputs: the cross kernel,
    plus on the diagonal the product terms that hold a White primitive (zero across points, their variance
    product on the diagonal).  X in the factor's units (Xs / Xhead)."""
    r = X.shape[0]
    if not fac["prims"]:
        Xl = X.astype(LD)
        t = ((Xl[:, None, :] - Xl[None, :, :]) ** 2).sum(axis=2)
        K = LD(fac["variance"]) * np.exp(-t / 2)
    else:
        s2 = LD(fac["scale"]) ** 2
        K = R._kernel_values(dict(fac, Xs=X, M=r), X, X.shape[1], LD)[0] / s2
        white_terms = {p[1] for p in fac["prims"] if p[0] == R.K_WHITE}
        if white_terms:
            sub = dict(fac, Xs=X, M=r, prims=[p for p in fac["prims"] if p[1] in white_terms])
            K = K + np.diag(R._kernel_values(sub, X, X.shape[1], LD)[2] / s2)
    s2 = LD(fac["scale"]) * LD(fac["scale"])
    return s2 * (K + LD(fac["noise"]) * np.eye(r, dtype=LD))


def head_gram(fac):
    """scale^2 (K(X_S, X_S) + noise I) in long double."""
    return train_gram(fac, fac["Xhead"])


def check_head_factor(fac):
    """(rel, residual, cond): the relative difference of the product's L_S^-1 from the long-double one;
    |W A W^T - I|_2 of the product's factor W, which bounds the relative error of |W k|^2 against the exact
    k^T A^-1 k, so of the head variance's subtracted part; and cond_2(A), which bounds both to about
    |S| u cond(A) for any backward-stable factorisation.  (None, None, None) without a head subset."""
    A = head_gram(fac)
    if A.shape[0] == 0:
        return None, None, None
    Wl = lower_inverse_ld(cholesky_ld(A))
    W = fac["Whead"].astype(LD)
    rel = float(np.max(np.abs(W - Wl)) / np.max(np.abs(Wl)))
    E = W @ A @ W.T - np.eye(A.shape[0], dtype=LD)
    return rel, float(np.linalg.norm(E.astype(np.float64), 2)), float(np.linalg.cond(A.astype(np.float64)))


def full_factor_residual(fac, noise=None):
    """|L^-1 A L^-T - I|_2 of the product's full factor, A = scale^2 (K(X, X) + noise I) (O(M^3))."""
    if fac["M"] == 0:
        return 0.0
    A = train_gram(dict(fac, noise=fac["noise"] if noise is None else noise), fac["Xs"])
    W = fac["Linv"].astype(LD)
    return float(np.linalg.norm((W @ A @ W.T).astype(np.float64) - np.eye(fac["M"]), 2))


# ------------------------------------------------------------------------ V and L_V
def fn_spec(P, v_scale=1.0, lv="abs-linear", A=None, lv_scale=1.0, lv_const=None):
    """V = v_scale * x^T P x and one of the L_V forms screening_applicable accepts: "const" (lv_const),
    "abs-linear" |x A^T| (per output), "norm1" sum |x A^T|, "linear" x A^T (no abs), each times lv_scale."""
    return dict(P=np.asarray(P, dtype=np.float64), v_scale=float(v_scale), lv=lv,
                A=None if A is None else np.asarray(A, dtype=np.float64), lv_scale=float(lv_scale),
                lv_const=lv_const)


def V(spec, y):
    y = np.asarray(y, dtype=LD)
    return LD(spec["v_scale"]) * ((y @ spec["P"].astype(LD)) * y).sum(axis=1)


def LV(spec, y):
    """L_V's columns at y [n, D] (1 column for const and norm1)."""
    y = np.asarray(y, dtype=LD)
    if spec["lv"] == "const":
        return np.full((y.shape[0], 1), LD(spec["lv_const"]))
    t = y @ spec["A"].T.astype(LD)
    if spec["lv"] in ("abs-linear", "norm1"):
        t = np.abs(t)
    if spec["lv"] == "norm1":
        t = t.sum(axis=1, keepdims=True)
    return LD(spec["lv_scale"]) * t


def lv_threshold(spec, x):
    """L_V(x) as the threshold takes it (lyapunov_state_terms): the 1-norm of several columns."""
    t = LV(spec, x)
    return np.abs(t).sum(axis=1) if t.shape[1] > 1 else t[:, 0]


def threshold_fp64(lvx, lf, tau):
    """The device's threshold: fl(fl(-lv * fl(1 + lf)) * tau)."""
    lvx = np.asarray(lvx, dtype=np.float64)
    return (-lvx * (1.0 + np.asarray(lf, dtype=np.float64))) * float(tau)


def lf_for(lvx, target, tau):
    """The tabulated L_f that puts the threshold at `target`."""
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.asarray(target, dtype=np.float64) / (-np.asarray(lvx, dtype=np.float64) * float(tau)) - 1.0


# ------------------------------------------------------------------------ per-point quantities
def _gamma(out):
    fac = out["factor"]
    if fac["M"] == 0:
        return np.zeros(0, dtype=LD)
    return fac["Linv"].astype(LD).T @ out["alpha"].astype(LD)


def point_terms(tables, z):
    """mu* [n, D], sigma_prior [n, D], sigma_S [n, D], the largest kernel value [n, D] (the mean error bound's
    kbound for expressions) and |zs|^2 / 2 [n, D] at the fp64 query points z."""
    din = tables["din"]
    z = np.asarray(z, dtype=np.float64).reshape(-1, din)
    n, D = z.shape[0], len(tables["outputs"])
    mu, sp, ss = (np.zeros((n, D), dtype=LD) for _ in range(3))
    kmax, half = np.zeros((n, D)), np.zeros((n, D))
    cache = {}
    for o, out in enumerate(tables["outputs"]):
        fac = out["factor"]
        s = LD(fac["scale"])
        s2 = s * s
        if id(fac) not in cache:
            k, _, kss, _ = R._kernel_values(fac, z, din, LD)
            prior_var = LD(fac["variance"]) if not fac["prims"] else kss / s2
            r = fac["Whead"].shape[0] if "Whead" in fac else 0
            if r > 0:
                kS = R._kernel_values(dict(fac, Xs=fac["Xhead"], M=r), z, din, LD)[0]
                aS = kS @ fac["Whead"].astype(LD).T
                var_s = (kss - (aS * aS).sum(axis=1)) / s2
            else:
                var_s = np.broadcast_to(prior_var, (n,)).astype(LD)
            km = (np.max(np.abs(k), axis=1) / s2).astype(np.float64) if fac["M"] else np.zeros(n)
            zs = z / fac["lengthscales"] if not fac["prims"] else z
            cache[id(fac)] = (k, np.broadcast_to(prior_var, (n,)), var_s, km, (zs * zs).sum(axis=1) / 2)
        k, pv, vs, km, hz = cache[id(fac)]
        mx = LD(0)
        if out["prior"] is not None:
            mx = s * (z.astype(LD) * out["prior"].astype(LD)).sum(axis=1)
        dot = k @ _gamma(out) if fac["M"] else np.zeros(n, dtype=LD)
        mu[:, o] = (dot + mx) / s
        sp[:, o] = np.sqrt(pv)
        ss[:, o] = np.sqrt(np.maximum(vs, 0))
        kmax[:, o], half[:, o] = km, hz
    return dict(mu=mu, sigma_prior=sp, sigma_S=ss, kmax=kmax, half=half)


def sigma_full(tables, z):
    """The full posterior at z (O(M^2) per point): the reference dict of gp_posterior_reference.py."""
    return R.reference(tables, z)


def mean_error_term(tables, spec, terms, x):
    """4 sum_j |L_V(mu)_j| eps_j gamma_l1_j / |scale| (the fp64 mean's bound through L_V, DESIGN section 3.5)."""
    mu = terms["mu"]
    lv = LV(spec, mu).astype(np.float64)
    out = np.zeros(mu.shape[0])
    for j, o in enumerate(tables["outputs"]):
        fac = o["factor"]
        if fac["prims"]:
            eps, kb = 4.5e-16 + 7e-16 * (fac["M"] + 8), terms["kmax"][:, j]
        else:
            eps, kb = EPS_K + 4.5e-16 * (terms["half"][:, j] + fac.get("hmax", 0.0)) + 7e-16 * (fac["M"] + 8), 1.0
        l = lv[:, 0] if lv.shape[1] == 1 else lv[:, j]
        out += 4 * np.abs(l) * eps * kb * o.get("gamma_l1", 0.0) / abs(fac["scale"])
    return out


def screening_slack(spec, beta, mu, dm, shi):
    """filter.cu screening_slack restated: the change of the comparison over the box mu +- dm."""
    mu, dm, shi = (np.asarray(a, dtype=np.float64) for a in (mu, dm, shi))
    P = spec["P"]
    g = np.abs(mu @ (P + P.T))
    dv = (g * dm).sum(axis=1) + ((dm @ np.abs(P)) * dm).sum(axis=1)
    dv = dv * abs(spec["v_scale"])
    bs = np.abs(beta)[None, :] * shi
    dl = np.zeros(mu.shape[0])
    if spec["lv"] != "const":
        A = spec["A"]
        rows = dm @ np.abs(A).T
        if spec["lv"] == "norm1" or A.shape[0] == 1:
            dl = abs(spec["lv_scale"]) * rows.sum(axis=1) * bs.sum(axis=1)
        else:
            dl = abs(spec["lv_scale"]) * (rows * bs).sum(axis=1)
    with np.errstate(invalid="ignore"):
        return 1.000001 * (dv + dl)


def decision_terms(tables, spec, terms, x, thr):
    """The comparison's pieces at every point: D0, c [n, D], the sigma-free guard part g0 (so that
    G(s) = g0 + 1e-6 sum |c s|), and a magnitude for the long-double tolerance."""
    mu = terms["mu"]
    beta = np.array([o["beta"] for o in tables["outputs"]], dtype=LD)
    lv = LV(spec, mu)
    lvb = np.broadcast_to(lv, mu.shape) if lv.shape[1] == 1 else lv
    vm, vx = V(spec, mu), V(spec, x)
    thr = np.asarray(thr, dtype=LD)
    c = lvb * beta
    g0 = GUARD * (np.abs(vm) + np.abs(vx) + np.abs(thr) + np.abs(lvb * mu).sum(axis=1))
    return dict(D0=vm - vx, c=c, g0=g0, thr=thr, mag=np.abs(vm) + np.abs(vx) + np.abs(thr)
                + np.abs(lvb * mu).sum(axis=1))


def decrease_bound(spec, x, ref):
    """B: the full kernel's certified error of decrease = V(mu) - V(x) + sum_j L_V(mu)_j err_j, from the
    mean and err bounds of gp_posterior_reference.py (first and second order through V and L_V) plus the
    decision's own fp64 rounding, (2 D + 8) u times its magnitudes (test_gpu_gp_shapes.py _decrease_bound,
    for every V / L_V form of fn_spec)."""
    mu, err = ref["mean"], ref["err"]
    D = mu.shape[1]
    P = spec["P"].astype(LD)
    aP = np.abs(P) * abs(LD(spec["v_scale"]))
    x = np.asarray(x, dtype=LD)
    dmu = ref["mean_bound"].astype(LD)
    v, dv, beta = ref["var"], ref["var_bound"].astype(LD), ref["beta"]
    with np.errstate(invalid="ignore", divide="ignore"):
        derr = np.fmin(beta * dv / (np.sqrt(np.maximum(v, 0)) + np.sqrt(np.maximum(v - dv, 0))),
                          beta * np.sqrt(dv)) + 2 * U * err
    lv = LV(spec, mu)
    lvb = np.abs(np.broadcast_to(lv, mu.shape) if lv.shape[1] == 1 else lv)
    g = np.abs(mu @ (P + P.T)) * abs(LD(spec["v_scale"]))
    if spec["lv"] == "const":
        dl, al = np.zeros_like(mu), np.zeros_like(mu)
    else:
        A = np.abs(spec["A"].astype(LD)) * abs(LD(spec["lv_scale"]))
        dl, al = dmu @ A.T, np.abs(mu) @ A.T
        if spec["lv"] == "norm1" or A.shape[0] == 1:
            dl = np.broadcast_to(dl.sum(axis=1, keepdims=True), mu.shape)
            al = np.broadcast_to(al.sum(axis=1, keepdims=True), mu.shape)
    return ((g * dmu).sum(axis=1) + ((dmu @ aP) * dmu).sum(axis=1) + (dl * (err + derr)).sum(axis=1)
            + (lvb * derr).sum(axis=1)
            + (2 * D + 8) * U * 1.01 * (((np.abs(x) @ aP) * np.abs(x)).sum(axis=1)
                                         + ((np.abs(mu) @ aP) * np.abs(mu)).sum(axis=1)
                                         + ((lvb + al) * err).sum(axis=1)))


def edges(dt, s, guard=GUARD, c=None):
    """(D_hi(s), D_lo(s), G(s)) at every point; `guard` and `c` replaceable for the mutants."""
    cs = (dt["c"] if c is None else c) * np.asarray(s, dtype=LD)
    return (dt["D0"] + np.maximum(cs, 0).sum(axis=1), dt["D0"] + np.minimum(cs, 0).sum(axis=1),
            guard * (dt["mag"] + np.abs(cs).sum(axis=1)))


# ------------------------------------------------------------------------ placements
def assign(n, eligible, seed=0, weights=None):
    """One placement per point from a fixed rule: the points eligible for a placement are dealt round-robin
    (in a seeded random order) over the placements they are eligible for.  eligible: dict name -> bool [n]."""
    names = [p for p in PLACEMENTS if p != "neutral"]
    out = np.array(["neutral"] * n, dtype=object)
    order = np.random.default_rng(seed).permutation(n)
    counts = {p: 0 for p in names}
    w = weights or {}
    for i in order:
        opts = [p for p in names if eligible.get(p) is not None and eligible[p][i]]
        if not opts:
            continue
        p = min(opts, key=lambda q: (counts[q] / w.get(q, 1.0), names.index(q)))
        out[i] = p
        counts[p] += 1
    return out


def edge_targets(place, e1, e2, slack1, slack2, dfull, B, neutral):
    """The threshold each placement asks for.  e1 / e2: (D_hi, D_lo, G) at sigma_prior / sigma_S; slack1 /
    slack2: each stage's full restated slack (G plus its mean-error term); dfull, B: the exact decrease and
    the full kernel's certified error (NaN where not computed); neutral: the threshold elsewhere."""
    t = np.array(neutral, dtype=LD)
    for stage, (hi, lo, G), S in (("s1", e1, slack1), ("hd", e2, slack2)):
        for edge, E, sgn in (("hi", hi, 1), ("lo", lo, -1)):
            for kind, off in (("hair", -1e-6 * G), ("guard", 0.5 * G), ("live", 10 * S)):
                m = place == "%s_%s_%s" % (stage, edge, kind)
                t[m] = (E + sgn * off)[m]
    for name, k in TRUE_K.items():
        m = place == name
        t[m] = (dfull + k * B)[m]
    return t


def certify(tables, spec, x, terms, thr):
    """(decision terms, (D_hi, D_lo, G) at sigma_prior, the same at sigma_S) for thresholds thr."""
    dt = decision_terms(tables, spec, terms, x, thr)
    return dt, edges(dt, terms["sigma_prior"]), edges(dt, terms["sigma_S"])


def exact_decrease(tables, spec, z, d, terms, rows, dfull, B, sfull=None):
    """Fill dfull / B (NaN-initialised [n]) and, if given, sigma_full [n, D] at `rows` from the full posterior
    (O(M^2) per point).  Returns sigma_full at the rows not computed before (None if there are none)."""
    rows = np.asarray(rows, dtype=np.int64)
    rows = rows[np.isnan(np.asarray(dfull[rows], dtype=np.float64))]
    if rows.size == 0:
        return
    ref = sigma_full(tables, z[rows])
    sub = {k: v[rows] for k, v in terms.items()}
    dt = decision_terms(tables, spec, sub, z[rows, :d], np.zeros(rows.size))
    sig = np.sqrt(np.maximum(ref["var"], 0))
    dfull[rows] = dt["D0"] + (dt["c"] * sig).sum(axis=1)
    B[rows] = decrease_bound(spec, z[rows, :d], ref)
    if sfull is not None:
        sfull[rows] = sig
    return sig


def plan(tables, spec, z, d, tau, lf_neutral, extra1, extra2, seed=0, head_classes=True, lo_head=None,
         terms=None, true_weight=1.0, gap_extra=None, focus=None, sfull=None):
    """One placement per point and its threshold target.  extra1 / extra2 [n]: each stage's restated slack
    beyond the 1e-6 guard (mean-error term or screening_slack; inf: that stage cannot decide the point).
    Excluded (neutral): L_V(x) = 0, and head placements where the head edge lies within 20 slacks of stage
    1's (sigma_S ~ sigma_prior: far from data, or no head subset).  Returns a dict with place, target, lf,
    the terms, and dfull / B filled at the true-edge placements."""
    n = z.shape[0]
    x = z[:, :d]
    terms = point_terms(tables, z) if terms is None else terms
    lvx = lv_threshold(spec, x).astype(np.float64)
    neutral = threshold_fp64(lvx, np.full(n, lf_neutral), tau)
    ok = np.isfinite(lvx) & (np.abs(lvx) > 1e-9 * np.max(np.abs(lvx)))
    if focus is not None:                 # placements only there (the rest keeps the neutral threshold)
        ok &= focus
    dt, e1, e2 = certify(tables, spec, x, terms, neutral)
    S1 = (e1[2] + extra1).astype(np.float64)
    S2 = (e2[2] + extra2).astype(np.float64)
    S1gap = S1 if gap_extra is None else (e1[2] + gap_extra).astype(np.float64)
    el = {}
    for edge, k in (("hi", 0), ("lo", 1)):
        gap = np.abs(np.asarray(e1[k] - e2[k], dtype=np.float64))
        for kind in ("hair", "guard", "live"):
            el["s1_%s_%s" % (edge, kind)] = ok & (np.isfinite(S1) if kind == "live" else ok)
            use = head_classes and (edge == "hi" or lo_head is None or lo_head)
            # a head edge apart from stage 1's (a live one so far that stage 1 cannot decide it)
            apart = gap > (20 * S1gap if kind == "live" else 2 * e1[2].astype(np.float64))
            el["hd_%s_%s" % (edge, kind)] = ok & use & apart & np.isfinite(S2)
    for name in TRUE_K:
        el[name] = ok
    place = assign(n, el, seed, {name: true_weight for name in TRUE_K})
    dfull = np.full(n, np.nan, dtype=LD)
    B = np.full(n, np.nan, dtype=LD)
    exact_decrease(tables, spec, z, d, terms, np.flatnonzero(np.isin(place, list(TRUE_K))), dfull, B, sfull)
    target = edge_targets(place, e1, e2, S1, S2, dfull, B, neutral)
    for _ in range(2):                    # G depends on |thr| (1e-6 of it): settle the targets
        dt, e1, e2 = certify(tables, spec, x, terms, target)
        target = edge_targets(place, e1, e2, S1, S2, dfull, B, neutral)
    t64 = target.astype(np.float64)
    lf = np.where(place == "neutral", lf_neutral, lf_for(lvx, t64, tau))
    lf = np.where(ok, lf, lf_neutral)
    return dict(place=place, target=target, lf=lf, lvx=lvx, terms=terms, dfull=dfull, B=B, x=x, S1=S1, S2=S2)


# ------------------------------------------------------------------------ the audit
def audit(place, stage, flag, thr, e1, e2, dfull=None, B=None, full_flag=None, tol_mag=None):
    """Every expectation of the filter, as a pure function of the placements, the observed stage (1: stage 1,
    2: head, 3: refine) and flag of every point.  e1 / e2: (D_hi, D_lo, G) at sigma_prior and sigma_S from the
    exact mean; dfull / B (NaN where not computed): the exact decrease at sigma_full and the full kernel's
    error bound; full_flag: the full sweep's flags.  Returns (failures: list of strings, report: dict)."""
    fails, rep = [], {}
    thr = np.asarray(thr, dtype=LD)
    stage = np.asarray(stage)
    flag = np.asarray(flag).astype(bool)
    tol = TOL * (np.asarray(tol_mag, dtype=LD) if tol_mag is not None else np.abs(thr))

    def fail(what, mask):
        idx = np.flatnonzero(mask)
        if idx.size:
            fails.append("%s: %d points, e.g. %s" % (what, idx.size, idx[:8].tolist()))

    for s, (hi, lo, G) in ((1, e1), (2, e2)):
        dec = stage == s
        neg_m = thr - hi                     # exact margin of a negative decision
        pos_m = lo - thr                     # ... of a non-negative one
        margin = np.where(flag, neg_m, pos_m)
        fail("stage %d soundness" % s, dec & (margin < -tol))
        fail("stage %d guard (margin < 0.5 G)" % s, dec & (margin < 0.5 * G))
        rep["stage %d decided" % s] = int(dec.sum())
        with np.errstate(invalid="ignore", divide="ignore"):
            ratio = margin / G
        rep["stage %d min margin / G" % s] = float(np.min(ratio[dec])) if dec.any() else float("nan")
        tag = "s1" if s == 1 else "hd"
        for edge, out in (("hi", True), ("lo", False)):
            fail("%s_%s_hair decided by its stage with the edge's outcome" % (tag, edge),
                 (place == "%s_%s_hair" % (tag, edge)) & dec & (flag == out))
            fail("%s_%s_guard decided by its stage" % (tag, edge), (place == "%s_%s_guard" % (tag, edge)) & dec)
            live = place == "%s_%s_live" % (tag, edge)
            fail("%s_%s_live not decided by stage <= %d with the edge's outcome" % (tag, edge, s),
                 live & ~((stage <= s) & (flag == out)))
    if dfull is not None:
        dfull = np.asarray(dfull, dtype=LD)
        known = ~np.isnan(dfull.astype(np.float64))
        exact = np.zeros(len(thr), dtype=bool)
        exact[known] = dfull[known] < thr[known]
        for name in TRUE_K:
            if name not in RECORDED:
                fail("%s flag != exact outcome" % name, (place == name) & known & (flag != exact))
        clear = known & (np.abs(dfull - thr) > np.asarray(B, dtype=LD))
        fail("flag != exact outcome clear of B", clear & (flag != exact))
        rep["exact outcome checked"] = int(clear.sum())
    if full_flag is not None:
        full_flag = np.asarray(full_flag).astype(bool)
        rec = np.isin(place, RECORDED)
        fail("flag != full sweep's", ~rec & (flag != full_flag))
        rep["+-0.01B disagreements"] = int((rec & (flag != full_flag)).sum())
    rep["classes"] = {p: int((place == p).sum()) for p in PLACEMENTS}
    return fails, rep


def stages_from_lists(n, list_a, list_b):
    """1 / 2 / 3 per point from the filter's lists (stage 1: not in list A; head: in A, not in B)."""
    st = np.ones(n, dtype=np.int64)
    st[np.asarray(list_a, dtype=np.int64)] = 2
    st[np.asarray(list_b, dtype=np.int64)] = 3
    return st
