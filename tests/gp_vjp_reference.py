"""Extended-precision reference of the GP posterior's reverse mode (``slb_gp_vjp``, csrc/gp_grad.cu) and a
computed bound of its rounding error at every point and input column.

Inputs are the tables the kernels read, as ``gp_posterior_reference.stack_tables`` reads them back from the
device (``fac.Xs``, the UNPACKED ``fac.Linv`` -- so that an error of ``slb_pack_factor`` or of the kernel's
decoding of the packed groups shows as a difference --, scale, lengthscales, kss, the ``slb_kernel`` normal
form, each output's beta and prior-mean row), plus each output's ``_gamma_dev`` (``vjp_tables``).  The
reference repeats the kernel's mathematics (header of gp_grad.cu) in ``np.longdouble``.  For output o on
factor f with cotangents g_o (mean) and h_o (err), with K = s^2 k(X, z), a = L^-1 K, b_c = L^-1 d_c K:

    mean part  G_c = sum_o g_o m_o,c + s sum_j (sum_{o on f} g_o gamma_o,j) d_c k_f(z, x_j)   (per factor f)
    var_f      = (s^2 k**(z) - sum_i a_i^2) / s^2                    (computed again, as the err kernel does)
    d_c var_f  = d_c k**(z) - (2 / s^2) sum_i a_i b_i,c
    err part   E_c = sum_o h_o beta_o / (2 sqrt(var_f(o))) d_c var_f(o)

Kernel gradients carry the product rule inside each term: d_c prod_p v_p = sum_p d_c v_p prod_{q != p} v_q.
Stationary primitives: delta_c = (z_c - x_c) w_c^2, d_c v = s(r) delta_c with s = -v (RBF), -e / r (Matern
1/2, e = var exp(-r)), -3 e (Matern 3/2, e = var exp(-sqrt3 r)), -(5/3)(1 + sqrt5 r) e (Matern 5/2, e = var
exp(-sqrt5 r)), r = sqrt(r^2 + 1e-12) as gpflow forms it; the diagonal of a stationary primitive is constant.
Linear: d_c = w_c x_c across points, 2 w_c z_c on the diagonal (the only nonzero d k** among the primitives).
Constant and White: zero gradient.  An inactive column has w_c = 0 and so an exactly zero kernel gradient.
The plain RBF works in zs = z / l, formed in fp64 as the kernel forms it: d_c k = -k (zs_c - Xs_c) / l_c.
Squared distances come from the differences, never from the expansion, so that points on and next to
training inputs are references too.

Error bound (standard model as in gp_posterior_reference: u = 2^-53, a sum of n terms in any order is off by
at most gamma_n sum |terms|, gamma_n <= 1.01 n u):

* Kernel values K_j, k** and their budgets e_j, e** are gp_posterior_reference's.  A kernel gradient
  d_c v = s delta_c of a stationary primitive: delta_c has 3 roundings (difference, two products by w_c),
  the product s delta_c one; s carries the value's relative budget rho (the exp's argument error and the
  ulps of exp and variance, as for the value) plus the roundings of its own factor: Matern 1/2 the relative
  error eps of r (as the value's eps_s) and the division, Matern 3/2 one product, Matern 5/2 eps of 1 + sqrt5
  r, the rounded 5/3 and two products.  So |d d_c v| <= |d_c v| (rho + eps_extra + 4u), and where the exp
  flushes (argument > 700) the budget is |d_c v| itself.  Linear: one product (2 w_c is exact).  The
  plain RBF: rho of its value plus the difference, the product by k and the division by l_c, 4u.
* A term's gradient from perturbed factors, by the product rule: sum_p (|d v_p| + e'_p) prod_{q != p}
  (|v_q| + e_q) - sum_p |d v_p| prod |v_q|, plus 3P u times that first sum for the kernel's P steps of
  (term * dv, fma, term *= v); the sum over T terms adds T u (|g| + budget); the product by s^2 two more u.
* Mean part: w_j = sum_o g_o gamma_o,j by D_f FMAs is off by 1.01 D_f u sum |g_o gamma_o,j|; the lanes' split
  sum and the butterfly over M rows of w_j d_c k_j: 1.01 M u sum |w_j d_c k_j| + sum |w_j| e'_j
  + sum e_w,j (|d_c k_j| + e'_j); the factor's s^2 acc / s three more u; the sum over factors and the
  prior-mean FMAs, n_t terms in all: 1.01 n_t u sum |terms|.
* Err part: A = |L^-1| |K|, B_c = |L^-1| |d_c K|, E = |L^-1| e, E'_c = |L^-1| e'_c (each contraction has
  at most M + 8 terms with the zero padding).  sum a^2: C_VAR u (M + 8) sum A^2 + 2 sum A E + sum E^2, and
  sum a b_c: C_VAR u (M + 8) sum A B_c + sum (A E'_c + B_c E) + sum E E'_c (C_VAR = 3.1: the contraction,
  the product and the reduction, with the O(u^2) terms).  var is bounded exactly as in the forward (dv);
  d_c var: [e**_c + 2 bound(sum a b_c) + 2u (|d_c k**| + 2 |sum a b_c|)] / s^2 + 2u |d_c var| (subtraction,
  rounded s^2, division).
* 1 / sqrt(var) where var is certified positive (var > dv): the computed var lies in [var - dv, var + dv],
  so 1 / sqrt is off by the relative rho_v = sqrt(var / (var - dv)) - 1; the coefficient h beta / (2 sqrt)
  adds 3 roundings (product, sqrt, division): rho_c = 1.01 (rho_v + 3u).  Each output's term
  coef d_c var is off by |coef| (dd (1 + rho_c) + |d_c var| rho_c), and the kernel's FMAs over the outputs
  add 1.01 D u sum |terms| (with their budgets).
* Both cotangents: the err kernel adds its sum to the mean kernel's result, one more u |sum|.

Rule where var is not certified positive (var <= dv, the interval given by var and its bound contains 0):
no value claim is made for the err part of that point (err-only and both modes); the point is counted in
``uncertified``.  A reference var of exactly 0 (a Linear-only kernel at z = 0) must give a non-finite err
gradient in every column, as torch's sqrt backward does (2 sqrt(0) = 0: inf times the gradient, NaN where
that is 0).  The mean-only mode always has a claim.

``fp64_other_order`` evaluates the same operation in plain fp64 numpy in another order (reversed
contractions and sums, numpy's exp) and must lie inside the bound; ``mutations`` perturbs the reference in
ways a subtly wrong kernel could, and ``mutation_ratio`` reports by how much each perturbation exceeds the
bound.
"""
import numpy as np

import gp_posterior_reference as R

LD, U = R.LD, R.U
C_VAR = R.C_VAR
FLUSH = 700


def vjp_tables(stack):
    """gp_posterior_reference.stack_tables plus each output's gamma (``_gamma_dev``, the mean kernel's
    weights)."""
    tables = R.stack_tables(stack)
    members = getattr(stack, "functions", [stack])
    for out, member in zip(tables["outputs"], members):
        gp = member.gaussian_process
        out["gamma"] = gp._gamma_dev.cpu().numpy()[:out["factor"]["M"]].astype(np.float64)
    return tables


def add_gamma(tables):
    """gamma = L^-T alpha for tables built on the host (the relation update_cache keeps on the device)."""
    for out in tables["outputs"]:
        out["gamma"] = out["factor"]["Linv"].T @ out["alpha"]
    return tables


# ------------------------------------------------------------------------ kernel gradients and their budget
def _prim_grad(kind, var, w, zz, X, din, dtype, diag):
    """Value, value budget, gradient [.., din] and gradient budget of one primitive (cross form [n, M], or
    diagonal form [n])."""
    n = zz.shape[0]
    shape = (n,) if diag else (n, X.shape[0])
    zero = np.zeros(shape, dtype=dtype)
    gzero = np.zeros(shape + (din,), dtype=dtype)
    if kind == R.K_LINEAR:
        if diag:
            prod = w * zz * zz
            g = 2 * w * zz
        else:
            prod = (w * zz)[:, None, :] * X[None, :, :]
            g = np.broadcast_to(w * X, shape + (din,)).astype(dtype)
        v = prod.sum(axis=-1)
        return v, (din + 1) * U * np.abs(prod).sum(axis=-1), g, U * np.abs(g)
    if kind == R.K_CONSTANT:
        return np.full(shape, var), zero, gzero, gzero
    if kind == R.K_WHITE:
        return (np.full(shape, var) if diag else zero), zero, gzero, gzero
    if diag:
        return np.full(shape, var), zero, gzero, gzero
    diff = zz[:, None, :] - X[None, :, :]
    df = diff * w
    r2 = (df * df).sum(axis=2)
    delta = df * w
    theta = (din + 4) * U
    if kind == R.K_RBF:
        v = var * np.exp(-r2 / 2)
        rho = theta * r2 / 2 * 1.01 + 3 * U
        s, extra, arg = -v, 0.0, r2 / 2
    else:
        c = R._MATERN_C[kind].astype(dtype) if dtype is LD else dtype(float(R._MATERN_C[kind]))
        r = np.sqrt(r2 + dtype(1e-12))
        sr = c * r
        eps = ((din + 4) / 2 + 3) * U
        e = var * np.exp(-sr)
        rho = (sr * eps) * 1.01 + 2 * U
        arg = sr
        if kind == R.K_MATERN12:
            v, poly_eps = e, 0.0
            s, extra = -e / r, eps + U
        elif kind == R.K_MATERN32:
            v, poly_eps = (1 + sr) * e, 3 * U + 2 * eps
            s, extra = -3 * e, U
        else:
            v, poly_eps = (1 + sr + sr * sr / 3) * e, 3 * U + 2 * eps
            s, extra = -(dtype(5) / 3) * (1 + sr) * e, eps + 4 * U
        rho = rho + poly_eps + U                            # the value's budget (gp_posterior_reference)
    ev = np.abs(v) * rho
    ev = np.where(arg > FLUSH, np.abs(v) + 1e-300, ev)
    g = s[..., None] * delta
    eg = np.abs(g) * (rho + extra + 4 * U)[..., None]
    eg = np.where((arg > FLUSH)[..., None], np.abs(g) + 1e-300, eg)
    return v, ev, g, eg


def _expr_grad(fac, zz, X, din, dtype, diag, mutate=None):
    """Gradient [.., din] of the covariance expression and its budget, unscaled (product rule inside each
    term)."""
    terms = {}
    for kind, term, var, w in fac["prims"]:
        terms.setdefault(term, []).append((kind, dtype(var), w.astype(dtype)))
    n = zz.shape[0]
    shape = (n, din) if diag else (n, X.shape[0], din)
    g = np.zeros(shape, dtype=dtype)
    eg = np.zeros(shape, dtype=dtype)
    for prims in terms.values():
        parts = [_prim_grad(kind, var, w, zz, X, din, dtype, diag) for kind, var, w in prims]
        P = len(parts)
        tg = np.zeros(shape, dtype=dtype)
        hi = np.zeros(shape, dtype=dtype)
        lo = np.zeros(shape, dtype=dtype)
        for p in range(P):
            if mutate == "drop_product_term" and P > 1 and p == 0:
                continue
            other = np.ones(shape[:-1], dtype=dtype)
            ohi = np.ones(shape[:-1], dtype=dtype)
            olo = np.ones(shape[:-1], dtype=dtype)
            for q in range(P):
                if q != p:
                    other = other * parts[q][0]
                    ohi = ohi * (np.abs(parts[q][0]) + parts[q][1])
                    olo = olo * np.abs(parts[q][0])
            tg = tg + parts[p][2] * other[..., None]
            hi = hi + (np.abs(parts[p][2]) + parts[p][3]) * ohi[..., None]
            lo = lo + np.abs(parts[p][2]) * olo[..., None]
        g = g + tg
        eg = eg + (hi - lo) + 3 * P * U * hi
    T = len(terms)
    eg = eg + T * U * (np.abs(g) + eg)
    return g, eg


def _inactive(fac):
    """Columns on which no primitive of the expression acts (all weights 0)."""
    W = np.array([w for _, _, _, w in fac["prims"]])
    return (W == 0).all(axis=0)


def _cross_grads(fac, z, din, dtype, mutate=None):
    """d_c k(z, x_j) [n, M, din] (unscaled) and its budget."""
    X = fac["Xs"].astype(dtype)
    if not fac["prims"]:
        l = fac["lengthscales"]
        zs = (z / l).astype(dtype)                           # fp64 division, as the kernel does
        diff = zs[:, None, :] - X[None, :, :]
        t = (diff * diff).sum(axis=2)
        k = dtype(fac["variance"]) * np.exp(-t / 2)
        g = -k[..., None] * diff / l.astype(dtype)
        rho = (din + 3) * U * t / 2 * 1.01 + 2 * U
        eg = np.abs(g) * (rho + 4 * U)[..., None]
        eg = np.where((t / 2 > FLUSH)[..., None], np.abs(g) + 1e-300, eg)
        return g, eg
    return _expr_grad(fac, z.astype(dtype), X, din, dtype, False, mutate)


def _diag_grads(fac, z, din, dtype, mutate=None):
    """d_c k**(z) [n, din] (unscaled) and its budget; zero for the plain RBF."""
    n = z.shape[0]
    if not fac["prims"] or mutate == "drop_kdiag_grad":
        return np.zeros((n, din), dtype=dtype), np.zeros((n, din), dtype=dtype)
    return _expr_grad(fac, z.astype(dtype), None, din, dtype, True, mutate)


def _leak_fac(fac, mutate):
    """The factor with the leak applied to the value too (the mutation changes the weights)."""
    if mutate != "leak_inactive" or not fac["prims"]:
        return fac
    inact = _inactive(fac)
    prims = [(k, t, v, np.where(inact, 1e-2, w) if k not in (R.K_CONSTANT, R.K_WHITE) else w)
             for k, t, v, w in fac["prims"]]
    return dict(fac, prims=prims)


# ------------------------------------------------------------------------ the two parts of the VJP
def _factors(tables):
    out = []
    for o in tables["outputs"]:
        if not any(o["factor"] is f for f in out):
            out.append(o["factor"])
    return out


def _sum(x, axis, order):
    """A sum along `axis`, in reversed order for the fp64 cross-check (np.sum is pairwise)."""
    if order == "forward":
        return x.sum(axis=axis)
    return np.flip(x, axis=axis).sum(axis=axis)


def _parts(tables, z, gm, ge, dtype, mutate=None, order="forward"):
    """Mean part, err part [n, din], their bounds, the err part's claim mask and the zero-variance mask."""
    din = tables["din"]
    z = np.asarray(z, dtype=np.float64).reshape(-1, din)
    n = z.shape[0]
    outs = tables["outputs"]
    D = len(outs)
    gm = np.asarray(gm, dtype=np.float64).reshape(n, D).astype(dtype)
    ge = np.asarray(ge, dtype=np.float64).reshape(n, D).astype(dtype)
    if mutate == "swap_cotangents":
        i, j = _cotangent_pair(tables)
        gm[:, [i, j]], ge[:, [i, j]] = gm[:, [j, i]], ge[:, [j, i]]
    gmean = np.zeros((n, din), dtype=dtype)
    bmean = np.zeros((n, din), dtype=dtype)
    mterms = np.zeros((n, din), dtype=dtype)
    nterms = 0
    gerr = np.zeros((n, din), dtype=dtype)
    berr = np.zeros((n, din), dtype=dtype)
    eterms = np.zeros((n, din), dtype=dtype)
    claim = np.ones(n, dtype=bool)
    zero_var = np.zeros(n, dtype=bool)
    for fac0 in _factors(tables):
        fac = _leak_fac(fac0, mutate)
        M = fac["M"]
        mine = [o for o, out in enumerate(outs) if out["factor"] is fac0]
        s = dtype(fac["scale"])
        s2 = s * s
        dk, edk = _cross_grads(fac, z, din, dtype, mutate)           # [n, M, din]
        if mutate == "drop_last_row" and M:
            dk, edk = dk.copy(), edk.copy()
            dk[:, M - 1] = 0
            edk[:, M - 1] = 0
        # ---- mean part: one weight per row, folded over the outputs on this factor
        w = np.zeros((n, M), dtype=dtype)
        ew = np.zeros((n, M), dtype=dtype)
        for o in mine:
            gam = outs[o]["gamma"].astype(dtype)
            w = w + gm[:, o:o + 1] * gam[None, :]
            ew = ew + np.abs(gm[:, o:o + 1] * gam[None, :])
        ew = 1.01 * len(mine) * U * ew
        prod = w[..., None] * dk
        acc = _sum(prod, 1, order)
        eacc = (1.01 * M * U * np.abs(prod).sum(axis=1) + (np.abs(w)[..., None] * edk).sum(axis=1)
                + (ew[..., None] * (np.abs(dk) + edk)).sum(axis=1))
        part = s * acc
        gmean = gmean + part
        bmean = bmean + s * eacc + 3 * U * np.abs(part)
        mterms = mterms + np.abs(part) + s * eacc
        nterms += 1
        # ---- err part
        if not mine:
            continue
        k, e, kss, ekss = R._kernel_values(fac, z, din, dtype)        # s^2 k, s^2 k**
        dkss, edkss = _diag_grads(fac, z, din, dtype, mutate)
        dkss = s2 * dkss
        edkss = s2 * edkss * (1 + 2 * U) + 2 * U * np.abs(dkss)
        dK = s2 * dk
        edK = s2 * edk * (1 + 2 * U) + 2 * U * np.abs(dK)
        if mutate == "drop_last_row" and M:
            k, e = k.copy(), e.copy()
            k[:, M - 1] = 0
            e[:, M - 1] = 0
        L = fac["Linv"].astype(dtype)
        if mutate == "swap_packed_columns":
            L = L.copy()
            for g0 in range(0, M - 5, 8):
                L[:, [g0 + 1, g0 + 5]] = L[:, [g0 + 5, g0 + 1]]
        KK = np.concatenate((k[..., None], dK), axis=2)               # [n, M, 1 + din]
        EE = np.concatenate((e[..., None], edK), axis=2)
        cols = n * (1 + din)
        flat = KK.transpose(1, 0, 2).reshape(M, cols)
        unflat = lambda x: x.reshape(M, n, 1 + din).transpose(1, 0, 2)     # [n, M(i), 1 + din]
        if order == "forward":
            ab = unflat(L @ flat)
        else:
            ab = unflat(L[:, ::-1] @ flat[::-1])
        aL = np.abs(L)
        AB = unflat(aL @ np.abs(flat))
        EAB = unflat(aL @ EE.transpose(1, 0, 2).reshape(M, cols))
        if mutate == "drop_last_block" and M:
            keep = np.ones(M, dtype=bool)
            keep[8 * ((M - 1) // 8):] = False
            ab, AB, EAB = ab[:, keep], AB[:, keep], EAB[:, keep]
        a, A, E = ab[:, :, :1], AB[:, :, :1], EAB[:, :, :1]
        S = _sum(a * ab, 1, order)                                    # [n, 1 + din]: sum a^2, sum a b_c
        m8 = M + 8
        bS = (C_VAR * U * m8 * (A * AB).sum(axis=1) + (A * EAB).sum(axis=1) + (AB * E).sum(axis=1)
              + (E * EAB).sum(axis=1))
        var = (kss - S[:, 0]) / s2
        bvar = (bS[:, 0] + ekss + 2 * U * np.abs(kss)) / s2 + 2 * U * np.abs(var)
        two = {"two_over_s2_to_one_over_s2": 1, "two_over_s2_to_one_over_s": 1 / s}.get(mutate, 2)
        if mutate == "two_over_s2_to_one_over_s":
            dvar = dkss / s2 - two * S[:, 1:]
        else:
            dvar = (dkss - two * S[:, 1:]) / s2
        bdvar = ((edkss + 2 * bS[:, 1:] + 2 * U * (np.abs(dkss) + 2 * np.abs(S[:, 1:]))) / s2
                 + 2 * U * np.abs(dvar))
        ok = var > bvar
        claim &= ok
        zero_var |= var == 0
        with np.errstate(divide="ignore", invalid="ignore"):
            rv = np.where(ok, np.sqrt(var / np.where(ok, var - bvar, 1)) - 1, 0)
            rc = 1.01 * (rv + 3 * U)
            for o in mine:
                coef = ge[:, o] * dtype(outs[o]["beta"]) / (2 * np.sqrt(var))     # NaN where var < 0
                term = coef[:, None] * dvar
                eterm = np.abs(coef)[:, None] * (bdvar * (1 + rc[:, None]) + np.abs(dvar) * rc[:, None])
                gerr = gerr + term
                berr = berr + eterm
                eterms = eterms + np.abs(term) + eterm
    # prior-mean FMAs
    for o, out in enumerate(outs):
        prior = out["prior"]
        if mutate == "move_prior":
            prior = outs[(o + 1) % D]["prior"]
        if prior is None:
            continue
        t = gm[:, o:o + 1] * prior.astype(dtype)[None, :]
        gmean = gmean + t
        mterms = mterms + np.abs(t)
        nterms += 1
    bmean = bmean + 1.01 * nterms * U * mterms
    berr = berr + 1.01 * D * U * eterms
    if mutate == "swap_points" and n > 1:
        perm = np.arange(n)
        h = n // 2
        perm[0:2 * h:2], perm[1:2 * h:2] = np.arange(1, 2 * h, 2), np.arange(0, 2 * h, 2)
        gerr, berr, claim = gerr[perm], berr[perm], claim[perm]
    return dict(mean=gmean, mean_bound=bmean, err=gerr, err_bound=berr, claim=claim, zero_var=zero_var)


def reference(tables, z, gm, ge, mutate=None):
    """Long-double VJP at the fp64 points z [n, d_in] for cotangents gm, ge [n, D]: dict of the mean part,
    the err part and their sum [n, d_in], their bounds, ``claim`` (err part certified) and ``zero_var``."""
    r = _parts(tables, z, gm, ge, LD, mutate)
    r["both"] = r["mean"] + r["err"]
    r["both_bound"] = r["mean_bound"] + r["err_bound"] + U * (np.abs(r["both"]) + r["mean_bound"] + r["err_bound"])
    return r


def fp64_other_order(tables, z, gm, ge):
    """The same operation in plain fp64 numpy, summed in another order: mean part, err part, their sum."""
    r = _parts(tables, z, gm, ge, np.float64, order="reversed")
    return r["mean"], r["err"], r["mean"] + r["err"]


# ------------------------------------------------------------------------ comparisons
def _ratio(obs, want, bound):
    obs = np.asarray(obs, dtype=LD)
    d = np.abs(obs - want)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(d == 0, 0, d / bound)
    return np.where(np.isnan(obs), np.inf, r)


def ratios(ref, mean=None, err=None, both=None):
    """Largest |observed - reference| / bound over points and columns, for each mode given.  Err and both
    modes: only where the err part is certified; a zero reference variance must give non-finite columns."""
    out = {}
    if mean is not None:
        out["mean"] = float(np.max(_ratio(mean, ref["mean"], ref["mean_bound"]), initial=0.0))
    for key, obs in (("err", err), ("both", both)):
        if obs is None:
            continue
        obs = np.asarray(obs)
        r = _ratio(obs, ref[key], ref["%s_bound" % key])[ref["claim"]]
        worst = float(np.max(r, initial=0.0))
        zv = ref["zero_var"]
        if zv.any() and np.isfinite(obs[zv]).any():
            worst = np.inf
        out[key] = worst
    return out


def worst(r):
    return max(r.values()) if r else 0.0


def uncertified(ref):
    """Points where no value claim is made on the err part (var not certified positive)."""
    return int((~ref["claim"]).sum())


def check_not_too_tight(tables, z, gm, ge):
    """Ratio of the fp64 other-order evaluation's deviation to the bound (must be <= 1)."""
    ref = reference(tables, z, gm, ge)
    m, e, b = fp64_other_order(tables, z, gm, ge)
    return worst(ratios(ref, mean=m, err=e, both=b))


# ------------------------------------------------------------------------ mutations
MUTATIONS = ("drop_last_row", "drop_last_block", "swap_packed_columns", "swap_points", "swap_cotangents",
             "drop_product_term", "drop_kdiag_grad", "two_over_s2_to_one_over_s2", "two_over_s2_to_one_over_s",
             "move_prior", "leak_inactive")


def _cotangent_pair(tables):
    """Two outputs on one factor with data: their cotangents swapped move both parts."""
    outs = tables["outputs"]
    for i, a in enumerate(outs):
        for j, b in enumerate(outs):
            if i < j and a["factor"] is b["factor"] and a["factor"]["M"]:
                return i, j
    return None


def applicable_mutations(tables, n):
    """The perturbations that change anything for this stack and point count."""
    facs = _factors(tables)
    data = [f for f in facs if f["M"]]
    out = []
    if data:
        out += ["drop_last_row", "drop_last_block", "two_over_s2_to_one_over_s2"]
    if any(f["M"] >= 6 for f in facs):
        out.append("swap_packed_columns")
    linear = [f for f in facs if any(p[0] == R.K_LINEAR for p in f["prims"])]
    if n > 1 and (data or linear):                          # otherwise the err part is 0 everywhere
        out.append("swap_points")
    if _cotangent_pair(tables) is not None:
        out.append("swap_cotangents")
    if any(_product_term(f) for f in data):
        out.append("drop_product_term")
    if linear:
        out.append("drop_kdiag_grad")
    if any(f["scale"] != 1.0 for f in data):
        out.append("two_over_s2_to_one_over_s")
    priors = [o["prior"] for o in tables["outputs"]]
    if len(priors) > 1 and any(p is not None for p in priors) and \
            any(not _same(priors[o], priors[(o + 1) % len(priors)]) for o in range(len(priors))):
        out.append("move_prior")
    if any(f["prims"] and _inactive(f).any() and any(p[0] not in (R.K_CONSTANT, R.K_WHITE) for p in f["prims"])
           for f in data):
        out.append("leak_inactive")
    return out


def _same(a, b):
    if a is None or b is None:
        return a is None and b is None
    return np.array_equal(a, b)


def _product_term(fac):
    """A term of two or more primitives whose first primitive has a gradient."""
    terms = {}
    for p in fac["prims"]:
        terms.setdefault(p[1], []).append(p)
    return any(len(t) > 1 and t[0][0] not in (R.K_CONSTANT, R.K_WHITE) for t in terms.values())


def mutation_ratio(tables, z, gm, ge, mutation, ref=None):
    """Largest deviation of the perturbed reference from the reference, relative to the bound, over the
    mean-only and err-only modes: a kernel with that defect would be caught where this is > 1."""
    ref = reference(tables, z, gm, ge) if ref is None else ref
    mut = reference(tables, z, gm, ge, mutate=mutation)
    err = mut["err"].astype(np.float64)
    err[ref["zero_var"]] = np.nan
    return worst(ratios(ref, mean=mut["mean"].astype(np.float64), err=err))


def mutation_ratios(tables, z, gm, ge):
    n = np.asarray(z).reshape(-1, tables["din"]).shape[0]
    ref = reference(tables, z, gm, ge)
    return {m: mutation_ratio(tables, z, gm, ge, m, ref) for m in applicable_mutations(tables, n)}
