"""Extended-precision reference of the GP posterior kernel (``gp_tile_kernel``, csrc/gp_tile.cuh) and a
computed bound of the kernel's rounding error at every point and output.

Inputs are the product's own tables read back from the device: the scaled training inputs ``fac.Xs``,
``fac.Linv``, ``alpha`` (``GPRCached._alpha_dev``), and from the stack descriptor the lengthscales, variance,
scale, beta, prior-mean row and the covariance expression's normal form (``slb_kernel``).  The reference
repeats the kernel's arithmetic in ``np.longdouble`` (64-bit significand here):

    k_j = s^2 kappa(z, x_j),  a = L^-1 k,  mean = (a . alpha + s m(z)) / s,  var = (s^2 k** - sum a^2) / s^2,
    err = beta sqrt(var).

For the plain RBF, ``zs = z / l`` is formed in fp64 as the kernel forms it.  Covariance expressions follow
gpflow 0.4.0 (DESIGN section 3.3): ``r = sqrt(r^2 + 1e-12)`` for Matern, Linear with ARD weights, White zero
across points, diagonal ``k** = variance`` for stationary primitives.  The squared distance is taken from
the differences, not from the oracle's ``|x|^2 + |x'|^2 - 2 x.x'`` expansion: next to a training input that
expansion cancels to an absolute error of ~1e-19 |x|^2 even in long double, which through ``sqrt(. + 1e-12)``
is a relative error of ~1e-13 of a Matern value, far above the fp64 budget being tested.  Both start from
the same factor, so the comparison measures the kernel's error alone, not the Cholesky factorisation's.

Error bound (standard model: every fp64 operation rounds with relative error at most u = 2^-53;
gamma_n = n u / (1 - n u) <= 1.01 n u for n u <= 0.01; a sum of n terms in ANY order, and therefore the DMMA
accumulation, whose order is treated as arbitrary, is off by at most gamma_n sum |terms|):

* e_j, the budget of one generated kernel value |k^_j - k_j|.  An exp argument x with relative error
  theta moves exp(x) by the factor exp(|x| theta); the product value is then bounded as
  |x| theta (1 + 2u) + 2u (two ulps) -- ``exp_neg_tab`` is within one ulp of exp (tools/exp_neg_tab_check.c),
  one more for the primitives' scalar products.  Plain RBF: t = sum (zs - xs)^2 by d_in FMAs on rounded
  differences, theta <= (d_in + 3) u, so e_j = |k_j| ((d_in + 3) u t_j / 2 * 1.01 + 4u) (exp, times variance,
  times s^2, one spare), and e_j = |k_j| where exp_neg_tab flushes (t_j / 2 > 700).  Expressions: per
  primitive, stationary r^2 = sum ((z - x) w)^2 has theta <= (d_in + 4) u; RBF as above; Matern
  s = c sqrt(r^2 + 1e-12) has relative error eps_s <= ((d_in + 4) / 2 + 3) u (add, sqrt, the rounded
  constant c), the exp factor then (s eps_s + 2u), the polynomial 1 + s + s^2/3 by FMAs 3u + 2 eps_s, times
  variance u; Linear sum w_c z_c x_c by FMAs is off by (d_in + 1) u sum |w_c z_c x_c| (absolute: no
  relative bound survives cancellation); Constant and White are exact.  A term's product of values
  v_p +- e_p is bounded by prod(|v_p| + e_p) - prod |v_p| plus P u prod(|v_p| + e_p) for its P roundings,
  the sum of T terms adds T u sum |term|, and the factor s^2 one more u |k|.  The diagonal k** is exact
  for stationary primitives and Constant/White, Linear as above; for the plain RBF k** = s^2 v is one
  rounded product.
* Ak = |L^-1| |k|, Ek = |L^-1| e.  a_i = sum_j L_ij k^_j over at most M terms: |a^_i - a_i| <= gamma_M Ak_i
  + Ek_i (to first order).  Both reductions run over at most M + 8 terms (zero-padded rows add zeros).
  a . alpha: gamma_{M+8} sum Ak |alpha| + sum |alpha| (gamma_M Ak + Ek), i.e. c_mean u (M + 8)
  sum Ak |alpha| + sum Ek |alpha| with c_mean = 2 * 1.01 -> 2.1.  sum a^2: gamma_{M+8} sum Ak^2 +
  2 sum Ak (gamma_M Ak + Ek) + sum Ek^2, i.e. c_var u (M + 8) sum Ak^2 + 2 sum Ak Ek + sum Ek^2 with
  c_var = 3 * 1.01 -> 3.1 (the 0.1 also absorbs the O(u^2) products of the first-order terms).
* mean = (a . alpha + s m(z)) / s with m(z) = sum_c z_c p_c by d_in rounded products and adds and one more
  product by s: (d_in + 2) u sum |z_c p_c|; the final add and division: 2u |mean|.
  |d mean| <= [c_mean u (M + 8) sum Ak |alpha| + sum Ek |alpha|] / s + (d_in + 2) u sum |z_c p_c|
              + 2u |mean| (+ 2u for the 1.01 of gamma)
* var = (s^2 k** - sum a^2) / s^2 with s^2 rounded once: the subtraction and division 2u |var|, the rounded
  s^2 in k** and in the division u s^2 k** / s^2 each:
  |d var| <= [c_var u (M + 8) sum Ak^2 + 2 sum Ak Ek + sum Ek^2 + e_kss + 2u s^2 k**] / s^2 + 2u |var|
* err = beta sqrt(var): |sqrt(v^) - sqrt(v)| = |v^ - v| / (sqrt(v^) + sqrt(v)); where var > 4 |d var| the
  bound beta |d var| / (sqrt(var) + sqrt(var - |d var|)) + 2u err is used (sqrt and the product by beta);
  elsewhere (err / beta)^2 is compared with var instead, within |d var| + 4u (err / beta)^2.

``check_not_too_tight`` evaluates the same operation in plain fp64 numpy in another order (reversed
contraction, pairwise sums, numpy's exp) and requires it inside the bound; ``mutations`` perturbs the
reference in ways a subtly wrong kernel could (a dropped row, a dropped 8-row block, two points of a tile
swapped, two outputs' alpha swapped) and ``mutation_ratio`` reports by how much each perturbation exceeds
the bound -- a bound loose enough to hide them fails the tests that use it.
"""
import numpy as np

LD = np.longdouble
U = 2.0 ** -53
C_MEAN, C_VAR = 2.1, 3.1
K_RBF, K_MATERN12, K_MATERN32, K_MATERN52, K_LINEAR, K_CONSTANT, K_WHITE = range(7)
_MATERN_C = {K_MATERN12: np.sqrt(LD(1)), K_MATERN32: np.sqrt(LD(3)), K_MATERN52: np.sqrt(LD(5))}


# ------------------------------------------------------------------------ the device tables, read back
def stack_tables(stack):
    """Host copies of everything the kernel reads for a ``GaussianProcess`` / ``FunctionStack``: one dict
    per output with its factor's tables (shared factors are shared dicts)."""
    desc = stack.gp_stack()
    members = getattr(stack, "functions", [stack])
    din = int(desc.input_dim)
    factors = {}
    outs = []
    for o, member in enumerate(members):
        gp = member.gaussian_process
        gp._ensure()
        fi = int(desc.outputs[o].factor)
        if fi not in factors:
            F = desc.factors[fi]
            fac = gp._factor
            prims = [(int(F.kernel.prims[i].kind), int(F.kernel.prims[i].term), float(F.kernel.prims[i].variance),
                      np.array([F.kernel.prims[i].w[c] for c in range(din)], dtype=np.float64))
                     for i in range(int(F.kernel.num_prims))]
            factors[fi] = dict(M=int(F.M), Xs=fac.Xs.cpu().numpy().reshape(-1, din).astype(np.float64),
                               Linv=fac.Linv.cpu().numpy().reshape(int(F.M), int(F.M)),
                               lengthscales=np.array([F.lengthscales[c] for c in range(din)]),
                               variance=float(F.variance), scale=float(F.scale), kss=float(F.kss),
                               prims=prims, index=fi)
        fac = factors[fi]
        prior = None if gp._prior_dev is None else gp._prior_dev.cpu().numpy().astype(np.float64)
        outs.append(dict(factor=fac, beta=float(desc.outputs[o].beta),
                         alpha=gp._alpha_dev.cpu().numpy()[:fac["M"]].astype(np.float64), prior=prior))
    return dict(din=din, outputs=outs)


# ------------------------------------------------------------------------ kernel values and their budget
def _kernel_values(fac, z, din, dtype):
    """k [n, M] (times s^2), its budget e [n, M], k** [n] and its budget, in `dtype` arithmetic."""
    X = fac["Xs"].astype(dtype)
    n, M = z.shape[0], fac["M"]
    s2 = dtype(fac["scale"]) * dtype(fac["scale"])
    if not fac["prims"]:                                      # plain RBF on lengthscale-divided inputs
        zs = (z / fac["lengthscales"]).astype(dtype)          # fp64 division, as the kernel does
        t = ((zs[:, None, :] - X[None, :, :]) ** 2).sum(axis=2)
        k = s2 * (dtype(fac["variance"]) * np.exp(-t / 2))
        e = np.abs(k) * ((din + 3) * U * t / 2 * 1.01 + 4 * U)
        e = np.where(t / 2 > 700, np.abs(k) + 1e-300, e)
        kss = np.full(n, dtype(fac["kss"]))
        return k, e, kss, U * np.abs(kss)
    zz = z.astype(dtype)
    total = np.zeros((n, M), dtype=dtype)
    etotal = np.zeros((n, M), dtype=dtype)
    dtotal = np.zeros(n, dtype=dtype)
    edtotal = np.zeros(n, dtype=dtype)
    terms = {}
    for kind, term, var, w in fac["prims"]:
        terms.setdefault(term, []).append((kind, dtype(var), w.astype(dtype)))
    for prims in terms.values():
        vals, errs, dvals, derrs = [], [], [], []
        for kind, var, w in prims:
            if kind == K_LINEAR:
                prod = (w * zz)[:, None, :] * X[None, :, :]
                v = prod.sum(axis=2)
                ev = (din + 1) * U * np.abs(prod).sum(axis=2)
                dprod = w * zz * zz
                dv, dev_ = dprod.sum(axis=1), (din + 1) * U * np.abs(dprod).sum(axis=1)
            elif kind in (K_CONSTANT, K_WHITE):
                v = np.full((n, M), var if kind == K_CONSTANT else dtype(0))
                ev = np.zeros((n, M), dtype=dtype)
                dv, dev_ = np.full(n, var), np.zeros(n, dtype=dtype)
            else:
                r2 = (((zz[:, None, :] - X[None, :, :]) * w) ** 2).sum(axis=2)
                theta = (din + 4) * U
                if kind == K_RBF:
                    v = var * np.exp(-r2 / 2)
                    ev = np.abs(v) * (theta * r2 / 2 * 1.01 + 3 * U)
                    ev = np.where(r2 / 2 > 700, np.abs(v) + 1e-300, ev)
                else:
                    c = _MATERN_C[kind].astype(dtype) if dtype is LD else dtype(float(_MATERN_C[kind]))
                    s = c * np.sqrt(r2 + dtype(1e-12))
                    eps_s = ((din + 4) / 2 + 3) * U
                    if kind == K_MATERN12:
                        poly, epoly = dtype(1), 0.0
                    elif kind == K_MATERN32:
                        poly, epoly = 1 + s, 3 * U + 2 * eps_s
                    else:
                        poly, epoly = 1 + s + s * s / 3, 3 * U + 2 * eps_s
                    v = var * poly * np.exp(-s)
                    ev = np.abs(v) * ((s * eps_s) * 1.01 + 2 * U + epoly + U)
                    ev = np.where(s > 700, np.abs(v) + 1e-300, ev)
                dv, dev_ = np.full(n, var), np.zeros(n, dtype=dtype)
            vals.append(v); errs.append(ev); dvals.append(dv); derrs.append(dev_)
        P = len(prims)
        hi = np.prod([np.abs(v) + ev for v, ev in zip(vals, errs)], axis=0)
        lo = np.prod([np.abs(v) for v in vals], axis=0)
        term_v = np.prod(vals, axis=0)
        total = total + term_v
        etotal = etotal + (hi - lo) + P * U * hi
        dhi = np.prod([np.abs(v) + ev for v, ev in zip(dvals, derrs)], axis=0)
        dlo = np.prod([np.abs(v) for v in dvals], axis=0)
        dtotal = dtotal + np.prod(dvals, axis=0)
        edtotal = edtotal + (dhi - dlo) + P * U * dhi
    T = len(terms)
    # the sum of the terms: T u sum |term| <= T u (|total| + error); then s^2 times it
    etotal = etotal + T * U * (np.abs(total) + etotal)
    edtotal = edtotal + T * U * (np.abs(dtotal) + edtotal)
    k = s2 * total
    e = s2 * etotal * (1 + 2 * U) + U * np.abs(k)
    kss = s2 * dtotal
    ekss = s2 * edtotal * (1 + 2 * U) + U * np.abs(kss)
    return k, e, kss, ekss


# ------------------------------------------------------------------------ the posterior
def _posterior(tables, z, dtype, mutate=None, order="forward"):
    """mean, var [n, D] (and the bound's ingredients) in `dtype` arithmetic."""
    din = tables["din"]
    z = np.asarray(z, dtype=np.float64).reshape(-1, din)
    n, D = z.shape[0], len(tables["outputs"])
    mean = np.zeros((n, D), dtype=dtype)
    var = np.zeros((n, D), dtype=dtype)
    bm = np.zeros((n, D), dtype=dtype)
    bv = np.zeros((n, D), dtype=dtype)
    cache = {}
    for o, out in enumerate(tables["outputs"]):
        fac = out["factor"]
        if id(fac) not in cache:
            M = fac["M"]
            k, e, kss, ekss = _kernel_values(fac, z, din, dtype)
            L = fac["Linv"].astype(dtype)
            keep = np.ones(M, dtype=bool)
            if mutate == "drop_last_row" and M:
                keep[M - 1] = False
            elif mutate == "drop_first_row" and M:
                keep[0] = False
            elif mutate == "drop_last_block" and M:
                keep[8 * ((M - 1) // 8):] = False
            if mutate == "drop_first_row" and M:
                k = k.copy()
                k[:, 0] = 0                      # row and column 0 of the factor gone
            if order == "forward":
                a = k @ L.T                      # [n, M]
            else:                                # another summation order (fp64 cross-check)
                a = np.stack([L[i, ::-1] @ k[:, ::-1].T for i in range(M)], axis=1) if M else k[:, :0]
            Ak = np.abs(k) @ np.abs(L).T
            Ek = e @ np.abs(L).T
            cache[id(fac)] = (a, Ak, Ek, kss, ekss, keep)
        a, Ak, Ek, kss, ekss, keep = cache[id(fac)]
        M = fac["M"]
        s = dtype(fac["scale"])
        s2 = s * s
        alpha = out["alpha"].astype(dtype)
        if mutate == "swap_alpha" and out.get("swap_with") is not None:
            alpha = tables["outputs"][out["swap_with"]]["alpha"].astype(dtype)
        ak, aAk, aEk = a[:, keep], Ak[:, keep], Ek[:, keep]
        al = alpha[keep]
        if order == "forward":
            dot = ak @ al
            ssq = (ak * ak).sum(axis=1)
        else:
            dot = np.array([np.sum((ak[p] * al)[::-1]) for p in range(n)], dtype=dtype)
            ssq = np.array([np.sum((ak[p] * ak[p])[::-1]) for p in range(n)], dtype=dtype)
        mx = np.zeros(n, dtype=dtype)
        emx = np.zeros(n, dtype=dtype)
        if out["prior"] is not None:
            pz = z.astype(dtype) * out["prior"].astype(dtype)
            mx = s * pz.sum(axis=1)
            emx = (din + 2) * U * np.abs(pz).sum(axis=1)
        mean[:, o] = (dot + mx) / s
        var[:, o] = (kss - ssq) / s2
        m8 = M + 8
        bm[:, o] = ((C_MEAN * U * m8 * (aAk @ np.abs(al)) + aEk @ np.abs(al)) / s + emx
                    + 2 * U * np.abs(mean[:, o]))
        bv[:, o] = ((C_VAR * U * m8 * (aAk * aAk).sum(axis=1) + 2 * (aAk * aEk).sum(axis=1)
                     + (aEk * aEk).sum(axis=1) + ekss + 2 * U * np.abs(kss)) / s2 + 2 * U * np.abs(var[:, o]))
    return mean, var, bm, bv


def reference(tables, z, mutate=None):
    """Long-double posterior at the fp64 query points z [n, d_in]: dict of mean, var, err (= beta sqrt(var))
    [n, D] and their bounds mean_bound, var_bound (float64)."""
    mean, var, bm, bv = _posterior(tables, z, LD, mutate)
    beta = np.array([o["beta"] for o in tables["outputs"]], dtype=LD)
    if mutate == "swap_points" and mean.shape[0] > 1:
        perm = np.arange(mean.shape[0])
        perm[0::2][:mean.shape[0] // 2], perm[1::2][:mean.shape[0] // 2] = \
            np.arange(1, 2 * (mean.shape[0] // 2), 2), np.arange(0, 2 * (mean.shape[0] // 2), 2)
        mean, var = mean[perm], var[perm]
    err = beta * np.sqrt(np.maximum(var, 0))
    return dict(mean=mean, var=var, err=err, beta=beta, mean_bound=bm.astype(np.float64),
                var_bound=bv.astype(np.float64))


def fp64_other_order(tables, z):
    """The same operation in plain fp64 numpy, summed in another order: mean, var [n, D]."""
    mean, var, _, _ = _posterior(tables, z, np.float64, order="reversed")
    return mean, var


# ------------------------------------------------------------------------ comparisons
def ratios(ref, mean=None, var=None, err=None):
    """Largest |observed - reference| / bound over points and outputs, for each quantity given."""
    out = {}
    if mean is not None:
        out["mean"] = float(np.max(np.abs(np.asarray(mean, dtype=LD) - ref["mean"]) / ref["mean_bound"],
                                   initial=0.0))
    if var is not None:
        out["var"] = float(np.max(np.abs(np.asarray(var, dtype=LD) - ref["var"]) / ref["var_bound"], initial=0.0))
    if err is not None:
        e = np.asarray(err, dtype=LD)
        beta, v, dv = ref["beta"], ref["var"], ref["var_bound"].astype(LD)
        sqrt_ok = v > 4 * dv
        with np.errstate(invalid="ignore", divide="ignore"):
            be = beta * dv / (np.sqrt(np.where(sqrt_ok, v, 1)) + np.sqrt(np.where(sqrt_ok, v - dv, 1))) \
                + 2 * U * ref["err"]
            r1 = np.abs(e - ref["err"]) / be
            e2 = (e / beta) ** 2
            r2 = np.abs(e2 - v) / (dv + 4 * U * e2)
        r = np.where(sqrt_ok, r1, r2)
        r = np.where(np.isnan(e), np.inf, r)
        out["err"] = float(np.max(r, initial=0.0))
    return out


def worst(r):
    return max(r.values()) if r else 0.0


def check_not_too_tight(tables, z):
    """Ratio of the fp64 other-order evaluation's deviation to the bound (must be <= 1)."""
    ref = reference(tables, z)
    mean, var = fp64_other_order(tables, z)
    return worst(ratios(ref, mean=mean, var=var))


MUTATIONS = ("drop_last_row", "drop_first_row", "drop_last_block", "swap_points", "swap_alpha")


def _pair_outputs(tables):
    """Mark, for the alpha swap, one pair of outputs that share a factor and have different alpha."""
    outs = tables["outputs"]
    for o in outs:
        o["swap_with"] = None
    for i, a in enumerate(outs):
        for j, b in enumerate(outs):
            if i < j and a["factor"] is b["factor"] and a["factor"]["M"] and not np.array_equal(a["alpha"], b["alpha"]):
                a["swap_with"], b["swap_with"] = j, i
                return True
    return False


def applicable_mutations(tables, n):
    """The perturbations that change anything for this stack and point count."""
    out = []
    if any(o["factor"]["M"] for o in tables["outputs"]):
        out += ["drop_last_row", "drop_first_row", "drop_last_block"]
    if n > 1:
        out.append("swap_points")
    if _pair_outputs(tables):
        out.append("swap_alpha")
    return out


def mutation_ratio(tables, z, mutation):
    """Largest deviation of the perturbed reference from the reference, relative to the bound (mean and
    var): a kernel with that defect would be caught where this is > 1."""
    _pair_outputs(tables)
    ref = reference(tables, z)
    mut = reference(tables, z, mutate=mutation)
    return worst(ratios(ref, mean=mut["mean"].astype(np.float64), var=mut["var"].astype(np.float64)))


def mutation_ratios(tables, z):
    n = np.asarray(z).reshape(-1, tables["din"]).shape[0]
    return {m: mutation_ratio(tables, z, m) for m in applicable_mutations(tables, n)}


def query_points(tables, n, rng, spread=1.2):
    """n query points: half of them within ~1e-3 of training inputs (the first, the last, the last 8-row
    block and a few random rows of every factor), the rest uniform in the box -- so that the mutations,
    which drop exactly those rows, move the posterior."""
    din = tables["din"]
    z = rng.uniform(-spread, spread, (n, din))
    raw = []
    for o in tables["outputs"]:
        fac = o["factor"]
        M = fac["M"]
        if not M:
            continue
        X = fac["Xs"] * (fac["lengthscales"] if not fac["prims"] else 1.0)
        rows = [M - 1, 0] + list(range(8 * ((M - 1) // 8), M)) + list(rng.integers(0, M, 4))
        raw += [X[r] for r in rows]
    near = min(len(raw), (n + 1) // 2)
    for i in range(near):
        z[i] = raw[i] + 1e-3 * rng.standard_normal(din)
    return z
