"""Extended-precision reference of the posterior mean in the form ``slb_gp_mean`` evaluates (the Bellman
sweep's staged pipeline, csrc/gp_mean_staged.cuh), with a computed bound of the kernel's rounding error at
every point and output.

Inputs are the product's own device tables read back: per factor the staged rows ``Xf`` (plain RBF:
``[x / l, h]`` with ``h = -|x / l|^2 / 2``; covariance expressions: the raw inputs), per output ``gamma_f``
(the folded weights ``scale^2 v gamma``, or ``scale^2 gamma`` for expressions) and the prior-mean row.  In
``np.longdouble``:

    plain RBF:    k_j = exp(h_j + zs . xs_j - |zs|^2 / 2),   zs = z / l formed in fp64 as the kernel does;
    expressions:  k_j = kappa(z, x_j) (``gp_posterior_reference._kernel_values`` without the s^2 fold);
    mean = (sum_j k_j gamma_f[j] + scale (z . m)) / scale.

Error bound (u = 2^-53, every fp64 operation rounds by at most u):
* a plain kernel value: the argument is a chain of d_in + 1 FMAs and one add on fp64 inputs, off by at
  most (d_in + 3) u (|h_j| + sum |zs_c xs_jc| + |zs|^2 / 2); exp moves by that (times 1.01) and the table
  exp adds one ulp, two with the spare: e_j = k_j ((d_in + 3) u A_j 1.01 + 2 u);  e_j = k_j + 1e-300
  where the argument is below -700 (the table flushes).  Expression values take the budget of
  ``gp_posterior_reference`` divided by the fold.
* the dot product over at most M + 8 rows (two interleaved FMA chains, zero-padded rows add zeros):
  (M + 8) u 1.01 sum |k_j gamma_j| + sum |gamma_j| e_j;
* the prior term: d_in + 1 roundings of sum |z_c m_c| times |scale|, one more each for the final
  add and the division.
The bound is compared against the worst case over the points of |device - reference| / bound; two
mutations (a dropped training row, two outputs' weights swapped) must exceed it by 10x or more.
"""
import numpy as np

import gp_posterior_reference as GR

LD = np.longdouble
U = 2.0 ** -53


def staged_tables(stack):
    """Host copies of the staged tables of a ``GaussianProcess`` / ``FunctionStack``."""
    desc = stack.gp_stack()
    members = getattr(stack, "functions", [stack])
    din = int(desc.input_dim)
    post = GR.stack_tables(stack)
    outs = []
    for o, member in enumerate(members):
        gp = member.gaussian_process
        fac = gp._factor
        M = int(desc.factors[int(desc.outputs[o].factor)].M)
        width = din if fac.plain is False else din + 1
        Xf = fac.Xf.cpu().numpy().reshape(-1, width)[:M].astype(np.float64)
        gf = gp._gamma_f_dev.cpu().numpy()[:M].astype(np.float64)
        F = desc.factors[int(desc.outputs[o].factor)]
        outs.append(dict(M=M, plain=bool(fac.plain), Xf=Xf, gamma_f=gf, scale=float(F.scale),
                         lengthscales=np.array([F.lengthscales[c] for c in range(din)]),
                         fold=float(gp._scale) ** 2 * (float(gp.kern.variance) if fac.plain else 1.0),
                         prior=post["outputs"][o]["prior"], post=post["outputs"][o]))
    return dict(din=din, outputs=outs, post=post)


def _unit_kernel(out, z, din):
    """k [n, M] and its budget e [n, M] in long double (without the fold)."""
    if out["M"] == 0:
        n = z.shape[0]
        return np.zeros((n, 0), dtype=LD), np.zeros((n, 0), dtype=LD)
    if out["plain"]:
        zs = (z / out["lengthscales"]).astype(LD)          # fp64 division, as the kernel does
        xs, h = out["Xf"][:, :din].astype(LD), out["Xf"][:, din].astype(LD)
        dot = zs @ xs.T
        zz = (zs * zs).sum(axis=1) / 2
        arg = h[None, :] + dot - zz[:, None]
        k = np.exp(arg)
        A = np.abs(h)[None, :] + np.abs(zs) @ np.abs(xs).T + zz[:, None]
        e = k * ((din + 3) * U * A * 1.01 + 2 * U)
        e = np.where(arg < -700, k + LD(1e-300), e)
        return k, e
    k, e, _, _ = GR._kernel_values(out["post"]["factor"], z, din, LD)
    s2 = LD(out["scale"]) * LD(out["scale"])
    return k / s2, e / s2 * (1 + 4 * U)


def reference(tables, z, mutate=None):
    """mean [n, D] in long double and its bound [n, D]; ``mutate``: "drop_row" (the last training row of
    output 0 is left out) or "swap_gamma" (outputs 0 and 1 exchange their weights)."""
    din = tables["din"]
    z = np.asarray(z, dtype=np.float64).reshape(-1, din)
    n, D = z.shape[0], len(tables["outputs"])
    mean = np.zeros((n, D), dtype=LD)
    bound = np.zeros((n, D), dtype=LD)
    gammas = [o["gamma_f"] for o in tables["outputs"]]
    if mutate == "swap_gamma":
        gammas[0], gammas[1] = gammas[1], gammas[0]
    for o, out in enumerate(tables["outputs"]):
        k, e = _unit_kernel(out, z, din)
        g = gammas[o].astype(LD)
        if mutate == "drop_row" and o == 0:
            k, e, g = k[:, :-1], e[:, :-1], g[:-1]
        dot = k @ g if out["M"] else np.zeros(n, dtype=LD)
        adot = np.abs(k) @ np.abs(g) if out["M"] else np.zeros(n, dtype=LD)
        ebody = (np.abs(g)[None, :] * e).sum(axis=1) if out["M"] else np.zeros(n, dtype=LD)
        s = LD(out["scale"])
        prior = np.zeros(n, dtype=LD)
        aprior = np.zeros(n, dtype=LD)
        if out["prior"] is not None:
            pm = out["prior"].astype(LD)
            prior = s * (z.astype(LD) @ pm)
            aprior = abs(s) * (np.abs(z.astype(LD)) @ np.abs(pm))
        num = dot + prior
        mean[:, o] = num / s
        b = (out["M"] + 8) * U * 1.01 * adot + ebody + (din + 2) * U * aprior + 2 * U * (np.abs(num) + adot)
        bound[:, o] = (b / abs(s)) * 1.05 + LD(1e-300)
    return mean, bound


def gamma_gap_bound(tables, z):
    """Bound of |exact gamma form - exact a . alpha form| from the fp64 rounding of gamma = L^-T alpha
    ((M + 2) u 1.01 (|L^-1|^T |alpha|)_j per weight, times the fold), divided by scale."""
    din = tables["din"]
    z = np.asarray(z, dtype=np.float64).reshape(-1, din)
    out_b = np.zeros((z.shape[0], len(tables["outputs"])))
    for o, out in enumerate(tables["outputs"]):
        if out["M"] == 0:
            continue
        k, _ = _unit_kernel(out, z, din)
        fac = out["post"]["factor"]
        w = np.abs(fac["Linv"]).T @ np.abs(out["post"]["alpha"])
        out_b[:, o] = (np.abs(k).astype(np.float64) @ w) * (out["M"] + 2) * U * 1.01 * out["fold"] / out["scale"]
    return out_b * 1.05


def ratio(device, mean, bound):
    return float(np.max(np.abs(device.astype(LD) - mean) / bound)) if device.size else 0.0
