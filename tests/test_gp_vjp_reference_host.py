"""CPU checks of the VJP reference (tests/gp_vjp_reference.py) on tables built on the host.

The reference is checked against two independent derivatives of the posterior -- long-double central
differences of gp_posterior_reference.reference and float64 torch autograd through a direct restatement of
the posterior -- and its bound from both sides: an fp64 numpy evaluation in another summation order lies
inside it (not too tight), and every perturbation a subtly wrong kernel could make exceeds it by at least
10x somewhere (not vacuous)."""
import numpy as np
import pytest
import torch

import gp_posterior_reference as R
import gp_vjp_reference as V
from test_gp_posterior_reference_host import EXPRESSIONS, _tables

KINDS = ["rbf"] + EXPRESSIONS
LD = np.longdouble


def _vtables(*args, **kw):
    return V.add_gamma(_tables(*args, **kw))


def _cotangents(tables, n, seed):
    rng = np.random.default_rng(seed)
    D = len(tables["outputs"])
    return rng.normal(size=(n, D)), rng.normal(size=(n, D))


def _away(tables, z, rmin):
    """Rows of z at distance >= rmin from every training input (Matern 1/2's r = 0 region has a curvature
    of 1 / sqrt(1e-12) that no finite difference resolves)."""
    keep = np.ones(len(z), dtype=bool)
    for o in tables["outputs"]:
        fac = o["factor"]
        if fac["M"]:
            X = fac["Xs"] * (fac["lengthscales"] if not fac["prims"] else 1.0)
            keep &= np.sqrt(((z[:, None] - X[None]) ** 2).sum(axis=2)).min(axis=1) >= rmin
    return z[keep]


def _objective(tables, z, gm, ge):
    ref = R.reference(tables, z)
    return (ref["mean"] * gm.astype(LD)).sum(axis=1) + (ref["err"] * ge.astype(LD)).sum(axis=1)


def _central_differences(tables, z, gm, ge, h=2.0 ** -17):
    out = np.zeros(z.shape, dtype=LD)
    for c in range(z.shape[1]):
        zp, zm = z.copy(), z.copy()
        zp[:, c] += h
        zm[:, c] -= h
        step = (zp[:, c].astype(LD) - zm[:, c].astype(LD))
        out[:, c] = (_objective(tables, zp, gm, ge) - _objective(tables, zm, gm, ge)) / step
    return out


def _torch_posterior(tables, z):
    """mean, err [n, D] in float64 torch from the tables, differentiable in z."""
    outs = []
    errs = []
    for o in tables["outputs"]:
        fac = o["factor"]
        s = fac["scale"]
        M = fac["M"]
        X = torch.tensor(fac["Xs"])
        if not fac["prims"]:
            zs = z / torch.tensor(fac["lengthscales"])
            k = fac["variance"] * torch.exp(-((zs[:, None] - X[None]) ** 2).sum(dim=2) / 2)
            kss = torch.full((z.shape[0],), fac["variance"], dtype=torch.float64)
        else:
            k, kss = 0.0, 0.0
            for t in sorted({p[1] for p in fac["prims"]}):
                tk, tkss = 1.0, 1.0
                for kind, _, var, w in (p for p in fac["prims"] if p[1] == t):
                    w = torch.tensor(w)
                    if kind == R.K_LINEAR:
                        v, vd = (z * w) @ X.T, ((z * w) * z).sum(dim=1)
                    elif kind == R.K_CONSTANT:
                        v, vd = torch.full((z.shape[0], M), var, dtype=torch.float64), var
                    elif kind == R.K_WHITE:
                        v, vd = torch.zeros((z.shape[0], M), dtype=torch.float64), var
                    else:
                        r2 = (((z[:, None] - X[None]) * w) ** 2).sum(dim=2)
                        r = torch.sqrt(r2 + 1e-12)
                        c = {R.K_MATERN32: 3 ** 0.5, R.K_MATERN52: 5 ** 0.5}.get(kind, 1.0)
                        v = {R.K_RBF: lambda: var * torch.exp(-r2 / 2), R.K_MATERN12: lambda: var * torch.exp(-r),
                             R.K_MATERN32: lambda: var * (1 + c * r) * torch.exp(-c * r),
                             R.K_MATERN52: lambda: var * (1 + c * r + c * c * r * r / 3) * torch.exp(-c * r)}[kind]()
                        vd = var
                    tk, tkss = tk * v, tkss * vd
                k, kss = k + tk, kss + tkss
            kss = kss * torch.ones(z.shape[0], dtype=torch.float64)
        mx = z @ torch.tensor(o["prior"]) if o["prior"] is not None else 0.0
        if M:
            a = (s * s * k) @ torch.tensor(fac["Linv"]).T
            mean = (a @ torch.tensor(o["alpha"]) + s * mx) / s
            var = (s * s * kss - (a * a).sum(dim=1)) / (s * s)
        else:
            mean, var = mx + 0.0 * z[:, 0], kss
        outs.append(mean)
        errs.append(o["beta"] * torch.sqrt(var))
    return torch.stack(outs, dim=1), torch.stack(errs, dim=1)


def _close(got, want, rtol, what):
    """Per column, relative to the column's largest magnitude over the batch."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    scale = np.maximum(np.abs(want).max(axis=0), 1e-300)
    err = np.abs(got - want).max(axis=0)
    assert (err <= rtol * scale).all(), (what, err / scale)


@pytest.mark.parametrize("kind", KINDS)
def test_agrees_with_central_differences_and_torch_autograd(kind):
    """Mean and err parts at every d_in against long-double central differences of the forward reference
    and float64 autograd of an independent torch restatement; scale 1.7, a prior mean, shared factor."""
    for din in range(1, 7):
        tables = _vtables(din, 23, [kind, kind], seed=10 * din, scale=1.7)
        z = _away(tables, np.random.default_rng(din).uniform(-1.2, 1.2, (40, din)), 0.05)
        assert len(z) >= 4, (kind, din)
        gm, ge = _cotangents(tables, len(z), din)
        ref = V.reference(tables, z, gm, ge)
        assert ref["claim"].all()
        fd = _central_differences(tables, z, gm, ge)
        _close(ref["both"], fd, 1e-7, (kind, din, "central differences"))
        zt = torch.tensor(z, requires_grad=True)
        mean, err = _torch_posterior(tables, zt)
        gmt = torch.autograd.grad((mean * torch.tensor(gm)).sum(), zt, retain_graph=True)[0]
        get = torch.autograd.grad((err * torch.tensor(ge)).sum(), zt)[0]
        _close(ref["mean"], gmt.numpy(), 1e-9, (kind, din, "mean part, autograd"))
        _close(ref["err"], get.numpy(), 1e-8, (kind, din, "err part, autograd"))


MS = [0, 1, 5, 7, 8, 9, 127, 128, 129, 257]


def _cases():
    out = []
    for din in range(1, 7):
        for i, M in enumerate(MS):
            out.append((din, M, ["rbf", "rbf"]))
            out.append((din, M, [EXPRESSIONS[(din + i) % len(EXPRESSIONS)]] * 2))
    return out


def _near_points(tables, n, seed):
    """Half the points next to (1e-7) or on training inputs, the rest from query_points."""
    rng = np.random.default_rng(seed)
    z = R.query_points(tables, n, rng)
    fac = tables["outputs"][0]["factor"]
    if fac["M"]:
        X = fac["Xs"] * (fac["lengthscales"] if not fac["prims"] else 1.0)
        rows = rng.integers(0, fac["M"], n // 4)
        z[:len(rows)] = X[rows]
        z[len(rows):2 * len(rows)] = X[rows] + 1e-7 * rng.standard_normal((len(rows), tables["din"]))
    return z


@pytest.mark.parametrize("din,M,kinds", _cases())
def test_fp64_in_another_order_lies_inside_the_bound(din, M, kinds):
    tables = _vtables(din, M, kinds, seed=din * 100 + M, shared=True, scale=0.3 if M % 2 else 1.7)
    z = _near_points(tables, 24, M)
    gm, ge = _cotangents(tables, len(z), M)
    assert V.check_not_too_tight(tables, z, gm, ge) <= 1.0


@pytest.mark.parametrize("din,M,kinds", [(1, 9, ["rbf", "rbf"]), (2, 9, ["six", "six"]), (3, 257, ["rbf", "rbf"]),
                                         (4, 64, ["matern12", "matern12"]), (5, 13, ["linear", "linear"]),
                                         (6, 130, ["white_matern32", "white_matern32"]),
                                         (3, 40, ["constant_rbf", "constant_rbf"]), (2, 17, ["six", "six"])])
def test_every_mutation_exceeds_the_bound(din, M, kinds):
    """Shared factors (so the cotangent swap applies), scale 1.7, a prior mean; the points start next to
    the training inputs."""
    tables = _vtables(din, M, kinds, seed=7 * din + M, shared=True, scale=1.7)
    z = R.query_points(tables, 48, np.random.default_rng(din))
    gm, ge = _cotangents(tables, len(z), din)
    ratios = V.mutation_ratios(tables, z, gm, ge)
    want = {"drop_last_row", "drop_last_block", "swap_packed_columns", "swap_points", "swap_cotangents",
            "two_over_s2_to_one_over_s2", "two_over_s2_to_one_over_s", "move_prior"}
    if kinds[0] == "six":
        want |= {"drop_product_term", "drop_kdiag_grad"}
    if kinds[0] == "linear":
        want.add("drop_kdiag_grad")
    if kinds[0] == "matern12" and din > 1:
        want.add("leak_inactive")
    assert set(ratios) >= want, ratios
    assert min(ratios.values()) >= 10.0, ratios


def test_zero_variance_rule():
    """A Linear-only kernel at z = 0 has var = 0 exactly: no claim there, and the rule wants non-finite
    columns (torch's sqrt backward); finite values are refused.  Other points keep their claim."""
    tables = _vtables(2, 5, ["linear"], seed=3)
    z = np.random.default_rng(0).uniform(-1, 1, (6, 2))
    z[2] = 0.0
    gm, ge = _cotangents(tables, 6, 0)
    ref = V.reference(tables, z, gm, ge)
    assert ref["zero_var"].tolist() == [False, False, True, False, False, False]
    assert not ref["claim"][2] and ref["claim"].sum() == 5 and V.uncertified(ref) == 1
    err = ref["err"].astype(np.float64)
    err[2] = np.nan
    assert V.worst(V.ratios(ref, err=err)) <= 1.0
    err[2] = 0.0
    assert V.ratios(ref, err=err)["err"] == np.inf
