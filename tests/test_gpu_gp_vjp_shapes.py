"""The GP posterior's reverse mode (``slb_gp_vjp``, csrc/gp_grad.cu) at every shape it is compiled or launched
for, against the long-double reference and the per-point, per-column error bound of
tests/gp_vjp_reference.py, in all three cotangent modes (mean only, err only, both).

Coverage (compiled shape or run-time path -> test):

===============================================================  ============================================
gp_vjp_mean_kernel / gp_vjp_err_kernel<DIN>, DIN 1..6, plain      test_every_input_dimension (every kind meets
RBF and every expression kind; err tiles of P = 64 / (1 + DIN)    every d_in; M at the 128-row j-panel and
points; M at the panel edges; n at P - 1, P, P + 1, 2P + 1 and    256-row i-panel edges and 513; n at the tile
the mean kernel's 4-point blocks                                  edges)
M = 0 .. 2000 across every 8-row group, j-panel and i-panel edge  test_rows_and_panels (d_in = 3)
n in the thousands                                                test_many_points
stacks of 1..6 outputs: one factor, one each, shared factors      test_stacks
interleaved, an empty-data output, a prior mean on alternate
outputs, distinct beta, scale 0.3 / 1 / 1.7
noise variance 1e-6 (tiny var next to the data)                   test_small_noise
===============================================================  ============================================

Query points in every case: uniform over and beyond the data, next to training inputs (1e-3), exactly on
them, within 1e-7 of them, far enough that exp flushes, and training inputs moved in inactive columns only.
A module-scope fixture prints the largest observed-error / bound ratio of each section, the smallest
mutation / bound ratio and the number of points whose err part is not certified (``pytest -s``).
"""
import numpy as np
import pytest
import torch

import gp_posterior_reference as R
import gp_vjp_reference as V
import safe_learning_b200 as sl
from safe_learning_b200 import _device as dev
from test_gpu_gp_vjp import _kernel

pytestmark = pytest.mark.gpu

KINDS = ["rbf", "matern12", "matern32", "matern52", "linear", "constant", "white", "rbf_sub", "notebook", "six"]
EDGES = [127, 128, 129, 255, 256, 257, 513]
MS = [0, 1, 7, 8, 9, 127, 128, 129, 255, 256, 257, 511, 512, 513, 2000]
SCALES = [0.3, 1.0, 1.7]
MUT_POINTS = 24
MUT_MAX_M = 300

_REPORT = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for key in sorted(_REPORT):
        print("%-40s %.3g" % (key, _REPORT[key]))


def _note(key, value, smallest=False):
    old = _REPORT.get(key)
    if old is None or (value < old if smallest else value > old):
        _REPORT[key] = value


def _count(key, value):
    _REPORT[key] = _REPORT.get(key, 0) + value


def _tile(din):
    return 64 // (1 + din)


def _stack(din, M, kinds, factors=None, seed=0, priors=None, scale=1.0, betas=None, noise=0.01, empty=None):
    """FunctionStack on one data set: output o has the kernel kinds[factors[o]] (outputs with the same factor
    id share one factor), a prior mean where priors[o] (all by default), beta betas[o]; output `empty` has
    no data."""
    factors = list(range(len(kinds))) if factors is None else factors
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1, 1, (M, din))
    gps = []
    for o, fid in enumerate(factors):
        kern = _kernel(kinds[fid], din, np.random.default_rng(seed + 100 + fid))
        Xo = X[:0] if o == empty else X
        Y = np.sin(Xo @ rng.normal(size=din) + o)[:, None] + 0.05 * rng.normal(size=(Xo.shape[0], 1))
        p = rng.normal(size=(1, din))
        mean = sl.LinearSystem(p) if priors is None or priors[o] else None
        gp = sl.GPRCached(Xo, Y, kern, mean_function=mean, noise_variance=noise, scale=scale)
        gps.append(sl.GaussianProcess(gp, beta=2.0 if betas is None else betas[o]))
    return sl.FunctionStack(gps)


def _inputs(fac):
    return fac["Xs"] * (fac["lengthscales"] if not fac["prims"] else 1.0)


def _points(tables, n, seed):
    """n query points: gp_posterior_reference.query_points (first half next to the first, last and last-group
    rows of every factor, the rest uniform over and beyond the data), then from the end: exactly on training
    inputs, within 1e-7 of them, far away (every exp flushes), and training inputs moved in the inactive
    columns of an expression only."""
    rng = np.random.default_rng(seed)
    din = tables["din"]
    z = R.query_points(tables, n, rng, spread=1.5)
    special = [np.sign(rng.uniform(-1, 1, din)) * 2000.0]
    for o in tables["outputs"]:
        fac = o["factor"]
        if not fac["M"]:
            continue
        X = _inputs(fac)
        for j in rng.integers(0, fac["M"], 2):
            special += [X[j], X[j] + 1e-7 * rng.standard_normal(din)]
        if fac["prims"] and V._inactive(fac).any():
            x = X[rng.integers(0, fac["M"])].copy()
            x[V._inactive(fac)] = rng.uniform(-1.5, 1.5, int(V._inactive(fac).sum()))
            special.append(x)
    k = min(len(special), n // 2)
    if k:
        z[n - k:] = np.array(special[:k])
    return z


def _check(section, stack, z, seed=0, mutations=True):
    """All three modes within the bound where the err part is certified (the rule of gp_vjp_reference
    elsewhere); every applicable mutation exceeds the bound 10x on the first points."""
    tables = V.vjp_tables(stack)
    n, D = z.shape[0], len(tables["outputs"])
    rng = np.random.default_rng(seed)
    gm, ge = rng.normal(size=(n, D)), rng.normal(size=(n, D))
    x = torch.tensor(z, device=dev.device())
    gmt, get = (torch.tensor(g, device=dev.device()) for g in (gm, ge))
    got = dict(mean=stack.vjp_device(x, gmt, None), err=stack.vjp_device(x, None, get),
               both=stack.vjp_device(x, gmt, get))
    got = {k: v.cpu().numpy() for k, v in got.items()}
    ref = V.reference(tables, z, gm, ge)
    r = V.ratios(ref, **got)
    for mode, value in r.items():
        _note("%s (%s): error / bound" % (section, mode), value)
    _count("%s: points uncertified" % section, V.uncertified(ref))
    _count("%s: points" % section, n)
    assert V.worst(r) <= 1.0, r
    assert np.isfinite(got["mean"]).all()
    if mutations and max(o["factor"]["M"] for o in tables["outputs"]) <= MUT_MAX_M:
        k = min(n, MUT_POINTS)
        mut = V.mutation_ratios(tables, z[:k], gm[:k], ge[:k])
        for name, value in mut.items():
            _note("mutation / bound (min): %s" % name, value, smallest=True)
        assert min(mut.values(), default=np.inf) >= 10.0, mut
    return tables


# ------------------------------------------------------------------------ every d_in, kind, panel and tile edge
@pytest.mark.parametrize("din", range(1, 7))
def test_every_input_dimension(din):
    """Every kind at every d_in (two outputs on one factor, a prior mean on the first only); M rotates
    through the panel edges and n through the err tile's edges and the mean kernel's 4-point blocks, so each
    d_in meets every M edge and every n edge."""
    P = _tile(din)
    ns = [P - 1, P, P + 1, 2 * P + 1, 3, 4, 5]
    for j, kind in enumerate(KINDS):
        M = EDGES[(din + j) % len(EDGES)]
        n = ns[(din + 2 * j) % len(ns)]
        stack = _stack(din, M, [kind], factors=[0, 0], seed=100 * din + j, priors=[True, False],
                       scale=SCALES[j % 3], betas=[2.0, 1.5])
        assert stack.gp_stack().num_factors == 1
        _check("input dimensions", stack, _points(V.vjp_tables(stack), n, j), seed=j)


@pytest.mark.parametrize("M", MS)
def test_rows_and_panels(M):
    """d_in = 3 (P = 16): M across every 8-row group, j-panel and i-panel boundary up to ~2000 rows; plain
    RBF and the notebook kernel."""
    for j, kind in enumerate(("rbf", "notebook")):
        n = 24 if M > 600 else [15, 16, 17, 33, 5][(MS.index(M) + j) % 5]
        stack = _stack(3, M, [kind], factors=[0, 0], seed=M + j, priors=[j == 0, j == 1], scale=SCALES[M % 3],
                       betas=[1.5, 2.5])
        _check("rows and panels", stack, _points(V.vjp_tables(stack), n, M), seed=M)


def test_many_points():
    """n in the thousands: many err tiles and mean blocks, the last tile partial (3001 = 187 * 16 + 9)."""
    stack = _stack(3, 100, ["six", "rbf"], seed=5, scale=1.7, betas=[2.0, 3.0])
    _check("many points", stack, _points(V.vjp_tables(stack), 3001, 5), mutations=False)


# ------------------------------------------------------------------------ stacks
LAYOUTS = ["one factor", "one each", "interleaved", "empty output"]


@pytest.mark.parametrize("D", range(1, 7))
@pytest.mark.parametrize("layout", LAYOUTS)
def test_stacks(D, layout):
    """Stacks of 1..6 outputs (d_in = 1 + (D % 6)): factors [0, .., 0], [0, 1, .., D - 1], [0, 1, 0, 2, 1, 0]
    or one factor each with an empty-data output; a prior mean on alternate outputs, distinct beta per
    output, scale 0.3 / 1 / 1.7."""
    din = 1 + D % 6
    kinds = ["six", "rbf", "notebook", "matern52", "linear", "rbf_sub"]
    factors = {"one factor": [0] * D, "one each": list(range(D)), "interleaved": [0, 1, 0, 2, 1, 0][:D],
               "empty output": list(range(D))}[layout]
    empty = D // 2 if layout == "empty output" else None
    i = LAYOUTS.index(layout)
    stack = _stack(din, 137, kinds, factors=factors, seed=10 * D + i, priors=[o % 2 == 0 for o in range(D)],
                   scale=SCALES[(D + i) % 3], betas=[1.0 + 0.5 * o for o in range(D)], empty=empty)
    desc = stack.gp_stack()
    assert desc.num_factors == len(set(factors))
    if empty is not None:
        assert desc.factors[desc.outputs[empty].factor].M == 0
    _check("stacks", stack, _points(V.vjp_tables(stack), 40, D), seed=D)


# ------------------------------------------------------------------------ tiny variance next to the data
@pytest.mark.parametrize("din", range(1, 7))
def test_small_noise(din):
    """Noise variance 1e-6: next to and on the data the variance is ~1e-6 of the prior's and d var cancels
    hard; certified points hold the bound, the others are counted.  Here |L^-1| |K| is ~1e4 times |a|, so
    the a-priori bound of var exceeds var next to the data and most err-part claims there are withdrawn:
    the mutations are checked in the other sections."""
    kind = KINDS[din % len(KINDS)]
    stack = _stack(din, 200, [kind, "rbf"], factors=[0, 1, 0], seed=din, scale=SCALES[din % 3], noise=1e-6,
                   betas=[2.0, 1.0, 3.0])
    _check("small noise", stack, _points(V.vjp_tables(stack), 48, din), seed=din, mutations=False)


def test_zero_variance_gives_nan():
    """A Linear-only kernel at z = 0: var = 0 exactly, the err columns are not finite (torch's sqrt
    backward), the other points hold the bound."""
    stack = _stack(2, 5, ["linear"], factors=[0], seed=3, priors=[False])
    z = np.random.default_rng(1).uniform(-1, 1, (20, 2))
    z[3] = 0.0
    tables = _check("zero variance", stack, z, mutations=False)
    ref = V.reference(tables, z, np.ones((20, 1)), np.ones((20, 1)))
    assert ref["zero_var"].tolist() == [i == 3 for i in range(20)]
