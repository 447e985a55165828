"""CPU checks of the GP posterior reference (tests/gp_posterior_reference.py) and of the host side of
``slb_debug_refine``.

The bound is checked from both sides without a GPU: an fp64 numpy evaluation of the same operation in
another summation order lies inside it (not too tight), and every perturbation a subtly wrong kernel could
make -- a dropped training row or 8-row block, two points swapped, two outputs' alpha swapped -- exceeds it
by at least 10x somewhere (not vacuous).  The tables are built here in numpy with the layout the product
keeps on the device (scaled inputs for the plain RBF, the slb_kernel normal form otherwise)."""
import numpy as np
import pytest

import gp_posterior_reference as R
from safe_learning_b200 import _native as nat

FAKE = 0x1000
MS = [0, 1, 3, 4, 5, 7, 8, 9, 255, 256, 257]
EXPRESSIONS = ["matern12", "matern32", "matern52", "linear", "constant_rbf", "white_matern32", "six"]


def _prims(kind, din, rng):
    """Normal form (kind, term, variance, w[din]) of the covariance expressions of test_gpu_gp_vjp."""
    ls = lambda: np.where(np.arange(din) < max(1, din - 1), 1.0 / rng.uniform(0.6, 1.6, din), 0.0)
    full = lambda: 1.0 / rng.uniform(0.6, 1.6, din)
    if kind in ("matern12", "matern32", "matern52"):
        k = {"matern12": R.K_MATERN12, "matern32": R.K_MATERN32, "matern52": R.K_MATERN52}[kind]
        return [(k, 0, 0.6, ls())]
    if kind == "linear":
        return [(R.K_LINEAR, 0, 1.0, rng.uniform(0.2, 1.0, din))]
    if kind == "constant_rbf":
        return [(R.K_CONSTANT, 0, 0.8, np.zeros(din)), (R.K_RBF, 1, 0.3, np.ones(din))]
    if kind == "white_matern32":
        return [(R.K_WHITE, 0, 0.2, np.zeros(din)), (R.K_MATERN32, 1, 0.5, np.ones(din))]
    if kind == "six":
        return [(R.K_RBF, 0, 0.5, full()), (R.K_MATERN32, 0, 1.0, ls()),
                (R.K_LINEAR, 1, 1.0, np.full(din, 0.3)), (R.K_MATERN12, 1, 0.4, np.eye(din)[din - 1]),
                (R.K_MATERN52, 2, 0.3, full()), (R.K_CONSTANT, 3, 0.2, np.zeros(din))]
    raise KeyError(kind)


def _gram(prims, X):
    """K(X, X) of a normal form in fp64 (noise added by the caller), gpflow arithmetic on differences."""
    M = X.shape[0]
    total = np.zeros((M, M))
    for t in sorted({p[1] for p in prims}):
        term = np.ones((M, M))
        for kind, _, var, w in (p for p in prims if p[1] == t):
            if kind == R.K_LINEAR:
                v = (X * w) @ X.T
            elif kind == R.K_CONSTANT:
                v = np.full((M, M), var)
            elif kind == R.K_WHITE:
                v = var * np.eye(M)
            else:
                r2 = (((X[:, None] - X[None]) * w) ** 2).sum(axis=2)
                r = np.sqrt(r2 + 1e-12)
                v = {R.K_RBF: lambda: var * np.exp(-r2 / 2), R.K_MATERN12: lambda: var * np.exp(-r),
                     R.K_MATERN32: lambda: var * (1 + np.sqrt(3) * r) * np.exp(-np.sqrt(3) * r),
                     R.K_MATERN52: lambda: var * (1 + np.sqrt(5) * r + 5 / 3 * r * r) * np.exp(-np.sqrt(5) * r)}[kind]()
            term = term * v
        total = total + term
    return total


def _tables(din, M, kinds, seed, shared=False, prior=True, scale=1.0):
    """Tables of a stack of len(kinds) outputs on one data set; kind "rbf" is the plain path."""
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1, 1, (M, din))
    factors, outs = [], []
    for o, kind in enumerate(kinds):
        if shared and factors:
            fac = factors[0]
        else:
            krng = np.random.default_rng(seed + 100 + o)
            if kind == "rbf":
                ls = krng.uniform(0.6, 1.6, din)
                Xs = X / ls
                K = 0.7 * np.exp(-((Xs[:, None] - Xs[None]) ** 2).sum(axis=2) / 2)
                fac = dict(prims=[], lengthscales=ls, variance=0.7, kss=scale * scale * 0.7, Xs=Xs)
            else:
                prims = _prims(kind, din, krng)
                K = _gram(prims, X)
                fac = dict(prims=prims, lengthscales=np.zeros(din), variance=0.0, kss=0.0, Xs=X)
            Kn = (K + 0.01 * np.eye(M)) * scale * scale
            Linv = np.linalg.inv(np.linalg.cholesky(Kn)) if M else np.zeros((0, 0))
            fac.update(M=M, Linv=np.tril(Linv), scale=scale, index=len(factors))
            factors.append(fac)
        p = rng.normal(size=din) if prior else None
        Y = np.sin(X @ rng.normal(size=din) + o) + 0.05 * rng.normal(size=M)
        target = scale * (Y - (X @ p if prior else 0.0))
        outs.append(dict(factor=fac, beta=2.0 if o % 2 == 0 else 1.5, alpha=fac["Linv"] @ target, prior=p))
    return dict(din=din, outputs=outs)


def _cases():
    out = []
    for din in range(1, 7):
        for i, M in enumerate(MS):
            out.append((din, M, ["rbf", "rbf"]))
            out.append((din, M, [EXPRESSIONS[(din + i) % len(EXPRESSIONS)]] * 2))
    return out


@pytest.mark.parametrize("din,M,kinds", _cases())
def test_fp64_in_another_order_lies_inside_the_bound(din, M, kinds):
    tables = _tables(din, M, kinds, seed=din * 100 + M)
    z = R.query_points(tables, 40, np.random.default_rng(M))
    assert R.check_not_too_tight(tables, z) <= 1.0


@pytest.mark.parametrize("kind", ["rbf"] + EXPRESSIONS)
def test_every_expression_kind_at_every_input_dimension(kind):
    for din in range(1, 7):
        tables = _tables(din, 57, [kind, kind], seed=din, scale=1.7)
        z = R.query_points(tables, 30, np.random.default_rng(din))
        assert R.check_not_too_tight(tables, z) <= 1.0, (kind, din)


@pytest.mark.parametrize("din,M,kinds", [(1, 1, ["rbf"]), (2, 9, ["six", "six"]), (3, 257, ["rbf", "rbf"]),
                                         (4, 64, ["matern12", "linear"]), (5, 5, ["rbf", "matern52"]),
                                         (6, 200, ["white_matern32", "constant_rbf"])])
def test_every_mutation_exceeds_the_bound(din, M, kinds):
    """Shared factors so that the alpha swap applies; the query points start next to the dropped rows."""
    tables = _tables(din, M, kinds, seed=7 * din + M, shared=True)
    z = R.query_points(tables, 64, np.random.default_rng(din))
    ratios = R.mutation_ratios(tables, z)
    assert set(ratios) >= {"drop_last_row", "drop_first_row", "drop_last_block", "swap_points"}
    if len(kinds) > 1:
        assert "swap_alpha" in ratios
    assert min(ratios.values()) >= 10.0, ratios


def test_reference_agrees_with_a_direct_solve():
    """Independent of the bound: mean and var against scipy's triangular solve on the noisy Gram matrix."""
    from scipy.linalg import solve_triangular
    tables = _tables(3, 40, ["rbf"], seed=3)
    out = tables["outputs"][0]
    fac = out["factor"]
    z = R.query_points(tables, 16, np.random.default_rng(1))
    zs = z / fac["lengthscales"]
    k = 0.7 * np.exp(-((zs[:, None] - fac["Xs"][None]) ** 2).sum(axis=2) / 2)
    L = np.linalg.inv(fac["Linv"])
    a = solve_triangular(L, k.T, lower=True)
    ref = R.reference(tables, z)
    np.testing.assert_allclose(ref["mean"][:, 0].astype(float), a.T @ out["alpha"] + z @ out["prior"], rtol=1e-9)
    np.testing.assert_allclose(ref["var"][:, 0].astype(float), 0.7 - (a * a).sum(axis=0), rtol=1e-7, atol=1e-12)


# ------------------------------------------------------------------------ slb_debug_refine (host side)
def _sweep(num_outputs=1):
    """A sweep descriptor whose checks pass up to the device work (tables at fake addresses)."""
    cfg = nat.SlbSweep()
    cfg.grid.ndim, cfg.grid.nindex = 2, 100
    for c in range(2):
        cfg.grid.num_points[c], cfg.grid.unit_maxes[c], cfg.grid.upper[c] = 10, 0.1, 1.0
    cfg.gp.num_outputs, cfg.gp.num_factors, cfg.gp.input_dim = num_outputs, 1 if num_outputs else 0, 3
    return cfg


def _refine(cfg, n_max=10, list_=FAKE, count=FAKE, negative=FAKE, workspace=FAKE):
    return nat.load().slb_debug_refine(None, cfg, 0, n_max, list_, count, negative, None, None, None, workspace)


def _rejected(rc, *words):
    err = nat.last_error()
    assert rc == 1, err
    for w in words:
        assert w in err, err


def test_debug_refine_symbol():
    lib = nat.load()
    assert hasattr(lib, "slb_debug_refine")
    assert len(nat.SIGNATURES["slb_debug_refine"][1]) == 11
    assert lib.slb_abi_version() == 6


def test_debug_refine_rejections():
    lib = nat.load()
    _rejected(lib.slb_debug_refine(None, None, 0, 1, FAKE, FAKE, FAKE, None, None, None, FAKE),
              "slb_debug_refine: null config")
    _rejected(_refine(_sweep(num_outputs=0)), "slb_debug_refine needs GP dynamics")
    for kw in ("list_", "count", "negative", "workspace"):
        _rejected(_refine(_sweep(), **{kw: None}), "slb_debug_refine: null list, count, negative or workspace")
    _rejected(_refine(_sweep(), n_max=-1), "slb_debug_refine: n_max -1 outside [0, 4194304]")
    chunk = lib.slb_filter_workspace(1 << 40) - lib.slb_filter_workspace(0)
    chunk //= (lib.slb_filter_workspace(1) - lib.slb_filter_workspace(0))
    assert chunk == 1 << 22
    _rejected(_refine(_sweep(), n_max=chunk + 1), "outside [0, 4194304]")
