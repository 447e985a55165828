"""CPU tests of the GP marginal likelihood: the numpy reference (tests/gp_lml_reference.py) against
scipy's multivariate normal and against central differences of itself, the host side of
GPRCached.hyperparameters / log_likelihood_and_gradient / optimize (paths, the chain rule from the
device kernel's descriptor slots to parameters, fixed parameters, the positive transform), and the
host checks of slb_gp_lml_grad.  No call here launches a kernel."""
import numpy as np
import pytest
import scipy.stats
import torch
from numpy.testing import assert_allclose

import gp_lml_reference as R
import oracle as O

SPECS = [
    '["rbf", 3, {"variance": 0.7, "lengthscales": [0.8, 1.3, 0.6], "ARD": true}]',
    '["rbf", 3, {"variance": 1.2, "lengthscales": 0.9}]',
    '["matern12", 2, {"variance": 0.5, "lengthscales": [0.7, 1.1], "active_dims": [0, 2], "ARD": true}]',
    '["matern32", 3, {"variance": 0.9, "lengthscales": 1.3}]',
    '["matern52", 1, {"variance": 0.6, "lengthscales": 0.8, "active_dims": [1]}]',
    '["linear", 3, {"variance": [0.3, 0.5, 0.2], "ARD": true}]',
    '["linear", 2, {"variance": 0.4, "active_dims": [0, 2]}]',
    '["add", ["constant", 3, {"variance": 0.3}], ["white", 3, {"variance": 0.05}], ["rbf", 3]]',
    # the notebook kernels: Linear(3, ARD) + Matern32(1, active_dims=[0]) * Linear(1), Matern32 * Linear
    '["add", ["linear", 3, {"variance": [0.02, 0.06, 0.015], "ARD": true}], '
    '["prod", ["matern32", 1, {"lengthscales": 1.0, "active_dims": [0]}], ["linear", 1, {"variance": 0.06}]]]',
    '["prod", ["matern32", 3, {"lengthscales": [1.1, 0.7, 1.4], "ARD": true}], ["linear", 3, {"variance": 0.5}]]',
]
PRIOR = np.array([[0.4, -0.2, 0.3]])


def _case(M, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1, 1, (M, 3))
    Y = np.sin(2 * X).sum(axis=1, keepdims=True) + 0.1 * rng.standard_normal((M, 1))
    return X, Y


@pytest.mark.parametrize("M", [0, 1, 7, 40])
@pytest.mark.parametrize("prior", [False, True])
@pytest.mark.parametrize("spec", SPECS)
def test_reference_lml_is_the_gaussian_logpdf(spec, prior, M):
    X, Y = _case(M, seed=M)
    kern = R.oracle_kernel(spec)
    mean = O.LinearMean(PRIOR) if prior else None
    noise = R.Noise(0.04)
    lml = R.log_likelihood(kern, noise, X, Y, mean)
    if M == 0:
        assert lml == 0.0
        return
    cov = kern.K(X) + 0.04 * np.eye(M)
    mu = mean(X)[:, 0] if prior else np.zeros(M)
    want = scipy.stats.multivariate_normal.logpdf(Y[:, 0], mean=mu, cov=cov)
    assert_allclose(lml, want, rtol=1e-12)


@pytest.mark.parametrize("prior", [False, True])
@pytest.mark.parametrize("spec", SPECS)
def test_reference_gradient_is_the_central_difference(spec, prior):
    X, Y = _case(30, seed=5)
    kern = R.oracle_kernel(spec)
    noise = R.Noise(0.04)
    mean = O.LinearMean(PRIOR) if prior else None
    _, grads = R.log_likelihood_and_gradient(kern, noise, X, Y, mean)
    for path, (owner, name) in R.parameters(kern, noise).items():
        value = np.atleast_1d(np.asarray(getattr(owner, name), dtype=np.float64)).copy()
        assert grads[path].shape == value.shape
        for c in range(value.size):
            h = 1e-4 * value[c]
            fd = []
            for s in (h, -h):
                v = value.copy()
                v[c] += s
                setattr(owner, name, v if np.ndim(getattr(owner, name)) else float(v[0]))
                fd.append(R.log_likelihood(kern, noise, X, Y, mean))
            setattr(owner, name, value if np.ndim(getattr(owner, name)) else float(value[0]))
            assert_allclose(grads[path][c], (fd[0] - fd[1]) / (2 * h), rtol=1e-6, atol=1e-6,
                            err_msg="%s[%d]" % (path, c))


def test_reference_gradient_of_an_empty_data_set_is_zero():
    kern = R.oracle_kernel(SPECS[8])
    lml, grads = R.log_likelihood_and_gradient(kern, R.Noise(0.1), np.zeros((0, 3)), np.zeros((0, 1)))
    assert lml == 0.0 and all(not np.any(g) for g in grads.values())


# ---------------------------------------------------------------- product host side
@pytest.fixture(scope="module")
def sl():
    import __graft_entry__
    __graft_entry__.build()
    import safe_learning_b200 as sl
    return sl


def _shared_model(sl):
    """(a + b) * c: c sits in both product terms (normal form a c + b c)."""
    k = sl.kernels
    a = k.RBF(2, variance=0.7, lengthscales=[0.8, 1.3], ARD=True)
    b = k.Linear(2, variance=0.4)
    c = k.Matern32(1, variance=0.9, lengthscales=1.5, active_dims=[1])
    gp = sl.GPR(np.zeros((0, 2)), np.zeros((0, 1)), (a + b) * c, noise_variance=0.01)
    return gp, a, b, c


def test_hyperparameter_paths_and_values(sl):
    gp, a, b, c = _shared_model(sl)
    hp = gp.hyperparameters()
    assert list(hp) == ["kern.kern_list[0].kern_list[0].variance", "kern.kern_list[0].kern_list[0].lengthscales",
                        "kern.kern_list[0].kern_list[1].variance", "kern.kern_list[1].variance",
                        "kern.kern_list[1].lengthscales", "likelihood.variance"]
    assert_allclose(hp["kern.kern_list[0].kern_list[0].lengthscales"], [0.8, 1.3])     # ARD: a vector
    assert hp["kern.kern_list[0].kern_list[1].variance"] == 0.4                        # scalar
    assert hp["kern.kern_list[1].lengthscales"] == 1.5 and hp["likelihood.variance"] == 0.01
    hp["kern.kern_list[0].kern_list[0].lengthscales"][0] = 99.0                       # a copy
    assert a.lengthscales[0] == 0.8
    single = sl.GPR(np.zeros((0, 1)), np.zeros((0, 1)), sl.kernels.RBF(1, variance=2.0))
    assert list(single.hyperparameters()) == ["kern.variance", "kern.lengthscales", "likelihood.variance"]
    bad = sl.GPR(np.zeros((0, 2)), np.zeros((0, 1)), sl.kernels.RBF(2, lengthscales=[1.0, 2.0]))
    with pytest.raises(ValueError, match="ARD is False"):
        bad.hyperparameters()


def test_slot_gradients_chain_to_parameters(sl, monkeypatch):
    """Descriptor slots -> parameters: d/dl = -(d/dw) / l^2, non-ARD sums its columns, the shared c
    sums its two occurrences, Linear's w is its variance, the noise slot is last."""
    gp, a, b, c = _shared_model(sl)
    S = 1 + sl._native.SLB_MAX_IN
    slots = np.random.default_rng(0).standard_normal(sl._native.SLB_GP_HYPER_SLOTS)
    monkeypatch.setattr(type(gp), "_log_likelihood", lambda self, want: (-3.5, slots))
    lml, g = gp.log_likelihood_and_gradient()
    # normal form: [a, c], [b, c] -> descriptor primitives 0: a, 1: c, 2: b, 3: c
    prim = lambda p: (slots[p * S], slots[p * S + 1:(p + 1) * S])
    assert lml == -3.5
    assert_allclose(g["kern.kern_list[0].kern_list[0].variance"], prim(0)[0])
    assert_allclose(g["kern.kern_list[0].kern_list[0].lengthscales"], -prim(0)[1][:2] / np.array([0.8, 1.3]) ** 2)
    assert_allclose(g["kern.kern_list[0].kern_list[1].variance"], prim(2)[1][0] + prim(2)[1][1])
    assert_allclose(g["kern.kern_list[1].variance"], prim(1)[0] + prim(3)[0])
    assert_allclose(g["kern.kern_list[1].lengthscales"], -(prim(1)[1][1] + prim(3)[1][1]) / 1.5 ** 2)
    assert_allclose(g["likelihood.variance"], slots[-1])
    assert np.shape(g["kern.kern_list[0].kern_list[0].lengthscales"]) == (2,)
    assert all(np.ndim(g[p]) == 0 for p in g if not p.endswith("[0].lengthscales"))


def _quadratic_objective(targets):
    """-LML = sum (log v - log t)^2 over every component: the optimum is v = t."""
    def fake(self):
        hp = self.hyperparameters()
        lml, grads = 0.0, {}
        for p, v in hp.items():
            v = np.asarray(v, dtype=np.float64)
            r = np.log(v) - np.log(targets[p])
            lml -= float(np.sum(r * r))
            grads[p] = -2 * r / v if v.ndim else float(-2 * r / v)
        return lml, grads
    return fake


def test_optimize_fixed_and_transform(sl, monkeypatch):
    gp, a, b, c = _shared_model(sl)
    start = gp.hyperparameters()
    targets = {p: np.asarray(v) * 1.7 for p, v in start.items()}
    monkeypatch.setattr(type(gp), "log_likelihood_and_gradient", _quadratic_objective(targets))
    res = gp.optimize(tol=1e-12, fixed=("likelihood.variance", "kern.kern_list[1].lengthscales"))
    assert res.success
    hp = gp.hyperparameters()
    for p in hp:
        want = start[p] if p in ("likelihood.variance", "kern.kern_list[1].lengthscales") else targets[p]
        assert_allclose(hp[p], want, rtol=1e-5, err_msg=p)
    assert gp.likelihood.variance == 0.01 and np.all(c.lengthscales == 1.5)
    assert_allclose(a.lengthscales, [0.8 * 1.7, 1.3 * 1.7], rtol=1e-6)          # written back
    assert_allclose(b.variance, [0.4 * 1.7] * 2, rtol=1e-6)


def test_optimize_softplus_round_trip_and_callback(sl, monkeypatch):
    """At the optimum already: scipy stops at x0, and softplus(softplus^-1(v)) writes v back."""
    gp, a, b, c = _shared_model(sl)
    start = gp.hyperparameters()
    monkeypatch.setattr(type(gp), "log_likelihood_and_gradient", _quadratic_objective(start))
    seen = []
    res = gp.optimize(callback=seen.append, maxiter=5)
    assert res.nit <= 1
    for p, v in gp.hyperparameters().items():
        assert_allclose(v, start[p], rtol=1e-12, err_msg=p)
    x0 = res.x
    assert_allclose(np.logaddexp(0.0, x0) + 1e-6, [0.7, 0.8, 1.3, 0.4, 0.9, 1.5, 0.01], rtol=1e-12)


def test_optimize_rejects_bad_starts_and_paths(sl):
    gp, a, b, c = _shared_model(sl)
    a.variance = 1e-6
    with pytest.raises(ValueError, match="kern.kern_list\\[0\\].kern_list\\[0\\].variance"):
        gp.optimize()
    a.variance = 0.7
    b.variance = np.array([0.4, -1.0])
    with pytest.raises(ValueError):
        gp.optimize()
    b.variance = np.array([0.4, 0.4])
    with pytest.raises(ValueError, match="unknown"):
        gp.optimize(fixed=("kern.nonsense",))
    gp.likelihood.variance = 0.0
    gp.optimize(fixed=("likelihood.variance",), maxiter=1)         # a fixed parameter may be anything


def test_optimize_restores_values_when_the_search_fails(sl, monkeypatch):
    gp, a, b, c = _shared_model(sl)
    start = gp.hyperparameters()
    calls = []

    def failing(self):
        calls.append(1)
        if len(calls) == 3:
            raise torch.linalg.LinAlgError("not positive-definite")
        return _quadratic_objective({p: np.asarray(v) * 3 for p, v in start.items()})(self)

    monkeypatch.setattr(type(gp), "log_likelihood_and_gradient", failing)
    with pytest.raises(torch.linalg.LinAlgError):
        gp.optimize()
    for p, v in gp.hyperparameters().items():
        assert_allclose(v, start[p], rtol=0, atol=0, err_msg=p)


def test_empty_data_set_likelihood(sl):
    gp, a, b, c = _shared_model(sl)
    before = sl._native.launch_count()
    assert gp.compute_log_likelihood() == 0.0
    lml, g = gp.log_likelihood_and_gradient()
    assert lml == 0.0 and all(not np.any(v) for v in g.values())
    assert sl._native.launch_count() == before


# ---------------------------------------------------------------- slb_gp_lml_grad host checks
def _kernel(nat, kinds=(0,), din=3):
    k = nat.SlbKernel()
    k.num_prims = len(kinds)
    for i, kind in enumerate(kinds):
        k.prims[i].kind, k.prims[i].term, k.prims[i].variance = kind, 0, 1.0
        for c in range(din):
            k.prims[i].w[c] = 1.0
    return k


def _call(nat, k, M=0, din=3, bufs=(None,) * 5):
    X, Kinv, alpha, grad, work = bufs
    return nat.load().slb_gp_lml_grad(None, X, M, din, k, Kinv, alpha, grad, work)


@pytest.mark.parametrize("case, message", [
    ("negative M", "negative M"),
    ("d_in 0", "d_in 0 outside 1..8"),
    ("d_in 9", "d_in 9 outside 1..8"),
    ("no primitives", "no primitives"),
    ("too many primitives", "7 kernel primitives outside 0..6"),
    ("unknown kind", "unknown kind 7"),
    ("term order", "term order"),
    ("first term", "terms start at 0"),
    ("negative weight", "negative weight"),
    ("weight beyond d_in", "column 3 beyond d_in = 3"),
    ("null buffers", "null X, Kinv, alpha, grad or workspace"),
])
def test_lml_grad_rejects_malformed_calls(sl, case, message):
    nat = sl._native
    k = _kernel(nat, kinds=(0, 4))
    M, din, bufs = 0, 3, (None,) * 5
    if case == "negative M":
        M = -1
    elif case == "d_in 0":
        din = 0
    elif case == "d_in 9":
        din = 9
    elif case == "no primitives":
        k.num_prims = 0
    elif case == "too many primitives":
        k.num_prims = 7
    elif case == "unknown kind":
        k.prims[1].kind = 7
    elif case == "term order":
        k.prims[1].term = 2
    elif case == "first term":
        k.prims[0].term = k.prims[1].term = 1
    elif case == "negative weight":
        k.prims[1].w[2] = -0.5
    elif case == "weight beyond d_in":
        k.prims[0].w[3] = 0.25
    elif case == "null buffers":
        M, bufs = 5, (0x1000, 0x2000, None, 0x3000, 0x4000)
    before = nat.launch_count()
    assert _call(nat, k, M, din, bufs) != 0
    assert message in nat.last_error(), nat.last_error()
    assert nat.launch_count() == before


def test_lml_grad_empty_data_set_launches_nothing(sl):
    nat = sl._native
    before = nat.launch_count()
    for kinds in ((0,), (1, 2, 3), (4, 5, 6)):
        assert _call(nat, _kernel(nat, kinds)) == 0
    assert nat.launch_count() == before
    assert nat.load().slb_gp_lml_grad_workspace(0) == 0
    assert nat.load().slb_gp_lml_grad_workspace(64) == 1 * nat.SLB_GP_HYPER_SLOTS * 8
    assert nat.load().slb_gp_lml_grad_workspace(65) == 3 * nat.SLB_GP_HYPER_SLOTS * 8
    assert nat.load().slb_gp_lml_grad_workspace(-1) == -1
