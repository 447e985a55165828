"""numpy reference of the GP log marginal likelihood and its analytic hyper-parameter gradient on the
oracle's kernels (``oracle.reference_path``: gpflow 0.4.0 arithmetic), for the tests of
``GPRCached.compute_log_likelihood`` / ``log_likelihood_and_gradient`` / ``optimize``.

It differentiates the kernel TREE (``Add`` / ``Prod`` nodes, product rule over a node's children), not
the sum-of-products normal form the device kernel works on, and names parameters by their tree paths
(``kern.kern_list[1].kern_list[0].lengthscales``, ``likelihood.variance``); a primitive object reached
by several paths is one parameter (its first path).  Gradients are per component (one value per active
column for lengthscales and the Linear variance); a non-ARD parameter's gradient is their sum."""
import numpy as np
import scipy.linalg

import oracle as O

LOWER = 1e-6          # gpflow 0.4.0 transforms.Log1pe lower bound
STATIONARY = (O.RBF, O.Matern12, O.Matern32, O.Matern52)


def _ard_factory(cls):
    def make(input_dim, **kwargs):
        k = cls(input_dim, **kwargs)
        k.ARD = bool(kwargs.get("ARD", False))       # the oracle's classes take ARD but do not keep it
        return k
    return make


class _Namespace(object):
    pass


ORACLE_KERNELS = _Namespace()
for _name in ("RBF", "Matern12", "Matern32", "Matern52", "Linear", "Constant", "White"):
    setattr(ORACLE_KERNELS, _name, _ard_factory(getattr(O, _name)))


def oracle_kernel(spec):
    """The oracle's kernel of a ``bench_workloads.build_kernel`` spec, primitives marked with ARD."""
    import bench_workloads as W
    return W.build_kernel(ORACLE_KERNELS, spec)


def kernel_set(din):
    """(name, builder) of the test kernels on d_in = din inputs: every primitive kind, ARD and scalar
    parameters, active_dims, sums, products, the notebook form Linear(ARD) + Matern32([0]) * Linear(1),
    a primitive shared by two product terms, and six primitives.  builder(ns) builds the kernel from
    ns's classes (``safe_learning_b200.kernels`` or ``ORACLE_KERNELS``)."""
    ls = np.linspace(0.6, 1.4, din)
    last = [din - 1]

    def rbf_ard(ns):
        return ns.RBF(din, variance=0.8, lengthscales=ls, ARD=True)

    def materns(ns):
        return (ns.Matern12(1, variance=0.5, lengthscales=0.9, active_dims=last)
                + ns.Matern32(din, variance=0.7, lengthscales=1.2)
                + ns.Matern52(din, variance=0.3, lengthscales=ls[::-1].copy(), ARD=True))

    def linear(ns):
        return (ns.Linear(din, variance=np.linspace(0.2, 0.6, din), ARD=True)
                + ns.Linear(1, variance=0.3, active_dims=last))

    def const_white(ns):
        return ns.Constant(din, variance=0.4) + ns.White(din, variance=0.05) + ns.RBF(din, variance=0.6)

    def notebook(ns):
        return (ns.Linear(din, variance=np.linspace(0.02, 0.06, din), ARD=True)
                + ns.Matern32(1, lengthscales=1.0, active_dims=[0]) * ns.Linear(1, variance=0.06))

    def product(ns):
        return ns.Matern32(din, variance=0.9, lengthscales=ls, ARD=True) * ns.Linear(din, variance=0.5)

    def shared(ns):
        c = ns.Linear(1, variance=0.7, active_dims=last)
        return (ns.RBF(din, variance=0.9, lengthscales=1.1)
                + ns.Matern52(1, variance=0.4, lengthscales=0.8, active_dims=[0])) * c

    def six(ns):
        return (ns.RBF(din, variance=0.9, lengthscales=ls, ARD=True) * ns.Matern12(1, lengthscales=1.3)
                * ns.Matern32(1, variance=1.1, lengthscales=0.9, active_dims=last)
                + ns.Matern52(din, variance=0.6, lengthscales=1.1) * ns.Linear(din, variance=0.4)
                * ns.Constant(din, variance=0.8))

    return [("rbf_ard", rbf_ard), ("materns", materns), ("linear", linear), ("const_white", const_white),
            ("notebook", notebook), ("product", product), ("shared", shared), ("six", six)]


def data(din, M, seed=0, noise_std=0.1):
    """Seeded inputs in [-1, 1]^din and targets of a smooth function plus noise [M, 1]."""
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1, 1, (M, din))
    Y = np.sin(2.0 * X).sum(axis=1, keepdims=True) + 0.3 * X[:, :1] + noise_std * rng.standard_normal((M, 1))
    return X, Y


def _params_of(prim):
    if isinstance(prim, STATIONARY):
        return ("variance", "lengthscales")
    return ("variance",)


def primitives(kern, path="kern"):
    """[(path, primitive)] in tree order, each object once."""
    out, seen = [], set()

    def walk(k, p):
        if isinstance(k, (O.Add, O.Prod)):
            for i, sub in enumerate(k.kern_list):
                walk(sub, "%s.kern_list[%d]" % (p, i))
        elif id(k) not in seen:
            seen.add(id(k))
            out.append((p, k))

    walk(kern, path)
    return out


def parameters(kern, noise):
    """{path: (owner, attribute)} of the kernel's parameters and the noise (``likelihood.variance``)."""
    out = {}
    for path, prim in primitives(kern):
        for name in _params_of(prim):
            out["%s.%s" % (path, name)] = (prim, name)
    out["likelihood.variance"] = (noise, "variance")
    return out


def _prim_derivatives(k, X):
    """K(X) of primitive k and {(id(k), name): [n, M, M]} derivative per parameter component."""
    M = X.shape[0]
    K = k.K(X)
    Xa = X[:, k.active_dims]
    if isinstance(k, STATIONARY):
        ls = k.lengthscales
        D = np.square(Xa[:, None, :] - Xa[None, :, :]) / ls ** 3          # [M, M, n]: (x_c - x'_c)^2 / l^3
        base = K / k.variance if k.variance != 0 else type(k)(k.input_dim, 1.0, ls, k.active_dims).K(X)
        if isinstance(k, O.RBF):
            fac = k.variance * base                                        # d K / d l_c = K D_c
        else:
            r = k.euclid_dist(X)
            if isinstance(k, O.Matern12):
                fac = k.variance * np.exp(-r) / r
            elif isinstance(k, O.Matern32):
                fac = 3.0 * k.variance * np.exp(-np.sqrt(3.) * r)
            else:
                fac = 5.0 / 3.0 * k.variance * (1. + np.sqrt(5.) * r) * np.exp(-np.sqrt(5.) * r)
        dls = np.moveaxis(fac[:, :, None] * D, 2, 0)
        return K, {(id(k), "variance"): base[None], (id(k), "lengthscales"): dls}
    if isinstance(k, O.Linear):
        return K, {(id(k), "variance"): np.einsum("ic,jc->cij", Xa, Xa)}
    if isinstance(k, O.Constant):
        return K, {(id(k), "variance"): np.ones((1, M, M))}
    if isinstance(k, O.White):
        return K, {(id(k), "variance"): np.eye(M)[None]}
    raise TypeError(type(k))


def kernel_derivatives(kern, X):
    """K(X) and {(id(prim), name): d K / d component [n, M, M]} by the product rule over the tree."""
    if isinstance(kern, O.Add):
        K, der = None, {}
        for sub in kern.kern_list:
            Ks, ds = kernel_derivatives(sub, X)
            K = Ks if K is None else K + Ks
            for key, v in ds.items():
                der[key] = der[key] + v if key in der else v
        return K, der
    if isinstance(kern, O.Prod):
        parts = [kernel_derivatives(sub, X) for sub in kern.kern_list]
        K, der = None, {}
        for i, (Ki, di) in enumerate(parts):
            K = Ki if K is None else K * Ki
            others = np.ones_like(Ki)
            for j, (Kj, _) in enumerate(parts):
                if j != i:
                    others = others * Kj
            for key, v in di.items():
                v = v * others[None]
                der[key] = der[key] + v if key in der else v
        return K, der
    return _prim_derivatives(kern, X)


class Noise(object):
    def __init__(self, variance):
        self.variance = float(variance)


def log_likelihood(kern, noise, X, Y, mean=None):
    """gpflow 0.4.0 GPR.build_likelihood: log N(Y | m(X), K(X) + noise I)."""
    M = X.shape[0]
    if M == 0:
        return 0.0
    d = Y[:, 0] - (mean(X)[:, 0] if mean is not None else 0.0)
    L = np.linalg.cholesky(kern.K(X) + np.eye(M) * noise.variance)
    a = scipy.linalg.solve_triangular(L, d, lower=True)
    return float(-0.5 * M * np.log(2 * np.pi) - np.sum(np.log(np.diag(L))) - 0.5 * a.dot(a))


def log_likelihood_and_gradient(kern, noise, X, Y, mean=None, with_magnitude=False):
    """(LML, {path: per-component gradient [n]}) and, if asked, {path: 1/2 sum_ij |W_ij| |d K_ij / d
    theta| per component}: the scale of the rounding a correct implementation may differ by."""
    params = parameters(kern, noise)
    M = X.shape[0]
    grads, mags = {}, {}
    if M == 0:
        for path, (owner, name) in params.items():
            n = np.size(getattr(owner, name))
            grads[path], mags[path] = np.zeros(n), np.zeros(n)
        return (0.0, grads, mags) if with_magnitude else (0.0, grads)
    K, der = kernel_derivatives(kern, X)
    Kn = K + np.eye(M) * noise.variance
    cho = scipy.linalg.cho_factor(Kn, lower=True)
    d = Y[:, 0] - (mean(X)[:, 0] if mean is not None else 0.0)
    alpha = scipy.linalg.cho_solve(cho, d)
    Kinv = scipy.linalg.cho_solve(cho, np.eye(M))
    W = np.outer(alpha, alpha) - Kinv
    lml = log_likelihood(kern, noise, X, Y, mean)
    for path, (owner, name) in params.items():
        dK = np.eye(M)[None] if owner is noise else der[(id(owner), name)]
        grads[path] = 0.5 * np.einsum("ij,cij->c", W, dK)
        mags[path] = 0.5 * np.einsum("ij,cij->c", np.abs(W), np.abs(dK))
    return (lml, grads, mags) if with_magnitude else (lml, grads)


# ---- the fit gpflow 0.4.0 Model.optimize runs, on the reference objective ------------------------------
def _softplus(x):
    return np.logaddexp(0.0, x) + LOWER


def _softplus_inv(y):
    ys = y - LOWER
    return ys + np.log(-np.expm1(-ys))


def pack(kern, noise, fixed=()):
    """free paths and the free vector of the current values (non-ARD values collapsed to one entry)."""
    params = parameters(kern, noise)
    free = [p for p in params if p not in fixed]
    values = []
    for p in free:
        owner, name = params[p]
        v = np.atleast_1d(np.asarray(getattr(owner, name), dtype=np.float64))
        values.append(v if getattr(owner, "ARD", False) else v[:1])
    return free, np.concatenate(values)


def _assign(kern, noise, free, y):
    params, k = parameters(kern, noise), 0
    for p in free:
        owner, name = params[p]
        old = getattr(owner, name)
        n = np.size(old) if getattr(owner, "ARD", False) else 1
        if np.ndim(old) == 0:
            setattr(owner, name, float(y[k]))
        else:
            setattr(owner, name, np.broadcast_to(y[k:k + n], np.shape(old)).copy())
        k += n


def objective(kern, noise, X, Y, mean, free, ard):
    """-LML and its gradient in the free space, for scipy.optimize.minimize(jac=True)."""
    def fun(x):
        _assign(kern, noise, free, _softplus(x))
        lml, grads = log_likelihood_and_gradient(kern, noise, X, Y, mean)
        g = np.concatenate([grads[p] if ard[p] else np.sum(grads[p], keepdims=True) for p in free])
        return -lml, -g * (1.0 / (1.0 + np.exp(-x)))
    return fun


def fit(kern, noise, X, Y, mean=None, fixed=(), maxiter=1000):
    """scipy L-BFGS-B on the reference objective; leaves the fitted values in kern / noise."""
    import scipy.optimize
    params = parameters(kern, noise)
    free, y0 = pack(kern, noise, fixed)
    ard = {p: bool(getattr(params[p][0], "ARD", False)) for p in free}
    res = scipy.optimize.minimize(objective(kern, noise, X, Y, mean, free, ard), _softplus_inv(y0),
                                  method="L-BFGS-B", jac=True, options=dict(maxiter=maxiter))
    _assign(kern, noise, free, _softplus(res.x))
    return res
