"""numpy reference of the joint log marginal likelihood of a GP with k target columns under one kernel and
noise (gpflow 0.4.0 ``GPR`` with ``Y`` [M, k]) and its analytic hyper-parameter gradient, for the tests of
``GPRCached.log_likelihood_and_gradient`` / ``optimize`` on multi-output models.  It builds on the one-column
reference (``tests/gp_lml_reference.py``): the same oracle kernels, parameter paths and kernel derivatives."""
import numpy as np
import scipy.linalg

from gp_lml_reference import kernel_derivatives, parameters


def log_likelihood_and_gradient_cols(kern, noise, X, Y, rows=None):
    """The LML sums the columns' log densities, -(kM/2) log 2 pi - k sum_i log L_ii - 1/2 sum_c |L^-1 d_c|^2,
    and W = sum_c alpha_c alpha_c^T - k K^-1 with alpha = K^-1 D, D = Y - X rows^T.  Returns (LML, grads, mags):
    {path: per-component gradient} and {path: 1/2 sum_ij |W|_ij |d K_ij / d theta|} with |W| taken term by term,
    the scale of the rounding a correct implementation may differ by."""
    params = parameters(kern, noise)
    M, k = Y.shape
    grads, mags = {}, {}
    if M == 0:
        for path, (owner, name) in params.items():
            n = np.size(getattr(owner, name))
            grads[path], mags[path] = np.zeros(n), np.zeros(n)
        return 0.0, grads, mags
    K, der = kernel_derivatives(kern, X)
    Kn = K + np.eye(M) * noise.variance
    D = Y - (X.dot(rows.T) if rows is not None else 0.0)
    L = np.linalg.cholesky(Kn)
    a = scipy.linalg.solve_triangular(L, D, lower=True)
    lml = float(-0.5 * k * M * np.log(2 * np.pi) - k * np.sum(np.log(np.diag(L))) - 0.5 * np.sum(a * a))
    cho = scipy.linalg.cho_factor(Kn, lower=True)
    alpha = scipy.linalg.cho_solve(cho, D)
    Kinv = scipy.linalg.cho_solve(cho, np.eye(M))
    W = alpha.dot(alpha.T) - k * Kinv
    Wabs = np.abs(alpha).dot(np.abs(alpha).T) + k * np.abs(Kinv)
    for path, (owner, name) in params.items():
        dK = np.eye(M)[None] if owner is noise else der[(id(owner), name)]
        grads[path] = 0.5 * np.einsum("ij,cij->c", W, dK)
        mags[path] = 0.5 * np.einsum("ij,cij->c", Wabs, np.abs(dK))
    return lml, grads, mags
