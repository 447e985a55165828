"""numpy/scipy fp64 restatement of the reference hot path (TEST INFRASTRUCTURE ONLY).

Reference: befelix/safe_learning @ f1aad5a, paths relative to its source tree.
All objects here are plain numpy callables: ``fun(points) -> ndarray`` where the
reference builds a TF1 graph node.  Operation order of the cheap element-wise
pieces (grid coordinates, linear maps, quadratic forms, barycentric weights, the
decrease / threshold formula) is written out explicitly -- left-to-right sums, one
rounding per multiply and per add, no BLAS, no FMA -- so that a device
implementation can reproduce it bit for bit.  The GP posterior goes through
LAPACK/BLAS like the reference goes through Eigen; parity there is to tolerance.

Pinned behaviours that the reference leaves open (SURVEY.md section 8a Q1-Q5):
stable V-sort (ties broken by flat index), NaN => unsafe.
"""

from __future__ import annotations

import itertools

import numpy as np
import scipy.linalg
import scipy.signal
import scipy.spatial

__all__ = [
    "config", "DimensionError", "GridWorld", "LinearSystem", "QuadraticFunction",
    "Saturation", "ConstantFunction", "ScaledFunction", "AbsFunction", "Norm1Function",
    "MaxAbsFunction",
    "RBF", "Matern12", "Matern32", "Matern52", "Linear", "Constant", "Bias", "White", "Add", "Prod",
    "LinearMean", "GPRCached", "GaussianProcess", "FunctionStack", "Triangulation",
    "InvertedPendulum", "CartPole", "LyapunovNetwork", "NeuralNetwork", "Lyapunov",
    "PolicyIteration",
    "batchify", "dlqr", "hstack_inputs", "stable_value_order", "prefix_rule",
    "perturb_actions", "get_safe_sample", "unique_rows", "smallest_boundary_value",
]


class _Config(object):
    """``safe_learning/configuration.py:8-32``: fp64 everywhere, 10 000-point batches."""

    np_dtype = np.float64
    gp_batch_size = 10000


config = _Config()
_EPS = np.finfo(np.float64).eps


class DimensionError(Exception):
    """``functions.py:575-576``."""


# --------------------------------------------------------------------------- helpers
def hstack_inputs(args):
    """[x, u] column concatenation, ``utilities.py:123-159`` (numpy branch)."""
    cols = [np.atleast_2d(np.asarray(a, dtype=np.float64)) for a in args]
    return cols[0] if len(cols) == 1 else np.hstack(cols)


def _seq_dot(points, matrix_rows):
    """``points @ matrix_rows.T`` with a fixed left-to-right sum and no FMA.

    points [B, k], matrix_rows [o, k] -> [B, o].  Stands in for ``tf.matmul`` at
    ``functions.py:1583`` / ``:1537`` with a defined summation order.
    """
    points = np.asarray(points, dtype=np.float64)
    rows = np.asarray(matrix_rows, dtype=np.float64)
    out = np.empty((points.shape[0], rows.shape[0]), dtype=np.float64)
    for o in range(rows.shape[0]):
        acc = points[:, 0] * rows[o, 0]
        for k in range(1, rows.shape[1]):
            acc = acc + points[:, k] * rows[o, k]
        out[:, o] = acc
    return out


def batchify(arrays, batch_size):
    """Ordered batches ``(start, [views])``; ``utilities.py:224-249``."""
    if not isinstance(arrays, (list, tuple)):
        arrays = (arrays,)
    start = 0
    while True:
        views = [arr[start:start + batch_size] for arr in arrays]
        if views[0].size == 0:
            return
        yield start, views
        start += batch_size


def dlqr(a, b, q, r):
    """Discrete LQR gain and cost-to-go; ``utilities.py:327-356``."""
    a, b, q, r = (np.atleast_2d(m) for m in (a, b, q, r))
    p = scipy.linalg.solve_discrete_are(a, b, q, r)
    btp = b.T.dot(p)
    k = np.linalg.solve(btp.dot(b) + r, btp.dot(a))
    return k, p


# --------------------------------------------------------------------------- grid
class GridWorld(object):
    """Regular grid; ``functions.py:579-817``.

    Flat index k <-> ijk = unravel(k, num_points), last dimension fastest
    (``:622-638``); coordinates are ``ijk * unit_maxes + offset`` with separate
    multiply and add (``:731``).
    """

    def __init__(self, limits, num_points):
        self.limits = np.atleast_2d(limits).astype(np.float64)
        self.num_points = np.broadcast_to(num_points, len(self.limits)).astype(np.int64)
        if np.any(self.num_points < 2):
            raise DimensionError("There must be at least 2 points in each dimension.")
        self.offset = self.limits[:, 0]
        self.unit_maxes = ((self.limits[:, 1] - self.offset)
                           / (self.num_points - 1)).astype(np.float64)
        self.offset_limits = np.stack((np.zeros_like(self.limits[:, 0]),
                                       self.limits[:, 1] - self.offset), axis=1)
        self.discrete_points = [np.linspace(lo, hi, n, dtype=np.float64)
                                for (lo, hi), n in zip(self.limits, self.num_points)]
        self.nrectangles = int(np.prod(self.num_points - 1))
        self.nindex = int(np.prod(self.num_points))
        self.ndim = len(self.limits)
        self._all_points = None

    def __len__(self):
        return self.nindex

    @property
    def all_points(self):
        """``functions.py:622-638`` (meshgrid ``indexing='ij'``, C order)."""
        if self._all_points is None:
            mesh = np.meshgrid(*self.discrete_points, indexing="ij")
            self._all_points = np.column_stack([m.ravel() for m in mesh]).astype(np.float64)
        return self._all_points

    def _check_dimensions(self, states):
        if not states.shape[1] == self.ndim:
            raise DimensionError("the input argument has the wrong dimensions.")

    def _center_states(self, states, clip=True):
        """``functions.py:691-712``."""
        states = np.atleast_2d(states).astype(np.float64)
        states = states - self.offset[None, :]
        if clip:
            np.clip(states, self.offset_limits[:, 0] + 2 * _EPS,
                    self.offset_limits[:, 1] - 2 * _EPS, out=states)
        return states

    def index_to_state(self, indices):
        """``functions.py:714-731``."""
        indices = np.atleast_1d(indices)
        ijk = np.vstack(np.unravel_index(indices, self.num_points)).T.astype(np.float64)
        return ijk * self.unit_maxes + self.offset

    def state_to_index(self, states):
        """``functions.py:733-752`` (clip, scale by 1/unit, rint, ravel)."""
        states = np.atleast_2d(states)
        self._check_dimensions(states)
        states = np.clip(states, self.limits[:, 0], self.limits[:, 1])
        states = (states - self.offset) * (1. / self.unit_maxes)
        ijk = np.rint(states).astype(np.int32)
        return np.ravel_multi_index(ijk.T, self.num_points)

    def state_to_rectangle(self, states):
        """``functions.py:754-776`` (digitize against the linspace values)."""
        ind = []
        for i, (pts, n) in enumerate(zip(self.discrete_points, self.num_points)):
            idx = np.digitize(states[:, i], pts) - 1
            np.clip(idx, 0, n - 2, out=idx)
            ind.append(idx)
        return np.ravel_multi_index(ind, self.num_points - 1)

    def rectangle_to_state(self, rectangles):
        """``functions.py:778-798``."""
        rectangles = np.atleast_1d(rectangles)
        ijk = np.vstack(np.unravel_index(rectangles, self.num_points - 1)).astype(np.float64)
        return (ijk.T * self.unit_maxes) + self.offset

    def rectangle_corner_index(self, rectangles):
        """``functions.py:800-817``."""
        ijk = np.vstack(np.unravel_index(rectangles, self.num_points - 1))
        return np.ravel_multi_index(np.atleast_2d(ijk), self.num_points)


# --------------------------------------------------------------------------- small functions
class LinearSystem(object):
    """``y = [x, u] . A^T``; ``functions.py:1546-1583``."""

    def __init__(self, matrices):
        if isinstance(matrices, np.ndarray):
            matrices = (matrices,)
        self.matrix = np.hstack([np.atleast_2d(m).astype(np.float64) for m in matrices])
        self.output_dim, self.input_dim = self.matrix.shape

    def __call__(self, *inputs):
        return _seq_dot(hstack_inputs(inputs), self.matrix)


class QuadraticFunction(object):
    """``sum((x P) * x, axis=1)``; ``functions.py:1513-1543``. P is NOT symmetrised."""

    def __init__(self, matrix):
        self.matrix = np.atleast_2d(matrix).astype(np.float64)
        self.ndim = self.matrix.shape[0]
        self.input_dim, self.output_dim = self.ndim, 1

    def __call__(self, *inputs):
        x = hstack_inputs(inputs)
        lin = _seq_dot(x, self.matrix.T)         # (x P)_c = sum_r x_r P[r, c]
        prod = lin * x
        acc = prod[:, 0]
        for c in range(1, prod.shape[1]):
            acc = acc + prod[:, c]
        return acc[:, None]

    def gradient(self, points):
        """``functions.py:1541-1543``."""
        return _seq_dot(np.atleast_2d(points), (self.matrix + self.matrix.T).T)


class Saturation(object):
    """``min(max(fun(x), lower), upper)``; ``functions.py:310-354``."""

    def __init__(self, fun, lower, upper):
        self.fun, self.lower, self.upper = fun, lower, upper
        self.input_dim, self.output_dim = fun.input_dim, fun.output_dim

    def __call__(self, *inputs):
        return np.minimum(np.maximum(self.fun(*inputs), self.lower), self.upper)


class ConstantFunction(object):
    """``functions.py:241-251``."""

    def __init__(self, constant):
        self.constant = constant

    def __call__(self, *inputs):
        x = hstack_inputs(inputs)
        return np.broadcast_to(np.asarray(self.constant, dtype=np.float64), (x.shape[0], 1)).copy()


class ScaledFunction(object):
    """``fun * c`` (``MultipliedFunction`` with a constant, ``functions.py:163-199``; ``__neg__`` ``:120-122``)."""

    def __init__(self, fun, factor):
        self.fun, self.factor = fun, float(factor)

    def __call__(self, *inputs):
        return self.fun(*inputs) * self.factor


class AbsFunction(object):
    """``tf.abs(fun(x))`` -- the per-dimension local Lipschitz lambda of
    ``examples/adaptive_safety_verification.ipynb`` cell 17."""

    def __init__(self, fun):
        self.fun = fun

    def __call__(self, *inputs):
        return np.abs(self.fun(*inputs))


class Norm1Function(object):
    """``tf.norm(fun(x), ord=1, axis=1, keepdims=True)`` (same notebook cell, else branch)."""

    def __init__(self, fun):
        self.fun = fun

    def __call__(self, *inputs):
        return _row_norm1(self.fun(*inputs))


class MaxAbsFunction(object):
    """``tf.reduce_max(tf.abs(fun(x)), axis=1, keepdims=True)``
    (``examples/inverted_pendulum.ipynb`` cell 14)."""

    def __init__(self, fun):
        self.fun = fun

    def __call__(self, *inputs):
        return np.max(np.abs(self.fun(*inputs)), axis=1, keepdims=True)


def _row_norm1(values):
    values = np.abs(values)
    acc = values[:, 0]
    for c in range(1, values.shape[1]):
        acc = acc + values[:, c]
    return acc[:, None]


# --------------------------------------------------------------------------- GP (gpflow 0.4.0 restated)
class Kernel(object):
    """``gpflow==0.4.0`` ``kernels.Kern`` algebra (third party, pinned ``requirements.txt:3``; not under
    the upstream sources, restated from its published arithmetic): every primitive works on the columns
    ``active_dims`` (default: the first ``input_dim``), ``k1 + k2`` / ``k1 * k2`` add / multiply the
    covariance matrices (``Add`` / ``Prod``).  Used by the reference's experiments
    (``examples/inverted_pendulum.ipynb`` cell 6, ``1d_region_of_attraction_estimate.ipynb`` cell 5)."""

    def __init__(self, input_dim, active_dims=None):
        self.input_dim = int(input_dim)
        if active_dims is None:
            active_dims = range(self.input_dim)
        elif isinstance(active_dims, slice):
            active_dims = range(*active_dims.indices(1 << 30))[:self.input_dim]
        self.active_dims = [int(a) for a in active_dims]

    def _slice(self, X, X2):
        X = X[:, self.active_dims]
        return X, (None if X2 is None else X2[:, self.active_dims])

    def __add__(self, other):
        return Add([self, other])

    def __mul__(self, other):
        return Prod([self, other])


class Add(Kernel):
    def __init__(self, kern_list):
        self.kern_list = list(kern_list)

    def K(self, X, X2=None):
        out = self.kern_list[0].K(X, X2)
        for k in self.kern_list[1:]:
            out = out + k.K(X, X2)
        return out

    def Kdiag(self, X):
        out = self.kern_list[0].Kdiag(X)
        for k in self.kern_list[1:]:
            out = out + k.Kdiag(X)
        return out


class Prod(Kernel):
    def __init__(self, kern_list):
        self.kern_list = list(kern_list)

    def K(self, X, X2=None):
        out = self.kern_list[0].K(X, X2)
        for k in self.kern_list[1:]:
            out = out * k.K(X, X2)
        return out

    def Kdiag(self, X):
        out = self.kern_list[0].Kdiag(X)
        for k in self.kern_list[1:]:
            out = out * k.Kdiag(X)
        return out


class Stationary(Kernel):
    """gpflow 0.4.0 ``Stationary``: ``square_dist`` by the ``|x|^2 + |x'|^2 - 2 x.x'`` expansion on
    lengthscale-divided inputs, ``euclid_dist = sqrt(square_dist + 1e-12)``, ``Kdiag = variance``."""

    def __init__(self, input_dim, variance=1.0, lengthscales=None, active_dims=None, ARD=False):
        Kernel.__init__(self, input_dim, active_dims)
        self.variance = float(variance)
        ls = 1.0 if lengthscales is None else lengthscales
        self.lengthscales = np.broadcast_to(np.asarray(ls, dtype=np.float64),
                                            (self.input_dim,)).copy()

    def square_dist(self, X, X2=None):
        X, X2 = self._slice(X, X2)
        X = X / self.lengthscales
        Xs = np.sum(np.square(X), axis=1)
        if X2 is None:
            return -2 * X.dot(X.T) + Xs[:, None] + Xs[None, :]
        X2 = X2 / self.lengthscales
        X2s = np.sum(np.square(X2), axis=1)
        return -2 * X.dot(X2.T) + Xs[:, None] + X2s[None, :]

    def euclid_dist(self, X, X2=None):
        return np.sqrt(self.square_dist(X, X2) + 1e-12)

    def Kdiag(self, X):
        return np.full(X.shape[0], self.variance, dtype=np.float64)


class RBF(Stationary):
    """``gpflow==0.4.0`` ``kernels.RBF``: ``K = variance * exp(-square_dist/2)``.  Defaults
    variance = lengthscales = 1.  Pinned by the golden vector ``tests/test_functions.py:237-261``."""

    def K(self, X, X2=None):
        return self.variance * np.exp(-self.square_dist(X, X2) / 2)


class Matern12(Stationary):
    def K(self, X, X2=None):
        return self.variance * np.exp(-self.euclid_dist(X, X2))


class Matern32(Stationary):
    def K(self, X, X2=None):
        r = self.euclid_dist(X, X2)
        return self.variance * (1. + np.sqrt(3.) * r) * np.exp(-np.sqrt(3.) * r)


class Matern52(Stationary):
    def K(self, X, X2=None):
        r = self.euclid_dist(X, X2)
        return self.variance * (1. + np.sqrt(5.) * r + 5. / 3. * np.square(r)) * np.exp(-np.sqrt(5.) * r)


class Linear(Kernel):
    """gpflow 0.4.0 ``kernels.Linear``: ``K = (X * variance) X2^T``, ``Kdiag = sum(X^2 * variance)``."""

    def __init__(self, input_dim, variance=1.0, active_dims=None, ARD=False):
        Kernel.__init__(self, input_dim, active_dims)
        self.variance = np.broadcast_to(np.asarray(variance, dtype=np.float64),
                                        (self.input_dim,)).copy()

    def K(self, X, X2=None):
        X, X2 = self._slice(X, X2)
        return (X * self.variance).dot((X if X2 is None else X2).T)

    def Kdiag(self, X):
        X, _ = self._slice(X, None)
        return np.sum(np.square(X) * self.variance, axis=1)


class Constant(Kernel):
    def __init__(self, input_dim, variance=1.0, active_dims=None):
        Kernel.__init__(self, input_dim, active_dims)
        self.variance = float(variance)

    def K(self, X, X2=None):
        return np.full((X.shape[0], (X if X2 is None else X2).shape[0]), self.variance)

    def Kdiag(self, X):
        return np.full(X.shape[0], self.variance, dtype=np.float64)


Bias = Constant


class White(Kernel):
    def __init__(self, input_dim, variance=1.0, active_dims=None):
        Kernel.__init__(self, input_dim, active_dims)
        self.variance = float(variance)

    def K(self, X, X2=None):
        if X2 is None:
            return self.variance * np.eye(X.shape[0])
        return np.zeros((X.shape[0], X2.shape[0]))

    def Kdiag(self, X):
        return np.full(X.shape[0], self.variance, dtype=np.float64)


class LinearMean(object):
    """A one-output linear prior mean ``m(z) = z . a`` -- what a
    ``LinearSystem((A[[j], :], B[[j], :]))`` mean function evaluates to
    (``examples/adaptive_safety_verification.ipynb`` cell 9)."""

    def __init__(self, row):
        self.row = np.asarray(row, dtype=np.float64).reshape(1, -1)

    def __call__(self, X):
        return _seq_dot(X, self.row)


class GPRCached(object):
    """GP regression with cached Cholesky; ``functions.py:357-458``.

    cache (``:395-411``): ``L = chol(scale^2 (K + noise I))``, ``alpha = L^-1 scale (Y - m(X))``.
    predict (``:417-458``): ``a = L^-1 scale^2 K(X, x*)``, ``mean = (a^T alpha + scale m(x*)) / scale``,
    ``var = (scale^2 Kdiag - sum a^2) / scale^2`` (latent variance, never clamped).
    """

    def __init__(self, x, y, kern, mean_function=None, noise_variance=1.0, scale=1.0):
        self.X = np.atleast_2d(np.asarray(x, dtype=np.float64))
        self.Y = np.atleast_2d(np.asarray(y, dtype=np.float64))
        self.kern = kern
        self.mean_function = mean_function
        self.noise_variance = float(noise_variance)
        self._scale = float(scale)
        self.update_cache()

    def _mean(self, X):
        if self.mean_function is None:
            return np.zeros((X.shape[0], 1), dtype=np.float64)
        return self.mean_function(X)

    def update_cache(self):
        if self.X.shape[0] == 0:        # empty data set: prior only (zero-size TF ops upstream)
            self.cholesky, self.alpha = np.zeros((0, 0)), np.zeros((0, 1))
            return
        kernel = self.kern.K(self.X) + np.eye(self.X.shape[0]) * self.noise_variance
        kernel = kernel * (self._scale ** 2)
        target = self._scale * (self.Y - self._mean(self.X))
        self.cholesky = np.linalg.cholesky(kernel)
        self.alpha = scipy.linalg.solve_triangular(self.cholesky, target, lower=True)

    def build_predict(self, Xnew):
        Xnew = np.atleast_2d(np.asarray(Xnew, dtype=np.float64))
        mx = self._scale * self._mean(Xnew)
        if self.X.shape[0] == 0:
            a = np.zeros((0, Xnew.shape[0]))
        else:
            Kx = (self._scale ** 2) * self.kern.K(self.X, Xnew)
            a = scipy.linalg.solve_triangular(self.cholesky, Kx, lower=True)
        fmean = a.T.dot(self.alpha) + mx
        Knew = (self._scale ** 2) * self.kern.Kdiag(Xnew)
        fvar = Knew - np.sum(np.square(a), axis=0)
        fvar = np.tile(fvar.reshape(-1, 1), (1, self.Y.shape[1]))
        return fmean / self._scale, fvar / (self._scale ** 2)


class GaussianProcess(object):
    """``functions.py:461-546``: ``(mean, beta * sqrt(var))``; inputs are concatenated."""

    def __init__(self, gaussian_process, beta=2.0):
        self.gaussian_process = gaussian_process
        self.beta = float(beta)
        self.input_dim = gaussian_process.X.shape[1]
        self.output_dim = gaussian_process.Y.shape[1]

    @property
    def X(self):
        return self.gaussian_process.X

    @property
    def Y(self):
        return self.gaussian_process.Y

    def __call__(self, *inputs):
        mean, var = self.gaussian_process.build_predict(hstack_inputs(inputs))
        with np.errstate(invalid="ignore"):
            std = self.beta * np.sqrt(var)          # var < 0 -> NaN, as tf.sqrt (:514)
        return mean, std

    def add_data_point(self, x, y):
        gp = self.gaussian_process
        gp.X = np.vstack((gp.X, np.atleast_2d(x)))
        gp.Y = np.vstack((gp.Y, np.atleast_2d(y)))
        gp.update_cache()


class FunctionStack(object):
    """``functions.py:254-307``: column-stack the (mean, error) pairs of 1-output GPs."""

    def __init__(self, functions):
        self.functions = list(functions)
        self.num_fun = len(self.functions)
        self.input_dim = self.functions[0].input_dim
        self.output_dim = sum(f.output_dim for f in self.functions)

    def __call__(self, *inputs):
        points = hstack_inputs(inputs)
        pairs = [f(points) for f in self.functions]
        return (np.concatenate([p[0] for p in pairs], axis=1),
                np.concatenate([p[1] for p in pairs], axis=1))

    def add_data_point(self, x, y):
        for fun, yi in zip(self.functions, np.asarray(y).squeeze()):
            fun.add_data_point(x, yi)


# --------------------------------------------------------------------------- triangulation
class _Delaunay1D(object):
    """``functions.py:935-978``."""

    def __init__(self, points):
        self.points = points
        self.nsimplex = len(points) - 1
        self._min, self._max = np.min(points), np.max(points)
        self.simplices = np.array([[0, 1]])

    def find_simplex(self, points):
        points = points.squeeze()
        outside = (points > self._max) | (points < self._min)
        return np.where(outside, -1, 0)


class Triangulation(object):
    """Piecewise-linear interpolation on a grid; ``functions.py:981-1226`` and the
    TF evaluation ``:1442-1499``.

    One unit hyper-rectangle is Delaunay-triangulated (Qhull, ``:1019-1023``); a query
    point is located by rectangle (``state_to_rectangle``) + simplex inside the unit
    cell (``find_simplex`` on ``centered % unit_maxes``, ``:1103-1130``), weights are
    ``w1 = (x - origin) . H_s``, ``w0 = 1 - sum(w1)`` (``:1488-1491``), the value is
    ``sum_k w_k * param[simplex_k]`` (``:1494-1499``).  ``project`` clips the query to the
    limits first (``:1479-1485``).
    """

    def __init__(self, discretization, vertex_values=None, project=False):
        self.discretization = disc = discretization
        self.input_dim = disc.ndim
        self.project = project
        if disc.ndim == 1:
            corners = np.array([[0.0], [disc.unit_maxes[0]]])
            self.triangulation = _Delaunay1D(corners)
        else:
            corners = np.array(list(itertools.product(*np.diag(disc.unit_maxes))),
                               dtype=np.float64)
            self.triangulation = scipy.spatial.Delaunay(corners)
        # simplex corner indices in grid numbering (:1064-1088)
        tri_points = np.atleast_2d(self.triangulation.points)
        mapping = disc.state_to_index(tri_points + disc.offset)
        self.unit_simplices = mapping[np.asarray(self.triangulation.simplices)]
        self.nsimplex_unit = int(self.triangulation.nsimplex)
        self.nsimplex = self.nsimplex_unit * disc.nrectangles
        # hyperplanes (:1090-1101)
        self.hyperplanes = np.empty((self.nsimplex_unit, disc.ndim, disc.ndim))
        for i, simplex in enumerate(self.unit_simplices):
            pts = disc.index_to_state(simplex)
            self.hyperplanes[i] = np.linalg.inv(pts[1:] - pts[:1])
        self._parameters = None
        self.parameters = vertex_values

    @property
    def nindex(self):
        return self.discretization.nindex

    @property
    def parameters(self):
        return self._parameters

    @parameters.setter
    def parameters(self, values):
        self._parameters = (None if values is None else
                            np.asarray(values, dtype=np.float64).reshape(self.nindex, -1))

    @property
    def output_dim(self):
        return None if self._parameters is None else self._parameters.shape[1]

    def find_simplex(self, points):
        disc = self.discretization
        rect = disc.state_to_rectangle(points)
        unit = disc._center_states(points, clip=True) % disc.unit_maxes
        ids = np.atleast_1d(self.triangulation.find_simplex(unit))
        return ids + rect * self.nsimplex_unit

    def simplices(self, indices):
        unit = np.remainder(indices, self.nsimplex_unit)
        out = self.unit_simplices[unit].copy()
        rect = np.floor_divide(indices, self.nsimplex_unit)
        corner = self.discretization.rectangle_corner_index(rect)
        if out.ndim > 1:
            corner = corner[:, None]
        return out + corner

    def weights(self, points):
        """Barycentric weights [B, d+1] and corner indices [B, d+1]."""
        points = np.atleast_2d(np.asarray(points, dtype=np.float64))
        ids = self.find_simplex(points)
        corners = self.simplices(ids)
        origins = self.discretization.index_to_state(corners[:, 0])
        planes = self.hyperplanes[ids % self.nsimplex_unit]
        if self.project:
            lim = self.discretization.limits
            points = np.minimum(np.maximum(points, lim[:, 0]), lim[:, 1])
        offset = points - origins
        d = self.input_dim
        w = np.empty((points.shape[0], d + 1))
        for c in range(d):
            acc = offset[:, 0] * planes[:, 0, c]
            for k in range(1, d):
                acc = acc + offset[:, k] * planes[:, k, c]
            w[:, c + 1] = acc
        acc = w[:, 1]
        for c in range(2, d + 1):
            acc = acc + w[:, c]
        w[:, 0] = 1 - acc
        return w, corners

    def __call__(self, *inputs):
        w, corners = self.weights(hstack_inputs(inputs))
        vals = self._parameters[corners]                     # [B, d+1, out]
        acc = w[:, 0, None] * vals[:, 0, :]
        for k in range(1, w.shape[1]):
            acc = acc + w[:, k, None] * vals[:, k, :]
        return acc

    def gradient(self, points):
        """``functions.py:1260-1326`` (``_get_weights_gradient`` + ``gradient``): per point the
        weights ``[d, d+1]`` are ``[-sum_c H[k, c], H[k, 0], ..., H[k, d-1]]`` of the simplex the
        point falls in; ``grad[i, l, k] = sum_v weights[i, k, v] * values[corner_v, l]``, the
        output axis squeezed for one column.  Pinned by ``tests/test_functions.py:582-624``."""
        points = np.atleast_2d(np.asarray(points, dtype=np.float64))
        ids = self.find_simplex(points)
        corners = self.simplices(ids)
        planes = self.hyperplanes[ids % self.nsimplex_unit]          # [B, d, d]
        d = self.input_dim
        hs = planes[:, :, 0]
        for c in range(1, d):
            hs = hs + planes[:, :, c]
        vals = self._parameters[corners]                             # [B, d+1, out]
        res = (-hs)[:, None, :] * vals[:, 0, :, None]                # [B, out, d]
        for c in range(d):
            res = res + planes[:, None, :, c] * vals[:, c + 1, :, None]
        if res.shape[1] == 1:
            res = res[:, 0, :]
        return res

    def gradient_function(self):
        return lambda *inputs: self.gradient(hstack_inputs(inputs))


# --------------------------------------------------------------------------- plants / Lyapunov NN
class InvertedPendulum(object):
    """``examples/utilities.py:144-289``: normalised 10-sub-step explicit Euler."""

    def __init__(self, mass, length, friction=0.0, dt=1 / 80, normalization=None):
        self.mass, self.length, self.friction, self.dt = mass, length, friction, dt
        self.gravity = 9.81
        self.normalization = normalization
        if normalization is not None:
            self.normalization = [np.array(n, dtype=np.float64) for n in normalization]
            self.inv_norm = [n ** -1 for n in self.normalization]
        self.input_dim, self.output_dim = 3, 2

    @property
    def inertia(self):
        return self.mass * self.length ** 2

    def linearize(self):
        """``examples/utilities.py:207-240``."""
        g, l, b, inertia = self.gravity, self.length, self.friction, self.inertia
        A = np.array([[0, 1], [g / l, -b / inertia]], dtype=np.float64)
        B = np.array([[0], [1 / inertia]], dtype=np.float64)
        if self.normalization is not None:
            Tx, Tu = map(np.diag, self.normalization)
            Tx_inv, Tu_inv = map(np.diag, self.inv_norm)
            A = np.linalg.multi_dot((Tx_inv, A, Tx))
            B = np.linalg.multi_dot((Tx_inv, B, Tu))
        sysd = scipy.signal.StateSpace(A, B, np.eye(2), np.zeros((2, 1))).to_discrete(self.dt)
        return sysd.A, sysd.B

    def __call__(self, *inputs):
        sa = hstack_inputs(inputs)
        state, action = sa[:, :2].copy(), sa[:, 2:3].copy()
        if self.normalization is not None:
            state = state * self.normalization[0]
            action = action * self.normalization[1]
        dt = self.dt / 10
        g_l = self.gravity / self.length
        for _ in range(10):
            angle, omega = state[:, 0:1], state[:, 1:2]
            acc = g_l * np.sin(angle) + action / self.inertia
            if self.friction > 0:
                acc = acc - self.friction / self.inertia * omega
            state = state + dt * np.concatenate((omega, acc), axis=1)
        if self.normalization is not None:
            state = state * self.inv_norm[0]
        return state


class CartPole(object):
    """``examples/utilities.py:292-437``."""

    def __init__(self, pendulum_mass, cart_mass, length, rot_friction=0.0, dt=0.01,
                 normalization=None):
        self.pendulum_mass, self.cart_mass, self.length = pendulum_mass, cart_mass, length
        self.rot_friction, self.dt, self.gravity = rot_friction, dt, 9.81
        self.normalization = normalization
        if normalization is not None:
            self.normalization = [np.array(n, dtype=np.float64) for n in normalization]
            self.inv_norm = [n ** -1 for n in self.normalization]
        self.input_dim, self.output_dim = 5, 4

    def linearize(self):
        m, M, L, b, g = (self.pendulum_mass, self.cart_mass, self.length,
                         self.rot_friction, self.gravity)
        A = np.array([[0, 0, 1, 0], [0, 0, 0, 1],
                      [0, g * m / M, 0, -b / (M * L)],
                      [0, g * (m + M) / (L * M), 0, -b * (m + M) / (m * M * L ** 2)]],
                     dtype=np.float64)
        B = np.array([0, 0, 1 / M, 1 / (M * L)]).reshape((-1, 1))
        if self.normalization is not None:
            Tx, Tu = map(np.diag, self.normalization)
            Tx_inv, Tu_inv = map(np.diag, self.inv_norm)
            A = np.linalg.multi_dot((Tx_inv, A, Tx))
            B = np.linalg.multi_dot((Tx_inv, B, Tu))
        Ad, Bd, _, _, _ = scipy.signal.cont2discrete((A, B, 0, 0), self.dt, method="zoh")
        return Ad, Bd

    def ode(self, state, action):
        m, M, L, b, g = (self.pendulum_mass, self.cart_mass, self.length,
                         self.rot_friction, self.gravity)
        theta, v, omega = state[:, 1:2], state[:, 2:3], state[:, 3:4]
        det = L * (M + m * np.square(np.sin(theta)))
        v_dot = (action - m * L * np.square(omega) * np.sin(theta) - b * omega * np.cos(theta)
                 + 0.5 * m * g * L * np.sin(2 * theta)) * L / det
        omega_dot = (action * np.cos(theta) - 0.5 * m * L * np.square(omega) * np.sin(2 * theta)
                     - b * (m + M) * omega / (m * L) + (m + M) * g * np.sin(theta)) / det
        return np.concatenate((v, omega, v_dot, omega_dot), axis=1)

    def __call__(self, *inputs):
        sa = hstack_inputs(inputs)
        state, action = sa[:, :4].copy(), sa[:, 4:5].copy()
        if self.normalization is not None:
            state = state * self.normalization[0]
            action = action * self.normalization[1]
        dt = self.dt / 10
        for _ in range(10):
            state = state + dt * self.ode(state, action)
        if self.normalization is not None:
            state = state * self.inv_norm[0]
        return state


class LyapunovNetwork(object):
    """``examples/utilities.py:48-104``: ``net <- act(net . [W^T W + eps I; W2]^T)``, ``V = |net|^2``.

    Weights are passed explicitly (``weights[i] = (W_posdef, W_extra or None)``);
    the reference draws them from a Xavier initialiser.
    """

    def __init__(self, input_dim, layer_dims, activations, weights, eps=1e-6):
        self.input_dim, self.output_dims = input_dim, list(layer_dims)
        self.activations, self.weights, self.eps = activations, weights, eps
        self.output_dim = 1

    def kernels(self):
        out = []
        for i, (w0, w1) in enumerate(self.weights):
            din = self.input_dim if i == 0 else self.output_dims[i - 1]
            k = w0.T.dot(w0) + self.eps * np.eye(din)
            if w1 is not None:
                k = np.concatenate([k, w1], axis=0)
            out.append(k)
        return out

    def __call__(self, *inputs):
        net = hstack_inputs(inputs)
        for k, act in zip(self.kernels(), self.activations):
            net = act(_seq_dot(net, k))
        sq = np.square(net)
        acc = sq[:, 0]
        for c in range(1, sq.shape[1]):
            acc = acc + sq[:, c]
        return acc[:, None]


class NeuralNetwork(object):
    """``functions.py:1665-1729`` forward pass with explicit parameters: ``tf.layers.dense`` with
    bias in the hidden layers only, bias-free output layer, ``output_scale``."""

    def __init__(self, layers, nonlinearities, weights, biases, output_scale=1., use_bias=True):
        self.layers, self.nonlinearities = list(layers), list(nonlinearities)
        self.weights, self.biases = weights, biases
        self.output_scale, self.use_bias = output_scale, use_bias
        self.input_dim, self.output_dim = layers[0], layers[-1]

    def __call__(self, *inputs):
        net = hstack_inputs(inputs)
        for i, (w, act) in enumerate(zip(self.weights, self.nonlinearities)):
            net = _seq_dot(net, np.asarray(w).T)
            if self.use_bias and i + 1 < len(self.weights):
                net = net + self.biases[i]
            if act is not None:
                net = act(net)
        return net * self.output_scale


# --------------------------------------------------------------------------- Lyapunov
def stable_value_order(values):
    """``np.argsort(self.values)`` (``lyapunov.py:512``) with the tie-break pinned: stable."""
    return np.argsort(values, kind="stable")


def prefix_rule(values, ok, initial=None):
    """Sort-free closed form of the ``can_shrink=True`` sweep (SURVEY Q1).

    ``ok[i] = negative[i] | initial[i]``.  Returns (safe_set, first_fail_position).
    """
    order = stable_value_order(values)
    ok_sorted = ok[order]
    p = int(np.argmin(ok_sorted)) if not ok_sorted.all() else len(ok_sorted)
    safe = np.zeros(len(values), dtype=bool)
    safe[order[:p]] = True
    if initial is not None:
        safe[initial] = True
    return safe, p


class Lyapunov(object):
    """``lyapunov.py:142-606``.  The adaptive branch (``:445-487, 540-582``) is restated with two
    refined checks, see ``refined_negative``; its parity is UNPINNED: the reference has no test for
    it and its graph tests the wrong tensor (dead code at ``:469-476``)."""

    def __init__(self, discretization, lyapunov_function, dynamics, lipschitz_dynamics,
                 lipschitz_lyapunov, tau, policy, initial_set=None, adaptive=False):
        self.adaptive = adaptive
        self.discretization = discretization
        self.policy = policy
        self.safe_set = np.zeros(discretization.nindex, dtype=bool)
        self.initial_safe_set = initial_set
        if initial_set is not None:
            self.safe_set[initial_set] = True
        self.tau = tau
        self.dynamics = dynamics
        self.lyapunov_function = lyapunov_function
        self.values = None
        self.c_max = 0.0
        self._lipschitz_dynamics = lipschitz_dynamics
        self._lipschitz_lyapunov = lipschitz_lyapunov
        self.update_values()
        self._refinement = np.zeros(discretization.nindex, dtype=int)
        if initial_set is not None:
            self._refinement[initial_set] = 1

    def lipschitz_dynamics(self, states):
        f = self._lipschitz_dynamics
        return f(states) if callable(f) else f

    def lipschitz_lyapunov(self, states):
        f = self._lipschitz_lyapunov
        return f(states) if callable(f) else f

    def threshold(self, states, tau=None):
        """``lyapunov.py:265-288``: ``-lv * (1 + lf) * tau`` (1-norm of a vector-valued lv)."""
        if tau is None:
            tau = self.tau
        lv = self.lipschitz_lyapunov(states)
        if callable(self._lipschitz_lyapunov) and lv.shape[1] > 1:
            lv = _row_norm1(lv)
        lf = self.lipschitz_dynamics(states)
        return -lv * (1. + lf) * tau

    def is_safe(self, state):
        return self.safe_set[self.discretization.state_to_index(state)]

    def update_values(self):
        """``lyapunov.py:305-322``."""
        self.values = np.asarray(self.lyapunov_function(self.discretization.all_points)).squeeze()

    def v_decrease_confidence(self, states, next_states):
        """``lyapunov.py:324-354``: lv is evaluated at the predicted MEAN."""
        if isinstance(next_states, (tuple, list)):
            next_states, error_bounds = next_states
            lv = self.lipschitz_lyapunov(next_states)
            prod = lv * error_bounds
            if np.ndim(prod) == 2 and prod.shape[1] > 1:
                acc = prod[:, 0]
                for c in range(1, prod.shape[1]):
                    acc = acc + prod[:, c]
                bound = acc[:, None]
            else:
                bound = np.reshape(prod, (-1, 1))
        else:
            bound = 0.0
        v_decrease = self.lyapunov_function(next_states) - self.lyapunov_function(states)
        return v_decrease, bound

    def v_decrease_bound(self, states, next_states):
        """``lyapunov.py:356-376``."""
        v_dot, err = self.v_decrease_confidence(states, next_states)
        return v_dot + err

    def negative(self, states):
        """The graph node ``tf_negative`` (``lyapunov.py:436-441``): strict <, NaN -> False."""
        actions = self.policy(states)
        next_states = self.dynamics(states, actions)
        decrease = self.v_decrease_bound(states, next_states)
        threshold = self.threshold(states, self.tau)
        with np.errstate(invalid="ignore"):
            return np.squeeze(np.less(decrease, threshold), axis=1)

    def full_grid_negative(self, batch_size=None):
        """``negative`` on every grid point, batched like the reference but with the early
        exit disabled (the full-grid rate of SURVEY section 8d)."""
        batch_size = batch_size or config.gp_batch_size
        out = np.empty(self.discretization.nindex, dtype=bool)
        for i, (idx,) in batchify((np.arange(self.discretization.nindex),), batch_size):
            out[i:i + len(idx)] = self.negative(self.discretization.index_to_state(idx))
        return out

    def decrease_and_threshold(self, states, tau=None):
        actions = self.policy(states)
        next_states = self.dynamics(states, actions)
        decrease = self.v_decrease_bound(states, next_states)
        threshold = np.broadcast_to(self.threshold(states, tau), decrease.shape)
        return decrease, threshold

    def required_refinement(self, states, safety_factor=1.):
        """``lyapunov.py:445-455``: ``n_req = ceil(max(safety_factor * threshold / decrease, 0))``,
        NaN -> 0."""
        decrease, threshold = self.decrease_and_threshold(states)
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = safety_factor * threshold / decrease
        ratio = np.where(np.isnan(ratio), 0.0, ratio)
        return np.ceil(np.maximum(ratio, 0)).ravel()

    def refinement_mesh(self, center, n):
        """``lyapunov.py:459-472``: the ``n^d`` points ``center + 0.5 (1 - 1/n) unit_maxes
        linspace(-1, 1, n)`` (``indexing='ij'``; ``linspace(-1, 1, 1) = [-1]`` times 0 for n = 1)."""
        lengths = self.discretization.unit_maxes.reshape((-1, 1))
        spacing = np.linspace(-1., 1., n).reshape(1, -1)
        border = 0.5 * (1 - 1 / n) * lengths * np.tile(spacing, [len(lengths), 1])
        mesh = np.meshgrid(*border, indexing="ij")
        points = np.stack([col.reshape(-1) for col in mesh], axis=1)
        return points + np.asarray(center).reshape(1, -1)

    def refined_negative(self, states, refinement, mode="mesh", known_safe=None):
        """The per-state refined check of ``lyapunov.py:457-481``.

        ``mode="reference"``: as written -- ``refined_safety_check`` builds the mesh (``:461-472``)
        but compares the OUTER ``decrease`` tensor (all fed states) with ``threshold(center,
        tau / n)`` and reduces over everything (``:474-478``), so one failing state in the fed
        slice fails every state.
        ``mode="mesh"``: the evident intent -- the decrease condition is evaluated on the mesh
        points of the cell with ``tau / n``: ``all_p v_decrease_bound(p) < threshold(p, tau / n)``,
        and "cells that correspond to known safe states" (``:548-551``: ``negative`` or in the
        initial safe set, ``known_safe``) are not re-checked -- as written they are re-checked
        with n = 1, which fails every initial state whose own decrease is not negative and ends
        the prefix there.
        """
        out = np.zeros(len(states), dtype=bool)
        if mode == "reference":
            decrease, _ = self.decrease_and_threshold(states)
        for i, (center, n) in enumerate(zip(states, refinement)):
            n = int(n)
            if mode != "reference" and known_safe is not None and known_safe[i]:
                out[i] = True
                continue
            with np.errstate(invalid="ignore"):
                if mode == "reference":
                    thr = self.threshold(center.reshape(1, -1), self.tau / n)
                    out[i] = bool(np.all(np.less(decrease, thr)))
                else:
                    dec, thr = self.decrease_and_threshold(self.refinement_mesh(center, n),
                                                           self.tau / n)
                    out[i] = bool(np.all(np.less(dec, thr)))
        return out

    def update_safe_set(self, can_shrink=True, max_refinement=1, safety_factor=1.,
                        refinement_mode="mesh"):
        """The host loop of ``lyapunov.py:497-606`` as written (batches, early break,
        ``c_max`` index quirks), including the adaptive branch ``:540-582``."""
        safety_factor = np.maximum(safety_factor, 1.)
        if can_shrink:
            safe_set = np.zeros_like(self.safe_set, dtype=bool)
            refinement = np.zeros_like(self._refinement, dtype=int)
            if self.initial_safe_set is not None:
                safe_set[self.initial_safe_set] = True
                refinement[self.initial_safe_set] = 1
        else:
            safe_set = self.safe_set
            refinement = self._refinement

        value_order = stable_value_order(self.values)
        safe_set = safe_set[value_order]
        refinement = refinement[value_order]

        i = bound = 0
        for i, (indices, safe_batch, refine_batch) in batchify(
                (value_order, safe_set, refinement), config.gp_batch_size):
            states = self.discretization.index_to_state(indices)
            negative = self.negative(states)
            safe_batch |= negative
            refine_batch[negative] = 1
            bound = int(np.argmin(safe_batch))
            refine_bound = 0
            if bound > 0 or not safe_batch[0]:
                if self.adaptive and max_refinement > 1:                       # :540-577
                    refine_batch[bound:] = self.required_refinement(states[bound:], safety_factor)
                    initial = np.zeros(self.discretization.nindex, dtype=bool)
                    if self.initial_safe_set is not None:
                        initial[self.initial_safe_set] = True
                    idx_safe = np.logical_or(negative, initial[indices])
                    refine_batch[idx_safe] = 1
                    to_check = np.logical_and(refine_batch >= 1,
                                              refine_batch <= max_refinement)[bound:]
                    stop = len(to_check) if np.all(to_check) else int(np.argmin(to_check))
                    if stop > 0:
                        refined_safe = self.refined_negative(states[bound:bound + stop],
                                                             refine_batch[bound:bound + stop],
                                                             refinement_mode,
                                                             idx_safe[bound:bound + stop])
                        refine_bound = len(refined_safe) if np.all(refined_safe) \
                            else int(np.argmin(refined_safe))
                        safe_batch[bound:bound + refine_bound] = True
                    if stop < len(to_check) or refine_bound < stop:
                        safe_batch[bound + refine_bound:] = False
                        refine_batch[bound + refine_bound:] = 0
                        break
                else:
                    safe_batch[bound:] = False
                    refine_batch[bound:] = 0
                    break

        max_index = i + bound + refine_bound - 1
        self.c_max = self.values[value_order[max_index]]

        safe_nodes = value_order[safe_set]
        self.safe_set[:] = False
        self.safe_set[safe_nodes] = True
        self._refinement[value_order] = refinement
        if self.initial_safe_set is not None:
            self.safe_set[self.initial_safe_set] = True
            self._refinement[self.initial_safe_set] = 1


# --------------------------------------------------------------------------- policy iteration
class PolicyIteration(object):
    """``reinforcement_learning.py:26-279`` (``future_values``, ``value_iteration``,
    ``discrete_policy_optimization``)."""

    def __init__(self, policy, dynamics, reward_function, value_function, gamma=0.98):
        self.policy, self.dynamics = policy, dynamics
        self.reward_function, self.value_function = reward_function, value_function
        self.gamma = gamma
        self.state_space = self.value_function.discretization.all_points

    def future_values(self, states, policy=None, actions=None, lyapunov=None,
                      lagrange_multiplier=1.):
        """``r(x, u) + gamma V(mean f(x, u))`` [``- lambda (decrease - threshold)``]; ``:65-114``."""
        if actions is None:
            actions = (policy or self.policy)(states)
        next_states = self.dynamics(states, actions)
        rewards = self.reward_function(states, actions)
        var = None
        if isinstance(next_states, tuple):
            next_states, var = next_states
        expected = self.value_function(next_states)
        updated = rewards + self.gamma * expected
        if lyapunov is not None:
            decrease = lyapunov.v_decrease_bound(states, (next_states, var))
            updated = updated - lagrange_multiplier * (decrease - lyapunov.threshold(states))
        return updated

    def value_iteration(self):
        """One synchronous (Jacobi) sweep; ``:135-140``. Returns the new vertex values."""
        new = self.future_values(self.state_space)
        self.value_function.parameters = new
        return new

    def discrete_policy_optimization(self, action_space, constraint=None):
        """``:213-279``: argmax over a discrete action set, first maximum wins."""
        states = self.policy.discretization.all_points
        action_space = np.asarray(action_space, dtype=np.float64)
        n_states, (n_opt, n_act) = states.shape[0], action_space.shape
        values = np.empty((n_states, n_opt))
        for i, action in enumerate(action_space):
            arr = np.broadcast_to(action, (n_states, n_act))
            values[:, i] = self.future_values(states, actions=arr)[:, 0]
            if constraint is not None:
                values[constraint(arr) < 0, i] = -np.inf
        best = action_space[np.argmax(values, axis=1)]
        self.policy.parameters = best
        return best


# --------------------------------------------------------------------------- safe sampling
def smallest_boundary_value(fun, discretization):
    """``lyapunov.py:22-56``: the smallest value of ``fun`` over the faces of the grid (per axis:
    that axis at its two end points, all others at every grid coordinate).  Pinned by
    ``tests/test_lyapunov.py:77-84``."""
    min_value = np.inf
    for i in range(discretization.ndim):
        tmp = list(discretization.discrete_points)
        tmp[i] = discretization.discrete_points[i][[0, -1]]
        columns = (x.ravel() for x in np.meshgrid(*tmp, indexing="ij"))
        min_value = min(min_value, float(np.min(fun(np.column_stack(list(columns))))))
    return min_value


def unique_rows(array):
    """``utilities.py:496-516``."""
    array = np.ascontiguousarray(array)
    dtype = np.dtype((np.void, array.dtype.itemsize * array.shape[1]))
    _, idx = np.unique(array.view(dtype=dtype), return_index=True)
    return array[idx]


def perturb_actions(states, actions, perturbations, limits=None):
    """``lyapunov.py:609-651``."""
    num_states, state_dim = states.shape
    states_new = np.repeat(states, len(perturbations), axis=0)
    actions_new = (np.repeat(actions, len(perturbations), axis=0)
                   + np.tile(perturbations, (num_states, 1)))
    state_actions = np.column_stack((states_new, actions_new))
    if limits is not None:
        limits = np.asarray(limits)
        acts = state_actions[:, state_dim:]
        np.clip(acts, limits[:, 0], limits[:, 1], out=acts)
        state_actions = unique_rows(state_actions)
    return state_actions


def get_safe_sample(lyapunov, perturbations, limits=None, positive=False, safe_states=None):
    """``lyapunov.py:657-797`` with the random sub-sampling factored out (pass ``safe_states``
    to evaluate a fixed candidate set).  Returns (state_action [1, n+m], bound)."""
    disc = lyapunov.discretization
    if safe_states is None:
        safe_states = disc.index_to_state(np.where(lyapunov.safe_set)[0])
    safe_actions = lyapunov.policy(safe_states)
    state_actions = perturb_actions(safe_states, safe_actions, perturbations, limits)
    mean, std = lyapunov.dynamics(state_actions)
    bound = np.sum(std, axis=1, keepdims=True)
    lv = lyapunov.lipschitz_lyapunov(mean)
    error = np.sum(lv * std, axis=1, keepdims=True)
    future = lyapunov.lyapunov_function(mean) + error
    maps_inside = (future < lyapunov.c_max)[:, 0]
    if not positive:
        maps_inside &= lyapunov.safe_set[disc.state_to_index(mean)]
    bound_safe = bound[maps_inside]
    if len(bound_safe) == 0:
        state_actions = perturb_actions(safe_states, safe_actions, np.array([[0.]]), limits)
        _, std = lyapunov.dynamics(state_actions)
        bound = np.sum(std, axis=1, keepdims=True)
        max_id = int(np.argmax(bound))
        return state_actions[[max_id]], bound[max_id].squeeze()
    max_id = int(np.argmax(bound_safe))
    return state_actions[maps_inside, :][[max_id]], bound_safe[max_id].squeeze()
