"""Stand-in for the slice of gpflow==0.4.0 that the reference's safe_learning package touches
(fixture generation only; see ../tensorflow/__init__.py).

``kernels.*`` (RBF, Matern, Linear, Constant, White, Add, Prod) and ``gpr.GPR.build_predict`` restate gpflow 0.4.0's published arithmetic
(third-party code that is not part of the reference); everything the reference itself
implements -- ``GPRCached`` caching and prediction, ``GaussianProcess`` beta scaling,
``FunctionStack`` -- runs from the reference's own source on top of this.
"""
import contextlib

import numpy as np
import tensorflow as tf

__version__ = "0.4.0-shim"


class _DataHolder(tf.Tensor):
    """param.DataHolder: an array that behaves as a tensor inside tf_mode and exposes .value."""

    def __init__(self, array, on_shape_change="raise"):
        tf.Tensor.__init__(self, None)
        self.value = np.array(array, dtype=np.float64)

    def _value(self, feed, cache):
        return self.value

    @property
    def shape(self):
        return self.value.shape


class _Param(object):
    DataHolder = _DataHolder

    @staticmethod
    def AutoFlow(*tf_arg_tuples):
        def wrap(method):
            def runner(self, *args):
                out = method(self, *args)
                if isinstance(out, (list, tuple)):
                    return [o.eval() if isinstance(o, tf.Tensor) else o for o in out]
                return out.eval()
            return runner
        return wrap


param = _Param()


class _MeanFunctions(object):
    class Zero(object):
        def __call__(self, X):
            return tf.Tensor(lambda f, c: np.zeros((tf._val(X, f, c).shape[0], 1)))


mean_functions = _MeanFunctions()


class _Kern(object):
    """gpflow 0.4.0 kernels.Kern: `active_dims` column selection (default: the first `input_dim`
    columns), `+` -> Add, `*` -> Prod.  K / Kdiag return lazy tensors of the numpy arithmetic."""

    def __init__(self, input_dim, active_dims=None):
        self.input_dim = int(input_dim)
        if active_dims is None:
            active_dims = slice(self.input_dim)
        self.active_dims = active_dims

    def _slice(self, x, x2):
        x = x[:, self.active_dims]
        return x, (None if x2 is None else x2[:, self.active_dims])

    def K(self, X, X2=None, presliced=False):
        def run(f, c):
            x = tf._val(X, f, c)
            x2 = None if X2 is None else tf._val(X2, f, c)
            return self._K(x, x2)
        return tf.Tensor(run)

    def Kdiag(self, X, presliced=False):
        return tf.Tensor(lambda f, c: self._Kdiag(tf._val(X, f, c)))

    def __add__(self, other):
        return _Add([self, other])

    def __mul__(self, other):
        return _Prod([self, other])


class _Combination(_Kern):
    def __init__(self, kern_list):
        self.kern_list = list(kern_list)


class _Add(_Combination):
    def _K(self, x, x2):
        out = self.kern_list[0]._K(x, x2)
        for k in self.kern_list[1:]:
            out = out + k._K(x, x2)
        return out

    def _Kdiag(self, x):
        out = self.kern_list[0]._Kdiag(x)
        for k in self.kern_list[1:]:
            out = out + k._Kdiag(x)
        return out


class _Prod(_Combination):
    def _K(self, x, x2):
        out = self.kern_list[0]._K(x, x2)
        for k in self.kern_list[1:]:
            out = out * k._K(x, x2)
        return out

    def _Kdiag(self, x):
        out = self.kern_list[0]._Kdiag(x)
        for k in self.kern_list[1:]:
            out = out * k._Kdiag(x)
        return out


class _Stationary(_Kern):
    """gpflow 0.4.0 Stationary: square_dist by the |x|^2 + |x'|^2 - 2 x.x' expansion on
    lengthscale-divided inputs; euclid_dist = sqrt(square_dist + 1e-12); Kdiag = variance."""

    def __init__(self, input_dim, variance=1.0, lengthscales=None, active_dims=None, ARD=False):
        _Kern.__init__(self, input_dim, active_dims)
        self.variance = float(variance)
        ls = 1.0 if lengthscales is None else lengthscales
        self.lengthscales = np.broadcast_to(np.asarray(ls, dtype=np.float64),
                                            (self.input_dim,)).copy()

    def square_dist(self, X, X2):
        X, X2 = self._slice(X, X2)
        X = X / self.lengthscales
        Xs = np.sum(np.square(X), axis=1)
        if X2 is None:
            return -2 * X.dot(X.T) + Xs[:, None] + Xs[None, :]
        X2 = X2 / self.lengthscales
        X2s = np.sum(np.square(X2), axis=1)
        return -2 * X.dot(X2.T) + Xs[:, None] + X2s[None, :]

    def euclid_dist(self, X, X2):
        return np.sqrt(self.square_dist(X, X2) + 1e-12)

    def _Kdiag(self, x):
        return np.full(x.shape[0], self.variance)


class _Kernels(object):
    class RBF(_Stationary):
        def _K(self, x, x2):
            return self.variance * np.exp(-self.square_dist(x, x2) / 2)

    class Matern12(_Stationary):
        def _K(self, x, x2):
            return self.variance * np.exp(-self.euclid_dist(x, x2))

    class Matern32(_Stationary):
        def _K(self, x, x2):
            r = self.euclid_dist(x, x2)
            return self.variance * (1. + np.sqrt(3.) * r) * np.exp(-np.sqrt(3.) * r)

    class Matern52(_Stationary):
        def _K(self, x, x2):
            r = self.euclid_dist(x, x2)
            return self.variance * (1.0 + np.sqrt(5.) * r + 5. / 3. * np.square(r)) \
                * np.exp(-np.sqrt(5.) * r)

    class Linear(_Kern):
        def __init__(self, input_dim, variance=1.0, active_dims=None, ARD=False):
            _Kern.__init__(self, input_dim, active_dims)
            self.variance = np.asarray(variance, dtype=np.float64) * \
                (np.ones(self.input_dim) if ARD else 1.0)

        def _K(self, x, x2):
            x, x2 = self._slice(x, x2)
            return (x * self.variance).dot((x if x2 is None else x2).T)

        def _Kdiag(self, x):
            x, _ = self._slice(x, None)
            return np.sum(np.square(x) * self.variance, 1)

    class Constant(_Kern):
        def __init__(self, input_dim, variance=1.0, active_dims=None):
            _Kern.__init__(self, input_dim, active_dims)
            self.variance = float(variance)

        def _K(self, x, x2):
            return np.full((x.shape[0], (x if x2 is None else x2).shape[0]), self.variance)

        def _Kdiag(self, x):
            return np.full(x.shape[0], self.variance)

    class White(_Kern):
        def __init__(self, input_dim, variance=1.0, active_dims=None):
            _Kern.__init__(self, input_dim, active_dims)
            self.variance = float(variance)

        def _K(self, x, x2):
            if x2 is None:
                return self.variance * np.eye(x.shape[0])
            return np.zeros((x.shape[0], x2.shape[0]))

        def _Kdiag(self, x):
            return np.full(x.shape[0], self.variance)

    Bias = Constant
    Add, Prod = _Add, _Prod


kernels = _Kernels()


class _Likelihood(object):
    def __init__(self):
        self.variance = 1.0        # gpflow default Gaussian likelihood variance


class _GPR(object):
    """gpflow 0.4.0 gpr.GPR: holds X, Y as DataHolders, kernel, mean function, likelihood."""

    def __init__(self, X, Y, kern, mean_function=None, name="name"):
        object.__setattr__(self, "X", _DataHolder(X))
        object.__setattr__(self, "Y", _DataHolder(Y))
        self.kern = kern
        self.mean_function = mean_function or mean_functions.Zero()
        self.likelihood = _Likelihood()
        self.name = name

    def __setattr__(self, key, value):
        current = self.__dict__.get(key)
        if isinstance(current, _DataHolder) and not isinstance(value, _DataHolder):
            current.value = np.array(value, dtype=np.float64)
        else:
            object.__setattr__(self, key, value)

    @contextlib.contextmanager
    def tf_mode(self):
        yield self

    def make_tf_array(self, x):
        return 0

    def get_feed_dict_keys(self):
        return {}

    def update_feed_dict(self, keys, feed_dict):
        pass

    def get_free_state(self):
        return np.zeros(1)

    def build_predict(self, Xnew, full_cov=False):
        """gpflow 0.4.0 GPR.build_predict (uncached): factorises K on every call."""
        Kx = self.kern.K(self.X, Xnew)
        K = self.kern.K(self.X) + tf.eye(tf.shape(self.X)[0], dtype=tf.float64) * self.likelihood.variance
        L = tf.cholesky(K)
        A = tf.matrix_triangular_solve(L, Kx, lower=True)
        V = tf.matrix_triangular_solve(L, self.Y - self.mean_function(self.X))
        fmean = tf.matmul(A, V, transpose_a=True) + self.mean_function(Xnew)
        fvar = self.kern.Kdiag(Xnew) - tf.reduce_sum(tf.square(A), 0)
        fvar = tf.tile(tf.reshape(fvar, (-1, 1)), [1, tf.shape(self.Y)[1]])
        return fmean, fvar

    def predict_f(self, Xnew):
        mean, var = self.build_predict(np.asarray(Xnew, dtype=np.float64))
        return mean.eval(), var.eval()


class _GprModule(object):
    GPR = _GPR


gpr = _GprModule()


class _Models(object):
    GPModel = _GPR


models = _Models()
