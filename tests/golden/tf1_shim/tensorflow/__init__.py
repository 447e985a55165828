"""numpy-backed stand-in for the slice of the TensorFlow 1.x API that
the reference's safe_learning package uses on the region-of-attraction path.

PURPOSE: fixture generation only (tests/golden/make_golden.py).  TF 1.x cannot be installed
in the build container (Python 3.12, no network); this shim lets the UNMODIFIED reference
modules be imported and executed so that their own Python logic -- graph construction order,
the update_safe_set batch loop, c_max indexing, GPRCached algebra, Triangulation lookup --
produces the golden vectors the oracle is pinned against.  Tensors are lazy closures evaluated
with numpy at ``eval``/``Session.run`` time; linear algebra goes to numpy/scipy (LAPACK), as
TF 1.x goes to Eigen.  Nothing here is shipped or imported by the product.
"""
import contextlib

import numpy as np
import scipy.linalg

class _DType(object):
    def __init__(self, np_dtype):
        self.as_numpy_dtype = np_dtype


float64 = _DType(np.float64)
int64 = _DType(np.int64)
int32 = _DType(np.int32)
bool = _DType(np.bool_)       # noqa: A001


def _np_dtype(dt):
    return getattr(dt, "as_numpy_dtype", dt)


# --------------------------------------------------------------------------- graph / scopes
class Graph(object):
    def __init__(self):
        self._names = {}

    def unique_name(self, name):
        n = self._names.get(name, 0)
        self._names[name] = n + 1
        return name if n == 0 else "%s_%d" % (name, n)


_GRAPH = Graph()
_SCOPES = []
_VARIABLES = []
_SESSIONS = []


def get_default_graph():
    return _GRAPH


def reset_default_graph():
    global _GRAPH
    _GRAPH = Graph()
    del _VARIABLES[:]


class _Scope(object):
    def __init__(self, name):
        self.original_name_scope = name
        self.name = name


@contextlib.contextmanager
def variable_scope(name_or_scope, *args, **kwargs):
    if isinstance(name_or_scope, _Scope):
        scope = name_or_scope
    elif isinstance(name_or_scope, str) and name_or_scope.endswith("/"):
        scope = _Scope(name_or_scope)          # re-entering an original_name_scope
    else:
        prefix = _SCOPES[-1].original_name_scope if _SCOPES else ""
        scope = _Scope(prefix + _GRAPH.unique_name(prefix + str(name_or_scope))[len(prefix):] + "/")
    _SCOPES.append(scope)
    try:
        yield scope
    finally:
        _SCOPES.pop()


@contextlib.contextmanager
def name_scope(name, *args, **kwargs):
    yield name


def make_template(name, func, create_scope_now_=False, **kwargs):
    return func


class GraphKeys(object):
    TRAINABLE_VARIABLES = "trainable_variables"


def get_collection(key, scope=None):
    return [v for v in _VARIABLES if scope is None or v._scope.startswith(scope)]


# --------------------------------------------------------------------------- tensors
class Tensor(object):
    def __init__(self, fn, name=None):
        self._fn = fn
        self.name = name

    # evaluation --------------------------------------------------------------------
    def _value(self, feed, cache):
        key = id(self)
        if key not in cache:
            cache[key] = np.asarray(feed[self]) if self in feed else self._fn(feed, cache)
        return cache[key]

    def eval(self, feed_dict=None, session=None):
        return self._value(dict(feed_dict or {}), {})

    @property
    def shape(self):
        return tuple(self.eval().shape)

    def get_shape(self):
        return self.shape

    __hash__ = object.__hash__
    __array_ufunc__ = None        # ndarray <op> Tensor must defer to Tensor.__r<op>__

    # operators ---------------------------------------------------------------------
    def __add__(self, o): return _binary(np.add, self, o)
    def __radd__(self, o): return _binary(np.add, o, self)
    def __sub__(self, o): return _binary(np.subtract, self, o)
    def __rsub__(self, o): return _binary(np.subtract, o, self)
    def __mul__(self, o): return _binary(np.multiply, self, o)
    def __rmul__(self, o): return _binary(np.multiply, o, self)
    def __truediv__(self, o): return _binary(np.divide, self, o)
    def __rtruediv__(self, o): return _binary(np.divide, o, self)
    def __neg__(self): return _unary(np.negative, self)
    def __lt__(self, o): return _binary(np.less, self, o)
    def __gt__(self, o): return _binary(np.greater, self, o)
    def __eq__(self, o): return self is o
    def __ne__(self, o): return self is not o

    def __getitem__(self, item):
        return Tensor(lambda f, c: self._value(f, c)[item])


def _val(x, feed, cache):
    if isinstance(x, Tensor):
        return x._value(feed, cache)
    if isinstance(x, (list, tuple)) and any(isinstance(e, Tensor) for e in x):
        return np.asarray([_val(e, feed, cache) for e in x])
    return np.asarray(x)


def _unary(op, a, **kw):
    return Tensor(lambda f, c: op(_val(a, f, c), **kw))


def _binary(op, a, b):
    with np.errstate(invalid="ignore", divide="ignore"):
        return Tensor(lambda f, c: op(_val(a, f, c), _val(b, f, c)))


class Variable(Tensor):
    def __init__(self, initial_value, name=None, dtype=None, **kwargs):
        Tensor.__init__(self, None, name)
        if isinstance(initial_value, Tensor):
            initial_value = initial_value.eval()
        self.value = np.array(initial_value, dtype=_np_dtype(dtype) if dtype else None)
        self._scope = _SCOPES[-1].original_name_scope if _SCOPES else ""
        _VARIABLES.append(self)

    def _value(self, feed, cache):
        return np.asarray(feed[self]) if self in feed else self.value


def placeholder(dtype, shape=None, name=None):
    dummy_shape = tuple(2 if s is None else int(s) for s in (shape if shape is not None else ()))
    dt = _np_dtype(dtype)
    return Tensor(lambda f, c: np.zeros(dummy_shape, dtype=dt), name)


def constant(value, dtype=None, shape=None, name=None):
    arr = np.array(value, dtype=_np_dtype(dtype) if dtype else None)
    return Tensor(lambda f, c: arr, name)


def convert_to_tensor(value, dtype=None, name=None):
    return value if isinstance(value, Tensor) else constant(value, dtype)


def assign(ref, value, validate_shape=None, name=None):
    def run(f, c):
        ref.value = np.array(_val(value, f, c))
        return ref.value
    return Tensor(run, name)


def variables_initializer(var_list, name=None):
    return Tensor(lambda f, c: None)


def control_dependencies(inputs):
    return contextlib.nullcontext()


def stop_gradient(x, name=None):
    return x


# --------------------------------------------------------------------------- sessions
class Session(object):
    def __init__(self, *args, **kwargs):
        pass

    def __enter__(self):
        _SESSIONS.append(self)
        return self

    def __exit__(self, *exc):
        _SESSIONS.pop()

    def close(self):
        if self in _SESSIONS:
            _SESSIONS.remove(self)

    def run(self, fetches, feed_dict=None):
        feed, cache = dict(feed_dict or {}), {}
        if isinstance(fetches, (list, tuple)):
            return [t._value(feed, cache) if isinstance(t, Tensor) else t for t in fetches]
        return fetches._value(feed, cache)


class InteractiveSession(Session):
    def __init__(self, *args, **kwargs):
        _SESSIONS.append(self)


def ConfigProto(*args, **kwargs):
    return None


def get_default_session():
    return _SESSIONS[-1] if _SESSIONS else None


# --------------------------------------------------------------------------- ops
def matmul(a, b, transpose_a=False, transpose_b=False, name=None):
    def run(f, c):
        x, y = _val(a, f, c), _val(b, f, c)
        return (x.T if transpose_a else x).dot(y.T if transpose_b else y)
    return Tensor(run, name)


def concat(values, axis, name=None):
    return Tensor(lambda f, c: np.concatenate([_val(v, f, c) for v in values], axis=axis), name)


def stack(values, axis=0, name=None):
    if isinstance(values, np.ndarray):
        return constant(values)
    return Tensor(lambda f, c: np.stack([_val(v, f, c) for v in values], axis=axis), name)


def unstack(value, axis=0, name=None):
    n = value.shape[axis]
    return [Tensor(lambda f, c, i=i: np.take(_val(value, f, c), i, axis=axis)) for i in range(n)]


def split(value, num_or_size_splits, axis=0, name=None):
    if isinstance(num_or_size_splits, int):
        n = num_or_size_splits
        return [Tensor(lambda f, c, i=i: np.split(_val(value, f, c), n, axis=axis)[i])
                for i in range(n)]
    cuts = np.cumsum(num_or_size_splits)[:-1]
    return [Tensor(lambda f, c, i=i: np.split(_val(value, f, c), cuts, axis=axis)[i])
            for i in range(len(num_or_size_splits))]


def _reduce(op):
    def fn(x, axis=None, keepdims=False, keep_dims=None, name=None):
        kd = keepdims if keep_dims is None else keep_dims
        return Tensor(lambda f, c: op(_val(x, f, c), axis=axis, keepdims=kd), name)
    return fn


reduce_sum = _reduce(np.sum)
reduce_max = _reduce(np.max)
reduce_min = _reduce(np.min)
reduce_all = _reduce(np.all)


def norm(x, ord="euclidean", axis=None, keepdims=False, keep_dims=None, name=None):
    kd = keepdims if keep_dims is None else keep_dims
    order = 2 if ord == "euclidean" else ord
    return Tensor(lambda f, c: np.linalg.norm(_val(x, f, c), ord=order, axis=axis, keepdims=kd))


def square(x, name=None): return _unary(np.square, x)
def abs(x, name=None): return _unary(np.abs, x)       # noqa: A001
def sin(x, name=None): return _unary(np.sin, x)
def cos(x, name=None): return _unary(np.cos, x)
def exp(x, name=None): return _unary(np.exp, x)
def tanh(x, name=None): return _unary(np.tanh, x)
def ceil(x, name=None): return _unary(np.ceil, x)
def is_nan(x, name=None): return _unary(np.isnan, x)
def zeros_like(x, dtype=None, name=None): return _unary(np.zeros_like, x)


def sqrt(x, name=None):
    def run(f, c):
        with np.errstate(invalid="ignore"):
            return np.sqrt(_val(x, f, c))
    return Tensor(run, name)


def maximum(a, b, name=None): return _binary(np.maximum, a, b)
def minimum(a, b, name=None): return _binary(np.minimum, a, b)
def multiply(a, b, name=None): return _binary(np.multiply, a, b)
def less(a, b, name=None): return _binary(np.less, a, b)


def clip_by_value(x, lo, hi, name=None):
    return Tensor(lambda f, c: np.clip(_val(x, f, c), _val(lo, f, c), _val(hi, f, c)))


def where(cond, x, y, name=None):
    return Tensor(lambda f, c: np.where(_val(cond, f, c), _val(x, f, c), _val(y, f, c)))


def squeeze(x, axis=None, name=None):
    return Tensor(lambda f, c: np.squeeze(_val(x, f, c), axis=axis), name)


def expand_dims(x, axis, name=None):
    return Tensor(lambda f, c: np.expand_dims(_val(x, f, c), axis), name)


def reshape(x, shape, name=None):
    return Tensor(lambda f, c: np.reshape(_val(x, f, c), tuple(int(s) for s in
                                                               np.atleast_1d(_val(shape, f, c)))))


def tile(x, multiples, name=None):
    return Tensor(lambda f, c: np.tile(_val(x, f, c), tuple(int(m) for m in
                                                            np.atleast_1d(_val(multiples, f, c)))))


def shape(x, name=None):      # noqa: F811
    return Tensor(lambda f, c: np.array(_val(x, f, c).shape, dtype=np.int64))


def cast(x, dtype, name=None):
    return Tensor(lambda f, c: _val(x, f, c).astype(_np_dtype(dtype)))


def eye(n, dtype=None, name=None):
    return Tensor(lambda f, c: np.eye(int(_val(n, f, c)), dtype=_np_dtype(dtype) if dtype else float))


def gather(params, indices, validate_indices=None, name=None):
    return Tensor(lambda f, c: _val(params, f, c)[_val(indices, f, c)])


def cholesky(x, name=None):
    return Tensor(lambda f, c: np.linalg.cholesky(_val(x, f, c)), name)


def matrix_triangular_solve(matrix, rhs, lower=True, adjoint=False, name=None):
    return Tensor(lambda f, c: scipy.linalg.solve_triangular(
        _val(matrix, f, c), _val(rhs, f, c), lower=lower, trans="T" if adjoint else "N"), name)


def matrix_diag_part(x, name=None): return _unary(np.diagonal, x)


def py_func(func, inp, Tout, stateful=True, name=None):
    state = {}

    def run_all(f, c):
        key = ("py_func", id(state))
        if key not in c:
            out = func(*[_val(i, f, c) for i in inp])
            c[key] = out if isinstance(out, (list, tuple)) else [out]
        return c[key]
    if isinstance(Tout, (list, tuple)):
        return [Tensor(lambda f, c, i=i: np.asarray(run_all(f, c)[i])) for i in range(len(Tout))]
    return Tensor(lambda f, c: np.asarray(run_all(f, c)[0]))


from . import contrib  # noqa: E402,F401


class _LayersStub(object):
    @staticmethod
    def dense(*args, **kwargs):
        raise NotImplementedError("tf.layers.dense is outside the shimmed path")


layers = _LayersStub()
