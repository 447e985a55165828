"""The few cvxpy names ``reinforcement_learning.py:142-178`` uses, on scipy's HiGHS ``linprog``:
affine expressions  A v + b  in one vector variable, ``<=`` constraints and a linear objective."""
import numpy as np
import scipy.optimize
import scipy.sparse as sp

OPTIMAL, INFEASIBLE, UNBOUNDED = "optimal", "infeasible", "unbounded"


class _Affine(object):
    """A v + b for the problem's one variable v (A sparse [m, n] or None for 0, b [m])."""
    __array_priority__ = 1000

    def __init__(self, A, b):
        self.A, self.b = A, np.asarray(b, dtype=np.float64).reshape(-1)

    def __add__(self, other):
        if isinstance(other, _Affine):
            A = self.A if other.A is None else (other.A if self.A is None else self.A + other.A)
            return _Affine(A, self.b + other.b)
        return _Affine(self.A, self.b + np.asarray(other, dtype=np.float64).reshape(-1))

    __radd__ = __add__

    def __rmul__(self, scalar):
        return _Affine(None if self.A is None else self.A * float(scalar), self.b * float(scalar))

    def __le__(self, other):
        return (self + (-1.0) * (other if isinstance(other, _Affine) else _Affine(None, other)))


class Variable(_Affine):
    def __init__(self, shape):
        self.shape = tuple(np.atleast_1d(shape))
        n = int(np.prod(self.shape))
        super().__init__(sp.identity(n, format="csr"), np.zeros(n))
        self.value = None


class Constant(object):
    __array_priority__ = 1000

    def __init__(self, value):
        self.value = sp.csr_matrix(value)

    def __mul__(self, expr):
        return _Affine(self.value @ expr.A, self.value @ expr.b)

    def __rmul__(self, scalar):
        return Constant(self.value * float(scalar))


def sum(expr):                                              # noqa: A001 (cvxpy's name)
    return _Affine(sp.csr_matrix(np.ones((1, expr.A.shape[0]))) @ expr.A, [np.sum(expr.b)])


class Maximize(object):
    def __init__(self, expr):
        self.expr = expr


class Problem(object):
    def __init__(self, objective, constraints):
        self.objective, self.constraints = objective, constraints
        self.status = None

    def solve(self, **options):
        A = sp.vstack([c.A for c in self.constraints]).tocsc()
        b = -np.concatenate([c.b for c in self.constraints])
        cost = -self.objective.expr.A.toarray().ravel()
        res = scipy.optimize.linprog(cost, A_ub=A, b_ub=b, bounds=(None, None), method="highs")
        self.status = {0: OPTIMAL, 2: INFEASIBLE, 3: UNBOUNDED}.get(res.status, "failed")
        self._result = res
        for var in _VARIABLES:
            var.value = None if res.x is None else res.x.reshape(var.shape)
        return None if res.x is None else -res.fun


_VARIABLES = []
_variable_init = Variable.__init__


def _tracked_init(self, shape):
    _variable_init(self, shape)
    del _VARIABLES[:]
    _VARIABLES.append(self)


Variable.__init__ = _tracked_init
