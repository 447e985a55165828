"""CPU tests of multi-output GPs (a ``GPRCached`` whose ``Y`` has k columns): the shape checks of the model,
the stack and ``FunctionStack.add_data_point``; the host checks of ``slb_gp_lml_grad_cols``; and the numpy
reference of the joint log marginal likelihood (tests/gp_lml_cols_reference.py) against the sum of its
one-column form and against central differences.  No call here launches a kernel."""
import numpy as np
import pytest
from numpy.testing import assert_allclose

import gp_lml_cols_reference as RC
import gp_lml_reference as R


@pytest.fixture(scope="module")
def sl():
    import __graft_entry__
    __graft_entry__.build()
    import safe_learning_b200 as sl
    return sl


def _gp(sl, M, k, mean_rows=None, din=3):
    rng = np.random.default_rng(M + k)
    X = rng.uniform(-1, 1, (M, din))
    Y = rng.standard_normal((M, k))
    mean = None if mean_rows is None else sl.LinearSystem(rng.uniform(-1, 1, (mean_rows, din)))
    return sl.GPRCached(X, Y, sl.RBF(din, lengthscales=[1.0] * din), mean_function=mean)


# ---------------------------------------------------------------- shapes
@pytest.mark.parametrize("k", [1, 2, 3, 6])
def test_k_columns_and_the_empty_data_set(sl, k):
    gp = _gp(sl, 12, k, mean_rows=k)
    assert gp.output_dim == k and gp.Y.shape == (12, k)
    assert sl.GaussianProcess(gp).output_dim == k
    empty = sl.GPRCached(np.empty((0, 3)), np.empty((0, k)), sl.RBF(3))
    assert empty.Y.shape == (0, k) and empty.output_dim == k


def test_rows_mismatch_raises(sl):
    X = np.zeros((5, 3))
    with pytest.raises(sl.DimensionError, match="one target row per input row"):
        sl.GPRCached(X, np.zeros((4, 2)), sl.RBF(3))
    with pytest.raises(sl.DimensionError, match="one target row per input row"):
        sl.GPRCached(X, np.zeros(5), sl.RBF(3))            # a 1-D y is one row, not five
    with pytest.raises(sl.DimensionError, match="one target row per input row"):
        sl.GPRCached(np.empty((0, 3)), np.zeros((1, 2)), sl.RBF(3))


def test_more_than_six_outputs_raise(sl):
    with pytest.raises(sl.DimensionError, match="1..6 outputs"):
        _gp(sl, 5, 7)
    gps = [sl.GaussianProcess(_gp(sl, 5, 4)), sl.GaussianProcess(_gp(sl, 5, 3))]
    stack = sl.FunctionStack(gps)
    assert stack.output_dim == 7
    with pytest.raises(sl.DimensionError, match="at most 6 stacked GP outputs, got 7"):
        stack.gp_stack()


@pytest.mark.parametrize("k, rows", [(1, 2), (2, 1), (3, 2), (2, 3)])
def test_mean_function_rows_must_match(sl, k, rows):
    with pytest.raises(sl.DimensionError, match="prior mean has %d rows for %d target columns" % (rows, k)):
        _gp(sl, 6, k, mean_rows=rows)


def test_mean_function_kind(sl):
    with pytest.raises(NotImplementedError):
        sl.GPRCached(np.zeros((2, 3)), np.zeros((2, 2)), sl.RBF(3), mean_function=sl.QuadraticFunction(np.eye(3)))


def test_add_data_point_split_checks_columns(sl):
    stack = sl.FunctionStack([sl.GaussianProcess(_gp(sl, 5, 2)), sl.GaussianProcess(_gp(sl, 5, 1))])
    with pytest.raises(sl.DimensionError, match="y has 2 columns, the stack has 3 outputs"):
        stack.add_data_point(np.zeros((1, 3)), np.zeros((1, 2)))


# ---------------------------------------------------------------- slb_gp_lml_grad_cols host checks
def _kernel(nat, din=3):
    k = nat.SlbKernel()
    k.num_prims = 1
    k.prims[0].kind, k.prims[0].term, k.prims[0].variance = 0, 0, 1.0
    for c in range(din):
        k.prims[0].w[c] = 1.0
    return k


@pytest.mark.parametrize("kcols, M, message", [
    (0, 0, "0 target columns outside 1..6"),
    (7, 5, "7 target columns outside 1..6"),
    (-1, 5, "-1 target columns outside 1..6"),
    (2, 5, "null X, Kinv, alpha, grad or workspace"),
    (2, -1, "negative M"),
])
def test_lml_grad_cols_rejects_malformed_calls(sl, kcols, M, message):
    nat = sl._native
    before = nat.launch_count()
    bufs = (0x1000, 0x2000, None, 0x3000, 0x4000)
    X, Kinv, alpha, grad, work = bufs
    assert nat.load().slb_gp_lml_grad_cols(None, X, M, 3, _kernel(nat), Kinv, alpha, kcols, grad, work) != 0
    assert message in nat.last_error(), nat.last_error()
    assert "slb_gp_lml_grad_cols" in nat.last_error()
    assert nat.launch_count() == before


@pytest.mark.parametrize("kcols", [1, 2, 6])
def test_lml_grad_cols_empty_data_set_launches_nothing(sl, kcols):
    nat = sl._native
    before = nat.launch_count()
    assert nat.load().slb_gp_lml_grad_cols(None, None, 0, 3, _kernel(nat), None, None, kcols, None, None) == 0
    assert nat.launch_count() == before
    gp = sl.GPRCached(np.empty((0, 3)), np.empty((0, kcols)), sl.RBF(3))
    lml, grads = gp.log_likelihood_and_gradient()
    assert lml == 0.0 and all(not np.any(v) for v in grads.values())
    assert nat.launch_count() == before


# ---------------------------------------------------------------- the joint LML reference
def _oracle_case(M, k, seed):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1, 1, (M, 3))
    Y = np.sin(2 * X[:, :1] + np.arange(k)) + 0.1 * rng.standard_normal((M, k))
    rows = rng.uniform(-0.5, 0.5, (k, 3))
    return X, Y, rows


@pytest.mark.parametrize("k", [1, 2, 4])
@pytest.mark.parametrize("M", [1, 9, 40])
def test_joint_reference_is_the_sum_of_the_columns(k, M):
    X, Y, rows = _oracle_case(M, k, M + k)
    for name, builder in R.kernel_set(3):
        kern, noise = builder(R.ORACLE_KERNELS), R.Noise(0.07)
        lml, grads, mags = RC.log_likelihood_and_gradient_cols(kern, noise, X, Y, rows)
        parts = [R.log_likelihood_and_gradient(kern, noise, X, Y[:, [c]], R.O.LinearMean(rows[c]))
                 for c in range(k)]
        assert_allclose(lml, sum(p[0] for p in parts), rtol=1e-12, atol=1e-12 * M * k)
        for path in grads:
            assert_allclose(grads[path], sum(p[1][path] for p in parts), rtol=0,
                            atol=1e-12 * (np.max(mags[path]) + 1.0), err_msg=(name, path))


def test_joint_reference_against_central_differences():
    X, Y, rows = _oracle_case(25, 3, 5)
    for name, builder in R.kernel_set(3):
        kern, noise = builder(R.ORACLE_KERNELS), R.Noise(0.07)
        _, grads, _ = RC.log_likelihood_and_gradient_cols(kern, noise, X, Y, rows)
        for path, (owner, attr) in R.parameters(kern, noise).items():
            base = np.array(getattr(owner, attr), dtype=np.float64, copy=True)
            flat = np.atleast_1d(base).copy()
            for c in range(flat.size):
                h = 1e-6 * max(1.0, abs(flat[c]))
                vals = []
                for sgn in (1, -1):
                    trial = flat.copy()
                    trial[c] += sgn * h
                    setattr(owner, attr, trial.reshape(np.shape(base)) if np.ndim(base) else float(trial[0]))
                    vals.append(RC.log_likelihood_and_gradient_cols(kern, noise, X, Y, rows)[0])
                setattr(owner, attr, base if np.ndim(base) else float(base))
                fd = (vals[0] - vals[1]) / (2 * h)
                assert_allclose(np.atleast_1d(grads[path])[c], fd, rtol=1e-5, atol=1e-6, err_msg=(name, path))
