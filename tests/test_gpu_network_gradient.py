"""GPU tests of ``NetworkGradient`` (``SLB_FLAG_GRADIENT`` on a LyapunovNetwork or a one-output
NeuralNetwork): the fused input gradient equals ``slb_function_vjp`` with cotangent 1 bit for bit and the
float64 torch-CPU autograd of ``network_grad_oracle.py`` to 1e-12; the post-op wrappers reduce it as numpy
does; and ``Norm1Function(V.gradient_function())`` as L_V makes the Lyapunov sweeps of
lyapunov_function_learning.ipynb fused (deterministic and GP dynamics, filtered, full and adaptive) with
the same results as the composed path through ``V.gradient``."""
import os
import sys

import numpy as np
import pytest
import torch
from numpy.testing import assert_array_equal

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import bench_workloads as W  # noqa: E402
import network_grad_oracle as G  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sl():
    import __graft_entry__
    __graft_entry__.build()
    import safe_learning_b200 as sl
    return sl


def _cuda(a):
    return torch.tensor(np.asarray(a, dtype=np.float64), device="cuda")


# ---------------------------------------------------------------- shapes
# ("lnn", input_dim, widths, activations) | ("mlp", layers, nonlinearities, use_bias, output_scale)
SHAPES = [
    ("lnn", 2, [64, 64, 64], ["tanh"] * 3),                          # lyapunov_function_learning
    ("lnn", 4, [64, 64, 64], ["tanh"] * 3),                          # C4
    ("lnn", 2, [64, 64, 64], ["relu"] * 3),
    ("lnn", 2, [2, 2], ["linear", "relu"]),
    ("lnn", 1, [1], ["tanh"]),                                       # in_dim 1, one layer
    ("lnn", 6, [64] * 8, ["tanh", "relu"] * 4),                      # in_dim 6, eight layers of 64
    ("lnn", 3, [7, 8, 31, 32, 33, 63], ["tanh", "relu", "linear", "tanh", "relu", "tanh"]),   # ragged
    ("mlp", [2, 64, 64, 1], ["relu", "relu", None], True, 1.0),      # value network [64, 64, 1]
    ("mlp", [2, 32, 32, 1], ["relu", "relu", "tanh"], False, 0.8),   # no bias, output_scale != 1
    ("mlp", [6, 31, 17, 1], ["tanh", "relu", None], True, -1.7),
    ("mlp", [1, 5, 1], ["tanh", "tanh"], True, 2.5),
    ("mlp", [4] + [64] * 7 + [1], ["tanh", "relu"] * 3 + ["tanh", None], True, 1.1),
]
N_POINTS = [1, 31, 33, 100000]


def _net(sl, shape, seed=0):
    if shape[0] == "lnn":
        _, din, widths, acts = shape
        return sl.LyapunovNetwork(din, widths, acts, seed=seed)
    _, layers, acts, bias, scale = shape
    net = sl.NeuralNetwork(layers, acts, output_scale=scale, use_bias=bias, seed=seed)
    if bias and len(layers) > 2:
        rng = np.random.default_rng(seed)
        net.biases = [rng.normal(scale=0.3, size=d) for d in layers[1:-1]]
    return net


def _vjp_in(net, x):
    from safe_learning_b200 import functions as F
    return F._function_vjp(net, x, torch.ones((x.shape[0], 1), dtype=torch.float64, device=x.device))[0]


def _points(net, n, seed):
    return _cuda(np.random.default_rng(seed).uniform(-1.5, 1.5, (n, net.input_dim)))


@pytest.mark.parametrize("shape", range(len(SHAPES)))
@pytest.mark.parametrize("n", N_POINTS)
def test_gradient_equals_vjp_bit_for_bit(sl, shape, n):
    net = _net(sl, SHAPES[shape], seed=shape)
    x = _points(net, n, seed=n)
    got = net.gradient_function().evaluate_device(x)
    assert got.shape == (n, net.input_dim)
    assert torch.equal(got, _vjp_in(net, x))


def test_relu_preactivation_of_exactly_zero_has_derivative_zero(sl):
    """x = 0 with zero biases: every first-layer pre-activation is exactly 0, ReLU' = 0 there (as TF's),
    so the gradient is 0 -- as the VJP's."""
    net = sl.NeuralNetwork([2, 16, 1], ["relu", None], seed=2)          # biases are drawn as zeros
    x = np.zeros((40, 2))
    x[::2] = np.random.default_rng(0).uniform(-1, 1, (20, 2))
    xt = _cuda(x)
    got = net.gradient_function().evaluate_device(xt)
    assert torch.equal(got, _vjp_in(net, xt))
    assert not got[1::2].any()
    lnn = sl.LyapunovNetwork(2, [4, 4], ["relu", "relu"], seed=1)
    zero = _cuda(np.zeros((3, 2)))
    assert not lnn.gradient_function().evaluate_device(zero).any()


def _oracle_grad(net, x):
    xt = torch.tensor(x, requires_grad=True)
    params = [p.detach().cpu() for p in net.parameters]
    if hasattr(net, "output_dims"):
        out = G.lyapunov_network(xt, params, net.input_dim, net.output_dims, net.activations, net.eps)
    else:
        kernels = [p for p, nm in zip(params, net.parameter_names) if nm.endswith("kernel")]
        biases = [p for p, nm in zip(params, net.parameter_names) if nm.endswith("bias")]
        out = G.mlp(xt, kernels, biases, net.nonlinearities, net.output_scale, net.use_bias)
    out.sum().backward()
    return xt.grad.numpy()


def _close(got, want, rtol=1e-12):
    """rtol with atol = rtol max|want| (entries that cancel to ~0)."""
    atol = rtol * max(float(np.max(np.abs(want))), 1e-300)
    np.testing.assert_allclose(got, want, rtol=rtol, atol=atol)


@pytest.mark.parametrize("shape", range(len(SHAPES)))
def test_gradient_matches_autograd_oracle(sl, shape):
    net = _net(sl, SHAPES[shape], seed=shape)
    x = np.random.default_rng(shape).uniform(-1.5, 1.5, (1000, net.input_dim))
    _close(net.gradient_function()(x), _oracle_grad(net, x))


@pytest.mark.parametrize("shape", [0, 1, 6, 7, 9])
def test_wrappers_reduce_the_gradient_as_numpy(sl, shape):
    net = _net(sl, SHAPES[shape], seed=shape)
    x = _points(net, 5000, seed=3)
    g = net.gradient_function()
    raw = g.evaluate_device(x).cpu().numpy()
    a = np.abs(raw)
    norm1 = a[:, 0].copy()
    for j in range(1, a.shape[1]):                     # the kernel's left-to-right sum
        norm1 = norm1 + a[:, j]
    cases = [(sl.AbsFunction(g), a), (sl.Norm1Function(g), norm1[:, None]),
             (sl.MaxAbsFunction(g), a.max(axis=1, keepdims=True)), (sl.ScaledFunction(g, -0.3), raw * -0.3),
             (-sl.Norm1Function(g), -norm1[:, None])]
    for fun, want in cases:
        got = fun.evaluate_device(x).cpu().numpy()
        assert got.shape == want.shape
        assert_array_equal(got, want)


def test_gradient_method_and_object(sl):
    net = sl.LyapunovNetwork(2, [64, 64, 64], ["tanh"] * 3, seed=4)
    x = np.random.default_rng(1).uniform(-1, 1, (300, 2))
    got = net.gradient(x)
    assert isinstance(got, np.ndarray) and got.shape == (300, 2)
    assert_array_equal(got, _vjp_in(net, _cuda(x)).cpu().numpy())
    assert_array_equal(net.gradient(_cuda(x)), got)
    with pytest.raises(sl.DimensionError):
        sl.NeuralNetwork([2, 8, 2], ["tanh", None]).gradient_function()(x)


# ---------------------------------------------------------------- the notebook's certification, fused
def _notebook(sl, num_points=251, seed=21):
    """lyapunov_function_learning.ipynb cells 13-20 on the product: pendulum plant, saturated LQR policy,
    V = LyapunovNetwork(2, [64, 64, 64], tanh), tau = sum(unit) / 2."""
    par = W.make_pendulum(num_points=num_points, M=8)
    pl = par["plant"]
    plant = sl.InvertedPendulum(normalization=[pl["state_norm"], pl["action_norm"]], **pl["true"])
    policy = sl.Saturation(sl.LinearSystem(-par["K"]), -1., 1.)
    V = sl.LyapunovNetwork(2, [64, 64, 64], ["tanh"] * 3, eps=1e-8, seed=seed)
    grid = sl.GridWorld(par["limits"], par["num_points"])

    def make(lv, dynamics=plant, **kw):
        return sl.Lyapunov(grid, V, dynamics, par["L_dyn"], lv, par["tau"], policy, par["initial"], **kw)
    return V, make


def _composed_lv(V):
    return lambda x: np.abs(V.gradient(x)).sum(1, keepdims=True)


def _run(lyap, **kw):
    lyap.update_values()
    neg, det = lyap.compute_negative(want_details=True)
    out = {k: det[k].cpu().numpy().copy() for k in ("decrease", "threshold")}
    out["negative"] = neg.cpu().numpy().copy()
    lyap.update_safe_set(**kw)
    out["safe_set"] = np.array(lyap.safe_set)
    out["c_max"] = lyap.feed_dict[lyap.c_max]
    out["values"] = np.array(lyap.values)
    return out


def _assert_same(a, b, keys=("negative", "decrease", "threshold", "safe_set", "c_max")):
    for k in keys:
        if k == "c_max":
            assert a[k] == b[k]
        else:
            assert_array_equal(a[k], b[k], err_msg=k)


def test_notebook_sweep_is_fused_and_equals_the_composed_path(sl):
    V, make = _notebook(sl)
    fused = make(sl.Norm1Function(V.gradient_function()))
    composed = make(_composed_lv(V))
    assert not fused._is_composed() and composed._is_composed()
    a, b = _run(fused), _run(composed)
    _assert_same(a, b)
    assert 0 < a["negative"].sum() < a["negative"].size           # the decision is not one-sided
    # L_V enters the threshold: it is not a constant multiple of tau
    assert np.unique(a["threshold"]).size > 1000


def test_in_place_sgd_step_reaches_the_fused_sweep(sl):
    V, make = _notebook(sl, num_points=101)
    fused = make(sl.Norm1Function(V.gradient_function()))
    before = _run(fused)
    opt = torch.optim.SGD(V.parameters, lr=0.05)
    x = _cuda(np.random.default_rng(3).uniform(-1, 1, (1000, 2)))
    loss = torch.mean(torch.abs(V.torch(x) - 0.1 * torch.sum(x * x, dim=1, keepdim=True)))
    opt.zero_grad()
    loss.backward()
    opt.step()
    after = _run(fused)
    assert not np.array_equal(after["threshold"], before["threshold"])
    _assert_same(after, _run(make(_composed_lv(V))))


# ---------------------------------------------------------------- GP dynamics: L_V at the predicted mean
def _near_threshold(det):
    dec, thr = det["decrease"], det["threshold"]
    scale = np.maximum(np.maximum(np.abs(dec), np.abs(thr)), 1e-300)
    return int(np.count_nonzero(np.abs(dec - thr) <= 1e-9 * scale))


def _gp_case(sl, num_points=101, M=200):
    par = W.make_pendulum(num_points=num_points, M=M)
    base = W.build_product(par)
    V = sl.LyapunovNetwork(2, [64, 64, 64], ["tanh"] * 3, eps=1e-8, seed=21)

    def make(lv, **kw):
        return sl.Lyapunov(base.discretization, V, base.dynamics, par["L_dyn"], lv, par["tau"], base.policy,
                           initial_set=par["initial"], **kw)
    return V, make


def _flags_and_set(lyap, filt, **kw):
    lyap.filter = filt
    neg = lyap.compute_negative().cpu().numpy().copy()
    lyap.update_safe_set(**kw)
    return neg, np.array(lyap.safe_set), lyap.feed_dict[lyap.c_max]


def test_gp_sweep_filtered_equals_full_and_composed(sl):
    V, make = _gp_case(sl)
    fused = make(sl.Norm1Function(V.gradient_function()))
    assert not fused._is_composed()
    cfg = fused.sweep_descriptor()
    from safe_learning_b200 import _native as nat
    assert nat.load().slb_filter_stage1(cfg) == 64                    # fp64 mean stage
    neg_f, safe_f, c_f = _flags_and_set(fused, True)
    neg_full, safe_full, c_full = _flags_and_set(fused, False)
    assert_array_equal(neg_f, neg_full)
    assert_array_equal(safe_f, safe_full)
    assert c_f == c_full
    _, det = fused.compute_negative(want_details=True)
    det = {k: det[k].cpu().numpy() for k in ("decrease", "threshold")}
    assert _near_threshold(det) == 0
    composed = make(_composed_lv(V))
    composed.update_safe_set()
    assert_array_equal(np.array(composed.safe_set), safe_full)
    assert composed.feed_dict[composed.c_max] == c_full
    assert 0 < neg_full.sum() < neg_full.size


def test_gp_adaptive_sweep_equals_composed(sl):
    V, make = _gp_case(sl, num_points=61, M=200)
    fused = make(sl.Norm1Function(V.gradient_function()), adaptive=True)
    _, safe_f, c_f = _flags_and_set(fused, True, max_refinement=3)
    _, safe_full, c_full = _flags_and_set(fused, False, max_refinement=3)
    assert_array_equal(safe_f, safe_full)
    assert c_f == c_full
    composed = make(_composed_lv(V), adaptive=True)
    composed.update_safe_set(max_refinement=3)
    assert_array_equal(np.array(composed.safe_set), safe_full)
    assert composed.feed_dict[composed.c_max] == c_full


def test_c4_shape_filtered_equals_full(sl):
    """bench_workloads.make_cartpole (16^4 grid, M = 200, V = LyapunovNetwork(4, [64, 64, 64])) with
    L_V = |dV/dx|_1 in place of the constant 1.0."""
    par = W.make_cartpole(num_points=16, M=200)
    base = W.build_product(par)
    V = base.lyapunov_function
    lyap = sl.Lyapunov(base.discretization, V, base.dynamics, par["L_dyn"],
                       sl.Norm1Function(V.gradient_function()), par["tau"], base.policy,
                       initial_set=par["initial"])
    neg_f, safe_f, c_f = _flags_and_set(lyap, True)
    neg_full, safe_full, c_full = _flags_and_set(lyap, False)
    assert_array_equal(neg_f, neg_full)
    assert_array_equal(safe_f, safe_full)
    assert c_f == c_full


# ---------------------------------------------------------------- a ReLU value network, and no backward
def test_maxabs_of_a_relu_value_network_gradient(sl):
    """MaxAbsFunction(value.gradient_function()): the L_V of inverted_pendulum.ipynb cell 14 for a
    [2, 64, 64, 1] ReLU value network."""
    net = sl.NeuralNetwork([2, 64, 64, 1], ["relu", "relu", None], seed=5)
    rng = np.random.default_rng(5)
    net.biases = [rng.normal(scale=0.3, size=64) for _ in range(2)]
    x = rng.uniform(-1, 1, (4000, 2))
    got = sl.MaxAbsFunction(net.gradient_function())(x)
    _close(got, np.abs(_oracle_grad(net, x)).max(axis=1, keepdims=True))


def test_backward_through_a_network_gradient_raises(sl):
    net = sl.LyapunovNetwork(2, [8, 8], ["tanh", "tanh"], seed=0)
    x = _cuda(np.random.default_rng(0).uniform(-1, 1, (16, 2))).requires_grad_(True)
    out = net.gradient_function().torch(x)
    assert torch.equal(out.detach(), net.gradient_function().evaluate_device(x.detach()))
    with pytest.raises(NotImplementedError, match="second derivative"):
        out.sum().backward()
