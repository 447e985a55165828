"""CPU tests of the trainable networks (``NeuralNetwork`` / ``LyapunovNetwork`` parameters, the two
constructor conventions, ``lipschitz``), of the torch-CPU oracle of ``network_grad_oracle.py``, and of
the host-side checks of ``slb_function_vjp`` (``csrc/network_grad.cu``)."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import network_grad_oracle as G  # noqa: E402
import oracle as O  # noqa: E402
import safe_learning_b200 as sl  # noqa: E402
from safe_learning_b200 import _native as nat  # noqa: E402

T64 = torch.float64


# ---------------------------------------------------------------- the oracle against the numpy forward
def test_oracle_mlp_forward_matches_reference_path():
    rng = np.random.default_rng(0)
    dims = [3, 17, 9, 2]
    ws = [rng.normal(size=(a, b)) / np.sqrt(a) for a, b in zip(dims[:-1], dims[1:])]
    bs = [rng.normal(size=b) for b in dims[1:-1]]
    x = rng.normal(size=(50, 3))
    ref = O.NeuralNetwork(dims, [np.tanh, lambda v: np.maximum(v, 0), None], ws, bs,
                          output_scale=0.7)(x)
    got = G.mlp(torch.tensor(x), [torch.tensor(w) for w in ws], [torch.tensor(b) for b in bs],
                ["tanh", "relu", "linear"], 0.7).numpy()
    np.testing.assert_allclose(got, ref, rtol=1e-13, atol=1e-13)


def test_oracle_lyapunov_forward_matches_reference_path():
    net = sl.LyapunovNetwork(2, [4, 4, 9], ["tanh", "relu", "tanh"], seed=3)
    x = np.random.default_rng(1).normal(size=(40, 2))
    ref = O.LyapunovNetwork(2, [4, 4, 9], [np.tanh, lambda v: np.maximum(v, 0), np.tanh],
                            net.weights)(x)
    got = G.lyapunov_network(torch.tensor(x), [torch.tensor(p.detach().cpu().numpy())
                                                for p in net.parameters],
                             2, [4, 4, 9], ["tanh", "relu", "tanh"]).numpy()
    np.testing.assert_allclose(got, ref, rtol=1e-13, atol=1e-13)


def test_oracle_plants_match_reference_path():
    x = np.random.default_rng(2).normal(size=(30, 3))
    norm = (np.array([1.0, 2.0]), np.array([0.5]))
    ref = O.InvertedPendulum(0.15, 0.5, 0.1, normalization=norm)(x)
    got = G.pendulum(torch.tensor(x), 0.15, 0.5, 0.1, normalization=norm).numpy()
    np.testing.assert_allclose(got, ref, rtol=1e-13, atol=1e-13)
    x = np.random.default_rng(3).normal(size=(30, 5))
    norm = (np.array([0.5, 0.3, 1.0, 2.0]), np.array([4.0]))
    ref = O.CartPole(0.175, 1.732, 0.28, 0.01, 0.01, normalization=norm)(x)
    got = G.cartpole(torch.tensor(x), 0.175, 1.732, 0.28, 0.01, 0.01, normalization=norm).numpy()
    np.testing.assert_allclose(got, ref, rtol=1e-13, atol=1e-13)


@pytest.mark.parametrize("which", ["mlp", "lnn", "pendulum", "cartpole"])
def test_oracle_autograd_matches_central_differences(which):
    rng = np.random.default_rng(4)
    if which == "mlp":
        ws = [torch.tensor(rng.normal(size=s)) for s in [(2, 5), (5, 3)]]
        bs = [torch.tensor(rng.normal(size=5))]
        x = torch.tensor(rng.normal(size=(6, 2)))
        f = lambda x: G.mlp(x, ws, bs, ["tanh", "linear"], 1.3)
    elif which == "lnn":
        wp = [torch.tensor(rng.normal(size=s)) for s in [(2, 2), (1, 2), (2, 3), (2, 3)]]
        x = torch.tensor(rng.normal(size=(6, 2)))
        f = lambda x: G.lyapunov_network(x, wp, 2, [3, 5], ["tanh", "tanh"])
    elif which == "pendulum":
        x = torch.tensor(rng.normal(size=(6, 3)))
        f = lambda x: G.pendulum(x, 0.15, 0.5, 0.1, normalization=([1.0, 2.0], [0.5]))
    else:
        x = torch.tensor(rng.normal(size=(6, 5)))
        f = lambda x: G.cartpole(x, 0.175, 1.732, 0.28, 0.01, 0.01)
    xg = x.clone().requires_grad_(True)
    f(xg).sum().backward()
    fd = G.central_difference(f, x.clone())
    np.testing.assert_allclose(xg.grad.numpy(), fd.numpy(), rtol=1e-6, atol=1e-8)


# ---------------------------------------------------------------- parameters
@pytest.mark.parametrize("use_bias", [True, False])
def test_mlp_parameter_order_and_shapes(use_bias):
    net = sl.NeuralNetwork([3, 16, 8, 2], ["relu", "tanh", None], use_bias=use_bias)
    shapes = [tuple(p.shape) for p in net.parameters]
    if use_bias:
        assert net.parameter_names == ["layer_0/kernel", "layer_0/bias", "layer_1/kernel",
                                       "layer_1/bias", "output/kernel"]
        assert shapes == [(3, 16), (16,), (16, 8), (8,), (8, 2)]
    else:
        assert net.parameter_names == ["layer_0/kernel", "layer_1/kernel", "output/kernel"]
        assert shapes == [(3, 16), (16, 8), (8, 2)]
    for p in net.parameters:
        assert p.dtype == T64 and p.requires_grad and p.is_leaf


def test_reference_convention_is_lazy_and_draws_like_the_eager_one():
    lazy = sl.NeuralNetwork([64, 64, 1], ["relu", "relu", None], seed=7)
    assert lazy.parameters == [] and lazy.weights == [] and not lazy.built
    assert lazy.output_dim == 1
    wrapped = sl.Saturation(lazy, -1., 1.)
    assert wrapped.input_dim is None
    with pytest.raises(sl.DimensionError, match="build"):
        lazy.descriptor()
    lazy.build(2)                         # what the first evaluation does with its points' width
    assert wrapped.input_dim == 2
    eager = sl.NeuralNetwork([2, 64, 64, 1], ["relu", "relu", None], seed=7)
    assert lazy.parameter_names == eager.parameter_names
    for a, b in zip(lazy.parameters, eager.parameters):
        assert torch.equal(a.detach().cpu(), b.detach().cpu())
    assert lazy.input_dim == 2


def test_unbuilt_network_is_not_quietly_taken_off_the_fused_path():
    """A fused consumer asking for the descriptor of a network whose input width is not known yet gets
    an error that says so, instead of a silent switch to the host loop."""
    from safe_learning_b200 import reinforcement_learning as rl
    lazy = sl.NeuralNetwork([8, 1], ["relu", None])
    with pytest.raises(sl.DimensionError, match="build"):
        rl._fusable(lazy)


def test_weights_and_biases_round_trip_and_bump_version():
    net = sl.NeuralNetwork([2, 5, 1], ["tanh", None], seed=1)
    w = [np.arange(10.0).reshape(2, 5), np.ones((5, 1))]
    v0 = net.version
    net.weights = w
    assert net.version != v0
    for a, b in zip(net.weights, w):
        assert np.array_equal(a, b)
    net.biases = [np.full(5, 0.25)]
    assert np.array_equal(net.biases[0], np.full(5, 0.25))
    assert np.array_equal(net.parameters[1].detach().cpu().numpy(), np.full(5, 0.25))
    v1 = net.version
    with torch.no_grad():
        net.parameters[0].add_(1.0)           # an optimizer's in-place step
    assert net.version != v1
    assert np.array_equal(net.weights[0], w[0] + 1.0)
    net.parameters = [torch.zeros(2, 5), np.zeros(5), np.zeros((5, 1))]
    assert all(not p.detach().cpu().numpy().any() for p in net.parameters)


@pytest.mark.parametrize("dims", [[2, 2, 2], [2, 64, 64, 64], [4, 4, 9, 9]])
def test_lyapunov_parameter_order_and_shapes(dims):
    net = sl.LyapunovNetwork(dims[0], dims[1:], ["tanh"] * (len(dims) - 1))
    names, shapes = [], []
    din = dims[0]
    for i, dout in enumerate(dims[1:]):
        names.append("weights_posdef_%d" % i)
        shapes.append((math.ceil((din + 1) / 2), din))
        if dout > din:
            names.append("weights_%d" % i)
            shapes.append((dout - din, din))
        din = dout
    assert net.parameter_names == names
    assert [tuple(p.shape) for p in net.parameters] == shapes
    for (w0, w1), k in zip(net.weights, net.kernels()):
        assert np.array_equal(k[:w0.shape[1]], w0.T.dot(w0) + net.eps * np.eye(w0.shape[1]))
        if w1 is not None:
            assert np.array_equal(k[w0.shape[1]:], w1)


def test_lyapunov_weights_round_trip():
    net = sl.LyapunovNetwork(2, [3, 3], ["tanh", "tanh"], seed=2)
    new = [(np.ones((2, 2)), np.full((1, 2), 2.0)), (np.eye(2, 3), None)]
    net.weights = new
    for (a0, a1), (b0, b1) in zip(net.weights, new):
        assert np.array_equal(a0, b0)
        assert (a1 is None and b1 is None) or np.array_equal(a1, b1)


@pytest.mark.parametrize("use_bias", [True, False])
def test_lipschitz_is_product_of_largest_singular_values(use_bias):
    net = sl.NeuralNetwork([2, 32, 32, 1], ["relu", "relu", None], use_bias=use_bias, seed=5)
    expect = np.prod([np.linalg.svd(w, compute_uv=False)[0] for w in net.weights])
    assert isinstance(net.lipschitz(), float)
    assert net.lipschitz() == pytest.approx(expect, rel=1e-14)


# ---------------------------------------------------------------- host-side checks of the C entry point
def _lib():
    return nat.load()


def _net_desc(kind=nat.FN_LYAPUNOV_NN, widths=(64, 64, 64), in_dim=2, out_dim=1):
    d = nat.SlbFunction()
    d.kind, d.in_dim, d.out_dim = kind, in_dim, out_dim
    d.cparams[0] = len(widths)
    for i, w in enumerate(widths):
        d.cparams[1 + i] = w
        d.cparams[9 + i] = 0
    d.cparams[17] = 1.0
    d.cparams[18] = 1.0
    d.matrix = 0x1000                        # never dereferenced: every case below fails on the host
    return d


def _vjp(desc, n=10, points=0x2000, gout=0x3000, gin=0x4000, gpar=None, ws=None):
    return _lib().slb_function_vjp(None, desc, points, n, gout, gin, gpar, None, ws)


def test_vjp_rejects_unsupported_kind():
    desc = nat.SlbFunction()
    desc.kind, desc.in_dim, desc.out_dim = nat.FN_QUADRATIC, 2, 1
    desc.matrix = 0x1000
    assert _vjp(desc) != 0
    assert "has no VJP" in nat.last_error()
    assert _lib().slb_function_vjp_workspace(desc, 10) == -1


def test_vjp_rejects_post_op_flags():
    desc = _net_desc()
    desc.flags = nat.FLAG_SCALE
    assert _vjp(desc) != 0
    assert "flags" in nat.last_error()


def test_vjp_rejects_null_points_or_cotangent():
    assert _vjp(_net_desc(), points=None) != 0
    assert "null points or cotangent" in nat.last_error()
    assert _vjp(_net_desc(), gout=None) != 0
    assert "null points or cotangent" in nat.last_error()


def test_vjp_rejects_negative_n():
    assert _vjp(_net_desc(), n=-1) != 0
    assert "negative n" in nat.last_error()
    assert _lib().slb_function_vjp_workspace(_net_desc(), -1) == -1


def test_vjp_rejects_parameter_gradient_of_a_plant():
    sl_p = sl.InvertedPendulum(0.15, 0.5, 0.1)
    desc = sl_p.descriptor()
    assert _vjp(desc, gpar=0x5000) != 0
    assert "no parameters" in nat.last_error()
    assert _lib().slb_function_vjp_workspace(desc, 1000) == 0


def test_vjp_rejects_missing_workspace():
    assert _vjp(_net_desc(), n=1000, gpar=0x5000, ws=None) != 0
    assert "workspace" in nat.last_error()


def test_vjp_rejects_bad_shapes():
    assert _vjp(_net_desc(widths=(64, 65))) != 0
    assert _vjp(_net_desc(kind=nat.FN_MLP, widths=(8, 7), out_dim=7)) != 0


@pytest.mark.parametrize("widths,in_dim,nparams,per_sm", [
    ((64, 64, 64), 2, 2 * 64 + 2 * 64 * 64, 2),
    ((64,) * 8, 8, 8 * 64 + 7 * 64 * 64, 1),
    ((1,), 1, 1, 8),
])
def test_vjp_workspace_size(widths, in_dim, nparams, per_sm):
    desc = _net_desc(widths=widths, in_dim=in_dim)
    lib = _lib()
    assert lib.slb_function_vjp_workspace(desc, 0) == 0
    assert lib.slb_function_vjp_workspace(desc, 32) == 0        # one tile: written in place
    assert lib.slb_function_vjp_workspace(desc, 33) == 2 * nparams * 8
    ctas = min(-(-63001 // 32), 132 * per_sm)
    assert lib.slb_function_vjp_workspace(desc, 63001) == ctas * nparams * 8


def test_vjp_signatures_are_declared():
    assert nat.SIGNATURES["slb_function_vjp_workspace"][0] is C.c_int64
    assert len(nat.SIGNATURES["slb_function_vjp"][1]) == 9
