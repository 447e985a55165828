"""GPU tests of ``slb_function_vjp`` and the trainable networks: gradients of the fused networks and
plants against torch-CPU autograd of the oracle restatement (``network_grad_oracle.py``), the
recomputed forward against ``slb_eval_function``, determinism of the parameter reduction, training
loops of the reference's notebooks step by step against the oracle, and the fused sweeps on the
trained weights."""
import os
import sys

import numpy as np
import pytest
import torch
from numpy.testing import assert_allclose, assert_array_equal

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import bench_workloads as W  # noqa: E402
import network_grad_oracle as G  # noqa: E402
import oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
TILE = 32


@pytest.fixture(scope="module")
def sl():
    import __graft_entry__
    __graft_entry__.build()
    import safe_learning_b200 as sl
    return sl


def _cpu(t):
    return t.detach().cpu()


def _close(got, want, rtol=1e-10):
    """rtol with atol = 1e-12 max|want| (entries that cancel to ~0)."""
    got, want = np.asarray(got), np.asarray(want)
    atol = 1e-12 * max(float(np.max(np.abs(want))) if want.size else 0.0, 1e-300)
    assert_allclose(got, want, rtol=rtol, atol=atol)


def _mlp_oracle(net, x, cot):
    """(grad_in, [grad per parameter], out) of the oracle at the network's current parameters."""
    params = [_cpu(p).clone().requires_grad_(True) for p in net.parameters]
    kernels = [p for p, nm in zip(params, net.parameter_names) if nm.endswith("kernel")]
    biases = [p for p, nm in zip(params, net.parameter_names) if nm.endswith("bias")]
    xt = torch.tensor(x, requires_grad=True)
    out = G.mlp(xt, kernels, biases, net.nonlinearities, net.output_scale, net.use_bias)
    (out * torch.tensor(cot)).sum().backward()
    return xt.grad.numpy(), [p.grad.numpy() for p in params], out.detach().numpy()


def _lnn_oracle(net, x, cot):
    params = [_cpu(p).clone().requires_grad_(True) for p in net.parameters]
    xt = torch.tensor(x, requires_grad=True)
    out = G.lyapunov_network(xt, params, net.input_dim, net.output_dims, net.activations, net.eps)
    (out * torch.tensor(cot)).sum().backward()
    return xt.grad.numpy(), [p.grad.numpy() for p in params], out.detach().numpy()


def _check_vjp(sl, net, n, seed=0):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1.5, 1.5, (n, net.input_dim))
    cot = rng.normal(size=(n, net.output_dim))
    gin, gpar, out = net.vjp(torch.tensor(x, device="cuda"), torch.tensor(cot, device="cuda"),
                             want_out=True)
    oracle = _lnn_oracle if isinstance(net, sl.LyapunovNetwork) else _mlp_oracle
    o_in, o_par, _ = oracle(net, x, cot)
    _close(_cpu(gin).numpy(), o_in)
    assert len(gpar) == len(o_par)
    for g, o in zip(gpar, o_par):
        assert tuple(g.shape) == o.shape
        _close(_cpu(g).numpy(), o)
    # recomputed forward: byte-identical to slb_eval_function
    ref = net.evaluate_device(torch.tensor(x, device="cuda"))
    assert torch.equal(out, ref)


# ---------------------------------------------------------------- shape grid
MLP_SHAPES = [
    ([1, 1], ["linear"], True, 1.0),
    ([3, 7, 2], ["tanh", "linear"], True, 2.5),
    ([2, 8, 8, 6], ["relu", "tanh", "linear"], True, 1.0),
    ([8, 31, 32, 33, 1], ["tanh", "relu", "tanh", "tanh"], True, 0.3),
    ([2, 63, 64, 3], ["relu", "relu", "linear"], False, -1.7),
    ([2, 64, 64, 1], ["relu", "relu", "linear"], True, 1.0),              # value net [64, 64, 1]
    ([2, 32, 32, 1], ["relu", "relu", "tanh"], False, 0.8),               # policy [32, 32, 1]
    ([4] + [64] * 7 + [5], ["tanh", "relu"] * 3 + ["tanh", "linear"], True, 1.1),   # 8 layers
    ([5, 1, 64, 1, 4], ["tanh", "linear", "relu", "tanh"], True, 1.0),
]
LNN_SHAPES = [
    (1, [1], ["tanh"]),
    (2, [64, 64, 64], ["tanh"] * 3),                                       # lyapunov_function_learning
    (4, [64, 64, 64], ["tanh"] * 3),                                       # C4
    (3, [7, 8, 31, 32, 33, 63], ["tanh", "relu", "linear", "tanh", "relu", "tanh"]),
    (8, [8, 8, 64, 64, 64, 64, 64, 64], ["tanh"] * 8),
    (2, [2, 2], ["linear", "relu"]),
]
N_GRID = [1, TILE - 1, TILE, TILE + 1, 1000]


@pytest.mark.parametrize("shape", range(len(MLP_SHAPES)))
@pytest.mark.parametrize("n", N_GRID)
def test_mlp_vjp_matches_oracle(sl, shape, n):
    dims, acts, bias, scale = MLP_SHAPES[shape]
    net = sl.NeuralNetwork(dims, acts, output_scale=scale, use_bias=bias, seed=shape)
    if bias and len(dims) > 2:
        rng = np.random.default_rng(shape)
        net.biases = [rng.normal(scale=0.3, size=d) for d in dims[1:-1]]
    _check_vjp(sl, net, n, seed=n)


@pytest.mark.parametrize("shape", range(len(LNN_SHAPES)))
@pytest.mark.parametrize("n", N_GRID)
def test_lyapunov_vjp_matches_oracle(sl, shape, n):
    din, dims, acts = LNN_SHAPES[shape]
    net = sl.LyapunovNetwork(din, dims, acts, seed=shape)
    _check_vjp(sl, net, n, seed=n)


@pytest.mark.parametrize("which", ["mlp", "lnn"])
def test_notebook_shapes_at_63001_points(sl, which):
    if which == "mlp":
        net = sl.NeuralNetwork([64, 64, 1], ["relu", "relu", None], seed=3)
        net.evaluate_device(torch.zeros((1, 2), dtype=torch.float64, device="cuda"))
    else:
        net = sl.LyapunovNetwork(2, [64, 64, 64], ["tanh"] * 3, seed=3)
    _check_vjp(sl, net, 251 ** 2, seed=5)


@pytest.mark.parametrize("kind,shape", [("mlp", 2), ("mlp", 3), ("mlp", 4), ("mlp", 7), ("mlp", 8),
                                        ("lnn", 3), ("lnn", 4)])
def test_vjp_with_many_tiles_per_cta_matches_oracle(sl, kind, shape):
    """63 001 points: every CTA accumulates several tiles into its workspace row (out = 6, odd widths,
    bias off with output_scale < 0, 8 layers)."""
    if kind == "mlp":
        dims, acts, bias, scale = MLP_SHAPES[shape]
        net = sl.NeuralNetwork(dims, acts, output_scale=scale, use_bias=bias, seed=shape)
        if bias:
            rng = np.random.default_rng(shape)
            net.biases = [rng.normal(scale=0.3, size=d) for d in dims[1:-1]]
    else:
        din, dims, acts = LNN_SHAPES[shape]
        net = sl.LyapunovNetwork(din, dims, acts, seed=shape)
    _check_vjp(sl, net, 63001, seed=shape)


def test_second_derivative_through_a_network_raises(sl):
    """The VJP kernel is not differentiable itself: a double backward raises instead of returning a
    gradient that treats the first derivative as a constant."""
    net = sl.LyapunovNetwork(2, [2, 4], ["tanh", "tanh"], seed=0)
    x = torch.tensor(np.random.default_rng(0).uniform(-1, 1, (8, 2)), device="cuda", requires_grad=True)
    (gx,) = torch.autograd.grad(net.torch(x).sum(), x, create_graph=True)
    with pytest.raises(RuntimeError):
        gx.sum().backward()


def test_relu_gradient_is_zero_at_exactly_zero(sl):
    """Points whose first-layer pre-activations are exactly 0 (x = 0, zero bias) get no gradient
    through those units, as TF's ReLU' = 0 at 0."""
    net = sl.NeuralNetwork([2, 16, 1], ["relu", None], seed=2)          # biases are drawn as zeros
    x = np.zeros((TILE + 3, 2))
    x[::2] = np.random.default_rng(0).uniform(-1, 1, (len(x[::2]), 2))
    cot = np.ones((len(x), 1))
    gin, gpar, _ = net.vjp(torch.tensor(x, device="cuda"), torch.tensor(cot, device="cuda"))
    o_in, o_par, _ = _mlp_oracle(net, x, cot)
    _close(_cpu(gin).numpy(), o_in)
    for g, o in zip(gpar, o_par):
        _close(_cpu(g).numpy(), o)
    zero = np.zeros((4, 2))
    gin, gpar, _ = net.vjp(torch.tensor(zero, device="cuda"), torch.ones((4, 1), dtype=torch.float64,
                                                                         device="cuda"))
    assert not _cpu(gin).numpy().any()
    assert all(not _cpu(g).numpy().any() for g in gpar)


@pytest.mark.parametrize("n", [TILE + 1, 63001])
def test_parameter_gradient_is_bit_reproducible(sl, n):
    net = sl.LyapunovNetwork(2, [64, 64, 64], ["tanh"] * 3, seed=1)
    rng = np.random.default_rng(7)
    x = torch.tensor(rng.uniform(-1, 1, (n, 2)), device="cuda")
    cot = torch.tensor(rng.normal(size=(n, 1)), device="cuda")
    a = net.vjp(x, cot)[1]
    b = net.vjp(x, cot)[1]
    for u, v in zip(a, b):
        assert torch.equal(u, v)


def test_zero_points_give_zero_parameter_gradient(sl):
    net = sl.NeuralNetwork([2, 8, 1], ["tanh", None], seed=1)
    gin, gpar, _ = net.vjp(torch.zeros((0, 2), dtype=torch.float64, device="cuda"),
                           torch.zeros((0, 1), dtype=torch.float64, device="cuda"))
    assert gin.shape == (0, 2)
    assert all(not _cpu(g).numpy().any() for g in gpar)


def test_lyapunov_gradient_method(sl):
    net = sl.LyapunovNetwork(2, [64, 64, 64], ["tanh"] * 3, seed=4)
    x = np.random.default_rng(1).uniform(-1, 1, (300, 2))
    o_in, _, _ = _lnn_oracle(net, x, np.ones((300, 1)))
    got = net.gradient(x)
    assert isinstance(got, np.ndarray) and got.shape == (300, 2)
    _close(got, o_in)


# ---------------------------------------------------------------- plants
PEND = dict(mass=0.15, length=0.5, friction=0.1, dt=0.01,
            normalization=[(np.deg2rad(30), np.sqrt(9.81 / 0.5)), (9.81 * 0.15 * 0.5 * 0.5,)])
CART = dict(pendulum_mass=0.175, cart_mass=1.732, length=0.28, rot_friction=0.01, dt=0.01,
            normalization=[(0.5, np.deg2rad(30), 1.0, 2.0), (5.0,)])


@pytest.mark.parametrize("which", ["pendulum", "pendulum_plain", "cartpole", "cartpole_plain"])
def test_plant_jacobian_matches_oracle(sl, which):
    rng = np.random.default_rng(3)
    if which.startswith("pendulum"):
        kw = dict(PEND) if which == "pendulum" else dict(mass=0.15, length=0.5)
        plant = sl.InvertedPendulum(**kw)
        f = lambda z: G.pendulum(z, kw["mass"], kw["length"], kw.get("friction", 0.0),
                                 kw.get("dt", 1 / 80), kw.get("normalization"))
        x = rng.uniform(-1, 1, (500, 3))
    else:
        kw = dict(CART) if which == "cartpole" else dict(pendulum_mass=0.175, cart_mass=1.732, length=0.28)
        plant = sl.CartPole(**kw)
        f = lambda z: G.cartpole(z, kw["pendulum_mass"], kw["cart_mass"], kw["length"],
                                 kw.get("rot_friction", 0.0), kw.get("dt", 0.01), kw.get("normalization"))
        x = rng.uniform(-1, 1, (500, 5))
    jac = _cpu(plant.jacobian_device(torch.tensor(x, device="cuda"))).numpy()
    want = torch.autograd.functional.jacobian(lambda z: f(z).sum(dim=0), torch.tensor(x))
    want = want.permute(1, 0, 2).numpy()                                      # [n, out, in]
    assert_allclose(jac, want, rtol=1e-12, atol=1e-12 * np.abs(want).max())
    # central differences of the fused forward
    h = 1e-6
    for i in range(x.shape[1]):
        e = np.zeros(x.shape[1])
        e[i] = h
        fd = (plant(x + e) - plant(x - e)) / (2 * h)
        assert_allclose(jac[:, :, i], fd, rtol=1e-6, atol=1e-8)
    # torch(): one VJP, and the recomputed forward equals the fused evaluation
    xt = torch.tensor(x, device="cuda", requires_grad=True)
    cot = torch.tensor(rng.normal(size=(500, plant.output_dim)), device="cuda")
    (plant.torch(xt) * cot).sum().backward()
    assert_allclose(_cpu(xt.grad).numpy(), np.einsum("no,noi->ni", _cpu(cot).numpy(), jac),
                    rtol=1e-12, atol=1e-14)
    import safe_learning_b200.functions as F
    _, _, out = F._function_vjp(plant, torch.tensor(x, device="cuda"), cot, want_in=False, want_out=True)
    assert torch.equal(out, plant.evaluate_device(x))


# ---------------------------------------------------------------- notebook training loops
def _relu_margin(kernels, biases, acts, x, use_bias):
    """min |pre-activation| over the ReLU layers of the oracle MLP (a ReLU kink within 1e-12 would
    let the two runs take different branches)."""
    net, margin = torch.tensor(x), np.inf
    with torch.no_grad():
        for i, w in enumerate(kernels):
            net = net @ w
            if use_bias and i + 1 < len(kernels):
                net = net + biases[i]
            if acts[i] == "relu":
                margin = min(margin, float(net.abs().min()))
            net = G.ACT[acts[i]](net)
    return margin


def _assert_same_side(gpu, cpu, what, step):
    """Entries within 1e-12 of a kink (|.| or max(., 0)) must sit on the same side of it in both runs,
    exactly 0 counting as its own side (both runs then take the subgradient 0); the count is reported."""
    gpu, cpu = np.asarray(gpu).ravel(), np.asarray(cpu).ravel()
    near = (np.abs(gpu) < 1e-12) | (np.abs(cpu) < 1e-12)
    assert np.array_equal(np.sign(gpu[near]), np.sign(cpu[near])), \
        "step %d: %d %s within 1e-12 of the kink, on different sides in the two runs" % (step, near.sum(), what)
    return int(near.sum())


def _assert_params_close(net, oracle_params, step):
    for p, q in zip(net.parameters, oracle_params):
        a, b = _cpu(p).numpy(), q.detach().numpy()
        assert_allclose(a, b, rtol=1e-9, atol=1e-9 * max(np.abs(b).max(), 1e-300),
                        err_msg="step %d" % step)


def _oracle_copy(net):
    return [_cpu(p).clone().requires_grad_(True) for p in net.parameters]


def _split(net, params):
    k = [p for p, nm in zip(params, net.parameter_names) if nm.endswith("kernel")]
    b = [p for p, nm in zip(params, net.parameter_names) if nm.endswith("bias")]
    return k, b


def _pendulum_setup(sl):
    plant = sl.InvertedPendulum(**PEND)
    f = lambda z: G.pendulum(z, PEND["mass"], PEND["length"], PEND["friction"], PEND["dt"],
                             PEND["normalization"])
    K = np.array([[-0.7, -0.4]])
    Pq = np.diag([-0.1, -0.1, -0.1])
    return plant, f, K, Pq


def test_value_function_loop_matches_oracle(sl):
    """reinforcement_learning_pendulum.ipynb cells 7-20: V [64, 64, 1] (relu, relu, None) on
    r + 0.95 V(f(x, pi(x))) with the target held fixed, scaled L1 objective, SGD lr 0.005, batch 100."""
    plant, f, K, Pq = _pendulum_setup(sl)
    vf = sl.NeuralNetwork([64, 64, 1], ["relu", "relu", None], name="value_function", seed=11)
    policy, reward = sl.LinearSystem(K), sl.QuadraticFunction(Pq)
    gamma, scaling = 0.95, 1 / 0.3
    rng = np.random.default_rng(0)
    x0 = torch.tensor(rng.uniform(-1, 1, (100, 2)), device="cuda")
    vf.torch(x0)                                           # first call creates the variables
    assert [tuple(p.shape) for p in vf.parameters] == [(2, 64), (64,), (64, 64), (64,), (64, 1)]
    theta = _oracle_copy(vf)
    opt = torch.optim.SGD(vf.parameters, lr=0.005)
    opt_c = torch.optim.SGD(theta, lr=0.005)
    Kt, Pt = torch.tensor(K), torch.tensor(Pq)
    for step in range(30):
        xb = rng.uniform(-1, 1, (100, 2))
        x = torch.tensor(xb, device="cuda")
        z = torch.cat([x, policy.torch(x)], dim=1)
        target = (reward.torch(z) + gamma * vf.torch(plant.torch(z))).detach()
        resid = vf.torch(x) - target
        obj = scaling * torch.mean(torch.abs(resid))
        opt.zero_grad()
        obj.backward()
        opt.step()
        # oracle
        xc = torch.tensor(xb)
        zc = torch.cat([xc, xc @ Kt.T], dim=1)
        kc, bc = _split(vf, theta)
        with torch.no_grad():
            tgt = torch.sum((zc @ Pt) * zc, dim=1, keepdim=True) + gamma * G.mlp(f(zc), kc, bc, vf.nonlinearities)
        res_c = G.mlp(xc, kc, bc, vf.nonlinearities) - tgt
        obj_c = scaling * torch.mean(torch.abs(res_c))
        opt_c.zero_grad()
        obj_c.backward()
        opt_c.step()
        margin = min(float(res_c.detach().abs().min()),
                     _relu_margin([k.detach() for k in kc], [b.detach() for b in bc], vf.nonlinearities, xb, True))
        assert margin > 1e-12, "step %d: a ReLU pre-activation or L1 residual within 1e-12 of 0" % step
        _assert_params_close(vf, theta, step)


def test_policy_loop_matches_oracle(sl):
    """Cells 34-38 of the same notebook: policy [64, 64, 1] (relu, relu, None, no bias) through the
    frozen value network and the pendulum, objective -(1 - gamma)/r_max mean(r + gamma V(f(x, pi(x)))),
    SGD lr 0.6."""
    plant, f, K, Pq = _pendulum_setup(sl)
    vf = sl.NeuralNetwork([2, 64, 64, 1], ["relu", "relu", None], seed=12)
    rng = np.random.default_rng(1)
    vf.biases = [rng.normal(scale=0.1, size=64), rng.normal(scale=0.1, size=64)]
    pol = sl.NeuralNetwork([64, 64, 1], ["relu", "relu", None], use_bias=False, name="policy", seed=13)
    reward = sl.QuadraticFunction(Pq)
    gamma = 0.95
    scaling = (1 - gamma) / 0.2
    pol.evaluate_device(torch.zeros((1, 2), dtype=torch.float64, device="cuda"))
    theta = _oracle_copy(pol)
    vk, vb = _split(vf, _oracle_copy(vf))
    vk, vb = [k.detach() for k in vk], [b.detach() for b in vb]
    opt = torch.optim.SGD(pol.parameters, lr=0.6)
    opt_c = torch.optim.SGD(theta, lr=0.6)
    Pt = torch.tensor(Pq)
    for step in range(30):
        xb = rng.uniform(-1, 1, (100, 2))
        x = torch.tensor(xb, device="cuda")
        z = torch.cat([x, pol.torch(x)], dim=1)
        obj = -scaling * torch.mean(reward.torch(z) + gamma * vf.torch(plant.torch(z)))
        opt.zero_grad()
        obj.backward()
        opt.step()
        xc = torch.tensor(xb)
        uc = G.mlp(xc, theta, [], pol.nonlinearities, use_bias=False)
        zc = torch.cat([xc, uc], dim=1)
        obj_c = -scaling * torch.mean(torch.sum((zc @ Pt) * zc, dim=1, keepdim=True)
                                      + gamma * G.mlp(f(zc), vk, vb, vf.nonlinearities))
        opt_c.zero_grad()
        obj_c.backward()
        opt_c.step()
        margin = min(_relu_margin([t.detach() for t in theta], [], pol.nonlinearities, xb, False),
                     _relu_margin(vk, vb, vf.nonlinearities, f(zc).detach().numpy(), True))
        assert margin > 1e-12, "step %d: a ReLU pre-activation within 1e-12 of 0" % step
        _assert_params_close(pol, theta, step)
    assert all(p.grad is not None for p in pol.parameters)


def test_lyapunov_pretraining_and_classification_loop_matches_oracle(sl):
    """lyapunov_function_learning.ipynb cells 25-26 (L1 pre-training towards 0.1 |x|^2 on the r <= 0.1
    ball of the 251^2 grid, SGD lr 0.1, batch 1000, 20 steps), then 10 steps of the cell-30 objective
    (perceptron loss on ROA labels plus the Lagrangian decrease loss with V at x and at f(x))."""
    plant, f, K, _ = _pendulum_setup(sl)
    policy = sl.LinearSystem(K)
    net = sl.LyapunovNetwork(2, [64, 64, 64], ["tanh"] * 3, eps=1e-8, seed=21)
    V = lambda x, th: G.lyapunov_network(x, th, 2, net.output_dims, net.activations, net.eps)
    # the Lyapunov object of cells 19-20 (L_v = |grad V|_1) exists before training: its cached
    # descriptors must follow the in-place SGD steps
    cert = _Certification(sl, net, plant, policy, K, V)
    before = cert.run()
    assert before["safe_set"].sum() > cert.initial.sum()
    grid = sl.GridWorld([[-1, 1], [-1, 1]], 251)
    pts = grid.all_points
    level = pts[np.linalg.norm(pts, axis=1) <= 0.1]
    theta = _oracle_copy(net)
    opt = torch.optim.SGD(net.parameters, lr=0.1)
    opt_c = torch.optim.SGD(theta, lr=0.1)
    rng = np.random.default_rng(2)
    kinks = 0
    for step in range(20):
        xb = level[rng.integers(0, len(level), 1000)]
        x = torch.tensor(xb, device="cuda")
        res_g = net.torch(x) - 0.1 * torch.sum(x * x, dim=1, keepdim=True)
        obj = torch.mean(torch.abs(res_g))
        opt.zero_grad()
        obj.backward()
        opt.step()
        xc = torch.tensor(xb)
        res = V(xc, theta) - 0.1 * torch.sum(xc * xc, dim=1, keepdim=True)
        obj_c = torch.mean(torch.abs(res))
        opt_c.zero_grad()
        obj_c.backward()
        opt_c.step()
        # the origin is a grid point of the ball: V(0) = 0.1 |0|^2 = 0 exactly in both runs
        kinks += _assert_same_side(_cpu(res_g).numpy(), res.detach().numpy(), "L1 residuals", step)
        _assert_params_close(net, theta, step)
    Kt = torch.tensor(K)
    c_max, lam, eps = 0.05, 1.0, 1e-8
    for step in range(10):
        xb = pts[rng.integers(0, len(pts), 1000)]
        labels = (np.linalg.norm(xb, axis=1, keepdims=True) < 0.5).astype(np.float64)
        x = torch.tensor(xb, device="cuda")
        lab = torch.tensor(labels, device="cuda")
        z = torch.cat([x, policy.torch(x)], dim=1)
        vx, vfx = net.torch(x), net.torch(plant.torch(z))
        hinge_g, dv_g = -(2 * lab - 1) * (c_max - vx), vfx - vx
        loss = torch.clamp(hinge_g, min=0) + lam * lab * torch.clamp(dv_g, min=0) / (vx + eps).detach()
        obj = torch.mean(loss)
        opt.zero_grad()
        obj.backward()
        opt.step()
        xc, labc = torch.tensor(xb), torch.tensor(labels)
        zc = torch.cat([xc, xc @ Kt.T], dim=1)
        vxc, vfxc = V(xc, theta), V(f(zc), theta)
        hinge = -(2 * labc - 1) * (c_max - vxc)
        dv = vfxc - vxc
        loss_c = torch.clamp(hinge, min=0) + lam * labc * torch.clamp(dv, min=0) / (vxc + eps).detach()
        opt_c.zero_grad()
        torch.mean(loss_c).backward()
        opt_c.step()
        kinks += _assert_same_side(_cpu(hinge_g).numpy(), hinge.detach().numpy(), "hinge arguments", 20 + step)
        kinks += _assert_same_side(_cpu(dv_g).numpy(), dv.detach().numpy(), "decreases", 20 + step)
        _assert_params_close(net, theta, 20 + step)
    print("entries within 1e-12 of a kink (same side in both runs): %d" % kinks)
    # the trained network: fused forward equals the numpy oracle, L_V from gradient() equals autograd
    x = pts[::97]
    w = net.weights
    onet = O.LyapunovNetwork(2, net.output_dims, [np.tanh] * 3, w, eps=net.eps)
    assert_allclose(net(x), onet(x), rtol=1e-13, atol=1e-15)
    xt = torch.tensor(x, requires_grad=True)
    V(xt, [_cpu(p) for p in net.parameters]).sum().backward()
    _close(net.gradient(x), xt.grad.numpy())
    # update_values / update_safe_set on the same Lyapunov object now certify the trained network
    after = cert.run()
    assert not np.array_equal(after["values"], before["values"])
    assert after["c_max"] != before["c_max"] or not np.array_equal(after["safe_set"], before["safe_set"])


class _Certification(object):
    """``Lyapunov(grid, V, pendulum, L_f, L_v, tau, policy, initial set)`` with L_v = |dV/dx|_1, on the
    GPU (``LyapunovNetwork.gradient``) and in the oracle (autograd of the torch-CPU restatement at the
    network's current weights); ``run`` updates both and checks they agree."""

    def __init__(self, sl, net, plant, policy, K, V):
        self.net, self.V = net, V
        limits = [[-1., 1.], [-1., 1.]]
        self.grid_c = O.GridWorld(limits, 41)
        self.initial = np.linalg.norm(self.grid_c.all_points, axis=1) < 0.15
        self.tau, self.l_f = 0.002, 1.0
        self.oplant = O.InvertedPendulum(PEND["mass"], PEND["length"], PEND["friction"], PEND["dt"],
                                         PEND["normalization"])
        self.opolicy = O.LinearSystem((K,))
        lv = lambda x: np.sum(np.abs(net.gradient(x)), axis=1, keepdims=True)
        self.gpu = sl.Lyapunov(sl.GridWorld(limits, 41), net, plant, self.l_f, lv, self.tau, policy,
                               self.initial)

    def _lv_oracle(self, params):
        def lv(x):
            xt = torch.tensor(np.asarray(x, dtype=np.float64), requires_grad=True)
            self.V(xt, params).sum().backward()
            return np.sum(np.abs(xt.grad.numpy()), axis=1, keepdims=True)
        return lv

    def run(self):
        net = self.net
        onet = O.LyapunovNetwork(2, net.output_dims, [np.tanh] * 3, net.weights, eps=net.eps)
        cpu = O.Lyapunov(self.grid_c, onet, self.oplant, self.l_f,
                         self._lv_oracle([_cpu(p) for p in net.parameters]), self.tau, self.opolicy,
                         self.initial)
        gpu = self.gpu
        gpu.update_values()
        assert_allclose(gpu.values, cpu.values, rtol=1e-12, atol=1e-14)
        gpu.values = cpu.values                  # identical sort keys (tanh differs by an ulp)
        gpu.update_safe_set()
        cpu.update_safe_set()
        assert_array_equal(gpu.safe_set, cpu.safe_set)
        assert gpu.feed_dict[gpu.c_max] == cpu.c_max
        return {"values": np.array(cpu.values), "safe_set": np.array(cpu.safe_set), "c_max": cpu.c_max}


# ---------------------------------------------------------------- fused paths on the trained weights
def test_fused_sweep_and_rollout_see_trained_policy(sl):
    """Train the [32, 32, 1] policy of inverted_pendulum.ipynb cell 9 in place (one SGD step on a
    Lyapunov-decrease objective through the GP mean), then run update_safe_set and compute_roa on the
    same object: both match the oracle built from the new weights."""
    par = W.make_pendulum(num_points=24, M=50, tau_scale=1 / 64.)
    gpu, cpu = W.build_product(par), W.build_oracle(par)
    net = sl.NeuralNetwork([2, 32, 32, 1], ["relu", "relu", "tanh"], output_scale=0.8, seed=4)
    gpu.policy = net
    gpu.update_safe_set()                                # caches descriptors of the initial weights
    x = torch.tensor(np.random.default_rng(3).uniform(-0.5, 0.5, (256, 2)), device="cuda")
    opt = torch.optim.SGD(net.parameters, lr=0.05)
    mean, _ = gpu.dynamics.torch(torch.cat([x, net.torch(x)], dim=1))
    obj = torch.mean(gpu.lyapunov_function.torch(mean))
    before = [_cpu(p).clone() for p in net.parameters]
    w0, b0 = net.weights, net.biases
    opt.zero_grad()
    obj.backward()
    opt.step()
    assert any(not torch.equal(a, _cpu(b)) for a, b in zip(before, net.parameters))
    cpu.policy = O.NeuralNetwork([2, 32, 32, 1], [lambda v: np.maximum(v, 0.0)] * 2 + [np.tanh],
                                 net.weights, net.biases, output_scale=0.8)
    gpu.update_safe_set()
    cpu.update_safe_set()
    assert_array_equal(gpu.safe_set, cpu.safe_set)
    assert gpu.feed_dict[gpu.c_max] == cpu.c_max
    # the sweep's decrease bounds follow the new weights, far outside the GP's rounding
    states = cpu.discretization.all_points
    relu = [lambda v: np.maximum(v, 0.0)] * 2 + [np.tanh]
    stale = O.NeuralNetwork([2, 32, 32, 1], relu, w0, b0, output_scale=0.8)
    dec_new = cpu.v_decrease_bound(states, cpu.dynamics(states, cpu.policy(states))).ravel()
    dec_old = cpu.v_decrease_bound(states, cpu.dynamics(states, stale(states))).ravel()
    _, det = gpu.compute_negative(want_details=True)
    dec_g = det["decrease"].cpu().numpy().ravel()
    assert_allclose(dec_g, dec_new, rtol=1e-5, atol=1e-12)
    assert np.max(np.abs(dec_old - dec_new)) > 100 * np.max(np.abs(dec_g - dec_new))
    # closed loop x <- f(x, pi(x)) with the trained policy
    plant, f, _, _ = _pendulum_setup(sl)
    states = np.random.default_rng(4).uniform(-0.3, 0.3, (200, 2))
    loop = sl.ClosedLoop(plant, net)
    assert loop.fused
    roa_g, traj_g = sl.compute_roa(states, loop, horizon=20, tol=0.1, no_traj=False)
    kc, bc = net.weights, net.biases
    s = states.copy()
    traj = [s]
    for _ in range(19):
        u = O.NeuralNetwork([2, 32, 32, 1], [lambda v: np.maximum(v, 0.0)] * 2 + [np.tanh], kc, bc,
                            output_scale=0.8)(s)
        s = O.InvertedPendulum(PEND["mass"], PEND["length"], PEND["friction"], PEND["dt"],
                               PEND["normalization"])(s, u)
        traj.append(s)
    assert_allclose(traj_g[:, :, -1], traj[-1], rtol=1e-12, atol=1e-12)
    assert_array_equal(roa_g, np.linalg.norm(traj[-1], axis=1) <= 0.1)


def test_policy_gradient_through_gp_dynamics_matches_central_differences(sl):
    """inverted_pendulum.ipynb cell 9 shape: d future_values(states, lyapunov=...) / d (sampled policy
    parameters) for a [32, 32, 1] policy through the GP mean, against central differences."""
    par = W.make_pendulum(num_points=24, M=50, tau_scale=1 / 64.)
    gpu = W.build_product(par)
    net = sl.NeuralNetwork([2, 32, 32, 1], ["tanh", "tanh", "tanh"], output_scale=0.8, seed=9)
    grid = sl.GridWorld([[-1, 1], [-1, 1]], 15)
    vtab = sl.Triangulation(grid, -np.sum(grid.all_points ** 2, axis=1, keepdims=True), project=True)
    rl = sl.PolicyIteration(net, gpu.dynamics, sl.QuadraticFunction(-0.1 * np.eye(3)), vtab, gamma=0.9)
    states = torch.tensor(np.random.default_rng(6).uniform(-0.4, 0.4, (64, 2)), device="cuda")

    def objective():
        return rl.future_values(states, lyapunov=gpu).sum()

    objective().backward()
    rng = np.random.default_rng(0)
    checked = 0
    for p in net.parameters:
        flat = p.detach().view(-1)
        for j in rng.choice(flat.numel(), size=min(3, flat.numel()), replace=False):
            old = float(flat[j])
            h = 1e-6
            with torch.no_grad():
                flat[j] = old + h
            up = float(objective())
            with torch.no_grad():
                flat[j] = old - h
            down = float(objective())
            with torch.no_grad():
                flat[j] = old
            fd = (up - down) / (2 * h)
            g = float(p.grad.view(-1)[j])
            assert abs(g - fd) <= 1e-5 * max(abs(fd), 1e-3), (p.shape, j, g, fd)
            checked += 1
    assert checked >= 10
