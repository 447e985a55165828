"""How function objects enter torch's autograd graph: ``slb_function_columns`` (the COLUMNS rule of
``include/slb200.h``, which sizes every evaluation and VJP buffer), the one autograd node behind
``Function.torch`` on the CPU (driven by a torch-CPU function object with one trainable tensor), and, on the
GPU, every fusable object's gradients against the rule that object states."""
import numpy as np
import pytest
import torch

import safe_learning_b200 as sl
from safe_learning_b200 import _native as nat
from safe_learning_b200 import functions as F

T64 = torch.float64


# ---------------------------------------------------------------- slb_function_columns
# slb200.h (slb_sweep): out_dim, except 1 for QUADRATIC and LYAPUNOV_NN, 2 for PENDULUM, 4 for CARTPOLE, and
# 1 after NORM1 or MAXABS
KIND_COLUMNS = {nat.FN_QUADRATIC: 1, nat.FN_LYAPUNOV_NN: 1, nat.FN_PENDULUM: 2, nat.FN_CARTPOLE: 4}


@pytest.mark.parametrize("kind", [nat.FN_NONE, nat.FN_CONSTANT, nat.FN_LINEAR, nat.FN_QUADRATIC,
                                  nat.FN_TRIANGULATION, nat.FN_PENDULUM, nat.FN_CARTPOLE, nat.FN_LYAPUNOV_NN,
                                  nat.FN_MLP])
@pytest.mark.parametrize("flags", [0, nat.FLAG_NORM1, nat.FLAG_MAXABS, nat.FLAG_GRADIENT,
                                   nat.FLAG_SATURATE | nat.FLAG_ABS | nat.FLAG_NORM1 | nat.FLAG_SCALE])
def test_function_columns_follow_the_header_rule(kind, flags):
    d = nat.SlbFunction()
    d.kind, d.in_dim, d.out_dim, d.flags = kind, 3, 5, flags
    want = 1 if flags & (nat.FLAG_NORM1 | nat.FLAG_MAXABS) else KIND_COLUMNS.get(kind, 5)
    assert nat.load().slb_function_columns(d) == want


def test_function_columns_of_null_is_an_error():
    lib = nat.load()
    assert lib.slb_function_columns(None) == -1
    assert "null function" in nat.last_error()


# ---------------------------------------------------------------- the autograd node, on the CPU
class _Affine(F.DeterministicFunction):
    """``tanh(x) W^T + b`` in torch on the CPU, with ``b`` its trainable tensor; records the ``_vjp``
    requests."""

    def __init__(self, w, b):
        super().__init__("affine")
        self.w, self.b = w, b
        self.output_dim, self.input_dim = w.shape
        self.requests = []

    def evaluate_device(self, points):
        return torch.tanh(points) @ self.w.T + self.b.detach()

    def jacobian_device(self, points):
        return self.w * (1 - torch.tanh(points) ** 2).unsqueeze(1)

    def _trainable_tensors(self):
        return [self.b]

    def _vjp(self, points, grad_out, want_in, want_params):
        self.requests.append((want_in, want_params))
        gin, _ = super()._vjp(points, grad_out, want_in, False)
        return gin, ([grad_out.sum(dim=0)] if want_params else [])


def _case(seed=0, n=7):
    rng = np.random.default_rng(seed)
    fun = _Affine(torch.tensor(rng.normal(size=(2, 3))), torch.tensor(rng.normal(size=2), requires_grad=True))
    return fun, torch.tensor(rng.normal(size=(n, 3))), torch.tensor(rng.normal(size=(n, 2)))


def test_gradients_reach_the_points_and_the_tensor():
    fun, x, g = _case()
    x.requires_grad_(True)
    y = fun.torch(x)
    assert torch.equal(y.detach(), fun.evaluate_device(x.detach()))
    y.backward(g)
    assert fun.requests == [(True, True)]
    assert torch.equal(x.grad, torch.einsum("no,noi->ni", g, fun.jacobian_device(x.detach())))
    assert torch.equal(fun.b.grad, g.sum(dim=0))


def test_vjp_is_asked_only_for_what_is_needed():
    fun, x, g = _case(1)
    fun.torch(x).backward(g)                          # the points need no gradient
    assert fun.requests == [(False, True)] and fun.b.grad is not None
    fun.b.requires_grad_(False)
    fun.requests.clear()
    x.requires_grad_(True)
    fun.torch(x).backward(g)                          # the tensor needs none
    assert fun.requests == [(True, False)] and x.grad is not None


def test_write_to_the_tensor_between_forward_and_backward_raises():
    fun, x, g = _case(2)
    y = fun.torch(x)
    with torch.no_grad():
        fun.b.add_(1.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        y.backward(g)
    assert fun.requests == []


def test_second_derivative_raises():
    """Also without trainable tensors: the VJP rule holds the Jacobian constant, so a second derivative
    through it would be silently wrong."""
    for trainable in (True, False):
        fun, x, _ = _case(3)
        fun.b.requires_grad_(trainable)
        x.requires_grad_(True)
        (gx,) = torch.autograd.grad((fun.torch(x) ** 2).sum(), x, create_graph=True)
        with pytest.raises(RuntimeError, match="once_differentiable"):
            gx.sum().backward()


def test_saturation_passes_the_tensor_gradient_through_its_mask():
    fun, x, g = _case(4, n=40)
    sat = sl.Saturation(fun, -0.5, 0.5)
    sat.evaluate_device = lambda p: torch.clamp(fun.evaluate_device(p), -0.5, 0.5)   # the fused forward
    x.requires_grad_(True)
    sat.torch(x).backward(g)
    inner = fun.evaluate_device(x.detach())
    free = ((inner > -0.5) & (inner < 0.5)).to(T64)
    assert 0 < free.sum() < free.numel()
    assert fun.requests == [(False, True)]
    assert torch.equal(fun.b.grad, (g * free).sum(dim=0))
    assert torch.equal(x.grad, torch.einsum("no,noi->ni", g * free, fun.jacobian_device(x.detach())))


def test_wrappers_build_a_network_in_the_reference_convention():
    lazy = sl.NeuralNetwork([8, 1], ["relu", None])
    (-sl.Saturation(lazy, -1., 1.))._build(3)       # what torch() does with its points' width
    assert lazy.built and lazy.input_dim == 3 and len(lazy.parameters) == 3


# ---------------------------------------------------------------- on the GPU: each object's rule, written out
def _linear():
    return sl.LinearSystem(np.array([[0.3, -1.2, 0.5], [0.7, 0.1, -0.4]]))


def _mlp():
    return sl.NeuralNetwork([3, 16, 2], ["tanh", None], seed=1)


def _tri(project=True, leaf=True):
    grid = sl.GridWorld([[-1.0, 1.0], [-0.8, 1.2], [-1.0, 0.5]], [4, 5, 3])
    tri = sl.Triangulation(grid, np.random.default_rng(2).normal(size=(grid.nindex, 1)), project=project)
    if leaf:
        tri.vertex_values
    return tri


OBJECTS = {
    "linear": _linear,
    "quadratic": lambda: sl.QuadraticFunction(np.array([[1.0, 0.2, 0.0], [-0.3, 0.5, 0.1], [0.0, 0.4, 2.0]])),
    "constant": lambda: sl.ConstantFunction([0.5, -1.0], input_dim=3),
    "pendulum": lambda: sl.InvertedPendulum(0.15, 0.5, 0.1, normalization=([1.0, 2.0], [0.5])),
    "cartpole": lambda: sl.CartPole(0.175, 1.732, 0.28, 0.01, 0.01),
    "tri": lambda: _tri(False, False),
    "tri_project": lambda: _tri(True, False),
    "tri_leaf": lambda: _tri(False, True),
    "tri_project_leaf": lambda: _tri(True, True),
    "mlp": _mlp,
    "lyapunov": lambda: sl.LyapunovNetwork(3, [3, 8], ["tanh", "tanh"], seed=1),
    "saturated_unbuilt_mlp": lambda: sl.Saturation(sl.NeuralNetwork([16, 1], ["tanh", None], seed=4), -0.3, 0.3),
}
for _name, _base in (("linear", _linear), ("mlp", _mlp), ("tri_leaf", _tri)):
    OBJECTS["saturation_" + _name] = lambda b=_base: sl.Saturation(b(), -0.3, 0.3)
    OBJECTS["abs_" + _name] = lambda b=_base: sl.AbsFunction(b())
    OBJECTS["norm1_" + _name] = lambda b=_base: sl.Norm1Function(b())
    OBJECTS["scaled_" + _name] = lambda b=_base: sl.ScaledFunction(b(), -1.7)


def _tensor_rule(fun, x, g):
    """The trainable tensors' gradients for the cotangent g of fun(x)."""
    if isinstance(fun, F._PostOp):
        return _tensor_rule(fun.fun, x, fun._inner_cotangent(fun.fun.evaluate_device(x), g))
    if isinstance(fun, F._TrainableNetwork):
        return fun._grads_like(F._function_vjp(fun, x, g, False, fun._packed_device().numel())[1],
                               fun.parameters)
    if isinstance(fun, sl.Triangulation) and fun._trainable_tensors():
        table = fun.vertex_values
        return [F._function_vjp(fun, x, g, want_in=False, nparams=table.numel())[1].view(table.shape)]
    return []


def _rule(fun, x, g):
    """(the points' gradient, the trainable tensors' gradients): one slb_function_vjp call for the plants and
    the networks, otherwise grad_out @ jacobian_device and _tensor_rule."""
    if isinstance(fun, (sl.InvertedPendulum, sl.CartPole)):
        return F._function_vjp(fun, x, g)[0], []
    if isinstance(fun, F._TrainableNetwork):
        gin, gflat, _ = F._function_vjp(fun, x, g, True, fun._packed_device().numel())
        return gin, fun._grads_like(gflat, fun.parameters)
    return torch.einsum("no,noi->ni", g, fun.jacobian_device(x)), _tensor_rule(fun, x, g)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(OBJECTS))
def test_torch_gradients_are_each_objects_rule(name):
    fun = OBJECTS[name]()
    rng = np.random.default_rng(5)
    x = torch.tensor(rng.uniform(-1.3, 1.3, (300, fun.input_dim or 3)), device="cuda")
    g = torch.tensor(rng.normal(size=(300, fun.output_dim)), device="cuda")
    xg = x.clone().requires_grad_(True)
    y = fun.torch(xg)
    y.backward(g)
    tensors = fun._trainable_tensors()
    assert torch.equal(y.detach(), fun.evaluate_device(x))
    gin, grads = _rule(fun, x, g)
    assert torch.equal(xg.grad, gin)
    assert len(grads) == len(tensors)
    assert bool(tensors) == any(k in name for k in ("mlp", "lyapunov", "leaf"))
    for t, want in zip(tensors, grads):
        assert torch.equal(t.grad, want)
    if name == "saturated_unbuilt_mlp":
        assert fun.fun.built and fun.input_dim == 3 and len(tensors) == 3


@pytest.mark.gpu
def test_triangulation_gradient_has_no_point_gradient():
    """TriangulationGradient states no Jacobian: its backward raises, as the einsum rule does."""
    fun = sl.TriangulationGradient(_tri())
    x = torch.tensor(np.random.default_rng(6).uniform(-1.0, 1.0, (50, 3)), device="cuda")
    g = torch.ones((50, 3), dtype=T64, device="cuda")
    assert fun._trainable_tensors() == []
    xg = x.clone().requires_grad_(True)
    y = fun.torch(xg)
    assert torch.equal(y.detach(), fun.evaluate_device(x))
    with pytest.raises(NotImplementedError, match="no device Jacobian"):
        y.backward(g)
    with pytest.raises(NotImplementedError, match="no device Jacobian"):
        _rule(fun, x, g)
