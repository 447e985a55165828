"""Function objects of the region-of-attraction path, as parameter containers for libslb200.

API surface follows ``safe_learning/functions.py`` of the reference (class names, constructor
arguments, attributes); cited line numbers are relative to the upstream safe_learning sources.  Where the
reference's objects emit TF1 graph nodes, these objects (a) describe themselves to the CUDA
kernels through an ``slb_function`` / ``slb_gp_stack`` descriptor and (b) evaluate eagerly on
the GPU when called with numpy arrays, returning numpy arrays.  There is no CPU path.

gpflow is replaced by small gpflow-free containers: the ``kernels`` (RBF, Matern12/32/52, Linear,
Constant, White, sums and products, ``active_dims``; arithmetic of ``gpflow==0.4.0``
``kernels``) and ``GPRCached`` (``functions.py:357-458``).
"""

from __future__ import annotations

import collections
import hashlib
import itertools
import weakref

import numpy as np
import scipy.signal
import scipy.sparse
import scipy.spatial
import torch

from . import _device as dev
from . import _native as nat
from .configuration import Configuration

config = Configuration()

__all__ = ["DimensionError", "GridWorld", "Function", "DeterministicFunction",
           "UncertainFunction", "ConstantFunction", "LinearSystem", "QuadraticFunction",
           "Saturation", "AbsFunction", "Norm1Function", "MaxAbsFunction", "ScaledFunction",
           "Triangulation", "TriangulationGradient", "PiecewiseConstant", "NetworkGradient",
           "Kernel", "RBF", "Matern12", "Matern32", "Matern52", "Linear", "Constant", "Bias",
           "White", "Sum", "Add", "Product", "Prod", "kernels", "Likelihood", "GPRCached", "GPR",
           "GaussianProcess", "FunctionStack", "PosteriorMean",
           "InvertedPendulum", "CartPole", "VanDerPol", "LyapunovNetwork", "NeuralNetwork",
           "concatenate_inputs"]


class DimensionError(Exception):
    """``functions.py:575-576``."""


def concatenate_inputs(inputs):
    """Column-concatenate call arguments ([x, u] layout; ``utilities.py:123-159``)."""
    cols = [np.atleast_2d(np.asarray(a, dtype=np.float64)) for a in inputs]
    return cols[0] if len(cols) == 1 else np.hstack(cols)


# =============================================================================== GridWorld
class GridWorld(object):
    """Regular grid (``functions.py:579-817``).

    The kernels never read coordinates from memory: ``descriptor()`` carries
    offset / unit_maxes / num_points and every thread rebuilds ``ijk * unit_maxes + offset``
    (``:731``) from its flat index.  The host-side helpers below are vectorised numpy index
    arithmetic (not a compute path).
    """

    def __init__(self, limits, num_points):
        self.limits = np.atleast_2d(limits).astype(np.float64)
        npts = np.broadcast_to(num_points, len(self.limits))
        self.num_points = npts.astype(np.int64, copy=True)
        if np.any(self.num_points < 2):
            raise DimensionError("There must be at least 2 points in each dimension.")
        if len(self.limits) > nat.SLB_MAX_DIM:
            raise DimensionError("at most %d grid dimensions are supported" % nat.SLB_MAX_DIM)
        self.offset = self.limits[:, 0]
        self.unit_maxes = (self.limits[:, 1] - self.offset) / (self.num_points - 1)
        self.offset_limits = np.stack((np.zeros(len(self.limits)),
                                       self.limits[:, 1] - self.offset), axis=1)
        self.discrete_points = [np.linspace(lo, hi, n, dtype=np.float64)
                                for (lo, hi), n in zip(self.limits, self.num_points)]
        self.nrectangles = int(np.prod(self.num_points - 1))
        self.nindex = int(np.prod(self.num_points))
        self.ndim = len(self.limits)
        self._all_points = None
        self._points_dev = None

    def __len__(self):
        return self.nindex

    # ---- descriptor for the kernels
    def descriptor(self, need_points=False):
        g = nat.SlbGrid()
        g.ndim = self.ndim
        g.nindex = self.nindex
        for c in range(self.ndim):
            g.num_points[c] = int(self.num_points[c])
            g.offset[c] = float(self.offset[c])
            g.unit_maxes[c] = float(self.unit_maxes[c])
            g.upper[c] = float(self.limits[c, 1])
        if need_points:
            if self._points_dev is None:
                self._points_dev = dev.to_device(np.concatenate(self.discrete_points))
            g.discrete_points = self._points_dev.data_ptr()
        return g

    # ---- reference API
    @property
    def all_points(self):
        """All grid points, C order, last dimension fastest (``:622-638``).  Host array; the
        sweeps do not use it."""
        if self._all_points is None:
            mesh = np.meshgrid(*self.discrete_points, indexing="ij")
            self._all_points = np.column_stack([m.ravel() for m in mesh])
        return self._all_points

    def sample_continuous(self, num_samples):
        rand = np.random.uniform(0, 1, size=(num_samples, self.ndim))
        return rand * np.diff(self.limits, axis=1).T + self.offset

    def sample_discrete(self, num_samples, replace=False):
        idx = np.random.choice(self.nindex, size=num_samples, replace=replace)
        return self.index_to_state(idx)

    def _check_dimensions(self, states):
        if not states.shape[1] == self.ndim:
            raise DimensionError("the input argument has the wrong dimensions.")

    def _center_states(self, states, clip=True):
        eps = np.finfo(np.float64).eps
        states = np.atleast_2d(states).astype(np.float64) - self.offset[None, :]
        if clip:
            np.clip(states, self.offset_limits[:, 0] + 2 * eps,
                    self.offset_limits[:, 1] - 2 * eps, out=states)
        return states

    def index_to_state(self, indices):
        ijk = np.stack(np.unravel_index(np.atleast_1d(indices), self.num_points), axis=1)
        return ijk.astype(np.float64) * self.unit_maxes + self.offset

    def state_to_index(self, states):
        states = np.atleast_2d(states)
        self._check_dimensions(states)
        clipped = np.clip(states, self.limits[:, 0], self.limits[:, 1])
        ijk = np.rint((clipped - self.offset) * (1. / self.unit_maxes)).astype(np.int32)
        return np.ravel_multi_index(ijk.T, self.num_points)

    def state_to_rectangle(self, states):
        cells = []
        for i, (pts, n) in enumerate(zip(self.discrete_points, self.num_points)):
            cells.append(np.clip(np.digitize(states[:, i], pts) - 1, 0, n - 2))
        return np.ravel_multi_index(cells, self.num_points - 1)

    def rectangle_to_state(self, rectangles):
        ijk = np.stack(np.unravel_index(np.atleast_1d(rectangles), self.num_points - 1), axis=1)
        return ijk.astype(np.float64) * self.unit_maxes + self.offset

    def rectangle_corner_index(self, rectangles):
        ijk = np.vstack(np.unravel_index(rectangles, self.num_points - 1))
        return np.ravel_multi_index(np.atleast_2d(ijk), self.num_points)


# =============================================================================== Function base
class Function(object):
    """Base class (``functions.py:31-122``): ``fun(*inputs)`` concatenates the inputs and
    evaluates on the GPU; ``+``/``*``/``-`` with scalars build fused wrappers."""

    input_dim = None
    output_dim = None

    def __init__(self, name="function"):
        self.name = name
        self.feed_dict = {}

    # descriptor protocol --------------------------------------------------------------
    def descriptor(self):
        """Return an ``slb_function``; device buffers it points to are owned by ``self``."""
        raise NotImplementedError("%s cannot be fused into the CUDA kernels"
                                  % type(self).__name__)

    @property
    def parameters(self):
        return []

    @property
    def version(self):
        """Changes whenever the descriptor would change (callers cache descriptors on it).
        Plain parameter containers are immutable after construction."""
        return 0

    # eager evaluation -----------------------------------------------------------------
    def __call__(self, *inputs):
        return self.evaluate_device(concatenate_inputs(inputs)).cpu().numpy()

    def evaluate_device(self, points):
        """points: numpy [n, in] or device tensor -> device tensor [n, out]."""
        lib = nat.load()
        desc = self.descriptor()
        pts = dev.to_device(points)
        if pts.dim() != 2 or pts.shape[1] != desc.in_dim:
            raise DimensionError("%s expects %d input columns, got shape %s"
                                 % (type(self).__name__, desc.in_dim, tuple(pts.shape)))
        out = dev.empty((pts.shape[0], lib.slb_function_columns(desc)))
        nat.check(lib.slb_eval_function(dev.stream(), desc, pts.data_ptr(), pts.shape[0],
                                        out.data_ptr()), "slb_eval_function")
        return out

    # differentiable application (torch autograd) --------------------------------------------
    def jacobian_device(self, points):
        """d out / d in at device points [n, in] -> device tensor [n, out, in] (the reference gets
        these from ``tf.gradients``; here every fusable object states its own)."""
        raise NotImplementedError("%s has no device Jacobian" % type(self).__name__)

    def torch(self, points):
        """``fun(points)`` on a device tensor [n, in] as one node of torch's autograd graph with
        inputs (points, ``_trainable_tensors()``): forward = the fused CUDA evaluation, backward =
        one ``_vjp`` call (``PolicyIteration.future_values`` with tensors,
        ``reinforcement_learning.py:65-114`` under ``tf.gradients`` in
        ``examples/inverted_pendulum.ipynb`` cell 17).  The backward is not differentiable itself:
        a second derivative raises."""
        if points.dim() == 2:
            self._build(points.shape[1])
        return _FusedApply.apply(points, self, *self._trainable_tensors())

    # the same forward as a torch expression of the points, differentiated instead of ``_vjp`` when a
    # backward runs with create_graph=True; None: a second derivative raises
    _torch_expression = None

    def _forward_device(self, points):
        """The forward of ``torch``'s node on contiguous device points."""
        return self.evaluate_device(points)

    def _build(self, input_dim):
        """Create whatever depends on the input width before ``torch`` collects the trainable
        tensors (a network in the reference's convention); nothing here."""

    def _trainable_tensors(self):
        """The leaf tensors ``torch(points)`` differentiates besides the points (none here)."""
        return []

    def _vjp(self, points, grad_out, want_in, want_params):
        """For the cotangent ``grad_out`` [n, out] of ``fun(points)``: (the points' gradient [n, in]
        if ``want_in`` else None, one gradient per ``_trainable_tensors()`` if ``want_params`` else
        []).  Here ``grad_out @ jacobian_device(points)`` and no tensors."""
        gin = torch.einsum("no,noi->ni", grad_out, self.jacobian_device(points)) if want_in else None
        return gin, []

    def _param_vjp(self, points, grad_out):
        """Gradients of ``sum(grad_out * fun(points))`` for each of ``_trainable_tensors()``."""
        return self._vjp(points, grad_out, False, True)[1]

    # algebra (``functions.py:112-122``) --------------------------------------------------
    def __neg__(self):
        return ScaledFunction(self, -1.0)

    def __mul__(self, other):
        if np.isscalar(other):
            return ScaledFunction(self, float(other))
        raise NotImplementedError("only multiplication by a scalar is fused on the GPU")

    __rmul__ = __mul__

    def __abs__(self):
        return AbsFunction(self)

    def __add__(self, other):
        raise NotImplementedError("AddedFunction (functions.py:125-160) is outside the fused "
                                  "hot path of this build")


class _FusedApply(torch.autograd.Function):
    """Fused CUDA evaluation of a Function object inside torch's autograd graph, with the object's
    trainable tensors as inputs: the one node behind ``Function.torch``.  An object whose forward
    returns a tuple (the GP posterior: mean and beta * sigma) gives one node with several outputs; its
    ``_vjp`` receives a tuple of cotangents, None for an output that does not reach the loss."""

    @staticmethod
    def forward(ctx, points, fun, *tensors):
        ctx.fun = fun
        if fun._torch_expression is not None:
            # the points themselves: a backward with create_graph differentiates the torch expression
            # on them, which needs their place in the graph
            ctx.save_for_backward(points, *tensors)
            ctx.set_materialize_grads(False)
            return fun._forward_device(points.detach().contiguous())
        points = points.detach().contiguous()
        ctx.save_for_backward(points, *tensors)      # torch refuses backward after an in-place update
        return fun._forward_device(points)

    @staticmethod
    def backward(ctx, *grad_outs):
        if torch.is_grad_enabled() and ctx.fun._torch_expression is not None:
            # create_graph=True through an object that states its forward in torch operations: the
            # first derivative as a graph, so that a second derivative exists
            points, outs = ctx.saved_tensors[0], ctx.fun._torch_expression(ctx.saved_tensors[0])
            outs = outs if isinstance(outs, tuple) else (outs,)
            used = [(o, g) for o, g in zip(outs, grad_outs) if g is not None and o.requires_grad]
            gin = None
            if used:
                (gin,) = torch.autograd.grad([o for o, _ in used], points, [g for _, g in used],
                                             create_graph=True, allow_unused=True)
            if gin is None:
                gin = torch.zeros_like(points)
            return (gin, None) + (None,) * (len(ctx.saved_tensors) - 1)
        return _FusedApply._backward_once(ctx, *grad_outs)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def _backward_once(ctx, *grad_outs):
        # the VJPs are not differentiable themselves: double backward raises instead of treating the
        # gradient as a constant
        points, ntensors = ctx.saved_tensors[0], len(ctx.saved_tensors) - 1
        if len(grad_outs) == 1:
            grad_out = grad_outs[0].contiguous()
        else:
            grad_out = tuple(None if g is None else g.contiguous() for g in grad_outs)
        gin, grads = ctx.fun._vjp(points, grad_out, ctx.needs_input_grad[0], any(ctx.needs_input_grad[2:]))
        return (gin, None) + tuple(grads or [None] * ntensors)


def _function_vjp(fun, points, grad_out, want_in=True, nparams=0, want_out=False):
    """One ``slb_function_vjp`` call: (grad_in [n, in] or None, grad_params [nparams] or None,
    recomputed forward [n, out] or None), device tensors."""
    lib = nat.load()
    desc = fun.descriptor()
    pts = dev.to_device(points)
    n = pts.shape[0]
    ncols = lib.slb_function_columns(desc)
    gout = dev.to_device(grad_out).reshape(n, ncols).contiguous()
    gin = dev.empty((n, desc.in_dim)) if want_in else None
    gpar = dev.empty((nparams,)) if nparams else None
    out = dev.empty((n, ncols)) if want_out else None
    ws = None
    if gpar is not None:
        size = lib.slb_function_vjp_workspace(desc, n)
        if size < 0:
            raise nat.NativeLibraryError("slb_function_vjp_workspace: %s" % nat.last_error())
        ws = torch.empty(size, dtype=torch.uint8, device=pts.device) if size else None
    nat.check(lib.slb_function_vjp(dev.stream(), desc, pts.data_ptr(), n, gout.data_ptr(), dev.ptr(gin),
                                   dev.ptr(gpar), dev.ptr(out), dev.ptr(ws)), "slb_function_vjp")
    return gin, gpar, out


def _unit_vjp_jacobian(fun, points):
    """[n, out, in] from out_dim VJPs with unit cotangents."""
    pts = dev.to_device(points)
    n, nout = pts.shape[0], fun.output_dim
    rows = []
    for o in range(nout):
        cot = dev.zeros((n, nout))
        cot[:, o] = 1.0
        rows.append(_function_vjp(fun, pts, cot)[0])
    return torch.stack(rows, dim=1)


class DeterministicFunction(Function):
    """``functions.py:233-238``."""


class UncertainFunction(Function):
    """``functions.py:202-230``."""

    def to_mean_function(self):
        """A callable returning only the first output, ``lambda *points: self(*points)[0]``
        (``functions.py:209-230``); ``GaussianProcess`` and ``FunctionStack`` return a fused
        ``PosteriorMean`` instead."""
        return lambda *points: self(*points)[0]


class ConstantFunction(DeterministicFunction):
    """``functions.py:241-251``."""

    def __init__(self, constant, input_dim=1, name="constant_function"):
        super().__init__(name)
        self.constant = np.atleast_1d(np.asarray(constant, dtype=np.float64)).ravel()
        self.input_dim, self.output_dim = input_dim, len(self.constant)

    def descriptor(self):
        d = nat.SlbFunction()
        d.kind, d.in_dim, d.out_dim = nat.FN_CONSTANT, self.input_dim, self.output_dim
        for i, v in enumerate(self.constant):
            d.cparams[i] = float(v)
        return d

    def jacobian_device(self, points):
        return dev.zeros((points.shape[0], self.output_dim, self.input_dim))


class LinearSystem(DeterministicFunction):
    """``y = [x, u] A^T`` (``functions.py:1546-1583``)."""

    def __init__(self, matrices, name="linear_system"):
        super().__init__(name)
        if isinstance(matrices, np.ndarray):
            matrices = (matrices,)
        self.matrix = np.hstack([np.atleast_2d(m).astype(np.float64) for m in matrices])
        self.output_dim, self.input_dim = self.matrix.shape
        self._matrix_dev = None

    def descriptor(self):
        if self._matrix_dev is None:
            self._matrix_dev = dev.to_device(self.matrix)
        d = nat.SlbFunction()
        d.kind, d.in_dim, d.out_dim = nat.FN_LINEAR, self.input_dim, self.output_dim
        d.matrix = self._matrix_dev.data_ptr()
        return d

    def jacobian_device(self, points):
        self.descriptor()
        return self._matrix_dev.unsqueeze(0).expand(points.shape[0], -1, -1)


class QuadraticFunction(DeterministicFunction):
    """``sum((x P) * x)`` with P as given, not symmetrised (``functions.py:1513-1543``)."""

    def __init__(self, matrix, name="quadratic"):
        super().__init__(name)
        self.matrix = np.atleast_2d(matrix).astype(np.float64)
        self.ndim = self.matrix.shape[0]
        self.input_dim, self.output_dim = self.ndim, 1
        self._matrix_dev = None

    def descriptor(self):
        if self._matrix_dev is None:
            self._matrix_dev = dev.to_device(self.matrix)
        d = nat.SlbFunction()
        d.kind, d.in_dim, d.out_dim = nat.FN_QUADRATIC, self.ndim, 1
        d.matrix = self._matrix_dev.data_ptr()
        return d

    def gradient(self, points=None):
        """``x (P + P^T)`` as a fusable LinearSystem (``:1541-1543``); evaluated when points
        are given."""
        grad = LinearSystem((self.matrix + self.matrix.T).T)
        return grad if points is None else grad(points)

    def jacobian_device(self, points):
        self.descriptor()
        sym = self._matrix_dev + self._matrix_dev.T
        return (points @ sym).unsqueeze(1)                          # x (P + P^T)


class _PostOp(DeterministicFunction):
    """A post-operation fused onto a wrapped function's descriptor.  The kernels apply
    saturate -> abs -> norm1 -> scale in that order (``slb200.h``), so wrappers must be
    nested in that order (``MaxAbsFunction`` takes the place of norm1)."""

    _order = 0

    def __init__(self, fun, name):
        super().__init__(name)
        if not isinstance(fun, Function):
            raise TypeError("%s wraps a Function object, got %r" % (type(self).__name__, fun))
        inner = getattr(fun, "_order", 0)
        if inner >= self._order:
            raise NotImplementedError(
                "%s around %s: post-operations fuse only in the order "
                "saturate -> abs -> norm1 -> scale" % (type(self).__name__, type(fun).__name__))
        self.fun = fun

    @property
    def input_dim(self):
        # read through, so that a wrapped network in the reference's convention reports the width
        # its first evaluation gives it
        return self.fun.input_dim

    @property
    def parameters(self):
        return self.fun.parameters

    @property
    def version(self):
        return (id(self.fun), self.fun.version, getattr(self, "lower", None),
                getattr(self, "upper", None), getattr(self, "factor", None))

    def _inner_cotangent(self, inner, grad_out):
        """The cotangent of the wrapped function's output ``inner`` [n, out] for the cotangent
        ``grad_out`` of this wrapper's output (the rule of ``jacobian_device``)."""
        raise NotImplementedError("%s does not pass gradients to the wrapped function's parameters"
                                  % type(self).__name__)

    def _build(self, input_dim):
        self.fun._build(input_dim)

    def _trainable_tensors(self):
        return self.fun._trainable_tensors()

    def _vjp(self, points, grad_out, want_in, want_params):
        """The points' gradient from this wrapper's ``jacobian_device``; the wrapped object's tensors'
        gradients are its VJP of the cotangent mapped through this wrapper."""
        gin, grads = super()._vjp(points, grad_out, want_in, False)
        if want_params:
            inner = self.fun.evaluate_device(points)
            grads = self.fun._param_vjp(points, self._inner_cotangent(inner, grad_out))
        return gin, grads


class Saturation(_PostOp):
    """``min(max(fun(x), lower), upper)`` (``functions.py:310-354``)."""

    _order = 1

    def __init__(self, fun, lower, upper, name="saturation"):
        super().__init__(fun, name)
        self.lower, self.upper = float(lower), float(upper)
        self.output_dim = fun.output_dim

    def descriptor(self):
        d = self.fun.descriptor()
        d.flags |= nat.FLAG_SATURATE
        d.lower, d.upper = self.lower, self.upper
        return d

    def _free(self, inner):
        # strictly inside the bounds; tf.clip_by_value also passes the gradient at equality (DESIGN.md
        # §3.11)
        return ((inner > self.lower) & (inner < self.upper)).to(torch.float64)

    def _inner_cotangent(self, inner, grad_out):
        return grad_out * self._free(inner)

    def jacobian_device(self, points):
        inner = self.fun.evaluate_device(points)
        return self.fun.jacobian_device(points) * self._free(inner).unsqueeze(2)


class AbsFunction(_PostOp):
    """``|fun(x)|`` element-wise -- the per-dimension Lipschitz lambda
    ``tf.abs(grad_lyapunov_function(x))`` of ``examples/adaptive_safety_verification.ipynb``
    cell 17, as a fusable object."""

    _order = 2

    def __init__(self, fun, name="abs"):
        super().__init__(fun, name)
        self.output_dim = fun.output_dim

    def descriptor(self):
        d = self.fun.descriptor()
        d.flags |= nat.FLAG_ABS
        return d

    def _inner_cotangent(self, inner, grad_out):
        return grad_out * torch.sign(inner)

    def jacobian_device(self, points):
        sign = torch.sign(self.fun.evaluate_device(points))
        return self.fun.jacobian_device(points) * sign.unsqueeze(2)


class Norm1Function(_PostOp):
    """``tf.norm(fun(x), ord=1, axis=1, keepdims=True)`` (same notebook cell)."""

    _order = 3

    def __init__(self, fun, name="norm1"):
        super().__init__(fun, name)
        self.output_dim = 1

    def descriptor(self):
        d = self.fun.descriptor()
        d.flags |= nat.FLAG_NORM1
        return d

    def _inner_cotangent(self, inner, grad_out):
        return grad_out * torch.sign(inner)                          # [n, 1] against [n, out]

    def jacobian_device(self, points):
        sign = torch.sign(self.fun.evaluate_device(points))
        return (self.fun.jacobian_device(points) * sign.unsqueeze(2)).sum(dim=1, keepdim=True)


class MaxAbsFunction(_PostOp):
    """``tf.reduce_max(tf.abs(fun(x)), axis=1, keepdims=True)`` -- the Lipschitz lambda of
    ``examples/inverted_pendulum.ipynb`` cell 14 (around ``value_function.gradient``), as a
    fusable object."""

    _order = 3

    def __init__(self, fun, name="maxabs"):
        super().__init__(fun, name)
        self.output_dim = 1

    def descriptor(self):
        d = self.fun.descriptor()
        d.flags |= nat.FLAG_MAXABS
        return d


class ScaledFunction(_PostOp):
    """``fun * c`` / ``-fun`` (``MultipliedFunction`` with a constant, ``functions.py:163-199``)."""

    _order = 4

    def __init__(self, fun, factor, name="scaled"):
        super().__init__(fun, name)
        self.factor = float(factor)
        self.output_dim = fun.output_dim

    def __getattr__(self, item):          # e.g. (-value_function).discretization
        if item in ("fun", "factor"):
            raise AttributeError(item)
        return getattr(self.fun, item)

    def descriptor(self):
        d = self.fun.descriptor()
        d.flags |= nat.FLAG_SCALE
        d.out_scale = self.factor
        return d

    def _inner_cotangent(self, inner, grad_out):
        return grad_out * self.factor

    def jacobian_device(self, points):
        return self.fun.jacobian_device(points) * self.factor


# =============================================================================== Triangulation
class _Delaunay1D(object):
    """Two-point stand-in for scipy's Delaunay in 1-D (``functions.py:935-978``)."""

    def __init__(self, points):
        self.points = points
        self.nsimplex = 1
        self.simplices = np.array([[0, 1]])


class _TriangulationTables(object):
    """Host-side tables of ``_Triangulation`` (``functions.py:1002-1101``): the unit
    hyper-rectangle is triangulated once by Qhull; the kernels take the resulting
    ``unit_simplices`` / ``hyperplanes`` instead of assuming a particular split."""

    def __init__(self, discretization, project=False, owner=None):
        self.discretization = disc = discretization
        self.input_dim = disc.ndim
        self.project = project
        self._owner = weakref.ref(owner) if owner is not None else None
        if disc.ndim == 1:
            self.triangulation = _Delaunay1D(np.array([[0.0], [disc.unit_maxes[0]]]))
        else:
            corners = np.array(list(itertools.product(*np.diag(disc.unit_maxes))))
            self.triangulation = scipy.spatial.Delaunay(corners)
        mapping = disc.state_to_index(np.atleast_2d(self.triangulation.points) + disc.offset)
        self.unit_simplices = mapping[np.asarray(self.triangulation.simplices)].astype(np.int64)
        self.nsimplex_unit = int(self.triangulation.nsimplex)
        self.nsimplex = self.nsimplex_unit * disc.nrectangles
        self.hyperplanes = np.empty((self.nsimplex_unit, disc.ndim, disc.ndim))
        for i, simplex in enumerate(self.unit_simplices):
            pts = disc.index_to_state(simplex)
            self.hyperplanes[i] = np.linalg.inv(pts[1:] - pts[:1])
        # Queries clipped in every dimension land on a unit-cell corner shared by several
        # simplices; which one Qhull's walk returns decides the (discontinuous) extrapolation
        # of a non-projected query, so ask Qhull once per corner pattern (functions.py:1120-1124).
        self.corner_simplex = np.zeros(2 ** disc.ndim, dtype=np.int32)
        if disc.ndim > 1:
            eps = np.finfo(np.float64).eps
            lo = disc.offset_limits[:, 0] + 2 * eps
            hi = disc.offset_limits[:, 1] - 2 * eps
            for pattern in range(2 ** disc.ndim):
                bits = np.array([(pattern >> c) & 1 for c in range(disc.ndim)], dtype=bool)
                unit = np.where(bits, hi, lo) % disc.unit_maxes
                self.corner_simplex[pattern] = int(self.triangulation.find_simplex(unit[None, :])[0])

    @property
    def limits(self):
        return self.discretization.limits

    @property
    def nindex(self):
        return self.discretization.nindex

    def parameter_derivative(self, points):
        """``_Triangulation.parameter_derivative`` (``functions.py:1228-1259``): the sparse [n, nindex]
        matrix B with ``tri(points) = B @ vertex_values``, in the reference's layout (rows
        ``repeat(arange(n), d + 1)``, cols the simplex vertices of each point, data the barycentric
        weights).  The rows are the forward evaluation's, computed on the device
        (``slb_triangulation_rows``)."""
        owner = self._owner() if self._owner is not None else None
        if owner is None:
            raise ValueError("parameter_derivative needs the Triangulation these tables belong to")
        lib = nat.load()
        desc = owner.descriptor()
        pts = dev.to_device(np.atleast_2d(np.asarray(points, dtype=np.float64)))
        if pts.shape[1] != self.input_dim:
            raise DimensionError("parameter_derivative expects %d input columns, got shape %s"
                                 % (self.input_dim, tuple(pts.shape)))
        n, nsimp = pts.shape[0], self.input_dim + 1
        cols = dev.empty((n, nsimp), torch.int64)
        weights = dev.empty((n, nsimp))
        nat.check(lib.slb_triangulation_rows(dev.stream(), desc, pts.data_ptr(), n, cols.data_ptr(),
                                             weights.data_ptr()), "slb_triangulation_rows")
        rows = np.repeat(np.arange(n), nsimp)
        return scipy.sparse.coo_matrix((weights.cpu().numpy().ravel(), (rows, cols.cpu().numpy().ravel())),
                                       shape=(n, self.nindex))


class _VertexTable(object):
    """The device vertex table [nindex, out] of ``Triangulation`` and ``PiecewiseConstant``: one buffer
    (``_param_dev``) that the descriptor points at, one writer (``_store``) and one trainable leaf.

    ``vertex_values`` hands out that buffer as a float64 leaf tensor with ``requires_grad``, for
    ``torch.optim``: from then on every writer (the ``parameters`` setter, ``value_iteration``,
    ``optimize_value_function``, ``discrete_policy_optimization``) copies into it in place, so the
    leaf, the descriptor and the optimizer keep seeing one tensor, and the version follows its
    in-place updates."""

    _param_dev = None
    _version = 0

    def _set_table(self, values):
        """Upload ``values`` (numpy or torch, reshaped to [nindex, -1])."""
        if isinstance(values, (list, tuple)) and len(values) == 1:
            values = values[0]
        if isinstance(values, torch.Tensor):
            vals = values.detach().to(dtype=torch.float64).reshape(self.nindex, -1)
            self._store(vals.to(dev.device()).contiguous().clone())
        else:
            vals = np.asarray(values, dtype=np.float64).reshape(self.nindex, -1)
            self._store(dev.to_device(vals))
        self._version += 1

    @property
    def vertex_values(self):
        """The vertex table [nindex, out] as a float64 leaf tensor with ``requires_grad`` -- the
        descriptor's buffer itself, so in-place ``torch.optim`` steps are what the fused sweeps read."""
        if self._param_dev is None:
            raise ValueError("%s has no vertex values" % type(self).__name__)
        if not self._param_dev.requires_grad:
            self._param_dev = self._param_dev.detach().clone().requires_grad_(True)
        return self._param_dev

    def _store(self, values):
        """The one writer of the vertex table (a device tensor [nindex, out]): swaps the buffer until
        ``vertex_values`` has been handed out, then copies into that leaf in place."""
        leaf = self._param_dev
        if leaf is not None and leaf.requires_grad:
            if tuple(values.shape) != tuple(leaf.shape):
                raise DimensionError("vertex values of shape %s for a table of shape %s (the "
                                     "vertex_values leaf keeps its shape)"
                                     % (tuple(values.shape), tuple(leaf.shape)))
            with torch.no_grad():
                leaf.copy_(values)
            return
        self._param_dev = values
        self.output_dim = int(values.shape[1])

    def _trainable_tensors(self):
        leaf = self._param_dev
        return [leaf] if leaf is not None and leaf.requires_grad else []

    def _table_vjp(self, points, grad_out):
        """The vertex table's gradient: one ``slb_function_vjp`` call (the transpose of the lookup,
        summed in a fixed order)."""
        _, gflat, _ = _function_vjp(self, points, grad_out, want_in=False, nparams=self._param_dev.numel())
        return [gflat.view(self._param_dev.shape).to(self._param_dev.device)]

    def _table_version(self):
        # the table is swapped (new device buffer) by value_iteration until vertex_values is handed out,
        # and updated in place after, so its address and its version counter are part of the descriptor
        # identity
        if self._param_dev is None:
            return (self._version, 0, 0)
        return (self._version, self._param_dev.data_ptr(), self._param_dev._version)


class Triangulation(_VertexTable, DeterministicFunction):
    """Piecewise-linear interpolation on a GridWorld (``functions.py:1372-1510``).

    The vertex values live in HBM (``_param_dev`` [nindex, out]); ``parameters`` exposes
    them like the reference's single tf.Variable: ``tri.parameters[0]`` is the [nindex, out]
    array, and assigning ``tri.parameters = values`` re-uploads.

    ``vertex_values`` hands out that buffer as a trainable leaf (``_VertexTable``).  ``torch(points)``
    differentiates the points and the vertex values.
    """

    def __init__(self, discretization, vertex_values, project=False, name="triangulation"):
        super().__init__(name)
        self.tri = _TriangulationTables(discretization, project=project, owner=self)
        self.input_dim = self.tri.input_dim
        self._param_dev = None
        self._hyper_dev = None
        self._simp_dev = None
        self._corner_dev = None
        self._version = 0
        self.output_dim = None
        if vertex_values is not None:
            self.parameters = vertex_values

    @property
    def project(self):
        return self.tri.project

    @project.setter
    def project(self, value):
        self.tri.project = value

    @property
    def discretization(self):
        return self.tri.discretization

    @property
    def nindex(self):
        return self.tri.nindex

    @property
    def parameters(self):
        if self._param_dev is None:
            return []
        return [self._param_dev.detach().cpu().numpy()]

    @parameters.setter
    def parameters(self, values):
        self._set_table(values)

    def _vjp(self, points, grad_out, want_in, want_params):
        """The points' gradient from ``jacobian_device``; the vertex table's from ``_table_vjp``."""
        gin, grads = super()._vjp(points, grad_out, want_in, False)
        if want_params:
            grads = self._table_vjp(points, grad_out)
        return gin, grads

    @property
    def version(self):
        return (self.project,) + self._table_version()

    def descriptor(self):
        if self._param_dev is None:
            raise ValueError("Triangulation has no vertex values")
        if self.input_dim > nat.SLB_MAX_DIM:
            raise DimensionError("Triangulation supports up to %d dims" % nat.SLB_MAX_DIM)
        if self._hyper_dev is None:
            self._hyper_dev = dev.to_device(self.tri.hyperplanes)
            self._simp_dev = dev.to_device(self.tri.unit_simplices, torch.int64)
            self._corner_dev = dev.to_device(self.tri.corner_simplex, torch.int32)
        d = nat.SlbFunction()
        d.kind, d.in_dim, d.out_dim = nat.FN_TRIANGULATION, self.input_dim, self.output_dim
        d.flags = nat.FLAG_PROJECT if self.project else 0
        d.matrix = self._param_dev.data_ptr()
        d.hyperplanes = self._hyper_dev.data_ptr()
        d.unit_simplices = self._simp_dev.data_ptr()
        d.corner_simplex = self._corner_dev.data_ptr() if self.input_dim > 1 else None
        d.nsimplex = self.tri.nsimplex_unit
        d.grid = self.discretization.descriptor(need_points=True)
        return d

    def gradient_function(self):
        """The gradient of the interpolant as a fusable function object (one value column)."""
        return TriangulationGradient(self)

    def gradient(self, points):
        """``Triangulation.gradient`` (``functions.py:1302-1326, 1506-1510``): the partial
        derivatives of the piecewise-linear interpolant, numpy ``[n, d]``."""
        return self.gradient_function()(points)

    def jacobian_device(self, points):
        if self.output_dim != 1:
            raise NotImplementedError("Jacobian of a multi-column Triangulation")
        grad = self.gradient_function().evaluate_device(points)       # [n, d]
        if self.project:      # clipped coordinates carry no gradient (tf.clip_by_value, :1479-1485)
            lim = dev.to_device(np.asarray(self.discretization.limits, dtype=np.float64))
            grad = grad * ((points >= lim[:, 0]) & (points <= lim[:, 1])).to(torch.float64)
        return grad.unsqueeze(1)


class TriangulationGradient(DeterministicFunction):
    """``x -> d Triangulation(x) / dx`` (piecewise constant; ``functions.py:1260-1326``), evaluated
    by the same simplex lookup as the value (``SLB_FLAG_GRADIENT``).  Its ``torch`` differentiates
    the points only: like the reference's ``py_func`` gradient, it passes no gradient to the vertex
    values."""

    def __init__(self, triangulation, name="triangulation_gradient"):
        super().__init__(name)
        if not isinstance(triangulation, Triangulation):
            raise TypeError("TriangulationGradient wraps a Triangulation")
        self.triangulation = triangulation
        self.input_dim = self.output_dim = triangulation.input_dim

    @property
    def parameters(self):
        return self.triangulation.parameters

    @property
    def version(self):
        return ("grad", self.triangulation.version)

    def descriptor(self):
        d = self.triangulation.descriptor()
        if d.out_dim != 1:
            raise DimensionError("the fused gradient needs a Triangulation with one value column")
        d.flags |= nat.FLAG_GRADIENT
        d.out_dim = self.input_dim
        return d


class PiecewiseConstant(_VertexTable, DeterministicFunction):
    """Nearest-vertex table on a GridWorld (``functions.py:820-932``): ``pwc(x)`` is the row of
    ``vertex_values`` at ``discretization.state_to_index(x)``, evaluated on the GPU by the same lookup in
    every sweep, rollout, Bellman kernel and VJP (``SLB_FN_PIECEWISE_CONSTANT``, DESIGN.md §3.15).

    ``parameters`` is the bare [nindex, out] array, as in the reference (the setter reshapes to
    ``(nindex, -1)``); ``vertex_values`` hands the device table out as a trainable leaf, as for
    ``Triangulation``.  A point with a NaN coordinate evaluates to NaN in every column (the reference
    raises from ``ravel_multi_index``); ``parameter_derivative`` raises ``ValueError`` for it, as the
    reference does.
    """

    def __init__(self, discretization, vertex_values=None, name="piecewise_constant"):
        super().__init__(name)
        self.discretization = discretization
        self.input_dim = discretization.ndim
        self.output_dim = None
        self.parameters = vertex_values

    @property
    def parameters(self):
        if self._param_dev is None:
            return None
        return self._param_dev.detach().cpu().numpy()

    @parameters.setter
    def parameters(self, values):
        if values is None:
            self._param_dev, self.output_dim = None, None
            self._version += 1
            return
        self._set_table(values)

    @property
    def limits(self):
        return self.discretization.limits

    @property
    def nindex(self):
        return self.discretization.nindex

    @property
    def version(self):
        return self._table_version()

    def descriptor(self):
        if self._param_dev is None:
            raise ValueError("PiecewiseConstant has no vertex values")
        d = nat.SlbFunction()
        d.kind, d.in_dim, d.out_dim = nat.FN_PIECEWISE_CONSTANT, self.input_dim, self.output_dim
        d.matrix = self._param_dev.data_ptr()
        d.grid = self.discretization.descriptor()
        for c, inv in enumerate(1. / self.discretization.unit_maxes):     # numpy's, as in state_to_index
            d.cparams[c] = float(inv)
        return d

    def parameter_derivative(self, points):
        """``PiecewiseConstant.parameter_derivative`` (``functions.py:889-913``): the sparse [n, nindex]
        matrix of ones with ``pwc(points) = B @ parameters``; the columns come from the device lookup
        (``slb_grid_nearest_index``)."""
        lib = nat.load()
        pts = dev.to_device(np.atleast_2d(np.asarray(points, dtype=np.float64)))
        if pts.shape[1] != self.input_dim:
            raise DimensionError("the input argument has the wrong dimensions.")
        n = pts.shape[0]
        idx = dev.empty((n,), torch.int64)
        nat.check(lib.slb_grid_nearest_index(dev.stream(), self.discretization.descriptor(), pts.data_ptr(),
                                             n, idx.data_ptr()), "slb_grid_nearest_index")
        cols = idx.cpu().numpy()
        if np.any(cols < 0):
            raise ValueError("invalid entry in coordinates array (a point with a NaN coordinate)")
        return scipy.sparse.coo_matrix((np.ones(n, dtype=np.int64), (np.arange(n), cols)),
                                       shape=(n, self.nindex))

    def gradient(self, points):
        """Always zero (``functions.py:915-932``): the reference's broadcast ``[n, input_dim]``."""
        return np.broadcast_to(0, (len(points), self.input_dim))

    def gradient_function(self):
        """The gradient as a fusable function object: the constant 0 in ``input_dim`` columns."""
        return ConstantFunction(np.zeros(self.input_dim), input_dim=self.input_dim)

    def jacobian_device(self, points):
        return dev.zeros((points.shape[0], self.output_dim, self.input_dim))

    def _vjp(self, points, grad_out, want_in, want_params):
        """The points' gradient is zero; the vertex table's comes from ``_table_vjp``."""
        gin = dev.zeros((points.shape[0], self.input_dim)) if want_in else None
        return gin, (self._table_vjp(points, grad_out) if want_params else [])


# =============================================================================== plants
def _pack_norm(cp, normalization, ns, base):
    """cparams[base:] = Tx[ns], Tu, 1/Tx[ns]; returns the flag value."""
    if normalization is None:
        return 0.0
    tx, tu = (np.asarray(n, dtype=np.float64).ravel() for n in normalization)
    inv = tx ** -1
    for i in range(ns):
        cp[base + i] = float(tx[i])
    cp[base + ns] = float(tu[0])
    for i in range(ns):
        cp[base + ns + 1 + i] = float(inv[i])
    return 1.0


class InvertedPendulum(DeterministicFunction):
    """Normalised inverted pendulum, 10 explicit-Euler sub-steps
    (``examples/utilities.py:144-289``)."""

    def __init__(self, mass, length, friction=0.0, dt=1 / 80, normalization=None,
                 name="inverted_pendulum"):
        super().__init__(name)
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
        """Discretised, normalised linearisation (``examples/utilities.py:207-240``)."""
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

    def descriptor(self):
        d = nat.SlbFunction()
        d.kind, d.in_dim, d.out_dim = nat.FN_PENDULUM, 3, 2
        cp = d.cparams
        cp[0] = self.gravity / self.length
        cp[1] = self.inertia
        cp[2] = self.friction / self.inertia
        cp[3] = self.dt / 10
        cp[9] = _pack_norm(cp, self.normalization, 2, 4)     # [4..5] Tx, [6] Tu, [7..8] 1/Tx
        cp[10] = 1.0 if self.friction > 0 else 0.0
        return d

    def jacobian_device(self, points):
        """d x+ / d [x, u] through the ten Euler sub-steps, [n, 2, 3] (``slb_function_vjp``)."""
        return _unit_vjp_jacobian(self, points)

    def _vjp(self, points, grad_out, want_in, want_params):
        """The points' gradient as one ``slb_function_vjp`` call (``jacobian_device`` makes one per
        output)."""
        return (_function_vjp(self, points, grad_out)[0] if want_in else None), []


class CartPole(DeterministicFunction):
    """Cart-pole (``examples/utilities.py:292-437``)."""

    def __init__(self, pendulum_mass, cart_mass, length, rot_friction=0.0, dt=0.01,
                 normalization=None, name="CartPole"):
        super().__init__(name)
        self.pendulum_mass, self.cart_mass, self.length = pendulum_mass, cart_mass, length
        self.rot_friction, self.dt, self.gravity = rot_friction, dt, 9.81
        self.state_dim, self.action_dim = 4, 1
        self.normalization = normalization
        if normalization is not None:
            self.normalization = [np.array(n, dtype=np.float64) for n in normalization]
            self.inv_norm = [n ** -1 for n in self.normalization]
        self.input_dim, self.output_dim = 5, 4

    def linearize(self):
        m, M, L, b, g = (self.pendulum_mass, self.cart_mass, self.length, self.rot_friction,
                         self.gravity)
        A = np.array([[0, 0, 1, 0], [0, 0, 0, 1], [0, g * m / M, 0, -b / (M * L)],
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

    def descriptor(self):
        d = nat.SlbFunction()
        d.kind, d.in_dim, d.out_dim = nat.FN_CARTPOLE, 5, 4
        cp = d.cparams
        cp[0], cp[1], cp[2] = self.pendulum_mass, self.cart_mass, self.length
        cp[3], cp[4], cp[5] = self.rot_friction, self.gravity, self.dt / 10
        cp[15] = _pack_norm(cp, self.normalization, 4, 6)    # [6..9] Tx, [10] Tu, [11..14] 1/Tx
        return d

    def jacobian_device(self, points):
        """d x+ / d [x, u] through the ten Euler sub-steps, [n, 4, 5] (``slb_function_vjp``)."""
        return _unit_vjp_jacobian(self, points)

    _vjp = InvertedPendulum._vjp


class VanDerPol(DeterministicFunction):
    """Van der Pol oscillator in reverse time, ``x' = -y``, ``y' = x + damping (x^2 - 1) y``, 10
    explicit-Euler sub-steps (``examples/utilities.py:440-519``).  Its region of attraction is
    bounded by the unstable limit cycle.

    Called as ``vdp(states, actions)`` with a one-column action that does not enter (the reference
    splits ``[x, u]`` as ``[2, 1]``); pair it with a one-column policy such as
    ``LinearSystem(np.zeros((1, 2)))``.  ``normalization`` is the state scale ``Tx`` only: the
    plant runs on ``x diag(Tx)`` and returns its result times ``diag(1 / Tx)``, as matrix products,
    so an infinite or NaN component makes the other column NaN."""

    def __init__(self, damping=1, dt=0.01, normalization=None, name="VanDerPol"):
        super().__init__(name)
        self.damping, self.dt = damping, dt
        self.state_dim, self.action_dim = 2, 0
        self.normalization = normalization
        if normalization is not None:
            self.normalization = np.array(normalization, dtype=np.float64)
            self.inv_norm = self.normalization ** -1
        self.input_dim, self.output_dim = 3, 2

    def normalize(self, state):
        """``state . diag(1 / Tx)`` on a numpy ``[n, 2]`` array (``:455-461``)."""
        if self.normalization is None:
            return state
        return np.matmul(state, np.diag(self.inv_norm))

    def denormalize(self, state):
        """``state . diag(Tx)`` on a numpy ``[n, 2]`` array (``:463-469``)."""
        if self.normalization is None:
            return state
        return np.matmul(state, np.diag(self.normalization))

    def linearize(self):
        """The discretised (zero-order hold), normalised linearisation ``Ad`` (``:471-487``)."""
        A = np.array([[0, -1], [1, -1]], dtype=np.float64)
        if self.normalization is not None:
            Tx, Tx_inv = np.diag(self.normalization), np.diag(self.inv_norm)
            A = np.linalg.multi_dot((Tx_inv, A, Tx))
        Ad, _, _, _, _ = scipy.signal.cont2discrete((A, np.zeros([2, 1]), 0, 0), self.dt, method="zoh")
        return Ad

    def descriptor(self):
        d = nat.SlbFunction()
        d.kind, d.in_dim, d.out_dim = nat.FN_VANDERPOL, 3, 2
        cp = d.cparams
        cp[0] = self.damping
        cp[1] = self.dt / 10
        if self.normalization is not None:                      # [2] flag, [3..4] Tx, [5..6] 1/Tx
            cp[2] = 1.0
            cp[3], cp[4] = (float(t) for t in self.normalization)
            cp[5], cp[6] = (float(t) for t in self.inv_norm)
        return d

    def jacobian_device(self, points):
        """d x+ / d [x, u] through the ten Euler sub-steps, [n, 2, 3] with a zero action column
        (``slb_function_vjp``)."""
        return _unit_vjp_jacobian(self, points)

    _vjp = InvertedPendulum._vjp


def _param_device():
    """Where network parameters live: the library's device when torch sees one (every evaluation
    needs it), otherwise the CPU, so that a network can be built and inspected on a host without a
    GPU."""
    return dev.device() if torch.cuda.is_available() else torch.device("cpu")


def _leaf(value):
    """A float64 leaf tensor with requires_grad on the parameter device (copies its input)."""
    if isinstance(value, torch.Tensor):
        t = value.detach().to(device=_param_device(), dtype=torch.float64).clone()
    else:
        t = torch.tensor(np.asarray(value, dtype=np.float64), device=_param_device())
    return t.requires_grad_(True)


class _TrainableNetwork(DeterministicFunction):
    """Parameters as torch leaf tensors (``parameters``), a descriptor rebuilt whenever one of them
    changes (``version`` follows ``torch.Tensor._version``, so in-place optimizer steps count), and
    ``torch(points)`` as one autograd node whose backward is one ``slb_function_vjp`` call for the
    points and every parameter."""

    # activation codes of the fused kernels (csrc/common.cuh)
    _ACT = {"tanh": 0, "relu": 1, "linear": 2, "identity": 2}

    @classmethod
    def _activation_names(cls, activations, what):
        """The kernel's names of ``activations`` (names or functions such as ``numpy.tanh``)."""
        names = []
        for act in activations:
            key = act if isinstance(act, str) else getattr(act, "__name__", "")
            if key not in cls._ACT:
                raise NotImplementedError("%s %r is not fused (tanh/relu/linear)" % (what, act))
            names.append(key)
        return names

    @staticmethod
    def _xavier(rng, rows, cols):
        """A Xavier-uniform ``[rows, cols]`` draw from ``rng`` (``tf.contrib.layers.xavier_initializer``)."""
        lim = np.sqrt(6.0 / (rows + cols))
        return rng.uniform(-lim, lim, size=(rows, cols))

    def _network_descriptor(self, kind, widths, activations, output_scale=1.0, use_bias=False):
        """The descriptor of a fused network (layout in csrc/common.cuh): layer i has output width
        ``widths[i]`` and activation ``activations[i]``; ``output_scale`` and ``use_bias`` are read for
        ``FN_MLP`` only."""
        d = nat.SlbFunction()
        d.kind, d.in_dim, d.out_dim = kind, self.input_dim, self.output_dim
        d.cparams[0] = len(widths)
        for i, (od, act) in enumerate(zip(widths, activations)):
            d.cparams[1 + i] = od
            d.cparams[9 + i] = self._ACT[act]
        d.cparams[17] = output_scale
        d.cparams[18] = 1.0 if use_bias else 0.0
        d.matrix = self._packed_device().data_ptr()
        return d

    def _init_params(self):
        self._params = []
        self._names = []
        self._set_count = 0
        self._packed = None
        self._packed_version = None

    @property
    def parameters(self):
        return list(self._params)

    @parameters.setter
    def parameters(self, values):
        values = list(values)
        if len(values) != len(self._params):
            raise ValueError("%s has %d parameter tensors, got %d"
                             % (type(self).__name__, len(self._params), len(values)))
        new = []
        for old, v in zip(self._params, values):
            t = _leaf(v)
            if tuple(t.shape) != tuple(old.shape):
                raise DimensionError("parameter shape %s, expected %s" % (tuple(t.shape), tuple(old.shape)))
            new.append(t)
        self._set_params(new)

    @property
    def parameter_names(self):
        """TF variable names of ``parameters``, in the reference's creation order."""
        return list(self._names)

    def _set_params(self, tensors):
        self._params = tensors
        self._set_count += 1

    @property
    def version(self):
        return (self._set_count,) + tuple(t._version for t in self._params)

    def _packed_device(self):
        """The descriptor's parameter buffer for the current parameter version."""
        v = self.version
        if self._packed is None or self._packed_version != v:
            self._packed = self._pack()
            self._packed_version = v
        return self._packed

    def jacobian_device(self, points):
        return _unit_vjp_jacobian(self, points)

    def _trainable_tensors(self):
        return list(self._params)

    def _vjp(self, points, grad_out, want_in, want_params):
        """One ``slb_function_vjp`` call for the points and every parameter."""
        gin, gflat, _ = _function_vjp(self, points, grad_out, want_in,
                                      self._packed_device().numel() if want_params else 0)
        return (gin.to(points.device) if gin is not None else None,
                self._grads_like(gflat, self._params) if want_params else [])

    def vjp(self, points, grad_out, want_out=False):
        """(grad_in [n, in], [grad of each parameter], recomputed forward or None) for the cotangent
        ``grad_out`` [n, out] (device tensors)."""
        gin, gflat, out = _function_vjp(self, points, grad_out, True, self._packed_device().numel(),
                                        want_out)
        return gin, self._grads_like(gflat, self._params), out

    def _grads_like(self, gflat, params):
        """The flat parameter gradient as one tensor per parameter, each on its parameter's device
        (a network built before ``torch.cuda.set_device`` keeps its leaves where they were made)."""
        return [g.to(p.device) for g, p in zip(self._unpack_grads(gflat), params)]

    def gradient_function(self):
        """``x -> d net(x) / dx`` as a fusable function object (a network with one output)."""
        return NetworkGradient(self)


class LyapunovNetwork(_TrainableNetwork):
    """Positive-definite network ``V(x) = |phi(x)|^2`` (``examples/utilities.py:48-104``):
    layer i applies ``act(net . [W_i^T W_i + eps I; W_i'']^T)``.

    ``weights[i] = (W_posdef, W_extra or None)`` with the reference's shapes
    (``[ceil((in+1)/2), in]`` and ``[out - in, in]``); when omitted they are drawn Xavier-uniform
    from ``seed`` (the reference uses ``tf.contrib.layers.xavier_initializer``).  ``activations``
    are 'tanh' | 'relu' | 'linear' (or ``numpy.tanh``).  ``parameters`` holds the same matrices as
    trainable tensors, in the reference's variable order ``weights_posdef_i``, ``weights_i``; the
    layer kernels are formed from them on the host once per parameter version.
    """

    def __init__(self, input_dim, layer_dims, activations, eps=1e-6, initializer=None,
                 name="lyapunov_network", weights=None, seed=0):
        super().__init__(name)
        self.input_dim, self.output_dim = int(input_dim), 1
        self.num_layers = len(layer_dims)
        self.output_dims = [int(v) for v in layer_dims]
        self.eps = eps
        if self.output_dims[0] < self.input_dim:
            raise ValueError("The first layer dimension must be at least the input dimension!")
        if np.any(np.diff(self.output_dims) < 0):
            raise ValueError("Each layer must maintain or increase the dimension of its input!")
        if max(self.output_dims) > 64 or self.num_layers > 8:
            raise DimensionError("LyapunovNetwork: at most 8 layers of width <= 64 are fused")
        self.activations = self._activation_names(activations, "activation")
        self.hidden_dims = [int(np.ceil(((self.input_dim if i == 0 else self.output_dims[i - 1])
                                         + 1) / 2)) for i in range(self.num_layers)]
        if weights is None:
            rng = np.random.default_rng(seed)
            weights = []
            for i in range(self.num_layers):
                din = self.input_dim if i == 0 else self.output_dims[i - 1]
                extra = self.output_dims[i] - din
                weights.append((self._xavier(rng, self.hidden_dims[i], din),
                                self._xavier(rng, extra, din) if extra > 0 else None))
        self._init_params()
        self.weights = weights

    def _layer_in(self, i):
        return self.input_dim if i == 0 else self.output_dims[i - 1]

    @property
    def weights(self):
        """``[(W_posdef, W_extra or None)]`` per layer, numpy copies of the current parameters."""
        out, it = [], iter(self._params)
        for i in range(self.num_layers):
            w0 = next(it).detach().cpu().numpy()
            w1 = next(it).detach().cpu().numpy() if self.output_dims[i] > self._layer_in(i) else None
            out.append((w0, w1))
        return out

    @weights.setter
    def weights(self, weights):
        params, names = [], []
        for i, (w0, w1) in enumerate(weights):
            din = self._layer_in(i)
            w0 = np.asarray(w0.detach().cpu().numpy() if isinstance(w0, torch.Tensor) else w0,
                            dtype=np.float64)
            if w0.ndim != 2 or w0.shape[1] != din:
                raise DimensionError("weights_posdef_%d must have %d columns, got shape %s"
                                     % (i, din, w0.shape))
            params.append(_leaf(w0))
            names.append("weights_posdef_%d" % i)
            if self.output_dims[i] > din:
                if w1 is None or tuple(np.shape(w1) if not hasattr(w1, "shape") else w1.shape) != \
                        (self.output_dims[i] - din, din):
                    raise DimensionError("weights_%d must have shape %s"
                                         % (i, (self.output_dims[i] - din, din)))
                params.append(_leaf(w1))
                names.append("weights_%d" % i)
        if len(weights) != self.num_layers:
            raise DimensionError("%d layers need %d weight pairs" % (self.num_layers, len(weights)))
        self._names = names
        self._set_params(params)

    def kernels(self):
        """Layer kernels ``[W^T W + eps I; W_extra]`` ([out_i, in_i])."""
        out = []
        for i, (w0, w1) in enumerate(self.weights):
            din = self._layer_in(i)
            k = w0.T.dot(w0) + self.eps * np.eye(din)
            if w1 is not None:
                k = np.concatenate([k, w1], axis=0)
            out.append(k)
        return out

    def _pack(self):
        return dev.to_device(np.concatenate([k.ravel() for k in self.kernels()]))

    def descriptor(self):
        return self._network_descriptor(nat.FN_LYAPUNOV_NN, self.output_dims, self.activations)

    def _unpack_grads(self, gflat):
        """dL/dK_i -> the leaves: dW_posdef = W (G + G^T) over the top in_i rows, dW_extra = G below."""
        grads, off, it = [], 0, iter(self._params)
        for i in range(self.num_layers):
            din, dout = self._layer_in(i), self.output_dims[i]
            G = gflat[off:off + dout * din].view(dout, din)
            off += dout * din
            top = G[:din]
            grads.append(next(it).detach() @ (top + top.T))
            if dout > din:
                next(it)
                grads.append(G[din:].clone())
        return grads

    def gradient(self, points):
        """dV/dx at the points, numpy ``[n, d]`` (``tf.gradients(V(x), x)`` of the notebooks), from
        ``gradient_function()``."""
        pts = dev.to_device(concatenate_inputs([points]) if not isinstance(points, torch.Tensor)
                            else points)
        return self.gradient_function().evaluate_device(pts).cpu().numpy()


class NeuralNetwork(_TrainableNetwork):
    """Dense MLP (``functions.py:1665-1729``): bias in the hidden layers only, no bias in the output
    layer, output multiplied by ``output_scale``; ``nonlinearities`` one per layer ('tanh' | 'relu' |
    None).

    Two conventions for ``layers``:
      - ``[in, h1, ..., out]`` with one nonlinearity per layer after the input: built at once;
      - the reference's ``[h1, ..., out]`` with as many nonlinearities as entries: every entry is a
        layer width, and the input width and the parameters are created at the first evaluation, as
        the reference's TF variables are (``parameters`` is ``[]`` before that).
    ``weights[i]`` has the TF layout ``[in_i, out_i]``, ``biases[i]`` ``[out_i]`` (hidden layers);
    both are drawn Xavier-uniform / zero from ``seed`` when omitted.  ``parameters`` holds them as
    trainable tensors in the reference's variable order (``layer_i/kernel``, ``layer_i/bias``, ...,
    ``output/kernel``).
    """

    def __init__(self, layers, nonlinearities, output_scale=1., use_bias=True,
                 name="neural_network", weights=None, biases=None, seed=0):
        super().__init__(name)
        self.layers = [int(v) for v in layers]
        self.nonlinearities = self._activation_names(
            ["linear" if act is None else act for act in nonlinearities], "nonlinearity")
        if len(self.nonlinearities) == len(self.layers):
            widths = list(self.layers)                       # reference convention: input inferred
        elif len(self.nonlinearities) == len(self.layers) - 1:
            widths = self.layers[1:]
        else:
            raise ValueError("one nonlinearity per layer after the input is required")
        self.output_scale = float(output_scale)
        self.use_bias = bool(use_bias)
        self.output_dim = widths[-1]
        if max(widths) > 64 or len(widths) > 8 or self.output_dim > nat.SLB_MAX_OUT:
            raise DimensionError("NeuralNetwork: at most 8 layers of width <= 64 are fused")
        self._widths = widths
        self._seed = seed
        self._init_params()
        self._biases_unused = None
        self.input_dim = None
        if len(self.nonlinearities) == len(self.layers) - 1:
            self._create(self.layers[0], weights, biases)
        elif weights is not None:
            self._create(int(np.shape(weights[0])[0]), weights, biases)
        elif biases is not None:
            raise ValueError("biases without weights need the [in, h1, ..., out] convention")

    @property
    def built(self):
        return self.input_dim is not None

    def _create(self, input_dim, weights=None, biases=None):
        """Create the parameters for input width ``input_dim`` (drawn from ``seed`` when omitted)."""
        self.input_dim = int(input_dim)
        if self.input_dim > nat.SLB_MAX_IN:
            raise DimensionError("NeuralNetwork: input width above %d" % nat.SLB_MAX_IN)
        dims = [self.input_dim] + self._widths
        rng = np.random.default_rng(self._seed)
        if weights is None:
            weights = [self._xavier(rng, din, dout) for din, dout in zip(dims[:-1], dims[1:])]
        if biases is None:
            biases = [np.zeros(d) for d in dims[1:-1]]
        self._dims = dims
        self._set_weights_biases(weights, biases)

    def build(self, input_dim):
        """Create the parameters for input width ``input_dim`` unless they exist (what the first
        evaluation does with its points' width).  A network in the reference's convention needs this,
        or one evaluation, before it is handed to a fused consumer (Lyapunov, PolicyIteration,
        ClosedLoop), which reads its descriptor."""
        if not self.built:
            self._create(input_dim)

    _build = build

    def _set_weights_biases(self, weights, biases):
        dims = self._dims
        weights = [np.asarray(w.detach().cpu().numpy() if isinstance(w, torch.Tensor) else w,
                              dtype=np.float64) for w in weights]
        biases = [np.asarray(b.detach().cpu().numpy() if isinstance(b, torch.Tensor) else b,
                             dtype=np.float64) for b in biases]
        if len(weights) != len(dims) - 1 or any(w.shape != (a, b) for w, a, b in
                                               zip(weights, dims[:-1], dims[1:])):
            raise DimensionError("weights must have shapes %s"
                                 % [(a, b) for a, b in zip(dims[:-1], dims[1:])])
        if len(biases) != len(dims) - 2 or any(b.shape != (d,) for b, d in zip(biases, dims[1:-1])):
            raise DimensionError("biases must have shapes %s" % [(d,) for d in dims[1:-1]])
        params, names = [], []
        for i, w in enumerate(weights[:-1]):
            params.append(_leaf(w))
            names.append("layer_%d/kernel" % i)
            if self.use_bias:
                params.append(_leaf(biases[i]))
                names.append("layer_%d/bias" % i)
        params.append(_leaf(weights[-1]))
        names.append("output/kernel")
        self._biases_unused = None if self.use_bias else biases
        self._names = names
        self._set_params(params)

    def _kernel_tensors(self):
        step = 2 if self.use_bias else 1
        return self._params[0:-1:step] + [self._params[-1]]

    @property
    def weights(self):
        """Layer kernels ``[in_i, out_i]``, numpy copies of the current parameters."""
        return [t.detach().cpu().numpy() for t in self._kernel_tensors()] if self.built else []

    @weights.setter
    def weights(self, weights):
        if not self.built:
            self._create(int(np.shape(weights[0])[0]), weights)
        else:
            self._set_weights_biases(weights, self.biases)

    @property
    def biases(self):
        """Hidden-layer biases ``[out_i]``, numpy copies of the current parameters."""
        if not self.built:
            return []
        if not self.use_bias:
            return [np.array(b) for b in self._biases_unused]
        return [t.detach().cpu().numpy() for t in self._params[1:-1:2]]

    @biases.setter
    def biases(self, biases):
        if not self.built:
            raise ValueError("the network creates its parameters at the first evaluation")
        self._set_weights_biases(self.weights, biases)

    def lipschitz(self):
        """Product over the layer kernels of their largest singular value (``functions.py:1742-1761``).
        Every kernel enters, also with ``use_bias=False`` (where the reference's pairing of
        parameters skips every second one)."""
        out = 1.0
        for w in self.weights:
            out *= float(np.linalg.svd(w, compute_uv=False).max())
        return out

    def _pack(self):
        parts = []
        for i, t in enumerate(self._params):
            name = self._names[i]
            parts.append(t.detach().T.reshape(-1) if name.endswith("kernel") else t.detach().reshape(-1))
        return torch.cat(parts).to(dev.device()).contiguous()

    def _unpack_grads(self, gflat):
        grads, off = [], 0
        for t, name in zip(self._params, self._names):
            if name.endswith("kernel"):
                din, dout = t.shape
                grads.append(gflat[off:off + din * dout].view(dout, din).T.contiguous())
                off += din * dout
            else:
                grads.append(gflat[off:off + t.shape[0]].clone())
                off += t.shape[0]
        return grads

    def descriptor(self):
        if not self.built:
            raise DimensionError("NeuralNetwork(%s): the input width is set by the first evaluation;"
                                 " call build(input_dim) or evaluate it once before fusing it"
                                 % self.layers)
        return self._network_descriptor(nat.FN_MLP, self._widths, self.nonlinearities, self.output_scale,
                                        self.use_bias)

    def evaluate_device(self, points):
        pts = dev.to_device(points)
        if pts.dim() == 2:
            self.build(pts.shape[1])
        return super().evaluate_device(pts)


class NetworkGradient(DeterministicFunction):
    """``x -> d net(x) / dx`` of a ``LyapunovNetwork`` or a one-output ``NeuralNetwork``
    (``tf.gradients(V(x), x)``: the Lipschitz lambda of ``lyapunov_function_learning.ipynb`` cell 19),
    evaluated inside the fused kernels (``SLB_FLAG_GRADIENT``): reverse mode through the network at
    each point, bit-identical to the network's VJP with cotangent 1.  Its ``torch`` evaluates; its
    backward (the network's second derivative) is not implemented."""

    def __init__(self, net, name="network_gradient"):
        super().__init__(name)
        if not isinstance(net, _TrainableNetwork):
            raise TypeError("NetworkGradient wraps a LyapunovNetwork or NeuralNetwork")
        self.net = net

    @property
    def input_dim(self):
        return self.net.input_dim

    @property
    def output_dim(self):
        return self.net.input_dim

    @property
    def parameters(self):
        return self.net.parameters

    @property
    def version(self):
        return ("grad", self.net.version)

    def descriptor(self):
        if self.net.output_dim != 1:
            raise DimensionError("the fused gradient needs a network with one output, not %d (the "
                                 "Jacobian of a multi-output network is not fused)" % self.net.output_dim)
        d = self.net.descriptor()                  # an unbuilt NeuralNetwork raises DimensionError
        if d.in_dim > nat.SLB_MAX_OUT:
            raise DimensionError("the fused gradient of a network has at most %d input columns, not %d"
                                 % (nat.SLB_MAX_OUT, d.in_dim))
        d.flags |= nat.FLAG_GRADIENT
        d.out_dim = d.in_dim
        return d

    def _trainable_tensors(self):
        return self.net._trainable_tensors()

    def _vjp(self, points, grad_out, want_in, want_params):
        raise NotImplementedError("the backward of NetworkGradient is the network's second derivative "
                                  "(a Hessian-vector product), which has no device kernel")


# =============================================================================== Gaussian processes
class Kernel(object):
    """Covariance function with the algebra of ``gpflow==0.4.0`` ``kernels`` (third-party code the
    reference hands to ``GPRCached``, ``functions.py:370-393``): primitives carry ``input_dim`` and
    ``active_dims`` (default: the first ``input_dim`` columns), ``+`` and ``*`` build sums and
    products.  The device evaluates the sum-of-products normal form (``slb_kernel``)."""

    def __add__(self, other):
        return Sum([self, other])

    def __mul__(self, other):
        return Product([self, other])

    def terms(self):
        """Normal form: list of product terms, each a list of primitives."""
        raise NotImplementedError

    def hyper_key(self):
        return tuple(tuple(p.hyper_key() for p in term) for term in self.terms())

    def is_plain_rbf(self, din):
        return False

    def primitives(self, path="kern"):
        """``(path, primitive)`` of every primitive object of the expression tree in tree order, each
        object once (at its first path): a primitive that product expansion puts in several terms is
        one set of parameters."""
        out, seen = [], set()
        for p, prim in self._walk(path):
            if id(prim) not in seen:
                seen.add(id(prim))
                out.append((p, prim))
        return out

    def K_device(self, X, X2=None):
        """K(X, X2) on raw inputs (device tensors), gpflow arithmetic."""
        total = None
        for term in self.terms():
            prod = None
            for p in term:
                k = p._K(X, X2)
                prod = k if prod is None else prod * k
            total = prod if total is None else total + prod
        return total

    def Kdiag_device(self, X):
        total = None
        for term in self.terms():
            prod = None
            for p in term:
                k = p._Kdiag(X)
                prod = k if prod is None else prod * k
            total = prod if total is None else total + prod
        return total

    def fill(self, kstruct, din):
        """Write the normal form into an ``slb_kernel``."""
        terms = self.terms()
        count = sum(len(t) for t in terms)
        if count > nat.SLB_MAX_KPRIM:
            raise NotImplementedError("kernel expands to %d primitives; the device descriptor "
                                      "holds %d" % (count, nat.SLB_MAX_KPRIM))
        i = 0
        for t, term in enumerate(terms):
            for p in term:
                if max(p.active_dims) >= din:
                    raise DimensionError("kernel active_dims %r outside the %d GP input columns"
                                         % (p.active_dims, din))
                prim = kstruct.prims[i]
                prim.kind, prim.term, prim.variance = p.KIND, t, p._scalar_variance()
                weights = p._weights()
                for c in range(nat.SLB_MAX_IN):
                    prim.w[c] = 0.0
                for c, w in zip(p.active_dims, weights):
                    prim.w[c] = float(w)
                i += 1
        kstruct.num_prims = count


class Sum(Kernel):
    def __init__(self, kern_list):
        self.kern_list = list(kern_list)

    def terms(self):
        return [term for k in self.kern_list for term in k.terms()]

    def _walk(self, path):
        for i, k in enumerate(self.kern_list):
            yield from k._walk("%s.kern_list[%d]" % (path, i))


Add = Sum


class Product(Kernel):
    def __init__(self, kern_list):
        self.kern_list = list(kern_list)

    def terms(self):
        out = [[]]
        for k in self.kern_list:
            out = [a + b for a in out for b in k.terms()]
        return out

    _walk = Sum._walk


Prod = Product


class _Primitive(Kernel):
    KIND = None

    def __init__(self, input_dim, active_dims=None):
        self.input_dim = int(input_dim)
        if active_dims is None:
            active_dims = range(self.input_dim)
        elif isinstance(active_dims, slice):
            active_dims = range(*active_dims.indices(1 << 30))[:self.input_dim]
        self.active_dims = [int(a) for a in active_dims]
        if len(self.active_dims) != self.input_dim:
            raise DimensionError("active_dims %r does not select input_dim = %d columns"
                                 % (self.active_dims, self.input_dim))

    PARAMS = ("variance",)        # hyper-parameter attributes, in GPRCached.hyperparameters() order

    def terms(self):
        return [[self]]

    def _walk(self, path):
        yield path, self

    def _slot_gradient(self, g_variance, g_w):
        """Gradients of this primitive's parameters from one descriptor occurrence's slot gradients
        (``slb_gp_lml_grad``: ``g_variance``, ``g_w[c]`` per input column), one value per component."""
        return {"variance": g_variance}

    def _slice(self, X):
        return X[:, self.active_dims]

    def _scalar_variance(self):
        return float(self.variance)

    def _weights(self):
        return np.zeros(self.input_dim)

    def hyper_key(self):
        return (self.KIND, tuple(self.active_dims), self._scalar_variance(),
                tuple(np.asarray(self._weights(), dtype=np.float64).tolist()))


class _Stationary(_Primitive):
    PARAMS = ("variance", "lengthscales")

    def __init__(self, input_dim, variance=1.0, lengthscales=None, active_dims=None, ARD=False):
        _Primitive.__init__(self, input_dim, active_dims)
        self.variance = float(variance)
        ls = 1.0 if lengthscales is None else lengthscales
        self.lengthscales = np.broadcast_to(np.asarray(ls, dtype=np.float64),
                                            (self.input_dim,)).copy()
        self.ARD = ARD

    def _weights(self):
        return 1.0 / self.lengthscales

    def _slot_gradient(self, g_variance, g_w):
        # w = 1 / l:  d / d l = -(d / d w) / l^2
        return {"variance": g_variance,
                "lengthscales": -np.asarray(g_w)[self.active_dims] / self.lengthscales ** 2}

    def hyper_key(self):
        return (self.KIND, tuple(self.active_dims), self.variance,
                tuple(self.lengthscales.tolist()))

    def _square_dist(self, X, X2):
        """gpflow ``Stationary.square_dist``: the |x|^2 + |x'|^2 - 2 x.x' expansion."""
        ls = torch.as_tensor(self.lengthscales, dtype=torch.float64, device=X.device)
        X = self._slice(X) / ls
        sq = (X * X).sum(dim=1)
        if X2 is None:
            return -2.0 * (X @ X.T) + sq[:, None] + sq[None, :]
        X2 = self._slice(X2) / ls
        sq2 = (X2 * X2).sum(dim=1)
        return -2.0 * (X @ X2.T) + sq[:, None] + sq2[None, :]

    def _euclid_dist(self, X, X2):
        return torch.sqrt(self._square_dist(X, X2) + 1e-12)

    def _Kdiag(self, X):
        return torch.full((X.shape[0],), self.variance, dtype=torch.float64, device=X.device)


class RBF(_Stationary):
    """Squared-exponential kernel with the arithmetic of ``gpflow==0.4.0`` ``kernels.RBF``:
    ``variance * exp(-0.5 * sum(((x - x') / lengthscales)^2))``, ``Kdiag = variance``,
    defaults 1 (``lengthscales`` scalar or ARD vector)."""
    KIND = nat.K_RBF

    def is_plain_rbf(self, din):
        return self.active_dims == list(range(din))

    def _K(self, X, X2=None):
        return self.variance * torch.exp(-self._square_dist(X, X2) / 2)

    def K_scaled(self, Xs):
        """K(X, X) from lengthscale-divided inputs (device tensor [M, d])."""
        sq = (Xs * Xs).sum(dim=1)
        dist = -2.0 * (Xs @ Xs.T) + sq[:, None] + sq[None, :]
        return self.variance * torch.exp(-dist / 2)


class Matern12(_Stationary):
    """``variance * exp(-r)``, ``r = sqrt(square_dist + 1e-12)`` (gpflow 0.4.0)."""
    KIND = nat.K_MATERN12

    def _K(self, X, X2=None):
        return self.variance * torch.exp(-self._euclid_dist(X, X2))


class Matern32(_Stationary):
    """``variance * (1 + sqrt(3) r) * exp(-sqrt(3) r)`` (gpflow 0.4.0)."""
    KIND = nat.K_MATERN32

    def _K(self, X, X2=None):
        r = self._euclid_dist(X, X2)
        return self.variance * (1. + np.sqrt(3.) * r) * torch.exp(-np.sqrt(3.) * r)


class Matern52(_Stationary):
    """``variance * (1 + sqrt(5) r + 5/3 r^2) * exp(-sqrt(5) r)`` (gpflow 0.4.0)."""
    KIND = nat.K_MATERN52

    def _K(self, X, X2=None):
        r = self._euclid_dist(X, X2)
        return self.variance * (1. + np.sqrt(5.) * r + 5. / 3. * r * r) * torch.exp(-np.sqrt(5.) * r)


class Linear(_Primitive):
    """gpflow 0.4.0 ``kernels.Linear``: ``K = (X * variance) X'^T`` on the active columns,
    ``variance`` a scalar or (``ARD=True``) one value per column."""
    KIND = nat.K_LINEAR

    def __init__(self, input_dim, variance=1.0, active_dims=None, ARD=False):
        _Primitive.__init__(self, input_dim, active_dims)
        self.ARD = ARD
        self.variance = np.broadcast_to(np.asarray(variance, dtype=np.float64),
                                        (self.input_dim,)).copy()

    def _scalar_variance(self):
        return 1.0

    def _weights(self):
        return self.variance

    def _slot_gradient(self, g_variance, g_w):
        return {"variance": np.asarray(g_w)[self.active_dims]}     # w_c is the column's variance

    def _K(self, X, X2=None):
        var = torch.as_tensor(self.variance, dtype=torch.float64, device=X.device)
        X = self._slice(X)
        X2 = X if X2 is None else self._slice(X2)
        return (X * var) @ X2.T

    def _Kdiag(self, X):
        var = torch.as_tensor(self.variance, dtype=torch.float64, device=X.device)
        X = self._slice(X)
        return (X * X * var).sum(dim=1)


class Constant(_Primitive):
    """gpflow 0.4.0 ``kernels.Constant`` / ``Bias``: ``K = variance`` everywhere."""
    KIND = nat.K_CONSTANT

    def __init__(self, input_dim, variance=1.0, active_dims=None):
        _Primitive.__init__(self, input_dim, active_dims)
        self.variance = float(variance)

    def _K(self, X, X2=None):
        n2 = X.shape[0] if X2 is None else X2.shape[0]
        return torch.full((X.shape[0], n2), self.variance, dtype=torch.float64, device=X.device)

    def _Kdiag(self, X):
        return torch.full((X.shape[0],), self.variance, dtype=torch.float64, device=X.device)


Bias = Constant


class White(_Primitive):
    """gpflow 0.4.0 ``kernels.White``: ``variance * I`` for ``K(X)``, zeros against new points."""
    KIND = nat.K_WHITE

    def __init__(self, input_dim, variance=1.0, active_dims=None):
        _Primitive.__init__(self, input_dim, active_dims)
        self.variance = float(variance)

    def _K(self, X, X2=None):
        if X2 is None:
            return self.variance * torch.eye(X.shape[0], dtype=torch.float64, device=X.device)
        return torch.zeros((X.shape[0], X2.shape[0]), dtype=torch.float64, device=X.device)

    def _Kdiag(self, X):
        return torch.full((X.shape[0],), self.variance, dtype=torch.float64, device=X.device)


class _KernelNamespace(object):
    """``gpflow.kernels``-style access: ``safe_learning_b200.kernels.Matern32(...)``."""
    RBF, Matern12, Matern32, Matern52 = RBF, Matern12, Matern32, Matern52
    Linear, Constant, Bias, White, Add, Prod = Linear, Constant, Bias, White, Add, Prod


kernels = _KernelNamespace()


class Likelihood(object):
    """Gaussian likelihood holder (``gp.likelihood.variance``, default 1 like gpflow)."""

    def __init__(self, variance=1.0):
        self.variance = float(variance)


# gpflow 0.4.0's positive transform (transforms.Log1pe): value = softplus(free) + 1e-6
_POSITIVE_LOWER = 1e-6


def _param_value(owner, name):
    """Copy of hyper-parameter ``owner.name``: a float, or one value per column when ``owner.ARD``."""
    value = np.asarray(getattr(owner, name), dtype=np.float64)
    if value.ndim == 0:
        return float(value)
    if getattr(owner, "ARD", False):
        return value.copy()
    if np.any(value != value[0]):
        raise ValueError("%s.%s holds %s although ARD is False: a non-ARD parameter is one value"
                         % (type(owner).__name__, name, value.tolist()))
    return float(value[0])


def _set_param_value(owner, name, value):
    old = getattr(owner, name)
    if np.ndim(old) == 0:
        setattr(owner, name, float(value))
    else:
        setattr(owner, name, np.broadcast_to(np.asarray(value, dtype=np.float64), np.shape(old)).copy())


class _Factor(object):
    """Device-resident Cholesky state of one (X, kernel, noise, scale) combination."""

    __slots__ = ("key", "M", "nrb", "Xs", "L", "Linv", "Wpack", "Whead", "Wheadp", "Xhead", "head_rows",
                 "Xf", "hmax", "appends", "plain", "floor_rel")


_FACTOR_CACHE = {}
_FACTOR_CACHE_MAX = 8


def _remember_factor(fac):
    if len(_FACTOR_CACHE) >= _FACTOR_CACHE_MAX:
        _FACTOR_CACHE.pop(next(iter(_FACTOR_CACHE)))
    _FACTOR_CACHE[fac.key] = fac


class GPRCached(object):
    """GP regression with the factor cached in HBM (``functions.py:357-458``).

    ``update_cache`` (``:395-415``) builds ``L = chol(scale^2 (K + noise I))`` with torch's
    cuSOLVER/cuBLAS on the device (library plumbing, between sweeps), forms ``L^-1`` and packs
    it into the fragment order the sweep kernel streams (``slb_pack_factor``), and
    ``alpha = L^-1 scale (Y - m(X))``.  GPs that share X, kernel, noise and scale share one
    factor (the stacked GPs of a ``FunctionStack`` often do).

    ``Y`` may have k = 1..``SLB_MAX_OUT`` columns (gpflow's ``GPR`` with several targets): one kernel and
    noise for all of them, hence one factor; each column has its own ``alpha`` / ``gamma`` tables, stored
    as one 2-D device tensor per kind with a row per column (a 1-D tensor for k = 1).  A ``LinearSystem``
    prior mean then has k rows, row c being column c's prior mean.
    """

    def __init__(self, x, y, kern, mean_function=None, scale=1., name="GPRCached",
                 noise_variance=1.0):
        self.name = name
        self._X = np.atleast_2d(np.asarray(x, dtype=np.float64))
        self._Y = self._checked_targets(y, self._X.shape[0])
        if not isinstance(kern, Kernel):
            raise TypeError("kern must be built from safe_learning_b200 kernels (RBF, Matern12/32/52, "
                            "Linear, Constant, White and their sums / products), got %r"
                            % type(kern).__name__)
        if mean_function is not None and not isinstance(mean_function, LinearSystem):
            raise NotImplementedError("prior mean must be None or a LinearSystem with one row per output")
        if mean_function is not None and mean_function.output_dim != self._Y.shape[1]:
            raise DimensionError("the prior mean has %d rows for %d target columns: row c is column c's "
                                 "prior mean" % (mean_function.output_dim, self._Y.shape[1]))
        if self._X.shape[1] > nat.SLB_MAX_IN:
            raise DimensionError("GP input dimension above %d" % nat.SLB_MAX_IN)
        self.kern = kern
        self.mean_function = mean_function
        self.likelihood = Likelihood(noise_variance)
        self._scale = float(scale)
        self._factor = None
        self._alpha_dev = None
        self._gamma_dev = None
        self._gamma_f_dev = None
        self._gamma_l1_cols = [0.0]
        self._prior_dev = None
        self._stale = True
        self._version = 0
        self._hyper_seen = None

    @staticmethod
    def _checked_targets(y, rows):
        """``y`` as a float64 [rows, k] array, 1 <= k <= SLB_MAX_OUT (a 1-D ``y`` is one row)."""
        y = np.atleast_2d(np.asarray(y, dtype=np.float64))
        if y.ndim != 2 or y.shape[0] != rows:
            raise DimensionError("Y has shape %s but X has %d rows: one target row per input row"
                                 % (y.shape, rows))
        if not 1 <= y.shape[1] <= nat.SLB_MAX_OUT:
            raise DimensionError("Y has %d columns; a GP has 1..%d outputs" % (y.shape[1], nat.SLB_MAX_OUT))
        return y

    @property
    def output_dim(self):
        """k, the number of target columns."""
        return self._Y.shape[1]

    # data ------------------------------------------------------------------------------
    @property
    def X(self):
        return self._X

    @X.setter
    def X(self, value):
        self._X = np.atleast_2d(np.asarray(value, dtype=np.float64))
        self._stale = True

    @property
    def Y(self):
        return self._Y

    @Y.setter
    def Y(self, value):
        self._Y = np.atleast_2d(np.asarray(value, dtype=np.float64))
        self._stale = True

    @property
    def cholesky(self):
        self._ensure()
        return self._factor.L.cpu().numpy()

    @property
    def alpha(self):
        """``L^-1 scale (Y - m(X))``, [M, k]."""
        self._ensure()
        return self._alpha_dev.reshape(self.output_dim, -1)[:, :self._X.shape[0]].T.cpu().numpy()

    # factorisation -----------------------------------------------------------------------
    def _factor_key(self):
        digest = hashlib.sha1(np.ascontiguousarray(self._X).tobytes()).hexdigest()
        return (digest, self._X.shape, self.kern.hyper_key(), self.likelihood.variance,
                self._scale)

    def _hyper_state(self):
        return (self.kern.hyper_key(), self.likelihood.variance, self._scale)

    def _ensure(self):
        """Refresh the factor if data (setters mark it stale) or hyper-parameters changed."""
        if self._stale or self._factor is None or self._hyper_seen != self._hyper_state():
            self.update_cache()

    @property
    def version(self):
        self._ensure()
        return self._version

    def update_cache(self):
        """``functions.py:395-415`` on the device."""
        lib = nat.load()
        key = self._factor_key()
        M, din = self._X.shape
        fac = _FACTOR_CACHE.get(key)
        if fac is None:
            fac = _Factor()
            fac.key, fac.M, fac.nrb = key, M, (M + 7) // 8
            fac.plain = self.kern.is_plain_rbf(din)
            fac.appends = 0
            if M == 0:
                # empty data set (the notebooks start from np.empty((0, d))): prior only
                fac.Xs = dev.zeros((0, din))
                fac.L = fac.Linv = dev.zeros((0, 0))
                fac.Wpack = dev.zeros((1,))
                self._head(fac, None)
            else:
                if fac.plain:
                    fac.Xs = dev.to_device(self._X / self.kern.lengthscales)
                    kernel = self.kern.K_scaled(fac.Xs)
                else:
                    fac.Xs = dev.to_device(self._X)
                    kernel = self.kern.K_device(fac.Xs)
                kernel_noisy = kernel + torch.eye(M, dtype=torch.float64, device=kernel.device) \
                    * self.likelihood.variance
                kernel_noisy = kernel_noisy * (self._scale ** 2)
                fac.L = torch.linalg.cholesky(kernel_noisy)
                fac.Linv = torch.linalg.solve_triangular(
                    fac.L, torch.eye(M, dtype=torch.float64, device=kernel.device),
                    upper=False).contiguous()
                self._pack(fac, kernel)
            _remember_factor(fac)
        self._finish_cache(fac)

    def _pack(self, fac, kernel=None, head_from=None):
        """Device tables derived from ``L^-1``: the DMMA-ordered packed factor and the tables of
        the decision filter (``_head``).  ``kernel``: ``K(X, X)`` without noise if the caller has
        it; ``head_from``: an older factor of the same model whose head subset is kept."""
        lib = nat.load()
        fac.Wpack = dev.empty((int(lib.slb_packed_len(fac.M)),))
        nat.check(lib.slb_pack_factor(dev.stream(), fac.Linv.data_ptr(), fac.M,
                                      fac.Wpack.data_ptr()), "slb_pack_factor")
        self._head(fac, kernel, head_from)

    def _head(self, fac, kernel, head_from=None):
        """Tables of the decision filter (``slb_lyapunov_sweep_filtered``, csrc/filter.cu).

        * Head subset: the posterior variance given ANY subset S of the training set bounds the
          full posterior variance from above.  S = the first ``min(M, SLB_HEAD_RANK)`` points in
          pivoted-Cholesky order of ``K(X, X)`` (greedy: the point with the largest variance given
          the ones already chosen), factored on its own: ``Whead = chol(scale^2 (K_SS + noise
          I))^-1`` (stored transposed = column-major, zero padded), ``Xhead = Xs[S]``.  A factor
          grown by ``append_data`` keeps the subset of the factor it grew from.
        * ``Xf``: the training inputs as the filter's mean stage streams them (TMA bulk copies:
          rows padded to a multiple of 4, 16-byte aligned); for the plain RBF each row carries
          ``-|x / l|^2 / 2`` so that the squared distance expands into three FMAs.
        * ``floor_rel``: certified lower bound of posterior variance / prior variance that
          decides whether the filter may be used at all (``Lyapunov._filter_enabled``)."""
        R = nat.SLB_HEAD_RANK
        M, din = fac.M, self._X.shape[1]
        r = min(M, R)
        fac.Whead = dev.zeros((R, R))
        fac.Xhead = dev.zeros((R, din))
        fac.Wheadp = dev.zeros((R * R,))
        fac.head_rows = r
        Mp = max(8 * ((M + 7) // 8), 8)
        width = din + 1 if fac.plain else din
        fac.Xf = dev.zeros((Mp, width))
        fac.hmax = 0.0
        if M == 0:
            fac.floor_rel = 1.0
            return
        fac.Xf[:M, :din] = fac.Xs
        if fac.plain:
            half = -0.5 * (fac.Xs * fac.Xs).sum(dim=1)
            fac.Xf[:M, din] = half
            fac.hmax = float(-half.min().item())
        fac.Wheadp = dev.zeros((R * R,))
        if head_from is not None and head_from.head_rows == r:
            fac.Whead, fac.Wheadp, fac.Xhead = head_from.Whead, head_from.Wheadp, head_from.Xhead
        else:
            if kernel is None:
                kernel = self.kern.K_scaled(fac.Xs) if fac.plain else self.kern.K_device(fac.Xs)
            subset = self._pivoted_subset(kernel, r)
            fac.Xhead[:r] = fac.Xs.index_select(0, subset)
            k_ss = kernel.index_select(0, subset).index_select(1, subset)
            k_ss = (k_ss + torch.eye(r, dtype=torch.float64, device=k_ss.device)
                    * self.likelihood.variance) * (self._scale ** 2)
            l_ss = torch.linalg.cholesky(k_ss)
            linv = torch.linalg.solve_triangular(
                l_ss, torch.eye(r, dtype=torch.float64, device=k_ss.device), upper=False)
            fac.Whead[:r, :r] = linv.T                    # Whead[j, i] = L_S^-1[i, j]
            # the same matrix in DMMA A-fragment order (head stage of the filter): [b, s, T/4, T%4]
            full = dev.zeros((R, R))
            full[:r, :r] = linv
            fac.Wheadp = full.reshape(R // 8, 8, R // 4, 4).permute(0, 2, 1, 3).contiguous().reshape(-1)
        # var(z) >= k(z,z) s / (M k(z,z) + s), s = noise variance (M noisy observations AT z are
        # the most informative data set): relative to k(z,z) at least s / (M kmax + s).  When
        # that is not far above fp64 rounding of the O(M^2) contraction the reference's
        # "negative variance -> NaN -> unsafe" corner (functions.py:451) is reachable and the
        # filter, which bounds the variance from above only, is not used.  Neither is it with
        # non-finite or absurdly large inputs (the expanded distance needs moderate magnitudes).
        noise = float(self.likelihood.variance)
        if fac.plain:
            kmax = float(self.kern.variance)
        else:
            kmax = float(self.kern.Kdiag_device(fac.Xs).max().item())
        fac.floor_rel = noise / (fac.M * kmax + noise) if (kmax > 0 or noise > 0) else 0.0
        if not bool(torch.isfinite(fac.Xs).all()) or float(fac.Xs.abs().max().item()) > 1e100:
            fac.floor_rel = 0.0

    @staticmethod
    def _pivoted_subset(kernel, r):
        """Indices of the first ``r`` pivots of the pivoted Cholesky factorisation of the symmetric
        positive semi-definite ``kernel`` (device tensor [M, M]) -> int64 device tensor [r]: one
        kernel launch (``slb_pivoted_subset``), no host synchronisation."""
        lib = nat.load()
        M = kernel.shape[0]
        kernel = kernel.contiguous()
        picks = dev.zeros((r,), torch.int64)
        scratch = dev.empty((M * (r + 1),))
        nat.check(lib.slb_pivoted_subset(dev.stream(), kernel.data_ptr(), M, r, picks.data_ptr(),
                                         scratch.data_ptr()), "slb_pivoted_subset")
        return picks

    def _append_rows(self, x_new):
        """Rank-one growth of the cached factor for each appended observation (SURVEY.md 8f
        item 2) -- O(M^2) on the device instead of the O(M^3) refactorisation of
        ``functions.py:395-415``:  L' = [[L, 0], [l^T, lam]],  l = L^-1 k,  lam = sqrt(k** - l.l),
        L'^-1 = [[L^-1, 0], [-(l^T L^-1) / lam, 1 / lam]].  Returns the new factor, or None when
        a full refit is due (every 256 appends, or if the pivot is not safely positive)."""
        old = self._factor
        if old is None or self._hyper_seen != self._hyper_state():
            return None
        key = self._factor_key()
        cached = _FACTOR_CACHE.get(key)
        if cached is not None:
            return cached
        x_new = np.atleast_2d(np.asarray(x_new, dtype=np.float64))
        if old.appends + len(x_new) > 256 or old.M + len(x_new) != self._X.shape[0]:
            return None
        s2 = self._scale ** 2
        Xs, L, Linv = old.Xs, old.L, old.Linv
        if old.M == 0:
            return None
        for row in x_new:
            M = Xs.shape[0]
            if old.plain:
                xs = dev.to_device((row / self.kern.lengthscales)[None, :])
                # same expansion as RBF.K_scaled (gpflow square_dist)
                dist = -2.0 * (Xs @ xs.T)[:, 0] + (Xs * Xs).sum(dim=1) + (xs * xs).sum()
                k = s2 * (self.kern.variance * torch.exp(-dist / 2))
                kss = s2 * (self.kern.variance + self.likelihood.variance)
            else:
                xs = dev.to_device(row[None, :])
                k = s2 * self.kern.K_device(Xs, xs)[:, 0]
                kss = s2 * (self.kern.Kdiag_device(xs)[0] + self.likelihood.variance)
            l = Linv @ k
            lam2 = kss - torch.dot(l, l)
            if not bool(lam2 > 1e-12 * kss):
                return None
            lam = torch.sqrt(lam2)
            L_new = torch.zeros((M + 1, M + 1), dtype=torch.float64, device=L.device)
            L_new[:M, :M] = L
            L_new[M, :M] = l
            L_new[M, M] = lam
            Linv_new = torch.zeros_like(L_new)
            Linv_new[:M, :M] = Linv
            Linv_new[M, :M] = -(l @ Linv) / lam
            Linv_new[M, M] = 1.0 / lam
            Xs, L, Linv = torch.cat((Xs, xs), dim=0), L_new, Linv_new
        fac = _Factor()
        fac.key, fac.M, fac.nrb = key, Xs.shape[0], (Xs.shape[0] + 7) // 8
        fac.Xs, fac.L, fac.Linv = Xs.contiguous(), L, Linv.contiguous()
        fac.appends, fac.plain = old.appends + len(x_new), old.plain
        self._pack(fac, None, head_from=old if old.head_rows == nat.SLB_HEAD_RANK else None)
        _remember_factor(fac)
        return fac

    def append_data(self, x, y):
        """Append observations; grows the cached factor incrementally when possible."""
        self._X = np.vstack((self._X, np.atleast_2d(x)))
        self._Y = np.vstack((self._Y, np.atleast_2d(y)))
        was_fresh = not self._stale
        self._stale = True
        fac = self._append_rows(x) if was_fresh else None
        if fac is None:
            self.update_cache()
        else:
            self._finish_cache(fac)

    def _finish_cache(self, fac):
        """alpha / gamma / prior mean for this GP's targets on factor `fac` (functions.py:405-409).

        Each kind of table is one device tensor with a row per target column, every row zero padded
        to a multiple of 8 doubles (16-byte aligned, as the filter's bulk copies need); for k = 1 it is
        the 1-D row itself.  Column c is solved on its own, ``L^-1 t_c``, so that it is the same bits
        as a one-column GP's table on the same factor."""
        M, k = fac.M, self.output_dim
        self._factor = fac
        target = dev.to_device(self._Y)
        if self.mean_function is not None:
            if M:
                target = target - self.mean_function.evaluate_device(self._X)
            self._prior_dev = dev.to_device(self.mean_function.matrix.reshape(-1))
        else:
            self._prior_dev = None
        target = self._scale * target
        # the filter's mean weights: scale^2 gamma, times the RBF variance on the plain path
        # (whose kernel values are then <= 1), zero padded to the row count of Xf; and the bound
        # sum_i (|L^-1|^T |alpha|)_i of everything that rounds when the mean is summed
        fold = self._scale ** 2 * (float(self.kern.variance) if fac.plain else 1.0)
        alpha_t = dev.zeros((k, max(8 * fac.nrb, 8)))
        gamma_t = dev.zeros((k, max(M, 1) if k == 1 else max(8 * fac.nrb, 8)))
        gamma_f_t = dev.zeros((k, fac.Xf.shape[0]))
        self._gamma_l1_cols = [0.0] * k
        for c in range(k):
            alpha = fac.Linv @ target[:, c:c + 1].contiguous()
            gamma = fac.Linv.T @ alpha
            alpha_t[c, :M] = alpha[:, 0]
            if M:
                gamma_t[c, :M] = gamma[:, 0]
                gamma_f_t[c, :M] = fold * gamma[:, 0]
                self._gamma_l1_cols[c] = abs(fold) * float((fac.Linv.abs().T @ alpha.abs()).sum().item())
        one = (lambda t: t[0]) if k == 1 else (lambda t: t)
        self._alpha_dev, self._gamma_dev, self._gamma_f_dev = one(alpha_t), one(gamma_t), one(gamma_f_t)
        self._stale = False
        self._hyper_seen = self._hyper_state()
        self._version += 1

    # differentiable prediction -------------------------------------------------------------
    def torch_predict(self, points):
        """``build_predict`` (``functions.py:417-458``) on a device tensor [n, d_in] in torch
        operations (cuBLAS / cuSOLVER on the cached factor), differentiable with respect to
        ``points``: latent mean and variance, [n, k] each (the one variance tiled over the k columns,
        like the reference's ``tf.tile``)."""
        self._ensure()
        fac, s, k = self._factor, self._scale, self.output_dim
        s2 = s * s
        mx = 0.0
        if self.mean_function is not None:
            self.mean_function.descriptor()
            mx = s * (points @ self.mean_function._matrix_dev.T)               # :439
        kss = s2 * self.kern.Kdiag_device(points)                                # :450
        if fac.M == 0:
            return (mx / s + 0.0 * points[:, :1]).expand(-1, k), (kss / s2).unsqueeze(1).expand(-1, k)
        x_train = dev.to_device(self._X)
        kx = s2 * self.kern.K_device(x_train, points)                            # :438  [M, n]
        a = torch.linalg.solve_triangular(fac.L, kx, upper=False)                # :441
        alpha = self._alpha_dev.reshape(k, -1)[:, :fac.M].T
        fmean = (a.T @ alpha + mx) / s                                           # :442, :455
        fvar = (kss - (a * a).sum(dim=0)) / s2                                   # :451, :456
        return fmean, fvar.unsqueeze(1).expand(-1, k)

    # descriptor pieces -------------------------------------------------------------------
    def fill_factor(self, f):
        self._ensure()
        fac = self._factor
        f.M, f.nrb = fac.M, fac.nrb
        f.Xs, f.Wpack = fac.Xs.data_ptr(), fac.Wpack.data_ptr()
        f.Whead, f.Xhead, f.head_rows = fac.Whead.data_ptr(), fac.Xhead.data_ptr(), fac.head_rows
        f.Wheadp = fac.Wheadp.data_ptr()
        f.Xf, f.hmax = fac.Xf.data_ptr(), fac.hmax
        f.scale = self._scale
        if fac.plain:
            for c, ls in enumerate(self.kern.lengthscales):
                f.lengthscales[c] = float(ls)
            f.variance = self.kern.variance
            f.kss = (self._scale ** 2) * self.kern.variance
            f.kernel.num_prims = 0
        else:
            self.kern.fill(f.kernel, self._X.shape[1])
        return fac.key

    def fill_output(self, o, factor_index, beta, column=0):
        """Output slot ``o`` for target column ``column``: row ``column`` of every per-column table."""
        self._ensure()

        def row(t):
            return t.data_ptr() + 8 * column * t.shape[-1]
        o.factor, o.beta = factor_index, float(beta)
        o.alpha = row(self._alpha_dev)
        o.gamma = row(self._gamma_dev)
        o.prior_mean = None if self._prior_dev is None else row(self._prior_dev.view(self.output_dim, -1))
        o.gamma_f, o.gamma_l1 = row(self._gamma_f_dev), self._gamma_l1_cols[column]

    # hyper-parameters and the log marginal likelihood (gpflow 0.4.0 GPR.build_likelihood) ------------
    def _hyper_params(self):
        """``(path, owner, attribute)`` of every hyper-parameter, in ``hyperparameters()`` order."""
        out = [("%s.%s" % (path, name), prim, name)
               for path, prim in self.kern.primitives() for name in prim.PARAMS]
        out.append(("likelihood.variance", self.likelihood, "variance"))
        return out

    def hyperparameters(self):
        """Ordered dict from a path relative to the model (``kern.variance``,
        ``kern.kern_list[1].kern_list[0].lengthscales``, ``likelihood.variance``) to a copy of the
        value: a float, or one value per active column for an ARD primitive.  A primitive that
        appears in several product terms is listed once."""
        return collections.OrderedDict((path, _param_value(owner, name))
                                       for path, owner, name in self._hyper_params())

    def _set_hyperparameters(self, values):
        where = {path: (owner, name) for path, owner, name in self._hyper_params()}
        for path, value in values.items():
            _set_param_value(*where[path], value)

    def _log_likelihood(self, want_grad):
        """LML and, if ``want_grad``, its gradient in ``slb_gp_lml_grad``'s descriptor slots.  Its own
        factorisation of ``K + noise I`` (torch / cuSOLVER): the cached posterior factor and the filter
        tables are not touched.  A matrix that is not positive definite raises
        ``torch.linalg.LinAlgError``.  With k target columns the LML is the sum of the columns' log
        densities under the one kernel and noise (gpflow's ``GPR``), and the gradient is one fused pass
        (``slb_gp_lml_grad_cols``)."""
        lib = nat.load()
        M, din = self._X.shape
        k = self.output_dim
        kstruct = nat.SlbKernel()
        self.kern.fill(kstruct, din)
        slots = np.zeros(nat.SLB_GP_HYPER_SLOTS)
        if M == 0:
            if want_grad:           # the descriptor checks still run; nothing is launched
                nat.check(lib.slb_gp_lml_grad_cols(None, None, 0, din, kstruct, None, None, k, None, None),
                          "slb_gp_lml_grad_cols")
            return 0.0, slots
        X = dev.to_device(self._X)
        K = self.kern.K_device(X) + torch.eye(M, dtype=torch.float64, device=X.device) * self.likelihood.variance
        L = torch.linalg.cholesky(K)
        d = dev.to_device(self._Y)
        if self.mean_function is not None:
            d = d - self.mean_function.evaluate_device(self._X)
        a = torch.linalg.solve_triangular(L, d, upper=False)
        lml = -0.5 * k * M * np.log(2 * np.pi) - k * torch.log(torch.diagonal(L)).sum() - 0.5 * (a * a).sum()
        if want_grad:
            alpha = torch.cholesky_solve(d, L).contiguous()                     # [M, k] row-major
            kinv = torch.cholesky_inverse(L).contiguous()
            work = dev.empty((int(lib.slb_gp_lml_grad_workspace(M)) // 8,))
            grad = dev.empty((nat.SLB_GP_HYPER_SLOTS,))
            nat.check(lib.slb_gp_lml_grad_cols(dev.stream(), X.data_ptr(), M, din, kstruct, kinv.data_ptr(),
                                               alpha.data_ptr(), k, grad.data_ptr(), work.data_ptr()),
                      "slb_gp_lml_grad_cols")
            slots = grad.cpu().numpy()
        return float(lml.item()), slots

    def compute_log_likelihood(self):
        """Log marginal likelihood ``log N(Y | m(X), K(X) + noise I)`` (gpflow's name); 0 for an
        empty data set.  ``scale`` does not enter (the reference scales only the prediction cache)."""
        return self._log_likelihood(False)[0]

    def log_likelihood_and_gradient(self):
        """``(LML, {path: d LML / d parameter})``, each gradient shaped like its parameter in
        ``hyperparameters()``: the fused kernel's slot gradients chained to the parameters (``d / d l =
        -(d / d w) / l^2``, a non-ARD value sums its columns, a shared primitive sums its terms)."""
        lml, slots = self._log_likelihood(True)
        stride = 1 + nat.SLB_MAX_IN
        per_prim = {}
        flat = [p for term in self.kern.terms() for p in term]
        for i, prim in enumerate(flat):
            acc = per_prim.setdefault(id(prim), {})
            for name, g in prim._slot_gradient(slots[i * stride], slots[i * stride + 1:(i + 1) * stride]).items():
                acc[name] = acc.get(name, 0.0) + np.asarray(g, dtype=np.float64)
        grads = collections.OrderedDict()
        for path, owner, name in self._hyper_params():
            g = slots[-1] if owner is self.likelihood else per_prim[id(owner)][name]
            grads[path] = float(np.sum(g)) if np.ndim(_param_value(owner, name)) == 0 else g.copy()
        return lml, grads

    def optimize(self, method="L-BFGS-B", tol=None, callback=None, maxiter=1000, fixed=()):
        """Fit the kernel and noise hyper-parameters by maximising the log marginal likelihood
        (gpflow 0.4.0 ``Model.optimize``): ``scipy.optimize.minimize(jac=True)`` of ``-LML`` in the
        free space of gpflow's positive transform (``softplus(x) + 1e-6``); ``callback`` receives that
        free vector.  ``fixed``: paths of ``hyperparameters()`` held at their values (gpflow's
        ``param.fixed = True``, e.g. ``"likelihood.variance"`` for a known measurement noise).  The
        fitted values are written back into the kernel objects and ``likelihood``; the next sweep
        refits the posterior.  Returns scipy's ``OptimizeResult``.  A free parameter at or below 1e-6
        raises ``ValueError``; if the search fails (e.g. a Cholesky failure) the original values are
        restored and the error propagates."""
        import scipy.optimize
        import scipy.special
        start = self.hyperparameters()
        unknown = [p for p in fixed if p not in start]
        if unknown:
            raise ValueError("fixed: unknown hyper-parameter path(s) %s; known: %s" % (unknown, list(start)))
        free = [p for p in start if p not in fixed]
        low = [p for p in free if np.any(np.asarray(start[p]) <= _POSITIVE_LOWER)]
        if low:
            raise ValueError("hyper-parameter(s) %s start at or below the positive transform's floor %g"
                             % (low, _POSITIVE_LOWER))
        shapes = [np.shape(start[p]) for p in free]
        y0 = np.concatenate([np.ravel(start[p]) for p in free])
        ys = y0 - _POSITIVE_LOWER
        x0 = ys + np.log(-np.expm1(-ys))              # softplus^-1

        def unpack(x):
            y = np.logaddexp(0.0, x) + _POSITIVE_LOWER
            out, k = {}, 0
            for p, shape in zip(free, shapes):
                n = int(np.prod(shape))
                out[p] = float(y[k]) if shape == () else y[k:k + n].reshape(shape)
                k += n
            return out

        def objective(x):
            self._set_hyperparameters(unpack(x))
            lml, grads = self.log_likelihood_and_gradient()
            g = np.concatenate([np.ravel(grads[p]) for p in free])
            return -lml, -g * scipy.special.expit(x)

        try:
            result = scipy.optimize.minimize(objective, x0, method=method, jac=True, tol=tol, callback=callback,
                                             options=dict(maxiter=maxiter))
        except BaseException:
            self._set_hyperparameters(start)
            raise
        self._set_hyperparameters(unpack(result.x))
        return result

    def variance_floor(self):
        """Certified lower bound of posterior variance / prior variance (see ``_head``)."""
        self._ensure()
        return self._factor.floor_rel

    # host copies of the cached tables ------------------------------------------------------
    _CACHE_FIELDS = ("Xs", "Wpack", "Whead", "Wheadp", "Xhead", "Xf", "alpha", "gamma", "gamma_f")

    def _cache_tables(self):
        fac = self._factor
        return (fac.Xs, fac.Wpack, fac.Whead, fac.Wheadp, fac.Xhead, fac.Xf, self._alpha_dev,
                self._gamma_dev, self._gamma_f_dev)

    def export_cache(self, pinned=True):
        """Host copies (torch CPU tensors, page-locked if ``pinned``) of the device tables a sweep
        reads: scaled training inputs, packed ``L^-1``, its head block, ``alpha`` and ``gamma``
        (what ``update_cache`` leaves in HBM, ``functions.py:395-415``).  Together with
        ``import_cache`` this checkpoints / restores the cached state without a refit."""
        self._ensure()
        fac = self._factor
        out = {}
        for name, t in zip(self._CACHE_FIELDS, self._cache_tables()):
            host = t.detach().cpu()
            out[name] = host.pin_memory() if pinned and torch.cuda.is_available() else host
        return out

    def import_cache(self, tables):
        """Copy tables produced by ``export_cache`` (same data set and hyper-parameters, hence same
        shapes) back into the device buffers: asynchronous H2D copies on the current stream."""
        self._ensure()
        fac = self._factor
        for name, dst in zip(self._CACHE_FIELDS, self._cache_tables()):
            src = tables[name]
            if not isinstance(src, torch.Tensor):
                src = torch.from_numpy(np.ascontiguousarray(src, dtype=np.float64))
            if tuple(src.shape) != tuple(dst.shape):
                raise DimensionError("import_cache: %s has shape %s, the cached table %s"
                                     % (name, tuple(src.shape), tuple(dst.shape)))
            dst.copy_(src, non_blocking=True)
        return sum(int(tables[k].numel()) * 8 for k in self._CACHE_FIELDS)


GPR = GPRCached     # the uncached gpflow.gpr.GPR of the notebooks maps onto the cached one

def _table_slots(gps):
    """(owner, attribute) of every cached device table of a list of GPRCached models, each table
    once (stacked GPs may share a factor)."""
    slots, seen = [], set()
    for gp in gps:
        gp._ensure()
        fac = gp._factor
        for owner, names in ((fac, ("Xs", "Wpack", "Whead", "Wheadp", "Xhead", "Xf")),
                             (gp, ("_alpha_dev", "_gamma_dev", "_gamma_f_dev"))):
            for name in names:
                if (id(owner), name) not in seen:
                    seen.add((id(owner), name))
                    slots.append((owner, name))
    return slots


class PackedCache(object):
    """All cached GP tables of a model (or stack) in ONE contiguous device arena with a page-locked
    host mirror, so that checkpoint / restore is a single copy each way.  Building it re-homes the
    tables into the arena (their device pointers change: descriptors are rebuilt)."""

    ALIGN = 32                     # doubles: 256-byte table alignment (TMA bulk copies need 16 bytes)

    def __init__(self, gps, pinned=True):
        self.gps = list(gps)
        # the packed factors L^-1 (90% of the bytes; read by the O(M^2) posterior only) go last, so
        # that restore() can send them on a second stream behind the tables the filter stages read
        slots = _table_slots(self.gps)
        self.slots = ([sl for sl in slots if sl[1] != "Wpack"] + [sl for sl in slots if sl[1] == "Wpack"])
        offsets, total = [], 0
        self.split = None
        for owner, name in self.slots:
            if name == "Wpack" and self.split is None:
                self.split = total
            offsets.append(total)
            total += -(-max(getattr(owner, name).numel(), 1) // self.ALIGN) * self.ALIGN
        if self.split is None:
            self.split = total
        self.arena = dev.zeros((total,))
        self.views = []
        for (owner, name), off in zip(self.slots, offsets):
            old = getattr(owner, name)
            view = self.arena[off:off + old.numel()].view(old.shape)
            view.copy_(old)
            setattr(owner, name, view)
            self.views.append(view)
        for gp in self.gps:
            gp._version += 1       # the descriptors point at the old buffers
        host = self.arena.cpu()
        self.host = host.pin_memory() if pinned and torch.cuda.is_available() else host
        self.nbytes = int(total) * 8
        self.token = tuple(id(gp._factor) for gp in self.gps)
        self._side = None
        self._pinned = bool(self.host.is_pinned())

    def valid(self):
        return (self.token == tuple(id(gp._factor) for gp in self.gps)
                and all(getattr(o, n) is v for (o, n), v in zip(self.slots, self.views)))

    def restore(self, overlap=True):
        """Host mirror -> device arena, asynchronously.  With ``overlap`` (default, page-locked
        mirror) the small tables travel on the current stream and the packed factors on a second
        one; every launch that reads the packed factors waits for that copy inside the library
        (``slb_record_factor_dependency``), so a sweep enqueued right after this call runs its filter
        stages while the factors are still arriving.  Returns the bytes copied."""
        total = self.arena.numel()
        lib = nat.load()
        cur = torch.cuda.current_stream().cuda_stream
        if not (overlap and self._pinned and 0 < self.split < total):
            nat.check(lib.slb_restore_tables(self.arena.data_ptr(), self.host.data_ptr(), 8 * total, 8 * total,
                                             cur, None), "slb_restore_tables")
            return self.nbytes
        if self._side is None:
            self._side = torch.cuda.Stream()
        nat.check(lib.slb_restore_tables(self.arena.data_ptr(), self.host.data_ptr(), 8 * self.split,
                                         8 * total, cur, self._side.cuda_stream), "slb_restore_tables")
        dev.note_factor_dependency()
        return self.nbytes




def _build_stack(gps, betas):
    """slb_gp_stack for a list of GPRCached models (factor sharing by key): a GP with k target columns
    takes k consecutive outputs on its one factor, all with its beta."""
    stack = nat.SlbGpStack()
    total = sum(gp.output_dim for gp in gps)
    if total > nat.SLB_MAX_OUT:
        raise DimensionError("at most %d stacked GP outputs, got %d" % (nat.SLB_MAX_OUT, total))
    stack.num_outputs = total
    stack.input_dim = gps[0].X.shape[1]
    keys = []
    o = 0
    for gp, beta in zip(gps, betas):
        if gp.X.shape[1] != stack.input_dim:
            raise DimensionError("stacked GPs must share the input dimension")
        gp._ensure()
        key = gp._factor.key
        if key not in keys:
            gp.fill_factor(stack.factors[len(keys)])
            keys.append(key)
        for c in range(gp.output_dim):
            gp.fill_output(stack.outputs[o], keys.index(key), beta, c)
            o += 1
    stack.num_factors = len(keys)
    return stack


def _gp_predict(stack, points, want_var=False):
    lib = nat.load()
    pts = dev.to_device(points)
    if pts.dim() != 2 or pts.shape[1] != stack.input_dim:
        raise DimensionError("GP expects %d input columns, got %s"
                             % (stack.input_dim, tuple(pts.shape)))
    n, D = pts.shape[0], stack.num_outputs
    mean, err = dev.empty((n, D)), dev.empty((n, D))
    nat.check(lib.slb_gp_predict(dev.stream(), stack, pts.data_ptr(), n, mean.data_ptr(),
                                 err.data_ptr(), 1 if want_var else 0), "slb_gp_predict")
    return mean, err


def _gp_vjp(stack, points, grad_mean=None, grad_err=None):
    """One ``slb_gp_vjp`` call: the points' gradient [n, d_in] (device tensor) for the cotangents of
    the mean and of beta * sigma ([n, D] each, either may be None)."""
    lib = nat.load()
    pts = dev.to_device(points).contiguous()
    if pts.dim() != 2 or pts.shape[1] != stack.input_dim:
        raise DimensionError("GP expects %d input columns, got %s"
                             % (stack.input_dim, tuple(pts.shape)))
    n, D = pts.shape[0], stack.num_outputs
    gm = None if grad_mean is None else dev.to_device(grad_mean).reshape(n, D).contiguous()
    ge = None if grad_err is None else dev.to_device(grad_err).reshape(n, D).contiguous()
    gin = dev.empty((n, stack.input_dim))
    if n == 0:                        # (empty tensors have no data pointer to pass)
        return gin
    size = lib.slb_gp_vjp_workspace(stack, n)
    if size < 0:
        raise nat.NativeLibraryError("slb_gp_vjp_workspace: %s" % nat.last_error())
    ws = torch.empty(size, dtype=torch.uint8, device=pts.device) if size else None
    nat.check(lib.slb_gp_vjp(dev.stream(), stack, pts.data_ptr(), n, dev.ptr(gm), dev.ptr(ge),
                             gin.data_ptr(), dev.ptr(ws)), "slb_gp_vjp")
    return gin


class _GaussianProcessNode(UncertainFunction):
    """What ``GaussianProcess`` and ``FunctionStack`` share as one node of torch's autograd graph."""

    def _members(self):
        raise NotImplementedError

    def torch(self, points):
        """Stacked (mean, beta * sigma) [n, D] each, differentiable with respect to ``points``
        (``functions.py:278-291, 507-515``): one autograd node whose forward is ``slb_gp_predict``
        (equal to ``predict_device`` bit for bit) and whose backward is one ``slb_gp_vjp`` call; an
        output that does not reach the loss costs nothing (a mean-only objective is O(M d_in) per
        point).  A backward with create_graph=True differentiates ``GPRCached.torch_predict`` instead,
        so second derivatives exist."""
        return _FusedApply.apply(points, self)

    def _forward_device(self, points):
        return self.predict_device(points)

    def _torch_expression(self, points):
        """(mean, beta * sigma) in torch operations on the cached factor (``torch_predict``)."""
        parts = [f.gaussian_process.torch_predict(points) for f in self._members()]
        return (torch.cat([m for m, _ in parts], dim=1),
                torch.cat([f.beta * torch.sqrt(v) for f, (_, v) in zip(self._members(), parts)], dim=1))

    def vjp_device(self, points, grad_mean=None, grad_err=None):
        """grad_mean^T d mean / d points + grad_err^T d (beta sigma) / d points, [n, d_in]."""
        return _gp_vjp(self.gp_stack(), points, grad_mean, grad_err)

    def _vjp(self, points, grad_out, want_in, want_params):
        if not want_in:
            return None, []
        grad_mean, grad_err = grad_out
        return _gp_vjp(self.gp_stack(), points.detach(), grad_mean, grad_err), []

    def to_mean_function(self):
        """The posterior mean as a deterministic function (``functions.py:209-230``): a
        ``PosteriorMean`` on this GP, which the rollouts and the Bellman sweeps fuse as dynamics."""
        return PosteriorMean(self)


class GaussianProcess(_GaussianProcessNode):
    """``(mean, beta * sqrt(var))`` of a GP (``functions.py:461-546``), [n, k] each for a model with k
    target columns (the one sigma in every column)."""

    def __init__(self, gaussian_process, beta=2., name="gaussian_process"):
        super().__init__(name)
        if not isinstance(gaussian_process, GPRCached):
            raise TypeError("gaussian_process must be a safe_learning_b200 GPRCached/GPR model")
        self.gaussian_process = gaussian_process
        self.beta = float(beta)
        self.n_dim = self.input_dim = gaussian_process.X.shape[1]
        self.output_dim = gaussian_process.Y.shape[1]

    @property
    def X(self):
        return self.gaussian_process.X

    @property
    def Y(self):
        return self.gaussian_process.Y

    def gp_stack(self):
        return _build_stack([self.gaussian_process], [self.beta])

    def variance_floor(self):
        return self.gaussian_process.variance_floor()

    def export_cache(self, pinned=True):
        """See ``FunctionStack.export_cache``."""
        return PackedCache([self.gaussian_process], pinned)

    def import_cache(self, tables):
        return FunctionStack.import_cache(self, tables)

    @property
    def version(self):
        return (id(self.gaussian_process), self.gaussian_process.version, self.beta)

    def __call__(self, *inputs):
        mean, err = _gp_predict(self.gp_stack(), concatenate_inputs(inputs))
        return mean.cpu().numpy(), err.cpu().numpy()

    def predict_device(self, points, want_var=False):
        return _gp_predict(self.gp_stack(), points, want_var)

    def _members(self):
        return [self]

    def update_feed_dict(self):
        """Reference hook (``functions.py:517-523``): hyper-parameters travel in the
        descriptor here, so this only refreshes the cached factor."""
        self.gaussian_process._ensure()

    def add_data_point(self, x, y):
        """Append observations and refresh the factor (``functions.py:525-546``)."""
        self.gaussian_process.append_data(x, y)


class FunctionStack(_GaussianProcessNode):
    """Stack of GPs, their outputs side by side (``functions.py:254-307``); a member with k target
    columns contributes k outputs."""

    def __init__(self, functions, name="function_stack"):
        super().__init__(name)
        self.functions = list(functions)
        for f in self.functions:
            if not isinstance(f, GaussianProcess):
                raise TypeError("FunctionStack fuses GaussianProcess members only")
        self.num_fun = len(self.functions)
        self.input_dim = self.functions[0].input_dim
        self.output_dim = sum(f.output_dim for f in self.functions)

    def gp_stack(self):
        return _build_stack([f.gaussian_process for f in self.functions],
                            [f.beta for f in self.functions])

    def variance_floor(self):
        return min(f.variance_floor() for f in self.functions)

    def export_cache(self, pinned=True):
        """Checkpoint of everything a sweep reads from the cached GPs (scaled training inputs,
        packed ``L^-1``, filter tables, ``alpha``, ``gamma`` -- what ``update_cache`` leaves in HBM,
        ``functions.py:395-415``) as a ``PackedCache``: the tables are re-homed into one contiguous
        device arena mirrored by one page-locked host buffer, so ``import_cache`` is a single H2D
        copy.  (``GPRCached.export_cache`` gives per-table host tensors instead.)"""
        return PackedCache([f.gaussian_process for f in self.functions], pinned)

    def import_cache(self, tables):
        """Restore the cached tables from ``export_cache``'s result (same data set and hyper-
        parameters); returns the bytes copied host -> device."""
        if isinstance(tables, PackedCache):
            if not tables.valid():
                raise DimensionError("import_cache: the GP cache was refitted since export_cache")
            return tables.restore()
        gps = [f.gaussian_process for f in getattr(self, "functions", [self])]
        return sum(gp.import_cache(t) for gp, t in zip(gps, tables))

    @property
    def version(self):
        return tuple(f.version for f in self.functions)

    def __call__(self, *inputs):
        mean, err = _gp_predict(self.gp_stack(), concatenate_inputs(inputs))
        return mean.cpu().numpy(), err.cpu().numpy()

    def predict_device(self, points, want_var=False):
        return _gp_predict(self.gp_stack(), points, want_var)

    def _members(self):
        return self.functions

    def add_data_point(self, x, y):
        """Append observations to every member: ``y`` holds the stack's outputs side by side, and each
        member takes its ``output_dim`` columns."""
        if all(f.output_dim == 1 for f in self.functions):
            for fun, yi in zip(self.functions, np.asarray(y).squeeze()):
                fun.add_data_point(x, yi)
            return
        y = np.asarray(y, dtype=np.float64)
        y = y.reshape(-1, self.output_dim) if y.ndim < 2 else y
        if y.shape[1] != self.output_dim:
            raise DimensionError("y has %d columns, the stack has %d outputs" % (y.shape[1], self.output_dim))
        start = 0
        for fun in self.functions:
            fun.add_data_point(x, y[:, start:start + fun.output_dim])
            start += fun.output_dim


def _gp_mean(stack, points):
    """One ``slb_gp_mean`` call: the posterior mean [n, D] (device tensor) at device points."""
    lib = nat.load()
    pts = dev.to_device(points).contiguous()
    if pts.dim() != 2 or pts.shape[1] != stack.input_dim:
        raise DimensionError("GP expects %d input columns, got %s"
                             % (stack.input_dim, tuple(pts.shape)))
    n = pts.shape[0]
    mean = dev.empty((n, stack.num_outputs))
    nat.check(lib.slb_gp_mean(dev.stream(), stack, pts.data_ptr() if n else None, n,
                              mean.data_ptr() if n else None), "slb_gp_mean")
    return mean


class PosteriorMean(DeterministicFunction):
    """The posterior mean of a ``GaussianProcess`` or ``FunctionStack`` as a deterministic function,
    ``gp.to_mean_function()`` (``functions.py:209-230``): ``f(x, u)`` or ``f(z)`` returns the numpy
    mean ``[n, D]``.  ``compute_roa``, ``reward_rollout``, ``compute_trajectory`` and ``PolicyIteration``
    fuse it as dynamics; ``Lyapunov`` takes it down the composed path (a nominal decrease, no error
    term).  It has no ``descriptor``: the kernels take it as a GP stack (``gp_stack()``), as dynamics
    only.

    The mean is ``(sum_j k_j gamma_j + scale m(z)) / scale`` with ``gamma = scale^2 v L^-T alpha``
    folded per output (``slb_gp_mean``, the form of the Bellman sweep), not the full posterior's
    ``a^T alpha``: it agrees with ``gp(z)[0]`` within the bound of DESIGN.md §3.16, not bit for bit.
    It is the same function in every entry point, so a rollout of h steps equals h compositions of
    one-step evaluations bit for bit.  The GP is held, not copied: ``add_data_point`` on it is
    picked up (``version`` follows the GP's)."""

    def __init__(self, gaussian_process, name="mean_function"):
        super().__init__(name)
        if not isinstance(gaussian_process, _GaussianProcessNode):
            raise TypeError("PosteriorMean takes a GaussianProcess or FunctionStack")
        self.gaussian_process = gaussian_process
        self.input_dim = gaussian_process.input_dim
        self.output_dim = gaussian_process.output_dim

    def gp_stack(self):
        return self.gaussian_process.gp_stack()

    @property
    def version(self):
        return self.gaussian_process.version

    def __call__(self, *inputs):
        return self.evaluate_device(concatenate_inputs(inputs)).cpu().numpy()

    def evaluate_device(self, points):
        return _gp_mean(self.gp_stack(), points)

    def _torch_expression(self, points):
        """The mean in torch operations on the cached factor (for create_graph=True backwards)."""
        return self.gaussian_process._torch_expression(points)[0]

    def _vjp(self, points, grad_out, want_in, want_params):
        if not want_in:
            return None, []
        return _gp_vjp(self.gp_stack(), points.detach(), grad_out, None), []

    def jacobian_device(self, points):
        """[n, D, d_in] from D mean-only VJPs with unit cotangents."""
        pts = dev.to_device(points).contiguous()
        stack = self.gp_stack()
        n, nout = pts.shape[0], stack.num_outputs
        rows = []
        for o in range(nout):
            cot = dev.zeros((n, nout))
            cot[:, o] = 1.0
            rows.append(_gp_vjp(stack, pts, cot, None))
        return torch.stack(rows, dim=1)
