"""CPU tests of the network gradient descriptor (``SLB_FLAG_GRADIENT`` on ``SLB_FN_LYAPUNOV_NN`` and on a
one-output ``SLB_FN_MLP``, include/slb200.h): its column count, the host checks that accept or reject it,
and how the sweep entry points take it as ``lipschitz_lyapunov``.

As in test_descriptor_checks_host.py, every call is for an empty range (or n = 0) with fake, never
dereferenced device pointers: the entry points return before any CUDA call."""
import pytest

import safe_learning_b200 as sl
from safe_learning_b200 import _native as nat


def _lib():
    return nat.load()


def _net(kind=nat.FN_LYAPUNOV_NN, in_dim=2, widths=(64, 64, 64), flags=nat.FLAG_GRADIENT, out_dim=None,
         addr=0x1000):
    """A network descriptor; with the gradient flag out_dim defaults to in_dim (NetworkGradient's)."""
    d = nat.SlbFunction()
    d.kind, d.in_dim, d.flags = kind, in_dim, flags
    d.out_dim = out_dim if out_dim is not None else (in_dim if flags & nat.FLAG_GRADIENT else widths[-1])
    d.cparams[0] = len(widths)
    for i, w in enumerate(widths):
        d.cparams[1 + i] = w
        d.cparams[9 + i] = 0
    d.cparams[17] = 1.0
    d.cparams[18] = 1.0
    d.matrix = addr
    return d


def _eval(desc):
    return _lib().slb_eval_function(None, desc, None, 0, None)


def _rejected(rc, *words):
    err = nat.last_error()
    assert rc == 1, err
    for w in words:
        assert w in err, err


# ---------------------------------------------------------------- columns
@pytest.mark.parametrize("kind, widths", [(nat.FN_LYAPUNOV_NN, (64, 64, 64)), (nat.FN_MLP, (64, 64, 1))])
@pytest.mark.parametrize("in_dim", [1, 2, 4, 6])
@pytest.mark.parametrize("post, want", [(0, None), (nat.FLAG_NORM1, 1), (nat.FLAG_MAXABS, 1),
                                        (nat.FLAG_SCALE, None), (nat.FLAG_ABS | nat.FLAG_NORM1 | nat.FLAG_SCALE, 1)])
def test_gradient_columns(kind, widths, in_dim, post, want):
    d = _net(kind, in_dim, widths, nat.FLAG_GRADIENT | post)
    assert _lib().slb_function_columns(d) == (in_dim if want is None else want)
    assert _eval(d) == 0, nat.last_error()


def test_columns_without_the_flag_are_unchanged():
    assert _lib().slb_function_columns(_net(flags=0)) == 1
    assert _lib().slb_function_columns(_net(nat.FN_MLP, 3, (8, 2), flags=0)) == 2


# ---------------------------------------------------------------- rejections
def test_gradient_of_a_two_output_mlp_is_rejected():
    _rejected(_eval(_net(nat.FN_MLP, 3, (8, 2))), "one-output NeuralNetwork", "3 inputs to 2 outputs")


@pytest.mark.parametrize("kind, widths", [(nat.FN_LYAPUNOV_NN, (8, 8)), (nat.FN_MLP, (8, 1))])
@pytest.mark.parametrize("in_dim", [7, 8])
def test_gradient_wider_than_max_out_is_rejected(kind, widths, in_dim):
    name = "LyapunovNetwork" if kind == nat.FN_LYAPUNOV_NN else "NeuralNetwork"
    _rejected(_eval(_net(kind, in_dim, widths)), name, "%d inputs and 1 output" % in_dim,
              "SLB_MAX_OUT = %d" % nat.SLB_MAX_OUT)


def test_gradient_with_out_dim_other_than_in_dim_is_rejected():
    _rejected(_eval(_net(in_dim=3, out_dim=1)), "needs out_dim 3", "got 1")


@pytest.mark.parametrize("kind, widths", [(nat.FN_LYAPUNOV_NN, (64, 64, 64)), (nat.FN_MLP, (64, 64, 1))])
def test_vjp_of_a_network_gradient_is_rejected(kind, widths):
    d = _net(kind, 2, widths)
    rc = _lib().slb_function_vjp(None, d, 0x2000, 10, 0x3000, 0x4000, None, None, None)
    _rejected(rc, "Hessian-vector product")
    assert _lib().slb_function_vjp_workspace(d, 10) == -1
    assert "Hessian-vector product" in nat.last_error()


def _linear(f, n_in, n_out, flags=0, addr=0x5000):
    f.kind, f.in_dim, f.out_dim, f.flags, f.matrix = nat.FN_LINEAR, n_in, n_out, flags, addr


@pytest.mark.parametrize("kind", ["linear", "quadratic", "pendulum", "cartpole"])
def test_gradient_flag_stays_rejected_on_other_kinds(kind):
    d = nat.SlbFunction()
    if kind == "linear":
        _linear(d, 2, 2, nat.FLAG_GRADIENT)
    elif kind == "quadratic":
        d.kind, d.in_dim, d.out_dim, d.flags, d.matrix = nat.FN_QUADRATIC, 2, 1, nat.FLAG_GRADIENT, 0x5000
    elif kind == "pendulum":
        d.kind, d.in_dim, d.out_dim, d.flags = nat.FN_PENDULUM, 3, 2, nat.FLAG_GRADIENT
    else:
        d.kind, d.in_dim, d.out_dim, d.flags = nat.FN_CARTPOLE, 5, 4, nat.FLAG_GRADIENT
    _rejected(_eval(d), "gradient flag is only defined for Triangulation, LyapunovNetwork and one-output "
                        "NeuralNetwork", "kind %d" % d.kind)


# ---------------------------------------------------------------- as lipschitz_lyapunov of a sweep
def _sweep(d=2, gp=False):
    cfg = nat.SlbSweep()
    g = cfg.grid
    g.ndim, g.nindex = d, 5 ** d
    for c in range(d):
        g.num_points[c], g.unit_maxes[c] = 5, 0.5
    _linear(cfg.policy, d, 1, addr=0x1000)
    if gp:
        s = cfg.gp
        s.num_outputs, s.num_factors, s.input_dim = d, 1, d + 1
        f = s.factors[0]
        f.M, f.nrb, f.scale, f.variance = 0, 0, 1.0, 1.0
        for c in range(d + 1):
            f.lengthscales[c] = 1.0
        for o in range(d):
            s.outputs[o].factor = 0
            s.outputs[o].alpha = 0x9000 + 0x100 * o
    else:
        _linear(cfg.dynamics, d + 1, d, addr=0x2000)
    cfg.lyapunov = _net(in_dim=d, flags=0, out_dim=1, addr=0x3000)
    cfg.lv_const, cfg.lf_const, cfg.tau = 1.0, 0.5, 0.01
    return cfg


def _entries():
    lib = _lib()
    return [lambda c: lib.slb_lyapunov_sweep(None, c, 0, 0, None, None, None, None, None, None),
            lambda c: lib.slb_lyapunov_sweep_filtered(None, c, 0, 0, None, None, None, None),
            lambda c: lib.slb_lyapunov_points(None, c, None, 0, None, None, None, None, None, None)]


@pytest.mark.parametrize("entry", range(3))
@pytest.mark.parametrize("d", [2, 4])
@pytest.mark.parametrize("post", [0, nat.FLAG_ABS, nat.FLAG_NORM1, nat.FLAG_MAXABS])
def test_sweep_accepts_a_network_gradient_as_lipschitz_v(entry, d, post):
    cfg = _sweep(d, gp=entry == 1)
    cfg.lipschitz_v = _net(in_dim=d, flags=nat.FLAG_GRADIENT | post, addr=0x3000)
    assert _entries()[entry](cfg) == 0, nat.last_error()


@pytest.mark.parametrize("entry", range(3))
def test_sweep_rejects_a_gradient_of_another_width(entry):
    cfg = _sweep(2, gp=entry == 1)
    cfg.lipschitz_v = _net(in_dim=3, flags=nat.FLAG_GRADIENT | nat.FLAG_NORM1, addr=0x3000)
    _rejected(_entries()[entry](cfg), "lipschitz_lyapunov", "expects 2 inputs, function takes 3")


@pytest.mark.parametrize("network_v", [False, True])
def test_filter_reports_fp64_stages_for_a_network_gradient(network_v):
    """The fp32 screening stage takes a QUADRATIC V with a constant or LINEAR L_V only: with L_V = |dV/dx|_1
    of a network the filtered sweep runs its fp64 mean stage (64), then the head stage and refine."""
    cfg = _sweep(2, gp=True)
    for f in range(cfg.gp.num_factors):
        cfg.gp.factors[f].M = 500
    if not network_v:
        cfg.lyapunov.kind, cfg.lyapunov.out_dim, cfg.lyapunov.flags = nat.FN_QUADRATIC, 1, 0
    _linear(cfg.lipschitz_v, 2, 2, nat.FLAG_NORM1)
    assert _lib().slb_filter_stage1(cfg) == (64 if network_v else 32)      # the LINEAR L_V is screened
    cfg.lipschitz_v = _net(in_dim=2, flags=nat.FLAG_GRADIENT | nat.FLAG_NORM1, addr=0x3000)
    assert _lib().slb_filter_stage1(cfg) == 64


# ---------------------------------------------------------------- the Python object, without a GPU
def test_network_gradient_object_shape_and_errors():
    net = sl.LyapunovNetwork(2, [64, 64, 64], ["tanh"] * 3, seed=0)
    g = net.gradient_function()
    assert isinstance(g, sl.NetworkGradient)
    assert g.input_dim == g.output_dim == 2
    assert g.parameters == net.parameters
    assert g.version == ("grad", net.version)
    two = sl.NeuralNetwork([3, 8, 2], ["tanh", None])
    with pytest.raises(sl.DimensionError, match="one output"):
        two.gradient_function().descriptor()
    lazy = sl.NeuralNetwork([64, 1], ["relu", None])
    with pytest.raises(sl.DimensionError, match="build"):
        lazy.gradient_function().descriptor()
    with pytest.raises(TypeError):
        sl.NetworkGradient(sl.LinearSystem(([1.0, 2.0],)))


def test_value_operator_rejects_a_network_gradient():
    """The value operator's assembly kernel is compiled without the network gradient: slb_value_operator
    rejects one (here a reward |d net / d[x, u]|_1) instead of evaluating it."""
    cfg = nat.SlbBellman()
    g = cfg.grid
    g.ndim, g.nindex = 2, 25
    for c in range(2):
        g.num_points[c], g.unit_maxes[c] = 5, 0.5
    _linear(cfg.policy, 2, 1, addr=0x1000)
    _linear(cfg.dynamics, 3, 2, addr=0x2000)
    cfg.reward = _net(in_dim=3, flags=nat.FLAG_GRADIENT | nat.FLAG_NORM1, addr=0x3000)
    v = cfg.value
    v.kind, v.in_dim, v.out_dim = nat.FN_TRIANGULATION, 2, 1
    v.matrix, v.hyperplanes, v.unit_simplices, v.nsimplex = 0x4000, 0x5000, 0x6000, 2
    v.grid = cfg.grid
    v.grid.discrete_points = 0x7000
    cfg.gamma = 0.9
    rc = _lib().slb_value_operator(None, cfg, 0, 0, 0x8000, 0x9000, 0xa000, 0xb000)
    _rejected(rc, "slb_value_operator", "network gradient")
