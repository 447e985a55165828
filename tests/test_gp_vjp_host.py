"""CPU tests of the GP posterior's reverse mode (``slb_gp_vjp`` / ``slb_gp_vjp_workspace``,
include/slb200.h): the symbols, the ABI version and the host checks that run before any device work.

Every call uses fake, never dereferenced device pointers and returns before any CUDA call."""
import pytest

from safe_learning_b200 import _native as nat

FAKE = 0x1000


def _lib():
    return nat.load()


def _stack(num_outputs=2, input_dim=3, M=8):
    """A plain-RBF stack whose outputs share one factor (tables at fake addresses)."""
    s = nat.SlbGpStack()
    s.num_outputs, s.num_factors, s.input_dim = num_outputs, 1 if num_outputs else 0, input_dim
    f = s.factors[0]
    f.M, f.nrb = M, (M + 7) // 8
    f.Xs, f.Wpack = FAKE, FAKE
    f.scale, f.variance, f.kss = 1.0, 1.0, 1.0
    for c in range(input_dim):
        f.lengthscales[c] = 1.0
    for o in range(num_outputs):
        s.outputs[o].factor, s.outputs[o].beta = 0, 2.0
        s.outputs[o].alpha = s.outputs[o].gamma = FAKE
    return s


def _vjp(stack, n=4, points=FAKE, gmean=FAKE, gerr=FAKE, gin=FAKE):
    return _lib().slb_gp_vjp(None, stack, points, n, gmean, gerr, gin, None)


def _rejected(rc, *words):
    err = nat.last_error()
    assert rc == 1, err
    for w in words:
        assert w in err, err


def test_symbols_and_abi_version():
    lib = _lib()
    assert hasattr(lib, "slb_gp_vjp") and hasattr(lib, "slb_gp_vjp_workspace")
    assert lib.slb_abi_version() == 6 == nat.ABI_VERSION


def test_workspace_is_zero_for_a_mean_only_call():
    """The kernels keep their partial sums on chip: no workspace for any stack or point count."""
    for n in (0, 1, 4099, 1 << 20):
        assert _lib().slb_gp_vjp_workspace(_stack(), n) == 0, nat.last_error()
    assert _lib().slb_gp_vjp_workspace(_stack(M=0), 10) == 0


def test_workspace_rejections():
    lib = _lib()
    assert lib.slb_gp_vjp_workspace(None, 4) == -1
    assert "slb_gp_vjp_workspace: null gp" in nat.last_error()
    assert lib.slb_gp_vjp_workspace(_stack(num_outputs=0), 4) == -1
    assert "no outputs" in nat.last_error()
    assert lib.slb_gp_vjp_workspace(_stack(), -1) == -1
    assert "negative n" in nat.last_error()


def test_null_stack():
    _rejected(_lib().slb_gp_vjp(None, None, FAKE, 4, FAKE, FAKE, FAKE, None), "slb_gp_vjp: null gp")


def test_stack_without_outputs():
    _rejected(_vjp(_stack(num_outputs=0)), "slb_gp_vjp", "no outputs")


def test_invalid_stack_is_rejected_by_the_shared_validator():
    s = _stack()
    s.factors[0].nrb = 5
    _rejected(_vjp(s), "bad M/nrb")


def test_negative_n():
    _rejected(_vjp(_stack(), n=-3), "slb_gp_vjp: negative n (-3)")


def test_both_cotangents_null():
    _rejected(_vjp(_stack(), gmean=None, gerr=None), "slb_gp_vjp: both cotangents are NULL")
    _rejected(_vjp(_stack(), n=0, gmean=None, gerr=None), "both cotangents are NULL")


@pytest.mark.parametrize("which", ["points", "gin"])
def test_null_buffers(which):
    _rejected(_vjp(_stack(), **{which: None}), "slb_gp_vjp: null points or grad_points")


def test_null_gamma_with_a_mean_cotangent():
    s = _stack()
    s.outputs[1].gamma = None
    _rejected(_vjp(s), "slb_gp_vjp: GP output 1: null gamma")


def test_input_dim_beyond_the_compiled_kernels():
    _rejected(_vjp(_stack(input_dim=7)), "GP input_dim 7 not compiled (1..6)")


def test_zero_points_launch_nothing():
    assert _vjp(_stack(), n=0, points=None, gin=None) == 0, nat.last_error()
    assert _vjp(_stack(), n=0, points=None, gerr=None, gin=None) == 0, nat.last_error()
