"""CPU tests of the shape checks on slb_sweep / slb_bellman descriptors (include/slb200.h): the column
count every host check shares with the kernels (slb_fn_columns, csrc/light.cu), and the checks that
every sweep entry point runs before it returns for an empty range.

Every call here is for an empty index range (or n = 0) with fake, never dereferenced device
pointers: the entry points return before any CUDA call whether or not a check exists, so no call can
launch a kernel."""
import pytest

from safe_learning_b200 import _native as nat


def _grid(g, d):
    g.ndim, g.nindex = d, 5 ** d
    for c in range(d):
        g.num_points[c], g.unit_maxes[c] = 5, 0.5


def _linear(f, n_in, n_out, addr, flags=0):
    f.kind, f.in_dim, f.out_dim, f.flags = nat.FN_LINEAR, n_in, n_out, flags
    f.matrix = addr


def _quadratic(f, n_in, addr):
    f.kind, f.in_dim, f.out_dim = nat.FN_QUADRATIC, n_in, 1
    f.matrix = addr


def _gp(gp, d, input_dim):
    """A d-output GP stack on one factor without training points (M = 0: no table is read)."""
    gp.num_outputs, gp.num_factors, gp.input_dim = d, 1, input_dim
    f = gp.factors[0]
    f.M, f.nrb, f.scale, f.variance = 0, 0, 1.0, 1.0
    for c in range(input_dim):
        f.lengthscales[c] = 1.0
    for o in range(d):
        gp.outputs[o].factor = 0
        gp.outputs[o].alpha = 0x9000 + 0x100 * o


def _policy(f, d, flags, out):
    _linear(f, d, out, 0x1000, flags)


def _sweep(d=2, policy_flags=0, policy_out=1, gp_in=None, dyn_out=None):
    """GP dynamics with input_dim gp_in, else linear dynamics on [x, u] (u one column) with dyn_out
    columns."""
    cfg = nat.SlbSweep()
    _grid(cfg.grid, d)
    _policy(cfg.policy, d, policy_flags, policy_out)
    if gp_in is not None:
        _gp(cfg.gp, d, gp_in)
    else:
        _linear(cfg.dynamics, d + 1, d if dyn_out is None else dyn_out, 0x2000)
    _quadratic(cfg.lyapunov, d, 0x3000)
    cfg.lv_const, cfg.lf_const, cfg.tau = 1.0, 0.5, 0.01
    return cfg


def _bellman(d=2, policy_flags=0, policy_out=1, gp_in=None, dyn_out=None):
    cfg = nat.SlbBellman()
    _grid(cfg.grid, d)
    _policy(cfg.policy, d, policy_flags, policy_out)
    if gp_in is not None:
        _gp(cfg.gp, d, gp_in)
    else:
        _linear(cfg.dynamics, d + 1, d if dyn_out is None else dyn_out, 0x2000)
    _quadratic(cfg.reward, d + 1, 0x3000)
    v = cfg.value
    v.kind, v.in_dim, v.out_dim = nat.FN_TRIANGULATION, d, 1
    v.matrix, v.hyperplanes, v.unit_simplices, v.nsimplex = 0x4000, 0x5000, 0x6000, 2
    _grid(v.grid, d)
    v.grid.discrete_points = 0x7000
    cfg.gamma = 0.9
    return cfg


def _lyapunov_sweep(cfg):
    return nat.load().slb_lyapunov_sweep(None, cfg, 0, 0, None, None, None, None, None, None)


def _lyapunov_sweep_filtered(cfg):
    return nat.load().slb_lyapunov_sweep_filtered(None, cfg, 0, 0, None, None, None, None)


def _lyapunov_points(cfg):
    return nat.load().slb_lyapunov_points(None, cfg, None, 0, None, None, None, None, None, None)


def _bellman_sweep(cfg):
    return nat.load().slb_bellman_sweep(None, cfg, 0, 0, None)


SWEEPS = [_lyapunov_sweep, _lyapunov_sweep_filtered, _lyapunov_points]


def _rejected(rc, *words):
    err = nat.last_error()
    assert rc == 1, err
    for w in words:
        assert w in err, err


# ---------------------------------------------------------------- the action width of a reduced policy
@pytest.mark.parametrize("entry", SWEEPS)
def test_sweep_rejects_gp_sized_by_out_dim_of_a_maxabs_policy(entry):
    """MAXABS reduces a two-column policy to one action column: the GP takes d + 1 inputs, not d + 2
    (the kernel would read z[d + 1], which nothing writes)."""
    cfg = _sweep(policy_flags=nat.FLAG_MAXABS, policy_out=2, gp_in=4)
    _rejected(entry(cfg), "GP input_dim 4", "state 2 + action 1")


@pytest.mark.parametrize("entry", SWEEPS)
@pytest.mark.parametrize("flag", [nat.FLAG_MAXABS, nat.FLAG_NORM1])
def test_sweep_accepts_gp_sized_by_the_columns_of_a_reduced_policy(entry, flag):
    cfg = _sweep(policy_flags=flag, policy_out=2, gp_in=3)
    assert entry(cfg) == 0, nat.last_error()


@pytest.mark.parametrize("flag", [nat.FLAG_MAXABS, nat.FLAG_NORM1])
def test_bellman_rejects_gp_sized_by_out_dim_of_a_reduced_policy(flag):
    cfg = _bellman(policy_flags=flag, policy_out=2, gp_in=4)
    _rejected(_bellman_sweep(cfg), "GP stack shape (2 outputs, 4 inputs)", "state 2 + action 1")


@pytest.mark.parametrize("flag", [nat.FLAG_MAXABS, nat.FLAG_NORM1])
def test_bellman_accepts_gp_sized_by_the_columns_of_a_reduced_policy(flag):
    cfg = _bellman(policy_flags=flag, policy_out=2, gp_in=3)
    assert _bellman_sweep(cfg) == 0, nat.last_error()


def test_fixed_action_width_is_policy_out_dim():
    """With fixed_action the policy is not evaluated: out_dim is the action dimension, whatever the
    flags say."""
    cfg = _bellman(policy_flags=nat.FLAG_MAXABS, policy_out=2, gp_in=4)
    _quadratic(cfg.reward, 4, 0x3000)
    cfg.fixed_action = 1
    assert _bellman_sweep(cfg) == 0, nat.last_error()


# ---------------------------------------------------------------- deterministic dynamics
@pytest.mark.parametrize("cols", [1, 3])
def test_sweep_rejects_dynamics_without_d_columns(cols):
    cfg = _sweep(dyn_out=cols)
    _rejected(_lyapunov_sweep(cfg), "dynamics return %d columns" % cols, "state has 2")
    _rejected(_lyapunov_points(cfg), "dynamics return %d columns" % cols, "state has 2")


@pytest.mark.parametrize("cols", [1, 3])
def test_bellman_rejects_dynamics_without_d_columns(cols):
    _rejected(_bellman_sweep(_bellman(dyn_out=cols)), "dynamics return %d columns" % cols, "state has 2")


def test_deterministic_descriptors_are_accepted():
    assert _lyapunov_sweep(_sweep()) == 0, nat.last_error()
    assert _lyapunov_points(_sweep()) == 0, nat.last_error()
    assert _bellman_sweep(_bellman()) == 0, nat.last_error()


# ---------------------------------------------------------------- L_V, reward and value widths
def test_sweep_rejects_a_two_column_lipschitz_v_in_three_dimensions():
    cfg = _sweep(d=3)
    _linear(cfg.lipschitz_v, 3, 2, 0x8000)
    _rejected(_lyapunov_sweep(cfg), "lipschitz_lyapunov returns 2 columns", "state's 3")


@pytest.mark.parametrize("cols, flags", [(1, 0), (3, 0), (3, nat.FLAG_ABS), (2, nat.FLAG_NORM1),
                                         (3, nat.FLAG_MAXABS)])
def test_sweep_accepts_lipschitz_v_with_one_or_d_columns(cols, flags):
    cfg = _sweep(d=3)
    _linear(cfg.lipschitz_v, 3, cols, 0x8000, flags)
    assert _lyapunov_sweep(cfg) == 0, nat.last_error()


def test_bellman_rejects_a_two_column_reward():
    cfg = _bellman()
    _linear(cfg.reward, 3, 2, 0x3000)
    _rejected(_bellman_sweep(cfg), "reward_function returns 2 columns", "expected 1")


def test_bellman_rejects_a_two_column_value():
    cfg = _bellman()
    cfg.value.out_dim = 2
    _rejected(_bellman_sweep(cfg), "value_function returns 2 columns", "expected 1")


# ---------------------------------------------------------------- empty ranges are validated too
@pytest.mark.parametrize("entry", SWEEPS)
def test_sweep_validates_an_empty_range(entry):
    cfg = _sweep()
    cfg.policy.kind = nat.FN_NONE
    _rejected(entry(cfg), "a policy is required")


def test_filtered_sweep_validates_its_tables_for_an_empty_range():
    cfg = _sweep(gp_in=3)
    cfg.gp.factors[0].M, cfg.gp.factors[0].nrb = 8, 1
    cfg.gp.factors[0].Xs, cfg.gp.factors[0].Wpack = 0xa000, 0xb000
    _rejected(_lyapunov_sweep_filtered(cfg), "staged table Xf")


def test_empty_range_still_checks_the_range():
    cfg = _sweep()
    rc = nat.load().slb_lyapunov_sweep(None, cfg, 26, 26, None, None, None, None, None, None)
    _rejected(rc, "slb_lyapunov_sweep: index range [26, 26) outside the grid (nindex 25)")


# ---------------------------------------------------------------- the shared column count
@pytest.mark.parametrize("kind, n_in, n_out, cparams", [
    (nat.FN_QUADRATIC, 2, 1, {}),
    (nat.FN_LYAPUNOV_NN, 2, 1, {0: 1, 1: 4}),
    (nat.FN_PENDULUM, 3, 2, {}),
    (nat.FN_CARTPOLE, 5, 4, {}),
])
def test_eval_function_accepts_every_fixed_width_kind(kind, n_in, n_out, cparams):
    f = nat.SlbFunction()
    f.kind, f.in_dim, f.out_dim, f.matrix = kind, n_in, n_out, 0x1000
    for i, v in cparams.items():
        f.cparams[i] = v
    assert nat.load().slb_eval_function(None, f, None, 0, None) == 0, nat.last_error()


def test_rollout_column_counts_come_from_the_shared_count():
    """A NORM1 two-column policy gives one action column; pendulum dynamics return two columns."""
    lib = nat.load()
    cfg = _bellman(policy_flags=nat.FLAG_NORM1, policy_out=2)
    assert lib.slb_rollout(None, cfg, None, 0, 0, 5, None, 1e-3, None, None, None, None) == 0, \
        nat.last_error()
    pend = cfg.dynamics
    pend.kind, pend.in_dim, pend.out_dim, pend.matrix = nat.FN_PENDULUM, 3, 2, None
    assert lib.slb_rollout(None, cfg, None, 0, 0, 5, None, 1e-3, None, None, None, None) == 0, \
        nat.last_error()
    cfg.policy.flags = 0
    _rejected(lib.slb_rollout(None, cfg, None, 0, 0, 5, None, 1e-3, None, None, None, None),
              "dynamics", "expects 4 inputs")
