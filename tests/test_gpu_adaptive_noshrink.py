"""GPU tests of ``update_safe_set(can_shrink=False)`` with adaptive refinement (``lyapunov.py:497-606`` with
``:507-510, :540-582``): the kernels ``slb_no_shrink_scan`` / ``slb_no_shrink_resolve`` alone against a numpy
restatement of the batch loop; the product against the oracle in both refinement readings (GP and
deterministic plants, seeded previous sets, the composed path); the notebook loop of
``adaptive_safety_verification.ipynb`` cells 23-25; and the reference-generated fixture."""
import os
import sys

import numpy as np
import pytest
import torch
from numpy.testing import assert_array_equal

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import bench_workloads as W  # noqa: E402
import oracle as O  # noqa: E402
import safe_learning_b200 as sl  # noqa: E402
from adaptive_noshrink_cases import build, fixture_cases, load_fixture, replay_fixture  # noqa: E402
from safe_learning_b200 import _device as dev, _native as nat  # noqa: E402

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------ the kernels alone
def restated_loop(values, negative, prev_safe, prev_refine, initial, n_req, refined, batch, R):
    """The reference's batch loop over per-point inputs, with the mesh reading of the refined check:
    ``known`` cells pass, others pass iff ``2 <= n_req <= R`` and their ``refined`` flag is set
    (n_req = 1 re-checks the centre at tau, which is ``negative``).  Returns (safe, refinement,
    sorted position of c_max)."""
    n = len(values)
    order = np.argsort(values, kind="stable")
    known = negative | initial
    safe, refine = prev_safe[order].copy(), prev_refine[order].astype(np.float64)
    start = bound = refine_bound = 0
    for start in range(0, n, batch):
        sel = order[start:start + batch]
        safe_b, refine_b = safe[start:start + batch], refine[start:start + batch]   # views
        safe_b |= negative[sel]
        refine_b[negative[sel]] = 1
        bound = int(np.argmin(safe_b))
        refine_bound = 0
        if not (bound > 0 or not safe_b[0]):
            continue
        if R == 1:
            safe_b[bound:] = False
            refine_b[bound:] = 0
            break
        refine_b[bound:] = n_req[sel[bound:]]
        refine_b[known[sel]] = 1
        to_check = ((refine_b >= 1) & (refine_b <= R))[bound:]
        stop = len(to_check) if to_check.all() else int(np.argmin(to_check))
        if stop > 0:
            fed = sel[bound:bound + stop]
            ok = known[fed] | ((n_req[fed] >= 2) & refined[fed])
            refine_bound = len(ok) if ok.all() else int(np.argmin(ok))
            safe_b[bound:bound + refine_bound] = True
        if stop < len(to_check) or refine_bound < stop:
            safe_b[bound + refine_bound:] = False
            refine_b[bound + refine_bound:] = 0
            break
    out_safe = np.zeros(n, dtype=bool)
    out_safe[order] = safe
    out_refine = np.zeros(n, dtype=np.int64)
    out_refine[order] = refine.astype(np.int64)
    out_safe[initial] = True
    out_refine[initial] = 1
    return out_safe, out_refine, start + bound + refine_bound - 1


def _random_inputs(rng, n, R):
    values = rng.integers(0, max(2, n // 8), n).astype(np.float64)      # heavily tied
    values[rng.random(n) < 0.05] = -0.0
    p_neg = rng.choice([0.5, 0.9, 0.99, 1.0])
    negative = rng.random(n) < p_neg
    initial = rng.random(n) < 0.05
    prev_safe = initial | (rng.random(n) < rng.choice([0.0, 0.3, 0.8]))
    prev_refine = np.where(prev_safe, rng.integers(0, R + 3, n), rng.integers(0, 2, n))
    n_req = rng.choice(np.array([0., 1., 2., 3., 4., 5., 9., 16., 17., 40., np.inf]), n,
                       p=[.05, .05, .3, .2, .1, .1, .05, .05, .04, .03, .03])
    refined = rng.random(n) < rng.choice([0.7, 0.97, 1.0])
    return values, negative, prev_safe, prev_refine, initial, n_req, refined


def run_kernels(values, negative, prev_safe, prev_refine, initial, n_req, refined, batch, R):
    lib = nat.load()
    n = len(values)
    v = dev.to_device(values)
    order = torch.sort(v, stable=True).indices
    u8 = lambda a: dev.to_device(a.astype(np.uint8), torch.uint8)  # noqa: E731
    neg, prev, init = u8(negative), u8(prev_safe), u8(initial)
    nreq = dev.to_device(n_req) if R > 1 else None
    pref = dev.to_device(prev_refine.astype(np.int64), torch.int64)
    ws = dev.empty((int(lib.slb_no_shrink_workspace(n, batch)) // 8,), torch.int64)
    cand = torch.full((n,), 7, dtype=torch.uint8, device=dev.device())
    nat.check(lib.slb_no_shrink_scan(dev.stream(), order.data_ptr(), neg.data_ptr(), prev.data_ptr(),
                                     init.data_ptr(), dev.ptr(nreq), n, batch, R, ws.data_ptr(),
                                     cand.data_ptr()), "slb_no_shrink_scan")
    cand_host = cand.cpu().numpy()
    # the refined flags are only defined at the candidates: poison the rest
    ref = np.where(cand_host == 1, refined, rng_poison(n)).astype(np.uint8)
    safe = dev.empty((n,), torch.uint8)
    refinement = dev.empty((n,), torch.int64)
    result = dev.empty((2,), torch.int64)
    nat.check(lib.slb_no_shrink_resolve(dev.stream(), order.data_ptr(), v.data_ptr(), neg.data_ptr(),
                                        prev.data_ptr(), pref.data_ptr(), init.data_ptr(), dev.ptr(nreq),
                                        u8(ref).data_ptr(), n, batch, R, ws.data_ptr(), safe.data_ptr(),
                                        refinement.data_ptr(), result[0:1].data_ptr(),
                                        result[1:2].data_ptr()), "slb_no_shrink_resolve")
    res = result.cpu().numpy()
    return (safe.cpu().numpy().astype(bool), refinement.cpu().numpy(), int(res[0]),
            float(res[1:2].view(np.float64)[0]), cand_host)


def rng_poison(n):
    return np.random.default_rng(n).random(n) < 0.5


@pytest.mark.parametrize("R", [1, 4, 16])
def test_kernels_against_restated_loop(R):
    rng = np.random.default_rng(R)
    for trial in range(12):
        n = int(rng.choice([1, 2, 63, 64, 65, 300, 1000, 4097]))
        inputs = _random_inputs(rng, n, R)
        values = inputs[0]
        for batch in (1, 7, 64, n, n + 5):
            safe, refinement, pos, c_max, cand = run_kernels(*inputs, batch, R)
            exp_safe, exp_refine, exp_pos = restated_loop(*inputs, batch, R)
            msg = "R=%d n=%d batch=%d trial=%d" % (R, n, batch, trial)
            assert set(np.unique(cand)) <= {0, 1}, msg          # every point written
            if R == 1:
                assert not cand.any(), msg
            assert_array_equal(safe, exp_safe, err_msg=msg)
            assert_array_equal(refinement, exp_refine, err_msg=msg)
            assert pos == exp_pos, msg
            assert c_max == values[np.argsort(values, kind="stable")[exp_pos]], msg


def test_kernels_candidates_stop_at_the_first_hopeless_batch():
    """A batch whose first unverified point cannot be refined ends the loop: no later point is a
    candidate, and the refined flags of the points before it decide nothing after it."""
    n, batch, R = 40, 8, 4
    values = np.arange(n, dtype=np.float64)
    negative = np.ones(n, dtype=bool)
    negative[[3, 12, 13, 30]] = False
    n_req = np.full(n, 3.0)
    n_req[13] = 9.0                          # hopeless: batch 1 stops the loop
    zeros = np.zeros(n, dtype=bool)
    refined = np.ones(n, dtype=bool)
    safe, refinement, pos, _, cand = run_kernels(values, negative, zeros, np.zeros(n, np.int64), zeros,
                                                 n_req, refined, batch, R)
    assert np.flatnonzero(cand).tolist() == [3, 12]
    assert safe[:13].all() and not safe[13:].any()
    assert refinement[3] == 3 and refinement[12] == 3 and refinement[13] == 0 and pos == 12


# ------------------------------------------------------------------ the product against the oracle
@pytest.fixture
def batch64():
    old = (sl.config.gp_batch_size, O.config.gp_batch_size)
    sl.config.gp_batch_size = O.config.gp_batch_size = 64
    yield
    sl.config.gp_batch_size, O.config.gp_batch_size = old


def _compare(gpu, cpu, what):
    assert_array_equal(gpu.safe_set, cpu.safe_set, err_msg=what)
    assert_array_equal(gpu._refinement, cpu._refinement, err_msg=what)
    assert gpu.feed_dict[gpu.c_max] == cpu.c_max, what


def _seed_previous(gpu, cpu, rng, R):
    prev = cpu.safe_set | (rng.random(cpu.safe_set.size) < 0.2)
    refine = np.where(prev, rng.integers(1, R + 1, prev.size), rng.integers(0, 2, prev.size))
    for lyap in (gpu, cpu):
        lyap.safe_set = prev.copy()
        lyap._refinement = refine.copy()


@pytest.mark.parametrize("mode", ["mesh", "reference"])
@pytest.mark.parametrize("plant", ["gp", "linear"])
@pytest.mark.parametrize("tau_scale,max_refinement,safety_factor",
                         [(1 / 60., 4, 2.0), (1 / 30., 8, 2.0), (1 / 30., 4, 2.0), (1 / 60., 12, 4.0)])
def test_no_shrink_vs_oracle(batch64, mode, plant, tau_scale, max_refinement, safety_factor):
    par = W.make_pendulum(num_points=[26, 21], M=90, tau_scale=tau_scale)
    gpu, cpu = build(sl, par, plant, "product"), build(O, par, plant, "oracle")
    gpu.refinement_mode = mode
    R, s = max_refinement, safety_factor
    gpu.update_safe_set(True, R, s)
    cpu.update_safe_set(True, R, s, refinement_mode=mode)
    _compare(gpu, cpu, "can_shrink=True")
    for step in range(2):
        gpu.update_safe_set(False, R, s)
        cpu.update_safe_set(False, R, s, refinement_mode=mode)
        _compare(gpu, cpu, "no-shrink %d" % step)
    _seed_previous(gpu, cpu, np.random.default_rng(int(1 / tau_scale) + R), R)
    for step in range(2):
        gpu.update_safe_set(False, R, s, 4)                 # parallel_iterations: accepted, ignored
        cpu.update_safe_set(False, R, s, refinement_mode=mode)
        _compare(gpu, cpu, "seeded no-shrink %d" % step)
    # R = 1 and adaptive=False take the same kernels (the plain branch)
    gpu.update_safe_set(False, 1, s)
    cpu.update_safe_set(False, 1, s, refinement_mode=mode)
    _compare(gpu, cpu, "R = 1")


def test_no_shrink_composed_path_vs_oracle(batch64):
    """L_V as a numpy lambda: the sweep and the mesh checks take the composed path."""
    par = W.make_pendulum(num_points=[23, 19], M=60, tau_scale=1 / 40.)
    two_p = 2 * par["P"]
    l_v = lambda x: np.abs(np.asarray(x).dot(two_p.T))  # noqa: E731
    gpu, cpu = build(sl, par, "gp", "product", l_v), build(O, par, "gp", "oracle", l_v)
    assert gpu._is_composed()
    gpu.update_safe_set(True, 8, 2.0)
    cpu.update_safe_set(True, 8, 2.0, refinement_mode="mesh")
    _compare(gpu, cpu, "can_shrink=True")
    _seed_previous(gpu, cpu, np.random.default_rng(3), 8)
    gpu.update_safe_set(False, 8, 2.0)
    cpu.update_safe_set(False, 8, 2.0, refinement_mode="mesh")
    _compare(gpu, cpu, "no-shrink")


def test_notebook_loop_cells_23_to_25(batch64):
    """adaptive_safety_verification.ipynb cells 23-25 at test size: N_max 16, a safe sample with
    positive=True, add_data_point of the true plant's step, then update_safe_set(False, 16, 1.)."""
    par = W.make_pendulum(num_points=[31, 27], M=40, tau_scale=1 / 30.)
    gpu, cpu = build(sl, par, "gp", "product"), build(O, par, "gp", "oracle")
    gpu.update_safe_set(True, 16, 1.)
    cpu.update_safe_set(True, 16, 1., refinement_mode="mesh")
    _compare(gpu, cpu, "cell 23")
    perturbations = np.array([[-0.2], [-0.05], [0.0], [0.05], [0.2]])
    limits = np.array([[-1., 1.]])
    pl = par["plant"]
    sizes = []
    for rnd in range(4):
        for _ in range(3):
            sa_g, _ = sl.get_safe_sample(gpu, perturbations, limits, positive=True)
            sa_c, _ = O.get_safe_sample(cpu, perturbations, limits, positive=True)
            assert_array_equal(sa_g, sa_c)
            y = W._pendulum_step(sa_c, state_norm=pl["state_norm"], action_norm=pl["action_norm"],
                                 **pl["true"])
            gpu.dynamics.add_data_point(sa_c, y)
            cpu.dynamics.add_data_point(sa_c, y)
        gpu.update_safe_set(False, 16, 1.)
        cpu.update_safe_set(False, 16, 1., refinement_mode="mesh")
        _compare(gpu, cpu, "round %d" % rnd)
        sizes.append(int(cpu.safe_set.sum()))
    assert sizes[-1] > int(par["initial"].sum())


def test_errors_before_launch():
    grid = sl.GridWorld([[-1, 1]], 3)
    lyap = sl.Lyapunov(grid, sl.QuadraticFunction(np.array([[1.0]])), sl.LinearSystem(np.array([[1, 1.]])),
                       0.4, 0.3, 0.5, sl.LinearSystem(np.array([[-.1]])), adaptive=True)
    before = nat.launch_count()
    with pytest.raises(NotImplementedError, match="initial safe set"):
        lyap.update_safe_set(can_shrink=False, max_refinement=4)
    assert nat.launch_count() == before


# ------------------------------------------------------------------ the reference-generated fixture
FIX, PAR = load_fixture()


def _product_reference(lyap, can_shrink, R, s):
    lyap.refinement_mode = "reference"
    lyap.update_safe_set(can_shrink, R, s)


@pytest.mark.parametrize("case", fixture_cases(FIX), ids=lambda c: c[0])
def test_product_reference_mode_reproduces_fixture(case):
    replay_fixture(sl, "product", FIX, PAR, case, _product_reference)
