"""One step of update_safe_set on a single process (slb_safe_set_step) folds the first-fail key inside the
filter's decision kernels -- stage 1, the head stage and the refine pass each fold the points they decide --
and applies the prefix rule on it.  Its key (key_value, key_index, n_ok), prefix statistics and safe set
must equal those of slb_first_fail + slb_apply_prefix on the same flags, and its flags those of the plain
filtered sweep: on C2 and its tau / 64 variant, with both refine launches doing the work, with and without
an initial safe set, on ranges that start and end mid-row, on a range longer than one pass of the filter,
on grids where every point or no point is safe, with a shared factor.  The pendulum grid is symmetric and
V(x) = V(-x), so V has ties everywhere and the index decides between them.
"""
import numpy as np
import pytest

import bench_workloads as W
from test_gpu_parity import sl  # noqa: F401

pytestmark = pytest.mark.gpu

CHUNK = 1 << 22          # points per pass of the filter (csrc/filter.cu)


def _step_and_reference(lyap, begin, end, initial):
    """(key, prefix stats, safe set, flags) of slb_safe_set_step and of the reference on its flags."""
    import torch
    from safe_learning_b200 import _device as dev
    from safe_learning_b200 import _native as nat
    lib = nat.load()
    cfg = lyap.sweep_descriptor()
    assert lyap._filter_enabled(cfg)
    st = dev.stream()
    n = end - begin
    values = lyap._values_dev[begin - lyap._begin:end - lyap._begin]
    init = None if initial is None else dev.to_device(initial[begin:end].astype(np.uint8), torch.uint8)
    ws = dev.empty((int(lib.slb_filter_workspace(n)) // 8 + 1,), torch.int64)
    ws.fill_(0x5a5a5a5a5a5a5a5a)          # the step zeroes what it needs itself
    fstats = dev.zeros((4,), torch.int64)
    neg = dev.empty((n,), torch.uint8)
    key, stats = dev.zeros((4,), torch.int64), dev.zeros((4,), torch.int64)
    key.fill_(7)
    stats.fill_(7)
    safe = dev.empty((n,), torch.uint8)
    nat.check(lib.slb_safe_set_step(st, cfg, begin, end, neg.data_ptr(), values.data_ptr(), dev.ptr(init),
                                    ws.data_ptr(), fstats.data_ptr(), key.data_ptr(), safe.data_ptr(),
                                    stats.data_ptr()), "slb_safe_set_step")
    # the plain filtered sweep gives the same flags
    plain = dev.empty((n,), torch.uint8)
    nat.check(lib.slb_lyapunov_sweep_filtered(st, cfg, begin, end, plain.data_ptr(), None, ws.data_ptr(),
                                              fstats.data_ptr()), "slb_lyapunov_sweep_filtered")
    # the reference: first-fail reduction and prefix rule on the step's flags
    ffws = dev.empty((int(lib.slb_first_fail_workspace(n)) // 8 + 1,), torch.int64)
    rkey, rstats = dev.zeros((4,), torch.int64), dev.zeros((4,), torch.int64)
    rsafe = dev.empty((n,), torch.uint8)
    nat.check(lib.slb_first_fail(st, values.data_ptr(), neg.data_ptr(), dev.ptr(init), n, begin,
                                 ffws.data_ptr(), rkey.data_ptr()), "slb_first_fail")
    nat.check(lib.slb_apply_prefix(st, values.data_ptr(), dev.ptr(init), n, begin, rkey.data_ptr(),
                                   rsafe.data_ptr(), ffws.data_ptr(), rstats.data_ptr()), "slb_apply_prefix")
    torch.cuda.synchronize()
    assert np.array_equal(neg.cpu().numpy(), plain.cpu().numpy())
    assert key.cpu().tolist() == rkey.cpu().tolist()
    assert stats.cpu().tolist() == rstats.cpu().tolist()
    assert np.array_equal(safe.cpu().numpy(), rsafe.cpu().numpy())
    return key.cpu().numpy(), neg.cpu().numpy()


def _failing_ties(lyap, begin, end, initial, flags):
    """Failing points (neither negative nor initial) that share their V with another failing point."""
    v = lyap._values_dev[begin - lyap._begin:end - lyap._begin].cpu().numpy()
    ok = flags.astype(bool)
    if initial is not None:
        ok |= initial[begin:end]
    _, counts = np.unique(v[~ok], return_counts=True)
    return int(counts[counts > 1].sum())


def _c2(tau_scale=1.0, shared=False, num_points=256, M=500):
    par = W.make_pendulum(num_points=num_points, M=M, shared_hypers=shared, tau_scale=tau_scale)
    return W.build_product(par), par


def _initial_mask(par):
    return np.asarray(par["initial"], dtype=bool)


@pytest.mark.parametrize("tau_scale", [1.0, 1 / 64.], ids=["c2", "c2-tau64"])
@pytest.mark.parametrize("with_initial", [False, True], ids=["no-initial", "initial"])
def test_fused_key_c2(sl, tau_scale, with_initial):
    lyap, par = _c2(tau_scale)
    n = lyap.discretization.nindex
    initial = _initial_mask(par) if with_initial else None
    key, flags = _step_and_reference(lyap, 0, n, initial)
    assert key[1] != np.iinfo(np.int64).max, "some point must fail"
    assert 0 < key[2] < n
    assert _failing_ties(lyap, 0, n, initial, flags) > 0, "failing points with equal V: the index decides"


@pytest.mark.parametrize("with_initial", [False, True], ids=["no-initial", "initial"])
def test_fused_key_mid_row_ranges(sl, with_initial):
    lyap, par = _c2(1 / 64.)
    initial = _initial_mask(par) if with_initial else None
    for begin, end in ((37, 256 * 200 + 101), (256 * 100 + 5, 256 * 256 - 3), (1000, 1001)):
        _step_and_reference(lyap, begin, end, initial)


def test_fused_key_persistent_refine(sl):
    """tau / 64: the refine list (~2 800 points) takes 32-point tiles; a split of 0 sends it to the
    persistent 64-point launch."""
    from safe_learning_b200 import _native as nat
    lib = nat.load()
    lyap, par = _c2(1 / 64.)
    n = lyap.discretization.nindex
    lib.slb_debug_refine_split(0)
    try:
        for initial in (None, _initial_mask(par)):
            _step_and_reference(lyap, 0, n, initial)
    finally:
        lib.slb_debug_refine_split(32 * 132)


def test_fused_key_longer_than_a_pass(sl):
    lyap, par = _c2(1.0, num_points=2100, M=100)
    n = lyap.discretization.nindex
    assert n - 2 * 977 > CHUNK
    _step_and_reference(lyap, 977, n - 977, _initial_mask(par))
    _step_and_reference(lyap, 977, n - 977, None)


def test_fused_key_all_and_none_safe(sl):
    lyap, par = _c2(1.0)
    n = lyap.discretization.nindex
    key, _ = _step_and_reference(lyap, 0, n, np.ones(n, dtype=bool))
    assert key[0] == -1                  # UINT64_MAX: no point fails
    assert key[1] == np.iinfo(np.int64).max and key[2] == n
    # a threshold nothing reaches: no point is negative
    lyap, par = _c2(1e6)
    key, flags = _step_and_reference(lyap, 0, n, None)
    assert not flags.any()
    assert key[2] == 0 and key[1] != np.iinfo(np.int64).max


def test_fused_key_shared_factor(sl):
    lyap, par = _c2(1.0, shared=True)
    n = lyap.discretization.nindex
    _step_and_reference(lyap, 0, n, _initial_mask(par))
    _step_and_reference(lyap, 0, n, None)


@pytest.mark.parametrize("tau_scale", [1.0, 1 / 64.], ids=["c2", "c2-tau64"])
def test_update_safe_set_through_step(sl, tau_scale):
    """update_safe_set takes slb_safe_set_step, also when it replays the step as a CUDA graph: its safe
    set and its count are those of the reference on the plain sweep's flags."""
    lyap, par = _c2(tau_scale)
    n = lyap.discretization.nindex
    _step_and_reference(lyap, 0, n, _initial_mask(par))
    for _ in range(3):                   # plain, captured, replayed
        lyap.update_safe_set()
        safe = lyap.safe_set.copy()
        sweep = lyap.last_sweep
    assert int(sweep["n_safe"]) == int(safe.sum())
    assert np.array_equal(safe, _reference_safe_set(lyap, _initial_mask(par)))


def _reference_safe_set(lyap, initial):
    """slb_first_fail + slb_apply_prefix on the plain filtered sweep's flags, as a host mask."""
    import torch
    from safe_learning_b200 import _device as dev
    from safe_learning_b200 import _native as nat
    lib = nat.load()
    n = lyap.discretization.nindex
    st = dev.stream()
    flags = lyap.compute_negative()
    init = dev.to_device(initial.astype(np.uint8), torch.uint8)
    ffws = dev.empty((int(lib.slb_first_fail_workspace(n)) // 8 + 1,), torch.int64)
    rkey, rstats = dev.zeros((4,), torch.int64), dev.zeros((4,), torch.int64)
    rsafe = dev.empty((n,), torch.uint8)
    nat.check(lib.slb_first_fail(st, lyap._values_dev.data_ptr(), flags.data_ptr(), init.data_ptr(), n, 0,
                                 ffws.data_ptr(), rkey.data_ptr()), "slb_first_fail")
    nat.check(lib.slb_apply_prefix(st, lyap._values_dev.data_ptr(), init.data_ptr(), n, 0, rkey.data_ptr(),
                                   rsafe.data_ptr(), ffws.data_ptr(), rstats.data_ptr()), "slb_apply_prefix")
    torch.cuda.synchronize()
    return rsafe.cpu().numpy().astype(bool)
