"""The factored grid mean: stage 1 of the filtered sweep on a 2-D grid with RBF factors on [x0, x1, u] and a
saturated linear policy computes the GP mean of a tile of grid points from per-axis tables of kernel values
contracted in fp64 (csrc/filter.cu, filter_grid_mean_kernel), with a certified fp64-class error bound.
Its flags must equal the full posterior's (and those of the fp32 screening kernel that bit 5 of
slb_debug_filter_stages forces in its place) on grids that the tiles do not divide, on index ranges that
start and end mid-row, across training-set sizes, tau regimes and policy regimes; and its probed means
must lie within their bounds.
"""
import numpy as np
import pytest
from numpy.testing import assert_array_equal

import bench_workloads as W
from test_gpu_parity import sl  # noqa: F401

pytestmark = pytest.mark.gpu

FORCE_FP32 = 3 | 32


def _scheme(gpu):
    from safe_learning_b200 import _native as nat
    return nat.load().slb_filter_mean_scheme(gpu.sweep_descriptor())


def _flags(gpu, mask=3, begin=None, end=None):
    from safe_learning_b200 import _native as nat
    lib = nat.load()
    lib.slb_debug_filter_stages(mask)
    try:
        if begin is None:
            return gpu.compute_negative().cpu().numpy().copy()
        return gpu.compute_negative_range(begin, end).cpu().numpy().copy()
    finally:
        lib.slb_debug_filter_stages(3)


def _full(gpu, begin=None, end=None):
    gpu.filter = False
    try:
        return _flags(gpu, 3, begin, end)
    finally:
        gpu.filter = "auto"


def _scaled(par, k_scale):
    """The policy gain times k_scale: 0.01 leaves every point unsaturated, 30 saturates almost all."""
    par = dict(par)
    par["K"] = np.asarray(par["K"]) * k_scale
    return par


def _build(par, k_scale=1.0):
    return W.build_product(_scaled(par, k_scale))


@pytest.mark.parametrize("tau_scale", [1.0, 1 / 8., 1 / 48., 0.0])
@pytest.mark.parametrize("M", [0, 1, 8, 40, 64, 65, 100, 200, 256, 500])
def test_grid_mean_flags_equal_full_posterior(sl, M, tau_scale):
    from safe_learning_b200 import _native as nat
    par = W.make_pendulum(num_points=[45, 37], M=max(M, 1), tau_scale=tau_scale, seed=M + 11)
    if M == 0:
        par["X"], par["Y"] = par["X"][:0], par["Y"][:0]
    gpu = W.build_product(par)
    assert gpu._filter_enabled(gpu.sweep_descriptor())
    assert _scheme(gpu) == nat.MEAN_GRID_FACTORED
    gpu.reset_filter_stats()
    fast = _flags(gpu)
    stats = gpu.filter_stats
    assert stats["prior"] + stats["head"] + stats["refined"] == stats["points"] == 45 * 37
    assert_array_equal(fast, _full(gpu))
    assert_array_equal(fast, _flags(gpu, FORCE_FP32))


@pytest.mark.parametrize("k_scale", [0.01, 1.0, 30.0], ids=["unsaturated", "mixed", "saturated"])
@pytest.mark.parametrize("case", ["distinct", "shared factor", "no prior mean", "scaled targets",
                                  "short lengthscales"])
def test_grid_mean_policy_regimes(sl, case, k_scale):
    kw = dict(num_points=[70, 83], M=300, tau_scale=1 / 16., seed=5)
    if case == "shared factor":
        kw["shared_hypers"] = True
    if case == "no prior mean":
        kw["with_prior_mean"] = False
    if case == "scaled targets":
        kw["scale"] = 7.5
    par = W.make_pendulum(**kw)
    if case == "short lengthscales":
        par["lengthscales"] = [[0.2, 0.15, 0.4], [0.25, 0.12, 0.3]]
    gpu = _build(par, k_scale)
    if not gpu._filter_enabled(gpu.sweep_descriptor()):
        pytest.skip("variance floor below the filter's limit for this case")
    fast = _flags(gpu)
    assert_array_equal(fast, _full(gpu))
    assert_array_equal(fast, _flags(gpu, FORCE_FP32))


@pytest.mark.parametrize("begin,end", [(5, 45 * 37 - 3), (37 * 7 + 11, 37 * 30 + 2), (100, 101),
                                       (36, 38), (0, 37 * 17)])
def test_grid_mean_index_ranges(sl, begin, end):
    """Ranges that start and end mid-row (chunked passes, multi-rank slabs)."""
    par = W.make_pendulum(num_points=[45, 37], M=120, tau_scale=1 / 8., seed=2)
    gpu = W.build_product(par)
    fast = _flags(gpu, 3, begin, end)
    assert_array_equal(fast, _full(gpu, begin, end))
    assert_array_equal(fast, _flags(gpu, FORCE_FP32, begin, end))


def _probe(gpu, n, D=2):
    import torch
    from safe_learning_b200 import _native as nat, _device as dev
    lib = nat.load()
    mu = torch.zeros((n, D), dtype=torch.float64, device=dev.device())
    dm = torch.full((n, D), -1.0, dtype=torch.float64, device=dev.device())
    try:
        lib.slb_debug_screening_probe(mu.data_ptr(), dm.data_ptr())
        fast = gpu.compute_negative().cpu().numpy().copy()
        torch.cuda.synchronize()
    finally:
        lib.slb_debug_screening_probe(None, None)
    return fast, mu.cpu().numpy(), dm.cpu().numpy()


@pytest.mark.parametrize("k_scale", [0.01, 1.0, 30.0], ids=["unsaturated", "mixed", "saturated"])
@pytest.mark.parametrize("case", ["pendulum", "short lengthscales", "shared factor", "scaled targets",
                                  "large noise-free gammas"])
def test_grid_mean_within_its_certified_bound(sl, case, k_scale):
    """The fp64 posterior mean lies within the probed bound of every point, and the bound is
    fp64-class (relative to the scale of the mean) on every tile the bound admits."""
    kw = dict(num_points=[61, 53], M=300, tau_scale=1 / 16., seed=7)
    if case == "shared factor":
        kw["shared_hypers"] = True
    if case == "scaled targets":
        kw["scale"] = 7.5
    if case == "large noise-free gammas":
        kw["noise_std"] = 2e-4
    par = W.make_pendulum(**kw)
    if case == "short lengthscales":
        par["lengthscales"] = [[0.2, 0.15, 0.4], [0.25, 0.12, 0.3]]
    from safe_learning_b200 import _native as nat
    par = _scaled(par, k_scale)
    gpu = W.build_product(par)
    cpu = W.build_oracle(par)
    if not gpu._filter_enabled(gpu.sweep_descriptor()):
        pytest.skip("variance floor below the filter's limit for this case")
    n = gpu.discretization.nindex
    fast, mu, dm = _probe(gpu, n)
    assert (dm >= 0).all(), "the grid kernel did not write every point"
    states = cpu.discretization.all_points
    mean64, _ = gpu.dynamics(states, cpu.policy(states))
    finite = np.isfinite(dm)
    if case != "short lengthscales" and k_scale <= 1:     # (a steep policy widens the affine tiles' rho)
        assert finite.all(), "every tile of these grids is admissible: %g finite" % finite.mean()
    assert finite.mean() > 0.25, "most points left to the fp64 stages: %g" % finite.mean()
    err = np.abs(mu - mean64)
    assert (err[finite] <= dm[finite]).all(), "mean outside its certified bound: max ratio %g" % (
        (err[finite] / dm[finite]).max())
    # fp64-class: far below the fp32 screening kernel's bound at the same points
    nat.load().slb_debug_filter_stages(FORCE_FP32)
    try:
        _, _, dm32 = _probe(gpu, n)
    finally:
        nat.load().slb_debug_filter_stages(3)
    both = finite & np.isfinite(dm32)
    assert both.mean() > 0.25
    assert (dm[both] <= 1e-4 * dm32[both]).all(), "bound not fp64-class: max ratio to fp32 %g" % (
        (dm[both] / dm32[both]).max())
    assert_array_equal(fast, _full(gpu))


def test_grid_mean_fallback_for_inadmissible_tiles(sl):
    """Lengthscales far below a tile's extent leave the exponent range the bound is derived for: the
    tile's points get dm = inf and take the fp64 route, with the same flags."""
    par = W.make_pendulum(num_points=[61, 53], M=200, tau_scale=1 / 16., seed=3)
    par["lengthscales"] = [[0.02, 0.015, 0.04], [0.025, 0.012, 0.03]]
    gpu = W.build_product(par)
    if not gpu._filter_enabled(gpu.sweep_descriptor()):
        pytest.skip("variance floor below the filter's limit for this case")
    fast, mu, dm = _probe(gpu, gpu.discretization.nindex)
    assert np.isinf(dm).any()
    assert_array_equal(fast, _full(gpu))
