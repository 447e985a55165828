"""The work-item schedule of the factored grid mean (csrc/filter.cu, filter_grid_mean_kernel): a tile's
(factor, regime) items alternate between the CTA's two warp groups.  C2 gives each group one factor; these
cases give the groups other shares -- one shared factor whose regimes run on both groups at once, tiles
with all three regimes (an odd number of items), grids the tiles do not divide and ranges that start and
end mid-row.  Flags must equal the full posterior's and the forced fp32 kernel's, the probed mean must lie
within its bound of the fp64 posterior, and two sweeps must probe the same bytes.
"""
import numpy as np
import pytest
from numpy.testing import assert_array_equal

import bench_workloads as W
from test_gpu_grid_mean import FORCE_FP32, _flags, _full, _probe, _scaled, _scheme
from test_gpu_parity import sl  # noqa: F401

pytestmark = pytest.mark.gpu


def _regimes(gpu, cpu):
    """Per tile of 16 x 16 points, the set of policy regimes (low, high, affine) its points are in."""
    d = gpu.sweep_descriptor()
    n0, n1 = d.grid.num_points[0], d.grid.num_points[1]
    x = cpu.discretization.all_points
    u = cpu.policy(x)[:, 0]
    lo, hi = u.min(), u.max()
    reg = np.where(u == lo, 0, np.where(u == hi, 1, 2)).reshape(n0, n1)
    return [set(np.unique(reg[i:i + 16, k:k + 16])) for i in range(0, n0, 16) for k in range(0, n1, 16)]


CASES = {
    # one factor, mixed tiles: the low / high regime and the affine one run on the two groups together
    "shared factor, mixed": dict(kw=dict(num_points=[70, 83], M=300, shared_hypers=True), k=3.0),
    # tiles holding all three regimes: three items per factor, one group takes two of them
    "three regimes": dict(kw=dict(num_points=[45, 37], M=200), k=40.0),
    "three regimes, shared": dict(kw=dict(num_points=[45, 37], M=200, shared_hypers=True), k=40.0),
    "distinct, mixed": dict(kw=dict(num_points=[61, 53], M=120), k=3.0),
}


def _build(case):
    spec = CASES[case]
    par = W.make_pendulum(tau_scale=1 / 16., seed=9, **spec["kw"])
    par = _scaled(par, spec["k"])
    return W.build_product(par), W.build_oracle(par)


@pytest.mark.parametrize("case", sorted(CASES))
def test_item_schedules(sl, case):
    from safe_learning_b200 import _native as nat
    gpu, cpu = _build(case)
    if not gpu._filter_enabled(gpu.sweep_descriptor()):
        pytest.skip("variance floor below the filter's limit for this case")
    assert _scheme(gpu) == nat.MEAN_GRID_FACTORED
    tiles = _regimes(gpu, cpu)
    if "mixed" in case:
        assert any(len(t) >= 2 for t in tiles), "no mixed tile"
    if "three" in case:
        assert any(len(t) == 3 for t in tiles), "no tile with all three regimes"
    n = gpu.discretization.nindex
    fast, mu, dm = _probe(gpu, n)
    assert (dm >= 0).all(), "the grid kernel did not write every point"
    _, mu2, dm2 = _probe(gpu, n)
    assert mu.tobytes() == mu2.tobytes() and dm.tobytes() == dm2.tobytes(), "two sweeps differ"
    states = cpu.discretization.all_points
    mean64, _ = gpu.dynamics(states, cpu.policy(states))
    finite = np.isfinite(dm)
    assert finite.mean() > 0.25, "most points left to the fp64 stages: %g" % finite.mean()
    err = np.abs(mu - mean64)
    assert (err[finite] <= dm[finite]).all(), "mean outside its certified bound: max ratio %g" % (
        (err[finite] / dm[finite]).max())
    assert_array_equal(fast, _full(gpu))
    assert_array_equal(fast, _flags(gpu, FORCE_FP32))


@pytest.mark.parametrize("begin,end", [(5, 70 * 83 - 3), (83 * 7 + 11, 83 * 30 + 2), (83 * 16 - 1, 83 * 16 + 1),
                                       (200, 201)])
def test_item_schedules_on_ranges(sl, begin, end):
    """Ranges that start and end mid-row (multi-rank slabs) on a grid of mixed tiles and one shared factor."""
    gpu, _ = _build("shared factor, mixed")
    fast = _flags(gpu, 3, begin, end)
    assert_array_equal(fast, _full(gpu, begin, end))
    assert_array_equal(fast, _flags(gpu, FORCE_FP32, begin, end))
