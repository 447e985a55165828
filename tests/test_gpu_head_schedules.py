"""The head stage of the filtered sweep has two schedules (csrc/filter.cu, filter_head_kernel): the split
schedule (a warp per group of 8 list entries and factor, the fp64 means on the spare warps) that it takes
for short lists, and the round loop (a warp per group, factor after factor) for long ones.  Bits 3 and 4 of
slb_debug_filter_stages force one or the other; both must give the same flags and the same statistics, on a
short list (C2 as bench.py builds it) and on one with several groups per warp of the grid (tau / 64).
"""
import numpy as np
import pytest

import bench_workloads as W
from test_gpu_parity import _sweep_details, sl  # noqa: F401

pytestmark = pytest.mark.gpu

SPLIT, ROUNDS = 3 | 8, 3 | 16


def _sweep(gpu, lib, mask):
    lib.slb_debug_filter_stages(mask)
    try:
        gpu.reset_filter_stats()
        flags = gpu.compute_negative().cpu().numpy().copy()
        return flags, dict(gpu.filter_stats)
    finally:
        lib.slb_debug_filter_stages(3)


@pytest.mark.parametrize("tau_scale", [1.0, 1 / 64.], ids=["c2", "c2-tau64"])
def test_head_schedules_agree(sl, tau_scale):
    from safe_learning_b200 import _native as nat
    lib = nat.load()
    par = W.make_pendulum(num_points=[256, 256], M=500, shared_hypers=False, tau_scale=tau_scale)
    gpu = W.build_product(par)
    assert gpu._filter_enabled(gpu.sweep_descriptor())
    full = _sweep_details(gpu)["negative"]
    auto_flags, auto_stats = _sweep(gpu, lib, 3)
    split_flags, split_stats = _sweep(gpu, lib, SPLIT)
    round_flags, round_stats = _sweep(gpu, lib, ROUNDS)
    list_a = auto_stats["points"] - auto_stats["prior"]
    if tau_scale < 1:
        assert list_a > 8 * 132 * 16, "the list must hold more than one group per warp of the grid"
    else:
        assert list_a <= 8 * 132 * 16
    assert np.array_equal(split_flags, round_flags)
    assert np.array_equal(auto_flags, split_flags)
    assert np.array_equal(auto_flags.astype(bool), full)
    for key in ("prior", "head", "refined", "points"):
        assert split_stats[key] == round_stats[key] == auto_stats[key], key
