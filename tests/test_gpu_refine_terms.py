"""The refine pass of the filtered sweep takes each list-B point's z = [x, policy(x)], V(x) and threshold from
the point's list-A entry instead of recomputing them (csrc/gp_tile.cuh, gp_tile_body), and on the closed form
(the factored grid mean) finishes its tiles with the register-only evaluators (gp_tile_closed_kernel).  Every
first-stage plan stores those terms in its own way, so each is forced in turn -- the fp64 mean, the fp32
screening, the factored grid mean, and both head-stage schedules -- and on C2 (as bench.py builds it) must
give the flags and V(x) of the unfiltered full posterior, and a step (slb_safe_set_step) the first-fail key
and safe set that the reference reduction gives on the full posterior's flags.
"""
import numpy as np
import pytest

import bench_workloads as W
from test_gpu_parity import _sweep_details, sl  # noqa: F401

pytestmark = pytest.mark.gpu

MEAN_FP64, MEAN_FP32, MEAN_GRID = 1, 2, 3
# slb_debug_filter_stages: bit 2 fp64 mean, bit 3 / 4 head split schedule / round loop, bit 5 fp32 screening
PLANS = {"grid": (3, MEAN_GRID), "grid-split": (3 | 8, MEAN_GRID), "grid-rounds": (3 | 16, MEAN_GRID),
         "fp32": (3 | 32, MEAN_FP32), "fp32-rounds": (3 | 32 | 16, MEAN_FP32), "fp64": (3 | 4, MEAN_FP64),
         "fp64-split": (3 | 4 | 8, MEAN_FP64)}


@pytest.fixture(scope="module")
def c2(sl):  # noqa: F811
    par = W.make_pendulum(num_points=256, M=500, shared_hypers=False)
    gpu = W.build_product(par)
    assert gpu._filter_enabled(gpu.sweep_descriptor())
    return gpu, _sweep_details(gpu)


@pytest.mark.parametrize("plan", list(PLANS))
def test_refine_pass_reads_the_first_stage_terms(c2, plan):
    import torch
    from safe_learning_b200 import _device as dev
    from safe_learning_b200 import _native as nat
    gpu, full = c2
    lib = nat.load()
    mask, scheme = PLANS[plan]
    lib.slb_debug_filter_stages(mask)
    try:
        cfg = gpu.sweep_descriptor()
        assert lib.slb_filter_mean_scheme(cfg) == scheme
        begin, end = gpu._begin, gpu._end
        n = end - begin
        st = dev.stream()
        ws = dev.empty((int(lib.slb_filter_workspace(n)) // 8 + 1,), torch.int64)
        fstats = dev.zeros((4,), torch.int64)
        neg = dev.empty((n,), torch.uint8)
        values = dev.empty((n,))
        nat.check(lib.slb_lyapunov_sweep_filtered(st, cfg, begin, end, neg.data_ptr(), values.data_ptr(),
                                                  ws.data_ptr(), fstats.data_ptr()), "slb_lyapunov_sweep_filtered")
        # a step: the key folded by the three stages and the refine pass
        vdev = gpu._values_dev
        key, stats = dev.zeros((4,), torch.int64), dev.zeros((4,), torch.int64)
        safe, sneg = dev.empty((n,), torch.uint8), dev.empty((n,), torch.uint8)
        nat.check(lib.slb_safe_set_step(st, cfg, begin, end, sneg.data_ptr(), vdev.data_ptr(), None, ws.data_ptr(),
                                        dev.zeros((4,), torch.int64).data_ptr(), key.data_ptr(), safe.data_ptr(),
                                        stats.data_ptr()), "slb_safe_set_step")
        # the reference reduction on the full posterior's flags
        fneg = dev.to_device(full["negative"].astype(np.uint8), torch.uint8)
        ffws = dev.empty((int(lib.slb_first_fail_workspace(n)) // 8 + 1,), torch.int64)
        rkey, rstats = dev.zeros((4,), torch.int64), dev.zeros((4,), torch.int64)
        rsafe = dev.empty((n,), torch.uint8)
        nat.check(lib.slb_first_fail(st, vdev.data_ptr(), fneg.data_ptr(), None, n, begin, ffws.data_ptr(),
                                     rkey.data_ptr()), "slb_first_fail")
        nat.check(lib.slb_apply_prefix(st, vdev.data_ptr(), None, n, begin, rkey.data_ptr(), rsafe.data_ptr(),
                                       ffws.data_ptr(), rstats.data_ptr()), "slb_apply_prefix")
        torch.cuda.synchronize()
    finally:
        lib.slb_debug_filter_stages(3)
    assert int(fstats.cpu()[2]) > 0, "the refine pass must have points to refine"
    assert np.array_equal(neg.cpu().numpy().astype(bool), full["negative"])
    assert np.array_equal(sneg.cpu().numpy().astype(bool), full["negative"])
    assert np.array_equal(values.cpu().numpy(), full["values"])
    assert key.cpu().tolist() == rkey.cpu().tolist()
    assert stats.cpu().tolist() == rstats.cpu().tolist()
    assert np.array_equal(safe.cpu().numpy(), rsafe.cpu().numpy())
