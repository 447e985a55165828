"""Every kernel that folds the first-fail key as it decides points (slb_safe_set_step: stage 1's three mean
kernels, the head stage, the refine pass of gp_tile_kernel, and apply_prefix_kernel that reads the record)
keeps the stack frame it had before the fold and no local memory (no GPU: ``cuobjdump -res-usage`` on the
built library).  The bounds are the frames of the same kernels without the fold, from ptxas for sm_90a with
CUDA 12.9 (one exception, noted below); the fold adds two ballots, ten shuffles and two atomics per warp."""
import re

from test_stage_kernel_resources_host import usage  # noqa: F401

# kernel name pattern -> largest STACK (bytes) over its instantiations without the fold
FRAMES = {
    r"filter_grid_mean_kernelILi2EE": 0,
    r"filter_mean_kernelILi\dEE": 3584,
    r"filter_mean32_kernelILi\dELi\dEE": 3488,
    r"filter_head_kernelILi\dELi0EE": 480,
    r"filter_head_kernelILi\dELi[1-9]EE": 64,
    # 3392-3440 B without the fold; the 64-point tile with covariance expressions at d_in = 6 takes 16 B more
    r"gp_tile_kernelILi\dELb0ELb[01]ELi(32|64)EE": 3456,
    r"apply_prefix_kernelILb[01]EE": 0,
}


def test_fold_sites_keep_their_frames(usage):  # noqa: F811
    for pattern, frame in FRAMES.items():
        hits = {k: v for k, v in usage.items() if re.search(pattern, k)}
        assert hits, "no kernel matches %r" % pattern
        for name, res in hits.items():
            assert res["STACK"] <= frame and res["LOCAL"] == 0, (name, res)
