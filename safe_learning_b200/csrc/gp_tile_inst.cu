// gp_tile_inst.cu -- one translation unit per GP input dimension and tile size (compiled with
// -DSLB_TILE_DIN=1..6 -DSLB_TP=64|32, in parallel): the instantiations of gp_tile_kernel
// (gp_tile.cuh) -- plain RBF, covariance expressions, and (d_in = 3, 64 points) the phase-timing
// build.
#include "gp_tile.cuh"

#ifndef SLB_TILE_DIN
#error "compile with -DSLB_TILE_DIN=<1..6>"
#endif

#define SLB_CAT2(a, b) a##b
#define SLB_CAT(a, b) SLB_CAT2(a, b)

#define SLB_TILE_NAME SLB_CAT(SLB_CAT(SLB_CAT(slb_gp_tile_launch_, SLB_TILE_DIN), _), SLB_TP)

int SLB_TILE_NAME(cudaStream_t st, const slb_sweep& cfg, const slb_gp_args& a, bool kexpr,
                  bool timing) {
#if SLB_TILE_DIN == 3 && SLB_TP == 64
    if (timing) return launch_gp_tile<3, true, false>(st, cfg, a);
#else
    if (timing) {
        slb_set_error("phase timing is compiled for d_in = 3, 64-point tiles only");
        return 1;
    }
#endif
    return kexpr ? launch_gp_tile<SLB_TILE_DIN, false, true>(st, cfg, a)
                 : launch_gp_tile<SLB_TILE_DIN, false, false>(st, cfg, a);
}
