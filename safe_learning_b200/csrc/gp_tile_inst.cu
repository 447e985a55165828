// gp_tile_inst.cu -- one translation unit per GP input dimension and tile size (compiled with
// -DSLB_TILE_DIN=1..6 -DSLB_TP=64|32, in parallel): the unit's instantiation of slb_gp_tile_launch
// (gp_args.h) and through it of gp_tile_kernel (gp_tile.cuh) -- plain RBF, covariance expressions,
// (d_in = 3) the closed-form refine pass and (d_in = 3, 64 points) the phase-timing build.
#include "gp_tile.cuh"

#ifndef SLB_TILE_DIN
#error "compile with -DSLB_TILE_DIN=<1..6>"
#endif

template <int DIN, int TPV>
int slb_gp_tile_launch(cudaStream_t st, const slb_sweep& cfg, const slb_gp_args& a, bool kexpr,
                       bool timing) {
#if SLB_TILE_DIN == 3 && SLB_TP == 64
    if (timing) return launch_gp_tile<3, true, false>(st, cfg, a);
#else
    if (timing) {
        slb_set_error("phase timing is compiled for d_in = 3, 64-point tiles only");
        return 1;
    }
#endif
#if SLB_TILE_DIN == 3
    // the refine pass of the filter's closed form (two outputs; gp_tile_body)
    if (a.closed) return launch_gp_tile<3, false, false, 2>(st, cfg, a);
#endif
    return kexpr ? launch_gp_tile<DIN, false, true>(st, cfg, a)
                 : launch_gp_tile<DIN, false, false>(st, cfg, a);
}

template int slb_gp_tile_launch<SLB_TILE_DIN, SLB_TP>(cudaStream_t, const slb_sweep&, const slb_gp_args&,
                                                      bool, bool);
