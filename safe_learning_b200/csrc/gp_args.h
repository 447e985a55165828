// gp_args.h -- launch arguments of gp_tile_kernel (gp_tile.cuh), shared between the per-dimension
// translation units (gp_tile_inst.cu) and the dispatcher (gp_sweep.cu).
#pragma once
#include <stdint.h>

enum { MODE_SWEEP_GRID = 0, MODE_SWEEP_STATES = 1, MODE_PREDICT = 2 };
enum { SLB_SPLIT_ITEMS = 512, SLB_SPLIT_MAX = 8, SLB_SPLIT_TICKET_BYTES = 2048 };
// bytes of the split workspace: partial sums of SLB_SPLIT_ITEMS CTAs (64-point upper bound per tile)
#define SLB_SPLIT_PARTIAL_BYTES ((size_t)SLB_SPLIT_ITEMS * SLB_MAX_OUT * (1 + SLB_MAX_OUT) * 64 * sizeof(double))
// slb_debug_refine_timing: marks per CTA of the row-split refine launch
enum { SLB_REFINE_MARKS = 16 };

// Terms of one point the decision filter (filter.cu) left undecided, carried from stage 1 to the head stage
// and, for the points of list B, to the refine pass.  Every mean scheme stores z = [x, policy(x)], thr =
// threshold(x) and vx = V(x) as the tile prologue computes them; the other fields per scheme (filter.cu).
struct filter_side { double dec0, thr, guard, vx, coef[SLB_MAX_OUT], z[SLB_MAX_IN], dm[SLB_MAX_OUT]; };

struct slb_gp_args {
    const double* points;   // MODE_SWEEP_STATES: [n, d]; MODE_PREDICT: [n, d_in]
    int64_t n;
    int64_t idx_begin;
    int32_t mode;
    int32_t want_var;
    uint8_t* negative;
    double* values;
    double* decrease;
    double* threshold;
    double* mean;
    double* err;
    const int64_t* index_list;           // refine mode: the tile's points are index_list[rel]
    const unsigned long long* count;     // refine mode: number of list entries (read on the device)
    int64_t count_min, count_max;        // refine mode: this launch works iff count_min < *count <= count_max
    // refine mode, short lists: the rows of L^-1 of one point tile are split over up to SLB_SPLIT_MAX
    // CTAs (equal triangular areas); every CTA leaves its partial sums in `split_partial`
    // [CTA][factor][1 + MAX_OUT][tile points], the last one to arrive at `split_ticket[tile]` adds
    // them in group order and finishes the tile.  NULL: no split.  Grids of at most
    // SLB_SPLIT_ITEMS CTAs.
    double* split_partial;
    int* split_ticket;
    slb_fold_target fold;   // refine mode: rec != nullptr folds every decided point (common.cuh)
    // refine pass of the filtered sweep: the stage-1 terms of list entry i are side[side_slot[i]] (its list A
    // entry); the tile reads them instead of evaluating the policy and V.  NULL: computed from the index.
    const filter_side* side;
    const int64_t* side_slot;
    // with side: the sweep is the filter's closed form (grid_mean_applicable, two outputs, d_in = 3), and the
    // tile is finished by the register-only evaluators
    int32_t closed;
    unsigned long long* marks;   // slb_debug_refine_timing: [CTA][SLB_REFINE_MARKS] %globaltimer, or NULL
    long long* timing;      // diagnostics: [tile][warp][8]: cycles in {generate, contract, epilogue, total}, globaltimer ns {start, end}, cycles waiting at barriers, 0
};

// The GP tile kernel for input dimension DIN and TPV points per CTA.  Each (DIN, TPV) is instantiated
// in a translation unit of its own (gp_tile_inst.cu), so each has a symbol of its own: templates of
// gp_tile.cuh's unnamed namespace are weak symbols shared by all units of that source file.
template <int DIN, int TPV>
int slb_gp_tile_launch(cudaStream_t st, const slb_sweep& cfg, const slb_gp_args& a, bool kexpr, bool timing);

