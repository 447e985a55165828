// filter.cu -- certified decision filter in front of the O(M^2) GP posterior of the Lyapunov sweep.
//
// The reference evaluates, for every grid point (lyapunov.py:436-441, functions.py:417-458, 507-515)
//     negative = V(mu) - V(x) + sum_j L_V(mu)_j beta_j sigma_j  <  -L_V(x) (1 + L_f) tau
// and all of its cost is sigma_j = sqrt(k** - |L^-1 k|^2): M^2 flops per point and Cholesky factor,
// against M for the mean mu = k . (L^-T alpha).  But the comparison is monotone in every sigma_j, and
//     0 <= sigma_j <= sigma_j given ANY subset of the training set <= prior sigma_j.  So:
//   stage 1  the posterior mean mu of every grid point, V(mu), L_V(mu); decide every point whose outcome
//            is the same for sigma = 0 and the prior sigma; the rest is compacted into list A.  One of
//            three mean schemes per sweep (stage1_plan):
//              SLB_MEAN_FP64  (filter_mean_kernel, thread per point) all M kernel values in fp64, one
//                exp each -- the cost of a Bellman sweep (gp_mean_staged.cuh).  Runs whenever the other
//                two cannot: covariance expressions, a V or L_V without a closed-form bound over a box
//                of means (screening_applicable), head tables that do not fit in shared memory.  Its
//                list A entries are complete: every term of the comparison (filter_side);
//              SLB_MEAN_FP32_SCREENED  (filter_mean32_kernel, thread per point) the fp32 mean of
//                gp_mean_staged.cuh with its certified bound dm;
//              SLB_MEAN_GRID_FACTORED  (filter_grid_mean_kernel, CTA per 16 x 16 tile) the factored fp64
//                mean of gp_mean_grid.cuh with its fp64-class bound: 2-D grids, z = [x0, x1, u], a linear
//                policy (grid_mean_applicable).
//              The last two decide a point when the outcome is the same over the whole box mu +- dm
//              (screened_outcome) and leave list A entries in the screened layout: z, threshold, V(x),
//              the screened mean in coef and its bound in dm;
//   stage 2  (filter_head_kernel, one CTA per SM, a warp per 8 entries of list A) the posterior variance
//            given a HEAD SUBSET of at most SLB_HEAD_RANK training points (chosen by the host in pivoted-
//            Cholesky order, its own small factor: slb_gp_factor.Wheadp / Xhead); decide with the
//            tighter bound -- screened entries first over their box, then, unless their mean is
//            fp64-class already, with the mean recomputed in fp64 by the whole CTA (head_round_means).
//            Two schedules: a warp per group, or per (group, factor) pair when the list is short;
//   rest     compacted into list B for the full fp64 posterior (gp_tile_kernel, gp_sweep.cu), which takes
//            z, V(x) and the threshold from the entry's list A terms (slot_b).
// Certification.  A point is only decided when the outcome holds with a guard band that covers
// (a) 1e-6 relative to the magnitudes involved (five orders above the rounding differences between
// two fp64 evaluation orders of the posterior; the GP tolerance of the parity contract is 1e-5) and
// (b) a computed bound of the error of stage 1's mean: it is summed as k . gamma with a kernel
// value accurate to EPS_K relative (expanded squared distance, table-driven exp with a cubic
// remainder -- tools/exp_neg_fast_check.c), so |mean error| <= (EPS_K + M 2^-52) sum_j |k_j
// gamma_j| <= (...) |gamma|_1 (slb_gp_output.gamma_l1, k <= 1 after folding the variances into
// gamma), entering the comparison through L_V(mu).  Anything non-finite goes to the full path, so
// the flags equal those of slb_lyapunov_sweep bit for bit.
// The training inputs / gamma slices are block-wide shared-memory landings: they are brought in
// by TMA bulk copies (cp.async.bulk + mbarrier, bulk_copy.cuh), double buffered, issued by one
// thread while the block works on the previous slice.
#define SLB_EVAL_NOINLINE 1
#include "common.cuh"

#include <atomic>
#include <string.h>
#include <type_traits>

#include "gp_mean_staged.cuh"
#include "gp_mean_grid.cuh"
#include "gp_args.h"

namespace {

constexpr int FT = 64;                 // stage 1: threads per CTA = points per CTA (1024 CTAs at
                                       // 256 x 256, 7 resident per SM)
constexpr int HR = SLB_HEAD_RANK;
constexpr int HT = 512;                // stage 2: threads per CTA
constexpr int HW = HT / 32;            // ... its 16 warps
constexpr int HP = 8;                  // ... list entries per warp and round: the n dimension of a DMMA
constexpr int HEAD_CTAS = SLB_NUM_SMS;  // one CTA per SM (it stages the head factors in shared memory)
constexpr int64_t CHUNK = 1 << 22;     // points per pass of the three stages (bounds the workspace)
// workspace: [0, 64) the counts, then the refine pass's tile tickets, the fold record of a step
// (slb_safe_set_step: zeroed by the same memset as the counts and tickets), the refine pass's partial
// sums, then the lists
constexpr int64_t WS_FOLD = 64 + SLB_SPLIT_TICKET_BYTES;
constexpr int64_t WS_PARTIAL = WS_FOLD + 128;
constexpr int64_t WS_HEAD = WS_PARTIAL + (int64_t)SLB_SPLIT_PARTIAL_BYTES;   // bytes before the lists
static_assert(sizeof(slb_fold) <= WS_PARTIAL - WS_FOLD && WS_FOLD % 16 == 0, "fold record slot");


// terms of one undecided point (filter_side, gp_args.h): z, thr and vx in every layout.  fp64 mean stage: dec0 =
// V(mu) - V(x), guard and coef as decide() reads them.  Screened stages: coef[j] = screened mean of output j,
// dm[j] = its certified bound (the head stage rebuilds the mean-dependent terms from them, and from an fp64
// mean where needed)

// What stage1_plan decides for a sweep: the mean scheme of stage 1 (which fixes the layout of list A) and
// the shared memory of a head CTA, as offsets in doubles from its base.  [0, 4) there: three mbarriers
// and the CTA's two counters.
struct filter_plan {
    int mean_scheme;                   // SLB_MEAN_*.  FP64: list A entries are complete.  The other two:
                                       // the screened layout; GRID_FACTORED: an entry whose bounds dm are
                                       // all finite carries an fp64-class mean (no recompute), counts[2]
                                       // is the number of the other entries
    int factors_staged;                // factors whose head tables fit in shared memory (the others are
                                       // read from global memory)
    int mean_off[SLB_MAX_OUT];         // screened: offset of factor f's [Xf | gamma_f ...] block in mbuf
    int mean_doubles;                  // screened: size of mbuf
    int tabs;                          // [512] of exp_neg_fast, [64] of exp_neg_tab: one landing
    int kbuf;                          // [HW][HR][HP] kernel values of a warp's group
    int sd;                            // split schedule: [HW * HP][SLB_MAX_OUT] sigma by entry and factor
    int wbuf, xbuf;                    // [staged][HR * HR] packed head factors, [staged][HR * d_in] inputs
    int mbuf, mu, merr;                // screened: the mean tables, [HW * HP][SLB_MAX_OUT] fp64 means of a
                                       // round's entries and their error bounds
    int need;                          // screened: ints, [2] counters (round parity) then the slots to recompute
    int doubles;                       // all of it: the CTA's dynamic shared memory
};

struct filter_args {
    int64_t n;
    int64_t idx_begin;
    uint8_t* negative;
    double* values;
    int64_t* list_a;                   // undecided after stage 1 (index relative to the range)
    filter_side* side_a;               // their terms, same order
    int64_t* list_b;                   // undecided after stage 2 -> full posterior
    int64_t* slot_b;                   // ... the list A slot of each (the refine pass reads its terms)
    unsigned long long* counts;        // [0] entries of list_a, [1] entries of list_b, [2] see filter_plan
    unsigned long long* stats;         // nullptr or [4], see slb200.h
    int chunk_rows;                    // training rows per staged slice (multiple of 8)
    int max_outputs_per_factor;
    filter_plan plan;
    int prefetch_factors;              // head stage: warm L2 with the packed factors for the refine pass
    double* probe_mu;                  // slb_debug_screening_probe: nullptr or [n, D] screened means ...
    double* probe_dm;                  // ... and their certified error bounds (inf: point left to fp64)
    unsigned long long* timing;        // slb_debug_head_timing: nullptr or [HEAD_CTAS + 1][8] %globaltimer
    unsigned long long* timing1;       // slb_debug_stage1_timing: nullptr or [tiles][8] %globaltimer
    int head_schedule;                 // head stage: 0 chosen from the list length, 1 split, 2 round loop
    slb_fold_target fold;              // rec != nullptr: every kernel folds the points it decides (common.cuh)
};

// slb_debug_head_timing: timing[slot] = the latest %globaltimer (ns) at which a warp passed a mark.
// Head CTA c writes row c at the marks below, stage 1 writes row HEAD_CTAS, slot 0 when it leaves.
enum { HM_ENTRY, HM_TABLES, HM_BOUND0, HM_BOUND, HM_SCREENED, HM_MEANS, HM_DECIDED, HM_EXIT };
SLB_DEV void timing_mark(const filter_args& a, int slot) {
    if (a.timing == nullptr || (threadIdx.x & 31) != 0) return;
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    atomicMax(a.timing + slot, t);
}
SLB_DEV void head_mark(const filter_args& a, int mark) { timing_mark(a, blockIdx.x * 8 + mark); }
// slb_debug_stage1_timing: the same, per tile of the factored grid mean (row blockIdx.x); work item k
// (one factor and regime) marks S1_ITEM + min(k, 3)
enum { S1_ENTRY, S1_PROLOGUE, S1_ITEM, S1_MEANS = S1_ITEM + 4, S1_EXIT };
SLB_DEV void stage1_mark(const filter_args& a, int mark) {
    if (a.timing1 == nullptr || (threadIdx.x & 31) != 0) return;
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    atomicMax(a.timing1 + blockIdx.x * 8 + mark, t);
}

// outcome for err_j = beta_j sigma_j with sigma_j in [0, shi_j]:  +1 decided negative (True),
// 0 decided not negative (False), -1 undecided.  term_j = L_V(mu)_j beta_j sigma_j lies between 0 and
// coef_j shi_j; anything non-finite stays undecided (NaN compares false on both sides).
SLB_DEV int decide(const filter_side& t, const double* shi, int d) {
    double ub = 0.0, lb = 0.0;
    for (int j = 0; j < d; ++j) {
        const double e = t.coef[j] * shi[j];
        ub += fmax(e, 0.0);
        lb += fmin(e, 0.0);
        if (!(e == e)) { ub = e; lb = e; break; }        // NaN: poison both sums
    }
    const double slack = t.guard + 1e-6 * (fabs(ub) + fabs(lb));
    if (t.dec0 + ub + slack < t.thr) return 1;
    if (t.dec0 + lb - slack >= t.thr) return 0;
    return -1;
}

// warp-aggregated append of the lanes with `take` to a device list; returns the slot (or -1)
SLB_DEV long long list_append(bool take, unsigned long long* counter) {
    const unsigned ballot = __ballot_sync(0xffffffffu, take);
    if (ballot == 0) return -1;
    const int lane = threadIdx.x & 31;
    unsigned long long base = 0;
    if (lane == __ffs(ballot) - 1) base = atomicAdd(counter, (unsigned long long)__popc(ballot));
    base = __shfl_sync(0xffffffffu, base, __ffs(ballot) - 1);
    return take ? (long long)(base + __popc(ballot & ((1u << lane) - 1))) : -1;
}

SLB_DEV void count_stat(bool hit, unsigned long long* slot) {
    const unsigned ballot = __ballot_sync(0xffffffffu, hit);
    if (ballot != 0 && (threadIdx.x & 31) == 0) atomicAdd(slot, (unsigned long long)__popc(ballot));
}

// V(mu), L_V(mu) -> the terms of the comparison that depend on the mean: dec0 = V(mu) - V(x), the
// coefficient of every sigma_j, and the guard band (1e-6 relative + the mean's own error bound
// through L_V(mu), x 4)                                                      (lyapunov.py:344-352)
SLB_DEV void mean_decision_terms(const slb_sweep& cfg, filter_side& t, double vx, const double* mu,
                                 const double* mean_err) {
    const int D = cfg.gp.num_outputs;
    double vm[1];
    eval_fn_small(cfg.lyapunov, mu, vm);
    t.dec0 = f64sub(vm[0], vx);
    double lvmu = 0.0;                      // sum_j |L_V(mu)_j mu_j|: scale of V's sensitivity to mu
    double lverr = 0.0;                     // sum_j |L_V(mu)_j| mean_err_j
    {
        double lv[SLB_MAX_OUT];
        int nl = 1;
        if (cfg.lipschitz_v.kind != SLB_FN_NONE) nl = eval_fn_small(cfg.lipschitz_v, mu, lv);
        else lv[0] = cfg.lv_const;
        for (int j = 0; j < SLB_MAX_OUT; ++j) {
            const double l = j < D ? (nl == 1 ? lv[0] : lv[j]) : 0.0;
            t.coef[j] = j < D ? l * cfg.gp.outputs[j].beta : 0.0;
            if (j < D) { lvmu += fabs(l * mu[j]); lverr += fabs(l) * mean_err[j]; }
        }
    }
    t.guard = 1e-6 * (fabs(vm[0]) + fabs(vx) + fabs(t.thr) + lvmu) + 4.0 * lverr + 1e-300;
}

// ---- the decision of a screened list A entry, in closed form ----------------------------------------------
// The sweeps screening_applicable accepts (D <= 4 outputs, V QUADRATIC, L_V absent or LINEAR on them): the
// terms and outcome above with compile-time D and every operand in registers -- the per-point decision of
// both screened stage-1 kernels and of the head stage behind them.  Same arithmetic, same order as
// mean_decision_terms / decide.
template <int D>
struct cf_terms { double dec0, thr, guard, coef[D]; };

// mean_decision_terms
template <int D>
SLB_DEV void cf_mean_terms(const slb_sweep& cfg, cf_terms<D>& t, double vx, const double (&mu)[D],
                           const double (&mean_err)[D]) {
    const double vm = eval_quadratic_reg<D>(cfg.lyapunov, mu);
    t.dec0 = f64sub(vm, vx);
    int nl = 1;
    slb_vec<SLB_MAX_LIN_OUT> lv;
    lv.v[0] = cfg.lv_const;
    if (cfg.lipschitz_v.kind != SLB_FN_NONE) lv = eval_linear_reg<D, SLB_MAX_LIN_OUT>(cfg.lipschitz_v, mu, nl);
    double lvmu = 0.0, lverr = 0.0;
#pragma unroll
    for (int j = 0; j < D; ++j) {
        const double l = nl == 1 ? lv.v[0] : lv.v[j];
        t.coef[j] = l * cfg.gp.outputs[j].beta;
        lvmu += fabs(l * mu[j]);
        lverr += fabs(l) * mean_err[j];
    }
    t.guard = 1e-6 * (fabs(vm) + fabs(vx) + fabs(t.thr) + lvmu) + 4.0 * lverr + 1e-300;
}

// A screened stage knows the mean only to within dm_j (certified, gp_mean_staged.cuh / gp_mean_grid.cuh).
// For V = x^T P x (QUADRATIC, optional scale) and L_V constant or a LINEAR map with abs / 1-norm / scale
// (screening_applicable) the change of the comparison over the box mu +- dm is bounded in closed form:
// |V(mu + e) - V(mu)| <= sum_i |((P + P^T) mu)_i| dm_i + sum_ij |P_ij| dm_i dm_j;  |L_V(mu + e)_j -
// L_V(mu)_j| <= |scale| sum_i |A_ji| dm_i (all rows for the 1-norm), which enters with beta_j sigma_j <=
// beta_j shi_j.  Returns the amount to add to the guard band.  The slack is that of the same sums over four
// lanes, the lanes beyond D zero: for D < 4 a mean, bound or scale that is not finite makes it NaN (0 * inf),
// which `poison` and `0.0 * sc` restate.
template <int D>
SLB_DEV double screening_slack(const slb_sweep& cfg, const double (&mu)[D], const double (&dm)[D],
                               const double (&shi)[D]) {
    const slb_function& V = cfg.lyapunov;
    double poison = 0.0;
    if constexpr (D < 4) {
#pragma unroll
        for (int i = 0; i < D; ++i) poison += 0.0 * mu[i] + 0.0 * dm[i];
    }
    double bs[D];                                           // beta_j shi_j
#pragma unroll
    for (int j = 0; j < D; ++j) bs[j] = f64mul(fabs(cfg.gp.outputs[j].beta), shi[j]);
    double dv = 0.0;
#pragma unroll
    for (int i = 0; i < D; ++i) {
        double gi = 0.0;
#pragma unroll
        for (int r = 0; r < D; ++r) gi += mu[r] * (__ldg(V.matrix + r * D + i) + __ldg(V.matrix + i * D + r));
        dv += fabs(gi) * dm[i];
#pragma unroll
        for (int j = 0; j < D; ++j) dv += fabs(__ldg(V.matrix + i * D + j)) * dm[i] * dm[j];
    }
    dv += poison;
    if (V.flags & SLB_FLAG_SCALE) dv *= fabs(V.out_scale);
    double dl = 0.0;
    const slb_function& L = cfg.lipschitz_v;
    if (L.kind == SLB_FN_LINEAR) {
        const double sc = (L.flags & SLB_FLAG_SCALE) ? fabs(L.out_scale) : 1.0;
        const int mo = L.out_dim;
        double row[SLB_MAX_LIN_OUT];                       // row[o] = sum_i |A_oi| dm_i
#pragma unroll
        for (int o = 0; o < SLB_MAX_LIN_OUT; ++o) {
            row[o] = 0.0;
#pragma unroll
            for (int i = 0; i < D; ++i)
                if (o < mo) row[o] += fabs(__ldg(L.matrix + o * D + i)) * dm[i];
        }
        if ((L.flags & SLB_FLAG_NORM1) || mo == 1) {
            double sb = bs[0];
#pragma unroll
            for (int j = 1; j < D; ++j) sb = f64add(sb, bs[j]);
            dl = sc * (row[0] + row[1] + row[2] + row[3]) * sb;
        } else {                                            // mo == D
#pragma unroll
            for (int j = 0; j < D; ++j) dl += sc * row[j] * bs[j];
            if constexpr (D < 4) dl += 0.0 * sc;
        }
    }
    return 1.000001 * (dv + dl);
}

// decide
template <int D>
SLB_DEV int cf_decide(const cf_terms<D>& t, const double (&shi)[D]) {
    double ub = 0.0, lb = 0.0;
#pragma unroll
    for (int j = 0; j < D; ++j) {
        const double e = t.coef[j] * shi[j];
        ub += fmax(e, 0.0);
        lb += fmin(e, 0.0);
        if (!(e == e)) { ub = e; lb = e; }                 // NaN: both sums stay NaN from here on
    }
    const double slack = t.guard + 1e-6 * (fabs(ub) + fabs(lb));
    if (t.dec0 + ub + slack < t.thr) return 1;
    if (t.dec0 + lb - slack >= t.thr) return 0;
    return -1;
}

// the comparison over the box mu +- dm and every sigma_j in [0, shi_j]
template <int D>
SLB_DEV int screened_outcome(const slb_sweep& cfg, double vx, double thr, const double (&mu)[D],
                             const double (&dm)[D], const double (&shi)[D]) {
    cf_terms<D> t;
    t.thr = thr;
    double zero[D];
#pragma unroll
    for (int j = 0; j < D; ++j) zero[j] = 0.0;
    cf_mean_terms<D>(cfg, t, vx, mu, zero);
    t.guard += screening_slack<D>(cfg, mu, dm, shi);
    return cf_decide<D>(t, shi);
}

// prior_sigma_bound for plain RBF factors
template <int D>
SLB_DEV void cf_prior_sigma(const slb_gp_stack& gp, double (&shi)[D]) {
#pragma unroll
    for (int j = 0; j < D; ++j) shi[j] = sqrt(gp.factors[gp.outputs[j].factor].variance);
}

// for_outputs_on_factor over D outputs: the outputs' indices in registers
template <int D, class Fn>
SLB_DEV void cf_for_outputs_on_factor(const slb_gp_stack& gp, int f, Fn&& fn) {
    unsigned mask = 0;
#pragma unroll
    for (int o = 0; o < D; ++o)
        if (gp.outputs[o].factor == f) mask |= 1u << o;
    const auto call = [&](auto no) {
        constexpr int NO = decltype(no)::value;
        int outs[NO];
        unsigned m = mask;
#pragma unroll
        for (int q = 0; q < NO; ++q) { outs[q] = __ffs(m) - 1; m &= m - 1; }
        fn(no, outs);
    };
    switch (__popc(mask)) {
    case 1: call(std::integral_constant<int, 1>{}); break;
    case 2: if constexpr (D >= 2) call(std::integral_constant<int, 2>{}); break;
    case 3: if constexpr (D >= 3) call(std::integral_constant<int, 3>{}); break;
    case 4: if constexpr (D >= 4) call(std::integral_constant<int, 4>{}); break;
    default: break;
    }
}

// ---- stage 1: what its three kernels share -----------------------------------------------------------
// x of a grid point, V(x), threshold(x), u = policy(x), z = [x, u]          (lyapunov.py:436, 284-288).
// Returns whether z is sane: the expanded squared distance needs moderate magnitudes; NaN / huge inputs
// go to the full path.
template <int DIN>
SLB_DEV bool stage1_point(const slb_sweep& cfg, int64_t index, double* z, double* vx, double* thr) {
    grid_index_to_state(cfg.grid, index, z);
    lyapunov_state_terms(cfg, z, index, vx, thr);
    double u[SLB_MAX_OUT];
    const int m = eval_fn_small(cfg.policy, z, u);
    for (int c = 0; c < m; ++c) z[cfg.grid.ndim + c] = u[c];
    bool sane = true;
#pragma unroll
    for (int c = 0; c < DIN; ++c) sane &= fabs(z[c]) < 1e100;
    return sane;
}

// sigma_j <= prior sigma_j at z, for every output     (functions.py:450 without data)
template <int DIN>
SLB_DEV void prior_sigma_bound(const slb_gp_stack& gp, const double* z, double* shi) {
    for (int j = 0; j < gp.num_outputs; ++j) {
        const slb_gp_factor& F = gp.factors[gp.outputs[j].factor];
        shi[j] = sqrt(F.kernel.num_prims > 0 ? kernel_expr_diag<DIN>(F.kernel, z) : F.variance);
    }
}

// a point leaves stage 1: its flag and V(x); an undecided one is appended to list A (returns its slot,
// -1 otherwise: the caller writes the entry's terms)
SLB_DEV long long stage1_finish(const filter_args& a, bool valid, int64_t rel, int outcome, double vx) {
    const bool undecided = valid && outcome < 0;
    if (valid) {
        a.negative[rel] = outcome > 0 ? 1 : 0;
        if (a.values != nullptr) a.values[rel] = vx;
    }
    const long long slot = list_append(undecided, a.counts + 0);
    if (undecided) a.list_a[slot] = rel;
    if (a.fold.rec != nullptr) fold_decided(a.fold, valid && outcome >= 0, outcome > 0, rel, a.idx_begin);
    if (a.stats != nullptr) {
        count_stat(valid && !undecided, a.stats + 0);
        count_stat(valid, a.stats + 3);
    }
    return slot;
}

// ... from the fp32 screening kernel (z, thr: the point's input and threshold), with its mean mu and certified
// bound dm (SLB_MAX_OUT wide, D used): the comparison over the box and the prior sigma, the list A entry in
// the screened layout (the head stage rebuilds the mean-dependent terms), the probe
template <int DIN, int D>
SLB_DEV void stage1_screened_finish(const slb_sweep& cfg, const filter_args& a, bool valid, bool sane, int64_t rel,
                                    const double* z, double thr, double vx, const double* mu_in,
                                    const double* dm_in) {
    double mu[D], dm[D], shi[D];
#pragma unroll
    for (int j = 0; j < D; ++j) { mu[j] = mu_in[j]; dm[j] = dm_in[j]; }
    if (a.probe_mu != nullptr && valid) {
#pragma unroll
        for (int o = 0; o < D; ++o) {
            a.probe_mu[rel * D + o] = mu[o];
            a.probe_dm[rel * D + o] = sane ? dm[o] : f64_inf();
        }
    }
    cf_prior_sigma<D>(cfg.gp, shi);
    const int screened = screened_outcome<D>(cfg, vx, thr, mu, dm, shi);
    const long long slot = stage1_finish(a, valid, rel, sane ? screened : -1, vx);
    if (slot >= 0) {
        filter_side* dst = a.side_a + slot;
        dst->vx = vx;
        dst->thr = thr;
#pragma unroll
        for (int c = 0; c < DIN; ++c) dst->z[c] = z[c];
#pragma unroll
        for (int j = 0; j < D; ++j) {
            dst->coef[j] = mu[j];
            dst->dm[j] = sane ? dm[j] : f64_inf();
        }
    }
}

template <int DIN>
__global__ void __launch_bounds__(FT, 7)
filter_mean_kernel(const __grid_constant__ slb_sweep cfg, const filter_args a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    prefetch_descriptor_operands(cfg);
    mean_pipe P;
    double *tab512, *tab64;
    mean_pipe_setup(P, smem_raw, DIN, a.chunk_rows, a.max_outputs_per_factor, cfg.gp, &tab512, &tab64);
    uint64_t* bar = P.bar;
    if (threadIdx.x == 0) mean_pipe_init(P, tab512);
    mean_pipe_start<DIN>(cfg.gp, P);                                   // slice 0 -> buffer 0
    __syncthreads();

    const int64_t rel0 = (int64_t)blockIdx.x * FT + threadIdx.x;
    const bool valid = rel0 < a.n;
    const int64_t rel = valid ? rel0 : a.n - 1;   // every thread stays for the block barriers
    filter_side t;
    double vx;
    const bool sane = stage1_point<DIN>(cfg, a.idx_begin + rel, t.z, &vx, &t.thr);

    // ---- posterior mean of every output (functions.py:439-442 as k . L^-T alpha)
    slb_bulk::mbar_wait(bar + 2, 0);              // exp tables have landed
    double mu[SLB_MAX_OUT];
    double mean_err[SLB_MAX_OUT];
    gp_mean_staged<DIN, true>(cfg.gp, t.z, mu, mean_err, tab512, tab64, P);

    mean_decision_terms(cfg, t, vx, mu, mean_err);

    double shi[SLB_MAX_OUT];
    prior_sigma_bound<DIN>(cfg.gp, t.z, shi);
    t.vx = vx;
    const long long slot = stage1_finish(a, valid, rel, sane ? decide(t, shi, cfg.gp.num_outputs) : -1, vx);
    if (slot >= 0) a.side_a[slot] = t;
    timing_mark(a, HEAD_CTAS * 8);
}

// ---- stage 1, fp32 screening variant ---------------------------------------------------------------
// Same role as filter_mean_kernel with the mean from the fp32 scheme of gp_mean_staged.cuh (three FFMA
// and one MUFU.EX2 per kernel value instead of twelve fp64 operations) and its certified error bound
// dm: a point is decided when the comparison has the same outcome for every mean in mu +- dm and every
// sigma between 0 and the prior's (screening_slack).  The undecided points go to list A with z,
// threshold and V(x) only; the head stage recomputes their mean in fp64 (warp-cooperatively, on ~8% of
// the grid at C2), so everything downstream of this kernel is the fp64 arithmetic of the other path.
// D = the number of outputs (screening_applicable: 1..4): the decision is the closed form.
template <int DIN, int D>
__global__ void __launch_bounds__(FT, 7)
filter_mean32_kernel(const __grid_constant__ slb_sweep cfg, const filter_args a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ double s_cen[SLB_MAX_IN];
    prefetch_descriptor_operands(cfg);
    mean_pipe P;
    mean32_bufs B;
    mean32_bufs_setup<DIN>(B, mean_pipe_setup(P, smem_raw, DIN, a.chunk_rows, a.max_outputs_per_factor, cfg.gp,
                                              nullptr, nullptr), a.chunk_rows, FT / 32);
    if (threadIdx.x == 0) mean_pipe_init(P, nullptr);
    mean_pipe_start<DIN>(cfg.gp, P);                                   // slice 0 -> buffer 0

    const int64_t rel0 = (int64_t)blockIdx.x * FT + threadIdx.x;
    const bool valid = rel0 < a.n;
    const int64_t rel = valid ? rel0 : a.n - 1;   // every thread stays for the block barriers
    double z[SLB_MAX_IN], vx, thr;
    bool sane = stage1_point<DIN>(cfg, a.idx_begin + rel, z, &vx, &thr);
    // the CTA's centre: the query point of its middle thread
    if (threadIdx.x == FT / 2) {
#pragma unroll
        for (int c = 0; c < DIN; ++c) s_cen[c] = z[c];
    }
    __syncthreads();                              // centre visible; barriers initialised
    double zcen[DIN];
#pragma unroll
    for (int c = 0; c < DIN; ++c) zcen[c] = s_cen[c];

    double mu[SLB_MAX_OUT], dm[SLB_MAX_OUT];
    gp_mean32_staged<DIN>(cfg.gp, z, zcen, mu, dm, sane, P, B);
    stage1_screened_finish<DIN, D>(cfg, a, valid, sane, rel, z, thr, vx, mu, dm);
    timing_mark(a, HEAD_CTAS * 8);
}

// ---- stage 1, factored grid mean (gp_mean_grid.cuh): one CTA per GR x GC tile of a 2-D grid -------------
// Thread t owns point t of the tile (row-major: the flag and V(x) stores are contiguous along the grid's
// axis 1) in the prologue and the decision; in between, the tile's work items (factor, regime) alternate
// between the two warp groups, which meet the points' z / regime and leave their mu / dm in shared memory.
// D = the number of outputs (= 2, the grid's dimension).  The kernel runs the closed form only
// (grid_mean_applicable): the prologue and the decision keep every per-point operand in registers.
constexpr int GRID_OUTPUTS = 2;        // a 2-D grid's GP stack has two outputs (slb_validate_sweep)

template <int D>
__global__ void __launch_bounds__(GT, 2)
filter_grid_mean_kernel(const __grid_constant__ slb_sweep cfg, const filter_args a) {
    static_assert(D == GRID_OUTPUTS, "the factored grid mean is written for z = [x0, x1, u]");
    stage1_mark(a, S1_ENTRY);
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double* smem = reinterpret_cast<double*>(smem_raw);
    double* tab = smem + GSMEM_TAB;                                      // [512] of exp_neg_fast
    double* zs = smem + GSMEM_Z;
    double* mus = smem + GSMEM_MU;
    double* dms = smem + GSMEM_DM;
    int* present = reinterpret_cast<int*>(smem + GSMEM_REG);
    int8_t* regs = reinterpret_cast<int8_t*>(present + GT / 32);
    for (int i = threadIdx.x; i < 512; i += GT) tab[i] = g_exp_tables[i];   // visible after the first barrier
    prefetch_descriptor_operands(cfg);
    // the training rows and weights every tile reads chunk by chunk: into L2 while the prologue runs
    for (int f = 0; f < cfg.gp.num_factors; ++f) {
        const size_t bytes = (size_t)padded_rows(cfg.gp.factors[f].M) * 4 * sizeof(double);
        for (size_t off = (size_t)threadIdx.x * 128; off < bytes; off += (size_t)GT * 128)
            asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char*>(cfg.gp.factors[f].Xf) + off));
    }
#pragma unroll
    for (int o = 0; o < D; ++o) {
        const size_t bytes = (size_t)padded_rows(cfg.gp.factors[cfg.gp.outputs[o].factor].M) * sizeof(double);
        for (size_t off = (size_t)threadIdx.x * 128; off < bytes; off += (size_t)GT * 128)
            asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char*>(cfg.gp.outputs[o].gamma_f) + off));
    }
    const slb_grid& g = cfg.grid;
    const int64_t n0 = g.num_points[0], n1 = g.num_points[1];
    const int64_t ntc = (n1 + GC - 1) / GC;
    const int64_t row0 = a.idx_begin / n1 + (int64_t)(blockIdx.x / ntc) * GR;
    const int64_t col0 = (int64_t)(blockIdx.x % ntc) * GC;
    const slb_function& pol = cfg.policy;

    // ---- the thread's point: x, V(x), threshold(x), u = policy(x); z and the regime go to shared memory
    const int pt = threadIdx.x;
    const int64_t gi = row0 + pt / GC, gk = col0 + pt % GC;
    const int64_t flat = gi * n1 + gk;
    const bool valid = gi < n0 && gk < n1 && flat >= a.idx_begin && flat < a.idx_begin + a.n;
    const int64_t rel = valid ? flat - a.idx_begin : 0;   // every thread stays for the block barriers
    // grid_index_to_state of (gi, gk) (a point outside the range computes a state it never uses)
    const double x[D] = {f64add(f64mul((double)gi, g.unit_maxes[0]), g.offset[0]),
                         f64add(f64mul((double)gk, g.unit_maxes[1]), g.offset[1])};
    double vx, thr;
    lyapunov_state_terms_closed<D>(cfg, x, a.idx_begin + rel, &vx, &thr);
    int cols;
    const double u = eval_linear_reg<D, 1>(pol, x, cols).v[0];
    // z must be sane: the expanded squared distance needs moderate magnitudes; NaN / huge inputs go to the
    // full path
    const bool sane = fabs(x[0]) < 1e100 && fabs(x[1]) < 1e100 && fabs(u) < 1e100;
    zs[pt * 3 + 0] = x[0];
    zs[pt * 3 + 1] = x[1];
    zs[pt * 3 + 2] = u;
    // the regime is the clip the policy computed: saturated points carry the constant itself
    {
        const double ulo = (pol.flags & SLB_FLAG_SCALE) ? f64mul(pol.lower, pol.out_scale) : pol.lower;
        const double uhi = (pol.flags & SLB_FLAG_SCALE) ? f64mul(pol.upper, pol.out_scale) : pol.upper;
        const int reg = !(valid && sane) ? -1
                        : (pol.flags & SLB_FLAG_SATURATE) && u == ulo ? 0
                        : (pol.flags & SLB_FLAG_SATURATE) && u == uhi ? 1 : 2;
        regs[pt] = (int8_t)reg;
        const unsigned rbits = __reduce_or_sync(0xffffffffu, reg >= 0 ? 1u << reg : 0u);
        if ((threadIdx.x & 31) == 0) present[threadIdx.x >> 5] = (int)rbits;
    }
#pragma unroll
    for (int o = 0; o < GNO; ++o) { mus[pt * GNO + o] = 0.0; dms[pt * GNO + o] = f64_inf(); }
    __syncthreads();                              // z, regimes and the exp table visible
    stage1_mark(a, S1_PROLOGUE);

    // ---- posterior means: the work items (factor ascending, then regime), item k on group k % GG
    int regimes = 0;
#pragma unroll
    for (int w = 0; w < GT / 32; ++w) regimes |= present[w];
    const int grp = threadIdx.x / GGT;
    int item = 0;
    for (int f = 0; f < cfg.gp.num_factors; ++f) {
        cf_for_outputs_on_factor<D>(cfg.gp, f, [&](auto no, const int* outs) {
            constexpr int NO = decltype(no)::value;
            for (int r = 0; r < 3; ++r) {
                if (!((regimes >> r) & 1)) continue;
                if (item % GG == grp) {
                    // four outputs in two passes of two: four accumulator sets do not fit 128 registers.  Every
                    // output's sum is its own, so its mean is the same in either pass.
                    constexpr int NP = NO == 4 ? 2 : NO;
#pragma unroll
                    for (int q0 = 0; q0 < NO; q0 += NP)
                        grid_mean_item<NP>(cfg, f, r, outs + q0, smem + grp * GGRP, tab, row0, col0, zs, regs, mus,
                                           dms);
                    stage1_mark(a, S1_ITEM + min(item, 3));
                }
                ++item;
            }
        });
    }
    __syncthreads();                              // every item's mu / dm visible
    stage1_mark(a, S1_MEANS);

    // ---- the comparison over mu +- dm and sigma_j in [0, prior sigma_j] (as filter_mean32_kernel)
    double mu[D], dm[D], shi[D];
#pragma unroll
    for (int j = 0; j < D; ++j) {
        mu[j] = mus[pt * GNO + j];
        dm[j] = sane ? dms[pt * GNO + j] : f64_inf();
    }
    if (a.probe_mu != nullptr && valid) {
#pragma unroll
        for (int o = 0; o < D; ++o) {
            a.probe_mu[rel * D + o] = mu[o];
            a.probe_dm[rel * D + o] = dm[o];
        }
    }
    cf_prior_sigma<D>(cfg.gp, shi);
    const int outcome = sane ? screened_outcome<D>(cfg, vx, thr, mu, dm, shi) : -1;
    const bool undecided = valid && outcome < 0;
    if (valid) {
        a.negative[rel] = outcome > 0 ? 1 : 0;
        if (a.values != nullptr) a.values[rel] = vx;
    }
    if (a.fold.rec != nullptr) fold_decided(a.fold, valid && outcome >= 0, outcome > 0, rel, a.idx_begin);
    bool fp64 = sane;                             // every bound finite: an fp64-class mean
#pragma unroll
    for (int j = 0; j < D; ++j) fp64 &= dm[j] < f64_inf();
    // per warp: list A entries, decided points, valid points, entries without an fp64-class mean; then the
    // CTA's first list A slot.  One global atomic per counter and CTA instead of one per warp.  They take
    // the place of z, which no one reads after the means.
    constexpr int NW = GT / 32;
    unsigned* s_cnt = reinterpret_cast<unsigned*>(zs);                       // [4][NW]
    unsigned long long* s_base = reinterpret_cast<unsigned long long*>(s_cnt + 4 * NW);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned und = __ballot_sync(0xffffffffu, undecided);
    {
        const unsigned dec = __ballot_sync(0xffffffffu, valid && !undecided);
        const unsigned val = __ballot_sync(0xffffffffu, valid);
        const unsigned open = __ballot_sync(0xffffffffu, undecided && !fp64);
        if (lane == 0) {
            s_cnt[0 * NW + warp] = __popc(und);
            s_cnt[1 * NW + warp] = __popc(dec);
            s_cnt[2 * NW + warp] = __popc(val);
            s_cnt[3 * NW + warp] = __popc(open);
        }
    }
    __syncthreads();
    if (threadIdx.x < 4) {
        unsigned total = 0;
#pragma unroll
        for (int w = 0; w < NW; ++w) total += s_cnt[threadIdx.x * NW + w];
        if (threadIdx.x == 0) *s_base = total != 0 ? atomicAdd(a.counts + 0, (unsigned long long)total) : 0;
        else if (total != 0 && threadIdx.x == 3) atomicAdd(a.counts + 2, (unsigned long long)total);
        else if (total != 0 && a.stats != nullptr) atomicAdd(a.stats + (threadIdx.x == 1 ? 0 : 3), (unsigned long long)total);
    }
    __syncthreads();
    if (undecided) {
        // the list A entry in the screened layout: V(x), the threshold, z, the mean and its bound (the head
        // stage rebuilds the mean-dependent terms)
        unsigned long long slot = *s_base + __popc(und & ((1u << lane) - 1));
        for (int w = 0; w < warp; ++w) slot += s_cnt[w];
        a.list_a[slot] = rel;
        filter_side* dst = a.side_a + slot;
        dst->vx = vx;
        dst->thr = thr;
        dst->z[0] = x[0];
        dst->z[1] = x[1];
        dst->z[2] = u;
#pragma unroll
        for (int j = 0; j < D; ++j) {
            dst->coef[j] = mu[j];
            dst->dm[j] = dm[j];
        }
    }
    timing_mark(a, HEAD_CTAS * 8);
    stage1_mark(a, S1_EXIT);
}

// ---- stage 2: variance given the head subset, one warp per HP undecided points ---------------------
// One CTA per SM, HW = 16 warps.  The head factors W = L_S^-1 (packed in DMMA fragment order, 32 KB each)
// and the subset's inputs are staged ONCE per CTA in shared memory by TMA bulk copies (read from global
// memory per point they cost an L2/HBM round trip per column); then the warps take the list in groups of
// HP = 8 entries: a = W k for the eight of them is one chain of DMMAs (the entries are its n dimension), so
// a fragment of W read from shared memory serves 8 points -- one point per warp makes the stage
// shared-memory-bandwidth bound.  The kernel values k_j of the HR subset points are computed two per lane
// and point and exchanged through shared memory ([row][point]: the B fragments as they lie); lane p < HP
// makes the decision of point p.

// screened lists: fp64 mean of one factor's NO outputs at the lane's point.  L lanes (a power of two,
// 4..32, consecutive in the warp) share a point: lane r of them takes rows r, r + L, ... of the
// factor's shared-memory copy [Xf | gamma_f ...] and the parts are summed by log2(L) shuffles.  The
// arithmetic of mean_factor<.., FAST = true>: expanded distance, exp_neg_fast, two partial sums.
template <int DIN, int NO>
SLB_DEV void head_mean_factor(const double* __restrict__ xf, int Mp, const double* zs, double zz, int r,
                              int L, const double* __restrict__ tab512, double* dot) {
    constexpr int W = DIN + 1;
    const double* __restrict__ gm = xf + (size_t)Mp * W;
    double d0[NO], d1[NO];
#pragma unroll
    for (int q = 0; q < NO; ++q) { d0[q] = 0.0; d1[q] = 0.0; }
    for (int j = r; j < Mp; j += 4 * L) {
        double arg[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int jc = min(j + L * u, Mp - 1);
            double row[W];
            load_row<W>(xf + jc * W, row);
            double acc = row[DIN] + zz;
#pragma unroll
            for (int c = 0; c < DIN; ++c) acc = fma(zs[c], row[c], acc);
            arg[u] = acc;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            bool far;
            double k = exp_neg_fast(arg[u], tab512, far);
            k = (far || j + L * u >= Mp) ? 0.0 : k;
            const int jc = min(j + L * u, Mp - 1);
#pragma unroll
            for (int q = 0; q < NO; ++q) {
                if (u & 1) d1[q] = fma(k, gm[q * Mp + jc], d1[q]);
                else d0[q] = fma(k, gm[q * Mp + jc], d0[q]);
            }
        }
    }
#pragma unroll
    for (int q = 0; q < NO; ++q) {
        double v = d0[q] + d1[q];
        for (int off = L >> 1; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
        dot[q] = v;
    }
}

// screened lists, once per round of the head kernel: the fp64 means of the entries the round could not
// decide from their screened means (`slots`: s = 8 w + p is entry p of warp w's group), by ALL warps of the
// CTA -- L = 512 / (number of entries) lanes per point, so a CTA with few of them (short lists: the stage's
// duration is the latency of one group) still spreads the M exps per point and factor over its threads.
// Results: mu_s / merr_s [slot][SLB_MAX_OUT] in shared memory.  The threads [tid0, tid0 + nthreads) of
// the CTA (whole warps) take part; `slots` nullptr: the entries are slots 0 .. nneed - 1.  D outputs.
template <int DIN, int D>
SLB_DEV void head_round_means(const slb_sweep& cfg, const filter_args& a, const int* slots, int nneed,
                              int64_t grp0, int64_t count, const double* mbuf, const double* tab512,
                              double* mu_s, double* merr_s, int tid0, int nthreads) {
    const int nf = cfg.gp.num_factors;
    int L = 32;                                // 512 threads: 32 lanes up to 16 entries, ..., 4 beyond 64
    while (L > 4 && nneed * L > nthreads) L >>= 1;
    const int r = threadIdx.x & (L - 1);
    const int per_warp = 32 / L;
    const int nloop = (nneed + per_warp - 1) / per_warp * per_warp;   // whole warps take part in the shuffles
    for (int i = ((int)threadIdx.x - tid0) / L; i < nloop; i += nthreads / L) {
        const bool live = i < nneed;
        const int slot = live ? (slots != nullptr ? slots[i] : i) : 0;
        const int64_t k = (grp0 + (int64_t)(slot / HP) * gridDim.x) * HP + (slot % HP);
        double z[DIN];
#pragma unroll
        for (int c = 0; c < DIN; ++c) z[c] = (live && k < count) ? a.side_a[k].z[c] : 0.0;
        for (int f = 0; f < nf; ++f) {
            const slb_gp_factor& F = cfg.gp.factors[f];
            double zs[DIN];
            double zz = 0.0;
#pragma unroll
            for (int c = 0; c < DIN; ++c) {
                zs[c] = z[c] / F.lengthscales[c];
                zz = fma(zs[c], zs[c], zz);
            }
            zz *= -0.5;
            const int Mp = padded_rows(F.M);
            const double* xf = mbuf + a.plan.mean_off[f];
            const auto factor_means = [&](auto no, const int* outs) {
                constexpr int NO = decltype(no)::value;
                double dot[NO];
                head_mean_factor<DIN, NO>(xf, Mp, zs, zz, r, L, tab512, dot);
                if (r == 0 && live) {
#pragma unroll                                     // dot and outs stay in registers
                    for (int q = 0; q < NO; ++q)
                        mean_output_finish<DIN>(F, cfg.gp.outputs[outs[q]], z, dot[q], zz, 1.0, false,
                                                &mu_s[slot * SLB_MAX_OUT + outs[q]],
                                                &merr_s[slot * SLB_MAX_OUT + outs[q]]);
                }
            };
            cf_for_outputs_on_factor<D>(cfg.gp, f, factor_means);
        }
    }
}

// lane p < HP owns list entry grp * HP + p: its terms, its index and the prior bound of every output's sigma
template <int DIN>
SLB_DEV void head_group_entries(const slb_sweep& cfg, const filter_args& a, int64_t grp, int64_t count,
                                filter_side& t, int64_t& rel, bool& mine, double* shi) {
    const int lane = threadIdx.x & 31;
    const int64_t k = grp * HP + min(lane, HP - 1);
    mine = lane < HP && k < count;
    t = filter_side{};
    rel = 0;
    if (mine) { t = a.side_a[k]; rel = a.list_a[k]; }
    prior_sigma_bound<DIN>(cfg.gp, t.z, shi);
    if (!mine)
        for (int j = 0; j < cfg.gp.num_outputs; ++j) shi[j] = 0.0;
}

// sigma of factor f (head_rows > 0) given its head subset, for the HP entries of a group on one warp
// (lane p: entry p's; the other lanes' values are meaningless)
template <int DIN, bool ALL_STAGED, bool PLAIN>
SLB_DEV double head_factor_sdev(const slb_sweep& cfg, const filter_args& a, int f, const double* z,
                                bool mine, const double* exptab, double* kw, const double* wbuf,
                                const double* xbuf, uint64_t* bar) {
    const int lane = threadIdx.x & 31;
    const slb_gp_factor& F = cfg.gp.factors[f];
    const int rows = F.head_rows;
    const bool general = !PLAIN && F.kernel.num_prims > 0;
    const double s2 = f64mul(F.scale, F.scale);
    // ALL_STAGED: the tables are known to be in shared memory (LDS instead of generic loads)
    const bool staged = ALL_STAGED || f < a.plan.factors_staged;
    const double* xh = xbuf + (size_t)f * HR * DIN;
    if (!ALL_STAGED && !staged) xh = F.Xhead;
    // kernel values of every point of the group against subset points lane and lane + 32
    // (functions.py:438); entries beyond the list carry zeros (never decided)
    double zown[DIN];                       // this lane's point in the factor's units (one division
#pragma unroll                              // per lane and dimension instead of one per point)
    for (int c = 0; c < DIN; ++c) zown[c] = general ? z[c] : z[c] / F.lengthscales[c];
#pragma unroll
    for (int p = 0; p < HP; ++p) {
        double zs[DIN];
#pragma unroll
        for (int c = 0; c < DIN; ++c) zs[c] = __shfl_sync(0xffffffffu, zown[c], p);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int j = lane + 32 * h;
            double kv = 0.0;
            if (j < rows) {
                const double* xr = xh + j * DIN;
                if (general) {
                    kv = kernel_expr_cross<DIN>(F.kernel, zs, xr, exptab);
                } else {
                    double a2 = 0.0;
#pragma unroll
                    for (int c = 0; c < DIN; ++c) { const double df = zs[c] - xr[c]; a2 = fma(df, df, a2); }
                    kv = F.variance * exp_neg_tab(-0.5 * a2, exptab);
                }
                kv = s2 * kv;
            }
            kw[j * HP + p] = kv;
        }
    }
    __syncwarp();
    double ssp = 0.0;                       // lane p: sum_i a_i^2 of point p
    // a = W k on the fp64 tensor pipe: W (64 x 64, lower triangular) pre-packed in DMMA
    // A-fragment order (row block b, k-step s: slb_gp_factor.Wheadp), the HP = 8 points are
    // the n dimension, k values [row][point] in shared memory are the B fragments as they
    // lie.  Only the blocks on or below the diagonal (s <= 2 b + 1) are multiplied: 72 DMMAs.
    const double* __restrict__ Wp = wbuf + (size_t)f * HR * HR;
    if (!ALL_STAGED && !staged) Wp = F.Wheadp;
    else slb_bulk::mbar_wait(bar + 1, 0);       // the packed factors have landed
    double acc[8][2];
#pragma unroll
    for (int b = 0; b < 8; ++b) { acc[b][0] = 0.0; acc[b][1] = 0.0; }
#pragma unroll
    for (int sk = 0; sk < 16; ++sk) {
        const double bf = kw[(4 * sk + (lane & 3)) * HP + (lane >> 2)];
#pragma unroll
        for (int b = sk / 2; b < 8; ++b) {
            const double af = Wp[(b * 16 + sk) * 32 + lane];
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                         : "+d"(acc[b][0]), "+d"(acc[b][1]) : "d"(af), "d"(bf));
        }
    }
    __syncwarp();
    // lane T holds rows 8 b + T/4 of points 2 (T%4), 2 (T%4) + 1: square, sum over b, then over
    // the 8 lanes that share T%4; lane p fetches point p's sum
    double v0 = 0.0, v1 = 0.0;
#pragma unroll
    for (int b = 0; b < 8; ++b) { v0 = fma(acc[b][0], acc[b][0], v0); v1 = fma(acc[b][1], acc[b][1], v1); }
#pragma unroll
    for (int off = 4; off < 32; off <<= 1) {
        v0 += __shfl_xor_sync(0xffffffffu, v0, off);
        v1 += __shfl_xor_sync(0xffffffffu, v1, off);
    }
    const double s0 = __shfl_sync(0xffffffffu, v0, (lane >> 1) & 3);
    const double s1 = __shfl_sync(0xffffffffu, v1, (lane >> 1) & 3);
    ssp = (lane & 1) ? s1 : s0;
    double kss = F.kss;
    if (general && mine) kss = s2 * kernel_expr_diag<DIN>(F.kernel, z);
    const double sdev = sqrt(f64sub(kss, ssp) / s2);          // NaN if negative
    return sdev;
}

// the sigma bounds of one group of HP list entries [g HP, g HP + HP) on one warp (lane p: entry p, loaded by
// head_group_entries), factor after factor; D outputs (CD > 0: screened entries, plain RBF factors)
template <int DIN, bool ALL_STAGED, int CD, int D>
SLB_DEV void head_group_bound(const slb_sweep& cfg, const filter_args& a, const double* z, bool mine,
                              const double* exptab, double* kw, const double* wbuf, const double* xbuf,
                              uint64_t* bar, double (&shi)[D]) {
    slb_bulk::mbar_wait(bar + 0, 0);            // exp tables and subset inputs have landed
    head_mark(a, HM_TABLES);
    for (int f = 0; f < cfg.gp.num_factors; ++f) {
        if (cfg.gp.factors[f].head_rows <= 0) continue;
        const double sdev = head_factor_sdev<DIN, ALL_STAGED, (CD > 0)>(cfg, a, f, z, mine, exptab, kw, wbuf, xbuf,
                                                                        bar);
#pragma unroll
        for (int j = 0; j < D; ++j)
            if (j < cfg.gp.num_outputs && cfg.gp.outputs[j].factor == f) shi[j] = sdev;
        if (f == 0) head_mark(a, HM_BOUND0);
    }
    head_mark(a, HM_BOUND);
}

// The decision of a list entry from what stage 1 left in it and the bound shi of every sigma, the same in
// both schedules.  A complete entry (fp64 mean stage): the comparison itself.
SLB_DEV int head_entry_decision(const slb_sweep& cfg, const filter_args&, filter_side& t, const double* shi,
                                bool mine, double&, bool& need) {
    need = false;
    return mine ? decide(t, shi, cfg.gp.num_outputs) : 0;
}

// A screened entry (D outputs): the entry's fields in registers, the decision of stage 1 (screened_outcome)
// over the box of its screened mean first -- most are decided by the tighter variance bound alone; `need`:
// it is still open and has no fp64-class mean, so head_mean_decision follows with vx = V(x).  Only z goes
// in before the sigma bounds; the other fields are loaded for the decision (fewer registers live across the
// DMMA chain).
template <int DIN, int D>
struct cf_entry { int k; int64_t rel; double vx, thr, z[DIN], mu[D], dm[D]; };   // k: list index, -1: none

template <int DIN, int D>
SLB_DEV void head_group_entries(const slb_sweep& cfg, const filter_args& a, int64_t grp, int64_t count,
                                cf_entry<DIN, D>& t, int64_t& rel, bool& mine, double (&shi)[D]) {
    const int lane = threadIdx.x & 31;
    const int64_t k = grp * HP + min(lane, HP - 1);
    mine = lane < HP && k < count;
    t.k = mine ? (int)k : -1;
#pragma unroll
    for (int c = 0; c < DIN; ++c) t.z[c] = mine ? a.side_a[k].z[c] : 0.0;
    rel = 0;                                    // t.rel, loaded with the decision's fields
    cf_prior_sigma<D>(cfg.gp, shi);
    if (!mine) {
#pragma unroll
        for (int j = 0; j < D; ++j) shi[j] = 0.0;
    }
}

template <int DIN, int D>
SLB_DEV int head_entry_decision(const slb_sweep& cfg, const filter_args& a, cf_entry<DIN, D>& t,
                                const double (&shi)[D], bool mine, double& vx, bool& need) {
    t.rel = 0;
    t.vx = 0.0;
    t.thr = 0.0;
#pragma unroll
    for (int j = 0; j < D; ++j) { t.mu[j] = 0.0; t.dm[j] = 0.0; }
    if (t.k >= 0) {
        t.rel = a.list_a[t.k];
        const filter_side* e = a.side_a + t.k;
        t.vx = e->vx;
        t.thr = e->thr;
#pragma unroll
        for (int j = 0; j < D; ++j) { t.mu[j] = e->coef[j]; t.dm[j] = e->dm[j]; }
    }
    vx = t.vx;
    const int screened = screened_outcome<D>(cfg, vx, t.thr, t.mu, t.dm, shi);
    const int outcome = mine ? screened : 0;
    // an entry of the factored grid kernel with finite bounds carries an fp64-class mean: decided from its
    // box or sent to the refine pass without recomputing the mean.  An fp32-screened mean is recomputed.
    bool finite = a.plan.mean_scheme == SLB_MEAN_GRID_FACTORED;
#pragma unroll
    for (int j = 0; j < D; ++j) finite &= t.dm[j] < f64_inf();
    need = mine && outcome < 0 && !finite;
    head_mark(a, HM_SCREENED);
    return outcome;
}

// ... and with the fp64 mean head_round_means left for its slot: the comparison of the fp64 mean stage
template <int DIN, int D>
SLB_DEV int head_mean_decision(const slb_sweep& cfg, cf_entry<DIN, D>& t, double vx, const double (&shi)[D],
                               const double* mu_s, const double* merr_s, int slot) {
    double mu[D], merr[D];
#pragma unroll
    for (int j = 0; j < D; ++j) {
        mu[j] = mu_s[slot * SLB_MAX_OUT + j];
        merr[j] = merr_s[slot * SLB_MAX_OUT + j];
    }
    cf_terms<D> terms;
    terms.thr = t.thr;
    cf_mean_terms<D>(cfg, terms, vx, mu, merr);
    return cf_decide<D>(terms, shi);
}

// the grid index of an entry (complete: the one head_group_entries loaded) and its list A slot (lane p of group
// grp holds entry grp HP + p)
SLB_DEV int64_t entry_rel(const filter_side&, int64_t rel) { return rel; }
template <int DIN, int D>
SLB_DEV int64_t entry_rel(const cf_entry<DIN, D>& t, int64_t) { return t.rel; }
SLB_DEV int64_t entry_slot(const filter_side&, int64_t grp) { return grp * HP + (threadIdx.x & 31); }
template <int DIN, int D>
SLB_DEV int64_t entry_slot(const cf_entry<DIN, D>& t, int64_t) { return t.k; }

// every copy lands in this CTA's shared memory before the CTA may leave
SLB_DEV void head_wait_landings(uint64_t* bar) {
    for (int b = 0; b < 3; ++b) slb_bulk::mbar_wait(bar + b, 0);
}

// a lane's final outcome: the flag of a decided point, list B (and its list A slot k) for an undecided one
// (warp-collective)
SLB_DEV void head_group_finish(const filter_args& a, bool mine, int outcome, int64_t rel, int64_t k,
                               unsigned* s_stat) {
    const int lane = threadIdx.x & 31;
    const bool undecided = mine && outcome < 0;
    if (mine && outcome >= 0) a.negative[rel] = outcome > 0 ? 1 : 0;
    if (a.fold.rec != nullptr) fold_decided(a.fold, mine && outcome >= 0, outcome > 0, rel, a.idx_begin);
    const long long slot = list_append(undecided, a.counts + 1);
    if (undecided) {
        a.list_b[slot] = rel;
        a.slot_b[slot] = k;
    }
    const unsigned dec = __ballot_sync(0xffffffffu, mine && !undecided);
    const unsigned und = __ballot_sync(0xffffffffu, undecided);
    if (lane == 0) {
        if (dec) atomicAdd(s_stat + 0, (unsigned)__popc(dec));
        if (und) atomicAdd(s_stat + 1, (unsigned)__popc(und));
    }
}

// CD = 0: complete list entries (SLB_MEAN_FP64).  CD = D > 0: screened entries of D outputs (both screened
// schemes), loaded into registers and decided by the closed form of stage 1, their fp64 means recomputed
// where the box leaves them open (head_round_means)
template <int DIN, int CD>
__global__ void __launch_bounds__(HT, 1)
filter_head_kernel(const __grid_constant__ slb_sweep cfg, const filter_args a) {
    constexpr int ND = CD > 0 ? CD : SLB_MAX_OUT;
    using entry_t = std::conditional_t<(CD > 0), cf_entry<DIN, ND>, filter_side>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    if (threadIdx.x == 0) head_mark(a, HM_ENTRY);
    prefetch_descriptor_operands(cfg);
    // three landings, each waited for just before its first use: (a) the exp tables and the subsets'
    // inputs (kernel values), (b) the packed head factors (DMMA), (c) screened lists: [Xf | gamma_f]
    const filter_plan& lay = a.plan;
    double* smem = reinterpret_cast<double*>(smem_raw);
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem);                 // [3]
    unsigned* s_stat = reinterpret_cast<unsigned*>(smem + 3);          // decided / undecided by this CTA
    double* tab512 = smem + lay.tabs;                                  // (screened lists: exp_neg_fast)
    double* exptab = tab512 + 512;
    double* kbuf = smem + lay.kbuf;
    double* wbuf = smem + lay.wbuf;
    double* xbuf = smem + lay.xbuf;
    double* mbuf = smem + lay.mbuf;
    const int nf = cfg.gp.num_factors;
    // screened lists: fp64 means are recomputed here only for entries without an fp64-class one (all of them
    // after the fp32 screening kernel, those the grid kernel left with dm = inf: counts[2])
    const bool means = CD > 0 && (lay.mean_scheme != SLB_MEAN_GRID_FACTORED || a.counts[2] != 0);
    if (threadIdx.x == 0) {
        for (int b = 0; b < 3; ++b) slb_bulk::mbar_init(bar + b, 1);
        slb_bulk::fence_barrier_init();
        slb_bulk::fence_proxy_async();
        unsigned xbytes = 576 * sizeof(double), wbytes = 0;
        for (int f = 0; f < lay.factors_staged; ++f)
            if (cfg.gp.factors[f].head_rows > 0) {
                xbytes += (unsigned)(HR * DIN) * sizeof(double);
                wbytes += (unsigned)(HR * HR) * sizeof(double);
            }
        slb_bulk::mbar_arrive_expect_tx(bar + 0, xbytes);
        slb_bulk::copy_g2s(tab512, g_exp_tables, 576 * sizeof(double), bar + 0);
        for (int f = 0; f < lay.factors_staged; ++f)
            if (cfg.gp.factors[f].head_rows > 0)
                slb_bulk::copy_g2s(xbuf + (size_t)f * HR * DIN, cfg.gp.factors[f].Xhead,
                                   HR * DIN * sizeof(double), bar + 0);
        slb_bulk::mbar_arrive_expect_tx(bar + 1, wbytes);
        for (int f = 0; f < lay.factors_staged; ++f)
            if (cfg.gp.factors[f].head_rows > 0)
                slb_bulk::copy_g2s(wbuf + (size_t)f * HR * HR, cfg.gp.factors[f].Wheadp,
                                   HR * HR * sizeof(double), bar + 1);
        slb_bulk::mbar_arrive_expect_tx(bar + 2, means ? (unsigned)lay.mean_doubles * sizeof(double) : 0u);
        if (means) {
            for (int f = 0; f < nf; ++f) {
                const slb_gp_factor& F = cfg.gp.factors[f];
                const int Mp = padded_rows(F.M);
                if (Mp == 0) continue;
                double* dst = mbuf + lay.mean_off[f];
                slb_bulk::copy_g2s(dst, F.Xf, (unsigned)(Mp * (DIN + 1)) * sizeof(double), bar + 2);
                dst += (size_t)Mp * (DIN + 1);
                for (int o = 0; o < cfg.gp.num_outputs; ++o) {
                    if (cfg.gp.outputs[o].factor != f) continue;
                    slb_bulk::copy_g2s(dst, cfg.gp.outputs[o].gamma_f, (unsigned)Mp * sizeof(double), bar + 2);
                    dst += Mp;
                }
            }
        }
    }
    // ---- behind the staging: the refine pass that follows streams every factor's packed L^-1 (1 MB at
    // M = 500); if it is not L2-resident by then (first sweep after a cache update, or evicted in
    // between) its CTAs start with HBM round trips in lockstep: prefetch it.
    if (a.prefetch_factors) {
        for (int f = 0; f < nf; ++f) {
            const slb_gp_factor& F = cfg.gp.factors[f];
            const char* base = reinterpret_cast<const char*>(F.Wpack);
            const size_t nbytes = (size_t)F.nrb * (F.nrb + 1) * 32 * sizeof(double);
            for (size_t off = ((size_t)blockIdx.x * HT + threadIdx.x) * 128; off < nbytes;
                 off += (size_t)gridDim.x * HT * 128)
                asm volatile("prefetch.global.L2 [%0];" ::"l"(base + off));
            // ... and the training inputs its generation phases stage panel by panel
            const char* xs = reinterpret_cast<const char*>(F.Xs);
            const size_t xbytes = (size_t)F.M * DIN * sizeof(double);
            if (blockIdx.x == (unsigned)f)
                for (size_t off = (size_t)threadIdx.x * 128; off < xbytes; off += (size_t)HT * 128)
                    asm volatile("prefetch.global.L2 [%0];" ::"l"(xs + off));
        }
        if (blockIdx.x == gridDim.x - 1 && threadIdx.x < cfg.gp.num_outputs) {
            const slb_gp_output& G = cfg.gp.outputs[threadIdx.x];
            const size_t abytes = (size_t)cfg.gp.factors[G.factor].M * sizeof(double);
            for (size_t off = 0; off < abytes; off += 128)
                asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char*>(G.alpha) + off));
        }
    }
    if (threadIdx.x < 2) s_stat[threadIdx.x] = 0;
    if constexpr (CD > 0)
        if (threadIdx.x < 2) reinterpret_cast<int*>(smem + lay.need)[threadIdx.x] = 0;
    __syncthreads();
    const int64_t count = (int64_t)a.counts[0];
    const int64_t nwarps = (int64_t)gridDim.x * HW;
    const int64_t ngroups = (count + HP - 1) / HP;
    // groups are dealt round-robin over the CTAs (group g: CTA g % gridDim, warp g / gridDim): a short
    // list spreads over all SMs instead of filling the 16 warps of the first few
    if ((int64_t)blockIdx.x >= ngroups) {                              // no group for this CTA
        head_wait_landings(bar);
        if (threadIdx.x == 0) head_mark(a, HM_EXIT);
        return;
    }
    const int warp = threadIdx.x >> 5;
    double* kw = kbuf + warp * HR * HP;
    double* sd_s = smem + lay.sd;
    double* mu_s = smem + lay.mu;
    double* merr_s = smem + lay.merr;
    int* need_s = reinterpret_cast<int*>(smem + lay.need);
    // Short lists (one round, and a warp to spare beside one warp per group and factor: C2) are latency
    // bound: the split schedule gives every (group, factor) pair a warp of its own, and the spare warps
    // compute the fp64 means of all the round's entries meanwhile (used only where the screened box
    // leaves an entry open).  Longer lists keep the round loop below, factor after factor on one warp.
    const int ng_first = (int)min((int64_t)HW, (ngroups - blockIdx.x + gridDim.x - 1) / gridDim.x);
    const bool split = a.head_schedule == 1 ||
                       (a.head_schedule == 0 && ngroups <= nwarps && ng_first * nf < HW);
    if (split) {
        const int lane = threadIdx.x & 31;
        for (int64_t grp0 = blockIdx.x; grp0 < ngroups; grp0 += nwarps) {
            // this CTA's groups of the round: grp0 + i gridDim, i < ngr (group i's decisions on warp i)
            const int ngr = (int)min((int64_t)HW, (ngroups - grp0 + gridDim.x - 1) / gridDim.x);
            const int npairs = ngr * nf;
            const int nbw = min(npairs, HW);
            const bool early_means = means && nbw < HW;
            if (warp < nbw) {
                slb_bulk::mbar_wait(bar + 0, 0);
                head_mark(a, HM_TABLES);
                for (int p = warp; p < npairs; p += nbw) {
                    const int i = p / nf, f = p % nf;
                    if (cfg.gp.factors[f].head_rows <= 0) continue;
                    const int64_t k = (grp0 + (int64_t)i * gridDim.x) * HP + min(lane, HP - 1);
                    const bool mine = lane < HP && k < count;
                    double tz[DIN];
#pragma unroll
                    for (int c = 0; c < DIN; ++c) tz[c] = mine ? a.side_a[k].z[c] : 0.0;
                    const double sd =
                        lay.factors_staged == nf
                            ? head_factor_sdev<DIN, true, (CD > 0)>(cfg, a, f, tz, mine, exptab, kw, wbuf, xbuf, bar)
                            : head_factor_sdev<DIN, false, (CD > 0)>(cfg, a, f, tz, mine, exptab, kw, wbuf, xbuf, bar);
                    if (lane < HP) sd_s[(i * HP + lane) * SLB_MAX_OUT + f] = sd;
                    if (f == 0) head_mark(a, HM_BOUND0);
                }
                head_mark(a, HM_BOUND);
            } else if constexpr (CD > 0) {
                if (early_means) {
                    slb_bulk::mbar_wait(bar + 0, 0);
                    slb_bulk::mbar_wait(bar + 2, 0);
                    head_round_means<DIN, CD>(cfg, a, nullptr, ngr * HP, grp0, count, mbuf, tab512, mu_s, merr_s,
                                              nbw * 32, HT - nbw * 32);
                    head_mark(a, HM_MEANS);
                }
            }
            __syncthreads();
            if constexpr (CD > 0) {
                if (means && !early_means) {              // no warp to spare: the means after the bounds
                    slb_bulk::mbar_wait(bar + 0, 0);
                    slb_bulk::mbar_wait(bar + 2, 0);
                    head_round_means<DIN, CD>(cfg, a, nullptr, ngr * HP, grp0, count, mbuf, tab512, mu_s, merr_s, 0,
                                              HT);
                    head_mark(a, HM_MEANS);
                    __syncthreads();
                }
            }
            if (warp < ngr) {
                entry_t t;
                int64_t rel;
                bool mine;
                double shi[ND];
                head_group_entries<DIN>(cfg, a, grp0 + (int64_t)warp * gridDim.x, count, t, rel, mine, shi);
                const int slot = warp * HP + min(lane, HP - 1);
#pragma unroll
                for (int j = 0; j < ND; ++j) {
                    if (j >= cfg.gp.num_outputs) break;
                    const int f = cfg.gp.outputs[j].factor;
                    if (cfg.gp.factors[f].head_rows > 0) shi[j] = sd_s[slot * SLB_MAX_OUT + f];
                }
                double vx = 0.0;
                bool need;
                int outcome = head_entry_decision(cfg, a, t, shi, mine, vx, need);
                if constexpr (CD > 0)
                    if (need) outcome = head_mean_decision(cfg, t, vx, shi, mu_s, merr_s, slot);
                head_mark(a, HM_DECIDED);
                head_group_finish(a, mine, outcome, entry_rel(t, rel),
                                  entry_slot(t, grp0 + (int64_t)warp * gridDim.x), s_stat);
            }
            __syncthreads();                              // sd_s, mu_s are the next round's
        }
    } else {
        // round: warp w takes group grp0 + w gridDim (every warp of the CTA makes the same number of rounds)
        int round = 0;
        for (int64_t grp0 = blockIdx.x; grp0 < ngroups; grp0 += nwarps, ++round) {
            const int64_t grp = grp0 + (int64_t)warp * gridDim.x;
            const bool active = grp < ngroups;
            const int lane = threadIdx.x & 31;
            entry_t t;
            int64_t rel = 0;
            bool mine = false, need = false;
            double shi[ND];
            double vx = 0.0;
            int outcome = 0;
            if (active) {
                head_group_entries<DIN>(cfg, a, grp, count, t, rel, mine, shi);
                if (lay.factors_staged == nf)
                    head_group_bound<DIN, true, CD>(cfg, a, t.z, mine, exptab, kw, wbuf, xbuf, bar, shi);
                else
                    head_group_bound<DIN, false, CD>(cfg, a, t.z, mine, exptab, kw, wbuf, xbuf, bar, shi);
                outcome = head_entry_decision(cfg, a, t, shi, mine, vx, need);
                if (need) need_s[2 + atomicAdd(need_s + (round & 1), 1)] = warp * HP + lane;
            }
            if constexpr (CD > 0) {
                if (threadIdx.x == 0) need_s[(round + 1) & 1] = 0;       // the next round's counter
                __syncthreads();
                const int nneed = need_s[round & 1];
                if (nneed > 0) {
                    // the rest gets its mean in fp64 (all warps), then the same comparison as the fp64 path
                    slb_bulk::mbar_wait(bar + 2, 0);
                    head_round_means<DIN, CD>(cfg, a, need_s + 2, nneed, grp0, count, mbuf, tab512, mu_s, merr_s, 0, HT);
                    head_mark(a, HM_MEANS);
                    __syncthreads();
                    if (need) outcome = head_mean_decision(cfg, t, vx, shi, mu_s, merr_s, warp * HP + lane);
                }
            }
            if (active) {
                head_mark(a, HM_DECIDED);
                head_group_finish(a, mine, outcome, entry_rel(t, rel), entry_slot(t, grp), s_stat);
            }
        }
    }
    // one pair of global atomics per CTA (one per point serialised on the counter's L2 line)
    head_wait_landings(bar);
    __syncthreads();
    if (a.stats != nullptr && threadIdx.x < 2 && s_stat[threadIdx.x] != 0)
        atomicAdd(a.stats + 1 + threadIdx.x, (unsigned long long)s_stat[threadIdx.x]);
    if (threadIdx.x == 0) head_mark(a, HM_EXIT);
}

double* g_probe_mu = nullptr;          // slb_debug_screening_probe
double* g_probe_dm = nullptr;
unsigned long long* g_head_timing = nullptr;   // slb_debug_head_timing
unsigned long long* g_stage1_timing = nullptr; // slb_debug_stage1_timing
int g_filter_stages = 3;               // slb_debug_filter_stages: bit 0 head stage, bit 1 refine pass,
                                       // bit 2 forces the fp64 mean stage (no fp32 screening), bit 3 /
                                       // bit 4 force the head stage's split schedule / round loop,
                                       // bit 5 the fp32 screening kernel where the grid kernel would run

// The fp32 screening kernel needs closed-form bounds of V and L_V over a box of means
// (screening_slack): plain RBF factors, V = QUADRATIC (optional scale) on the GP outputs, L_V constant
// or LINEAR with abs / 1-norm / scale only.  Everything else keeps the fp64 mean stage.
bool screening_applicable(const slb_sweep& cfg) {
    if (g_filter_stages & 4) return false;
    const int D = cfg.gp.num_outputs;
    for (int f = 0; f < cfg.gp.num_factors; ++f)
        if (cfg.gp.factors[f].kernel.num_prims > 0) return false;
    const slb_function& V = cfg.lyapunov;
    if (D > 4) return false;                   // screening_slack is written out for up to 4 outputs
    if (V.kind != SLB_FN_QUADRATIC || V.in_dim != D || (V.flags & ~(uint32_t)SLB_FLAG_SCALE)) return false;
    const slb_function& L = cfg.lipschitz_v;
    if (L.kind == SLB_FN_NONE) return true;
    if (L.kind != SLB_FN_LINEAR || L.in_dim != D) return false;
    if (L.flags & ~(uint32_t)(SLB_FLAG_ABS | SLB_FLAG_NORM1 | SLB_FLAG_SCALE)) return false;
    if (L.out_dim > 4) return false;
    return (L.flags & SLB_FLAG_NORM1) || L.out_dim == 1 || L.out_dim == D;
}

// The factored grid kernel replaces the fp32 screening kernel (same list A layout) where kernel values
// factor over the grid axes: a 2-D grid (so two outputs), z = [x0, x1, u] with plain RBF factors
// (screening_applicable) and u = a x0 + b x1, optionally saturated and scaled.  Its per-point terms are
// the closed form of the register-only evaluators (common.cuh), so L_f is a constant, a table or a LINEAR
// map as well.
bool grid_mean_applicable(const slb_sweep& cfg) {
    if (g_filter_stages & 32) return false;
    const slb_function& P = cfg.policy;
    const slb_function& Lf = cfg.lipschitz_f;
    const bool lf_closed = Lf.kind == SLB_FN_NONE || cfg.lf_values != nullptr ||
                           (Lf.kind == SLB_FN_LINEAR && Lf.in_dim == 2 && Lf.out_dim <= SLB_MAX_LIN_OUT &&
                            Lf.matrix != nullptr &&
                            !(Lf.flags & ~(uint32_t)(SLB_FLAG_SATURATE | SLB_FLAG_ABS | SLB_FLAG_NORM1 |
                                                     SLB_FLAG_SCALE)));
    return screening_applicable(cfg) && cfg.grid.ndim == 2 && cfg.gp.input_dim == 3 &&
           P.kind == SLB_FN_LINEAR && P.in_dim == 2 && P.out_dim == 1 && P.matrix != nullptr &&
           !(P.flags & ~(uint32_t)(SLB_FLAG_SATURATE | SLB_FLAG_SCALE)) && lf_closed;
}

// Which stage 1 runs and the shared-memory layout of the head stage (one CTA per SM): which factors' head
// tables are staged, and -- for a screened stage 1 -- every factor's [Xf | gamma_f] next to them.  Screening
// is only used when all of it fits (otherwise the fp64 mean stage runs, whose list entries are complete).
filter_plan stage1_plan(const slb_sweep& cfg) {
    const int din = cfg.gp.input_dim, nf = cfg.gp.num_factors;
    const int budget = 226 * 1024 / (int)sizeof(double);
    const int slots = HW * HP * SLB_MAX_OUT;
    filter_plan p = {};
    p.mean_scheme = SLB_MEAN_FP64;
    p.factors_staged = nf;
    while (p.factors_staged > 0 && 4 + 576 + HW * HR * HP + slots + p.factors_staged * (HR * HR + HR * din) > budget)
        --p.factors_staged;
    int off = 4;
    p.tabs = off;   off += 576;
    p.kbuf = off;   off += HW * HR * HP;
    p.sd = off;     off += slots;
    p.wbuf = off;   off += p.factors_staged * HR * HR;
    p.xbuf = off;   off += p.factors_staged * HR * din;
    p.doubles = off;
    if (!screening_applicable(cfg) || p.factors_staged != nf) return p;
    int tables = 0;
    for (int f = 0; f < nf; ++f) {
        int no = 0;
        for (int o = 0; o < cfg.gp.num_outputs; ++o) no += cfg.gp.outputs[o].factor == f;
        p.mean_off[f] = tables;
        tables += ((cfg.gp.factors[f].M + 7) & ~7) * (din + 1 + no);
    }
    const int need = (HW * HP + 4) * (int)sizeof(int) / (int)sizeof(double);
    if (off + tables + 2 * slots + need > budget) return p;
    p.mean_scheme = grid_mean_applicable(cfg) ? SLB_MEAN_GRID_FACTORED : SLB_MEAN_FP32_SCREENED;
    p.mean_doubles = tables;
    p.mbuf = off;   off += tables;
    p.mu = off;     off += slots;
    p.merr = off;   off += slots;
    p.need = off;   off += need;
    p.doubles = off;
    return p;
}

// D = 0: the fp64 mean stage.  D > 0: a screened plan's D outputs (the closed-form kernels)
template <int DIN, int D>
int launch_filter(cudaStream_t st, const slb_sweep& cfg, const filter_args& a) {
    static std::atomic<bool> configured[64];
    int device = 0;
    SLB_CUDA(cudaGetDevice(&device));
    if (device < 0 || device >= 64 || !configured[device].load(std::memory_order_acquire)) {
        if constexpr (D == 0)
            SLB_CUDA(cudaFuncSetAttribute(filter_mean_kernel<DIN>,
                                          cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        else
            SLB_CUDA(cudaFuncSetAttribute(filter_mean32_kernel<DIN, D>,
                                          cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        SLB_CUDA(cudaFuncSetAttribute(filter_head_kernel<DIN, D>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        if constexpr (DIN == 3 && D == GRID_OUTPUTS) {
            SLB_CUDA(cudaFuncSetAttribute(filter_grid_mean_kernel<GRID_OUTPUTS>,
                                          cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)grid_mean_smem_bytes()));
            // all of the unified L1 / shared memory as shared: two 111 KB CTAs per SM
            SLB_CUDA(cudaFuncSetAttribute(filter_grid_mean_kernel<GRID_OUTPUTS>,
                                          cudaFuncAttributePreferredSharedMemoryCarveout,
                                          (int)cudaSharedmemCarveoutMaxShared));
        }
        if (device >= 0 && device < 64) configured[device].store(true, std::memory_order_release);
    }
    const int64_t blocks = (a.n + FT - 1) / FT;
    switch (a.plan.mean_scheme) {
    case SLB_MEAN_GRID_FACTORED:
        // grid_mean_applicable: d_in = 3 and two outputs
        SLB_CHECK(DIN == 3 && D == GRID_OUTPUTS, "filtered sweep: the factored grid mean needs d_in = 3 and %d outputs",
                  GRID_OUTPUTS);
        if constexpr (DIN == 3 && D == GRID_OUTPUTS) {
            // tiles of GR rows x GC columns over the rows the range touches (it may start and end mid-row)
            const int64_t n1 = cfg.grid.num_points[1];
            const int64_t r0 = a.idx_begin / n1, r1 = (a.idx_begin + a.n - 1) / n1;
            const int64_t tiles = ((r1 - r0) / GR + 1) * ((n1 + GC - 1) / GC);
            filter_grid_mean_kernel<GRID_OUTPUTS><<<(unsigned)tiles, GT, grid_mean_smem_bytes(), st>>>(cfg, a);
        }
        break;
    case SLB_MEAN_FP32_SCREENED:
        if constexpr (D > 0)
            filter_mean32_kernel<DIN, D><<<(unsigned)blocks, FT,
                                           mean32_smem_bytes(DIN, a.max_outputs_per_factor, a.chunk_rows, FT / 32),
                                           st>>>(cfg, a);
        break;
    default:
        if constexpr (D == 0)
            filter_mean_kernel<DIN><<<(unsigned)blocks, FT,
                                      mean_smem_bytes(DIN, a.max_outputs_per_factor, a.chunk_rows), st>>>(cfg, a);
    }
    SLB_LAUNCH_CHECK();
    if (!(g_filter_stages & 1)) return 0;
    filter_head_kernel<DIN, D><<<HEAD_CTAS, HT, (size_t)a.plan.doubles * sizeof(double), st>>>(cfg, a);
    SLB_LAUNCH_CHECK();
    return 0;
}

// The instantiation of a plan: d_in = d + m (slb_validate_sweep: m >= 1, so d_in >= 2) and, for a screened
// plan, its D = d outputs (screening_applicable: D <= 4), D = d_in - m with m <= SLB_MAX_ACT = 2
static_assert(SLB_MAX_ACT == 2, "the screened instantiations cover m = 1, 2");
int dispatch_filter(cudaStream_t st, const slb_sweep& cfg, const filter_args& a) {
    return slb_dispatch_dim<2, 6>(cfg.gp.input_dim, "GP input_dim", [&](auto din) {
        constexpr int DIN = decltype(din)::value;
        if (a.plan.mean_scheme == SLB_MEAN_FP64) return launch_filter<DIN, 0>(st, cfg, a);
        constexpr int DLO = DIN - 2 > 1 ? DIN - 2 : 1, DHI = DIN - 1 < 4 ? DIN - 1 : 4;
        return slb_dispatch_dim<DLO, DHI>(cfg.gp.num_outputs, "screened filter: outputs", [&](auto d) {
            return launch_filter<DIN, decltype(d)::value>(st, cfg, a);
        });
    });
}

}  // namespace

// light.cu: the prefix rule on the key a step folded into `rec` (slb_safe_set_step)
int slb_launch_apply_prefix_folded(cudaStream_t st, const double* values, const uint8_t* initial, int64_t n,
                                   int64_t idx_begin, slb_fold* rec, slb_fail_key* key, uint8_t* safe,
                                   slb_prefix_stats* stats);

// gp_sweep.cu: the full posterior on the compacted list (count read on the device)
int slb_launch_refine(cudaStream_t st, const slb_sweep& cfg, int64_t n_max, int64_t idx_begin,
                      const int64_t* list, const unsigned long long* count, uint8_t* negative,
                      double* values, double* mean, double* err, double* split_partial, int* split_ticket,
                      const slb_fold_target& fold, const filter_side* side, const int64_t* side_slot,
                      bool closed);

extern "C" {

int slb_debug_filter_stages(int32_t mask) {
    g_filter_stages = mask;
    return 0;
}

int slb_filter_stage1(const slb_sweep* cfg) {
    const int scheme = slb_filter_mean_scheme(cfg);
    return scheme == SLB_MEAN_NONE ? 0 : scheme == SLB_MEAN_FP64 ? 64 : 32;
}

int slb_filter_mean_scheme(const slb_sweep* cfg) {
    if (cfg == nullptr || cfg->gp.num_outputs <= 0) return SLB_MEAN_NONE;
    return stage1_plan(*cfg).mean_scheme;
}

int slb_debug_screening_probe(double* mu_dev, double* dm_dev) {
    g_probe_mu = (mu_dev != nullptr && dm_dev != nullptr) ? mu_dev : nullptr;
    g_probe_dm = g_probe_mu != nullptr ? dm_dev : nullptr;
    return 0;
}

int slb_debug_head_timing(void* buffer_dev) {
    g_head_timing = static_cast<unsigned long long*>(buffer_dev);
    return 0;
}

int slb_debug_stage1_timing(void* buffer_dev) {
    g_stage1_timing = static_cast<unsigned long long*>(buffer_dev);
    return 0;
}

int64_t slb_filter_workspace(int64_t n) {
    if (n < 0) n = 0;
    if (n > CHUNK) n = CHUNK;     // longer ranges are swept in passes of CHUNK points
    // [0] |list A|, [1] |list B| (uint64, 64 bytes reserved), tile tickets and partial sums of the
    // row-split refine pass, list A, list B, the list A slots of list B, terms of list A
    return WS_HEAD + n * (int64_t)(3 * sizeof(int64_t) + sizeof(filter_side));
}

int slb_debug_filter_lists(int64_t n, int64_t* offsets) {
    SLB_CHECK(offsets != nullptr, "slb_debug_filter_lists: null offsets");
    SLB_CHECK(n >= 0 && n <= CHUNK, "slb_debug_filter_lists: n %lld outside [0, %lld] (one pass)", (long long)n,
              (long long)CHUNK);
    // the layout slb_lyapunov_sweep_filtered carves out of its workspace (cap = n for one pass)
    offsets[0] = 0;
    offsets[1] = WS_HEAD;
    offsets[2] = WS_HEAD + n * (int64_t)sizeof(int64_t);
    return 0;
}

}  // extern "C"

// slb_lyapunov_sweep_filtered, and the sweep of slb_safe_set_step with fold.rec != nullptr: the record at
// WS_FOLD is zeroed with the first pass's counts and accumulates over all passes
static int filtered_sweep(cudaStream_t st, const slb_sweep* cfg, int64_t idx_begin, int64_t idx_end,
                          uint8_t* negative_dev, double* values_dev, void* workspace_dev, int64_t* stats_dev,
                          slb_fold_target fold) {
    int m;
    if (slb_validate_sweep(cfg, false, &m)) return 1;
    if (slb_validate_range("slb_lyapunov_sweep_filtered", idx_begin, idx_end, cfg->grid.nindex)) return 1;
    SLB_CHECK(cfg->gp.num_outputs > 0, "slb_lyapunov_sweep_filtered needs GP dynamics "
              "(deterministic dynamics have nothing to filter: use slb_lyapunov_sweep)");
    if (slb_validate_staged_tables(&cfg->gp, "filtered sweep")) return 1;
    int nomax = 1;
    for (int f = 0; f < cfg->gp.num_factors; ++f) {
        // (Whead has no device reader since the head stage multiplies the packed Wheadp only; the field stays
        // part of the descriptor: the parity tests take their reference from it)
        const slb_gp_factor& F = cfg->gp.factors[f];
        SLB_CHECK(F.M == 0 || (F.Whead != nullptr && F.Wheadp != nullptr && F.Xhead != nullptr),
                  "filtered sweep: GP factor %d lacks the filter tables (Whead / Wheadp / Xhead)", f);
        SLB_CHECK(F.M == 0 || ((reinterpret_cast<uintptr_t>(F.Wheadp) & 15) == 0 &&
                               (reinterpret_cast<uintptr_t>(F.Xhead) & 15) == 0),
                  "filtered sweep: GP factor %d: Wheadp / Xhead must be 16-byte aligned", f);
        SLB_CHECK(F.head_rows >= 0 && F.head_rows <= SLB_HEAD_RANK && F.head_rows <= F.M,
                  "filtered sweep: GP factor %d has %d head rows (0..min(M, %d))", f, F.head_rows,
                  SLB_HEAD_RANK);
        int no = 0;
        for (int o = 0; o < cfg->gp.num_outputs; ++o) no += cfg->gp.outputs[o].factor == f;
        if (no > nomax) nomax = no;
    }
    for (int o = 0; o < cfg->gp.num_outputs; ++o)
        SLB_CHECK(cfg->gp.outputs[o].gamma_l1 >= 0.0, "filtered sweep: GP output %d has no gamma_l1", o);
    const int64_t n_all = idx_end - idx_begin;
    if (n_all == 0) return 0;
    SLB_CHECK(negative_dev != nullptr && workspace_dev != nullptr,
              "slb_lyapunov_sweep_filtered: negative_dev and workspace_dev are required");
    char* ws = static_cast<char*>(workspace_dev);
    const int64_t cap = n_all < CHUNK ? n_all : CHUNK;
    filter_args a;
    memset(&a, 0, sizeof(a));
    a.counts = reinterpret_cast<unsigned long long*>(ws);
    int* tickets = reinterpret_cast<int*>(ws + 64);
    double* partial = reinterpret_cast<double*>(ws + WS_PARTIAL);
    a.list_a = reinterpret_cast<int64_t*>(ws + WS_HEAD);
    a.list_b = a.list_a + cap;
    a.slot_b = a.list_b + cap;
    a.side_a = reinterpret_cast<filter_side*>(a.slot_b + cap);
    a.stats = reinterpret_cast<unsigned long long*>(stats_dev);
    // rows per staged slice: two buffers of (d_in + 1 + outputs per factor) doubles per row within
    // ~24 KB, so that 7 CTAs stay resident per SM
    const int din = cfg->gp.input_dim;
    a.chunk_rows = mean_chunk_rows(din, nomax, 24);
    a.max_outputs_per_factor = nomax;
    a.plan = stage1_plan(*cfg);
    a.prefetch_factors = (g_filter_stages & 2) ? 1 : 0;
    a.head_schedule = (g_filter_stages >> 3) & 3;
    a.probe_mu = g_probe_mu;
    a.probe_dm = g_probe_dm;
    a.timing = g_head_timing;
    a.timing1 = g_stage1_timing;
    for (int64_t off = 0; off < n_all; off += CHUNK) {
        const int64_t n = n_all - off < CHUNK ? n_all - off : CHUNK;
        const bool first_fold = fold.rec != nullptr && off == 0;
        SLB_CUDA(cudaMemsetAsync(a.counts, 0, first_fold ? WS_PARTIAL : WS_FOLD, st));
        a.n = n; a.idx_begin = idx_begin + off;
        a.negative = negative_dev + off;
        a.values = values_dev ? values_dev + off : nullptr;
        a.fold = fold;
        if (fold.rec != nullptr) {
            a.fold.values = fold.values + off;
            a.fold.initial = fold.initial ? fold.initial + off : nullptr;
        }
        int rc = dispatch_filter(st, *cfg, a);
        if (rc) return rc;
        if (!(g_filter_stages & 2)) continue;
        rc = slb_launch_refine(st, *cfg, n, idx_begin + off, a.list_b, a.counts + 1,
                               negative_dev + off, values_dev ? values_dev + off : nullptr,
                               nullptr, nullptr, partial, tickets, a.fold, a.side_a, a.slot_b,
                               a.plan.mean_scheme == SLB_MEAN_GRID_FACTORED);
        if (rc) return rc;
    }
    return 0;
}

extern "C" {

int slb_lyapunov_sweep_filtered(void* stream, const slb_sweep* cfg, int64_t idx_begin,
                                int64_t idx_end, uint8_t* negative_dev, double* values_dev,
                                void* workspace_dev, int64_t* stats_dev) {
    return filtered_sweep((cudaStream_t)stream, cfg, idx_begin, idx_end, negative_dev, values_dev, workspace_dev,
                          stats_dev, slb_fold_target{});
}

int slb_safe_set_step(void* stream, const slb_sweep* cfg, int64_t idx_begin, int64_t idx_end,
                      uint8_t* negative_dev, const double* values_dev, const uint8_t* initial_dev,
                      void* workspace_dev, int64_t* stats_dev, slb_fail_key* key_dev, uint8_t* safe_dev,
                      slb_prefix_stats* prefix_stats_dev) {
    SLB_CHECK(cfg != nullptr, "slb_safe_set_step: null config");
    SLB_CHECK(idx_end > idx_begin, "slb_safe_set_step: empty range [%lld, %lld)", (long long)idx_begin,
              (long long)idx_end);
    SLB_CHECK(values_dev != nullptr && workspace_dev != nullptr && key_dev != nullptr && safe_dev != nullptr &&
                  prefix_stats_dev != nullptr,
              "slb_safe_set_step: null values, workspace, key, safe set or statistics");
    cudaStream_t st = (cudaStream_t)stream;
    slb_fold* rec = reinterpret_cast<slb_fold*>(static_cast<char*>(workspace_dev) + WS_FOLD);
    const int rc = filtered_sweep(st, cfg, idx_begin, idx_end, negative_dev, nullptr, workspace_dev, stats_dev,
                                  slb_fold_target{values_dev, initial_dev, rec});
    if (rc) return rc;
    return slb_launch_apply_prefix_folded(st, values_dev, initial_dev, idx_end - idx_begin, idx_begin, rec,
                                          key_dev, safe_dev, prefix_stats_dev);
}

int slb_debug_refine(void* stream, const slb_sweep* cfg, int64_t idx_begin, int64_t n_max,
                     const int64_t* list_dev, const unsigned long long* count_dev,
                     uint8_t* negative_dev, double* values_dev, double* mean_dev, double* err_dev,
                     void* workspace_dev) {
    SLB_CHECK(cfg != nullptr, "slb_debug_refine: null config");
    SLB_CHECK(cfg->gp.num_outputs > 0, "slb_debug_refine needs GP dynamics (the refine pass is the GP posterior)");
    SLB_CHECK(n_max >= 0 && n_max <= CHUNK, "slb_debug_refine: n_max %lld outside [0, %lld]", (long long)n_max,
              (long long)CHUNK);
    SLB_CHECK(list_dev != nullptr && count_dev != nullptr && negative_dev != nullptr && workspace_dev != nullptr,
              "slb_debug_refine: null list, count, negative or workspace");
    int m;
    if (slb_validate_sweep(cfg, false, &m)) return 1;
    if (slb_validate_range("slb_debug_refine", idx_begin, idx_begin + n_max, cfg->grid.nindex)) return 1;
    // the same workspace layout, and the same zeroed tickets, as one pass of the filtered sweep
    cudaStream_t st = (cudaStream_t)stream;
    char* ws = static_cast<char*>(workspace_dev);
    SLB_CUDA(cudaMemsetAsync(ws + 64, 0, SLB_SPLIT_TICKET_BYTES, st));
    return slb_launch_refine(st, *cfg, n_max, idx_begin, list_dev, count_dev, negative_dev, values_dev, mean_dev,
                             err_dev, reinterpret_cast<double*>(ws + WS_PARTIAL), reinterpret_cast<int*>(ws + 64),
                             slb_fold_target{}, nullptr, nullptr, false);
}

}  // extern "C"
