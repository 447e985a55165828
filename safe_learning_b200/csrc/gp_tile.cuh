// gp_tile.cuh -- the dominant kernel: GP posterior (mean + variance) of a 64-point tile and,
// in sweep mode, the fused Lyapunov decision.
//
// Replaces, per 10 000-point Session.run of the reference (paths relative to upstream safe_learning):
//   gpflow kern.K(X, Xnew)                       functions.py:438   -> k-row generation phase
//   tf.matrix_triangular_solve(L, Kx)            functions.py:441   -> a = L^-1 k as DMMA GEMM
//   a^T alpha (+ prior mean), Kdiag - sum a^2    functions.py:442,450-451 -> panel epilogue
//   beta * sqrt(var)                             functions.py:514
//   FunctionStack concat                         functions.py:278-291
//   v_decrease_bound < threshold                 lyapunov.py:436-441 -> tile epilogue
//
// Design (H100, fp64 pipe bound -- see DESIGN.md section 3.1):
//   * one CTA = 64 grid points x all M training points, 8 warps, 1 CTA/SM (~178 KB shared
//     memory).
//   * W = L^-1 (lower triangular) is pre-packed in DMMA.8x8x4 A-fragment order, two k-steps
//     per 128-bit element (slb_pack_factor); each warp streams ITS rows of W straight from L2
//     into registers with coalesced 512 B loads through a static three-deep register ring --
//     W is used by exactly one warp per CTA, so it never needs shared memory.
//   * the k-row tile K[j, p] = s^2 v exp(-|z_p - X_j|^2 / 2) is generated once per 256-row
//     j-panel into shared memory in a pair-interleaved layout (conflict-free 128-bit
//     B-fragment reads), with a branch-free table-driven exp, four evaluations in flight.
//   * a 256-row i-panel of a = W k lives in registers (32 rows x 64 points per warp = 64 fp64
//     accumulators per thread); row blocks are dealt to warps round-robin from the bottom of the
//     panel so the triangular work is balanced across warps and across SMSPs.  sum a^2 and
//     a.alpha are reduced by a butterfly reduce-scatter in the panel epilogue into per-warp
//     running sums (no block barrier per panel); `a` is never stored.
//   * first-wave CTAs prefetch the packed factor into L2 (cold-L2 launches otherwise stream it
//     from HBM in lockstep); eval_fn is not inlined here to keep the cold code small.
#pragma once
#define SLB_EVAL_NOINLINE 1
#include "common.cuh"

#include <string.h>

#include <atomic>


#include "gp_args.h"

namespace {

#ifndef SLB_TP
#define SLB_TP SLB_TILE_POINTS
#endif
constexpr int TP = SLB_TP;            // points per CTA: 64 for sweeps; 32 for the refine pass of the
                                      // filtered sweep, whose short point list would otherwise fill
                                      // only a fraction of the SMs (one translation unit each)
static_assert(TP == 32 || TP == 64, "TP must be 32 or 64");
constexpr int PANEL = 256;            // rows per i-panel, columns per j-panel
// K-row tile layout in shared memory: k-steps are handled in PAIRS (8 rows of K).  Row j of a
// panel lives at pair m = j / 8, half h = (j / 4) % 2, fragment row r = j % 4; element (j, p) is
// Ks[((m * 4 + r) * KSTR + p) * 2 + h], so one 128-bit load gives a lane its B fragments of both
// k-steps of a pair.  KSTR = 66: (r * 66 + c) mod 8 is distinct for r in 0..3, c in 0..1, i.e. the
// eight lanes of a quarter-warp hit eight different 16-byte bank groups (conflict-free LDS.128).
constexpr int KSTR = TP + 2;
constexpr int NW = 8;                 // warps per CTA
constexpr int NT = NW * 32;
constexpr int RQ = 32 / NW;           // 8-row blocks per warp per 256-row panel (RQ * NW = 32)
constexpr int NB = TP / 8;            // 8-point column blocks per warp tile
constexpr int CTAS_PER_SM = 1;
constexpr int NRED = 1 + SLB_MAX_OUT;
constexpr int PREFETCH_CTAS = SLB_NUM_SMS * CTAS_PER_SM;    // one wave

constexpr size_t SMEM_KS = (size_t)(PANEL / 8) * 4 * KSTR * 2 * sizeof(double);
constexpr size_t SMEM_Z = (size_t)SLB_MAX_IN * TP * sizeof(double);
constexpr size_t SMEM_RED = (size_t)NW * TP * NRED * sizeof(double);
constexpr size_t SMEM_TOT = (size_t)NRED * TP * sizeof(double);
constexpr size_t SMEM_POST = (size_t)2 * SLB_MAX_OUT * TP * sizeof(double);
constexpr size_t SMEM_EXPTAB = 64 * sizeof(double);
constexpr size_t SMEM_XP = (size_t)PANEL * SLB_MAX_IN * sizeof(double);
constexpr size_t SMEM_KEXPR = (sizeof(slb_kernel) + 15) / 16 * 16;
constexpr size_t SMEM_PRE = (size_t)4 * TP * sizeof(double);
constexpr size_t SMEM_TOTAL = SMEM_KS + SMEM_Z + SMEM_RED + SMEM_TOT + SMEM_POST + SMEM_EXPTAB +
                              SMEM_XP + SMEM_KEXPR + SMEM_PRE;

SLB_DEV double2 ldg_stream2(const double2* p) {
    double2 v;
    asm volatile("ld.global.nc.L1::no_allocate.v2.f64 {%0, %1}, [%2];"
                 : "=d"(v.x), "=d"(v.y) : "l"(p));
    return v;
}

SLB_DEV void dmma884(double& c0, double& c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

// depth of the register ring that streams L^-1 ahead of the DMMAs: the 32-point tiles of the refine
// pass do half the math per streamed byte, so they need more bytes in flight to cover the L2 latency
constexpr int RING = TP == 64 ? 3 : 5;
constexpr int BG = 4;                 // column blocks whose B fragments are loaded together

// Pairs [m0, m1) of k-steps of the current j-panel for row blocks q >= Q0 of this warp.
// Per pair and row block ONE 128-bit global load brings the A fragments of both k-steps
// (the packed factor stores them adjacent), per column block ONE 128-bit shared load brings both
// B fragments.  The A prefetch ring (RING pairs ahead) is unrolled with static registers: no
// rotation moves (tools/dmma_mix.cu, "wide", measures this load pattern in isolation).
template <int Q0>
SLB_DEV void mma_run(double (&acc)[RQ][NB][2], const double2* const (&ap)[RQ], int m0, int m1,
                     const double2* ks_lane) {
    double2 ar[RING][RQ];
    const int m1m = m1 - 1;
#pragma unroll
    for (int d = 0; d < RING; ++d) {
        const int md = min(m0 + d, m1m);
#pragma unroll
        for (int q = Q0; q < RQ; ++q) ar[d][q] = ldg_stream2(ap[q] + md * 32);
    }
    int m = m0;
#pragma unroll 1
    while (true) {
#pragma unroll
        for (int d = 0; d < RING; ++d) {
            if (m >= m1) return;
            const double2* kb = ks_lane + m * (4 * KSTR);
#pragma unroll
            for (int half = 0; half < NB; half += BG) {
                double2 b[BG];
#pragma unroll
                for (int nb = 0; nb < BG; ++nb) b[nb] = kb[(half + nb) * 8];
#pragma unroll
                for (int q = Q0; q < RQ; ++q)
#pragma unroll
                    for (int nb = 0; nb < BG; ++nb)
                        dmma884(acc[q][half + nb][0], acc[q][half + nb][1], ar[d][q].x, b[nb].x);
#pragma unroll
                for (int q = Q0; q < RQ; ++q)
#pragma unroll
                    for (int nb = 0; nb < BG; ++nb)
                        dmma884(acc[q][half + nb][0], acc[q][half + nb][1], ar[d][q].y, b[nb].y);
            }
            const int mp = min(m + RING, m1m);
#pragma unroll
            for (int q = Q0; q < RQ; ++q) ar[d][q] = ldg_stream2(ap[q] + mp * 32);
            ++m;
        }
    }
}

// Sum the 2 NBT per-thread values v[2 nb + e] (column 8 nb + 2 (T%4) + e of the warp tile) over the 8
// lanes that share T%4 (lane bits 4, 3, 2) and add them to red_q[column * NRED].  Reduce-scatter:
// every step halves the values a lane still carries (send one half, keep and add the other) --
// NBT = 8: 8+4+2 shuffles instead of 3 per value, every lane ends with two finished columns;
// NBT = 4: one column per lane.
template <int NBT>
SLB_DEV void row_lane_reduce(const double (&v)[2 * NBT], int lane, double* red_q) {
    constexpr int NV = 2 * NBT;
    const bool g2 = (lane & 16) != 0, g1 = (lane & 8) != 0, g0 = (lane & 4) != 0;
    double w8[NV / 2], w4[NV / 4];
#pragma unroll
    for (int i = 0; i < NV / 2; ++i) {
        const double send = g2 ? v[i] : v[i + NV / 2];
        const double keep = g2 ? v[i + NV / 2] : v[i];
        w8[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
    }
#pragma unroll
    for (int i = 0; i < NV / 4; ++i) {
        const double send = g1 ? w8[i] : w8[i + NV / 4];
        const double keep = g1 ? w8[i + NV / 4] : w8[i];
        w4[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
    }
    if constexpr (NBT == 8) {
        double w2[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const double send = g0 ? w4[i] : w4[i + 2];
            const double keep = g0 ? w4[i + 2] : w4[i];
            w2[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
        }
        // value index 2g + e  <->  nb = g = lane / 4, column 8g + 2(T%4) + e
        double* slot = red_q + (8 * (lane >> 2) + 2 * (lane & 3)) * NRED;
        slot[0] += w2[0];
        slot[NRED] += w2[1];
    } else {
        static_assert(NBT == 4, "written for 8 or 4 column blocks");
        const double send = g0 ? w4[0] : w4[1];
        const double keep = g0 ? w4[1] : w4[0];
        const double w1 = keep + __shfl_xor_sync(0xffffffffu, send, 4);
        // value index g = lane / 4  <->  nb = g / 2, e = g % 2
        const int g = lane >> 2;
        red_q[(8 * (g >> 1) + 2 * (lane & 3) + (g & 1)) * NRED] += w1;
    }
}

// slb_debug_refine_timing: marks[CTA][slot] = the latest %globaltimer (ns) at which a warp of the CTA passed
// the mark; the 32-point refine tiles only.  RM_GEN / RM_MMA + k: j-panel k (k = 3: the last ones) generated /
// contracted; RM_FINISHER: 1 in the CTA that finished its tile
enum { RM_ENTRY, RM_PROLOGUE, RM_GEN, RM_MMA = RM_GEN + 4, RM_PARTIAL = RM_MMA + 4, RM_TICKET, RM_FACTORS, RM_DECIDED,
       RM_EXIT, RM_FINISHER };
static_assert(RM_FINISHER < SLB_REFINE_MARKS, "refine marks");
SLB_DEV void refine_mark(const slb_gp_args& a, int slot) {
    if (TP != 32 || a.marks == nullptr || (threadIdx.x & 31) != 0) return;
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    atomicMax(a.marks + blockIdx.x * SLB_REFINE_MARKS + slot, t);
}

// One tile (or one row / factor share of it) on the calling CTA: the body of gp_tile_kernel.  CD > 0: the
// refine pass of the filter's closed form (CD outputs), which reads its terms from stage 1's list A entries and
// finishes the tile with the register-only evaluators.
template <int DIN, bool TIMING, bool KEXPR, int CD>
SLB_DEV void gp_tile_body(const slb_sweep& cfg, const slb_gp_args& a, unsigned char* smem_raw,
                          const int64_t tile_index, const int64_t npts, const int grp, const int G,
                          const int fsel, const int FS, const bool first_tile) {
    double* Ks = reinterpret_cast<double*>(smem_raw);
    double* zraw = Ks + (PANEL / 8) * 4 * KSTR * 2;   // [SLB_MAX_IN][TP]
    double* red = zraw + SLB_MAX_IN * TP;             // [NW][TP][NRED]
    double* tot = red + NW * TP * NRED;               // [NRED][TP]
    double* post = tot + NRED * TP;                   // mean [MAX_OUT][TP], err [MAX_OUT][TP]
    double* exptab = post + 2 * SLB_MAX_OUT * TP;     // 2^(j/64), j = 0..63
    double* Xp = exptab + 64;                         // scaled training inputs of the j-panel
    // covariance expression of the current factor (KEXPR): shared memory serves the primitive
    // loop's dynamically indexed reads as broadcasts, the kernel-parameter bank does not
    slb_kernel* kexpr = reinterpret_cast<slb_kernel*>(Xp + PANEL * SLB_MAX_IN);
    // decision terms per point: V(x), threshold(x) (stage 1), V(mu), error bound (tile epilogue)
    double* pre = reinterpret_cast<double*>(reinterpret_cast<unsigned char*>(kexpr) + SMEM_KEXPR);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // small operands behind pointers / in the constant bank: start their (cold) loads now, they are
    // consumed by stage 1 and by the first generation phase
    prefetch_descriptor_operands(cfg);
    const double exp_entry = c_exp2_tab[tid & 63];
    const int64_t tile0 = tile_index * TP;
    const int D = cfg.gp.num_outputs;
    long long t_gen = 0, t_mma = 0, t_epi = 0, t_mark = 0, t_sync = 0, t_s0 = 0;
    const long long t_start = TIMING ? clock64() : 0;
    long long g_start = 0;
    if (TIMING) asm volatile("mov.u64 %0, %globaltimer;" : "=l"(g_start));

    // ---- stage 0: warm L2.  Every CTA streams the whole packed L^-1 (1 MB per factor at
    // M=500); if it is not L2-resident when the launch starts (first sweep after add_data_point,
    // or after anything else evicted it) the first wave of CTAs would pull it from HBM at
    // streaming latency, in lockstep.
    // The first-wave CTAs therefore prefetch disjoint 128-byte lines of it into L2 while the
    // k-row generation phase runs; the demand loads then hit.
    if (first_tile && blockIdx.x < PREFETCH_CTAS) {
        for (int f = 0; f < cfg.gp.num_factors; ++f) {
            const slb_gp_factor& F = cfg.gp.factors[f];
            const char* base = reinterpret_cast<const char*>(F.Wpack);
            const size_t nbytes = (size_t)F.nrb * (F.nrb + 1) * 32 * sizeof(double);
            for (size_t off = ((size_t)blockIdx.x * NT + tid) * 128; off < nbytes;
                 off += (size_t)PREFETCH_CTAS * NT * 128)
                asm volatile("prefetch.global.L2 [%0];" ::"l"(base + off));
        }
    }

    if (tid < 64) exptab[tid] = exp_entry;

    // ---- stage 1: query points z = [x, policy(x)]  (lyapunov.py:436-437, utilities.py:143)
    if (tid < 2 * TP && (CD > 0 || a.side != nullptr)) {
        // refine pass of the filtered sweep: stage 1 computed the point's z, V(x) and threshold with the
        // arithmetic below and left them in its list A entry
        const int p = tid & (TP - 1);
        int64_t i = tile0 + p;
        if (i > npts - 1) i = npts - 1;
        const filter_side* e = a.side + a.side_slot[i];
        if (tid < TP) {
#pragma unroll
            for (int c = 0; c < DIN; ++c) zraw[c * TP + p] = e->z[c];
        } else {
            pre[p] = e->vx;
            pre[TP + p] = e->thr;
        }
    } else if constexpr (CD == 0) {
        if (tid < TP) {
            int64_t rel = tile0 + tid;
            if (rel > npts - 1) rel = npts - 1;
            if (a.index_list != nullptr) rel = a.index_list[rel];
            double z[SLB_MAX_IN];
            if (a.mode == MODE_PREDICT) {
#pragma unroll
                for (int c = 0; c < DIN; ++c) z[c] = a.points[rel * DIN + c];
            } else {
                const int d = cfg.grid.ndim;
                double x[SLB_MAX_DIM];
                if (a.mode == MODE_SWEEP_GRID) {
                    grid_index_to_state(cfg.grid, a.idx_begin + rel, x);
                } else {
                    for (int c = 0; c < d; ++c) x[c] = a.points[rel * d + c];
                }
                double u[SLB_MAX_OUT];
                const int m = eval_fn_small(cfg.policy, x, u);
                for (int c = 0; c < d; ++c) z[c] = x[c];
                for (int c = 0; c < m; ++c) z[d + c] = u[c];
            }
#pragma unroll
            for (int c = 0; c < DIN; ++c) zraw[c * TP + tid] = z[c];
        } else if (tid < 2 * TP && a.mode != MODE_PREDICT) {
            // warps 2-3, concurrently: the terms of the decision that need only x
            const int p = tid - TP;
            int64_t rel = tile0 + p;
            if (rel > npts - 1) rel = npts - 1;
            if (a.index_list != nullptr) rel = a.index_list[rel];
            const int d = cfg.grid.ndim;
            double x[SLB_MAX_DIM];
            if (a.mode == MODE_SWEEP_GRID) {
                grid_index_to_state(cfg.grid, a.idx_begin + rel, x);
            } else {
                for (int c = 0; c < d; ++c) x[c] = a.points[rel * d + c];
            }
            lyapunov_state_terms(cfg, x, a.mode == MODE_SWEEP_GRID ? a.idx_begin + rel : -1, &pre[p],
                                 &pre[TP + p]);
        }
    }
    __syncthreads();
    refine_mark(a, RM_PROLOGUE);

    // Row blocks are dealt by `wslot`; warps w and w+4 share an SMSP (and its fp64 pipe), so
    // their slots sum to 7 and every SMSP gets the same share of the triangular panels.
    const int wg_ = warp & 3, wr_ = warp >> 2;
    const int wslot = wr_ == 0 ? wg_ : 7 - wg_;
    const int p_gen = tid & (TP - 1);
    const int jg = tid / TP;                          // 0..NT/TP-1
    const double2* ks_lane = reinterpret_cast<const double2*>(Ks) + (lane & 3) * KSTR + (lane >> 2);

    // ---- factor epilogue: mean and error bound of the outputs on factor f from tot[] (sum a^2, then
    // a . alpha per output)                                     (functions.py:439-456, 514)
    auto factor_epilogue = [&](int f, bool general, double s2) {
        const slb_gp_factor& F = cfg.gp.factors[f];
        if (tid < TP) {
            int qty = 1;
            for (int o = 0; o < D; ++o) {
                const slb_gp_output& Go = cfg.gp.outputs[o];
                if (Go.factor != f) continue;
                double mx = 0.0;                                   // functions.py:439
                if (Go.prior_mean != nullptr) {
                    mx = f64mul(zraw[tid], Go.prior_mean[0]);
                    for (int c = 1; c < DIN; ++c)
                        mx = f64add(mx, f64mul(zraw[c * TP + tid], Go.prior_mean[c]));
                    mx = f64mul(F.scale, mx);
                }
                const double fmean = f64add(tot[qty * TP + tid], mx) / F.scale;   // :442, :455
                double kss = F.kss;
                if (general) {
                    double zt[DIN];
#pragma unroll
                    for (int c = 0; c < DIN; ++c) zt[c] = zraw[c * TP + tid];
                    kss = s2 * kernel_expr_diag<DIN>(*kexpr, zt);
                }
                const double fvar = f64sub(kss, tot[tid]) / s2;                    // :450-451, :456
                post[o * TP + tid] = fmean;
                post[(SLB_MAX_OUT + o) * TP + tid] =
                    a.want_var ? fvar : f64mul(Go.beta, sqrt(fvar));              // :514
                ++qty;
            }
        }
    };

    const bool split = G * FS > 1;
    for (int f = 0; f < cfg.gp.num_factors; ++f) {
        if (fsel >= 0 && f != fsel) continue;      // another CTA of the tile owns this factor
        const slb_gp_factor& F = cfg.gp.factors[f];
        const int M = F.M, nrb = F.nrb;
        const int nk4 = (M + 3) >> 2;
        const double s2 = f64mul(F.scale, F.scale);
        const double variance = F.variance;
        const double* __restrict__ Xs = F.Xs;

        const bool general = KEXPR && F.kernel.num_prims > 0;
        if (general) {
            __syncthreads();                          // previous factor's readers are done
            const int* src = reinterpret_cast<const int*>(&F.kernel);
            for (int i = tid; i < (int)(sizeof(slb_kernel) / sizeof(int)); i += NT)
                reinterpret_cast<int*>(kexpr)[i] = src[i];
            __syncthreads();
        }
        double zs[DIN];
#pragma unroll
        for (int c = 0; c < DIN; ++c)
            zs[c] = general ? zraw[c * TP + p_gen] : zraw[c * TP + p_gen] / F.lengthscales[c];
        // red[warp][col][qty] holds THIS warp's running partial sums over its row blocks of all
        // panels of the factor; only the owning warp touches it, so the panel epilogues need no
        // barrier and warps that finish a triangular panel early move straight on.
        for (int i = lane; i < TP * NRED; i += 32) red[warp * TP * NRED + i] = 0.0;
        __syncwarp();
        int resident = -1;

        // row blocks of this CTA: all of them, or (split refine) the grp-th of G ranges of equal
        // triangular area, boundaries at nrb sqrt(k / G)
        int rlo = 0, rhi = nrb;
        if (G > 1) {
            rlo = __double2int_rd((double)nrb * sqrt((double)grp / (double)G));
            rhi = grp + 1 == G ? nrb : __double2int_rd((double)nrb * sqrt((double)(grp + 1) / (double)G));
        }
        for (int pbeg = rlo; pbeg < rhi; pbeg += 32) {
            double acc[RQ][NB][2];
#pragma unroll
            for (int q = 0; q < RQ; ++q)
#pragma unroll
                for (int nb = 0; nb < NB; ++nb) { acc[q][nb][0] = 0.0; acc[q][nb][1] = 0.0; }

            const int pend = min(pbeg + 32, rhi);
            int bq[RQ];
#pragma unroll
            for (int q = 0; q < RQ; ++q) bq[q] = pend - 1 - wslot - NW * (RQ - 1 - q);

            const int jp_last = (pend - 1) >> 5;          // the j-panel holding the diagonal of row pend - 1
            for (int jp = 0; jp <= jp_last; ++jp) {
                const int nkp = min(64, nk4 - 64 * jp);
                if (jp != resident) {
                    // ---- generation phase: K[j, p] for j in this panel (functions.py:438)
                    if (TIMING) t_s0 = clock64();
                    __syncthreads();
                    if (TIMING) { t_mark = clock64(); t_sync += t_mark - t_s0; }
                    const int j0 = PANEL * jp;
                    const int nj = min(PANEL, M - j0);
                    // stage the panel's training inputs in shared memory with one coalesced pass:
                    // every row is needed once by every warp, and read straight from global the
                    // first toucher of each row pays an L2 round trip inside the exp dependency
                    // chain
                    for (int i = tid; i < nj * DIN; i += NT) Xp[i] = Xs[(size_t)j0 * DIN + i];
                    __syncthreads();
                    // thread (p_gen, jg): fragment row r = jg % 4 of the pairs m = jg / 4 (mod PS),
                    // both halves (rows 8m + r and 8m + 4 + r); GP pairs per iteration = 2 GP
                    // interleaved exps
                    constexpr int PS = NT / TP / 4;      // pair stride between a thread's pairs
                    static_assert(NT / TP == 4 * PS, "generation needs a multiple of 4 groups");
                    const int gr = jg & 3, gpo = jg >> 2;
                    const int npairs = (nkp + 1) >> 1;
                    double2* ks2 = reinterpret_cast<double2*>(Ks);
                    constexpr int GP = 2;            // pairs per iteration = 2 GP interleaved exps
                    if (general) {
                        // covariance expression on the raw inputs, GP pairs = 2 GP rows per batch
                        for (int mm = gpo; mm < npairs; mm += GP * PS) {
                            const double* xr[2 * GP];
#pragma unroll
                            for (int u = 0; u < 2 * GP; ++u) {
                                const int jj = 8 * (mm + PS * (u >> 1)) + 4 * (u & 1) + gr;
                                xr[u] = Xp + min(jj, nj - 1) * DIN;
                            }
                            double kv[2 * GP];
                            kernel_expr_cross_n<DIN, 2 * GP>(*kexpr, zs, xr, exptab, kv);
#pragma unroll
                            for (int u = 0; u < 2 * GP; ++u) {
                                const int jj = 8 * (mm + PS * (u >> 1)) + 4 * (u & 1) + gr;
                                kv[u] = jj < nj ? s2 * kv[u] : 0.0;   // zero rows pad the last pair
                            }
#pragma unroll
                            for (int g = 0; g < GP; ++g)
                                if (mm + PS * g < npairs)
                                    ks2[((mm + PS * g) * 4 + gr) * KSTR + p_gen] =
                                        make_double2(kv[2 * g], kv[2 * g + 1]);
                        }
                    } else
                    for (int mm = gpo; mm < npairs; mm += GP * PS) {
                        double t2[2 * GP];
#pragma unroll
                        for (int u = 0; u < 2 * GP; ++u) {
                            const int jj = min(8 * (mm + PS * (u >> 1)) + 4 * (u & 1) + gr, nj - 1);
                            const double* xr = Xp + jj * DIN;
                            double acc2 = 0.0;
#pragma unroll
                            for (int c = 0; c < DIN; ++c) {
                                const double df = zs[c] - xr[c];
                                acc2 = fma(df, df, acc2);
                            }
                            t2[u] = acc2;
                        }
                        double kv[2 * GP];
#pragma unroll
                        for (int u = 0; u < 2 * GP; ++u) {
                            const int jj = 8 * (mm + PS * (u >> 1)) + 4 * (u & 1) + gr;
                            const double k = s2 * (variance * exp_neg_tab(-0.5 * t2[u], exptab));
                            kv[u] = jj < nj ? k : 0.0;          // zero rows pad the last pair
                        }
#pragma unroll
                        for (int g = 0; g < GP; ++g)
                            if (mm + PS * g < npairs)
                                ks2[((mm + PS * g) * 4 + gr) * KSTR + p_gen] =
                                    make_double2(kv[2 * g], kv[2 * g + 1]);
                    }
                    resident = jp;
                    if (TIMING) { t_s0 = clock64(); t_gen += t_s0 - t_mark; }
                    __syncthreads();
                    if (TIMING) t_sync += clock64() - t_s0;
                    refine_mark(a, RM_GEN + min(jp, 3));
                }
                if (TIMING) t_mark = clock64();
                // ---- contraction phase: acc[rows of this warp, 64 points] += W[rows, panel] K
                // active pairs of k-steps per row block: block b needs columns j <= 8b + 7, i.e.
                // pairs <= b; in the diagonal j-panel that is (b - pbeg) + 1 pairs
                const int npairs_mma = (nkp + 1) >> 1;
                int mend[RQ];
                const double2* ap[RQ];
#pragma unroll
                for (int q = 0; q < RQ; ++q) {
                    // row block b needs the pairs of k-steps <= b: in j-panel jp that is b - 32 jp + 1
                    const bool valid = bq[q] >= pbeg;
                    const int me = valid ? min(npairs_mma, max(0, bq[q] - 32 * jp + 1)) : 0;
                    mend[q] = me;
                    const int64_t b = valid ? bq[q] : 0;
                    ap[q] = reinterpret_cast<const double2*>(F.Wpack) +
                            (b * (b + 1) / 2 + 32 * jp) * 32 + lane;
                }
                int mprev = 0;
                if (mend[0] > mprev) { mma_run<0>(acc, ap, mprev, mend[0], ks_lane); mprev = mend[0]; }
                if (mend[1] > mprev) { mma_run<1>(acc, ap, mprev, mend[1], ks_lane); mprev = mend[1]; }
                if (mend[2] > mprev) { mma_run<2>(acc, ap, mprev, mend[2], ks_lane); mprev = mend[2]; }
                if (mend[3] > mprev) { mma_run<3>(acc, ap, mprev, mend[3], ks_lane); mprev = mend[3]; }
                if (TIMING) t_mma += clock64() - t_mark;
                refine_mark(a, RM_MMA + min(jp, 3));
            }
            if (TIMING) t_mark = clock64();

            // ---- panel epilogue: sum_i a_i^2 and sum_i a_i alpha_i   (functions.py:442, 451)
            int qty = 0;
            for (int o = -1; o < D; ++o) {
                double al[RQ] = {};
                if (o >= 0) {
                    if (cfg.gp.outputs[o].factor != f) continue;
                    const double* alpha = cfg.gp.outputs[o].alpha;
#pragma unroll
                    for (int q = 0; q < RQ; ++q)
                        if (bq[q] >= pbeg) al[q] = __ldg(alpha + 8 * bq[q] + (lane >> 2));
                }
                // per-thread sums over this warp's row blocks: 2 NB values, column 8nb + 2(T%4) + e
                constexpr int NV = 2 * NB;
                double v[NV];
#pragma unroll
                for (int nb = 0; nb < NB; ++nb) {
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        double t = 0.0;
#pragma unroll
                        for (int q = 0; q < RQ; ++q) {
                            const double x = acc[q][nb][e];
                            t = fma(x, (o < 0) ? x : al[q], t);
                        }
                        v[nb * 2 + e] = t;
                    }
                }
                row_lane_reduce<NB>(v, lane, red + (size_t)warp * TP * NRED + qty);
                ++qty;
            }
            __syncwarp();
            if (TIMING) t_epi += clock64() - t_mark;
        }

        // ---- cross-warp reduction in a fixed order (deterministic)
        if (TIMING) t_s0 = clock64();
        __syncthreads();
        if (TIMING) t_sync += clock64() - t_s0;
        if (tid < TP) {
            for (int r = 0; r < NRED; ++r) {
                double s = 0.0;
#pragma unroll
                for (int w = 0; w < NW; ++w) s += red[(w * TP + tid) * NRED + r];
                tot[r * TP + tid] = s;
            }
        }
        __syncthreads();

        if (split) {
            // split refine: this CTA's share of the factor's sums; the tile is finished below
            double* part = a.split_partial + ((size_t)blockIdx.x * SLB_MAX_OUT + f) * (NRED * TP);
            for (int i = tid; i < NRED * TP; i += NT) part[i] = tot[i];
            __syncthreads();
            refine_mark(a, RM_PARTIAL);
            continue;
        }
        factor_epilogue(f, general, s2);
        __syncthreads();
    }

    if (split) {
        // ---- split refine: the last CTA of the tile adds the partial sums in group order
        __shared__ int s_ticket;
        __threadfence();
        __syncthreads();
        if (tid == 0) s_ticket = atomicAdd(a.split_ticket + tile_index, 1);
        __syncthreads();
        refine_mark(a, RM_TICKET);
        if (s_ticket != G * FS - 1) {
            refine_mark(a, RM_EXIT);
            if (TIMING && lane == 0) {             // row-group CTAs that do not finish the tile
                long long* t = a.timing + ((size_t)blockIdx.x * NW + warp) * 8;
                long long g_end;
                asm volatile("mov.u64 %0, %globaltimer;" : "=l"(g_end));
                t[0] = t_gen; t[1] = t_mma; t[2] = t_epi; t[3] = clock64() - t_start;
                t[4] = g_start; t[5] = g_end; t[6] = t_sync; t[7] = 1;
            }
            return;
        }
        __threadfence();
        if (tid == 0) a.split_ticket[tile_index] = 0;                  // ready for the next launch
        for (int f = 0; f < cfg.gp.num_factors; ++f) {
            const slb_gp_factor& F = cfg.gp.factors[f];
            for (int i = tid; i < NRED * TP; i += NT) {
                double sum = 0.0;
                // the CTAs that worked on factor f: all G * FS of the tile, or the G of its factor slot
                const size_t cta0 = (size_t)tile_index * (G * FS) + (FS > 1 ? (size_t)f * G : 0);
                for (int g2 = 0; g2 < G; ++g2)
                    sum += __ldcg(a.split_partial + ((cta0 + g2) * SLB_MAX_OUT + f) * (NRED * TP) + i);
                tot[i] = sum;
            }
            const bool general = KEXPR && F.kernel.num_prims > 0;
            if (general) {
                const int* src = reinterpret_cast<const int*>(&F.kernel);
                for (int i = tid; i < (int)(sizeof(slb_kernel) / sizeof(int)); i += NT)
                    reinterpret_cast<int*>(kexpr)[i] = src[i];
            }
            __syncthreads();
            factor_epilogue(f, general, f64mul(F.scale, F.scale));
            __syncthreads();
        }
        refine_mark(a, RM_FACTORS);
    }

    if (TIMING && lane == 0) {
        long long* t = a.timing + ((size_t)blockIdx.x * NW + warp) * 8;
        long long g_end;
        asm volatile("mov.u64 %0, %globaltimer;" : "=l"(g_end));
        t[0] = t_gen; t[1] = t_mma; t[2] = t_epi; t[3] = clock64() - t_start;
        t[4] = g_start; t[5] = g_end; t[6] = t_sync; t[7] = 0;
    }
    // ---- tile epilogue: V(mu) on warps 0-1, the error bound on warps 2-3, then the decision
    {
        const int p = tid & (TP - 1);
        const bool live = tile0 + p < npts;
        int64_t rel = live ? tile0 + p : 0;
        if (a.index_list != nullptr) rel = a.index_list[rel];
        if constexpr (CD > 0) {
            // the closed form: lyapunov_decide's arithmetic by the register-only evaluators
            if (tid < 2 * TP && live) {
                double mu[CD], er[CD];
#pragma unroll
                for (int o = 0; o < CD; ++o) {
                    mu[o] = post[o * TP + p];
                    er[o] = post[(SLB_MAX_OUT + o) * TP + p];
                }
                if (tid < TP) {
                    if (a.mean != nullptr) for (int o = 0; o < CD; ++o) a.mean[rel * CD + o] = mu[o];
                    if (a.err != nullptr) for (int o = 0; o < CD; ++o) a.err[rel * CD + o] = er[o];
                    pre[2 * TP + p] = eval_quadratic_reg<CD>(cfg.lyapunov, mu);
                } else {
                    pre[3 * TP + p] = lyapunov_error_bound_closed<CD>(cfg, mu, er);
                }
            }
        } else if (tid < 2 * TP && live) {
            double mu[SLB_MAX_OUT], er[SLB_MAX_OUT];
            for (int o = 0; o < D; ++o) {
                mu[o] = post[o * TP + p];
                er[o] = post[(SLB_MAX_OUT + o) * TP + p];
            }
            if (tid < TP) {
                if (a.mean != nullptr) for (int o = 0; o < D; ++o) a.mean[rel * D + o] = mu[o];
                if (a.err != nullptr) for (int o = 0; o < D; ++o) a.err[rel * D + o] = er[o];
                if (a.mode != MODE_PREDICT) {
                    double vm[1];
                    eval_fn_small(cfg.lyapunov, mu, vm);
                    pre[2 * TP + p] = vm[0];
                }
            } else if (a.mode != MODE_PREDICT) {
                pre[3 * TP + p] = lyapunov_error_bound(cfg, mu, er);
            }
        }
        if (a.mode == MODE_PREDICT) return;
        __syncthreads();
        bool neg = false;
        if (tid < TP && live) {
            const slb_decision r =
                lyapunov_combine(pre[p], pre[TP + p], pre[2 * TP + p], pre[3 * TP + p]);
            neg = r.negative;
            a.negative[rel] = r.negative ? 1 : 0;
            if (a.values != nullptr) a.values[rel] = r.vx;
            if (a.decrease != nullptr) a.decrease[rel] = r.decrease;
            if (a.threshold != nullptr) a.threshold[rel] = r.threshold;
        }
        // refine pass of a step that folds its key (filter.cu): the warps of the tile's points (TP is a
        // multiple of 32)
        if (a.fold.rec != nullptr && tid < TP) fold_decided(a.fold, live, neg, rel, a.idx_begin);
        refine_mark(a, RM_DECIDED);
        if (split) {
            refine_mark(a, RM_EXIT);
            if (TP == 32 && a.marks != nullptr && tid == 0) a.marks[blockIdx.x * SLB_REFINE_MARKS + RM_FINISHER] = 1;
        }
    }
}

// The kernel: the tiles of this CTA (refine mode: from the list length and the split), one after the other.
// KEXPR: at least one factor carries a covariance expression (slb_kernel) instead of the plain
// RBF; the RBF-only instantiation keeps the lean generation loop.
template <int DIN, bool TIMING, bool KEXPR, int CD>
SLB_DEV void gp_tile_run(const slb_sweep& cfg, const slb_gp_args& a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    int64_t tile_index = blockIdx.x;
    int64_t tile_end = tile_index + 1, tile_step = 1;
    int grp = 0, G = 1;                // row group of this CTA / groups per tile (split refine)
    int fsel = -1, FS = 1;             // split refine with spare CTAs left: this CTA's factor / factors
                                       // dealt to separate CTAs (FS = 1: every CTA does all factors)
    // refine mode (slb_lyapunov_sweep_filtered): the point list was compacted by the filter
    // kernel, its length lives in device memory; CTAs beyond it leave before the first barrier
    int64_t npts = a.n;
    if (a.count != nullptr) {
        prefetch_descriptor_operands(cfg);
        npts = (int64_t)*a.count;
        // one launch per tile size; only the one whose range holds the list length does work
        if (npts <= a.count_min || npts > a.count_max) return;
        const int64_t ntiles = (npts + TP - 1) / TP;
        if (a.split_partial != nullptr) {
            // short list: spread every tile's rows over as many CTAs as the grid has to spare
            int64_t spare = (int64_t)gridDim.x / ntiles;
            // the factors of a stack are independent until the tile epilogue: with CTAs to spare they
            // go to different CTAs first (half the generation phases and barriers in every CTA's
            // serial chain), the rest of the spare CTAs splits the rows
            const int nfac = cfg.gp.num_factors;
            if (nfac > 1 && spare >= 2 * nfac) {
                FS = nfac;
                spare /= nfac;
            }
            G = (int)(spare < 1 ? 1 : (spare > SLB_SPLIT_MAX ? SLB_SPLIT_MAX : spare));
            const int per_tile = G * FS;
            if ((int64_t)blockIdx.x >= ntiles * per_tile) return;
            tile_index = blockIdx.x / per_tile;
            tile_end = tile_index + 1;
            const int rem = (int)(blockIdx.x % per_tile);
            grp = rem % G;
            if (FS > 1) fsel = rem / G;
        } else {
            // unsplit refine launches are persistent: the grid is one CTA per SM (the list length is
            // not known to the host; a grid sized for the longest possible list costs empty CTAs
            // when it is not this launch's turn), every CTA walks the tiles in strides
            tile_end = ntiles;
            tile_step = gridDim.x;
        }
        if (tile_index * TP >= npts) return;
        refine_mark(a, RM_ENTRY);
    }
    for (int64_t tile = tile_index; tile < tile_end; tile += tile_step) {
        gp_tile_body<DIN, TIMING, KEXPR, CD>(cfg, a, smem_raw, tile, npts, grp, G, fsel, FS, tile == tile_index);
        if (tile + tile_step < tile_end) __syncthreads();     // shared memory is reused by the next tile
    }
}

// TPV (= TP) only makes the kernel's NAME unique per translation unit: the units for the two tile
// sizes are compiled from this one source file, nvcc derives the prefix of internal-linkage
// kernels from the file name, and equally named kernels of different modules were resolved to
// the same device function (observed: the 64-point launch ran the 32-point code).
template <int DIN, bool TIMING, bool KEXPR, int TPV>
__global__ void __launch_bounds__(NT, CTAS_PER_SM)
gp_tile_kernel(const __grid_constant__ slb_sweep cfg, const slb_gp_args a) {
    gp_tile_run<DIN, TIMING, KEXPR, 0>(cfg, a);
}

// the refine pass of the filter's closed form, CD outputs (gp_tile_body; plain RBF factors)
template <int DIN, int CD, int TPV>
__global__ void __launch_bounds__(NT, CTAS_PER_SM)
gp_tile_closed_kernel(const __grid_constant__ slb_sweep cfg, const slb_gp_args a) {
    gp_tile_run<DIN, false, false, CD>(cfg, a);
}

// TPV: see gp_tile_kernel -- nvcc emits templates of this unnamed namespace as WEAK symbols under a
// prefix derived from the source file name, so the two tile-size units would otherwise share
// one launch function (the first one linked: every refine pass ran with 64-point tiles).
template <int DIN, bool TIMING, bool KEXPR, int CD = 0, int TPV = TP>
int launch_gp_tile(cudaStream_t st, const slb_sweep& cfg, const slb_gp_args& a) {
    static_assert(TPV == TP, "TPV only disambiguates the symbol");
    // the opt-in to > 48 KB of dynamic shared memory is a per-device function attribute
    // (atomic flags: sweeps may be issued from several host threads)
    static std::atomic<bool> configured[64];
    void (*kernel)(slb_sweep, slb_gp_args) = gp_tile_kernel<DIN, TIMING, KEXPR, TP>;
    if constexpr (CD > 0) kernel = gp_tile_closed_kernel<DIN, CD, TP>;
    int device = 0;
    SLB_CUDA(cudaGetDevice(&device));
    if (device < 0 || device >= 64 || !configured[device].load(std::memory_order_acquire)) {
        SLB_CUDA(cudaFuncSetAttribute(kernel,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)SMEM_TOTAL));
        if (device >= 0 && device < 64) configured[device].store(true, std::memory_order_release);
    }
    int64_t tiles = (a.n + TP - 1) / TP;
    // unsplit refine launches are persistent (see gp_tile_kernel): one CTA per SM
    if (a.count != nullptr && a.split_partial == nullptr && tiles > PREFETCH_CTAS) tiles = PREFETCH_CTAS;
    kernel<<<(unsigned)tiles, NT, SMEM_TOTAL, st>>>(cfg, a);
    SLB_LAUNCH_CHECK();
    return 0;
}

}  // namespace
