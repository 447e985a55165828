// gp_mean_grid.cuh -- GP posterior mean of a FunctionStack on a tile of a 2-D grid, contracted in fp64 from
// per-axis tables of kernel values, with a certified fp64-class error bound: the third mean scheme of the
// decision filter (filter.cu, filter_grid_mean_kernel), beside the per-point fp64 and fp32 means of
// gp_mean_staged.cuh.  tools/grid_mean_probe.py and tests/test_grid_mean_bound_host.py restate the tile
// constants and the bound below.
#pragma once
#include "gp_mean_staged.cuh"

// ---- the factored grid mean ---------------------------------------------------------------------------
// On a 2-D grid with plain RBF factors on z = [x0, x1, u] and the policy u = clip(a x0 + b x1, lo, hi)
// (a LINEAR map, optionally saturated and scaled), the kernel values of a tile of grid points factor
// into per-axis tables and the mean of the tile is a small matrix product on the fp64 tensor pipe.
// In a factor's units (w = z / l; xs_j the staged training rows) and on a region where the policy is
// affine, w2 = alpha w0 + beta w1 + const (alpha = a' l0 / l2, beta = b' l1 / l2, a' b' the scaled
// row; alpha = beta = 0 where u is saturated, a constant).  Centre the tile at cw (cw2 the affine value
// there), xi = w0 - cw0, eta = w1 - cw1, D_j = cw - xs_j; the exponent -|w - xs_j|^2 / 2 expands to
//     -|D_j|^2 / 2  -  xi p_j  -  eta q_j  -  (xi^2 + eta^2 + (alpha xi + beta eta)^2) / 2,
//     p_j = D_j0 + alpha D_j2,  q_j = D_j1 + beta D_j2,
// so  mean_o[i, k] = Q[i, k] sum_j (gamma_oj exp(-|D_j|^2 / 2) E0[i, j]) E1[k, j],
//     E0[i, j] = exp(-xi_i p_j),  E1[k, j] = exp(-eta_k q_j),  Q = exp(-(...) / 2) <= 1:
// The tables run on the uniform offsets xi_i = (i - 8) h0, h0 = unit0 / l0 (eta likewise): a column of
// E0 is g^(i - 8), g = exp(-h0 p_j), from two exponentials and 15 products -- 5 M exponentials per tile
// and regime (two per table column, one weight) instead of GR GC M -- and GR GC M fp64 FMAs in DMMA
// m8n8k4 (warp w of a group: the 8 x 8 block (w / GCB, w % GCB) of the tile; its C fragment is two points
// of each lane).  A tile computes every regime its points are in (saturated low / high, affine), each
// point keeps its own.  Its work items are its (factor, regime) pairs -- factors ascending, regimes 0, 1, 2
// as its points need them -- dealt in turn to the CTA's two warp groups, each with its own tables and
// named barrier: an item's arithmetic does not depend on the group that runs it, and the summation order
// within an item is fixed, so two runs are bit-identical.
// Certified bound (u = 2^-53, rho = max|xi| sqrt(1 + alpha^2) + max|eta| sqrt(1 + beta^2) >= |w - cw|,
// s_j = |D_j|, Sg = gamma_l1 >= sum_j |gamma_oj|):
//   each term: the weight and Q from one exp_neg_fast each (EPS_K relative; its reduction x = n ln2 / 512
//     + r is the same for positive arguments, |x| <= 294 here), each table entry a power |o| <= 8 of one
//     (8 (EPS_K + 2 u)), three products; arguments from D (one rounding each), K, p, q (fma chains), h p
//     and xi = fl(o h): relative error <= 18 EPS_K + u (3.5 (s_j + rho)^2 + 43) of the exact k_j;
//     k_j <= exp(-max(s_j - rho, 0)^2 / 2), so its contribution is <= (18 EPS_K + u (3.5 (sqrt(rho^2 + 2)
//     + rho)^2 + 43)) |gamma_j|;
//   the M-term sum (two DMMA chains): <= (Mp + 4) u sum_j |gamma_j| k_j (the tables' product exceeds k_j
//     by 1 / Q, the final product with Q takes it back);
//   the point itself: the grid's w0 = fl(x0 / l0) is within dev (computed, + 2 u |xi|) of cw0 + xi (w1
//     likewise; on the affine region w2 moves by |alpha| dev + |beta| dev with them); the policy's
//     fl(fl(x0 a) + fl(x1 b)) scaled, alpha, beta and cw2 are within 10 u (|alpha| W0 + |beta| W1) of
//     the affine w2 (W = max |w| over the tile); |d k_j / d w_c| <= 1, so each enters times sum |gamma|;
//   dropped rows (|D_j|^2 > GRID_K_DROP: weight 0): each k_j <= exp(-(sqrt(K_DROP) - rho)^2 / 2);
//     products that leave the fp64 range downwards: < 1e-150 (Mp + 1) absolute (|table args| <=
//     rho sqrt(K_DROP) <= 294);
//   the other evaluation orders of the same mean (gamma itself and the a . alpha form of the full
//     posterior, its expanded distance): 7e-16 (M + 8) + 4.5e-16 (|w|^2 / 2 + hmax), as mean_output_finish.
// dm = 1.05 (sum of the above) Sg / |scale|.  A tile and regime with rho > GRID_RHO_MAX or a non-finite
// constant leaves its points to the fp64 route (dm = inf), like points the prologue finds insane.
constexpr int GR = 16, GC = 16;        // grid rows (axis 0) x columns (axis 1, contiguous) per CTA tile
constexpr int GCB = GC / 8;            // column blocks
constexpr int GG = 2;                  // warp groups per CTA: the tile's work items alternate between them
constexpr int GGT = GR * GC / 2;       // threads per group: one warp per 8 x 8 block, two points per thread
constexpr int GT = GG * GGT;           // threads per CTA: one per point in the prologue and the decision (two
                                       // CTAs per SM: one's barriers and round trips hide behind the other)
constexpr int GJ = 128;                // training rows per chunk of the tables
constexpr int GNO = 4;                 // outputs per factor (screening_applicable: at most 4 outputs)
constexpr double GRID_RHO_MAX = 12.0;
constexpr double GRID_K_DROP = 600.0;
constexpr int GFS = 36;                // doubles per fragment (32 used): the recurrence's column stores hit
                                       // every bank pair once, the contraction's loads stay contiguous
constexpr int GTAB = (GR / 8) * (GJ / 4) * GFS;   // one table of a chunk, in fragments
constexpr int GGRP = 2 * GTAB + GNO * GJ + 2 * GJ + 2 * (GR + GC);   // doubles of one group's item state
// the CTA's dynamic shared memory, in doubles: [GG][GGRP] the groups' item state, [512] the exp table,
// [GR GC][3] z of the tile's points, [GR GC][GNO] their means mu and bounds dm, then [GT / 32] ints: the
// regimes present in each warp's points, and [GR GC] bytes: the points' regimes.  111.3 KB: two CTAs per SM
// with their 1 KB of static shared memory and 1 KB reserved each (228 KB).
constexpr int GSMEM_TAB = GG * GGRP;
constexpr int GSMEM_Z = GSMEM_TAB + 512;
constexpr int GSMEM_MU = GSMEM_Z + GR * GC * 3;
constexpr int GSMEM_DM = GSMEM_MU + GR * GC * GNO;
constexpr int GSMEM_REG = GSMEM_DM + GR * GC * GNO;
static_assert(GR == 16 && GC == 16, "the recurrence runs 8 steps each way from the tile's centre");
static_assert(GT == GR * GC, "one point per thread in the prologue and the decision");
static_assert(GGT == GJ, "one training row per group thread and chunk");

inline size_t grid_mean_smem_bytes() {
    return (size_t)GSMEM_REG * sizeof(double) + (GT / 32) * sizeof(int) + GR * GC;
}

// the barrier of warp group grp alone (barrier 0 is __syncthreads'; constant ids: three barriers in all)
SLB_DEV void grid_group_sync(int grp) {
    if (grp == 0) asm volatile("bar.sync 1, %0;" ::"n"(GGT) : "memory");
    else asm volatile("bar.sync 2, %0;" ::"n"(GGT) : "memory");
}

// one work item of the tile -- factor f with NO outputs (compile-time: accumulators in registers), regime r
// -- on the calling thread's warp group (its item state at gsm); writes mu / dm [point][output] of the
// tile's points in regime r for the factor's outputs.  z / reg: [point] as the prologue left them.
template <int NO>
SLB_DEV void grid_mean_item(const slb_sweep& cfg, int f, int r, const int* outs, double* gsm, const double* tab,
                            int64_t row0, int64_t col0, const double* z, const int8_t* reg, double* mu, double* dm) {
    const slb_gp_factor& F = cfg.gp.factors[f];
    const slb_grid& g = cfg.grid;
    const slb_function& pol = cfg.policy;
    const int grp = threadIdx.x / GGT, gt = threadIdx.x % GGT;
    const int lane = gt & 31, warp = gt >> 5;
    const int rb = warp / GCB, cb = warp % GCB;
    double* e0f = gsm;                         // [GR / 8][J / 4][GFS]: DMMA A fragments
    double* e1f = e0f + GTAB;                  // [GC / 8][J / 4][GFS]: DMMA B fragments
    double* wg = e1f + GTAB;                   // [NO][GJ] gamma_oj exp(-|D_j|^2 / 2)
    double* pq = wg + GNO * GJ;                // [2][GJ]
    double* xi = pq + 2 * GJ;                  // [GR] xi of the tables: (i - GR / 2) h0
    double* eta = xi + GR;                     // [GC]
    double* dev = eta + GC;                    // [GR + GC] |w - cw - xi| of the grid's own points
    const double l0 = F.lengthscales[0], l1 = F.lengthscales[1], l2 = F.lengthscales[2];
    // the centre: grid point (GR / 2, GC / 2) of the tile, in the factor's units
    const double cw0 = f64add(f64mul((double)(row0 + GR / 2), g.unit_maxes[0]), g.offset[0]) / l0;
    const double cw1 = f64add(f64mul((double)(col0 + GC / 2), g.unit_maxes[1]), g.offset[1]) / l1;
    grid_group_sync(grp);                      // the group's previous item is done with the tables
    // the tables run on the uniform offsets xi_i = (i - GR / 2) h0, h0 = unit / l0 (a recurrence along the
    // axis); the grid's own points are within dev of them (a perturbation of the point, in the bound)
    const double h0 = g.unit_maxes[0] / l0, h1 = g.unit_maxes[1] / l1;
    if (gt < GR + GC) {
        const int c = gt < GR ? 0 : 1;
        const int i = c == 0 ? gt : gt - GR;
        const int64_t gi = (c == 0 ? row0 : col0) + i;
        const double x = f64add(f64mul((double)gi, g.unit_maxes[c]), g.offset[c]);   // grid_index_to_state
        const double ideal = (double)(i - GR / 2) * (c == 0 ? h0 : h1);
        xi[gt] = ideal;
        dev[gt] = fabs((x / (c == 0 ? l0 : l1) - (c == 0 ? cw0 : cw1)) - ideal);
    }
    grid_group_sync(grp);
    double mxi = 0.0, meta = 0.0, pert = 0.0;
#pragma unroll
    for (int r = 0; r < GR; ++r) mxi = fmax(mxi, fabs(xi[r]));
#pragma unroll
    for (int k = 0; k < GC; ++k) meta = fmax(meta, fabs(eta[k]));
#pragma unroll
    for (int k = 0; k < GR + GC; ++k) pert = fmax(pert, dev[k]);
    const int ti = rb * 8 + (lane >> 2);
    const int tk0 = cb * 8 + 2 * (lane & 3);
    const int Mp = padded_rows(F.M);
    const double u53 = 1.1102230246251565e-16;
    const double sc = (pol.flags & SLB_FLAG_SCALE) ? pol.out_scale : 1.0;
    {
        double alpha = 0.0, beta = 0.0, cw2;
        if (r == 2) {
            alpha = f64mul(f64mul(__ldg(pol.matrix + 0), sc), l0) / l2;
            beta = f64mul(f64mul(__ldg(pol.matrix + 1), sc), l1) / l2;
            cw2 = fma(alpha, cw0, f64mul(beta, cw1));
        } else {
            const double lim = r == 0 ? pol.lower : pol.upper;
            cw2 = ((pol.flags & SLB_FLAG_SCALE) ? f64mul(lim, pol.out_scale) : lim) / l2;
        }
        const double rho = mxi * sqrt(fma(alpha, alpha, 1.0)) + meta * sqrt(fma(beta, beta, 1.0));
        const bool ok = rho <= GRID_RHO_MAX && fabs(cw0) < 1e100 && fabs(cw1) < 1e100 && fabs(cw2) < 1e100 &&
                        fabs(alpha) < 1e100 && fabs(beta) < 1e100;
        double acc[NO][2][2];
#pragma unroll
        for (int q = 0; q < NO; ++q) { acc[q][0][0] = acc[q][0][1] = acc[q][1][0] = acc[q][1][1] = 0.0; }
        // the thread's training row of a chunk (GGT == GJ), loaded one chunk ahead: its L2 round trip runs
        // behind the previous chunk's tables and contraction
        double nx[3] = {0.0, 0.0, 0.0}, ng[NO];
#pragma unroll
        for (int q = 0; q < NO; ++q) ng[q] = 0.0;
        if (ok && gt < Mp) {
            const double2 x01 = *reinterpret_cast<const double2*>(F.Xf + (size_t)gt * 4);
            nx[0] = x01.x; nx[1] = x01.y; nx[2] = F.Xf[(size_t)gt * 4 + 2];
#pragma unroll
            for (int q = 0; q < NO; ++q) ng[q] = cfg.gp.outputs[outs[q]].gamma_f[gt];
        }
        for (int j0 = 0; ok && j0 < Mp; j0 += GJ) {
            const int J = min(GJ, Mp - j0), J4 = J >> 2;
            grid_group_sync(grp);              // the previous chunk's tables are consumed
            if (gt < J) {
                const double d0 = cw0 - nx[0], d1 = cw1 - nx[1], d2 = cw2 - nx[2];
                const double K = fma(d0, d0, fma(d1, d1, d2 * d2));
                const bool keep = K <= GRID_K_DROP;          // dropped rows: weight 0, tables of ones
                bool far;
                const double w = keep ? exp_neg_fast(-0.5 * K, tab, far) : 0.0;
                pq[gt] = keep ? fma(alpha, d2, d0) : 0.0;
                pq[GJ + gt] = keep ? fma(beta, d2, d1) : 0.0;
#pragma unroll
                for (int q = 0; q < NO; ++q) wg[q * GJ + gt] = ng[q] * w;
            }
            const int jn = j0 + GJ + gt;
            if (jn < Mp) {
                const double2 x01 = *reinterpret_cast<const double2*>(F.Xf + (size_t)jn * 4);
                nx[0] = x01.x; nx[1] = x01.y; nx[2] = F.Xf[(size_t)jn * 4 + 2];
#pragma unroll
                for (int q = 0; q < NO; ++q) ng[q] = cfg.gp.outputs[outs[q]].gamma_f[jn];
            }
            grid_group_sync(grp);
            // one table column (training row jj, axis c) per task: exp(-o h p) = g^o for the offsets
            // o = -8 .. 7 from two exps g = exp(-h p), 1 / g = exp(h p) and products outwards from o = 0
            for (int task = gt; task < 2 * J; task += GGT) {
                const int c = task >= J ? 1 : 0, jj = task - c * J;
                const double t = (c ? h1 : h0) * pq[c * GJ + jj];
                bool far;
                const double gd = exp_neg_fast(-t, tab, far), gu = exp_neg_fast(t, tab, far);
                double* col = (c ? e1f : e0f) + (jj >> 2) * GFS + (jj & 3);   // + block (m / 8) J4 GFS + (m % 8) 4
                col[J4 * GFS] = 1.0;                                          // m = 8: o = 0
                double v = 1.0;
#pragma unroll
                for (int o = 1; o < 8; ++o) { v *= gd; col[J4 * GFS + o * 4] = v; }      // m = 8 + o
                v = 1.0;
#pragma unroll
                for (int o = 1; o <= 8; ++o) { v *= gu; col[(8 - o) * 4] = v; }          // m = 8 - o
            }
            grid_group_sync(grp);
            const double* pa = e0f + rb * J4 * GFS + lane;
            const double* pb = e1f + cb * J4 * GFS + lane;
#pragma unroll 2
            for (int s = 0; s < J4; s += 2) {            // J4 is even (rows padded to 8)
                double af[2][NO], bf[2];
#pragma unroll
                for (int t = 0; t < 2; ++t) {
                    const double a0 = pa[(s + t) * GFS];
                    bf[t] = pb[(s + t) * GFS];
#pragma unroll
                    for (int q = 0; q < NO; ++q) af[t][q] = a0 * wg[q * GJ + 4 * (s + t) + (lane & 3)];
                }
#pragma unroll
                for (int q = 0; q < NO; ++q) {
                    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                                 : "+d"(acc[q][0][0]), "+d"(acc[q][0][1]) : "d"(af[0][q]), "d"(bf[0]));
                    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                                 : "+d"(acc[q][1][0]), "+d"(acc[q][1][1]) : "d"(af[1][q]), "d"(bf[1]));
                }
            }
        }
        // the bound of this tile and regime (relative to gamma_l1, see above)
        const double W0 = fabs(cw0) + mxi, W1 = fabs(cw1) + meta;
        const double W2 = r == 2 ? fabs(alpha) * W0 + fabs(beta) * W1 : fabs(cw2);
        const double sq = sqrt(rho * rho + 2.0) + rho, kd = sqrt(GRID_K_DROP) - rho;
        const double eps = 1.05 * (18.2 * EPS_K + u53 * (1.01 * (3.5 * sq * sq + 43.0) + 1.02 * (Mp + 4)) +
                                   1.01 * pert * (r == 2 ? 2.0 + fabs(alpha) + fabs(beta) : 2.0) +
                                   u53 * (2.0 * (mxi + meta) + (r == 2 ? 10.0 * W2 : 2.0 * W2)) +
                                   4.5e-16 * (0.5 * (W0 * W0 + W1 * W1 + W2 * W2) + F.hmax) + 7e-16 * (F.M + 8) +
                                   exp(-0.5 * kd * kd));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int p = ti * GC + tk0 + h;
            if (reg[p] != r) continue;
            const double x0 = xi[ti], e1 = eta[tk0 + h];
            const double v = fma(alpha, x0, beta * e1);
            bool far;
            const double Q = exp_neg_fast(-0.5 * fma(x0, x0, fma(e1, e1, v * v)), tab, far);
#pragma unroll
            for (int q = 0; q < NO; ++q) {
                const slb_gp_output& G = cfg.gp.outputs[outs[q]];
                const double m =
                    f64add(f64mul(acc[q][0][h] + acc[q][1][h], Q), prior_mean_term<3>(F, G, z + 3 * p)) / F.scale;
                const double bound = ok && eps < 1e-3
                                         ? (eps * G.gamma_l1 + 1e-150 * (Mp + 1)) / fabs(F.scale) + 1e-300
                                         : f64_inf();
                mu[p * GNO + outs[q]] = m;         // outs[q] < GNO (grid_mean_applicable: at most 4 outputs)
                dm[p * GNO + outs[q]] = bound;
            }
        }
    }
}
