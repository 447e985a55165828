// bellman_tile.cu -- PolicyIteration.discrete_policy_optimization (reinforcement_learning.py:213-279)
// with the action factored out of the exponent.
//
// The reference evaluates future_values(states, a_i) once per action a_i (:266-270): n_A sweeps, each
// with D M kernel values (one exp each) per state.  For the (ARD) RBF kernel of the GP dynamics
//     k([x, a], [X_j, A_j]) = v exp(-|x - X_j|^2 / 2) exp(-|a - A_j|^2 / 2)        (scaled inputs)
// so the GP mean of output o for state s and action i is a dense contraction
//     mean_o[i, s] = sum_j G_o[i, j] kx[j, s],   G_o[i, j] = gamma_o,j v exp(-|a_i - A_j|^2 / 2)
// with kx[j, s] = exp(-|x_s - X_j|^2 / 2) generated ONCE per state: M exps instead of n_A M, and
// an [n_A x M] x [M x states] fp64 GEMM on the tensor pipe (DMMA.8x8x4) instead of n_A M more
// exps.  At C3 size (512 x 512 states, n_A = 101, M = 500, two factors): 5.3e10 flop against
// 2.6e10 exp.
//   * pack kernel: G_o in DMMA A-fragment order, k-steps paired (the layout of slb_pack_factor);
//   * tile kernel: CTA = 64 states, 8 warps; per output the kx tile of a 128-row chunk is generated
//     into shared memory (pair-interleaved B-fragment layout of gp_tile.cuh), every warp owns up to
//     two 8-action row blocks x 64 states of the product; the means land in shared memory, then
//     r(x, a) + gamma V(mean) for every (state, action) pair, the constraint (:272-275) and
//     np.argmax's first-maximum / first-NaN rule (:278).
#define SLB_EVAL_NOINLINE 1
#include "common.cuh"

#include <atomic>

namespace {

constexpr int BS = 64;                 // states per CTA
constexpr int BNT = 256;               // threads per CTA
constexpr int BNW = BNT / 32;
constexpr int BCH = 128;               // training rows per generated chunk (16 pairs of k-steps)
constexpr int BKSTR = BS + 2;          // see gp_tile.cuh: conflict-free 128-bit B-fragment reads
constexpr int BNB = BS / 8;            // 8-state column blocks
constexpr int BMAXRB = 16;             // row blocks (8 actions each) per pass: two per warp

struct argmax_args {
    int64_t idx_begin, n;
    const double* actions;             // [n_actions, m]
    int n_actions, m;
    const double* constraint;          // [n_actions, n] or nullptr
    int32_t* best;
    double* best_value;
    const double* gpack[SLB_MAX_OUT];  // per output: packed G (all row blocks, all pairs)
    int nrb;                           // row blocks = ceil(n_actions / 8)
};

SLB_DEV void dmma884(double& c0, double& c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

// np.argmax order on (value, index): NaN counts as the maximum, the first one wins
SLB_DEV bool better(double v, int i, double bv, int bi) {
    const bool vn = v != v, bn = bv != bv;
    if (vn || bn) return vn && (!bn || i < bi);
    return v > bv || (v == bv && i < bi);
}

// G_o[i, j] = gamma_f[o][j] exp(-|a_i / l_a - A_j|^2 / 2) in A-fragment order: block (b, kp) holds
// 32 lanes x 2 doubles; lane T, half h <-> row 8b + T/4, column 8kp + 4h + T%4
__global__ void __launch_bounds__(256)
bellman_pack_actions_kernel(const __grid_constant__ slb_gp_stack gp, int o, int d,
                            const double* __restrict__ actions, int n_actions, int m, int nrb,
                            int npairs, double* __restrict__ out) {
    const int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int64_t total = (int64_t)nrb * npairs * 64;
    if (e >= total) return;
    const int h = (int)(e & 1), lane = (int)((e >> 1) & 31);
    const int64_t blk = e >> 6;
    const int kp = (int)(blk % npairs), b = (int)(blk / npairs);
    const int i = 8 * b + (lane >> 2), j = 8 * kp + 4 * h + (lane & 3);
    const slb_gp_output& G = gp.outputs[o];
    const slb_gp_factor& F = gp.factors[G.factor];
    double v = 0.0;
    if (i < n_actions && j < F.M) {
        double a2 = 0.0;
        for (int c = 0; c < m; ++c) {
            const double df = actions[i * m + c] / F.lengthscales[d + c] - F.Xs[(size_t)j * (d + m) + d + c];
            a2 = fma(df, df, a2);
        }
        v = G.gamma_f[j] * exp(-0.5 * a2);
    }
    out[e] = v;
}

template <int DS>
__global__ void __launch_bounds__(BNT, 1)
bellman_argmax_tile_kernel(const __grid_constant__ slb_bellman cfg, const argmax_args a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double* Ks = reinterpret_cast<double*>(smem_raw);                  // [(BCH/8) * 4 * BKSTR * 2]
    double* Xp = Ks + (BCH / 8) * 4 * BKSTR * 2;                       // [BCH][DS]
    double* exptab = Xp + BCH * DS;                                    // [64]
    double* xraw = exptab + 64;                                        // [DS][BS]
    double* cand_v = xraw + DS * BS;                                   // [4][BS]
    int* cand_i = reinterpret_cast<int*>(cand_v + 4 * BS);             // [4][BS]
    double* Cm = reinterpret_cast<double*>(cand_i + 4 * BS);           // [D][8 nrb_pass][BS] means

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t tile0 = (int64_t)blockIdx.x * BS;
    const int D = cfg.gp.num_outputs;
    const int din = DS + a.m;
    load_exp_table(exptab);
    if (tid < BS) {
        int64_t rel = tile0 + tid;
        if (rel > a.n - 1) rel = a.n - 1;
        double x[SLB_MAX_DIM];
        grid_index_to_state(cfg.grid, a.idx_begin + rel, x);
#pragma unroll
        for (int c = 0; c < DS; ++c) xraw[c * BS + tid] = x[c];
    }
    __syncthreads();

    const int p_gen = tid & (BS - 1), jg = tid >> 6;                   // generation: point, fragment row
    const double2* ks_lane = reinterpret_cast<const double2*>(Ks) + (lane & 3) * BKSTR + (lane >> 2);
    double bestv = 0.0;
    int besti = -1;

    // passes of up to BMAXRB row blocks (128 actions); n_A = 101 is one pass
    for (int rb0 = 0; rb0 < a.nrb; rb0 += BMAXRB) {
        const int nrbp = min(BMAXRB, a.nrb - rb0);
        for (int o = 0; o < D; ++o) {
            const slb_gp_output& G = cfg.gp.outputs[o];
            const slb_gp_factor& F = cfg.gp.factors[G.factor];
            const int M = F.M;
            const int npairs = (M + 7) >> 3;
            double xs[DS];
#pragma unroll
            for (int c = 0; c < DS; ++c) xs[c] = xraw[c * BS + p_gen] / F.lengthscales[c];
            // this warp's row blocks of the pass: warp and warp + 8
            double acc[2][BNB][2];
#pragma unroll
            for (int q = 0; q < 2; ++q)
#pragma unroll
                for (int nb = 0; nb < BNB; ++nb) { acc[q][nb][0] = 0.0; acc[q][nb][1] = 0.0; }
            const bool on0 = warp < nrbp, on1 = warp + BNW < nrbp;
            const double2* ap0 = reinterpret_cast<const double2*>(a.gpack[o]) +
                                 (size_t)(rb0 + warp) * npairs * 32 + lane;
            const double2* ap1 = ap0 + (size_t)BNW * npairs * 32;
            for (int c0 = 0; c0 < M; c0 += BCH) {
                const int nj = min(BCH, M - c0);
                const int npc = (nj + 7) >> 3;
                __syncthreads();                                       // Ks / Xp readers are done
                for (int i = tid; i < nj * DS; i += BNT)
                    Xp[i] = F.Xs[(size_t)(c0 + i / DS) * din + i % DS];
                __syncthreads();
                // kx[j, s] for the chunk: thread (p_gen, jg) fills fragment row jg of every pair
                double2* ks2 = reinterpret_cast<double2*>(Ks);
                for (int mm = 0; mm < npc; mm += 2) {
                    double kv[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const int jj = 8 * (mm + (u >> 1)) + 4 * (u & 1) + jg;
                        const double* xr = Xp + min(jj, nj - 1) * DS;
                        double a2 = 0.0;
#pragma unroll
                        for (int c = 0; c < DS; ++c) { const double df = xs[c] - xr[c]; a2 = fma(df, df, a2); }
                        kv[u] = a2;
                    }
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        const int jj = 8 * (mm + (u >> 1)) + 4 * (u & 1) + jg;
                        const double k = exp_neg_tab(-0.5 * kv[u], exptab);
                        kv[u] = jj < nj ? k : 0.0;
                    }
                    ks2[(mm * 4 + jg) * BKSTR + p_gen] = make_double2(kv[0], kv[1]);
                    if (mm + 1 < npc) ks2[((mm + 1) * 4 + jg) * BKSTR + p_gen] = make_double2(kv[2], kv[3]);
                }
                __syncthreads();
                // contraction over the chunk's pairs; A fragments one pair ahead
                if (on0) {
                    const int pk0 = c0 >> 3;
                    double2 a0 = __ldg(ap0 + (size_t)pk0 * 32);
                    double2 a1 = on1 ? __ldg(ap1 + (size_t)pk0 * 32) : make_double2(0.0, 0.0);
                    for (int mm = 0; mm < npc; ++mm) {
                        const int nx = min(mm + 1, npc - 1);
                        const double2 n0 = __ldg(ap0 + (size_t)(pk0 + nx) * 32);
                        const double2 n1 = on1 ? __ldg(ap1 + (size_t)(pk0 + nx) * 32) : make_double2(0.0, 0.0);
                        const double2* kb = ks_lane + mm * (4 * BKSTR);
#pragma unroll
                        for (int half = 0; half < BNB; half += 4) {
                            double2 b[4];
#pragma unroll
                            for (int nb = 0; nb < 4; ++nb) b[nb] = kb[(half + nb) * 8];
#pragma unroll
                            for (int nb = 0; nb < 4; ++nb) {
                                dmma884(acc[0][half + nb][0], acc[0][half + nb][1], a0.x, b[nb].x);
                                dmma884(acc[1][half + nb][0], acc[1][half + nb][1], a1.x, b[nb].x);
                            }
#pragma unroll
                            for (int nb = 0; nb < 4; ++nb) {
                                dmma884(acc[0][half + nb][0], acc[0][half + nb][1], a0.y, b[nb].y);
                                dmma884(acc[1][half + nb][0], acc[1][half + nb][1], a1.y, b[nb].y);
                            }
                        }
                        a0 = n0; a1 = n1;
                    }
                }
            }
            // means of this output -> Cm[o][local action][state]
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                if (!(q == 0 ? on0 : on1)) continue;
                const int row = 8 * (warp + q * BNW) + (lane >> 2);
                double* crow = Cm + ((size_t)o * 8 * BMAXRB + row) * BS;
#pragma unroll
                for (int nb = 0; nb < BNB; ++nb)
                    *reinterpret_cast<double2*>(crow + 8 * nb + 2 * (lane & 3)) =
                        make_double2(acc[q][nb][0], acc[q][nb][1]);
            }
        }
        __syncthreads();
        // ---- r(x, a) + gamma V(mean) for every (state, action) of the pass  (:95-104, :266-275)
        {
            const int s = tid & (BS - 1), g = tid >> 6;
            const int64_t rel = min(tile0 + s, a.n - 1);
            double z[SLB_MAX_IN];
#pragma unroll
            for (int c = 0; c < DS; ++c) z[c] = xraw[c * BS + s];
            const int i_end = min(a.n_actions, 8 * (rb0 + nrbp));
            // state part of every output's linear prior mean (the action terms follow per action, in
            // the same left-to-right order as the unfactored path)
            double mstate[SLB_MAX_OUT], scale[SLB_MAX_OUT];
            const double* pm[SLB_MAX_OUT];
            for (int o = 0; o < D; ++o) {
                const slb_gp_output& G = cfg.gp.outputs[o];
                scale[o] = cfg.gp.factors[G.factor].scale;
                pm[o] = G.prior_mean;
                mstate[o] = 0.0;
                if (pm[o] != nullptr) {
                    mstate[o] = f64mul(z[0], pm[o][0]);
                    for (int c = 1; c < DS; ++c) mstate[o] = f64add(mstate[o], f64mul(z[c], pm[o][c]));
                }
            }
            for (int i = 8 * rb0 + g; i < i_end; i += 4) {
                for (int c = 0; c < a.m; ++c) z[DS + c] = a.actions[i * a.m + c];
                double mu[SLB_MAX_OUT], r[SLB_MAX_OUT], v[SLB_MAX_OUT];
                for (int o = 0; o < D; ++o) {
                    double mx = 0.0;
                    if (pm[o] != nullptr) {
                        mx = mstate[o];
                        for (int c = DS; c < din; ++c) mx = f64add(mx, f64mul(z[c], pm[o][c]));
                        mx = f64mul(scale[o], mx);
                    }
                    const double dot = Cm[((size_t)o * 8 * BMAXRB + (i - 8 * rb0)) * BS + s];
                    mu[o] = f64add(dot, mx) / scale[o];
                }
                eval_fn_small(cfg.reward, z, r);
                eval_fn(cfg.value, mu, v);
                double val = f64add(r[0], f64mul(cfg.gamma, v[0]));
                if (a.constraint != nullptr && a.constraint[(int64_t)i * a.n + rel] < 0.0) val = -INFINITY;
                if (besti < 0 || better(val, i, bestv, besti)) { bestv = val; besti = i; }
            }
        }
        __syncthreads();                                               // Cm is rewritten by the next pass
    }
    {
        const int s = tid & (BS - 1), g = tid >> 6;
        cand_v[g * BS + s] = bestv;
        cand_i[g * BS + s] = besti;
    }
    __syncthreads();
    if (tid < BS && tile0 + tid < a.n) {
        double bv = cand_v[tid];
        int bi = cand_i[tid];
        for (int g = 1; g < 4; ++g) {
            const double v = cand_v[g * BS + tid];
            const int i = cand_i[g * BS + tid];
            if (i >= 0 && (bi < 0 || better(v, i, bv, bi))) { bv = v; bi = i; }
        }
        a.best[tile0 + tid] = bi;
        if (a.best_value != nullptr) a.best_value[tile0 + tid] = bv;
    }
}

constexpr size_t tile_smem(int ds, int D) {
    return ((size_t)(BCH / 8) * 4 * BKSTR * 2 + (size_t)BCH * ds + 64 + (size_t)ds * BS + 4 * BS) *
               sizeof(double) + 4 * BS * sizeof(int) + (size_t)D * 8 * BMAXRB * BS * sizeof(double);
}
// A Bellman GP stack has one output per state dimension (slb_validate_bellman), so the means of a
// pass take D = d slices of Cm: from d = 3 on the tile no longer fits, and only DS = 1, 2 exist.
static_assert(tile_smem(2, 2) <= 227 * 1024 && tile_smem(3, 3) > 227 * 1024,
              "factored argmax: state dimensions 1..2 fit the CTA, 3 does not");

template <int DS>
int launch_argmax_tile(cudaStream_t st, const slb_bellman& cfg, const argmax_args& a) {
    static std::atomic<bool> configured[64];
    int device = 0;
    SLB_CUDA(cudaGetDevice(&device));
    if (device < 0 || device >= 64 || !configured[device].load(std::memory_order_acquire)) {
        SLB_CUDA(cudaFuncSetAttribute(bellman_argmax_tile_kernel<DS>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
        if (device >= 0 && device < 64) configured[device].store(true, std::memory_order_release);
    }
    const size_t smem = tile_smem(DS, cfg.gp.num_outputs);
    const int64_t tiles = (a.n + BS - 1) / BS;
    bellman_argmax_tile_kernel<DS><<<(unsigned)tiles, BNT, smem, st>>>(cfg, a);
    SLB_LAUNCH_CHECK();
    return 0;
}

}  // namespace

// light.cu: can this argmax take the factored path, and how much workspace does it need?
bool slb_argmax_factorable(const slb_bellman& cfg, int m, int n_actions) {
    if (cfg.gp.num_outputs <= 0 || n_actions < 2) return false;
    const int d = cfg.grid.ndim;
    if (d < 1 || d > 2 || m < 1) return false;
    for (int f = 0; f < cfg.gp.num_factors; ++f)
        if (cfg.gp.factors[f].kernel.num_prims > 0 || cfg.gp.factors[f].M == 0) return false;
    for (int o = 0; o < cfg.gp.num_outputs; ++o)
        if (cfg.gp.outputs[o].gamma_f == nullptr) return false;
    return tile_smem(d, cfg.gp.num_outputs) <= 227 * 1024;
}

int64_t slb_argmax_workspace_bytes(const slb_bellman& cfg, int n_actions) {
    const int64_t nrb = (n_actions + 7) / 8;
    int64_t total = 0;
    for (int o = 0; o < cfg.gp.num_outputs; ++o) {
        const int M = cfg.gp.factors[cfg.gp.outputs[o].factor].M;
        total += nrb * ((M + 7) / 8) * 64 * (int64_t)sizeof(double);
    }
    return total;
}

int slb_launch_argmax_factored(cudaStream_t st, const slb_bellman& cfg, int64_t idx_begin, int64_t n,
                               const double* actions, int n_actions, int m, const double* constraint,
                               int32_t* best, double* best_value, void* workspace) {
    argmax_args a;
    a.idx_begin = idx_begin; a.n = n; a.actions = actions; a.n_actions = n_actions; a.m = m;
    a.constraint = constraint; a.best = best; a.best_value = best_value;
    a.nrb = (n_actions + 7) / 8;
    double* ws = static_cast<double*>(workspace);
    const int d = cfg.grid.ndim;
    for (int o = 0; o < SLB_MAX_OUT; ++o) a.gpack[o] = nullptr;
    for (int o = 0; o < cfg.gp.num_outputs; ++o) {
        const int M = cfg.gp.factors[cfg.gp.outputs[o].factor].M;
        const int npairs = (M + 7) / 8;
        const int64_t total = (int64_t)a.nrb * npairs * 64;
        bellman_pack_actions_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(
            cfg.gp, o, d, actions, n_actions, m, a.nrb, npairs, ws);
        SLB_LAUNCH_CHECK();
        a.gpack[o] = ws;
        ws += total;
    }
    return slb_dispatch_dim<1, 2>(d, "factored argmax: state dimension", [&](auto D) {
        return launch_argmax_tile<D>(st, cfg, a);
    });
}
