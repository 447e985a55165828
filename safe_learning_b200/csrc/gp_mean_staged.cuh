// gp_mean_staged.cuh -- GP posterior mean of a FunctionStack at one query point per thread, with the
// training rows streamed through shared memory by TMA bulk copies (cp.async.bulk + mbarrier, double
// buffered, issued by one thread while the block consumes the previous slice).  Shared by the
// decision filter of the Lyapunov sweep (filter.cu: FAST = reduced-accuracy exp with a computed
// error bound) and the Bellman sweep (light.cu: FAST = false, the <= 1 ulp table exp).
//   mean_o = (sum_j k_j gamma_f[o][j] + scale m_o(z)) / scale,  gamma_f = scale^2 v L^-T alpha
// (functions.py:439-442, reinforcement_learning.py:98-99); plain RBF factors use the expanded squared
// distance k_j = exp(h_j + zs . xs_j - |zs|^2 / 2) on rows [xs_j, h_j] (slb_gp_factor.Xf).
#pragma once
#include "common.cuh"
#include "bulk_copy.cuh"
#include "exp2_tab512.cuh"

constexpr int MEAN_UNROLL = 4;         // independent exp chains per thread (rows per iteration)
constexpr double EPS_K = 1.0e-13;      // certified relative error of exp_neg_fast incl. its argument

// exp(x) for -700 < x <= 0 (+ rounding) to 3.3e-14 relative (tools/exp_neg_fast_check.c):
// x = (512 q + i) ln2/512 + r, |r| <= ln2/1024;  exp(x) = 2^q T[i] (1 + r + r^2/2 + r^3/6).
// 7 fp64 operations (exp_neg_tab: 11).  `far` is set for x <= -700 (incl. -inf): the caller drops
// the term (the value is unspecified then).  NaN arguments are excluded by the caller.
SLB_DEV double exp_neg_fast(double x, const double* __restrict__ tab, bool& far) {
    const double MAGIC = 6755399441055744.0;                           // 1.5 * 2^52
    const double t = fma(x, 738.6598609351493, MAGIC);                 // 512 / ln2
    const int n = __double2loint(t);
    const double nd = t - MAGIC;
    const double r = fma(nd, -0.0013538030870311431, x);               // ln2 / 512
    double q = fma(r, 1.0 / 6.0, 0.5);
    q = q * r;
    const double p = fma(q, r, r);                                     // e^r - 1
    const double T = tab[n & 511];
    const double v = fma(T, p, T);
    far = (unsigned)__double2hiint(x) > 0xC085E000u;                   // x < -700.0
    return __hiloint2double(__double2hiint(v) + ((n >> 9) << 20), __double2loint(v));
}

// ---- stage 1: mean, prior bound -----------------------------------------------------------------
// Staged slices: per factor the rows [c0, c0 + rows) of Xf (plain RBF: [x / l, -|x / l|^2 / 2],
// width DIN + 1; covariance expressions: the raw inputs, width DIN) and of gamma_f of every output on
// the factor.  Buffer b of slice t = t & 1; its mbarrier completes when the bytes have landed.
struct mean_pipe {
    uint64_t* bar;                     // [2]
    double* xbuf;                      // [2][C * (DIN + 1)]
    double* gbuf;                      // [2][nomax * C]
    int C, xstride, gstride;
    int t;                             // slices consumed so far
    int pf, pc0;                       // producer: factor and first row of the NEXT slice to issue
};

SLB_DEV int padded_rows(int M) { return (M + 7) & ~7; }

SLB_DEV int first_factor_with_data(const slb_gp_stack& gp, int f) {
    while (f < gp.num_factors && gp.factors[f].M == 0) ++f;
    return f;
}

SLB_DEV double f64_inf() { return __longlong_as_double(0x7ff0000000000000ll); }

// The outputs that live on factor f, their number a compile-time constant for the caller's running sums:
// fn(std::integral_constant<int, NO>, outs) with 1 <= NO <= MAXNO (a factor without outputs is skipped).
template <int MAXNO = SLB_MAX_OUT, class Fn>
SLB_DEV void for_outputs_on_factor(const slb_gp_stack& gp, int f, Fn&& fn) {
    static_assert(MAXNO <= 6, "one case per count");
    int outs[SLB_MAX_OUT];
    int no = 0;
    for (int o = 0; o < gp.num_outputs; ++o)
        if (gp.outputs[o].factor == f) outs[no++] = o;
    switch (no) {
    case 1: fn(std::integral_constant<int, 1>{}, outs); break;
    case 2: if constexpr (MAXNO >= 2) fn(std::integral_constant<int, 2>{}, outs); break;
    case 3: if constexpr (MAXNO >= 3) fn(std::integral_constant<int, 3>{}, outs); break;
    case 4: if constexpr (MAXNO >= 4) fn(std::integral_constant<int, 4>{}, outs); break;
    case 5: if constexpr (MAXNO >= 5) fn(std::integral_constant<int, 5>{}, outs); break;
    case 6: if constexpr (MAXNO >= 6) fn(std::integral_constant<int, 6>{}, outs); break;
    default: break;
    }
}

// scale * (z . prior_mean) of one output, in the operation order of functions.py:439-442
template <int DIN>
SLB_DEV double prior_mean_term(const slb_gp_factor& F, const slb_gp_output& G, const double* z) {
    if (G.prior_mean == nullptr) return 0.0;
    double mx = f64mul(z[0], G.prior_mean[0]);
#pragma unroll
    for (int c = 1; c < DIN; ++c) mx = f64add(mx, f64mul(z[c], G.prior_mean[c]));
    return f64mul(F.scale, mx);
}

// thread 0: issue the producer's next slice into buffer `b` and advance
template <int DIN>
SLB_DEV void issue_slice(const slb_gp_stack& gp, mean_pipe& P, int b) {
    if (P.pf >= gp.num_factors) return;
    const slb_gp_factor& F = gp.factors[P.pf];
    const int Mp = padded_rows(F.M);
    const int rows = min(P.C, Mp - P.pc0);
    const int W = F.kernel.num_prims > 0 ? DIN : DIN + 1;
    int no = 0;
    for (int o = 0; o < gp.num_outputs; ++o) no += gp.outputs[o].factor == P.pf;
    const unsigned xbytes = (unsigned)(rows * W * sizeof(double));
    const unsigned gbytes = (unsigned)(rows * sizeof(double));
    slb_bulk::mbar_arrive_expect_tx(P.bar + b, xbytes + no * gbytes);
    slb_bulk::copy_g2s(P.xbuf + b * P.xstride, F.Xf + (size_t)P.pc0 * W, xbytes, P.bar + b);
    int q = 0;
    for (int o = 0; o < gp.num_outputs; ++o) {
        if (gp.outputs[o].factor != P.pf) continue;
        slb_bulk::copy_g2s(P.gbuf + b * P.gstride + q * P.C, gp.outputs[o].gamma_f + P.pc0, gbytes,
                           P.bar + b);
        ++q;
    }
    P.pc0 += P.C;
    if (P.pc0 >= Mp) { P.pf = first_factor_with_data(gp, P.pf + 1); P.pc0 = 0; }
}

template <int W>
SLB_DEV void load_row(const double* __restrict__ p, double (&r)[W]) {
    if constexpr (W % 2 == 0) {
#pragma unroll
        for (int c = 0; c < W; c += 2) {
            const double2 v = *reinterpret_cast<const double2*>(p + c);
            r[c] = v.x; r[c + 1] = v.y;
        }
    } else {
#pragma unroll
        for (int c = 0; c < W; ++c) r[c] = p[c];
    }
}

// mean of one output from its finished dot product, and the bound of the mean's own error
// (functions.py:439-442): shared by the thread-per-point stage and the head stage's recomputation
template <int DIN>
SLB_DEV void mean_output_finish(const slb_gp_factor& F, const slb_gp_output& G, const double* z,
                                double dot, double zz, double kbound, bool general, double* mu,
                                double* mean_err) {
    *mu = f64add(dot, prior_mean_term<DIN>(F, G, z)) / F.scale;
    // |mean - exact| <= eps sum_i |k_i| (|L^-1|^T |alpha|)_i <= eps kbound gamma_l1: kernel
    // values to EPS_K (+ the expanded distance's rounding), the M-term sums here, in gamma
    // itself and in the a . alpha form of the full posterior each to (M + 2) 2^-53
    const double eps = (general ? 4.5e-16 : EPS_K + 4.5e-16 * (-zz + F.hmax)) + 7e-16 * (F.M + 8);
    *mean_err = eps * kbound * G.gamma_l1 / F.scale;
}

// one factor with NO outputs on it (compile-time, so the running dot products stay in registers)
template <int DIN, int NO, bool FAST>
SLB_DEV void mean_factor(const slb_gp_stack& gp, int f, const int* outs, const double* z, double* mu,
                         double* mean_err, const double* tab512, const double* tab64, mean_pipe& P) {
    const slb_gp_factor& F = gp.factors[f];
    const bool general = F.kernel.num_prims > 0;
    double zs[DIN];
    double zz = 0.0;
#pragma unroll
    for (int c = 0; c < DIN; ++c) {
        zs[c] = general ? z[c] : z[c] / F.lengthscales[c];
        zz = fma(zs[c], zs[c], zz);
    }
    zz *= -0.5;
    double dot[NO], dot2[NO];                  // two partial sums: half the loop-carried chain
#pragma unroll
    for (int q = 0; q < NO; ++q) { dot[q] = 0.0; dot2[q] = 0.0; }
    double kbound = general ? 0.0 : 1.0;       // max_i |k_i| (plain RBF: variances live in gamma_f)
    const int Mp = padded_rows(F.M);
    for (int c0 = 0; c0 < Mp; c0 += P.C) {
        const int rows = min(P.C, Mp - c0);
        const int b = P.t & 1;
        if (threadIdx.x == 0) issue_slice<DIN>(gp, P, b ^ 1);         // next slice, other buffer
        slb_bulk::mbar_wait(P.bar + b, (P.t >> 1) & 1);
        const double* __restrict__ xb = P.xbuf + b * P.xstride;
        const double* __restrict__ gb = P.gbuf + b * P.gstride;
        if (!general) {
            // k_j = exp(-|zs - xs_j|^2 / 2) = exp(h_j + zs . xs_j + zz), h_j = -|xs_j|^2 / 2 staged
            // with the row; variance and scale^2 are folded into gamma_f.  4 independent chains.
            constexpr int W = DIN + 1;
            for (int j0 = 0; j0 < rows; j0 += MEAN_UNROLL) {
                double arg[MEAN_UNROLL];
#pragma unroll
                for (int u = 0; u < MEAN_UNROLL; ++u) {
                    double row[W];
                    load_row<W>(xb + (j0 + u) * W, row);
                    double acc = row[DIN] + zz;
#pragma unroll
                    for (int c = 0; c < DIN; ++c) acc = fma(zs[c], row[c], acc);
                    arg[u] = acc;
                }
                double g[NO][MEAN_UNROLL];
#pragma unroll
                for (int q = 0; q < NO; ++q)
#pragma unroll
                    for (int u = 0; u < MEAN_UNROLL; u += 4) load_row<4>(gb + q * P.C + j0 + u, *reinterpret_cast<double(*)[4]>(&g[q][u]));
#pragma unroll
                for (int u = 0; u < MEAN_UNROLL; ++u) {
                    double k;
                    if constexpr (FAST) {
                        bool far;
                        k = exp_neg_fast(arg[u], tab512, far);
                        k = far ? 0.0 : k;
                    } else {
                        k = exp_neg_tab(arg[u], tab64);          // <= 1 ulp (Bellman sweeps)
                    }
#pragma unroll
                    for (int q = 0; q < NO; ++q) {
                        if (u & 1) dot2[q] = fma(k, g[q][u], dot2[q]);
                        else dot[q] = fma(k, g[q][u], dot[q]);
                    }
                }
            }
        } else {
            for (int j0 = 0; j0 < rows; j0 += 4) {
                const double* xr[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) xr[u] = xb + (j0 + u) * DIN;
                double kv[4];
                kernel_expr_cross_n<DIN, 4>(F.kernel, zs, xr, tab64, kv);
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    kbound = fmax(kbound, fabs(kv[u]));
#pragma unroll
                    for (int q = 0; q < NO; ++q) dot[q] = fma(kv[u], gb[q * P.C + j0 + u], dot[q]);
                }
            }
        }
        __syncthreads();                       // every thread is done with buffer b
        ++P.t;
    }
#pragma unroll
    for (int q = 0; q < NO; ++q)
        mean_output_finish<DIN>(F, gp.outputs[outs[q]], z, dot[q] + dot2[q], zz, kbound, general,
                                &mu[outs[q]], &mean_err[outs[q]]);
}

// thread 0 of the block: barriers of the pipeline + the bulk copy of the exp tables (bar[2]; none for a
// carve-up without tables: tab512 == nullptr); call once per kernel, before the first __syncthreads
SLB_DEV void mean_pipe_init(mean_pipe& P, double* tab512) {
    slb_bulk::mbar_init(P.bar + 0, 1);
    slb_bulk::mbar_init(P.bar + 1, 1);
    if (tab512 != nullptr) slb_bulk::mbar_init(P.bar + 2, 1);
    slb_bulk::fence_barrier_init();
    slb_bulk::fence_proxy_async();
    if (tab512 == nullptr) return;
    slb_bulk::mbar_arrive_expect_tx(P.bar + 2, 576 * sizeof(double));
    slb_bulk::copy_g2s(tab512, g_exp_tables, 576 * sizeof(double), P.bar + 2);
}

// start one evaluation of the stack's means: the producer goes back to the first factor and the
// first slice is issued into the buffer the consumer will look at next (free: its last reader
// passed a block barrier).  Called by every thread, before gp_mean_staged.
template <int DIN>
SLB_DEV void mean_pipe_start(const slb_gp_stack& gp, mean_pipe& P) {
    P.pf = first_factor_with_data(gp, 0);
    P.pc0 = 0;
    if (threadIdx.x == 0) issue_slice<DIN>(gp, P, P.t & 1);
}

// means of every output of the stack at z (all threads of the block take part in the barriers)
template <int DIN, bool FAST>
SLB_DEV void gp_mean_staged(const slb_gp_stack& gp, const double* z, double* mu, double* mean_err,
                            const double* tab512, const double* tab64, mean_pipe& P) {
    for (int f = 0; f < gp.num_factors; ++f)
        for_outputs_on_factor(gp, f, [&](auto no, const int* outs) {
            mean_factor<DIN, decltype(no)::value, FAST>(gp, f, outs, z, mu, mean_err, tab512, tab64, P);
        });
}

// shared-memory carve-up of the mean stage: [0, 32) mbarriers (2 slices, 1 exp tables), then the two
// exp tables (512 + 64 doubles; left out when tab512 == nullptr: the fp32 screening kernel needs none),
// the slice ring of the inputs and of the gammas.  Returns the first double behind the ring.
SLB_DEV double* mean_pipe_setup(mean_pipe& P, unsigned char* smem_raw, int din, int chunk_rows, int nomax,
                                const slb_gp_stack& gp, double** tab512, double** tab64) {
    P.bar = reinterpret_cast<uint64_t*>(smem_raw);
    P.xbuf = reinterpret_cast<double*>(smem_raw + 32);
    if (tab512 != nullptr) {
        *tab512 = P.xbuf;
        *tab64 = *tab512 + 512;
        P.xbuf = *tab64 + 64;
    }
    P.C = chunk_rows;
    P.xstride = P.C * (din + 1);
    P.gstride = P.C * nomax;
    P.gbuf = P.xbuf + 2 * P.xstride;
    P.t = 0;
    P.pf = first_factor_with_data(gp, 0);
    P.pc0 = 0;
    return P.gbuf + 2 * P.gstride;
}

// rows per staged slice and dynamic shared memory of a kernel built on the pipeline (host)
inline int mean_chunk_rows(int din, int nomax, int budget_kb) {
    const int rows = (budget_kb * 1024) / (2 * 8 * (din + 1 + nomax));
    return rows >= 256 ? 256 : (rows & ~7);
}
inline size_t mean_smem_bytes(int din, int nomax, int chunk_rows, bool exp_tables = true) {
    return 32 + (exp_tables ? (512 + 64) * sizeof(double) : 0) +
           (size_t)2 * chunk_rows * (din + 1 + nomax) * sizeof(double);
}

// ---- fp32 screening mean (filter.cu, filter_mean32_kernel) ---------------------------------------
// The decision filter only needs the mean to within a bound it can certify, and at 12 fp64
// operations per kernel value the fp64 mean stage is the largest part of a sweep.  Here the same
// slices are converted, once per CTA, to fp32 rows CENTERED on a point of the CTA,
//     xc_j = (xs_j - cs) s,  zc = (zs - cs) s,  s^2 = log2 e   (differences taken in fp64),
// so that k_j = 2^(-|xc_j|^2/2 + zc . xc_j) 2^(-|zc|^2/2): three FFMA and one MUFU.EX2 per kernel
// value, the last factor (E) applied once per point in fp64.  Error of the computed mean, with
// u = 2^-24, Z = |zc|^2 / 2, t_j = |zc - xc_j|^2 / 2 (so k_j = 2^-t_j):
//   argument: h_j rounds once, each of the DIN products carries two input roundings, each FFMA
//     rounds once: |arg error| <= u (DIN + 2.01) (|h_j| + sum_c |zc_c xc_jc|) <= u (DIN + 2.01)
//     (2 |h_j| + Z) <= u (DIN + 2.01) (4 t_j + 5 Z)      [|h_j| <= 2 t_j + 2 Z];
//   2^x: ex2.approx.ftz.f32 to 2^-22 (PTX ISA), budgeted 8 u; gamma rounds to fp32: u;
//   sums: F32_FLUSH terms per fp32 accumulator, then added into an fp64 sum: F32_FLUSH u;
//   with k_j t_j <= 1 / (e ln 2) = 0.531 and k_j <= 1:
//   |mean error| <= u [0.7 (DIN + 2.01) (2.13 + 5 Z) + 8 + 1 + F32_FLUSH + 2 + (8 + 0.7 Z)] sum_j |gamma_j| / scale
// (the last bracket: E = 2^-Z also comes from ex2.approx, its argument rounded to fp32)
// (0.7 > ln 2 turns the argument error into a relative error of 2^x; the last 2 covers the fp64
// steps and the terms flushed to zero).  sum_j |gamma_j| is accumulated by the CTA while it
// converts.  Points with Z > 40 (2^Z would leave the fp32 range) are left to the fp64 stages.
constexpr int F32_FLUSH = 16;

template <int DIN>
struct row32 { static constexpr int W = DIN + 1 <= 2 ? 2 : (DIN + 1 <= 4 ? 4 : 8); };

SLB_DEV float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

template <int W32>
SLB_DEV void load_row32(const float* __restrict__ p, float (&r)[W32]) {
    if constexpr (W32 == 2) {
        const float2 v = *reinterpret_cast<const float2*>(p);
        r[0] = v.x; r[1] = v.y;
    } else {
#pragma unroll
        for (int c = 0; c < W32; c += 4) {
            const float4 v = *reinterpret_cast<const float4*>(p + c);
            r[c] = v.x; r[c + 1] = v.y; r[c + 2] = v.z; r[c + 3] = v.w;
        }
    }
}

// fp32 landing of the current slice, and the block's scratch for sum |gamma|
struct mean32_bufs {
    float* xf;                         // [C][row32<DIN>::W]
    float* g;                          // [nomax][C]
    double* red;                       // [SLB_MAX_OUT][warps per CTA]
};

// One plain-RBF factor with NO outputs: mu (fp32-screened) and dmu, the certified bound of its error.
// `zcen`: the CTA's centre in input units (the same for every thread).  `ok` is cleared when the
// point is out of the fp32 range of the scheme.
template <int DIN, int NO>
SLB_DEV void mean32_factor(const slb_gp_stack& gp, int f, const int* outs, const double* z,
                           const double* zcen, double* mu, double* dmu, bool& ok, mean_pipe& P,
                           const mean32_bufs& B) {
    const slb_gp_factor& F = gp.factors[f];
    constexpr int W = DIN + 1, W32 = row32<DIN>::W;
    const double S = 1.2011224087864498;           // sqrt(log2 e)
    // per CTA and factor: the centre in the factor's units and S / lengthscale (one division per
    // dimension for the whole block instead of two per thread)
    __syncthreads();                           // B.red of the previous factor has been read
    if (threadIdx.x < DIN) {
        B.red[threadIdx.x] = zcen[threadIdx.x] / F.lengthscales[threadIdx.x];
        B.red[DIN + threadIdx.x] = S / F.lengthscales[threadIdx.x];
    }
    __syncthreads();
    double cs[DIN];
    float zc[DIN];
    double Z = 0.0;
#pragma unroll
    for (int c = 0; c < DIN; ++c) {
        cs[c] = B.red[c];
        // (z - centre) S / l: within 3e-16 relative of (z / l - cs) S, and the 1e-16 |cs| the rounded
        // centre is off by stays below 1e-12 for the magnitudes admitted here -- four orders under u
        const double zcd = (z[c] - zcen[c]) * B.red[DIN + c];
        zc[c] = (float)zcd;
        Z = fma(zcd, zcd, Z);
        if (!(fabs(cs[c]) < 1e4) || !(fabs(zcd) < 1e4)) ok = false;
    }
    Z *= 0.5;
    __syncthreads();                           // B.red is reused for sum |gamma| below
    float acc[NO][4];
    double dot[NO], g1[NO];
#pragma unroll
    for (int q = 0; q < NO; ++q) {
        dot[q] = 0.0; g1[q] = 0.0;
#pragma unroll
        for (int u = 0; u < 4; ++u) acc[q][u] = 0.0f;
    }
    const int Mp = padded_rows(F.M);
    for (int c0 = 0; c0 < Mp; c0 += P.C) {
        const int rows = min(P.C, Mp - c0);
        const int b = P.t & 1;
        if (threadIdx.x == 0) issue_slice<DIN>(gp, P, b ^ 1);         // next slice, other buffer
        slb_bulk::mbar_wait(P.bar + b, (P.t >> 1) & 1);
        const double* __restrict__ xb = P.xbuf + b * P.xstride;
        const double* __restrict__ gb = P.gbuf + b * P.gstride;
        // ---- convert the slice: centred fp32 rows [xc, -|xc|^2 / 2], fp32 gammas
        for (int r = threadIdx.x; r < rows; r += blockDim.x) {
            double row[W];
            load_row<W>(xb + r * W, row);
            float o[W32];
            double hh = 0.0;
#pragma unroll
            for (int c = 0; c < DIN; ++c) {
                const double xcd = (row[c] - cs[c]) * S;
                o[c] = (float)xcd;
                hh = fma(xcd, xcd, hh);
            }
            o[DIN] = (float)(-0.5 * hh);
#pragma unroll
            for (int c = DIN + 1; c < W32; ++c) o[c] = 0.0f;
            float* dst = B.xf + r * W32;
            if constexpr (W32 == 2) {
                *reinterpret_cast<float2*>(dst) = make_float2(o[0], o[1]);
            } else {
#pragma unroll
                for (int c = 0; c < W32; c += 4)
                    *reinterpret_cast<float4*>(dst + c) = make_float4(o[c], o[c + 1], o[c + 2], o[c + 3]);
            }
#pragma unroll
            for (int q = 0; q < NO; ++q) {
                const double gq = gb[q * P.C + r];
                B.g[q * P.C + r] = (float)gq;
                g1[q] += fabs(gq);
            }
        }
        __syncthreads();                       // fp32 slice complete
        // ---- kernel values and dot products: 4 independent chains, fp32 sums flushed into fp64
        const float* __restrict__ xf = B.xf;
        const float* __restrict__ gf = B.g;
        for (int jb = 0; jb < rows; jb += 4 * F32_FLUSH) {
            const int jend = min(jb + 4 * F32_FLUSH, rows);
            for (int j0 = jb; j0 < jend; j0 += 4) {
                float k[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    float row[W32];
                    load_row32<W32>(xf + (j0 + u) * W32, row);
                    float arg = row[DIN];
#pragma unroll
                    for (int c = 0; c < DIN; ++c) arg = fmaf(zc[c], row[c], arg);
                    k[u] = ex2_approx(arg);
                }
#pragma unroll
                for (int q = 0; q < NO; ++q) {
                    const float4 g = *reinterpret_cast<const float4*>(gf + q * P.C + j0);
                    acc[q][0] = fmaf(k[0], g.x, acc[q][0]);
                    acc[q][1] = fmaf(k[1], g.y, acc[q][1]);
                    acc[q][2] = fmaf(k[2], g.z, acc[q][2]);
                    acc[q][3] = fmaf(k[3], g.w, acc[q][3]);
                }
            }
#pragma unroll
            for (int q = 0; q < NO; ++q) {
                dot[q] += ((double)acc[q][0] + (double)acc[q][1]) + ((double)acc[q][2] + (double)acc[q][3]);
#pragma unroll
                for (int u = 0; u < 4; ++u) acc[q][u] = 0.0f;
            }
        }
        __syncthreads();                       // every thread is done with the fp32 slice and buffer b
        ++P.t;
    }
    // ---- sum_j |gamma_j| over the block (every thread converted a disjoint set of rows)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
    for (int q = 0; q < NO; ++q) {
        double v = g1[q];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
        if (lane == 0) B.red[q * nw + warp] = v;
    }
    __syncthreads();
    // E = 2^-Z on the SFU as well: relative error 2^-22 + ln2 u Z (the argument rounded to fp32)
    const double E = (double)ex2_approx(-(float)Z);
    const double u24 = 5.9604644775390625e-8;
    const double epsrel = u24 * (0.7 * (DIN + 2.01) * (2.13 + 5.0 * Z) + 11.0 + F32_FLUSH + 8.0 + 0.7 * Z);
    if (!(Z <= 40.0)) ok = false;
#pragma unroll
    for (int q = 0; q < NO; ++q) {
        double gsum = 0.0;
        for (int w = 0; w < nw; ++w) gsum += B.red[q * nw + w];
        const slb_gp_output& G = gp.outputs[outs[q]];
        mu[outs[q]] = f64add(E * dot[q], prior_mean_term<DIN>(F, G, z)) / F.scale;
        // + the products that left the fp32 range downwards (each < 2^-126 in the scaled sum)
        dmu[outs[q]] = (1.05 * epsrel * gsum + 1.3e-26 * Mp) / fabs(F.scale) + 1e-300;
    }
}

template <int DIN>
SLB_DEV void gp_mean32_staged(const slb_gp_stack& gp, const double* z, const double* zcen, double* mu,
                              double* dmu, bool& ok, mean_pipe& P, const mean32_bufs& B) {
    for (int f = 0; f < gp.num_factors; ++f)
        for_outputs_on_factor(gp, f, [&](auto no, const int* outs) {
            mean32_factor<DIN, decltype(no)::value>(gp, f, outs, z, zcen, mu, dmu, ok, P, B);
        });
}

// The fp32 screening kernel's buffers behind the pipeline's carve-up (no exp tables): the block scratch,
// then the fp32 slice.  Device layout and host size, side by side.
template <int DIN>
SLB_DEV void mean32_bufs_setup(mean32_bufs& B, double* behind_pipe, int chunk_rows, int warps) {
    B.red = behind_pipe;
    B.xf = reinterpret_cast<float*>(B.red + 8 * warps + 8);
    B.g = B.xf + chunk_rows * row32<DIN>::W;
}
inline size_t mean32_smem_bytes(int din, int nomax, int chunk_rows, int warps) {
    const int w32 = din + 1 <= 2 ? 2 : (din + 1 <= 4 ? 4 : 8);
    return mean_smem_bytes(din, nomax, chunk_rows, false) + (size_t)(8 * warps + 8) * sizeof(double) +
           (size_t)chunk_rows * (w32 + nomax) * sizeof(float);
}
