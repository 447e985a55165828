// gp_grad.cu -- reverse mode of slb_gp_predict (want_var = 0): the point gradient of the GP posterior
// mean and of beta * sigma, the gradient path behind training a policy against GP dynamics (the
// reference's tf.gradients through GaussianProcess / FunctionStack, functions.py:278-291, 417-458,
// 507-515, in examples/inverted_pendulum.ipynb cells 9 and 17).
//
// Units are those of the forward (gp_tile.cuh factor_epilogue): K = s^2 k(X, z) with s the GPRCached
// scale, a = L^-1 K, mean = (a . alpha + s z . m) / s = s k . gamma + z . m, var = (s^2 kdiag(z) - a . a)
// / s^2.  For output o on factor f and a point z:
//   d mean_o / dz = m_o + s sum_j gamma_o,j grad_z k_f(z, x_j)                                   (mean kernel)
//   d var_f / dz  = grad_z kdiag_f(z) - (2 / s^2) sum_i a_i (L^-1 grad_z K)_i                    (err kernel)
//   d (beta_o sqrt(var_f)) / dz = (g beta_o) / (2 sqrt(var_f)) * d var_f / dz   (torch's sqrt backward: a
//                                 zero variance gives inf * 0 = NaN, as torch does)
//
// Mean kernel: one warp per point, O(M d_in) per point and factor; the cotangents of all outputs on a
// factor are folded into one weight per training row (sum_o g_o gamma_o,j), so it costs one kernel
// gradient per row; the lanes split the rows and a butterfly adds their sums.  It writes grad_points
// (0 when grad_mean is NULL).
//
// Err kernel (only when grad_err is given): forward mode in z on the packed factor.  One CTA takes P =
// 64 / (1 + d_in) points, i.e. NC = P (1 + d_in) <= 64 right-hand sides: k and its d_in partial
// derivatives per point.  Per 256-row i-panel every thread owns one row i of L^-1 and NC fp64
// accumulators; per 128-row j-panel the CTA generates K and grad K into shared memory (read as
// broadcasts) and each thread streams its row's 8-column groups of the packed factor (slb_pack_factor:
// the 8 values of row i in k-step pair kp are 64 contiguous bytes).  The panel epilogue forms a_i^2 and
// a_i (L^-1 d_c K)_i per point, reduces them over the warp by a butterfly and over the 8 warps in warp
// order; the factor epilogue adds d (beta sigma) / dz to grad_points.  Every sum runs in a fixed order
// without atomics: two calls give bit-identical results.  No workspace, no transposed factor.
#include "common.cuh"

#include <string.h>

// gp_sweep.cu: waits for an in-flight restore of the packed factors (slb_record_factor_dependency)
int slb_wait_for_factors(cudaStream_t st);

namespace {

constexpr int MT = 128;           // threads per CTA of the mean kernel
constexpr int VT = 256;           // threads per CTA of the err kernel = rows per i-panel
constexpr int VW = VT / 32;
constexpr int JP = 128;           // rows per j-panel of the err kernel

template <int DIN>
struct ErrShape {
    static constexpr int Q = 1 + DIN;              // right-hand sides per point: k, d_1 k .. d_DIN k
    static constexpr int P = 64 / Q;               // points per CTA
    static constexpr int NC = P * Q;               // right-hand sides per CTA
    static constexpr int KS = (NC + 1) & ~1;       // row stride of the shared K panel (double2 reads)
    static constexpr size_t SMEM = ((size_t)JP * KS + P * DIN + VW * NC + NC + P * DIN) * sizeof(double);
};

// value and z-gradient of one primitive against a training row (cross form) or of its diagonal form;
// delta_c = (z_c - x_c) w_c^2, r = sqrt(r^2 + 1e-12) (slb200.h)
template <int DIN>
SLB_DEV double prim_grad(const slb_kernel_prim& P, const double* z, const double* x, bool diag, double (&dv)[DIN]) {
    const int kind = P.kind;
#pragma unroll
    for (int c = 0; c < DIN; ++c) dv[c] = 0.0;
    if (kind == SLB_K_LINEAR) {
        double v = 0.0;
#pragma unroll
        for (int c = 0; c < DIN; ++c) {
            v = fma(P.w[c] * z[c], diag ? z[c] : x[c], v);
            dv[c] = diag ? 2.0 * P.w[c] * z[c] : P.w[c] * x[c];
        }
        return v;
    }
    if (kind == SLB_K_CONSTANT) return P.variance;
    if (kind == SLB_K_WHITE) return diag ? P.variance : 0.0;
    if (diag) return P.variance;                  // stationary: constant diagonal
    double r2 = 0.0, delta[DIN];
#pragma unroll
    for (int c = 0; c < DIN; ++c) {
        const double df = (z[c] - x[c]) * P.w[c];
        r2 = fma(df, df, r2);
        delta[c] = df * P.w[c];
    }
    double v, s;                                  // grad = s * delta
    if (kind == SLB_K_RBF) {
        v = P.variance * exp(-0.5 * r2);
        s = -v;
    } else {
        const double r = sqrt(r2 + 1e-12);
        if (kind == SLB_K_MATERN12) {
            const double e = P.variance * exp(-r);
            v = e;
            s = -e / r;
        } else if (kind == SLB_K_MATERN32) {
            const double sr = 1.7320508075688772 * r;
            const double e = P.variance * exp(-sr);
            v = (1.0 + sr) * e;
            s = -3.0 * e;
        } else {
            const double sr = 2.23606797749979 * r;
            const double e = P.variance * exp(-sr);
            v = (1.0 + sr + (5.0 / 3.0) * (r * r)) * e;
            s = -(5.0 / 3.0) * (1.0 + sr) * e;
        }
    }
#pragma unroll
    for (int c = 0; c < DIN; ++c) dv[c] = s * delta[c];
    return v;
}

// sum over terms of products of primitives, with the product rule inside a term
template <int DIN>
SLB_DEV double kexpr_grad(const slb_kernel& K, const double* z, const double* x, bool diag, double (&g)[DIN]) {
    double total = 0.0, term = 1.0, gterm[DIN];
#pragma unroll
    for (int c = 0; c < DIN; ++c) { g[c] = 0.0; gterm[c] = 0.0; }
    int cur = 0;
    for (int i = 0; i < K.num_prims; ++i) {
        const slb_kernel_prim& P = K.prims[i];
        if (P.term != cur) {
            total += term;
#pragma unroll
            for (int c = 0; c < DIN; ++c) { g[c] += gterm[c]; gterm[c] = 0.0; }
            term = 1.0;
            cur = P.term;
        }
        double dv[DIN];
        const double v = prim_grad<DIN>(P, z, x, diag, dv);
#pragma unroll
        for (int c = 0; c < DIN; ++c) gterm[c] = fma(gterm[c], v, term * dv[c]);
        term *= v;
    }
    if (K.num_prims == 0) return 0.0;
#pragma unroll
    for (int c = 0; c < DIN; ++c) g[c] += gterm[c];
    return total + term;
}

// k_f(z, x_j) and its z-gradient: the plain RBF works in Xs = X / l (the factor's Xs), grad =
// -k (z / l - Xs_j) / l
template <int DIN>
SLB_DEV double cross_grad(const slb_gp_factor& F, const double* z, const double* zs, const double* xr,
                          double (&g)[DIN]) {
    if (F.kernel.num_prims > 0) return kexpr_grad<DIN>(F.kernel, z, xr, false, g);
    double r2 = 0.0;
#pragma unroll
    for (int c = 0; c < DIN; ++c) {
        const double df = zs[c] - xr[c];
        r2 = fma(df, df, r2);
    }
    const double k = F.variance * exp(-0.5 * r2);
#pragma unroll
    for (int c = 0; c < DIN; ++c) g[c] = -k * (zs[c] - xr[c]) / F.lengthscales[c];
    return k;
}

template <int DIN>
__global__ void __launch_bounds__(MT)
gp_vjp_mean_kernel(const __grid_constant__ slb_gp_stack gp, const double* __restrict__ points, int64_t n,
                   const double* __restrict__ gmean, double* __restrict__ gin) {
    // one warp per point: lane l takes training rows l, l + 32, ...; the lanes' sums are combined by a
    // butterfly (a fixed order)
    const int64_t p = (int64_t)blockIdx.x * (MT / 32) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (p >= n) return;
    const int D = gp.num_outputs;
    double z[DIN], g[DIN];
#pragma unroll
    for (int c = 0; c < DIN; ++c) { z[c] = points[p * DIN + c]; g[c] = 0.0; }
    if (gmean != nullptr) {
        for (int f = 0; f < gp.num_factors; ++f) {
            const slb_gp_factor& F = gp.factors[f];
            const bool plain = F.kernel.num_prims == 0;
            double zs[DIN], acc[DIN];
#pragma unroll
            for (int c = 0; c < DIN; ++c) { zs[c] = plain ? z[c] / F.lengthscales[c] : z[c]; acc[c] = 0.0; }
            double go[SLB_MAX_OUT];
            for (int o = 0; o < D; ++o) go[o] = gp.outputs[o].factor == f ? gmean[p * D + o] : 0.0;
            for (int j = lane; j < F.M; j += 32) {
                double w = 0.0;
                for (int o = 0; o < D; ++o)
                    if (gp.outputs[o].factor == f) w = fma(go[o], __ldg(gp.outputs[o].gamma + j), w);
                double dk[DIN];
                cross_grad<DIN>(F, z, zs, F.Xs + (size_t)j * DIN, dk);
#pragma unroll
                for (int c = 0; c < DIN; ++c) acc[c] = fma(w, dk[c], acc[c]);
            }
#pragma unroll
            for (int c = 0; c < DIN; ++c)
#pragma unroll
                for (int s = 16; s > 0; s >>= 1) acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], s);
            const double s2 = F.scale * F.scale;
#pragma unroll
            for (int c = 0; c < DIN; ++c) g[c] += s2 * acc[c] / F.scale;
        }
        for (int o = 0; o < D; ++o) {
            const double* m = gp.outputs[o].prior_mean;
            if (m == nullptr) continue;
            const double go = gmean[p * D + o];
#pragma unroll
            for (int c = 0; c < DIN; ++c) g[c] = fma(go, m[c], g[c]);
        }
    }
    if (lane < DIN) {
        double v = g[0];
#pragma unroll
        for (int c = 1; c < DIN; ++c) if (lane == c) v = g[c];
        gin[p * DIN + lane] = v;
    }
}

template <int DIN>
__global__ void __launch_bounds__(VT, 1)
gp_vjp_err_kernel(const __grid_constant__ slb_gp_stack gp, const double* __restrict__ points, int64_t n,
                  const double* __restrict__ gerr, double* __restrict__ gin) {
    using S = ErrShape<DIN>;
    constexpr int Q = S::Q, P = S::P, NC = S::NC, KS = S::KS;
    extern __shared__ __align__(16) double smem[];
    double* Kd = smem;                    // [JP][KS]: s^2 k and s^2 d_c k of row j0 + jj, column p Q + q
    double* zt = Kd + JP * KS;            // [P][DIN] the tile's points
    double* red = zt + P * DIN;           // [VW][NC] per-warp panel sums
    double* tot = red + VW * NC;          // [NC] sum_i a_i^2 (q = 0), sum_i a_i (L^-1 d_q K)_i
    double* gacc = tot + NC;              // [P][DIN] d (beta sigma) / dz summed over outputs
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t p0 = (int64_t)blockIdx.x * P;
    const int np = (int)min((int64_t)P, n - p0);
    const int D = gp.num_outputs;
    if (tid < P * DIN) {
        const int p = tid / DIN, c = tid % DIN;
        zt[tid] = points[(p0 + min(p, np - 1)) * DIN + c];
        gacc[tid] = 0.0;
    }
    for (int i = tid; i < JP * KS; i += VT) Kd[i] = 0.0;    // the padding column stays 0
    __syncthreads();

    for (int f = 0; f < gp.num_factors; ++f) {
        const slb_gp_factor& F = gp.factors[f];
        const int M = F.M;
        const bool plain = F.kernel.num_prims == 0;
        const double s2 = F.scale * F.scale;
        const double* __restrict__ W = F.Wpack;
        if (tid < NC) tot[tid] = 0.0;
        for (int i0 = 0; i0 < M; i0 += VT) {
            double acc[KS];
#pragma unroll
            for (int c = 0; c < KS; ++c) acc[c] = 0.0;
            const int i = i0 + tid;
            const int wlast = min(i0 + 32 * warp + 31, M - 1);      // last live row of this warp
            const int jlast = min(i0 + VT - 1, M - 1);
            for (int j0 = 0; j0 <= jlast; j0 += JP) {
                __syncthreads();                                  // readers of the previous panel are done
                // ---- generation: K and grad K of rows j0 .. j0 + JP - 1 against the P points
                for (int e = tid; e < JP * P; e += VT) {
                    const int jj = e / P, p = e - jj * P, j = j0 + jj;
                    double* dst = Kd + jj * KS + p * Q;
                    if (j < M) {
                        double z[DIN], zs[DIN], dk[DIN];
#pragma unroll
                        for (int c = 0; c < DIN; ++c) {
                            z[c] = zt[p * DIN + c];
                            zs[c] = plain ? z[c] / F.lengthscales[c] : z[c];
                        }
                        const double k = cross_grad<DIN>(F, z, zs, F.Xs + (size_t)j * DIN, dk);
                        dst[0] = s2 * k;
#pragma unroll
                        for (int c = 0; c < DIN; ++c) dst[1 + c] = s2 * dk[c];
                    } else {
#pragma unroll
                        for (int q = 0; q < Q; ++q) dst[q] = 0.0;
                    }
                }
                __syncthreads();
                // ---- contraction: acc += L^-1[i, j0 .. ] K[j0 .., :] over the columns this warp needs
                const int jend = min(JP, wlast - j0 + 1);
                const int b = i >> 3;
                const double* wrow = W + (((int64_t)b * (b + 1) / 2) * 32 + (i & 7) * 4) * 2;
                for (int jj = 0; jj < jend; jj += 8) {
                    const int kp = (j0 + jj) >> 3;
                    double w[8];
                    if (i < M && kp <= b) {
                        const double2* src = reinterpret_cast<const double2*>(wrow + (int64_t)kp * 64);
#pragma unroll
                        for (int h = 0; h < 4; ++h) {
                            const double2 t = __ldg(src + h);
                            w[2 * h] = t.x;
                            w[2 * h + 1] = t.y;
                        }
                    } else {
#pragma unroll
                        for (int u = 0; u < 8; ++u) w[u] = 0.0;
                    }
#pragma unroll
                    for (int u = 0; u < 8; ++u) {
                        // element u of the group is column 8 kp + 4 (u % 2) + u / 2 (slb_pack_factor)
                        const double2* kr = reinterpret_cast<const double2*>(Kd + (jj + 4 * (u & 1) + (u >> 1)) * KS);
#pragma unroll
                        for (int c2 = 0; c2 < KS / 2; ++c2) {
                            const double2 kv = kr[c2];
                            acc[2 * c2] = fma(w[u], kv.x, acc[2 * c2]);
                            acc[2 * c2 + 1] = fma(w[u], kv.y, acc[2 * c2 + 1]);
                        }
                    }
                }
            }
            // ---- panel epilogue: a_i^2 and a_i (L^-1 d_q K)_i, summed over the warp, then over warps
#pragma unroll
            for (int p = 0; p < P; ++p) {
                const double a = acc[p * Q];
#pragma unroll
                for (int q = 0; q < Q; ++q) {
                    double v = a * acc[p * Q + q];
#pragma unroll
                    for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
                    if (lane == 0) red[warp * NC + p * Q + q] = v;
                }
            }
            __syncthreads();
            if (tid < NC) {
                double s = 0.0;
#pragma unroll
                for (int w = 0; w < VW; ++w) s += red[w * NC + tid];
                tot[tid] += s;
            }
        }
        __syncthreads();
        // ---- factor epilogue: d (beta_o sqrt(var)) / dz for the outputs on this factor
        if (tid < np) {
            const int p = tid;
            double z[DIN], dkss[DIN];
#pragma unroll
            for (int c = 0; c < DIN; ++c) { z[c] = zt[p * DIN + c]; dkss[c] = 0.0; }
            double kss = F.kss;
            if (!plain) {
                double gd[DIN];
                kss = s2 * kexpr_grad<DIN>(F.kernel, z, z, true, gd);
#pragma unroll
                for (int c = 0; c < DIN; ++c) dkss[c] = s2 * gd[c];
            }
            const double var = (kss - tot[p * Q]) / s2;
            double dvar[DIN];
#pragma unroll
            for (int c = 0; c < DIN; ++c) dvar[c] = (dkss[c] - 2.0 * tot[p * Q + 1 + c]) / s2;
            for (int o = 0; o < D; ++o) {
                if (gp.outputs[o].factor != f) continue;
                const double coef = (gerr[(p0 + p) * D + o] * gp.outputs[o].beta) / (2.0 * sqrt(var));
#pragma unroll
                for (int c = 0; c < DIN; ++c) gacc[p * DIN + c] = fma(coef, dvar[c], gacc[p * DIN + c]);
            }
        }
        __syncthreads();
    }
    // grad_points already holds the mean kernel's result (stream order)
    if (tid < np * DIN) gin[p0 * DIN + tid] += gacc[tid];
}

int check_stack(const slb_gp_stack* gp, const char* who) {
    SLB_CHECK(gp != nullptr, "%s: null gp", who);
    if (slb_validate_gp(gp)) return 1;
    SLB_CHECK(gp->num_outputs > 0, "%s: GP stack has no outputs", who);
    return 0;
}

template <int DIN>
int launch_gp_vjp(cudaStream_t st, const slb_gp_stack& gp, const double* points, int64_t n, const double* gmean,
                  const double* gerr, double* gin) {
    constexpr int PPB = MT / 32;          // points per block of the mean kernel
    SLB_CHECK((n + PPB - 1) / PPB <= 0x7fffffff, "slb_gp_vjp: too many points for one launch");
    gp_vjp_mean_kernel<DIN><<<(unsigned)((n + PPB - 1) / PPB), MT, 0, st>>>(gp, points, n, gmean, gin);
    SLB_LAUNCH_CHECK();
    if (gerr == nullptr) return 0;
    using S = ErrShape<DIN>;
    if (slb_wait_for_factors(st)) return 1;
    SLB_CUDA(cudaFuncSetAttribute(gp_vjp_err_kernel<DIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)S::SMEM));
    const int64_t tiles = (n + S::P - 1) / S::P;
    SLB_CHECK(tiles <= 0x7fffffff, "slb_gp_vjp: too many points for one launch");
    gp_vjp_err_kernel<DIN><<<(unsigned)tiles, VT, S::SMEM, st>>>(gp, points, n, gerr, gin);
    SLB_LAUNCH_CHECK();
    return 0;
}

}  // namespace

extern "C" int64_t slb_gp_vjp_workspace(const slb_gp_stack* gp, int64_t n) {
    if (check_stack(gp, "slb_gp_vjp_workspace")) return -1;
    if (n < 0) { slb_set_error("slb_gp_vjp_workspace: negative n (%lld)", (long long)n); return -1; }
    return 0;       // the kernels keep their partial sums on chip
}

extern "C" int slb_gp_vjp(void* stream, const slb_gp_stack* gp, const double* points_dev, int64_t n,
                          const double* grad_mean_dev, const double* grad_err_dev, double* grad_points_dev,
                          void* workspace_dev) {
    (void)workspace_dev;
    if (check_stack(gp, "slb_gp_vjp")) return 1;
    SLB_CHECK(n >= 0, "slb_gp_vjp: negative n (%lld)", (long long)n);
    SLB_CHECK(grad_mean_dev != nullptr || grad_err_dev != nullptr,
              "slb_gp_vjp: both cotangents are NULL (pass grad_mean, grad_err or both)");
    SLB_CHECK(n == 0 || (points_dev != nullptr && grad_points_dev != nullptr),
              "slb_gp_vjp: null points or grad_points");
    if (n == 0) return 0;
    for (int o = 0; o < gp->num_outputs; ++o)
        SLB_CHECK(grad_mean_dev == nullptr || gp->factors[gp->outputs[o].factor].M == 0 || gp->outputs[o].gamma,
                  "slb_gp_vjp: GP output %d: null gamma", o);
    return slb_dispatch_dim<1, 6>(gp->input_dim, "slb_gp_vjp: GP input_dim", [&](auto DIN) {
        return launch_gp_vjp<DIN>((cudaStream_t)stream, *gp, points_dev, n, grad_mean_dev, grad_err_dev,
                                  grad_points_dev);
    });
}
