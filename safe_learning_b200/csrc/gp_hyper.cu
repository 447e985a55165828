// gp_hyper.cu -- gradient of the GP log marginal likelihood with respect to every slot of a covariance
// expression (slb_kernel), the device half of GPRCached.log_likelihood_and_gradient / optimize (gpflow 0.4.0
// GPR.build_likelihood).  With K = kern.K(X) + noise I, k target columns D = Y - m(X) [M, k],
// alpha = K^-1 D [M, k] and W = sum_c alpha_c alpha_c^T - k K^-1:
//   d LML / d theta = 1/2 sum_ij W_ij d K_ij / d theta,     d LML / d noise = 1/2 tr W.
// K^-1 and alpha come from the host's Cholesky (torch / cuSOLVER); this file reads K^-1 once, whatever k is.
//
// Tile kernel: one CTA per SLB_GP_HYPER_TILE x SLB_GP_HYPER_TILE tile (bi, bj), bi >= bj, of the lower
// triangle.  It stages the k alpha columns of its row and column panels, and per pair forms
// w = -k Kinv_ij, then w = fma(alpha_ic, alpha_jc, w) for c = 0 .. k-1 in that order.  k = 1 is its own
// instantiation (COLS = false) with the one-column arithmetic fma(alpha_i, alpha_j, -Kinv_ij) and one
// staged column: the same value as the loop's (-1 * x is -x), without its runtime trip count.  Thread t owns
// column t % HT of the tile and every (HTHREADS / HT)-th row, so a warp reads 32 consecutive doubles of a K^-1
// row.  Per pair (i >= j) it evaluates every primitive's value and what its
// partials need, forms each primitive's co-factor (the product of the other primitives of its term, by
// prefix and suffix products: no division, a zero variance is fine), and adds
//   c_ij * cofactor_p * d k_p / d slot   (c_ij = W_ij off the diagonal, which stands for (i, j) and (j, i);
//                                          c_ii = W_ii / 2)
// to per-slot accumulators in registers.  The CTA reduces them in a fixed order (butterfly within each warp,
// then the warps in order) and writes one partial per slot and tile to the workspace, slot-major.
// Sum kernel: one CTA per slot adds that slot's tile partials in a fixed order (strided per thread, then a
// shared-memory tree).  No atomics, no M x M x slots intermediate: two calls are bit-identical.
//
// The primitive arithmetic is written out here rather than taken from common.cuh: the forms there evaluate
// k through the shared-memory exp table with the variance folded in, and gp_grad.cu's differentiate in z.
#include "common.cuh"

namespace {

constexpr int HT = SLB_GP_HYPER_TILE;
constexpr int HTHREADS = 128;                 // threads per tile CTA: HT / (HTHREADS / HT) = 32 rows each
constexpr int HWARPS = HTHREADS / 32;
constexpr int PSTRIDE = 1 + SLB_MAX_IN;       // slots per primitive: variance, w[0 .. SLB_MAX_IN)
constexpr int NSLOT = SLB_GP_HYPER_SLOTS;     // ... and the noise last
constexpr int RT = 256;                       // threads of the sum kernel
static_assert(HTHREADS % HT == 0, "a tile column per thread");

// Value of primitive P on the pair (x, y) of K(X) (diag: i == j), and what its partials need:
//   base = d k / d variance (0 for LINEAR, whose variance slot is not a parameter),
//   g    = (d k / d r) / r for the stationary kinds, so that d k / d w_c = g w_c (x_c - y_c)^2
//          (r^2 = sum_c ((x_c - y_c) w_c)^2, Matern r = sqrt(r^2 + 1e-12) as gpflow);
//   LINEAR: d k / d w_c = x_c y_c.
template <int DIN>
SLB_DEV double prim_value(const slb_kernel_prim& P, const double* x, const double* y, bool diag, double& base,
                          double& g) {
    const int kind = P.kind;
    g = 0.0;
    if (kind == SLB_K_LINEAR) {
        double v = 0.0;
#pragma unroll
        for (int c = 0; c < DIN; ++c) v = fma(P.w[c] * x[c], y[c], v);
        base = 0.0;
        return v;
    }
    if (kind == SLB_K_CONSTANT) {
        base = 1.0;
        return P.variance;
    }
    if (kind == SLB_K_WHITE) {                   // K(X): variance * I, by index, not by equal inputs
        base = diag ? 1.0 : 0.0;
        return diag ? P.variance : 0.0;
    }
    double r2 = 0.0;
#pragma unroll
    for (int c = 0; c < DIN; ++c) {
        const double df = (x[c] - y[c]) * P.w[c];
        r2 = fma(df, df, r2);
    }
    if (kind == SLB_K_RBF) {
        const double e = exp(-0.5 * r2);
        base = e;
        g = -P.variance * e;
    } else {
        const double r = sqrt(r2 + 1e-12);
        if (kind == SLB_K_MATERN12) {
            const double e = exp(-r);
            base = e;
            g = -P.variance * e / r;
        } else if (kind == SLB_K_MATERN32) {
            const double sr = 1.7320508075688772 * r;
            const double e = exp(-sr);
            base = (1.0 + sr) * e;
            g = -3.0 * P.variance * e;
        } else {
            const double sr = 2.23606797749979 * r;
            const double e = exp(-sr);
            base = (1.0 + sr + (5.0 / 3.0) * (r * r)) * e;
            g = -(5.0 / 3.0) * P.variance * (1.0 + sr) * e;
        }
    }
    return P.variance * base;
}

// tile t of the lower triangle in row order: t = bi (bi + 1) / 2 + bj, bj <= bi
SLB_DEV void tile_coords(int64_t t, int& bi, int& bj) {
    int b = (int)((sqrt(8.0 * (double)t + 1.0) - 1.0) * 0.5);
    while ((int64_t)b * (b + 1) / 2 > t) --b;
    while ((int64_t)(b + 1) * (b + 2) / 2 <= t) ++b;
    bi = b;
    bj = (int)(t - (int64_t)b * (b + 1) / 2);
}

template <int DIN, bool COLS>
__global__ void __launch_bounds__(HTHREADS, 2)
gp_lml_grad_tile_kernel(const __grid_constant__ slb_kernel K, const double* __restrict__ X, int M,
                        const double* __restrict__ Kinv, const double* __restrict__ alpha, int kcols,
                        double* __restrict__ part) {
    constexpr int S = 1 + DIN;
    constexpr int NP = SLB_MAX_KPRIM;
    constexpr int KMAX = COLS ? SLB_MAX_OUT : 1;
    const int kc = COLS ? kcols : 1;
    __shared__ double xr[HT * DIN], xc[HT * DIN], ar[HT * KMAX], ac[HT * KMAX];
    __shared__ double red[HWARPS][NSLOT];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t t = blockIdx.x;
    int bi, bj;
    tile_coords(t, bi, bj);
    const int r0 = bi * HT, c0 = bj * HT;
    for (int e = tid; e < HT * DIN; e += HTHREADS) {
        const int k = e / DIN;
        xr[e] = r0 + k < M ? X[(int64_t)r0 * DIN + e] : 0.0;
        xc[e] = c0 + k < M ? X[(int64_t)c0 * DIN + e] : 0.0;
    }
    for (int e = tid; e < HT * kc; e += HTHREADS) {       // alpha is [M, kc] row-major
        const int k = e / kc;
        ar[e] = r0 + k < M ? alpha[(int64_t)r0 * kc + e] : 0.0;
        ac[e] = c0 + k < M ? alpha[(int64_t)c0 * kc + e] : 0.0;
    }
    __syncthreads();

    const int np = K.num_prims;
    double acc[NP][S], accn = 0.0;
#pragma unroll
    for (int p = 0; p < NP; ++p)
#pragma unroll
        for (int s = 0; s < S; ++s) acc[p][s] = 0.0;
    const int jj = tid % HT, j = c0 + jj;
    double y[DIN];
#pragma unroll
    for (int c = 0; c < DIN; ++c) y[c] = xc[jj * DIN + c];
    for (int ii = tid / HT; ii < HT; ii += HTHREADS / HT) {
        const int i = r0 + ii;
        if (i >= M || j >= M || j > i) continue;          // j > i only in a diagonal tile
        const bool diag = i == j;
        double wij;
        if constexpr (COLS) {
            wij = -(double)kc * __ldg(Kinv + (int64_t)i * M + j);
            for (int c = 0; c < kc; ++c) wij = fma(ar[ii * kc + c], ac[jj * kc + c], wij);
        } else {
            wij = fma(ar[ii], ac[jj], -__ldg(Kinv + (int64_t)i * M + j));
        }
        const double cij = diag ? 0.5 * wij : wij;
        if (diag) accn += cij;
        double x[DIN];
#pragma unroll
        for (int c = 0; c < DIN; ++c) x[c] = xr[ii * DIN + c];
        double v[NP], base[NP], g[NP], co[NP];
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            v[p] = 1.0;
            base[p] = g[p] = 0.0;
            if (p < np) v[p] = prim_value<DIN>(K.prims[p], x, y, diag, base[p], g[p]);
        }
        // co-factors: the product of the other primitives of the same term
        double run = 1.0;
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            if (p > 0 && p < np && K.prims[p].term != K.prims[p - 1].term) run = 1.0;
            co[p] = run;
            run *= v[p];
        }
        run = 1.0;
#pragma unroll
        for (int p = NP - 1; p >= 0; --p) {
            if (p + 1 < np && K.prims[p + 1].term != K.prims[p].term) run = 1.0;
            co[p] *= run;
            run *= v[p];
        }
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            if (p >= np) break;
            const slb_kernel_prim& P = K.prims[p];
            const double cf = cij * co[p];
            acc[p][0] = fma(cf, base[p], acc[p][0]);
            if (P.kind == SLB_K_LINEAR) {
#pragma unroll
                for (int c = 0; c < DIN; ++c) acc[p][1 + c] = fma(cf, x[c] * y[c], acc[p][1 + c]);
            } else if (P.kind != SLB_K_CONSTANT && P.kind != SLB_K_WHITE) {
                const double cg = cf * g[p];
#pragma unroll
                for (int c = 0; c < DIN; ++c) {
                    const double d = x[c] - y[c];
                    acc[p][1 + c] = fma(cg * P.w[c], d * d, acc[p][1 + c]);
                }
            }
        }
    }

    // fixed-order reduction: butterfly within each warp, then the warps in order
#pragma unroll
    for (int p = 0; p < NP; ++p) {
        if (p >= np) break;
#pragma unroll
        for (int s = 0; s < S; ++s) {
            double a = acc[p][s];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
            if (lane == 0) red[warp][p * PSTRIDE + s] = a;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) accn += __shfl_xor_sync(0xffffffffu, accn, o);
    if (lane == 0) red[warp][NSLOT - 1] = accn;
    __syncthreads();
    for (int s = tid; s < NSLOT; s += HTHREADS) {
        const int p = s / PSTRIDE, q = s - p * PSTRIDE;
        double sum = 0.0;
        if (s == NSLOT - 1 || (p < np && q < S)) {
#pragma unroll
            for (int w = 0; w < HWARPS; ++w) sum += red[w][s];
        }
        part[(int64_t)s * gridDim.x + t] = sum;
    }
}

__global__ void __launch_bounds__(RT)
gp_lml_grad_sum_kernel(const double* __restrict__ part, int64_t tiles, double* __restrict__ grad) {
    __shared__ double s[RT];
    const int tid = threadIdx.x;
    const double* src = part + (int64_t)blockIdx.x * tiles;
    double a = 0.0;
    for (int64_t t = tid; t < tiles; t += RT) a += src[t];
    s[tid] = a;
    __syncthreads();
#pragma unroll
    for (int w = RT / 2; w > 0; w >>= 1) {
        if (tid < w) s[tid] += s[tid + w];
        __syncthreads();
    }
    if (tid == 0) grad[blockIdx.x] = s[0];
}

int64_t tile_count(int32_t M) {
    const int64_t nb = ((int64_t)M + HT - 1) / HT;
    return nb * (nb + 1) / 2;
}

template <int DIN>
int launch_lml_grad(cudaStream_t st, const double* X, int M, const slb_kernel& K, const double* Kinv,
                    const double* alpha, int kc, double* grad, double* part) {
    const int64_t tiles = tile_count(M);
    SLB_CHECK(tiles <= 0x7fffffff, "slb_gp_lml_grad: M = %d needs too many tiles for one launch", M);
    if (kc == 1)
        gp_lml_grad_tile_kernel<DIN, false><<<(unsigned)tiles, HTHREADS, 0, st>>>(K, X, M, Kinv, alpha, 1, part);
    else
        gp_lml_grad_tile_kernel<DIN, true><<<(unsigned)tiles, HTHREADS, 0, st>>>(K, X, M, Kinv, alpha, kc, part);
    SLB_LAUNCH_CHECK();
    gp_lml_grad_sum_kernel<<<NSLOT, RT, 0, st>>>(part, tiles, grad);
    SLB_LAUNCH_CHECK();
    return 0;
}

}  // namespace

extern "C" int64_t slb_gp_lml_grad_workspace(int32_t M) {
    if (M < 0) {
        slb_set_error("slb_gp_lml_grad_workspace: negative M (%d)", M);
        return -1;
    }
    return tile_count(M) * NSLOT * (int64_t)sizeof(double);
}

namespace {

int lml_grad(const char* who, void* stream, const double* X_dev, int32_t M, int32_t d_in, const slb_kernel* kern,
             const double* Kinv_dev, const double* alpha_dev, int32_t k, double* grad_dev, void* workspace_dev) {
    SLB_CHECK(M >= 0, "%s: negative M (%d)", who, M);
    SLB_CHECK(d_in >= 1 && d_in <= SLB_MAX_IN, "%s: d_in %d outside 1..%d", who, d_in, SLB_MAX_IN);
    SLB_CHECK(k >= 1 && k <= SLB_MAX_OUT, "%s: %d target columns outside 1..%d", who, k, SLB_MAX_OUT);
    SLB_CHECK(kern != nullptr, "%s: null kernel descriptor", who);
    if (slb_validate_kernel(*kern, d_in, who)) return 1;
    SLB_CHECK(kern->num_prims >= 1,
              "%s: the covariance expression has no primitives (num_prims = 0 is the sweeps' plain-RBF "
              "form, which this call does not take)", who);
    for (int i = 0; i < kern->num_prims; ++i)
        for (int c = d_in; c < SLB_MAX_IN; ++c)
            SLB_CHECK(kern->prims[i].w[c] == 0.0, "%s: kernel primitive %d has weight %g in column %d beyond "
                      "d_in = %d", who, i, kern->prims[i].w[c], c, d_in);
    if (M == 0) return 0;
    SLB_CHECK(X_dev != nullptr && Kinv_dev != nullptr && alpha_dev != nullptr && grad_dev != nullptr &&
              workspace_dev != nullptr, "%s: null X, Kinv, alpha, grad or workspace with M = %d", who, M);
    return slb_dispatch_dim<1, 6>(d_in, "slb_gp_lml_grad: d_in", [&](auto DIN) {
        return launch_lml_grad<DIN>((cudaStream_t)stream, X_dev, M, *kern, Kinv_dev, alpha_dev, k, grad_dev,
                                    static_cast<double*>(workspace_dev));
    });
}

}  // namespace

extern "C" int slb_gp_lml_grad_cols(void* stream, const double* X_dev, int32_t M, int32_t d_in,
                                    const slb_kernel* kern, const double* Kinv_dev, const double* alpha_dev,
                                    int32_t k, double* grad_dev, void* workspace_dev) {
    return lml_grad("slb_gp_lml_grad_cols", stream, X_dev, M, d_in, kern, Kinv_dev, alpha_dev, k, grad_dev,
                    workspace_dev);
}

extern "C" int slb_gp_lml_grad(void* stream, const double* X_dev, int32_t M, int32_t d_in, const slb_kernel* kern,
                               const double* Kinv_dev, const double* alpha_dev, double* grad_dev,
                               void* workspace_dev) {
    return lml_grad("slb_gp_lml_grad", stream, X_dev, M, d_in, kern, Kinv_dev, alpha_dev, 1, grad_dev,
                    workspace_dev);
}
