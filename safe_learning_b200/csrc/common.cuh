// common.cuh -- shared device code of libslb200: error plumbing, GridWorld coordinates,
// the fused function objects (policy / V / Lipschitz / plants / reward / Triangulation),
// the Lyapunov decision formula and the order-preserving V key.
//
// Reference citations are relative to the upstream befelix/safe_learning sources @ f1aad5a.
// Bit-parity rule: the cheap element-wise pieces use __dmul_rn/__dadd_rn (never contracted
// into FMA) in the left-to-right order that oracle/reference_path.py writes out, so grid
// coordinates, linear maps, quadratic forms and barycentric weights are bit-identical to
// the CPU oracle.  Only the GP contraction (DMMA) and libm calls (exp/sin/cos/sqrt is exact)
// differ in rounding.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#include <type_traits>

#include "../../include/slb200.h"
#include "exp2_tab64.h"

// SMs of the target GPU (H100 SXM, sm_90a): the CTA count of one full wave of the one-CTA-per-SM
// launches (head stage, persistent refine tiles, L2 prefetch of the packed factors)
constexpr int SLB_NUM_SMS = 132;

// ----------------------------------------------------------------------------- host side
void slb_set_error(const char* fmt, ...);
void slb_count_launch();

#define SLB_CHECK(cond, ...)                                                     \
    do {                                                                         \
        if (!(cond)) { slb_set_error(__VA_ARGS__); return 1; }                   \
    } while (0)

#define SLB_CUDA(call)                                                           \
    do {                                                                         \
        cudaError_t e__ = (call);                                                \
        if (e__ != cudaSuccess) {                                                \
            slb_set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), \
                          __FILE__, __LINE__);                                   \
            return 2;                                                            \
        }                                                                        \
    } while (0)

#define SLB_LAUNCH_CHECK()                                                       \
    do {                                                                         \
        slb_count_launch();                                                      \
        SLB_CUDA(cudaGetLastError());                                            \
    } while (0)

int slb_validate_function(const slb_function* f, const char* what, int expect_in /* <=0: any */);
int slb_fn_columns(const slb_function& f);
int slb_validate_dynamics(const slb_function* f, const char* who, int d, int m);
// the covariance expression's own checks (primitive count, kinds, term order, weights of the first
// d_in columns non-negative); messages start with `who`
int slb_validate_kernel(const slb_kernel& K, int d_in, const char* who);
int slb_validate_gp(const slb_gp_stack* gp);
int slb_validate_staged_tables(const slb_gp_stack* gp, const char* who);
int slb_validate_grid(const slb_grid* g, bool need_points);
int slb_validate_range(const char* who, int64_t idx_begin, int64_t idx_end, int64_t nindex);
// validates an slb_sweep descriptor (explicit_states: a sweep of a state list), *m_out = action dimension
int slb_validate_sweep(const slb_sweep* cfg, bool explicit_states, int* m_out);

// Runs the kernel instantiation of a runtime dimension d: returns launch(std::integral_constant<int,
// d>{}) for d in the compiled range [LO, HI], else the error "<what> <d> not compiled (LO..HI)".
template <int LO, int HI, class F>
int slb_dispatch_dim(int d, const char* what, F&& launch) {
    SLB_CHECK(d >= LO && d <= HI, "%s %d not compiled (%d..%d)", what, d, LO, HI);
    if constexpr (LO < HI) {
        if (d > LO) return slb_dispatch_dim<LO + 1, HI>(d, what, launch);
    }
    return launch(std::integral_constant<int, LO>{});
}

// ----------------------------------------------------------------------------- device side
#define SLB_DEV __device__ __forceinline__

SLB_DEV double f64mul(double a, double b) { return __dmul_rn(a, b); }
SLB_DEV double f64add(double a, double b) { return __dadd_rn(a, b); }
SLB_DEV double f64sub(double a, double b) { return __dsub_rn(a, b); }

// Order-preserving map double -> uint64 (ascending).  -0.0 is canonicalised to +0.0 first
// so that it ties with +0.0 like np.argsort sees it (lyapunov.py:512).
SLB_DEV uint64_t value_key(double v) {
    if (v == 0.0) v = 0.0;
    uint64_t b = (uint64_t)__double_as_longlong(v);
    return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}
SLB_DEV double key_value(uint64_t k) {
    uint64_t b = (k & 0x8000000000000000ull) ? (k & 0x7fffffffffffffffull) : ~k;
    return __longlong_as_double((long long)b);
}

// ---- first-fail key folded where the flags are decided (filter.cu, gp_tile.cuh; read by light.cu)
// The key of a sweep is the lexicographic minimum of (value_key(V), flat index) over the points that are
// neither negative nor initial, n_ok the number of those that are.  The decision kernels fold every point
// when its flag becomes final, so the record holds the key once the last of them has finished.  It is
// stored complemented -- hi = ~value_key, lo = INT64_MAX - index -- so that a zeroed record is the
// identity (no failing point) and the minimum is a 128-bit maximum.  Minimum and sum do not depend on
// the order of the updates: the result is exact and deterministic.
struct __align__(16) slb_fold {
    unsigned long long lo, hi;         // complemented key (see above)
    unsigned long long n_ok;
    unsigned int ticket;               // apply_prefix_kernel: blocks that have added their statistics
    unsigned int _pad;
    unsigned long long acc[4];         // apply_prefix_kernel: slb_prefix_stats accumulated over its blocks
};
// What a sweep folds into: V of the range (the values the prefix rule orders by), the initial safe set
// (may be null) and the record; all indexed relative to the pass like the flags.  rec == nullptr: no fold.
struct slb_fold_target {
    const double* values;
    const uint8_t* initial;
    slb_fold* rec;
};

SLB_DEV unsigned long long atom_cas128(slb_fold* p, unsigned long long lo, unsigned long long hi,
                                       unsigned long long new_lo, unsigned long long new_hi,
                                       unsigned long long* got_hi) {
    unsigned long long got_lo;
    asm volatile("{\n\t.reg .b128 d, c, s;\n\t"
                 "mov.b128 c, {%2, %3};\n\t"
                 "mov.b128 s, {%4, %5};\n\t"
                 "atom.global.cas.b128 d, [%6], c, s;\n\t"
                 "mov.b128 {%0, %1}, d;\n\t}"
                 : "=l"(got_lo), "=l"(*got_hi)
                 : "l"(lo), "l"(hi), "l"(new_lo), "l"(new_hi), "l"(p)
                 : "memory");
    return got_lo;
}

// (kv, ki) into the record: 128-bit maximum of the complemented key.  hi only grows, so a key whose hi
// is below the one already there cannot win and costs one load, not an atomic.
SLB_DEV void fold_key(slb_fold* rec, uint64_t kv, int64_t ki) {
    const unsigned long long hi = ~kv, lo = (unsigned long long)(INT64_MAX - ki);
    unsigned long long cur_hi;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(cur_hi) : "l"(&rec->hi) : "memory");
    if (hi < cur_hi) return;
    unsigned long long cur_lo = 0;
    while (hi > cur_hi || (hi == cur_hi && lo > cur_lo)) {
        unsigned long long got_hi;
        const unsigned long long got_lo = atom_cas128(rec, cur_lo, cur_hi, lo, hi, &got_hi);
        if (got_lo == cur_lo && got_hi == cur_hi) return;
        cur_lo = got_lo;
        cur_hi = got_hi;
    }
}

// A warp's points whose flags are final (warp-collective: all 32 lanes call it).  `mine`: the lane holds
// such a point, `negative` its flag, rel its index relative to the pass starting at idx_begin.  One
// n_ok add and at most one key update per warp.
SLB_DEV void fold_decided(const slb_fold_target& t, bool mine, bool negative, int64_t rel, int64_t idx_begin) {
    const bool ok = mine && (negative || (t.initial != nullptr && t.initial[rel] != 0));
    const bool fail = mine && !ok;
    const unsigned okb = __ballot_sync(0xffffffffu, ok);
    const unsigned failb = __ballot_sync(0xffffffffu, fail);
    uint64_t kv = fail ? value_key(t.values[rel]) : ~0ull;
    int64_t ki = fail ? idx_begin + rel : INT64_MAX;
    if (failb != 0) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const uint64_t ov = __shfl_xor_sync(0xffffffffu, kv, off);
            const int64_t oi = __shfl_xor_sync(0xffffffffu, ki, off);
            if (ov < kv || (ov == kv && oi < ki)) { kv = ov; ki = oi; }
        }
    }
    if ((threadIdx.x & 31) != 0) return;
    if (okb != 0) atomicAdd(&t.rec->n_ok, (unsigned long long)__popc(okb));
    if (failb != 0) fold_key(t.rec, kv, ki);
}

// Table-driven exp(x) for x <= 0 (<= 1 ulp against glibc on 2e7 points, tools/exp_neg_tab_check.c):
// x = (64 k + j) ln2/64 + r, |r| <= ln2/128;  exp(x) = 2^k * T[j] * (1 + r + ... + r^5/120).
// 10 fp64 operations; T (64 correctly rounded doubles) is read from a shared-memory
// copy because the index differs per lane (constant memory would serialise).
__constant__ double c_exp2_tab[64] = {SLB_EXP2_TAB64};

SLB_DEV void load_exp_table(double* tab_smem) {
    for (int i = threadIdx.x; i < 64; i += blockDim.x) tab_smem[i] = c_exp2_tab[i];
}

SLB_DEV double exp_neg_tab(double x, const double* __restrict__ tab) {
    const double MAGIC = 6755399441055744.0;             // 1.5 * 2^52
    const double t = fma(x, 92.33248261689366, MAGIC);                  // 64 / ln2
    const int n = __double2loint(t);
    const double nd = t - MAGIC;
    double r = fma(nd, -0.01083042469326756, x);                          // ln2/64, high part (32 bits)
    r = fma(nd, -2.9815858269852933e-12, r);                                 // ln2/64, low part
    double p = 1.0 / 120.0;
    p = fma(p, r, 1.0 / 24.0);
    p = fma(p, r, 1.0 / 6.0);
    p = fma(p, r, 0.5);
    p = fma(p, r, 1.0);
    p = p * r;                                           // e^r - 1
    const double T = tab[n & 63];
    const double v = fma(T, p, T);
    const double s = __hiloint2double(__double2hiint(v) + ((n >> 6) << 20), __double2loint(v));
    return x < -700.0 ? 0.0 : s;
}

// ---- covariance expressions (slb_kernel): sum over terms of products of gpflow primitives ------
// cross form k(z, x) against a training row (kern.K(X, Xnew), functions.py:438)
template <int DIN>
SLB_DEV double kernel_expr_cross(const slb_kernel& K, const double* z, const double* x,
                                 const double* exptab) {
    double total = 0.0, term = 1.0;
    int cur = 0;
    for (int i = 0; i < K.num_prims; ++i) {
        const slb_kernel_prim& P = K.prims[i];
        if (P.term != cur) { total += term; term = 1.0; cur = P.term; }
        double v;
        if (P.kind == SLB_K_LINEAR) {
            v = 0.0;
#pragma unroll
            for (int c = 0; c < DIN; ++c) v = fma(P.w[c] * z[c], x[c], v);
        } else if (P.kind == SLB_K_CONSTANT) {
            v = P.variance;
        } else if (P.kind == SLB_K_WHITE) {
            v = 0.0;
        } else {
            double r2 = 0.0;
#pragma unroll
            for (int c = 0; c < DIN; ++c) {
                const double df = (z[c] - x[c]) * P.w[c];
                r2 = fma(df, df, r2);
            }
            if (P.kind == SLB_K_RBF) {
                v = P.variance * exp_neg_tab(-0.5 * r2, exptab);
            } else {
                const double r = sqrt(r2 + 1e-12);
                if (P.kind == SLB_K_MATERN12) {
                    v = P.variance * exp_neg_tab(-r, exptab);
                } else if (P.kind == SLB_K_MATERN32) {
                    const double sr = 1.7320508075688772 * r;
                    v = P.variance * (1.0 + sr) * exp_neg_tab(-sr, exptab);
                } else {
                    const double sr = 2.23606797749979 * r;
                    v = P.variance * (1.0 + sr + (5.0 / 3.0) * (r * r)) * exp_neg_tab(-sr, exptab);
                }
            }
        }
        term *= v;
    }
    return K.num_prims > 0 ? total + term : 0.0;
}

// U training rows at once: the primitive loop is outermost so its parameters are fetched once per
// batch and the U exp / sqrt chains of a primitive are independent (the one-row form above runs
// one dependent chain per primitive).
template <int DIN, int U>
SLB_DEV void kernel_expr_cross_n(const slb_kernel& K, const double* z, const double* const (&x)[U],
                                 const double* exptab, double (&out)[U]) {
    double total[U], term[U];
#pragma unroll
    for (int u = 0; u < U; ++u) { total[u] = 0.0; term[u] = 1.0; }
    int cur = 0;
    for (int i = 0; i < K.num_prims; ++i) {
        const slb_kernel_prim& P = K.prims[i];
        const int kind = P.kind;
        const double var = P.variance;
        if (P.term != cur) {
#pragma unroll
            for (int u = 0; u < U; ++u) { total[u] += term[u]; term[u] = 1.0; }
            cur = P.term;
        }
        double w[DIN];
#pragma unroll
        for (int c = 0; c < DIN; ++c) w[c] = P.w[c];
        double v[U];
        if (kind == SLB_K_LINEAR) {
#pragma unroll
            for (int c = 0; c < DIN; ++c) w[c] *= z[c];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                double a = 0.0;
#pragma unroll
                for (int c = 0; c < DIN; ++c) a = fma(w[c], x[u][c], a);
                v[u] = a;
            }
        } else if (kind == SLB_K_CONSTANT || kind == SLB_K_WHITE) {
#pragma unroll
            for (int u = 0; u < U; ++u) v[u] = kind == SLB_K_CONSTANT ? var : 0.0;
        } else {
            double r2[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                double a = 0.0;
#pragma unroll
                for (int c = 0; c < DIN; ++c) {
                    const double df = (z[c] - x[u][c]) * w[c];
                    a = fma(df, df, a);
                }
                r2[u] = a;
            }
            if (kind == SLB_K_RBF) {
#pragma unroll
                for (int u = 0; u < U; ++u) v[u] = var * exp_neg_tab(-0.5 * r2[u], exptab);
            } else {
                // s = c r with c = 1, sqrt(3), sqrt(5); polynomial 1, 1 + s, 1 + s + s^2 / 3
                const double cs = kind == SLB_K_MATERN12 ? 1.0
                                : kind == SLB_K_MATERN32 ? 1.7320508075688772 : 2.23606797749979;
                const double c1 = kind == SLB_K_MATERN12 ? 0.0 : 1.0;
                const double c2 = kind == SLB_K_MATERN52 ? 1.0 / 3.0 : 0.0;
#pragma unroll
                for (int u = 0; u < U; ++u) {
                    const double sr = cs * sqrt(r2[u] + 1e-12);
                    v[u] = var * fma(fma(c2, sr, c1), sr, 1.0) * exp_neg_tab(-sr, exptab);
                }
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) term[u] *= v[u];
    }
#pragma unroll
    for (int u = 0; u < U; ++u) out[u] = K.num_prims > 0 ? total[u] + term[u] : 0.0;
}

// diagonal form k(z, z) (kern.Kdiag(Xnew), functions.py:450)
template <int DIN>
SLB_DEV double kernel_expr_diag(const slb_kernel& K, const double* z) {
    double total = 0.0, term = 1.0;
    int cur = 0;
    for (int i = 0; i < K.num_prims; ++i) {
        const slb_kernel_prim& P = K.prims[i];
        if (P.term != cur) { total += term; term = 1.0; cur = P.term; }
        double v = P.variance;
        if (P.kind == SLB_K_LINEAR) {
            v = 0.0;
#pragma unroll
            for (int c = 0; c < DIN; ++c) v = fma(P.w[c] * z[c], z[c], v);
        }
        term *= v;
    }
    return K.num_prims > 0 ? total + term : 0.0;
}

// GridWorld.index_to_state (functions.py:714-731): ijk * unit_maxes + offset, two roundings.
SLB_DEV void grid_index_to_state(const slb_grid& g, int64_t idx, double* x) {
    if (g.nindex <= 0x7fffffffll) {        // 32-bit index arithmetic (same integers, ~5x fewer instructions)
        unsigned rest = (unsigned)idx;
#pragma unroll
        for (int c = SLB_MAX_DIM - 1; c >= 0; --c) {
            if (c < g.ndim) {
                const unsigned n = (unsigned)g.num_points[c];
                const unsigned q = rest / n;
                const unsigned i = rest - q * n;
                rest = q;
                x[c] = f64add(f64mul((double)i, g.unit_maxes[c]), g.offset[c]);
            }
        }
        return;
    }
#pragma unroll
    for (int c = SLB_MAX_DIM - 1; c >= 0; --c) {
        if (c < g.ndim) {
            const int64_t n = g.num_points[c];
            const int64_t i = idx % n;
            idx /= n;
            x[c] = f64add(f64mul((double)i, g.unit_maxes[c]), g.offset[c]);
        }
    }
}

// GridWorld.state_to_index (functions.py:733-752), the nearest vertex of x: clip to [offset, upper], then
// (x - offset) * inv with inv = 1. / unit_maxes as numpy computes it (two roundings, never contracted), then
// rint (half to even, like np.rint), then ravel.  np.clip keeps a NaN where fmin / fmax would drop it; a
// row with a NaN coordinate has no vertex and gives -1 (the reference raises from ravel_multi_index).  The
// per-axis index is kept inside the grid so that a descriptor with a wrong inv cannot read out of bounds;
// with numpy's inv it never leaves it.
SLB_DEV int64_t grid_nearest_index(const slb_grid& g, const double* inv, const double* x) {
    int64_t idx = 0;
    for (int c = 0; c < g.ndim; ++c) {
        const double xc = x[c];
        if (xc != xc) return -1;
        const double cl = xc < g.offset[c] ? g.offset[c] : (xc > g.upper[c] ? g.upper[c] : xc);
        const double k = rint(f64mul(f64sub(cl, g.offset[c]), inv[c]));
        const int64_t n = g.num_points[c];
        const int64_t i = k > 0.0 ? (k < (double)(n - 1) ? (int64_t)k : n - 1) : 0;
        idx = idx * n + i;
    }
    return idx;
}

// fmod(a, b) for a >= 0, b > 0, a / b < 2^52 -- bit-identical to fmod (whose result is exact): the
// quotient from one division (it can only come out one too large, when a / b rounds up to an
// integer), the remainder by an exact fma.  CUDA's fmod is a long software loop; the Triangulation
// lookup calls it once per dimension and dominated its cost.
SLB_DEV double fmod_exact_pos(double a, double b) {
    double q = floor(a / b);
    double r = fma(-q, b, a);
    if (r < 0.0) r = fma(-(q - 1.0), b, a);
    else if (r >= b) r = fma(-(q + 1.0), b, a);
    return r;
}

// ---- Triangulation (functions.py:1103-1158 lookup, :1473-1499 evaluation) ----------------
// The one lookup of the point xin in the Triangulation f, in three forms:
//   TRI_EVAL     f(xin), or its gradient, into out (every function object inlines this form);
//   TRI_WEIGHTS  stops after the barycentric weights: out = w[0..d], *corner = the rectangle's lowest
//                vertex, *simplex = the simplex (the rows of the value operator, value_opt.cu);
//   TRI_CELL     as TRI_WEIGHTS, but searches the simplex from unit coordinates taken relative to the
//                rectangle's own lowest vertex (clipped xin - that vertex): the value operator's
//                repair of rows whose `% unit_maxes` picked a simplex on the wrong side of the cell.
// The forms differ in `if constexpr` blocks only, so that TRI_EVAL compiles to this code written out
// by itself: routing it through helper functions changed register allocation (and added spills) in
// the kernels that inline it.
enum { TRI_EVAL, TRI_WEIGHTS, TRI_CELL };

template <int FORM>
SLB_DEV void tri_lookup(const slb_function& f, const double* xin, double* out, int64_t* corner_out = nullptr,
                        int* simplex_out = nullptr) {
    const slb_grid& g = f.grid;
    const int d = g.ndim;
    const double eps = 2.220446049250313e-16;
    double unit[SLB_MAX_DIM];
    int64_t corner = 0;
    int poff = 0;
    int pattern = 0;
    bool all_clipped = true;
    for (int c = 0; c < d; ++c) {
        const double* pts = g.discrete_points + poff;
        const int n = (int)g.num_points[c];
        poff += n;
        const double xc = xin[c];
        // np.digitize(x, pts) - 1 clipped to [0, n-2]   (functions.py:771-773)
        int k = (int)floor((xc - g.offset[c]) / g.unit_maxes[c]);
        k = k < 0 ? 0 : (k > n - 1 ? n - 1 : k);
        while (k + 1 <= n - 1 && pts[k + 1] <= xc) ++k;
        while (k >= 0 && pts[k] > xc) --k;            // k = -1 when x < pts[0]
        k = k < 0 ? 0 : (k > n - 2 ? n - 2 : k);
        corner = corner * g.num_points[c] + k;        // rectangle_corner_index (:800-817)
        // _center_states(clip=True) % unit_maxes          (:691-712, :1120-1123)
        double cen = f64sub(xc, g.offset[c]);
        const double lo = 2.0 * eps;
        const double hi = f64sub(f64sub(g.upper[c], g.offset[c]), 2.0 * eps);
        if (cen < lo) cen = lo;
        else if (cen > hi) { cen = hi; pattern |= 1 << c; }
        else all_clipped = false;
        unit[c] = fmod_exact_pos(cen, g.unit_maxes[c]);
    }
    if constexpr (FORM == TRI_CELL) {
        double base[SLB_MAX_DIM];
        grid_index_to_state(g, corner, base);
        for (int c = 0; c < d; ++c) unit[c] = f64sub(fmin(fmax(xin[c], g.offset[c]), g.upper[c]), base[c]);
        all_clipped = false;
    }
    // simplex inside the unit cell: first simplex whose barycentric weights are all >= -tol
    int best = 0;
    double best_min = -1e300;
    const bool tabled = all_clipped && f.corner_simplex != nullptr;
    if (tabled) best = f.corner_simplex[pattern];
    for (int s = 0; s < f.nsimplex && !tabled; ++s) {
        const int64_t v0 = f.unit_simplices[s * (d + 1)];
        double o[SLB_MAX_DIM];
        if (g.nindex <= 0x7fffffffll) {        // 32-bit index arithmetic (same integers)
            unsigned t = (unsigned)v0;
            for (int c = d - 1; c >= 0; --c) {
                const unsigned n = (unsigned)g.num_points[c];
                const unsigned qq = t / n;
                o[c] = (double)(t - qq * n) * g.unit_maxes[c];
                t = qq;
            }
        } else {
            int64_t t = v0;
            for (int c = d - 1; c >= 0; --c) {
                o[c] = (double)(t % g.num_points[c]) * g.unit_maxes[c];
                t /= g.num_points[c];
            }
        }
        const double* H = f.hyperplanes + (size_t)s * d * d;
        double wsum = 0.0, wmin = 1e300;
        for (int c = 0; c < d; ++c) {
            double w = 0.0;
            for (int k = 0; k < d; ++k) w += (unit[k] - o[k]) * H[k * d + c];
            wsum += w;
            wmin = fmin(wmin, w);
        }
        wmin = fmin(wmin, 1.0 - wsum);
        if (wmin > best_min) { best_min = wmin; best = s; }
        if (wmin >= -1e-12) break;
    }
    // weights with the ORIGINAL (optionally projected) point   (:1479-1491)
    const int64_t* simp = f.unit_simplices + (size_t)best * (d + 1);
    const double* H = f.hyperplanes + (size_t)best * d * d;
    double origin[SLB_MAX_DIM], off[SLB_MAX_DIM];
    grid_index_to_state(g, simp[0] + corner, origin);
    for (int c = 0; c < d; ++c) {
        double xc = xin[c];
        // clip as tf.clip_by_value does: a NaN coordinate stays NaN (fmin / fmax would return the limit)
        if (f.flags & SLB_FLAG_PROJECT) xc = xc < g.offset[c] ? g.offset[c] : (xc > g.upper[c] ? g.upper[c] : xc);
        off[c] = f64sub(xc, origin[c]);
    }
    double w[SLB_MAX_DIM + 1];
    for (int c = 0; c < d; ++c) {
        double acc = f64mul(off[0], H[c]);
        for (int k = 1; k < d; ++k) acc = f64add(acc, f64mul(off[k], H[k * d + c]));
        w[c + 1] = acc;
    }
    double acc = w[1];
    for (int c = 2; c <= d; ++c) acc = f64add(acc, w[c]);
    w[0] = f64sub(1.0, acc);
    if constexpr (FORM != TRI_EVAL) {
        for (int c = 0; c <= d; ++c) out[c] = w[c];
        *corner_out = corner;
        *simplex_out = best;
        return;
    }
    if (f.flags & SLB_FLAG_GRADIENT) {
        // Triangulation.gradient (:1260-1326): weights[k][0] = -sum_c H[k][c], weights[k][1 + c] =
        // H[k][c]; d/dx_k = sum_v weights[k][v] * value[vertex v]   (one output column).  A point with
        // a NaN coordinate has no simplex, so its gradient is NaN (DESIGN.md §3.2).
        bool nan = false;
        for (int c = 0; c < d; ++c) nan = nan || xin[c] != xin[c];
        if (nan) {
            for (int k = 0; k < d; ++k) out[k] = __longlong_as_double(0x7ff8000000000000ll);
            return;
        }
        for (int k = 0; k < d; ++k) {
            double hs = H[k * d];
            for (int c = 1; c < d; ++c) hs = f64add(hs, H[k * d + c]);
            double v = f64mul(-hs, f.matrix[simp[0] + corner]);
            for (int c = 0; c < d; ++c)
                v = f64add(v, f64mul(H[k * d + c], f.matrix[simp[c + 1] + corner]));
            out[k] = v;
        }
        return;
    }
    // gather vertex values and combine  (:1494-1499)
    const int od = f.out_dim;
    for (int o = 0; o < od; ++o) {
        double v = f64mul(w[0], f.matrix[(simp[0] + corner) * od + o]);
        for (int k = 1; k <= d; ++k)
            v = f64add(v, f64mul(w[k], f.matrix[(simp[k] + corner) * od + o]));
        out[o] = v;
    }
}

// ---- plants (examples/utilities.py:242-289 pendulum, :387-437 cart-pole) -----------------
// cparams layout is written by safe_learning_b200/functions.py (InvertedPendulum/CartPole).
SLB_DEV void eval_pendulum(const slb_function& f, const double* in, double* out) {
    const double* p = f.cparams;
    const double g_l = p[0], inertia = p[1], fric_i = p[2], dt = p[3];
    const bool has_norm = p[9] != 0.0, has_fric = p[10] != 0.0;
    double th = in[0], om = in[1], u = in[2];
    if (has_norm) { th = f64mul(th, p[4]); om = f64mul(om, p[5]); u = f64mul(u, p[6]); }
    const double ui = u / inertia;
    for (int i = 0; i < 10; ++i) {
        double acc = f64add(f64mul(g_l, sin(th)), ui);
        if (has_fric) acc = f64sub(acc, f64mul(fric_i, om));
        const double th_n = f64add(th, f64mul(dt, om));
        const double om_n = f64add(om, f64mul(dt, acc));
        th = th_n; om = om_n;
    }
    if (has_norm) { th = f64mul(th, p[7]); om = f64mul(om, p[8]); }
    out[0] = th; out[1] = om;
}

SLB_DEV void eval_cartpole(const slb_function& f, const double* in, double* out) {
    const double* p = f.cparams;
    const double m = p[0], M = p[1], L = p[2], b = p[3], g = p[4], dt = p[5];
    const bool has_norm = p[15] != 0.0;
    double s[4] = {in[0], in[1], in[2], in[3]};
    double u = in[4];
    if (has_norm) { for (int c = 0; c < 4; ++c) s[c] = f64mul(s[c], p[6 + c]); u = f64mul(u, p[10]); }
    for (int i = 0; i < 10; ++i) {
        const double th = s[1], v = s[2], om = s[3];
        const double st = sin(th), ct = cos(th), s2t = sin(2.0 * th);
        const double det = L * (M + m * (st * st));
        const double v_dot = (u - m * L * (om * om) * st - b * om * ct + 0.5 * m * g * L * s2t) * L / det;
        const double om_dot = (u * ct - 0.5 * m * L * (om * om) * s2t - b * (m + M) * om / (m * L)
                               + (m + M) * g * st) / det;
        s[0] = f64add(s[0], f64mul(dt, v));
        s[1] = f64add(s[1], f64mul(dt, om));
        s[2] = f64add(s[2], f64mul(dt, v_dot));
        s[3] = f64add(s[3], f64mul(dt, om_dot));
    }
    if (has_norm) for (int c = 0; c < 4; ++c) s[c] = f64mul(s[c], p[11 + c]);
    for (int c = 0; c < 4; ++c) out[c] = s[c];
}

// reverse-time Van der Pol (examples/utilities.py:440-519); cparams layout in include/slb200.h.  The
// (de)normalisation is the reference's tf.matmul(state, diag(T)), written out: each column adds the other
// component times 0, so an inf or NaN component turns the other column into NaN, as the matmul does.
SLB_DEV void vanderpol_scale(double& x, double& y, double tx, double ty) {
    const double xs = f64add(f64mul(x, tx), f64mul(y, 0.0));
    y = f64add(f64mul(x, 0.0), f64mul(y, ty));
    x = xs;
}

SLB_DEV void eval_vanderpol(const slb_function& f, const double* in, double* out) {
    const double* p = f.cparams;
    const double damping = p[0], dt = p[1];
    const bool has_norm = p[2] != 0.0;
    double x = in[0], y = in[1];
    if (has_norm) vanderpol_scale(x, y, p[3], p[4]);
    for (int i = 0; i < 10; ++i) {
        // x' = -y, y' = x + damping (x^2 - 1) y, rounded left to right; state + dt * derivative
        const double y_dot = f64add(x, f64mul(f64mul(damping, f64sub(f64mul(x, x), 1.0)), y));
        x = f64add(x, f64mul(dt, -y));
        y = f64add(y, f64mul(dt, y_dot));
    }
    if (has_norm) vanderpol_scale(x, y, p[5], p[6]);
    out[0] = x; out[1] = y;
}

// ---- the fused networks: LyapunovNetwork (examples/utilities.py:85-104: h <- act(h . K_l^T), V = |h|^2)
// and NeuralNetwork (functions.py:1702-1729: dense layers, output multiplied by output_scale).
// Descriptor layout, written by _TrainableNetwork._network_descriptor (functions.py) and read only through
// the accessors below: cparams [0] layers, [1 + l] output width of layer l, [9 + l] activation of layer l
// (0 tanh, 1 relu, 2 identity), [17] the MLP's output_scale, [18] the MLP's use_bias.  `matrix` packs per
// layer its weight [out, in] (one row per output; LyapunovNetwork's kernel [W^T W + eps I; W_extra], built
// on the host), then its bias [out] if it has one.
#define SLB_NN_MAX_LAYERS 8
#define SLB_NN_MAX_WIDTH 64
#define SLB_NN_HD __host__ __device__ __forceinline__

SLB_NN_HD int nn_layers(const slb_function& f) { return (int)f.cparams[0]; }
SLB_NN_HD int nn_out(const slb_function& f, int l) { return (int)f.cparams[1 + l]; }     // layer l's width
// width l of the network: l = 0 its input, l >= 1 the output of layer l - 1
SLB_NN_HD int nn_width(const slb_function& f, int l) { return l == 0 ? f.in_dim : nn_out(f, l - 1); }
SLB_NN_HD int nn_act(const slb_function& f, int l) { return (int)f.cparams[9 + l]; }
// with use_bias the MLP's hidden layers carry a bias; its output layer and LyapunovNetwork have none
SLB_NN_HD bool nn_use_bias(const slb_function& f) { return f.kind == SLB_FN_MLP && f.cparams[18] != 0.0; }
SLB_NN_HD bool nn_bias(const slb_function& f, int l) { return nn_use_bias(f) && l + 1 < nn_layers(f); }
SLB_NN_HD double nn_scale(const slb_function& f) { return f.cparams[17]; }     // MLP only
// doubles of a layer wi -> wo in the packed parameters: its weight [wo, wi], then its bias [wo] if it has one
SLB_NN_HD int64_t nn_layer_size(int wi, int wo, bool bias) { return (int64_t)wo * wi + (bias ? wo : 0); }

// The activations (0 tanh, 1 relu, 2 identity) and their derivatives from the activation's output h
// (tanh' = 1 - h^2, ReLU' = [h > 0], so 0 at exactly 0, as TF's).
SLB_DEV double activate(double acc, int act) {
    return act == 0 ? tanh(acc) : (act == 1 ? fmax(acc, 0.0) : acc);
}

SLB_DEV double activate_grad(double h, int act) {
    return act == 0 ? 1.0 - h * h : (act == 1 ? (h > 0.0 ? 1.0 : 0.0) : 1.0);
}

// One unit of a layer: act(x(0) w(0) + ... + x(n-1) w(n-1) [+ bias()]), products and sums rounded in
// ascending k (f64mul / f64add, never contracted).  The accessors read the unit's operands; bias() is
// called only when has_bias.  Every forward pass of the networks (eval_network, network_input_gradient's
// recompute, vjp_network_kernel in network_grad.cu) computes its units here, so their activations and
// ReLU masks agree bit for bit.
template <class X, class W, class B>
SLB_DEV double nn_unit(int n, X x, W w, bool has_bias, B bias, int act) {
    double acc = f64mul(x(0), w(0));
    for (int k = 1; k < n; ++k) acc = f64add(acc, f64mul(x(k), w(k)));
    if (has_bias) acc = f64add(acc, bias());
    return activate(acc, act);
}

// a layer wi -> wo at one point: g = act(W h [+ b]) from its packed parameters P
SLB_DEV void nn_layer(const double* P, int wi, int wo, bool bias, int act, const double* h, double* g) {
    const double* b = P + (size_t)wo * wi;
    for (int o = 0; o < wo; ++o) {
        const double* row = P + (size_t)o * wi;
        g[o] = nn_unit(wi, [&](int k) { return h[k]; }, [&](int k) { return row[k]; }, bias,
                       [&] { return b[o]; }, act);
    }
}

// KIND = f.kind.  LyapunovNetwork: out[0] = |h|^2; NeuralNetwork: out = h * output_scale (h = the last
// layer's output).  One instance per kind, so each inlines without the other's epilogue or bias test.
template <int KIND>
SLB_DEV void eval_network(const slb_function& f, const double* in, double* out) {
    double h[SLB_NN_MAX_WIDTH], g[SLB_NN_MAX_WIDTH];
    int width = f.in_dim;
    for (int k = 0; k < width; ++k) h[k] = in[k];
    const double* P = f.matrix;
    const int layers = nn_layers(f);
    const bool use_bias = KIND == SLB_FN_MLP && nn_use_bias(f);
    for (int l = 0; l < layers; ++l) {
        const int od = nn_out(f, l);
        const bool bias = use_bias && l + 1 < layers;
        nn_layer(P, width, od, bias, nn_act(f, l), h, g);
        P += nn_layer_size(width, od, bias);
        width = od;
        for (int k = 0; k < width; ++k) h[k] = g[k];
    }
    if constexpr (KIND == SLB_FN_MLP) {
        for (int k = 0; k < width; ++k) out[k] = f64mul(h[k], nn_scale(f));
    } else {
        double v = f64mul(h[0], h[0]);
        for (int k = 1; k < width; ++k) v = f64add(v, f64mul(h[k], h[k]));
        out[0] = v;
    }
}

// SLB_FLAG_GRADIENT on SLB_FN_LYAPUNOV_NN or a one-output SLB_FN_MLP: out = d f / d x at one point
// (in_dim columns).  Reverse mode in vjp_network_kernel's operation order (network_grad.cu) for the
// cotangent 1: the forward through nn_unit, delta = 2 h (LyapunovNetwork) or output_scale (MLP) times
// activate_grad(h), then per input k the fma chain over the layer's outputs in ascending order from 0.0.
// The result equals slb_function_vjp(grad_out = 1).grad_in bit for bit.
// Four width-64 arrays per thread: the activations are not stored, the forward is recomputed up to
// layer l + 1 for the backward step through layer l (L (L + 1) / 2 layer evaluations; 6 for three
// layers).  Never inlined, so the kernels that inline eval_fn carry one call site, not this body.
static __device__ __noinline__ int network_input_gradient(const slb_function& f, const double* in, double* out) {
    double h[SLB_NN_MAX_WIDTH], g[SLB_NN_MAX_WIDTH];          // forward: a layer's input and output
    double d[SLB_NN_MAX_WIDTH], e[SLB_NN_MAX_WIDTH];          // backward: delta of layer l, dV/d(its input)
    const int layers = nn_layers(f);
    const bool mlp = f.kind == SLB_FN_MLP, use_bias = nn_use_bias(f);
    for (int l = layers - 1; l >= 0; --l) {
        // forward through layers 0..l: h = the output of layer l, W = its weight [width, wi]
        int width = f.in_dim;
        for (int k = 0; k < width; ++k) h[k] = in[k];
        const double* P = f.matrix;
        const double* W = P;
        int wi = width;
        for (int j = 0; j <= l; ++j) {
            const int od = nn_out(f, j);
            const bool bias = use_bias && j + 1 < layers;
            nn_layer(P, width, od, bias, nn_act(f, j), h, g);
            W = P;
            wi = width;
            P += nn_layer_size(width, od, bias);
            width = od;
            for (int k = 0; k < width; ++k) h[k] = g[k];
        }
        const int act = nn_act(f, l);
        if (l == layers - 1) {
            for (int o = 0; o < width; ++o) d[o] = (mlp ? nn_scale(f) : 2.0 * h[o]) * activate_grad(h[o], act);
        } else {
            for (int o = 0; o < width; ++o) d[o] = e[o] * activate_grad(h[o], act);
        }
        for (int k = 0; k < wi; ++k) {
            double s = 0.0;
            for (int o = 0; o < width; ++o) s = fma(d[o], W[(size_t)o * wi + k], s);
            e[k] = s;
        }
    }
    for (int k = 0; k < f.in_dim; ++k) out[k] = e[k];
    return f.in_dim;
}

// Evaluate a fused function object. `in` has f.in_dim entries, `out` receives the result
// columns; returns the number of columns (in_dim for a network under SLB_FLAG_GRADIENT, 1 after
// NORM1 / MAXABS).  slb_fn_columns (light.cu) states
// that number on the host, where it sizes the kernels and checks shapes: a change to one must be
// made to the other.  In gp_sweep.cu (SLB_EVAL_NOINLINE) it
// is deliberately NOT inlined: the tile kernel calls it five times per point (policy, V twice,
// L_V twice) in cold prologue / epilogue code, and one shared copy keeps the kernel text small.
// The thread-per-point kernels of light.cu inline it (the call overhead would cost them more).
#ifdef SLB_EVAL_NOINLINE
#define SLB_EVAL_ATTR static __device__ __noinline__
#else
#define SLB_EVAL_ATTR static __device__ __forceinline__
#endif
SLB_EVAL_ATTR int eval_fn(const slb_function& f, const double* in, double* out) {
    int od = f.out_dim;
    switch (f.kind) {
    case SLB_FN_CONSTANT:
        for (int o = 0; o < od; ++o) out[o] = f.cparams[o];
        break;
    case SLB_FN_LINEAR:       // functions.py:1583   y_o = sum_k x_k A[o,k]
        for (int o = 0; o < od; ++o) {
            const double* row = f.matrix + o * f.in_dim;
            double acc = f64mul(in[0], row[0]);
            for (int k = 1; k < f.in_dim; ++k) acc = f64add(acc, f64mul(in[k], row[k]));
            out[o] = acc;
        }
        break;
    case SLB_FN_QUADRATIC: {  // functions.py:1537-1539   sum_c (sum_r x_r P[r,c]) * x_c
        const int n = f.in_dim;
        double total = 0.0;
        for (int c = 0; c < n; ++c) {
            double lin = f64mul(in[0], f.matrix[c]);
            for (int r = 1; r < n; ++r) lin = f64add(lin, f64mul(in[r], f.matrix[r * n + c]));
            const double prod = f64mul(lin, in[c]);
            total = (c == 0) ? prod : f64add(total, prod);
        }
        out[0] = total;
        od = 1;
        break;
    }
    case SLB_FN_TRIANGULATION:
        tri_lookup<TRI_EVAL>(f, in, out);
        break;
    case SLB_FN_PENDULUM:
        eval_pendulum(f, in, out); od = 2;
        break;
    case SLB_FN_CARTPOLE:
        eval_cartpole(f, in, out); od = 4;
        break;
    case SLB_FN_VANDERPOL:
        eval_vanderpol(f, in, out); od = 2;
        break;
    // SLB_NO_NETWORK_GRADIENT (value_opt.cu): the unit's host entry points reject network gradients, and
    // its kernels are compiled without the call (with it, ptxas gives value_operator_kernel<5, 6> 128
    // registers and about 850 bytes of spills)
    case SLB_FN_LYAPUNOV_NN:
#ifndef SLB_NO_NETWORK_GRADIENT
        if (f.flags & SLB_FLAG_GRADIENT) { od = network_input_gradient(f, in, out); break; }
#endif
        eval_network<SLB_FN_LYAPUNOV_NN>(f, in, out); od = 1;
        break;
    case SLB_FN_MLP:
#ifndef SLB_NO_NETWORK_GRADIENT
        if (f.flags & SLB_FLAG_GRADIENT) { od = network_input_gradient(f, in, out); break; }
#endif
        eval_network<SLB_FN_MLP>(f, in, out);
        break;
    // SLB_FN_PIECEWISE_CONSTANT (functions.py:875-887): the nearest vertex's row, NaN without a vertex; any
    // other kind: NaN.  The kind shares the default branch because a case of its own gave the generic
    // filter_head_kernel 4-8 more bytes of spills.
    default: {
        const int64_t v = f.kind == SLB_FN_PIECEWISE_CONSTANT ? grid_nearest_index(f.grid, f.cparams, in) : -1;
        for (int o = 0; o < od; ++o)
            out[o] = v < 0 ? __longlong_as_double(0x7ff8000000000000ll) : f.matrix[v * od + o];
        break;
    }
    }
    if (f.flags & SLB_FLAG_SATURATE)
        for (int o = 0; o < od; ++o) out[o] = fmin(fmax(out[o], f.lower), f.upper);
    if (f.flags & (SLB_FLAG_ABS | SLB_FLAG_NORM1))
        for (int o = 0; o < od; ++o) out[o] = fabs(out[o]);
    if (f.flags & SLB_FLAG_NORM1) {
        double acc = out[0];
        for (int o = 1; o < od; ++o) acc = f64add(acc, out[o]);
        out[0] = acc;
        od = 1;
    }
    if (f.flags & SLB_FLAG_MAXABS) {
        double acc = fabs(out[0]);
        for (int o = 1; o < od; ++o) acc = fmax(acc, fabs(out[o]));
        out[0] = acc;
        od = 1;
    }
    if (f.flags & SLB_FLAG_SCALE)
        for (int o = 0; o < od; ++o) out[o] = f64mul(out[o], f.out_scale);
    return od;
}

// Fast path in front of eval_fn for the small linear-algebra objects that make up the per-point
// prologue / epilogue of every sweep of the reference's experiments (policy = Saturation(LinearSystem),
// V = QuadraticFunction, L_V = abs(LinearSystem)): in_dim <= 4, out_dim <= 2, operands in registers,
// eval_fn's arithmetic operation for operation (bit-identical).  The generic interpreter costs a
// call, local-memory operand arrays and runtime-bounded loops per evaluation: five of them set
// the floor of the filter's mean stage (M = 0: tools/mean_floor_probe.py).
SLB_DEV int eval_fn_small(const slb_function& f, const double* in, double* out) {
    const int n = f.in_dim;
    if (f.kind == SLB_FN_LINEAR && n <= 4 && f.out_dim <= 2 &&
        !(f.flags & (SLB_FLAG_MAXABS | SLB_FLAG_GRADIENT))) {
        int od = f.out_dim;
        double x[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) x[k] = k < n ? in[k] : 0.0;
        double y[2];
#pragma unroll
        for (int o = 0; o < 2; ++o) {
            if (o < od) {
                const double* row = f.matrix + o * n;
                double acc = f64mul(x[0], __ldg(row));
#pragma unroll
                for (int k = 1; k < 4; ++k)
                    if (k < n) acc = f64add(acc, f64mul(x[k], __ldg(row + k)));
                y[o] = acc;
            } else {
                y[o] = 0.0;
            }
        }
        if (f.flags & SLB_FLAG_SATURATE) {
            y[0] = fmin(fmax(y[0], f.lower), f.upper);
            y[1] = fmin(fmax(y[1], f.lower), f.upper);
        }
        if (f.flags & (SLB_FLAG_ABS | SLB_FLAG_NORM1)) { y[0] = fabs(y[0]); y[1] = fabs(y[1]); }
        if (f.flags & SLB_FLAG_NORM1) {
            if (od == 2) y[0] = f64add(y[0], y[1]);
            od = 1;
        }
        if (f.flags & SLB_FLAG_SCALE) { y[0] = f64mul(y[0], f.out_scale); y[1] = f64mul(y[1], f.out_scale); }
        out[0] = y[0];
        if (od == 2) out[1] = y[1];
        return od;
    }
    if (f.kind == SLB_FN_QUADRATIC && n <= 4 && !(f.flags & ~SLB_FLAG_SCALE)) {
        double x[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) x[k] = k < n ? in[k] : 0.0;
        double total = 0.0;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            if (c < n) {
                double lin = f64mul(x[0], __ldg(f.matrix + c));
#pragma unroll
                for (int r = 1; r < 4; ++r)
                    if (r < n) lin = f64add(lin, f64mul(x[r], __ldg(f.matrix + r * n + c)));
                const double prod = f64mul(lin, x[c]);
                total = (c == 0) ? prod : f64add(total, prod);
            }
        }
        if (f.flags & SLB_FLAG_SCALE) total = f64mul(total, f.out_scale);
        out[0] = total;
        return 1;
    }
    return eval_fn(f, in, out);
}

// Register-only evaluators of the closed form the filter's factored grid path runs on (filter.cu,
// grid_mean_applicable): the saturated linear policy, V = x^T P x and a LINEAR L_V / L_f.  Shapes are
// compile-time, operands and results stay in registers and there is no fallback call: the host has proved
// the kind and flags.  Each is eval_fn_small's arithmetic operation for operation, and so bit-identical to
// eval_fn (for out_dim 3 and 4, which eval_fn_small leaves to eval_fn, eval_fn's own order).
template <int N> struct slb_vec { double v[N]; };
constexpr int SLB_MAX_LIN_OUT = 4;     // out_dim of a closed-form L_V / L_f (grid_mean_applicable)

// LINEAR, in_dim N, out_dim <= MO (run time), flags among SATURATE | ABS | NORM1 | SCALE.  Returns the
// columns; `cols` = their number (1 after NORM1).
template <int N, int MO>
SLB_DEV slb_vec<MO> eval_linear_reg(const slb_function& f, const double (&x)[N], int& cols) {
    const int od = f.out_dim;
    slb_vec<MO> y;
#pragma unroll
    for (int o = 0; o < MO; ++o) {
        y.v[o] = 0.0;
        if (o < od) {
            const double* row = f.matrix + o * N;
            double acc = f64mul(x[0], __ldg(row));
#pragma unroll
            for (int k = 1; k < N; ++k) acc = f64add(acc, f64mul(x[k], __ldg(row + k)));
            y.v[o] = acc;
        }
    }
    if (f.flags & SLB_FLAG_SATURATE) {
#pragma unroll
        for (int o = 0; o < MO; ++o) y.v[o] = fmin(fmax(y.v[o], f.lower), f.upper);
    }
    if (f.flags & (SLB_FLAG_ABS | SLB_FLAG_NORM1)) {
#pragma unroll
        for (int o = 0; o < MO; ++o) y.v[o] = fabs(y.v[o]);
    }
    cols = od;
    if (f.flags & SLB_FLAG_NORM1) {
#pragma unroll
        for (int o = 1; o < MO; ++o)
            if (o < od) y.v[0] = f64add(y.v[0], y.v[o]);
        cols = 1;
    }
    if (f.flags & SLB_FLAG_SCALE) {
#pragma unroll
        for (int o = 0; o < MO; ++o) y.v[o] = f64mul(y.v[o], f.out_scale);
    }
    return y;
}

// QUADRATIC, in_dim N, flags among SCALE:  sum_c (sum_r x_r P[r,c]) x_c
template <int N>
SLB_DEV double eval_quadratic_reg(const slb_function& f, const double (&x)[N]) {
    double total = 0.0;
#pragma unroll
    for (int c = 0; c < N; ++c) {
        double lin = f64mul(x[0], __ldg(f.matrix + c));
#pragma unroll
        for (int r = 1; r < N; ++r) lin = f64add(lin, f64mul(x[r], __ldg(f.matrix + r * N + c)));
        const double prod = f64mul(lin, x[c]);
        total = (c == 0) ? prod : f64add(total, prod);
    }
    if (f.flags & SLB_FLAG_SCALE) total = f64mul(total, f.out_scale);
    return total;
}

// The per-point prologue / epilogue of a sweep kernel reads a handful of small operands through
// pointers of the descriptor (policy / V / L_V / L_f matrices, prior-mean rows), one dependent global
// load after the other; after an L2 flush (or any eviction) each is an HBM round trip in every CTA's
// serial chain.  Touch them all at once when the kernel starts.
SLB_DEV void prefetch_descriptor_operands(const slb_sweep& cfg) {
    const int i = threadIdx.x;
    const void* p = nullptr;
    if (i == 0) p = cfg.policy.matrix;
    else if (i == 1) p = cfg.lyapunov.matrix;
    else if (i == 2) p = cfg.lipschitz_v.matrix;
    else if (i == 3) p = cfg.lipschitz_f.matrix;
    else if (i < 4 + cfg.gp.num_outputs && i < 4 + SLB_MAX_OUT) p = cfg.gp.outputs[i - 4].prior_mean;
    if (p != nullptr) asm volatile("prefetch.global.L1 [%0];" ::"l"(p));
}

// The Lyapunov decision for one state (lyapunov.py:265-288, 324-376, 441).
//   x [d]; mu [d] predicted mean; err [d] error bounds (beta*sigma) or nullptr when the
//   dynamics are deterministic.  Returns negative = decrease < threshold (false on NaN).
struct slb_decision { double vx, decrease, threshold; bool negative; };

// The decision of lyapunov.py:436-441 in three independent pieces (the tile kernel evaluates the
// x-only piece while the GP runs, and the two mean-dependent pieces on different warps):
// (1) V(x) and threshold(x) = -|L_V(x)|_1 (1 + L_f) tau                      :284-288
// `flat_index` is the point's flat grid index (for cfg.lf_values), or -1 for an explicit state.
SLB_DEV void lyapunov_state_terms(const slb_sweep& cfg, const double* x, int64_t flat_index,
                                  double* vx_out, double* threshold_out) {
    double tmp[SLB_MAX_OUT], vx[1];
    eval_fn_small(cfg.lyapunov, x, vx);
    *vx_out = vx[0];
    double lvx;
    if (cfg.lipschitz_v.kind != SLB_FN_NONE) {               // :284-286 (1-norm of a vector lv)
        const int nl = eval_fn_small(cfg.lipschitz_v, x, tmp);
        lvx = tmp[0];
        if (nl > 1) {
            lvx = fabs(tmp[0]);
            for (int j = 1; j < nl; ++j) lvx = f64add(lvx, fabs(tmp[j]));
        }
    } else {
        lvx = cfg.lv_const;
    }
    double lf = cfg.lf_const;                                // lyapunov.py:227-244, :287
    if (cfg.lf_values != nullptr && flat_index >= 0) {
        lf = cfg.lf_values[flat_index - cfg.lf_index_base];
    } else if (cfg.lipschitz_f.kind != SLB_FN_NONE) {
        eval_fn_small(cfg.lipschitz_f, x, tmp);
        lf = tmp[0];
    }
    *threshold_out = f64mul(f64mul(-lvx, f64add(1.0, lf)), cfg.tau);   // :288
}

// ... the same for the closed form (a state of D dims, V QUADRATIC, L_V and L_f absent or LINEAR with
// the flags eval_linear_reg takes): the register-only evaluators, the arithmetic above
template <int D>
SLB_DEV void lyapunov_state_terms_closed(const slb_sweep& cfg, const double (&x)[D], int64_t flat_index,
                                         double* vx_out, double* threshold_out) {
    *vx_out = eval_quadratic_reg<D>(cfg.lyapunov, x);
    double lvx = cfg.lv_const;
    if (cfg.lipschitz_v.kind != SLB_FN_NONE) {
        int nl;
        const slb_vec<SLB_MAX_LIN_OUT> lv = eval_linear_reg<D, SLB_MAX_LIN_OUT>(cfg.lipschitz_v, x, nl);
        lvx = lv.v[0];
        if (nl > 1) {
            lvx = fabs(lv.v[0]);
#pragma unroll
            for (int j = 1; j < SLB_MAX_LIN_OUT; ++j)
                if (j < nl) lvx = f64add(lvx, fabs(lv.v[j]));
        }
    }
    double lf = cfg.lf_const;
    if (cfg.lf_values != nullptr && flat_index >= 0) {
        lf = cfg.lf_values[flat_index - cfg.lf_index_base];
    } else if (cfg.lipschitz_f.kind != SLB_FN_NONE) {
        int nf;
        lf = eval_linear_reg<D, SLB_MAX_LIN_OUT>(cfg.lipschitz_f, x, nf).v[0];
    }
    *threshold_out = f64mul(f64mul(-lvx, f64add(1.0, lf)), cfg.tau);
}

// (2) sum_j L_V(mu)_j err_j, L_V evaluated at the predicted MEAN                :344-347
// ... from L_V(mu)'s nl columns lv (one column: the same factor for every j)
SLB_DEV double lyapunov_error_sum(const double* lv, int nl, const double* err, int d) {
    double bound = f64mul(lv[0], err[0]);
    for (int j = 1; j < d; ++j) bound = f64add(bound, f64mul(nl == 1 ? lv[0] : lv[j], err[j]));
    return bound;
}

SLB_DEV double lyapunov_error_bound(const slb_sweep& cfg, const double* mu, const double* err) {
    double lv[SLB_MAX_OUT];
    int nl = 1;
    lv[0] = cfg.lv_const;
    if (cfg.lipschitz_v.kind != SLB_FN_NONE) nl = eval_fn_small(cfg.lipschitz_v, mu, lv);
    return lyapunov_error_sum(lv, nl, err, cfg.grid.ndim);
}

// ... the same for the closed form (D outputs = the state's dims, L_V absent or LINEAR as in
// lyapunov_state_terms_closed)
template <int D>
SLB_DEV double lyapunov_error_bound_closed(const slb_sweep& cfg, const double (&mu)[D], const double (&err)[D]) {
    int nl = 1;
    slb_vec<SLB_MAX_LIN_OUT> lv;
    lv.v[0] = cfg.lv_const;
    if (cfg.lipschitz_v.kind != SLB_FN_NONE) lv = eval_linear_reg<D, SLB_MAX_LIN_OUT>(cfg.lipschitz_v, mu, nl);
    return lyapunov_error_sum(lv.v, nl, err, D);
}

// (3) V(mu); then decrease = (V(mu) - V(x)) + bound  and  negative = decrease < threshold
SLB_DEV slb_decision lyapunov_combine(double vx, double threshold, double vm, double bound) {
    slb_decision r;
    r.vx = vx;
    r.threshold = threshold;
    r.decrease = f64add(f64sub(vm, vx), bound);                // :351-352, :376
    r.negative = r.decrease < r.threshold;                   // :441 strict, NaN -> false
    return r;
}

SLB_DEV slb_decision lyapunov_decide(const slb_sweep& cfg, const double* x, int64_t flat_index,
                                     const double* mu, const double* err) {
    double vx, threshold, vm[1];
    lyapunov_state_terms(cfg, x, flat_index, &vx, &threshold);
    eval_fn_small(cfg.lyapunov, mu, vm);
    const double bound = err != nullptr ? lyapunov_error_bound(cfg, mu, err) : 0.0;
    return lyapunov_combine(vx, threshold, vm[0], bound);
}
