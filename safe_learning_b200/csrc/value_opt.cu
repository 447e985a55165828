// value_opt.cu -- PolicyIteration.optimize_value_function (reinforcement_learning.py:142-211):
// exact policy evaluation, the fixed point of  v = r + gamma T v  on the value function's grid.
//
// The reference solves the LP  max sum(v)  s.t.  v <= r + gamma T v  (cvxpy); with nonnegative
// barycentric rows (each sums to 1) and gamma < 1 its optimum is that fixed point (DESIGN.md §3.9).
//
//   assembly   one thread per vertex: u = pi(x_i), x_i+ = mean f(x_i, u), r_i = r(x_i, u) (fused, as in
//              the Bellman sweep), or x+ from a device array (composed); row i of T = the d + 1
//              barycentric weights of x_i+ (the Triangulation lookup of common.cuh), with rows whose
//              lookup extrapolates from the wrong simplex of the right cell (DESIGN.md §3.2 Q6)
//              re-searched from cell-relative unit coordinates.  A PiecewiseConstant value table gives
//              one-hot rows: the next state's nearest vertex (grid_nearest_index) with weight 1, stored
//              with a zero-weight second entry (the solver's narrowest row).
//   solve      v_{k+1} = r + gamma (w_0 v_k[c_0] + ... + w_d v_k[c_d]), non-contracted, in this order
//              (the arithmetic of one Bellman sweep), until the certified error
//              gamma rho / (1 - gamma rho) ||v_k - v_{k-1}||_inf  <=  tol max(1, ||v_k||_inf),
//              rho = max_i sum_j |w_ij|.  One CTA with both iterates in shared memory for small grids,
//              else one cooperative launch with a grid barrier per iteration.
// A network gradient (SLB_FLAG_GRADIENT on a network) is not compiled into the assembly kernel, and
// slb_value_operator rejects one as its policy, dynamics or reward.
#define SLB_NO_NETWORK_GRADIENT
#include "bellman.cuh"

#include <cooperative_groups.h>
#include <string.h>

namespace cg = cooperative_groups;

namespace {

constexpr int VT = 256;                   // assembly threads per block
constexpr int VS_THREADS = 1024;          // solver threads per block
constexpr int64_t VS_SMALL_MAX = 12288;   // one-CTA tier: 2 x 12288 doubles = 192 KB of shared memory
constexpr double W_TOL = 1e-12;           // barycentric tolerance of the simplex search

// stats slots (uint64, SLB_VALUE_STATS of them, see slb200.h)
enum { ST_MINW = 0, ST_RHO, ST_REPAIRED, ST_NAN, ST_ITERS, ST_DELTA, ST_BOUND, ST_STATUS, ST_TIER };

SLB_DEV unsigned long long dbits(double v) { return (unsigned long long)__double_as_longlong(v); }
SLB_DEV double bitsd(unsigned long long b) { return __longlong_as_double((long long)b); }
SLB_DEV unsigned long long umax(unsigned long long a, unsigned long long b) { return a > b ? a : b; }

// per-block accumulation of the assembly statistics, then one set of global atomics
struct row_stats {
    unsigned long long minw_inv, rho, repaired, nan;     // minw_inv = ~value_key(min weight)
};

SLB_DEV void stats_flush(row_stats& s, unsigned long long* __restrict__ stats) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        s.minw_inv = umax(s.minw_inv, __shfl_xor_sync(0xffffffffu, s.minw_inv, off));
        s.rho = umax(s.rho, __shfl_xor_sync(0xffffffffu, s.rho, off));
        s.repaired += __shfl_xor_sync(0xffffffffu, s.repaired, off);
        s.nan += __shfl_xor_sync(0xffffffffu, s.nan, off);
    }
    if ((threadIdx.x & 31) == 0) {
        atomicMax(stats + ST_MINW, s.minw_inv);
        atomicMax(stats + ST_RHO, s.rho);
        if (s.repaired) atomicAdd(stats + ST_REPAIRED, s.repaired);
        if (s.nan) atomicAdd(stats + ST_NAN, s.nan);
    }
}

// entries per row of T: d + 1 barycentric weights of a Triangulation, two for a PiecewiseConstant (its
// one-hot row and a zero-weight filler: slb_value_solve takes rows of 2 .. SLB_MAX_DIM + 1 entries)
SLB_DEV int operator_cols(const slb_function& f) {
    return f.kind == SLB_FN_PIECEWISE_CONSTANT ? 2 : f.grid.ndim + 1;
}

// Row of T for the next state xp: columns (vertex indices) and weights.  The reference's lookup
// (tri_lookup, common.cuh); when it yields a weight < -W_TOL although the point is inside the grid
// (or projected onto it), the point lies on a grid line where `% unit_maxes` rounded to ~unit_maxes
// and picked a simplex of the wrong side of the cell: search the cell again with unit coordinates
// taken relative to the cell's own lowest vertex (TRI_CELL).
// A PiecewiseConstant's row is the nearest vertex with weight 1, then the same vertex with weight 0: for a
// finite v, w_0 v + 0 v is v bit for bit, so the solver's arithmetic is that of the one-hot row.  A NaN
// next state has no vertex and gives vertex 0 with weight NaN, counted in the NaN slot like a
// Triangulation's NaN row.
template <typename IDX>
SLB_DEV void operator_row(const slb_function& f, const double* xp, IDX* __restrict__ cols,
                          double* __restrict__ W, row_stats& st) {
    const slb_grid& g = f.grid;
    const int d = g.ndim;
    if (f.kind == SLB_FN_PIECEWISE_CONSTANT) {
        const int64_t v = grid_nearest_index(g, f.cparams, xp);
        const double w = v < 0 ? __longlong_as_double(0x7ff8000000000000ll) : 1.0;
        cols[0] = cols[1] = (IDX)(v < 0 ? 0 : v);
        W[0] = w;
        W[1] = 0.0;
        st.minw_inv = umax(st.minw_inv, ~value_key(v < 0 ? w : 0.0));
        st.rho = umax(st.rho, dbits(fabs(w)));
        st.nan += v < 0;
        return;
    }
    int64_t corner;
    int s;
    double w[SLB_MAX_DIM + 1];
    tri_lookup<TRI_WEIGHTS>(f, xp, w, &corner, &s);
    double wmin = w[0];
    bool inside = true, bad = false;
    for (int k = 0; k < d; ++k) {
        wmin = fmin(wmin, w[k + 1]);
        inside = inside && xp[k] >= g.offset[k] && xp[k] <= g.upper[k];
        bad = bad || xp[k] != xp[k];
    }
    if (wmin < -W_TOL && ((f.flags & SLB_FLAG_PROJECT) || inside)) {
        tri_lookup<TRI_CELL>(f, xp, w, &corner, &s);
        st.repaired += 1;
    }
    const int64_t* simp = f.unit_simplices + (size_t)s * (d + 1);
    double a = fabs(w[0]);
    wmin = w[0];
    for (int k = 0; k <= d; ++k) {
        cols[k] = (IDX)(simp[k] + corner);
        W[k] = w[k];
        if (k > 0) { a = f64add(a, fabs(w[k])); wmin = fmin(wmin, w[k]); }
    }
    if (wmin != wmin) bad = true;
    st.minw_inv = umax(st.minw_inv, ~value_key(wmin));
    st.rho = umax(st.rho, dbits(a));                      // a >= 0 (NaN: above +inf)
    st.nan += bad;
}

template <int DIN, typename IDX>
__global__ void __launch_bounds__(VT)
value_operator_kernel(const __grid_constant__ slb_bellman cfg, int64_t idx_begin, int64_t n,
                      IDX* __restrict__ cols, double* __restrict__ weights, double* __restrict__ rewards,
                      unsigned long long* __restrict__ stats, int chunk_rows, int nomax) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    bellman_smem S;
    bellman_setup<DIN>(S, smem_raw, cfg, chunk_rows, nomax);
    const int64_t i0 = (int64_t)blockIdx.x * VT + threadIdx.x;
    const bool valid = i0 < n;
    const int64_t i = valid ? i0 : n - 1;       // every thread stays for the block barriers
    const int d = cfg.grid.ndim;
    const int nc = operator_cols(cfg.value);
    double x[SLB_MAX_DIM], u[SLB_MAX_OUT], mu[SLB_MAX_OUT], r[SLB_MAX_OUT];
    grid_index_to_state(cfg.grid, idx_begin + i, x);
    const int m = eval_fn(cfg.policy, x, u);
    bellman_transition<DIN>(cfg, x, u, m, S, mu, r);
    row_stats st = {0ull, 0ull, 0ull, 0ull};
    if (valid) {
        IDX c[SLB_MAX_DIM + 1];
        double w[SLB_MAX_DIM + 1];
        operator_row<IDX>(cfg.value, mu, c, w, st);
        for (int k = 0; k < nc; ++k) {
            cols[i * nc + k] = c[k];
            weights[i * nc + k] = w[k];
        }
        rewards[i] = r[0];
        st.nan += r[0] != r[0];
    }
    stats_flush(st, stats);
}

template <typename IDX>
__global__ void __launch_bounds__(VT)
value_operator_points_kernel(const __grid_constant__ slb_function f, const double* __restrict__ xp,
                             int64_t n, IDX* __restrict__ cols, double* __restrict__ weights,
                             unsigned long long* __restrict__ stats) {
    const int64_t i = (int64_t)blockIdx.x * VT + threadIdx.x;
    const int d = f.grid.ndim, nc = operator_cols(f);
    row_stats st = {0ull, 0ull, 0ull, 0ull};
    if (i < n) {
        double x[SLB_MAX_DIM];
        for (int k = 0; k < d; ++k) x[k] = xp[i * d + k];
        IDX c[SLB_MAX_DIM + 1];
        double w[SLB_MAX_DIM + 1];
        operator_row<IDX>(f, x, c, w, st);
        for (int k = 0; k < nc; ++k) {
            cols[i * nc + k] = c[k];
            weights[i * nc + k] = w[k];
        }
    }
    stats_flush(st, stats);
}

// ---- solver ----------------------------------------------------------------------------------
struct solve_args {
    int64_t n;
    int ncols;
    double gamma, tol;
    int64_t max_iters;
};

// r_i + gamma (w_0 v[c_0] + w_1 v[c_1] + ...): tri_lookup's and bellman_value's arithmetic
template <typename IDX>
SLB_DEV double apply_row(const IDX* __restrict__ cols, const double* __restrict__ W, double r, int ncols,
                         double gamma, const double* v, int64_t i) {
    const IDX* c = cols + i * ncols;
    const double* w = W + i * ncols;
    double s = f64mul(__ldg(w), v[__ldg(c)]);
    for (int k = 1; k < ncols; ++k) s = f64add(s, f64mul(__ldg(w + k), v[__ldg(c + k)]));
    return f64add(r, f64mul(gamma, s));
}

// the thread's share of the prologue: smallest weight, largest row sum of |w|, NaN in a weight, a
// reward or the start table (a NaN vertex value would keep the iteration from ever converging)
template <typename IDX>
SLB_DEV void scan_rows(const solve_args& a, const double* __restrict__ W, const double* __restrict__ R,
                       const double* __restrict__ V0, int64_t i, unsigned long long& minw_inv,
                       unsigned long long& rho, unsigned long long& nan) {
    const double* w = W + i * a.ncols;
    double s = fabs(w[0]), mn = w[0];
    for (int k = 1; k < a.ncols; ++k) { s = f64add(s, fabs(w[k])); mn = fmin(mn, w[k]); }
    if (s != s || R[i] != R[i] || V0[i] != V0[i]) nan = 1;
    minw_inv = umax(minw_inv, ~value_key(mn));
    rho = umax(rho, dbits(s));
}

SLB_DEV unsigned long long warp_max(unsigned long long v) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v = umax(v, __shfl_xor_sync(0xffffffffu, v, off));
    return v;
}

// status from the prologue (uniform across threads): 0 = iterate, else the final status
SLB_DEV int prologue_status(unsigned long long minw_inv, unsigned long long rho_bits,
                            unsigned long long nan, double gamma, double* q) {
    if (nan) return SLB_VALUE_NAN;
    const double minw = key_value(~minw_inv);
    if (minw < -W_TOL) return SLB_VALUE_NEGATIVE_WEIGHT;
    const double gr = f64mul(gamma, bitsd(rho_bits));
    if (!(gr < 1.0)) return SLB_VALUE_NOT_CONTRACTIVE;
    *q = gr / f64sub(1.0, gr);
    return 0;
}

SLB_DEV void write_stats(unsigned long long* stats, unsigned long long minw_inv, unsigned long long rho,
                         int64_t iters, double delta, double bound, int status, int tier) {
    stats[ST_MINW] = minw_inv;
    stats[ST_RHO] = rho;
    stats[ST_ITERS] = (unsigned long long)iters;
    stats[ST_DELTA] = dbits(delta);
    stats[ST_BOUND] = dbits(bound);
    stats[ST_STATUS] = (unsigned long long)status;
    stats[ST_TIER] = (unsigned long long)tier;
}

// One CTA: both iterates in shared memory, one barrier per iteration (the iterate being read and the
// reduction slots alternate, so no thread can overwrite what another still reads).
template <typename IDX>
__global__ void __launch_bounds__(VS_THREADS, 1)
value_solve_small_kernel(const solve_args a, const IDX* __restrict__ cols, const double* __restrict__ W,
                         const double* __restrict__ R, double* __restrict__ v_inout,
                         unsigned long long* __restrict__ stats) {
    extern __shared__ double vs[];                           // [2][n]
    __shared__ unsigned long long red[2][2][VS_THREADS / 32];
    __shared__ unsigned long long pro[3];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t n = a.n;
    if (tid < 3) pro[tid] = 0ull;
    unsigned long long minw_inv = 0ull, rho = 0ull, nan = 0ull;
    for (int64_t i = tid; i < n; i += VS_THREADS) {
        vs[i] = v_inout[i];
        scan_rows<IDX>(a, W, R, v_inout, i, minw_inv, rho, nan);
    }
    minw_inv = warp_max(minw_inv);
    rho = warp_max(rho);
    nan = warp_max(nan);
    __syncthreads();
    if (lane == 0) {
        atomicMax(&pro[0], minw_inv);
        atomicMax(&pro[1], rho);
        atomicMax(&pro[2], nan);
    }
    __syncthreads();
    minw_inv = pro[0]; rho = pro[1]; nan = pro[2];
    double q = 0.0;
    int status = prologue_status(minw_inv, rho, nan, a.gamma, &q);
    int64_t k = 0;
    double delta = 0.0, bound = 0.0;
    while (status == 0) {
        ++k;
        const double* cur = vs + ((k & 1) ? 0 : n);
        double* nxt = vs + ((k & 1) ? n : 0);
        unsigned long long dl = 0ull, vm = 0ull;
        for (int64_t i = tid; i < n; i += VS_THREADS) {
            const double nv = apply_row<IDX>(cols, W, __ldg(R + i), a.ncols, a.gamma, cur, i);
            nxt[i] = nv;
            dl = umax(dl, dbits(fabs(f64sub(nv, cur[i]))));
            vm = umax(vm, dbits(fabs(nv)));
        }
        dl = warp_max(dl);
        vm = warp_max(vm);
        if (lane == 0) { red[k & 1][0][warp] = dl; red[k & 1][1][warp] = vm; }
        __syncthreads();
        dl = 0ull; vm = 0ull;
        for (int j = 0; j < VS_THREADS / 32; ++j) {
            dl = umax(dl, red[k & 1][0][j]);
            vm = umax(vm, red[k & 1][1][j]);
        }
        delta = bitsd(dl);
        bound = f64mul(q, delta);
        if (bound <= f64mul(a.tol, fmax(1.0, bitsd(vm)))) break;       // NaN: never converges
        if (k >= a.max_iters) { status = SLB_VALUE_MAX_ITERS; break; }
    }
    if (k > 0) {
        const double* fin = vs + ((k & 1) ? n : 0);
        for (int64_t i = tid; i < n; i += VS_THREADS) v_inout[i] = fin[i];
    }
    if (tid == 0) write_stats(stats, minw_inv, rho, k, delta, bound, status, 1);
}

// Cooperative tier: the grid sweeps the rows, warp maxima go to global slots that rotate over three
// iterations (slot k % 3 is written in iteration k and read after its grid barrier; iteration k + 2
// clears it -- one barrier after that read and one before its next use in iteration k + 3).
template <typename IDX>
__global__ void __launch_bounds__(VS_THREADS, 1)
value_solve_coop_kernel(const solve_args a, const IDX* __restrict__ cols, const double* __restrict__ W,
                        const double* __restrict__ R, double* __restrict__ v_inout, double* __restrict__ v_alt,
                        unsigned long long* __restrict__ slots, unsigned long long* __restrict__ stats) {
    cg::grid_group grid = cg::this_grid();
    const int64_t n = a.n;
    const int64_t stride = (int64_t)gridDim.x * VS_THREADS;
    const int64_t first = (int64_t)blockIdx.x * VS_THREADS + threadIdx.x;
    const int lane = threadIdx.x & 31;
    unsigned long long minw_inv = 0ull, rho = 0ull, nan = 0ull;
    for (int64_t i = first; i < n; i += stride) scan_rows<IDX>(a, W, R, v_inout, i, minw_inv, rho, nan);
    minw_inv = warp_max(minw_inv);
    rho = warp_max(rho);
    nan = warp_max(nan);
    if (lane == 0) {
        atomicMax(slots + 0, minw_inv);
        atomicMax(slots + 1, rho);
        atomicMax(slots + 2, nan);
    }
    grid.sync();
    minw_inv = *(volatile unsigned long long*)(slots + 0);
    rho = *(volatile unsigned long long*)(slots + 1);
    nan = *(volatile unsigned long long*)(slots + 2);
    unsigned long long* iter_slots = slots + 4;              // [3][2]
    double q = 0.0;
    int status = prologue_status(minw_inv, rho, nan, a.gamma, &q);
    int64_t k = 0;
    double delta = 0.0, bound = 0.0;
    while (status == 0) {
        ++k;
        const double* cur = (k & 1) ? v_inout : v_alt;
        double* nxt = (k & 1) ? v_alt : v_inout;
        unsigned long long* slot = iter_slots + 2 * (k % 3);
        if (first == 0) {                                    // slot of iteration k + 1
            unsigned long long* next = iter_slots + 2 * ((k + 1) % 3);
            next[0] = 0ull;
            next[1] = 0ull;
        }
        unsigned long long dl = 0ull, vm = 0ull;
        for (int64_t i = first; i < n; i += stride) {
            const double c = cur[i];
            const double nv = apply_row<IDX>(cols, W, __ldg(R + i), a.ncols, a.gamma, cur, i);
            nxt[i] = nv;
            dl = umax(dl, dbits(fabs(f64sub(nv, c))));
            vm = umax(vm, dbits(fabs(nv)));
        }
        dl = warp_max(dl);
        vm = warp_max(vm);
        if (lane == 0) {
            if (dl) atomicMax(slot + 0, dl);
            if (vm) atomicMax(slot + 1, vm);
        }
        grid.sync();
        dl = *(volatile unsigned long long*)(slot + 0);
        vm = *(volatile unsigned long long*)(slot + 1);
        delta = bitsd(dl);
        bound = f64mul(q, delta);
        if (bound <= f64mul(a.tol, fmax(1.0, bitsd(vm)))) break;
        if (k >= a.max_iters) { status = SLB_VALUE_MAX_ITERS; break; }
    }
    if (k & 1)                                               // the last iterate is in v_alt
        for (int64_t i = first; i < n; i += stride) v_inout[i] = v_alt[i];
    if (first == 0) write_stats(stats, minw_inv, rho, k, delta, bound, status, 2);
}

}  // namespace

static bool wide_index(int64_t nindex) { return nindex > 0x7fffffffll; }

// the rows of T are the barycentric weights of a one-output Triangulation (projection allowed) or the
// one-hot rows of a one-output PiecewiseConstant, without post-op flags
static int validate_value_table(const slb_function& value, const char* who) {
    const bool tri = value.kind == SLB_FN_TRIANGULATION && !(value.flags & ~SLB_FLAG_PROJECT);
    const bool table = value.kind == SLB_FN_PIECEWISE_CONSTANT && value.flags == 0;
    SLB_CHECK((tri || table) && value.out_dim == 1,
              "%s: the value function must be a plain one-output Triangulation or PiecewiseConstant", who);
    return 0;
}

static bool network_gradient(const slb_function& f) {
    return (f.flags & SLB_FLAG_GRADIENT) && (f.kind == SLB_FN_LYAPUNOV_NN || f.kind == SLB_FN_MLP);
}

template <typename IDX>
static int launch_solve(cudaStream_t st, const solve_args& a, const void* cols, const double* W,
                        const double* R, double* v, void* workspace, unsigned long long* stats) {
    const IDX* c = static_cast<const IDX*>(cols);
    if (a.n <= VS_SMALL_MAX) {
        const size_t smem = 2 * (size_t)a.n * sizeof(double);
        SLB_CUDA(cudaFuncSetAttribute(value_solve_small_kernel<IDX>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        value_solve_small_kernel<IDX><<<1, VS_THREADS, smem, st>>>(a, c, W, R, v, stats);
        SLB_LAUNCH_CHECK();
        return 0;
    }
    double* v_alt = static_cast<double*>(workspace);
    unsigned long long* slots = reinterpret_cast<unsigned long long*>(v_alt + a.n);
    SLB_CUDA(cudaMemsetAsync(slots, 0, 16 * sizeof(uint64_t), st));
    int per_sm = 0;
    SLB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, value_solve_coop_kernel<IDX>,
                                                           VS_THREADS, 0));
    SLB_CHECK(per_sm >= 1, "slb_value_solve: the cooperative solver cannot be resident");
    const int64_t want = (a.n + VS_THREADS - 1) / VS_THREADS;
    const int blocks = (int)(want < (int64_t)per_sm * SLB_NUM_SMS ? want : (int64_t)per_sm * SLB_NUM_SMS);
    solve_args args = a;
    const IDX* cc = c;
    const double* WW = W;
    const double* RR = R;
    void* params[] = {(void*)&args, (void*)&cc, (void*)&WW, (void*)&RR, (void*)&v, (void*)&v_alt,
                      (void*)&slots, (void*)&stats};
    SLB_CUDA(cudaLaunchCooperativeKernel((const void*)value_solve_coop_kernel<IDX>, dim3(blocks),
                                         dim3(VS_THREADS), params, 0, st));
    SLB_LAUNCH_CHECK();
    return 0;
}

extern "C" {

int slb_value_operator(void* stream, const slb_bellman* cfg, int64_t idx_begin, int64_t idx_end,
                       void* cols_dev, double* weights_dev, double* rewards_dev, uint64_t* stats_dev) {
    int m;
    if (slb_validate_bellman(cfg, &m)) return 1;
    SLB_CHECK(!cfg->fixed_action, "slb_value_operator: the policy is evaluated, fixed_action must be 0");
    if (validate_value_table(cfg->value, "slb_value_operator")) return 1;
    SLB_CHECK(!network_gradient(cfg->policy) && !network_gradient(cfg->dynamics) && !network_gradient(cfg->reward),
              "slb_value_operator: a network gradient (SLB_FLAG_GRADIENT) is not compiled into the value operator");
    if (slb_validate_range("slb_value_operator", idx_begin, idx_end, cfg->grid.nindex)) return 1;
    SLB_CHECK(stats_dev != nullptr, "slb_value_operator: null stats");
    const int64_t n = idx_end - idx_begin;
    cudaStream_t st = (cudaStream_t)stream;
    SLB_CUDA(cudaMemsetAsync(stats_dev, 0, 4 * sizeof(uint64_t), st));
    if (n == 0) return 0;
    SLB_CHECK(cols_dev && weights_dev && rewards_dev, "slb_value_operator: null output");
    const int din = cfg->grid.ndim + m;
    int chunk_rows, nomax;
    const size_t smem = bellman_stage_config(*cfg, din, &chunk_rows, &nomax);
    const unsigned blocks = (unsigned)((n + VT - 1) / VT);
    const bool wide = wide_index(cfg->value.grid.nindex);
    unsigned long long* stats = reinterpret_cast<unsigned long long*>(stats_dev);
    return slb_dispatch_dim<2, 6>(din, "slb_value_operator: state+action dimension", [&](auto D) {
        if (wide) value_operator_kernel<D, int64_t><<<blocks, VT, smem, st>>>(
            *cfg, idx_begin, n, (int64_t*)cols_dev, weights_dev, rewards_dev, stats, chunk_rows, nomax);
        else value_operator_kernel<D, int32_t><<<blocks, VT, smem, st>>>(
            *cfg, idx_begin, n, (int32_t*)cols_dev, weights_dev, rewards_dev, stats, chunk_rows, nomax);
        SLB_LAUNCH_CHECK();
        return 0;
    });
}

int slb_value_operator_points(void* stream, const slb_function* value, const double* next_states_dev,
                              int64_t n, void* cols_dev, double* weights_dev, uint64_t* stats_dev) {
    SLB_CHECK(value != nullptr, "slb_value_operator_points: null value function");
    if (slb_validate_function(value, "value_function", 0)) return 1;
    if (validate_value_table(*value, "slb_value_operator_points")) return 1;
    SLB_CHECK(n >= 0, "slb_value_operator_points: negative n");
    SLB_CHECK(stats_dev != nullptr, "slb_value_operator_points: null stats");
    cudaStream_t st = (cudaStream_t)stream;
    SLB_CUDA(cudaMemsetAsync(stats_dev, 0, 4 * sizeof(uint64_t), st));
    if (n == 0) return 0;
    SLB_CHECK(next_states_dev && cols_dev && weights_dev, "slb_value_operator_points: null buffer");
    const unsigned blocks = (unsigned)((n + VT - 1) / VT);
    unsigned long long* stats = reinterpret_cast<unsigned long long*>(stats_dev);
    if (wide_index(value->grid.nindex))
        value_operator_points_kernel<int64_t><<<blocks, VT, 0, st>>>(*value, next_states_dev, n,
                                                                    (int64_t*)cols_dev, weights_dev, stats);
    else
        value_operator_points_kernel<int32_t><<<blocks, VT, 0, st>>>(*value, next_states_dev, n,
                                                                    (int32_t*)cols_dev, weights_dev, stats);
    SLB_LAUNCH_CHECK();
    return 0;
}

int64_t slb_value_solve_workspace(int64_t n, int32_t ncols) {
    if (n <= VS_SMALL_MAX || ncols < 2 || ncols > SLB_MAX_DIM + 1) return 0;     // one-CTA tier: none
    return n * (int64_t)sizeof(double) + 16 * (int64_t)sizeof(uint64_t);
}

int slb_value_solve(void* stream, int64_t n, int32_t ncols, const void* cols_dev, const double* weights_dev,
                    const double* rewards_dev, double gamma, double tol, int64_t max_iters,
                    double* v_inout_dev, void* workspace_dev, uint64_t* stats_dev) {
    SLB_CHECK(n >= 1, "slb_value_solve: need n >= 1 (got %lld)", (long long)n);
    SLB_CHECK(ncols >= 2 && ncols <= SLB_MAX_DIM + 1,
              "slb_value_solve: ncols %d outside 2..%d (dimension 1..%d)", ncols, SLB_MAX_DIM + 1,
              SLB_MAX_DIM);
    SLB_CHECK(gamma >= 0.0 && gamma < 1.0, "slb_value_solve: gamma %g outside [0, 1)", gamma);
    SLB_CHECK(tol > 0.0, "slb_value_solve: tol must be positive (got %g)", tol);
    SLB_CHECK(max_iters >= 1, "slb_value_solve: max_iters must be >= 1");
    SLB_CHECK(cols_dev && weights_dev && rewards_dev && v_inout_dev && stats_dev,
              "slb_value_solve: null buffer");
    SLB_CHECK(n <= VS_SMALL_MAX || workspace_dev != nullptr,
              "slb_value_solve: n = %lld needs a workspace of slb_value_solve_workspace bytes",
              (long long)n);
    const solve_args a = {n, ncols, gamma, tol, max_iters};
    cudaStream_t st = (cudaStream_t)stream;
    unsigned long long* stats = reinterpret_cast<unsigned long long*>(stats_dev);
    return wide_index(n) ? launch_solve<int64_t>(st, a, cols_dev, weights_dev, rewards_dev, v_inout_dev,
                                                  workspace_dev, stats)
                         : launch_solve<int32_t>(st, a, cols_dev, weights_dev, rewards_dev, v_inout_dev,
                                                  workspace_dev, stats);
}

}  // extern "C"
