// light.cu -- the bandwidth-/latency-bound kernels around the GP sweep, plus library plumbing:
//   deterministic-dynamics Lyapunov sweep      lyapunov.py:436-441 with a DeterministicFunction
//   first-fail reduction + prefix application   lyapunov.py:500-606 (sort-free, SURVEY.md Q1/Q4)
//   generic function evaluation                 Function.__call__, Lyapunov.update_values :305-322
//   GridWorld.index_to_state                    functions.py:714-731
//   Bellman sweep / argmax / max|dV|            reinforcement_learning.py:65-114,135-140,213-279
#include "common.cuh"
#include "bellman.cuh"

#include <float.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <atomic>

// ----------------------------------------------------------------------------- plumbing
static thread_local char g_err[512] = "";
static std::atomic<long long> g_slb_launches{0};
void slb_count_launch() { g_slb_launches.fetch_add(1, std::memory_order_relaxed); }

void slb_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int slb_validate_grid(const slb_grid* g, bool need_points) {
    SLB_CHECK(g->ndim >= 1 && g->ndim <= SLB_MAX_DIM, "grid ndim %d outside 1..%d", g->ndim,
              SLB_MAX_DIM);
    int64_t n = 1;
    for (int c = 0; c < g->ndim; ++c) {
        SLB_CHECK(g->num_points[c] >= 2, "grid needs >= 2 points per dimension (dim %d has %lld)",
                  c, (long long)g->num_points[c]);
        n *= g->num_points[c];
    }
    SLB_CHECK(n == g->nindex, "grid nindex %lld != prod(num_points) %lld", (long long)g->nindex,
              (long long)n);
    SLB_CHECK(!need_points || g->discrete_points != nullptr,
              "grid.discrete_points is required for a Triangulation");
    return 0;
}

int slb_validate_range(const char* who, int64_t idx_begin, int64_t idx_end, int64_t nindex) {
    SLB_CHECK(idx_begin >= 0 && idx_end >= idx_begin && idx_end <= nindex,
              "%s: index range [%lld, %lld) outside the grid (nindex %lld)", who, (long long)idx_begin,
              (long long)idx_end, (long long)nindex);
    return 0;
}

// SLB_FLAG_GRADIENT on a network with `outputs` outputs (network_input_gradient, common.cuh): x -> d f /
// d x has in_dim columns, and every kernel array that receives them before a reduction holds SLB_MAX_OUT
static int validate_network_gradient(const slb_function* f, const char* what, const char* name, int outputs) {
    SLB_CHECK(outputs == 1,
              "%s: the gradient flag needs a one-output %s; this one maps %d inputs to %d outputs (its "
              "derivative is a Jacobian)", what, name, f->in_dim, outputs);
    SLB_CHECK(f->in_dim <= SLB_MAX_OUT,
              "%s: the gradient of a %s with %d inputs and %d output has more than SLB_MAX_OUT = %d columns",
              what, name, f->in_dim, outputs, SLB_MAX_OUT);
    SLB_CHECK(f->out_dim == f->in_dim, "%s: the gradient of a %s with %d inputs and %d output needs out_dim %d, "
              "got %d", what, name, f->in_dim, outputs, f->in_dim, f->out_dim);
    return 0;
}

int slb_validate_function(const slb_function* f, const char* what, int expect_in) {
    SLB_CHECK(!(f->flags & SLB_FLAG_GRADIENT) || f->kind == SLB_FN_TRIANGULATION || f->kind == SLB_FN_LYAPUNOV_NN ||
              f->kind == SLB_FN_MLP,
              "%s: the gradient flag is only defined for Triangulation, LyapunovNetwork and one-output "
              "NeuralNetwork (kind %d)", what, f->kind);
    const bool grad = (f->flags & SLB_FLAG_GRADIENT) != 0;
    SLB_CHECK(!((f->flags & SLB_FLAG_NORM1) && (f->flags & SLB_FLAG_MAXABS)),
              "%s: norm1 and maxabs reductions are exclusive", what);
    switch (f->kind) {
    case SLB_FN_NONE:
        return 0;
    case SLB_FN_CONSTANT:
        SLB_CHECK(f->out_dim >= 1 && f->out_dim <= SLB_MAX_OUT, "%s: constant out_dim %d", what,
                  f->out_dim);
        return 0;
    case SLB_FN_LINEAR:
        SLB_CHECK(f->matrix != nullptr, "%s: LinearSystem without matrix", what);
        SLB_CHECK(f->out_dim >= 1 && f->out_dim <= SLB_MAX_OUT && f->in_dim >= 1 &&
                  f->in_dim <= SLB_MAX_IN, "%s: LinearSystem shape [%d,%d] unsupported", what,
                  f->out_dim, f->in_dim);
        break;
    case SLB_FN_QUADRATIC:
        SLB_CHECK(f->matrix != nullptr, "%s: QuadraticFunction without matrix", what);
        SLB_CHECK(f->in_dim >= 1 && f->in_dim <= SLB_MAX_IN, "%s: quadratic dim %d unsupported",
                  what, f->in_dim);
        break;
    case SLB_FN_TRIANGULATION:
        if (slb_validate_grid(&f->grid, true)) return 1;
        SLB_CHECK(f->matrix && f->hyperplanes && f->unit_simplices && f->nsimplex >= 1,
                  "%s: Triangulation tables missing", what);
        SLB_CHECK(f->in_dim == f->grid.ndim, "%s: Triangulation in_dim %d != grid ndim %d", what,
                  f->in_dim, f->grid.ndim);
        SLB_CHECK(f->out_dim >= 1 && f->out_dim <= SLB_MAX_OUT, "%s: Triangulation out_dim %d",
                  what, f->out_dim);
        SLB_CHECK(!(f->flags & SLB_FLAG_GRADIENT) || f->out_dim == f->grid.ndim,
                  "%s: Triangulation gradient needs one value column and out_dim = ndim (%d), got %d",
                  what, f->grid.ndim, f->out_dim);
        break;
    case SLB_FN_PIECEWISE_CONSTANT:
        if (slb_validate_grid(&f->grid, false)) return 1;
        SLB_CHECK(f->matrix != nullptr, "%s: PiecewiseConstant without vertex values", what);
        SLB_CHECK(f->in_dim == f->grid.ndim, "%s: PiecewiseConstant in_dim %d != grid ndim %d", what,
                  f->in_dim, f->grid.ndim);
        SLB_CHECK(f->out_dim >= 1 && f->out_dim <= SLB_MAX_OUT, "%s: PiecewiseConstant out_dim %d", what,
                  f->out_dim);
        SLB_CHECK(!(f->flags & SLB_FLAG_PROJECT), "%s: PiecewiseConstant clips by itself (no projection flag)",
                  what);
        for (int c = 0; c < f->grid.ndim; ++c)
            SLB_CHECK(f->cparams[c] > 0.0 && f->cparams[c] < INFINITY,
                      "%s: PiecewiseConstant needs cparams[%d] = 1 / unit_maxes, positive and finite (got %g)",
                      what, c, f->cparams[c]);
        break;
    case SLB_FN_PENDULUM:
        SLB_CHECK(f->in_dim == 3 && f->out_dim == 2, "%s: pendulum must map 3 -> 2", what);
        break;
    case SLB_FN_CARTPOLE:
        SLB_CHECK(f->in_dim == 5 && f->out_dim == 4, "%s: cart-pole must map 5 -> 4", what);
        break;
    case SLB_FN_VANDERPOL:
        SLB_CHECK(f->in_dim == 3 && f->out_dim == 2, "%s: Van der Pol must map 3 -> 2", what);
        break;
    case SLB_FN_LYAPUNOV_NN:
    case SLB_FN_MLP: {        // LyapunovNetwork has one output, NeuralNetwork its last layer's width
        const char* name = f->kind == SLB_FN_MLP ? "NeuralNetwork" : "LyapunovNetwork";
        SLB_CHECK(f->matrix != nullptr, "%s: %s without parameters", what, name);
        const int layers = nn_layers(*f);
        SLB_CHECK(layers >= 1 && layers <= SLB_NN_MAX_LAYERS, "%s: %s with %d layers (1..%d)", what, name,
                  layers, SLB_NN_MAX_LAYERS);
        SLB_CHECK(f->in_dim >= 1 && f->in_dim <= SLB_MAX_IN, "%s: %s input dim %d outside 1..%d", what, name,
                  f->in_dim, SLB_MAX_IN);
        for (int l = 1; l <= layers; ++l)
            SLB_CHECK(nn_width(*f, l) >= 1 && nn_width(*f, l) <= SLB_NN_MAX_WIDTH,
                      "%s: %s layer %d width %d outside 1..%d", what, name, l - 1, nn_width(*f, l),
                      SLB_NN_MAX_WIDTH);
        const int outputs = f->kind == SLB_FN_MLP ? nn_width(*f, layers) : 1;
        if (grad) {
            if (validate_network_gradient(f, what, name, outputs)) return 1;
        } else {
            SLB_CHECK(f->out_dim == outputs && outputs <= SLB_MAX_OUT,
                      "%s: %s with %d outputs needs out_dim %d (<= %d), got %d", what, name, outputs, outputs,
                      SLB_MAX_OUT, f->out_dim);
        }
        break;
    }
    default:
        slb_set_error("%s: function kind %d is not implemented in this build", what, f->kind);
        return 1;
    }
    SLB_CHECK(expect_in <= 0 || f->in_dim == expect_in, "%s: expects %d inputs, function takes %d",
              what, expect_in, f->in_dim);
    return 0;
}

// The columns eval_fn (common.cuh) returns for f: the kind's count, then 1 after NORM1 / MAXABS.
// A network gradient (SLB_FLAG_GRADIENT on LYAPUNOV_NN / MLP with out_dim = in_dim, the shape
// slb_validate_function requires) returns in_dim; a network descriptor that validation rejects keeps its
// kind's count.  Host code (and Python, through slb_function_columns) sizes kernels and checks shapes
// with this number and never with out_dim: a change to eval_fn's return value must be made here too.
int slb_fn_columns(const slb_function& f) {
    if (f.flags & (SLB_FLAG_NORM1 | SLB_FLAG_MAXABS)) return 1;
    switch (f.kind) {
    case SLB_FN_LYAPUNOV_NN: case SLB_FN_MLP:
        if ((f.flags & SLB_FLAG_GRADIENT) && f.out_dim == f.in_dim) return f.in_dim;
        return f.kind == SLB_FN_MLP ? f.out_dim : 1;
    case SLB_FN_QUADRATIC: return 1;
    case SLB_FN_PENDULUM: case SLB_FN_VANDERPOL: return 2;
    case SLB_FN_CARTPOLE: return 4;
    default: return f.out_dim;
    }
}

// deterministic dynamics: [x, u] (d + m inputs) -> the next state (d columns)
int slb_validate_dynamics(const slb_function* f, const char* who, int d, int m) {
    if (slb_validate_function(f, "dynamics", d + m)) return 1;
    SLB_CHECK(f->kind != SLB_FN_NONE, "%s: no dynamics given", who);
    SLB_CHECK(slb_fn_columns(*f) == d, "%s: dynamics return %d columns, the state has %d", who,
              slb_fn_columns(*f), d);
    return 0;
}

int slb_validate_kernel(const slb_kernel& K, int d_in, const char* who) {
    SLB_CHECK(K.num_prims >= 0 && K.num_prims <= SLB_MAX_KPRIM,
              "%s: %d kernel primitives outside 0..%d", who, K.num_prims, SLB_MAX_KPRIM);
    for (int i = 0; i < K.num_prims; ++i) {
        const slb_kernel_prim& P = K.prims[i];
        SLB_CHECK(P.kind >= SLB_K_RBF && P.kind <= SLB_K_WHITE,
                  "%s: kernel primitive %d has unknown kind %d", who, i, P.kind);
        const int prev = i == 0 ? 0 : K.prims[i - 1].term;
        SLB_CHECK(P.term == prev || P.term == prev + 1,
                  "%s: kernel primitives must be listed in term order", who);
        SLB_CHECK(i > 0 || P.term == 0, "%s: kernel terms start at 0", who);
        for (int c = 0; c < d_in; ++c)
            SLB_CHECK(P.w[c] >= 0.0, "%s: kernel primitive %d has a negative weight", who, i);
    }
    return 0;
}

int slb_validate_gp(const slb_gp_stack* gp) {
    if (gp->num_outputs == 0) return 0;
    SLB_CHECK(gp->num_outputs >= 1 && gp->num_outputs <= SLB_MAX_OUT, "GP outputs %d outside 1..%d",
              gp->num_outputs, SLB_MAX_OUT);
    SLB_CHECK(gp->num_factors >= 1 && gp->num_factors <= gp->num_outputs,
              "GP factors %d inconsistent with %d outputs", gp->num_factors, gp->num_outputs);
    SLB_CHECK(gp->input_dim >= 1 && gp->input_dim <= SLB_MAX_IN, "GP input_dim %d unsupported",
              gp->input_dim);
    for (int f = 0; f < gp->num_factors; ++f) {
        const slb_gp_factor& F = gp->factors[f];
        SLB_CHECK(F.M >= 0 && F.nrb == (F.M + 7) / 8, "GP factor %d: bad M/nrb (%d/%d)", f, F.M,
                  F.nrb);
        SLB_CHECK(F.M == 0 || (F.Xs != nullptr && F.Wpack != nullptr), "GP factor %d: null table", f);
        SLB_CHECK(F.scale > 0.0, "GP factor %d: scale must be positive", f);
        char who[32];
        snprintf(who, sizeof(who), "GP factor %d", f);
        if (slb_validate_kernel(F.kernel, gp->input_dim, who)) return 1;
        if (F.kernel.num_prims == 0) {
            for (int c = 0; c < gp->input_dim; ++c)
                SLB_CHECK(F.lengthscales[c] > 0.0, "GP factor %d: lengthscale[%d] must be positive",
                          f, c);
        }
    }
    for (int o = 0; o < gp->num_outputs; ++o) {
        const slb_gp_output& G = gp->outputs[o];
        SLB_CHECK(G.factor >= 0 && G.factor < gp->num_factors, "GP output %d: bad factor index", o);
        SLB_CHECK(G.alpha != nullptr, "GP output %d: null alpha", o);
    }
    return 0;
}

// The staged GP mean (gp_mean_staged.cuh) copies Xf of every factor and gamma_f of every output by
// TMA bulk copies: wherever a factor has training points they must be present and 16-byte aligned.
int slb_validate_staged_tables(const slb_gp_stack* gp, const char* who) {
    auto aligned = [](const double* p) { return p != nullptr && (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
    for (int f = 0; f < gp->num_factors; ++f)
        SLB_CHECK(gp->factors[f].M == 0 || aligned(gp->factors[f].Xf),
                  "%s: GP factor %d lacks the (16-byte aligned) staged table Xf", who, f);
    for (int o = 0; o < gp->num_outputs; ++o)
        SLB_CHECK(gp->factors[gp->outputs[o].factor].M == 0 || aligned(gp->outputs[o].gamma_f),
                  "%s: GP output %d lacks the (16-byte aligned) staged table gamma_f", who, o);
    return 0;
}

int slb_validate_sweep(const slb_sweep* cfg, bool explicit_states, int* m_out) {
    SLB_CHECK(cfg != nullptr, "lyapunov sweep: null config");
    if (slb_validate_grid(&cfg->grid, false)) return 1;
    const int d = cfg->grid.ndim;
    if (slb_validate_function(&cfg->policy, "policy", d)) return 1;
    SLB_CHECK(cfg->policy.kind != SLB_FN_NONE, "lyapunov sweep: a policy is required");
    if (slb_validate_function(&cfg->lyapunov, "lyapunov_function", d)) return 1;
    SLB_CHECK(cfg->lyapunov.kind != SLB_FN_NONE, "lyapunov sweep: a Lyapunov function is required");
    if (slb_validate_function(&cfg->lipschitz_v, "lipschitz_lyapunov", d)) return 1;
    const int nl = slb_fn_columns(cfg->lipschitz_v);
    SLB_CHECK(cfg->lipschitz_v.kind == SLB_FN_NONE || nl == 1 || nl == d,
              "lyapunov sweep: lipschitz_lyapunov returns %d columns, expected 1 or the state's %d", nl, d);
    if (slb_validate_function(&cfg->lipschitz_f, "lipschitz_dynamics", d)) return 1;
    SLB_CHECK(cfg->lf_values == nullptr || !explicit_states,
              "lf_values (L_f tabulated per grid index) needs an index-range sweep");
    const int m = slb_fn_columns(cfg->policy);
    SLB_CHECK(m >= 1 && m <= SLB_MAX_ACT, "policy output dim %d unsupported", m);
    if (cfg->gp.num_outputs > 0) {
        if (slb_validate_gp(&cfg->gp)) return 1;
        SLB_CHECK(cfg->gp.num_outputs == d,
                  "GP stack has %d outputs but the state has %d dims", cfg->gp.num_outputs, d);
        SLB_CHECK(cfg->gp.input_dim == d + m, "GP input_dim %d != state %d + action %d",
                  cfg->gp.input_dim, d, m);
    } else if (slb_validate_dynamics(&cfg->dynamics, "lyapunov sweep", d, m)) {
        return 1;
    }
    *m_out = m;
    return 0;
}

int slb_validate_bellman(const slb_bellman* cfg, int* m_out) {
    SLB_CHECK(cfg != nullptr, "bellman: null config");
    if (slb_validate_grid(&cfg->grid, false)) return 1;
    const int d = cfg->grid.ndim;
    int m;
    if (cfg->fixed_action) {
        m = cfg->policy.out_dim;
        SLB_CHECK(m >= 1 && m <= SLB_MAX_ACT, "bellman: fixed action dim %d unsupported", m);
    } else {
        if (slb_validate_function(&cfg->policy, "policy", d)) return 1;
        SLB_CHECK(cfg->policy.kind != SLB_FN_NONE, "bellman: a policy is required");
        m = slb_fn_columns(cfg->policy);
        SLB_CHECK(m >= 1 && m <= SLB_MAX_ACT, "bellman: policy output dim %d unsupported", m);
    }
    if (cfg->gp.num_outputs > 0) {
        if (slb_validate_gp(&cfg->gp)) return 1;
        SLB_CHECK(cfg->gp.num_outputs == d && cfg->gp.input_dim == d + m,
                  "bellman: GP stack shape (%d outputs, %d inputs) does not match state %d + action %d",
                  cfg->gp.num_outputs, cfg->gp.input_dim, d, m);
        if (slb_validate_staged_tables(&cfg->gp, "bellman")) return 1;
    } else if (slb_validate_dynamics(&cfg->dynamics, "bellman", d, m)) {
        return 1;
    }
    if (slb_validate_function(&cfg->reward, "reward_function", d + m)) return 1;
    SLB_CHECK(cfg->reward.kind != SLB_FN_NONE, "bellman: a reward function is required");
    SLB_CHECK(slb_fn_columns(cfg->reward) == 1, "bellman: reward_function returns %d columns, expected 1",
              slb_fn_columns(cfg->reward));
    if (slb_validate_function(&cfg->value, "value_function", d)) return 1;
    SLB_CHECK(cfg->value.kind != SLB_FN_NONE, "bellman: a value function is required");
    SLB_CHECK(slb_fn_columns(cfg->value) == 1, "bellman: value_function returns %d columns, expected 1",
              slb_fn_columns(cfg->value));
    *m_out = m;
    return 0;
}

// ----------------------------------------------------------------------------- kernels
namespace {

constexpr int LT = 256;

__global__ void __launch_bounds__(LT)
det_sweep_kernel(const __grid_constant__ slb_sweep cfg, const double* __restrict__ states, int64_t n,
                 int64_t idx_begin, uint8_t* __restrict__ negative, double* __restrict__ values,
                 double* __restrict__ decrease, double* __restrict__ threshold,
                 double* __restrict__ mean) {
    const int64_t i = (int64_t)blockIdx.x * LT + threadIdx.x;
    if (i >= n) return;
    const int d = cfg.grid.ndim;
    double z[SLB_MAX_IN], u[SLB_MAX_OUT], mu[SLB_MAX_OUT];
    if (states != nullptr) {
        for (int c = 0; c < d; ++c) z[c] = states[i * d + c];
    } else {
        grid_index_to_state(cfg.grid, idx_begin + i, z);
    }
    const int m = eval_fn(cfg.policy, z, u);
    for (int c = 0; c < m; ++c) z[d + c] = u[c];
    eval_fn(cfg.dynamics, z, mu);
    const slb_decision r = lyapunov_decide(cfg, z, states != nullptr ? -1 : idx_begin + i, mu, nullptr);
    negative[i] = r.negative ? 1 : 0;
    if (values != nullptr) values[i] = r.vx;
    if (decrease != nullptr) decrease[i] = r.decrease;
    if (threshold != nullptr) threshold[i] = r.threshold;
    if (mean != nullptr) for (int c = 0; c < d; ++c) mean[i * d + c] = mu[c];
}

// ---- deterministic-dynamics sweep, specialised ---------------------------------------------------
// The same decision as det_sweep_kernel for the composition of the reference's LQR experiments
// (SURVEY.md section 8d, deterministic variant of C2 / C5): d = 2, m = 1, policy = Saturation(
// LinearSystem), dynamics = LinearSystem on [x, u], V = QuadraticFunction, L_V = a constant or
// abs(LinearSystem) (one- or two-column), scalar L_f.  det_sweep_kernel interprets generic
// descriptors through local-memory operand arrays (1.6 KB stack, 64-bit index division, one byte
// written per thread); here the operands live in registers, the index
// arithmetic is one 32-bit division per 8 points and the 8 flags leave as one 8-byte store.  The
// arithmetic is eval_fn's, operation for operation (__dmul_rn / __dadd_rn, same order): bit-exact.
struct det_fast_params {
    const double* k;                   // policy row [2] (device)
    const double* a;                   // dynamics rows on [x0, x1, u]: [2][3]
    const double* p;                   // V's matrix [2][2]
    const double* lv;                  // L_V rows [lv_kind][2] (lv_kind 1, 2)
    double klo, khi;                   // saturation bounds
    double lv_const, lf, tau;
    int lv_kind;                       // 0: constant, 1: one abs-linear column, 2: two, 1-norm
    int lv_abs;                        // columns pass through fabs (SLB_FLAG_ABS | NORM1)
};

SLB_DEV double quad2(const double (&p)[2][2], double x0, double x1) {
    const double l0 = f64add(f64mul(x0, p[0][0]), f64mul(x1, p[1][0]));
    const double l1 = f64add(f64mul(x0, p[0][1]), f64mul(x1, p[1][1]));
    return f64add(f64mul(l0, x0), f64mul(l1, x1));
}

constexpr int DF_PTS = 8;              // points per thread (consecutive along the last grid axis)

__global__ void __launch_bounds__(LT)
det_sweep_fast_kernel(const __grid_constant__ slb_grid g, const det_fast_params qp, int64_t idx_begin,
                      int64_t n, uint8_t* __restrict__ negative, double* __restrict__ values) {
    const int64_t first = ((int64_t)blockIdx.x * LT + threadIdx.x) * DF_PTS;
    if (first >= n) return;
    // operand tables -> registers (warp-uniform loads, served by L1 after the first warp)
    struct { double k[2], a[2][3], p[2][2], lv[2][2], klo, khi, lv_const, lf, tau; int lv_kind, lv_abs; } q;
    q.k[0] = __ldg(qp.k); q.k[1] = __ldg(qp.k + 1);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
#pragma unroll
        for (int c = 0; c < 3; ++c) q.a[r][c] = __ldg(qp.a + 3 * r + c);
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            q.p[r][c] = __ldg(qp.p + 2 * r + c);
            q.lv[r][c] = r < qp.lv_kind ? __ldg(qp.lv + 2 * r + c) : 0.0;
        }
    }
    q.klo = qp.klo; q.khi = qp.khi; q.lv_const = qp.lv_const; q.lf = qp.lf; q.tau = qp.tau;
    q.lv_kind = qp.lv_kind; q.lv_abs = qp.lv_abs;
    const unsigned n1 = (unsigned)g.num_points[1];
    const unsigned flat = (unsigned)(idx_begin + first);
    unsigned i0 = flat / n1, i1 = flat - i0 * n1;
    unsigned long long flags = 0;
    const int count = (int)min((int64_t)DF_PTS, n - first);
#pragma unroll
    for (int t = 0; t < DF_PTS; ++t) {
        if (t < count) {
            const double x0 = f64add(f64mul((double)i0, g.unit_maxes[0]), g.offset[0]);
            const double x1 = f64add(f64mul((double)i1, g.unit_maxes[1]), g.offset[1]);
            double u = f64add(f64mul(x0, q.k[0]), f64mul(x1, q.k[1]));
            u = fmin(fmax(u, q.klo), q.khi);
            const double m0 = f64add(f64add(f64mul(x0, q.a[0][0]), f64mul(x1, q.a[0][1])), f64mul(u, q.a[0][2]));
            const double m1 = f64add(f64add(f64mul(x0, q.a[1][0]), f64mul(x1, q.a[1][1])), f64mul(u, q.a[1][2]));
            const double vx = quad2(q.p, x0, x1);
            const double vm = quad2(q.p, m0, m1);
            double lvx = q.lv_const;
            if (q.lv_kind >= 1) {
                double c0 = f64add(f64mul(x0, q.lv[0][0]), f64mul(x1, q.lv[0][1]));
                if (q.lv_abs) c0 = fabs(c0);
                lvx = c0;
                if (q.lv_kind == 2) {
                    const double c1 = f64add(f64mul(x0, q.lv[1][0]), f64mul(x1, q.lv[1][1]));
                    lvx = f64add(fabs(c0), fabs(c1));          // 1-norm of a vector-valued L_V (:284-286)
                }
            }
            const double thr = f64mul(f64mul(-lvx, f64add(1.0, q.lf)), q.tau);
            const double dec = f64add(f64sub(vm, vx), 0.0);     // lyapunov_combine with bound = 0
            if (dec < thr) flags |= 1ull << (8 * t);
            if (values != nullptr) values[first + t] = vx;
            if (++i1 == n1) { i1 = 0; ++i0; }
        }
    }
    if (count == DF_PTS && ((reinterpret_cast<uintptr_t>(negative) + first) & 7) == 0) {
        *reinterpret_cast<unsigned long long*>(negative + first) = flags;
    } else {
        for (int t = 0; t < count; ++t) negative[first + t] = (uint8_t)((flags >> (8 * t)) & 1);
    }
}

// host: does the sweep match the specialised composition?  Fills `q` from the device tables.
bool det_fast_applicable(const slb_sweep& cfg, const double* states, const double* decrease,
                         const double* threshold, const double* mean) {
    if (states || decrease || threshold || mean) return false;
    if (cfg.grid.ndim != 2 || cfg.grid.nindex > 0x7fffffffll) return false;
    const slb_function& P = cfg.policy, &F = cfg.dynamics, &V = cfg.lyapunov, &L = cfg.lipschitz_v;
    if (P.kind != SLB_FN_LINEAR || P.in_dim != 2 || P.out_dim != 1 || (P.flags & ~SLB_FLAG_SATURATE))
        return false;
    if (F.kind != SLB_FN_LINEAR || F.in_dim != 3 || F.out_dim != 2 || F.flags) return false;
    if (V.kind != SLB_FN_QUADRATIC || V.in_dim != 2 || V.flags) return false;
    if (cfg.lf_values != nullptr || cfg.lipschitz_f.kind != SLB_FN_NONE) return false;
    if (L.kind == SLB_FN_NONE) return true;
    if (L.kind != SLB_FN_LINEAR || L.in_dim != 2 || L.out_dim < 1 || L.out_dim > 2) return false;
    // one column: plain or abs; two columns reduce with the 1-norm in threshold() either way
    return (L.flags & ~(SLB_FLAG_ABS | SLB_FLAG_NORM1)) == 0;
}

__global__ void __launch_bounds__(LT)
eval_function_kernel(const __grid_constant__ slb_function fn, const double* __restrict__ points,
                     int64_t n, double* __restrict__ out, int ncols) {
    const int64_t i = (int64_t)blockIdx.x * LT + threadIdx.x;
    if (i >= n) return;
    double in[SLB_MAX_IN], o[SLB_MAX_OUT];
    for (int c = 0; c < fn.in_dim; ++c) in[c] = points[i * fn.in_dim + c];
    eval_fn(fn, in, o);
    for (int c = 0; c < ncols; ++c) out[i * ncols + c] = o[c];
}

__global__ void __launch_bounds__(LT)
index_to_state_kernel(const __grid_constant__ slb_grid g, int64_t idx_begin, int64_t n,
                      double* __restrict__ states) {
    const int64_t i = (int64_t)blockIdx.x * LT + threadIdx.x;
    if (i >= n) return;
    double x[SLB_MAX_DIM];
    grid_index_to_state(g, idx_begin + i, x);
    for (int c = 0; c < g.ndim; ++c) states[i * g.ndim + c] = x[c];
}

// ---- first-fail reduction ----------------------------------------------------------------
struct ff_partial { uint64_t kv; int64_t ki; int64_t nok; int64_t pad; };

SLB_DEV bool key_less(uint64_t av, int64_t ai, uint64_t bv, int64_t bi) {
    return av < bv || (av == bv && ai < bi);
}

SLB_DEV void ff_block_reduce(uint64_t& kv, int64_t& ki, int64_t& nok) {
    __shared__ uint64_t s_kv[32];
    __shared__ int64_t s_ki[32];
    __shared__ int64_t s_n[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        const uint64_t ov = __shfl_xor_sync(0xffffffffu, kv, off);
        const int64_t oi = __shfl_xor_sync(0xffffffffu, ki, off);
        nok += __shfl_xor_sync(0xffffffffu, nok, off);
        if (key_less(ov, oi, kv, ki)) { kv = ov; ki = oi; }
    }
    if (lane == 0) { s_kv[warp] = kv; s_ki[warp] = ki; s_n[warp] = nok; }
    __syncthreads();
    if (warp == 0) {
        const int nw = (blockDim.x + 31) >> 5;
        kv = lane < nw ? s_kv[lane] : ~0ull;
        ki = lane < nw ? s_ki[lane] : INT64_MAX;
        nok = lane < nw ? s_n[lane] : 0;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const uint64_t ov = __shfl_xor_sync(0xffffffffu, kv, off);
            const int64_t oi = __shfl_xor_sync(0xffffffffu, ki, off);
            nok += __shfl_xor_sync(0xffffffffu, nok, off);
            if (key_less(ov, oi, kv, ki)) { kv = ov; ki = oi; }
        }
    }
}

constexpr int FF_BLOCKS = 1024;

__global__ void __launch_bounds__(LT)
first_fail_partial_kernel(const double* __restrict__ values, const uint8_t* __restrict__ negative,
                          const uint8_t* __restrict__ initial, int64_t n, int64_t idx_begin,
                          ff_partial* __restrict__ partial) {
    uint64_t kv = ~0ull;
    int64_t ki = INT64_MAX, nok = 0;
    for (int64_t i = (int64_t)blockIdx.x * LT + threadIdx.x; i < n; i += (int64_t)gridDim.x * LT) {
        const bool ok = negative[i] != 0 || (initial != nullptr && initial[i] != 0);
        if (ok) {
            ++nok;
        } else {
            const uint64_t v = value_key(values[i]);
            const int64_t gi = idx_begin + i;
            if (key_less(v, gi, kv, ki)) { kv = v; ki = gi; }
        }
    }
    ff_block_reduce(kv, ki, nok);
    if (threadIdx.x == 0) { partial[blockIdx.x].kv = kv; partial[blockIdx.x].ki = ki;
                            partial[blockIdx.x].nok = nok; }
}

// Peer-memory key exchange (slb_exchange, slb200.h).  The payload words are written with plain
// system-scope stores, the sequence number behind a system-scope fence is the release flag.
SLB_DEV void st_sys(int64_t* p, int64_t v) {
    asm volatile("st.relaxed.sys.global.s64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
SLB_DEV void st_release_sys(int64_t* p, int64_t v) {
    asm volatile("st.release.sys.global.s64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
SLB_DEV int64_t ld_sys(const int64_t* p) {
    int64_t v;
    asm volatile("ld.relaxed.sys.global.s64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
SLB_DEV int64_t ld_acquire_sys(const int64_t* p) {
    int64_t v;
    asm volatile("ld.acquire.sys.global.s64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

__global__ void __launch_bounds__(FF_BLOCKS)
first_fail_final_kernel(const ff_partial* __restrict__ partial, int nparts,
                        slb_fail_key* __restrict__ result, const slb_exchange x) {
    __shared__ int64_t s_key[4];
    uint64_t kv = ~0ull;
    int64_t ki = INT64_MAX, nok = 0;
    if ((int)threadIdx.x < nparts) {
        kv = partial[threadIdx.x].kv; ki = partial[threadIdx.x].ki; nok = partial[threadIdx.x].nok;
    }
    ff_block_reduce(kv, ki, nok);
    if (threadIdx.x == 0) {
        result->key_value = kv; result->key_index = ki; result->n_ok = nok; result->_pad = 0;
        if (x.world > 1) {
            const int64_t seq = *x.seq_dev + 1;       // sweeps issued by this rank, this one included
            *x.seq_dev = seq;
            s_key[0] = (int64_t)kv; s_key[1] = ki; s_key[2] = nok; s_key[3] = seq;
        }
    }
    if (x.world <= 1) return;
    __syncthreads();
    // push: thread r stores this rank's key into slot [parity][rank] of rank r (its own included)
    if ((int)threadIdx.x < x.world) {
        const int64_t seq = s_key[3];
        int64_t* slot = reinterpret_cast<int64_t*>(
            x.slots[threadIdx.x] + (seq & 1) * x.world + x.rank);
        st_sys(slot + 0, s_key[0]);
        st_sys(slot + 1, s_key[1]);
        st_sys(slot + 2, s_key[2]);
        st_release_sys(slot + 3, seq);
    }
}

// Lexicographic min over the per-rank keys gathered by the caller's all-gather.
__global__ void combine_fail_keys_kernel(const slb_fail_key* __restrict__ gathered, int world,
                                         slb_fail_key* __restrict__ out) {
    if (threadIdx.x != 0) return;
    uint64_t kv = ~0ull;
    int64_t ki = INT64_MAX, nok = 0;
    for (int r = 0; r < world; ++r) {
        nok += gathered[r].n_ok;
        if (key_less(gathered[r].key_value, gathered[r].key_index, kv, ki)) {
            kv = gathered[r].key_value; ki = gathered[r].key_index;
        }
    }
    out->key_value = kv; out->key_index = ki; out->n_ok = nok; out->_pad = 0;
}

// X: the keys of all ranks arrive through peer memory (slb_exchange); every block waits for the
// `world` release flags of the current sweep in this rank's own slot array (local HBM/L2), reduces
// the keys (lexicographic min, n_ok sum) and block 0 publishes the winner to `key`.  A rank whose
// peer does not show up within ~10 s gives up and marks the result (key->_pad = -1).
// fold != nullptr (single process, slb_safe_set_step): the key comes from the record the decision kernels
// folded it into, block 0 publishes it to `key`; the statistics are added up in the record (zeroed with it)
// and the last block to finish copies them to `stats`.
template <bool X>
__global__ void __launch_bounds__(LT)
apply_prefix_kernel(const double* __restrict__ values, const uint8_t* __restrict__ initial, int64_t n,
                    int64_t idx_begin, slb_fail_key* __restrict__ key,
                    uint8_t* __restrict__ safe, slb_prefix_stats* __restrict__ stats,
                    const slb_exchange x, slb_fold* __restrict__ fold) {
    uint64_t kv;
    int64_t ki;
    if (fold != nullptr) {
        kv = ~fold->hi;
        ki = INT64_MAX - (int64_t)fold->lo;
        if (blockIdx.x == 0 && threadIdx.x == 0) {
            key->key_value = kv; key->key_index = ki; key->n_ok = (int64_t)fold->n_ok; key->_pad = 0;
        }
    } else if (X) {
        __shared__ int64_t s_k[SLB_MAX_RANKS][3];
        __shared__ int s_timeout;
        if (threadIdx.x == 0) s_timeout = 0;
        __syncthreads();
        const int64_t seq = *x.seq_dev;
        if ((int)threadIdx.x < x.world) {
            const int64_t* slot = reinterpret_cast<const int64_t*>(
                x.slots[x.rank] + (seq & 1) * x.world + threadIdx.x);
            unsigned long long t0, t1;
            asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t0));
            while (ld_acquire_sys(slot + 3) != seq) {
                asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t1));
                if (t1 - t0 > 10000000000ull) { s_timeout = 1; break; }
                __nanosleep(64);
            }
            s_k[threadIdx.x][0] = ld_sys(slot + 0);
            s_k[threadIdx.x][1] = ld_sys(slot + 1);
            s_k[threadIdx.x][2] = ld_sys(slot + 2);
        }
        __syncthreads();
        kv = ~0ull; ki = INT64_MAX;
        int64_t nok = 0;
        for (int r = 0; r < x.world; ++r) {
            nok += s_k[r][2];
            if (key_less((uint64_t)s_k[r][0], s_k[r][1], kv, ki)) { kv = (uint64_t)s_k[r][0]; ki = s_k[r][1]; }
        }
        if (blockIdx.x == 0 && threadIdx.x == 0) {
            key->key_value = kv; key->key_index = ki; key->n_ok = nok;
            key->_pad = s_timeout ? -1 : seq;
        }
    } else {
        kv = key->key_value;
        ki = key->key_index;
    }
    unsigned long long n_safe = 0, n_below = 0, max_below = 0, max_all = 0;
    for (int64_t i = (int64_t)blockIdx.x * LT + threadIdx.x; i < n; i += (int64_t)gridDim.x * LT) {
        const uint64_t v = value_key(values[i]);
        const bool below = key_less(v, idx_begin + i, kv, ki);
        const bool s = below || (initial != nullptr && initial[i] != 0);
        safe[i] = s ? 1 : 0;
        n_safe += s;
        n_below += below;
        if (below && v > max_below) max_below = v;
        if (v > max_all) max_all = v;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        n_safe += __shfl_xor_sync(0xffffffffu, n_safe, off);
        n_below += __shfl_xor_sync(0xffffffffu, n_below, off);
        const unsigned long long mb = __shfl_xor_sync(0xffffffffu, max_below, off);
        const unsigned long long ma = __shfl_xor_sync(0xffffffffu, max_all, off);
        if (mb > max_below) max_below = mb;
        if (ma > max_all) max_all = ma;
    }
    // block-level combine in shared memory, then four global atomics per block (one set per warp put
    // 8192 same-address atomics behind a 64 K-point sweep)
    __shared__ unsigned long long s_acc[4];
    if (threadIdx.x < 4) s_acc[threadIdx.x] = 0ull;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(&s_acc[0], n_safe);
        atomicAdd(&s_acc[1], n_below);
        atomicMax(&s_acc[2], max_below);
        atomicMax(&s_acc[3], max_all);
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    if (fold == nullptr) {
        atomicAdd(reinterpret_cast<unsigned long long*>(&stats->n_safe), s_acc[0]);
        atomicAdd(reinterpret_cast<unsigned long long*>(&stats->n_below), s_acc[1]);
        atomicMax(reinterpret_cast<unsigned long long*>(&stats->max_below), s_acc[2]);
        atomicMax(reinterpret_cast<unsigned long long*>(&stats->max_all), s_acc[3]);
        return;
    }
    unsigned long long* acc = fold->acc;
    atomicAdd(acc + 0, s_acc[0]);
    atomicAdd(acc + 1, s_acc[1]);
    atomicMax(acc + 2, s_acc[2]);
    atomicMax(acc + 3, s_acc[3]);
    __threadfence();
    if (atomicAdd(&fold->ticket, 1u) != gridDim.x - 1) return;
    __threadfence();
    stats->n_safe = (int64_t)__ldcg(acc + 0);
    stats->n_below = (int64_t)__ldcg(acc + 1);
    stats->max_below = __ldcg(acc + 2);
    stats->max_all = __ldcg(acc + 3);
}

// ---- Bellman sweep (bellman.cuh) ----------------------------------------------------------
template <int DIN>
__global__ void __launch_bounds__(LT, 2)
bellman_kernel(const __grid_constant__ slb_bellman cfg, int64_t idx_begin, int64_t n,
               double* __restrict__ out, int chunk_rows, int nomax) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    bellman_smem S;
    bellman_setup<DIN>(S, smem_raw, cfg, chunk_rows, nomax);
    const int64_t i0 = (int64_t)blockIdx.x * LT + threadIdx.x;
    const bool valid = i0 < n;
    const int64_t i = valid ? i0 : n - 1;       // every thread stays for the block barriers
    double x[SLB_MAX_DIM], u[SLB_MAX_OUT];
    grid_index_to_state(cfg.grid, idx_begin + i, x);
    int m;
    if (cfg.fixed_action) {
        m = cfg.policy.out_dim;
        for (int c = 0; c < m; ++c) u[c] = cfg.action[c];
    } else {
        m = eval_fn(cfg.policy, x, u);
    }
    const double v = bellman_value<DIN>(cfg, x, u, m, S);
    if (valid) out[i] = v;
}

template <int DIN>
__global__ void __launch_bounds__(LT, 2)
bellman_argmax_kernel(const __grid_constant__ slb_bellman cfg, int64_t idx_begin, int64_t n,
                      const double* __restrict__ actions, int n_actions, int m,
                      const double* __restrict__ constraint, int32_t* __restrict__ best,
                      double* __restrict__ best_value, int chunk_rows, int nomax) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    bellman_smem S;
    bellman_setup<DIN>(S, smem_raw, cfg, chunk_rows, nomax);
    const int64_t i0 = (int64_t)blockIdx.x * LT + threadIdx.x;
    const bool valid = i0 < n;
    const int64_t i = valid ? i0 : n - 1;       // every thread stays for the block barriers
    double x[SLB_MAX_DIM], u[SLB_MAX_ACT];
    grid_index_to_state(cfg.grid, idx_begin + i, x);
    int arg = 0;
    double vmax = 0.0;
    for (int a = 0; a < n_actions; ++a) {
        for (int c = 0; c < m; ++c) u[c] = actions[a * m + c];
        double v = bellman_value<DIN>(cfg, x, u, m, S);
        if (constraint != nullptr && constraint[(int64_t)a * n + i] < 0.0) v = -INFINITY;  // :272-275
        // np.argmax (:278): first maximum, and NaN counts as the maximum (first NaN wins)
        if (a == 0 || v > vmax || (v != v && vmax == vmax)) { vmax = v; arg = a; }
    }
    if (valid) {
        best[i] = arg;
        if (best_value != nullptr) best_value[i] = vmax;
    }
}

__global__ void __launch_bounds__(LT)
max_abs_diff_kernel(const double* __restrict__ a, const double* __restrict__ b, int64_t n,
                    unsigned long long* __restrict__ result) {
    double m = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * LT + threadIdx.x; i < n; i += (int64_t)gridDim.x * LT) {
        const double dlt = fabs(a[i] - b[i]);
        if (dlt > m || dlt != dlt) m = dlt;
    }
    unsigned long long bits = (unsigned long long)__double_as_longlong(m);   // m >= 0 or NaN
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        const unsigned long long o = __shfl_xor_sync(0xffffffffu, bits, off);
        if (o > bits) bits = o;
    }
    if ((threadIdx.x & 31) == 0) atomicMax(result, bits);
}

// ---- head subset of the decision filter: first r pivots of the pivoted Cholesky factorisation ----
// One CTA.  Step t: pivot = argmax of the remaining diagonal (ties: lowest index), column t of the
// partial factor  low[:, t] = (K[:, pivot] - low[:, :t] low[pivot, :t]) / sqrt(diag[pivot]),
// diag -= low[:, t]^2.  K is symmetric: its row `pivot` is read instead of the column (coalesced).
constexpr int PV_THREADS = 1024;

__global__ void __launch_bounds__(PV_THREADS)
pivoted_subset_kernel(const double* __restrict__ K, int M, int r, int64_t* __restrict__ picks,
                      double* __restrict__ low, double* __restrict__ diag) {
    __shared__ double s_val[32];
    __shared__ int s_idx[32];
    __shared__ double s_prow[SLB_HEAD_RANK];
    __shared__ int s_piv;
    __shared__ double s_dpiv;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int i = tid; i < M; i += PV_THREADS) diag[i] = K[(size_t)i * M + i];
    __syncthreads();
    for (int t = 0; t < r; ++t) {
        double bv = -INFINITY;
        int bi = 0x7fffffff;
        for (int i = tid; i < M; i += PV_THREADS) {
            const double v = diag[i];
            if (v > bv || (v == bv && i < bi)) { bv = v; bi = i; }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const double ov = __shfl_xor_sync(0xffffffffu, bv, off);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        if (lane == 0) { s_val[warp] = bv; s_idx[warp] = bi; }
        __syncthreads();
        if (warp == 0) {
            bv = s_val[lane]; bi = s_idx[lane];
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) {
                const double ov = __shfl_xor_sync(0xffffffffu, bv, off);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
                if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
            }
            if (lane == 0) { s_piv = bi; s_dpiv = bv; picks[t] = bi; }
        }
        __syncthreads();
        const int piv = s_piv;
        if (tid < t) s_prow[tid] = low[(size_t)piv * r + tid];
        __syncthreads();
        const double inv = 1.0 / sqrt(fmax(s_dpiv, 2.2250738585072014e-308));
        for (int i = tid; i < M; i += PV_THREADS) {
            double col = K[(size_t)piv * M + i];
            const double* li = low + (size_t)i * r;
            for (int j = 0; j < t; ++j) col = fma(-li[j], s_prow[j], col);
            col *= inv;
            low[(size_t)i * r + t] = col;
            // -inf marks the chosen points only: once the kernel's rank is exhausted the remaining diagonal
            // is rounding noise and col may overflow, so an unchosen point is clamped to the lowest finite
            // value (a repeated pick would make the "subset" count one observation twice and its variance
            // bound fall below the full posterior's)
            const double d = diag[i], nd = d - col * col;
            diag[i] = (i == piv || d == -INFINITY) ? -INFINITY
                      : nd >= -DBL_MAX ? nd : -DBL_MAX;
        }
        __syncthreads();
    }
}

inline unsigned blocks_for(int64_t n) { return (unsigned)((n + LT - 1) / LT); }

// The thread-per-point Bellman kernels (sweep, per-action argmax) at d_in = state + action dimension:
// launch(D, smem, chunk_rows, nomax) issues the kernel of dimension D with the staged-mean
// configuration of bellman_stage_config.
template <class F>
int launch_bellman(const slb_bellman& cfg, int m, F&& launch) {
    const int din = cfg.grid.ndim + m;
    int chunk_rows, nomax;
    const size_t smem = bellman_stage_config(cfg, din, &chunk_rows, &nomax);
    return slb_dispatch_dim<1, 6>(din, "bellman: state+action dimension", [&](auto D) {
        launch(D, smem, chunk_rows, nomax);
        SLB_LAUNCH_CHECK();
        return 0;
    });
}

bool g_det_fast = true;           // slb_debug_det_fast: A/B against the generic interpreter

}  // namespace

int slb_launch_det_sweep(cudaStream_t st, const slb_sweep& cfg, const double* states, int64_t n,
                         int64_t idx_begin, uint8_t* negative, double* values, double* decrease,
                         double* threshold, double* mean) {
    if (g_det_fast && det_fast_applicable(cfg, states, decrease, threshold, mean)) {
        const slb_function& L = cfg.lipschitz_v;
        det_fast_params q;
        memset(&q, 0, sizeof(q));
        q.k = cfg.policy.matrix; q.a = cfg.dynamics.matrix; q.p = cfg.lyapunov.matrix;
        const bool sat = (cfg.policy.flags & SLB_FLAG_SATURATE) != 0;
        q.klo = sat ? cfg.policy.lower : -INFINITY;
        q.khi = sat ? cfg.policy.upper : INFINITY;
        q.lv_const = cfg.lv_const; q.lf = cfg.lf_const; q.tau = cfg.tau;
        if (L.kind != SLB_FN_NONE) {
            q.lv = L.matrix;
            q.lv_kind = L.out_dim;
            q.lv_abs = (L.flags & (SLB_FLAG_ABS | SLB_FLAG_NORM1)) != 0;
        }
        const int64_t threads = (n + DF_PTS - 1) / DF_PTS;
        det_sweep_fast_kernel<<<blocks_for(threads), LT, 0, st>>>(cfg.grid, q, idx_begin, n, negative, values);
        SLB_LAUNCH_CHECK();
        return 0;
    }
    det_sweep_kernel<<<blocks_for(n), LT, 0, st>>>(cfg, states, n, idx_begin, negative, values,
                                                   decrease, threshold, mean);
    SLB_LAUNCH_CHECK();
    return 0;
}

// bellman_tile.cu
bool slb_argmax_factorable(const slb_bellman& cfg, int m, int n_actions);
int64_t slb_argmax_workspace_bytes(const slb_bellman& cfg, int n_actions);
int slb_launch_argmax_factored(cudaStream_t st, const slb_bellman& cfg, int64_t idx_begin, int64_t n,
                               const double* actions, int n_actions, int m, const double* constraint,
                               int32_t* best, double* best_value, void* workspace);

// The first-fail reduction (slb_first_fail, slb_first_fail_x) and the prefix application
// (slb_apply_prefix, slb_apply_prefix_x); `x` is the validated peer exchange of the _x forms, or
// nullptr for a single process.  `who` names the entry point in error messages.
static int first_fail(const char* who, void* stream, const double* values_dev, const uint8_t* negative_dev,
                      const uint8_t* initial_dev, int64_t n, int64_t idx_begin, void* workspace_dev,
                      slb_fail_key* result_dev, const slb_exchange* x) {
    SLB_CHECK(n >= 0, "%s: negative n", who);
    SLB_CHECK(workspace_dev && result_dev, "%s: null workspace/result", who);
    SLB_CHECK(n == 0 || (values_dev && negative_dev), "%s: null input", who);
    const int64_t want = (n + LT - 1) / LT;
    const int nparts = (int)(want < 1 ? 1 : (want > FF_BLOCKS ? FF_BLOCKS : want));
    cudaStream_t st = (cudaStream_t)stream;
    first_fail_partial_kernel<<<nparts, LT, 0, st>>>(values_dev, negative_dev, initial_dev, n, idx_begin,
                                                     (ff_partial*)workspace_dev);
    SLB_LAUNCH_CHECK();
    slb_exchange none;
    memset(&none, 0, sizeof(none));
    first_fail_final_kernel<<<1, FF_BLOCKS, 0, st>>>((const ff_partial*)workspace_dev, nparts, result_dev,
                                                     x != nullptr ? *x : none);
    SLB_LAUNCH_CHECK();
    return 0;
}

static int apply_prefix(const char* who, void* stream, const double* values_dev, const uint8_t* initial_dev,
                        int64_t n, int64_t idx_begin, slb_fail_key* key_dev, uint8_t* safe_dev,
                        slb_prefix_stats* stats_dev, const slb_exchange* x) {
    SLB_CHECK(n >= 0, "%s: negative n", who);
    SLB_CHECK(key_dev && stats_dev, "%s: null key/stats", who);
    SLB_CHECK(n == 0 || (values_dev && safe_dev), "%s: null buffer", who);
    cudaStream_t st = (cudaStream_t)stream;
    SLB_CUDA(cudaMemsetAsync(stats_dev, 0, sizeof(slb_prefix_stats), st));
    // an empty range launches nothing, except that a rank with an empty slab still takes part in the
    // exchange (one block, no points)
    if (n == 0 && x == nullptr) return 0;
    const int64_t want = (n + LT - 1) / LT;
    const unsigned blocks = (unsigned)(want > 2048 ? 2048 : (want < 1 ? 1 : want));
    slb_exchange none;
    memset(&none, 0, sizeof(none));
    if (x != nullptr && x->world > 1)
        apply_prefix_kernel<true><<<blocks, LT, 0, st>>>(values_dev, initial_dev, n, idx_begin, key_dev,
                                                         safe_dev, stats_dev, *x, nullptr);
    else
        apply_prefix_kernel<false><<<blocks, LT, 0, st>>>(values_dev, initial_dev, n, idx_begin, key_dev,
                                                          safe_dev, stats_dev, x != nullptr ? *x : none, nullptr);
    SLB_LAUNCH_CHECK();
    return 0;
}

// filter.cu (slb_safe_set_step): the prefix rule on the key folded into `rec` by the step's sweep, which
// also zeroed the record; no memset of its own
int slb_launch_apply_prefix_folded(cudaStream_t st, const double* values, const uint8_t* initial, int64_t n,
                                   int64_t idx_begin, slb_fold* rec, slb_fail_key* key, uint8_t* safe,
                                   slb_prefix_stats* stats) {
    const int64_t want = (n + LT - 1) / LT;
    const unsigned blocks = (unsigned)(want > 2048 ? 2048 : (want < 1 ? 1 : want));
    slb_exchange none;
    memset(&none, 0, sizeof(none));
    apply_prefix_kernel<false><<<blocks, LT, 0, st>>>(values, initial, n, idx_begin, key, safe, stats, none, rec);
    SLB_LAUNCH_CHECK();
    return 0;
}

static int validate_exchange(const slb_exchange* x, const char* who) {
    SLB_CHECK(x != nullptr, "%s: null exchange", who);
    SLB_CHECK(x->world >= 1 && x->world <= SLB_MAX_RANKS && x->rank >= 0 && x->rank < x->world,
              "%s: bad exchange (world %d, rank %d, at most %d ranks)", who, x->world, x->rank,
              SLB_MAX_RANKS);
    SLB_CHECK(x->seq_dev != nullptr, "%s: exchange without a sequence counter", who);
    for (int r = 0; r < x->world; ++r)
        SLB_CHECK(x->slots[r] != nullptr, "%s: exchange slot array of rank %d is not mapped", who, r);
    return 0;
}

extern "C" {

int slb_abi_version(void) { return SLB_ABI_VERSION; }
const char* slb_last_error(void) { return g_err; }
int64_t slb_launch_count(void) { return (int64_t)g_slb_launches.load(); }
void slb_note_graph_replay(int64_t kernels) { g_slb_launches.fetch_add(kernels); }

/* sizeof of every ABI struct, for bindings to verify their mirror:
   [grid, function, gp_factor, gp_output, gp_stack, sweep, bellman, fail_key, prefix_stats,
    exchange] */
int slb_struct_sizes(int64_t* out, int32_t n) {
    const int64_t sizes[10] = {sizeof(slb_grid), sizeof(slb_function), sizeof(slb_gp_factor),
                               sizeof(slb_gp_output), sizeof(slb_gp_stack), sizeof(slb_sweep),
                               sizeof(slb_bellman), sizeof(slb_fail_key), sizeof(slb_prefix_stats),
                               sizeof(slb_exchange)};
    for (int i = 0; i < n && i < 10; ++i) out[i] = sizes[i];
    return 10;
}

int slb_device_count(void) {
    int n = 0;
    const cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) {
        slb_set_error("cudaGetDeviceCount failed: %s (libslb200 has no CPU fallback)",
                      cudaGetErrorString(e));
        return -1;
    }
    return n;
}

int64_t slb_first_fail_workspace(int64_t n) {
    (void)n;
    return (int64_t)FF_BLOCKS * (int64_t)sizeof(ff_partial);
}

int slb_first_fail(void* stream, const double* values_dev, const uint8_t* negative_dev,
                   const uint8_t* initial_dev, int64_t n, int64_t idx_begin, void* workspace_dev,
                   slb_fail_key* result_dev) {
    return first_fail("slb_first_fail", stream, values_dev, negative_dev, initial_dev, n, idx_begin,
                      workspace_dev, result_dev, nullptr);
}

int slb_first_fail_x(void* stream, const double* values_dev, const uint8_t* negative_dev,
                     const uint8_t* initial_dev, int64_t n, int64_t idx_begin, void* workspace_dev,
                     slb_fail_key* result_dev, const slb_exchange* xchg) {
    if (validate_exchange(xchg, "slb_first_fail_x")) return 1;
    return first_fail("slb_first_fail_x", stream, values_dev, negative_dev, initial_dev, n, idx_begin,
                      workspace_dev, result_dev, xchg);
}

int slb_apply_prefix_x(void* stream, const double* values_dev, const uint8_t* initial_dev,
                       int64_t n, int64_t idx_begin, slb_fail_key* key_out_dev, uint8_t* safe_dev,
                       void* workspace_dev, slb_prefix_stats* stats_dev, const slb_exchange* xchg) {
    (void)workspace_dev;
    if (validate_exchange(xchg, "slb_apply_prefix_x")) return 1;
    return apply_prefix("slb_apply_prefix_x", stream, values_dev, initial_dev, n, idx_begin, key_out_dev,
                        safe_dev, stats_dev, xchg);
}

int slb_combine_fail_keys(void* stream, const slb_fail_key* gathered_dev, int32_t world,
                          slb_fail_key* out_dev) {
    SLB_CHECK(gathered_dev && out_dev && world >= 1, "slb_combine_fail_keys: bad arguments");
    combine_fail_keys_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(gathered_dev, world, out_dev);
    SLB_LAUNCH_CHECK();
    return 0;
}

int slb_apply_prefix(void* stream, const double* values_dev, const uint8_t* initial_dev, int64_t n,
                     int64_t idx_begin, const slb_fail_key* key_dev, uint8_t* safe_dev,
                     void* workspace_dev, slb_prefix_stats* stats_dev) {
    (void)workspace_dev;
    return apply_prefix("slb_apply_prefix", stream, values_dev, initial_dev, n, idx_begin,
                        const_cast<slb_fail_key*>(key_dev), safe_dev, stats_dev, nullptr);
}

int slb_function_columns(const slb_function* fn) {
    if (fn == nullptr) {
        slb_set_error("slb_function_columns: null function");
        return -1;
    }
    return slb_fn_columns(*fn);
}

int slb_eval_function(void* stream, const slb_function* fn, const double* points_dev, int64_t n,
                      double* out_dev) {
    SLB_CHECK(fn != nullptr, "slb_eval_function: null function");
    if (slb_validate_function(fn, "function", 0)) return 1;
    SLB_CHECK(fn->kind != SLB_FN_NONE, "slb_eval_function: empty function");
    SLB_CHECK(n >= 0, "slb_eval_function: negative n");
    if (n == 0) return 0;
    SLB_CHECK(points_dev && out_dev, "slb_eval_function: null buffer");
    eval_function_kernel<<<blocks_for(n), LT, 0, (cudaStream_t)stream>>>(*fn, points_dev, n, out_dev,
                                                                        slb_fn_columns(*fn));
    SLB_LAUNCH_CHECK();
    return 0;
}

int slb_index_to_state(void* stream, const slb_grid* grid, int64_t idx_begin, int64_t idx_end,
                       double* states_dev) {
    SLB_CHECK(grid != nullptr, "slb_index_to_state: null grid");
    if (slb_validate_grid(grid, false)) return 1;
    if (slb_validate_range("slb_index_to_state", idx_begin, idx_end, grid->nindex)) return 1;
    const int64_t n = idx_end - idx_begin;
    if (n == 0) return 0;
    SLB_CHECK(states_dev != nullptr, "slb_index_to_state: null output");
    index_to_state_kernel<<<blocks_for(n), LT, 0, (cudaStream_t)stream>>>(*grid, idx_begin, n,
                                                                         states_dev);
    SLB_LAUNCH_CHECK();
    return 0;
}

int slb_bellman_sweep(void* stream, const slb_bellman* cfg, int64_t idx_begin, int64_t idx_end,
                      double* out_dev) {
    int m;
    if (slb_validate_bellman(cfg, &m)) return 1;
    if (slb_validate_range("slb_bellman_sweep", idx_begin, idx_end, cfg->grid.nindex)) return 1;
    const int64_t n = idx_end - idx_begin;
    if (n == 0) return 0;
    SLB_CHECK(out_dev != nullptr, "slb_bellman_sweep: null output");
    return launch_bellman(*cfg, m, [&](auto D, size_t smem, int chunk_rows, int nomax) {
        bellman_kernel<D><<<blocks_for(n), LT, smem, (cudaStream_t)stream>>>(*cfg, idx_begin, n, out_dev,
                                                                            chunk_rows, nomax);
    });
}

int slb_debug_det_fast(int32_t enable) {
    g_det_fast = enable != 0;
    return 0;
}

int64_t slb_bellman_argmax_workspace(const slb_bellman* cfg, int32_t n_actions) {
    if (cfg == nullptr || n_actions < 1) return 0;
    const int m = cfg->policy.out_dim;
    return slb_argmax_factorable(*cfg, m, n_actions) ? slb_argmax_workspace_bytes(*cfg, n_actions) : 0;
}

int slb_bellman_argmax(void* stream, const slb_bellman* cfg, int64_t idx_begin, int64_t idx_end,
                       const double* actions_dev, int32_t n_actions, const double* constraint_dev,
                       int32_t* best_dev, double* best_value_dev, void* workspace_dev) {
    SLB_CHECK(cfg != nullptr && cfg->fixed_action, "slb_bellman_argmax: cfg.fixed_action must be set");
    int m;
    if (slb_validate_bellman(cfg, &m)) return 1;
    SLB_CHECK(n_actions >= 1 && actions_dev != nullptr, "slb_bellman_argmax: no actions");
    if (slb_validate_range("slb_bellman_argmax", idx_begin, idx_end, cfg->grid.nindex)) return 1;
    const int64_t n = idx_end - idx_begin;
    if (n == 0) return 0;
    SLB_CHECK(best_dev != nullptr, "slb_bellman_argmax: null output");
    if (workspace_dev != nullptr && slb_argmax_factorable(*cfg, m, n_actions))
        return slb_launch_argmax_factored((cudaStream_t)stream, *cfg, idx_begin, n, actions_dev,
                                          n_actions, m, constraint_dev, best_dev, best_value_dev,
                                          workspace_dev);
    return launch_bellman(*cfg, m, [&](auto D, size_t smem, int chunk_rows, int nomax) {
        bellman_argmax_kernel<D><<<blocks_for(n), LT, smem, (cudaStream_t)stream>>>(
            *cfg, idx_begin, n, actions_dev, n_actions, m, constraint_dev, best_dev, best_value_dev,
            chunk_rows, nomax);
    });
}

int slb_max_abs_diff(void* stream, const double* a_dev, const double* b_dev, int64_t n,
                     double* result_dev) {
    SLB_CHECK(result_dev != nullptr, "slb_max_abs_diff: null result");
    SLB_CHECK(n >= 0, "slb_max_abs_diff: negative n");
    cudaStream_t st = (cudaStream_t)stream;
    SLB_CUDA(cudaMemsetAsync(result_dev, 0, sizeof(double), st));
    if (n == 0) return 0;
    SLB_CHECK(a_dev && b_dev, "slb_max_abs_diff: null input");
    const int64_t want = (n + LT - 1) / LT;
    const unsigned blocks = (unsigned)(want > 1024 ? 1024 : want);
    max_abs_diff_kernel<<<blocks, LT, 0, st>>>(a_dev, b_dev, n,
                                               reinterpret_cast<unsigned long long*>(result_dev));
    SLB_LAUNCH_CHECK();
    return 0;
}

int slb_pivoted_subset(void* stream, const double* kernel_dev, int32_t M, int32_t r,
                       int64_t* picks_dev, double* scratch_dev) {
    SLB_CHECK(M >= 0 && r >= 0 && r <= M && r <= SLB_HEAD_RANK,
              "slb_pivoted_subset: need 0 <= r <= min(M, %d) (M %d, r %d)", SLB_HEAD_RANK, M, r);
    if (r == 0) return 0;
    SLB_CHECK(kernel_dev && picks_dev && scratch_dev, "slb_pivoted_subset: null buffer");
    pivoted_subset_kernel<<<1, PV_THREADS, 0, (cudaStream_t)stream>>>(
        kernel_dev, M, r, picks_dev, scratch_dev, scratch_dev + (size_t)M * r);
    SLB_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
