// network_grad.cu -- reverse-mode products (VJPs) of the fused networks and plants, the gradient
// path behind training NeuralNetwork / LyapunovNetwork with torch.optim (the reference trains them
// with TF optimisers through tf.gradients: reinforcement_learning_pendulum.ipynb cells 16-20, 34-38,
// lyapunov_function_learning.ipynb cells 25-30, inverted_pendulum.ipynb cell 17).
//
// Networks (SLB_FN_MLP, SLB_FN_LYAPUNOV_NN): one CTA walks tiles of TP points.  Per tile it
//   (1) recomputes the forward pass with every layer's activations in shared memory, column-major
//       [unit][point] with a padded stride, through nn_unit (common.cuh), the unit eval_network computes
//       with: the ReLU masks and tanh values it differentiates are exactly the forward's, and `out` is
//       bit-identical to slb_eval_function;
//   (2) runs the layers backwards: delta = dL/dh * act'(h) (tanh' = 1 - h^2, ReLU' = [h > 0], so 0 at
//       exactly 0, as TF's), the layer's weight gradient sum_p delta_p a_p^T (and sum_p delta_p for the
//       bias) accumulated into this CTA's row of the workspace, and dL/da = delta W for the layer below.
// Every CTA owns a fixed, n-determined set of tiles (tile t -> CTA t mod G) and the same thread owns
// the same parameter in every tile, so a CTA's partial sums are formed in a fixed order without any
// atomic; a second launch adds the G partial rows in CTA order.  Two calls with the same inputs give
// bit-identical gradients.  With G == 1 the CTA writes grad_params directly (no workspace).
//
// Plants (SLB_FN_PENDULUM, SLB_FN_CARTPOLE, SLB_FN_VANDERPOL): one thread per point, forward mode over
// the 3 or 5 inputs through the ten Euler sub-steps (state and tangents in registers), then
// grad_in = g^T J.
//
// SLB_FN_TRIANGULATION, SLB_FN_PIECEWISE_CONSTANT: the vertex-value gradient of triangulation_grad.cu.
#include "common.cuh"

#include <string.h>

// triangulation_grad.cu
int64_t slb_triangulation_vjp_workspace(const slb_function* fn, int64_t n);
int slb_triangulation_vjp(cudaStream_t st, const slb_function* fn, const double* points_dev, int64_t n,
                          const double* grad_out_dev, double* grad_in_dev, double* grad_params_dev,
                          double* out_dev, void* workspace_dev);

namespace {

constexpr int TP = 32;            // points per tile (one warp's worth: unit-major loops are conflict-free)
constexpr int TPS = TP + 1;       // padded column stride of the shared activation tables
constexpr int NT = 256;           // threads per CTA
constexpr int MAXL = SLB_NN_MAX_LAYERS;
constexpr int MAXW = SLB_NN_MAX_WIDTH;
constexpr size_t SMEM_OPTIN = 227 * 1024;

// activations of the largest network (input <= SLB_MAX_IN, 8 layers of 64) + two cotangent tables
constexpr size_t SMEM_MAX = (size_t)(SLB_MAX_IN + MAXL * MAXW) * TPS * sizeof(double)
                            + 2 * (size_t)MAXW * TPS * sizeof(double);
static_assert(SMEM_MAX <= SMEM_OPTIN, "network VJP tile exceeds the 227 KB shared-memory opt-in");

struct net_shape {
    int32_t kind;                 // SLB_FN_MLP or SLB_FN_LYAPUNOV_NN
    int32_t layers;
    int32_t width[MAXL + 1];      // width[0] = in_dim, width[l + 1] = output width of layer l
    int32_t act[MAXL];            // 0 tanh, 1 relu, 2 identity
    int32_t bias[MAXL];           // layer l carries a bias (MLP hidden layers with use_bias)
    int64_t woff[MAXL];           // offset of layer l's weight [out, in] in the packed parameters;
                                  // its bias (if any) follows at woff + out * in
    int32_t aoff[MAXL + 2];       // shared-memory offset (doubles) of activation table l; [layers + 1] = total
    int32_t maxw;
    int32_t _pad;
    int64_t nparams;
    double scale;                 // MLP output_scale
};

__global__ void __launch_bounds__(NT) vjp_network_kernel(
        const __grid_constant__ net_shape S, const double* __restrict__ P, const double* __restrict__ x,
        int64_t n, const double* __restrict__ gout, double* __restrict__ gin, double* __restrict__ out,
        double* __restrict__ partial, int64_t ntiles) {
    extern __shared__ double sm[];
    double* const dbuf0 = sm + S.aoff[S.layers + 1];          // two cotangent tables, used alternately
    double* const dbuf1 = dbuf0 + (size_t)S.maxw * TPS;
    const int tid = threadIdx.x;
    const int L = S.layers;
    double* my = partial != nullptr ? partial + (size_t)blockIdx.x * S.nparams : nullptr;
    bool first = true;
    for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int64_t p0 = tile * TP;
        const int np = (int)min((int64_t)TP, n - p0);
        const int in = S.width[0];
        for (int i = tid; i < in * TP; i += NT) {
            const int k = i / TP, p = i % TP;
            sm[k * TPS + p] = p < np ? x[(p0 + p) * in + k] : 0.0;
        }
        __syncthreads();
        // ---- forward
        for (int l = 0; l < L; ++l) {
            const int wi = S.width[l], wo = S.width[l + 1], act = S.act[l];
            const double* a_in = sm + S.aoff[l];
            double* a_out = sm + S.aoff[l + 1];
            const double* W = P + S.woff[l];
            const double* b = W + (size_t)wo * wi;
            for (int i = tid; i < wo * TP; i += NT) {
                const int o = i / TP, p = i % TP;
                const double* row = W + (size_t)o * wi;
                a_out[o * TPS + p] = nn_unit(wi, [&](int k) { return a_in[k * TPS + p]; },
                                             [&](int k) { return __ldg(row + k); }, S.bias[l],
                                             [&] { return __ldg(b + o); }, act);
            }
            __syncthreads();
        }
        // ---- output and the cotangent of the last activations
        const double* hL = sm + S.aoff[L];
        const int wL = S.width[L];
        if (S.kind == SLB_FN_MLP) {
            for (int i = tid; i < wL * TP; i += NT) {
                const int o = i / TP, p = i % TP;
                double g = 0.0;
                if (p < np) {
                    if (out != nullptr) out[(p0 + p) * wL + o] = f64mul(hL[o * TPS + p], S.scale);
                    g = gout[(p0 + p) * wL + o] * S.scale;
                }
                dbuf0[o * TPS + p] = g;
            }
        } else {                                   // V = sum_k h_k^2, dV/dh = 2h
            if (out != nullptr && tid < np) {
                double v = f64mul(hL[tid], hL[tid]);
                for (int k = 1; k < wL; ++k) v = f64add(v, f64mul(hL[k * TPS + tid], hL[k * TPS + tid]));
                out[p0 + tid] = v;
            }
            for (int i = tid; i < wL * TP; i += NT) {
                const int k = i / TP, p = i % TP;
                dbuf0[k * TPS + p] = p < np ? 2.0 * gout[p0 + p] * hL[k * TPS + p] : 0.0;
            }
        }
        __syncthreads();
        // ---- backward
        for (int l = L - 1; l >= 0; --l) {
            double* dA = ((L - 1 - l) & 1) ? dbuf1 : dbuf0;
            double* dB = ((L - 1 - l) & 1) ? dbuf0 : dbuf1;
            const int wi = S.width[l], wo = S.width[l + 1], act = S.act[l];
            const double* a_in = sm + S.aoff[l];
            const double* h = sm + S.aoff[l + 1];
            const double* W = P + S.woff[l];
            for (int i = tid; i < wo * TP; i += NT) {
                const int o = i / TP, p = i % TP;
                dA[o * TPS + p] *= activate_grad(h[o * TPS + p], act);
            }
            __syncthreads();
            if (my != nullptr) {                   // weight gradient (then bias): sum over the tile's points
                const int nw = wo * wi, nb = S.bias[l] ? wo : 0;
                for (int j = tid; j < nw + nb; j += NT) {
                    double s = 0.0;
                    if (j < nw) {
                        const int o = j / wi, k = j % wi;
                        for (int p = 0; p < np; ++p) s = fma(dA[o * TPS + p], a_in[k * TPS + p], s);
                    } else {
                        const int o = j - nw;
                        for (int p = 0; p < np; ++p) s += dA[o * TPS + p];
                    }
                    const int64_t idx = S.woff[l] + j;
                    my[idx] = first ? s : my[idx] + s;
                }
            }
            if (l > 0 || gin != nullptr) {         // dL/da_in = delta W
                for (int i = tid; i < wi * TP; i += NT) {
                    const int k = i / TP, p = i % TP;
                    double s = 0.0;
                    for (int o = 0; o < wo; ++o) s = fma(dA[o * TPS + p], __ldg(W + (size_t)o * wi + k), s);
                    if (l > 0) dB[k * TPS + p] = s;
                    else if (p < np) gin[(p0 + p) * in + k] = s;
                }
            }
            __syncthreads();
        }
        first = false;
    }
}

// grad[j] = sum over CTAs b = 0 .. G-1 (in that order) of partial[b][j]
__global__ void __launch_bounds__(NT) vjp_reduce_kernel(const double* __restrict__ partial, int G,
                                                        int64_t nparams, double* __restrict__ grad) {
    const int64_t j = (int64_t)blockIdx.x * NT + threadIdx.x;
    if (j >= nparams) return;
    double s = partial[j];
    for (int b = 1; b < G; ++b) s += partial[(size_t)b * nparams + j];
    grad[j] = s;
}

// ---- plants: forward-mode tangents T[c][i] = d state_c / d input_i
SLB_DEV void pendulum_jacobian(const slb_function& f, const double* in, double J[2][3]) {
    const double* p = f.cparams;
    const double g_l = p[0], inertia = p[1], fric_i = p[2], dt = p[3];
    const bool has_norm = p[9] != 0.0, has_fric = p[10] != 0.0;
    double th = in[0], om = in[1], u = in[2];
    double s_th = 1.0, s_om = 1.0, s_u = 1.0;
    if (has_norm) { s_th = p[4]; s_om = p[5]; s_u = p[6]; th *= s_th; om *= s_om; u *= s_u; }
    const double ui = u / inertia;
    double dth[3] = {s_th, 0.0, 0.0}, dom[3] = {0.0, s_om, 0.0};
    const double dui[3] = {0.0, 0.0, s_u / inertia};
    for (int it = 0; it < 10; ++it) {
        const double c = cos(th);
        double acc = g_l * sin(th) + ui;
        if (has_fric) acc -= fric_i * om;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            double dacc = g_l * c * dth[i] + dui[i];
            if (has_fric) dacc -= fric_i * dom[i];
            const double dth_n = dth[i] + dt * dom[i];
            dom[i] = dom[i] + dt * dacc;
            dth[i] = dth_n;
        }
        const double th_n = th + dt * om;
        om = om + dt * acc;
        th = th_n;
    }
    const double o_th = has_norm ? p[7] : 1.0, o_om = has_norm ? p[8] : 1.0;
#pragma unroll
    for (int i = 0; i < 3; ++i) { J[0][i] = dth[i] * o_th; J[1][i] = dom[i] * o_om; }
}

SLB_DEV void cartpole_jacobian(const slb_function& f, const double* in, double J[4][5]) {
    const double* p = f.cparams;
    const double m = p[0], M = p[1], L = p[2], b = p[3], g = p[4], dt = p[5];
    const bool has_norm = p[15] != 0.0;
    double s[4] = {in[0], in[1], in[2], in[3]};
    double u = in[4];
    double ds[4][5];
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int i = 0; i < 5; ++i) ds[c][i] = (c == i) ? (has_norm ? p[6 + c] : 1.0) : 0.0;
    const double su = has_norm ? p[10] : 1.0;
    if (has_norm) { for (int c = 0; c < 4; ++c) s[c] *= p[6 + c]; u *= su; }
    for (int it = 0; it < 10; ++it) {
        const double th = s[1], v = s[2], om = s[3];
        const double st = sin(th), ct = cos(th), s2t = sin(2.0 * th), c2t = cos(2.0 * th);
        const double det = L * (M + m * (st * st));
        const double n1 = u - m * L * (om * om) * st - b * om * ct + 0.5 * m * g * L * s2t;
        const double n2 = u * ct - 0.5 * m * L * (om * om) * s2t - b * (m + M) * om / (m * L) + (m + M) * g * st;
        const double v_dot = n1 * L / det;
        const double om_dot = n2 / det;
        const double inv_det2 = 1.0 / (det * det);
#pragma unroll
        for (int i = 0; i < 5; ++i) {
            const double dth = ds[1][i], dv = ds[2][i], dom = ds[3][i];
            const double du = (i == 4) ? su : 0.0;
            const double dn1 = du - m * L * (2.0 * om * dom * st + om * om * ct * dth)
                               - b * (dom * ct - om * st * dth) + m * g * L * c2t * dth;
            const double dn2 = du * ct - u * st * dth - 0.5 * m * L * (2.0 * om * dom * s2t + 2.0 * om * om * c2t * dth)
                               - b * (m + M) * dom / (m * L) + (m + M) * g * ct * dth;
            const double ddet = 2.0 * L * m * st * ct * dth;
            const double dv_dot = L * (dn1 * det - n1 * ddet) * inv_det2;
            const double dom_dot = (dn2 * det - n2 * ddet) * inv_det2;
            ds[0][i] += dt * dv;
            ds[1][i] += dt * dom;
            ds[2][i] += dt * dv_dot;
            ds[3][i] += dt * dom_dot;
        }
        s[0] += dt * v;
        s[1] += dt * om;
        s[2] += dt * v_dot;
        s[3] += dt * om_dot;
    }
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int i = 0; i < 5; ++i) J[c][i] = ds[c][i] * (has_norm ? p[11 + c] : 1.0);
}

// Van der Pol: the state's two inputs (the action column does not enter, its column of J is 0).  The
// (de)normalisation is diagonal, so its tangent is the scale itself.
SLB_DEV void vanderpol_jacobian(const slb_function& f, const double* in, double J[2][3]) {
    const double* p = f.cparams;
    const double damping = p[0], dt = p[1];
    const bool has_norm = p[2] != 0.0;
    const double s_x = has_norm ? p[3] : 1.0, s_y = has_norm ? p[4] : 1.0;
    double x = in[0] * s_x, y = in[1] * s_y;
    double dx[2] = {s_x, 0.0}, dy[2] = {0.0, s_y};
    for (int it = 0; it < 10; ++it) {
        const double y_dot = x + damping * (x * x - 1.0) * y;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const double dy_dot = dx[i] + damping * (2.0 * x * dx[i] * y + (x * x - 1.0) * dy[i]);
            const double dx_n = dx[i] - dt * dy[i];
            dy[i] = dy[i] + dt * dy_dot;
            dx[i] = dx_n;
        }
        const double x_n = x - dt * y;
        y = y + dt * y_dot;
        x = x_n;
    }
    const double o_x = has_norm ? p[5] : 1.0, o_y = has_norm ? p[6] : 1.0;
#pragma unroll
    for (int i = 0; i < 2; ++i) { J[0][i] = dx[i] * o_x; J[1][i] = dy[i] * o_y; }
    J[0][2] = 0.0; J[1][2] = 0.0;
}

__global__ void __launch_bounds__(NT) vjp_plant_kernel(const __grid_constant__ slb_function f,
                                                       const double* __restrict__ x, int64_t n,
                                                       const double* __restrict__ gout,
                                                       double* __restrict__ gin, double* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * NT + threadIdx.x;
    if (i >= n) return;
    double z[5], y[4];
    if (f.kind == SLB_FN_PENDULUM || f.kind == SLB_FN_VANDERPOL) {
        const bool vdp = f.kind == SLB_FN_VANDERPOL;
        for (int c = 0; c < 3; ++c) z[c] = x[i * 3 + c];
        if (out != nullptr) {
            if (vdp) eval_vanderpol(f, z, y); else eval_pendulum(f, z, y);
            out[i * 2] = y[0]; out[i * 2 + 1] = y[1];
        }
        if (gin != nullptr) {
            double J[2][3];
            if (vdp) vanderpol_jacobian(f, z, J); else pendulum_jacobian(f, z, J);
            const double g0 = gout[i * 2], g1 = gout[i * 2 + 1];
            for (int c = 0; c < 3; ++c) gin[i * 3 + c] = g0 * J[0][c] + g1 * J[1][c];
        }
    } else {
        for (int c = 0; c < 5; ++c) z[c] = x[i * 5 + c];
        if (out != nullptr) { eval_cartpole(f, z, y); for (int c = 0; c < 4; ++c) out[i * 4 + c] = y[c]; }
        if (gin != nullptr) {
            double J[4][5];
            cartpole_jacobian(f, z, J);
            double g[4];
            for (int o = 0; o < 4; ++o) g[o] = gout[i * 4 + o];
            for (int c = 0; c < 5; ++c) {
                double s = 0.0;
                for (int o = 0; o < 4; ++o) s = fma(g[o], J[o][c], s);
                gin[i * 5 + c] = s;
            }
        }
    }
}

// shape, parameter layout and shared-memory footprint of a network descriptor (validated before)
void network_shape(const slb_function& f, net_shape* S) {
    memset(S, 0, sizeof(*S));
    S->kind = f.kind;
    S->layers = nn_layers(f);
    int64_t off = 0;
    int32_t aoff = 0;
    S->maxw = 1;
    for (int l = 0; l <= S->layers; ++l) {
        S->width[l] = nn_width(f, l);
        S->aoff[l] = aoff;
        aoff += S->width[l] * TPS;
        if (S->width[l] > S->maxw) S->maxw = S->width[l];
    }
    for (int l = 0; l < S->layers; ++l) {
        S->act[l] = nn_act(f, l);
        S->bias[l] = nn_bias(f, l);
        S->woff[l] = off;
        off += nn_layer_size(S->width[l], S->width[l + 1], S->bias[l]);
    }
    S->aoff[S->layers + 1] = aoff;
    S->nparams = off;
    S->scale = f.kind == SLB_FN_MLP ? nn_scale(f) : 1.0;
}

size_t network_smem(const net_shape& S) {
    return ((size_t)S.aoff[S.layers + 1] + 2 * (size_t)S.maxw * TPS) * sizeof(double);
}

// CTAs of the parameter-gradient launch: one wave at the occupancy the tile's shared memory allows
// (a function of the shape and n only, so that the reduction order is reproducible)
int network_ctas(const net_shape& S, int64_t n) {
    const int64_t ntiles = (n + TP - 1) / TP;
    const size_t per_cta = network_smem(S) + 1024;              // + the runtime's reserved 1 KB
    int per_sm = (int)((228 * 1024) / per_cta);
    per_sm = per_sm < 1 ? 1 : (per_sm > 8 ? 8 : per_sm);
    return (int)(ntiles < (int64_t)SLB_NUM_SMS * per_sm ? ntiles : (int64_t)SLB_NUM_SMS * per_sm);
}

bool is_table(int kind) { return kind == SLB_FN_TRIANGULATION || kind == SLB_FN_PIECEWISE_CONSTANT; }

bool is_plant(int kind) {
    return kind == SLB_FN_PENDULUM || kind == SLB_FN_CARTPOLE || kind == SLB_FN_VANDERPOL;
}

int vjp_validate(const slb_function* fn, const char* what) {
    SLB_CHECK(fn != nullptr, "%s: null function", what);
    SLB_CHECK(fn->kind == SLB_FN_MLP || fn->kind == SLB_FN_LYAPUNOV_NN || fn->kind == SLB_FN_PENDULUM ||
              fn->kind == SLB_FN_CARTPOLE || fn->kind == SLB_FN_VANDERPOL || is_table(fn->kind),
              "%s: function kind %d has no VJP (NeuralNetwork, LyapunovNetwork, InvertedPendulum, CartPole, "
              "VanDerPol, Triangulation, PiecewiseConstant)", what, fn->kind);
    SLB_CHECK(!(fn->flags & SLB_FLAG_GRADIENT) || (fn->kind != SLB_FN_MLP && fn->kind != SLB_FN_LYAPUNOV_NN),
              "%s: the VJP of a network gradient (SLB_FLAG_GRADIENT) is a Hessian-vector product, which is "
              "not implemented", what);
    const uint32_t allowed = fn->kind == SLB_FN_TRIANGULATION ? SLB_FLAG_PROJECT : 0u;   // not a post-op
    SLB_CHECK((fn->flags & ~allowed) == 0,
              "%s: post-op flags 0x%x are not differentiated here (compose them in torch)", what, fn->flags);
    return slb_validate_function(fn, what, 0);
}

}  // namespace

extern "C" int64_t slb_function_vjp_workspace(const slb_function* fn, int64_t n) {
    if (vjp_validate(fn, "slb_function_vjp_workspace")) return -1;
    if (n < 0) { slb_set_error("slb_function_vjp_workspace: negative n"); return -1; }
    if (is_table(fn->kind)) return slb_triangulation_vjp_workspace(fn, n);
    if (is_plant(fn->kind)) return 0;
    net_shape S;
    network_shape(*fn, &S);
    const int G = network_ctas(S, n);
    return G > 1 ? (int64_t)G * S.nparams * (int64_t)sizeof(double) : 0;
}

extern "C" int slb_function_vjp(void* stream, const slb_function* fn, const double* points_dev, int64_t n,
                                const double* grad_out_dev, double* grad_in_dev, double* grad_params_dev,
                                double* out_dev, void* workspace_dev) {
    if (vjp_validate(fn, "slb_function_vjp")) return 1;
    SLB_CHECK(n >= 0, "slb_function_vjp: negative n (%lld)", (long long)n);
    cudaStream_t st = (cudaStream_t)stream;
    if (is_table(fn->kind)) {
        SLB_CHECK(n == 0 || (points_dev != nullptr && grad_out_dev != nullptr),
                  "slb_function_vjp: null points or cotangent");
        return slb_triangulation_vjp(st, fn, points_dev, n, grad_out_dev, grad_in_dev, grad_params_dev, out_dev,
                                     workspace_dev);
    }
    const bool plant = is_plant(fn->kind);
    SLB_CHECK(!plant || grad_params_dev == nullptr,
              "slb_function_vjp: the plants have no parameters (grad_params must be NULL)");
    SLB_CHECK(n == 0 || (points_dev != nullptr && grad_out_dev != nullptr),
              "slb_function_vjp: null points or cotangent");
    if (plant) {
        if (n == 0 || (grad_in_dev == nullptr && out_dev == nullptr)) return 0;
        vjp_plant_kernel<<<(unsigned)((n + NT - 1) / NT), NT, 0, st>>>(*fn, points_dev, n, grad_out_dev,
                                                                      grad_in_dev, out_dev);
        SLB_LAUNCH_CHECK();
        return 0;
    }
    net_shape S;
    network_shape(*fn, &S);
    if (n == 0) {
        if (grad_params_dev != nullptr)
            SLB_CUDA(cudaMemsetAsync(grad_params_dev, 0, (size_t)S.nparams * sizeof(double), st));
        return 0;
    }
    const int G = network_ctas(S, n);
    double* partial = nullptr;
    if (grad_params_dev != nullptr) {
        SLB_CHECK(G == 1 || workspace_dev != nullptr,
                  "slb_function_vjp: %lld points need slb_function_vjp_workspace = %lld bytes of workspace",
                  (long long)n, (long long)G * S.nparams * (long long)sizeof(double));
        partial = G == 1 ? grad_params_dev : (double*)workspace_dev;
    }
    if (grad_in_dev == nullptr && out_dev == nullptr && partial == nullptr) return 0;
    const size_t smem = network_smem(S);
    SLB_CUDA(cudaFuncSetAttribute(vjp_network_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int64_t ntiles = (n + TP - 1) / TP;
    vjp_network_kernel<<<G, NT, smem, st>>>(S, fn->matrix, points_dev, n, grad_out_dev, grad_in_dev, out_dev,
                                            partial, ntiles);
    SLB_LAUNCH_CHECK();
    if (partial != nullptr && G > 1) {
        vjp_reduce_kernel<<<(unsigned)((S.nparams + NT - 1) / NT), NT, 0, st>>>(partial, G, S.nparams,
                                                                               grad_params_dev);
        SLB_LAUNCH_CHECK();
    }
    return 0;
}
