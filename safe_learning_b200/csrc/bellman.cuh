// bellman.cuh -- one policy-evaluation transition per thread (reinforcement_learning.py:65-114),
// shared by the Bellman sweep / argmax (light.cu) and the value-operator assembly (value_opt.cu):
// u = pi(x), the mean next state f(x, u) (fused function or mean-only staged GP) and r(x, u).
#pragma once
#include "common.cuh"
#include "gp_mean_staged.cuh"

// host: validates an slb_bellman descriptor, *m_out = action dimension
int slb_validate_bellman(const slb_bellman* cfg, int* m_out);

// slice size and dynamic shared memory of the Bellman kernels' mean pipeline (< 48 KB: no opt-in)
static inline size_t bellman_stage_config(const slb_bellman& cfg, int din, int* chunk_rows, int* nomax) {
    int most = 1;
    for (int f = 0; f < cfg.gp.num_factors; ++f) {
        int no = 0;
        for (int o = 0; o < cfg.gp.num_outputs; ++o) no += cfg.gp.outputs[o].factor == f;
        if (no > most) most = no;
    }
    *nomax = most;
    *chunk_rows = mean_chunk_rows(din, most, 24);
    return mean_smem_bytes(din, most, *chunk_rows);
}

// The mean-only GP runs on the staged pipeline of gp_mean_staged.cuh (training rows and gamma streamed
// through shared memory by TMA bulk copies, expanded squared distance, the <= 1 ulp table exp).
struct bellman_smem {
    mean_pipe P;
    double* tab512;
    double* tab64;
};

template <int DIN>
SLB_DEV void bellman_setup(bellman_smem& S, unsigned char* smem_raw, const slb_bellman& cfg,
                           int chunk_rows, int nomax) {
    mean_pipe_setup(S.P, smem_raw, DIN, chunk_rows, nomax, cfg.gp, &S.tab512, &S.tab64);
    if (threadIdx.x == 0) mean_pipe_init(S.P, S.tab512);
    __syncthreads();
    slb_bulk::mbar_wait(S.P.bar + 2, 0);                       // exp tables have landed
}

// mu = mean f(x, u) (:94, :97-99), r = r(x, u) (:95)
template <int DIN>
SLB_DEV void bellman_transition(const slb_bellman& cfg, const double* x, const double* u, int m,
                                bellman_smem& S, double* mu, double* r) {
    const int d = cfg.grid.ndim;
    double z[SLB_MAX_IN], err[SLB_MAX_OUT];
    for (int c = 0; c < d; ++c) z[c] = x[c];
    for (int c = 0; c < m; ++c) z[d + c] = u[c];
    if (cfg.gp.num_outputs > 0) {
        mean_pipe_start<DIN>(cfg.gp, S.P);
        gp_mean_staged<DIN, false>(cfg.gp, z, mu, err, S.tab512, S.tab64, S.P);
    } else {
        eval_fn(cfg.dynamics, z, mu);
    }
    eval_fn(cfg.reward, z, r);
}

// r + gamma V(mu), written out in full rather than through bellman_transition: the sweep kernels'
// register allocation depends on the order of these local arrays
template <int DIN>
SLB_DEV double bellman_value(const slb_bellman& cfg, const double* x, const double* u, int m,
                             bellman_smem& S) {
    const int d = cfg.grid.ndim;
    double z[SLB_MAX_IN], mu[SLB_MAX_OUT], err[SLB_MAX_OUT], r[SLB_MAX_OUT], v[SLB_MAX_OUT];
    for (int c = 0; c < d; ++c) z[c] = x[c];
    for (int c = 0; c < m; ++c) z[d + c] = u[c];
    if (cfg.gp.num_outputs > 0) {
        mean_pipe_start<DIN>(cfg.gp, S.P);
        gp_mean_staged<DIN, false>(cfg.gp, z, mu, err, S.tab512, S.tab64, S.P);
    } else {
        eval_fn(cfg.dynamics, z, mu);
    }
    eval_fn(cfg.reward, z, r);                               // :95
    eval_fn(cfg.value, mu, v);                               // :101
    return f64add(r[0], f64mul(cfg.gamma, v[0]));                // :104
}
