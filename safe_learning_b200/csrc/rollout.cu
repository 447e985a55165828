// rollout.cu -- closed-loop rollouts  x <- f(x, pi(x))  from many start states at once:
//   compute_roa      examples/utilities.py:654-686  (end state within tol of the equilibrium,
//                                                    optionally the whole trajectory)
//   reward_rollout   examples/utilities.py:522-545  (discounted reward sum with the grid-wide
//                                                    early stop  max_i |temp_i| < tol)
//
// One thread per start state: the state (d <= 6) and the running reward sum stay in registers /
// the thread's stack for a whole chunk of RK steps, eval_fn is inlined (as in light.cu), the
// descriptors travel as __grid_constant__ parameters.  One launch per chunk; between chunks the
// state (and sum) wait in HBM, (d + 1) * 8 B per point, structure-of-arrays so that the loads and
// stores are coalesced.  Every step is eval_fn's arithmetic, so a rollout of h steps is bit-identical
// to h compositions of the library's one-step evaluations (slb_eval_function).
//
// The dynamics are either a fused function (DIN = 0: eval_fn) or the posterior mean of a GP stack
// (DIN = d_in = d + m, 1..6: the Bellman sweep's staged pipeline, bellman.cuh, set up once per launch
// and restarted per step; slb_gp_mean is its one-step form, so the same bit-identity holds).  The
// pipeline has block barriers: in the GP instantiations every thread stays to the end, threads past
// n clamp their index and store nothing.
//
// Early stop of reward_rollout without a host round trip per chunk: each chunk kernel writes, per
// step and per block, the maximum of |temp| (doubles >= 0 ordered by their bit patterns, so a NaN
// sorts above inf and never passes `< tol`, like np.max); a one-block finish kernel reduces the
// chunk's table and records the first step T* whose maximum is below tol.  The chunk after it
// re-runs the chunk holding T* from its saved start state and sums exactly up to T*; every later
// launch sees the control word and exits at once.  Cost: at most one extra chunk.
#include "bellman.cuh"

#include <string.h>

namespace {

constexpr int RT_MAX = 256;       // threads per block (fewer for small point counts)
constexpr int RK = 32;            // closed-loop steps per launch
constexpr int SECTOR = 4;         // doubles per 32-byte sector (trajectory staging)

// control word of one reward rollout (workspace): phase 0 = running, 1 = T* found in the chunk
// before the next launch (which re-runs it), 2 = done
struct roll_ctrl { int64_t stop; int32_t phase; int32_t _pad; };

struct roa_epilogue {
    double eq[SLB_MAX_DIM];
    double tol;
    int last;                     // this launch holds the final state: write flags
};

SLB_DEV void load_start(const slb_bellman& cfg, const double* __restrict__ states, int64_t idx_begin,
                        int64_t i, int d, double* x) {
    if (states != nullptr) {
        for (int c = 0; c < d; ++c) x[c] = states[i * d + c];
    } else {
        grid_index_to_state(cfg.grid, idx_begin + i, x);
    }
}

// u = pi(x) appended to z = [x, u]   (the one policy evaluation of a step)
SLB_DEV void apply_policy(const slb_bellman& cfg, double* z, int d) {
    double u[SLB_MAX_OUT];
    const int m = eval_fn(cfg.policy, z, u);
    for (int c = 0; c < m; ++c) z[d + c] = u[c];
}

// x <- f([x, u])
SLB_DEV void apply_dynamics(const slb_bellman& cfg, double* z, int d) {
    double y[SLB_MAX_OUT];
    eval_fn(cfg.dynamics, z, y);
    for (int c = 0; c < d; ++c) z[c] = y[c];
}

// x <- mean f([x, u]) of the GP stack (every thread of the block takes part: barriers)
template <int DIN>
SLB_DEV void apply_gp_mean(const slb_bellman& cfg, bellman_smem& S, double* z, int d) {
    double mu[SLB_MAX_OUT], err[SLB_MAX_OUT];
    mean_pipe_start<DIN>(cfg.gp, S.P);
    gp_mean_staged<DIN, false>(cfg.gp, z, mu, err, S.tab512, S.tab64, S.P);
    for (int c = 0; c < d; ++c) z[c] = mu[c];
}

// Trajectory output [n, d, horizon] (the reference's layout): consecutive steps of one coordinate
// are contiguous, so a thread's per-step stores are d * horizon * 8 B apart from its neighbours'.
// Each thread stages up to SECTOR steps per coordinate in shared memory and writes them once it
// reaches the end of a 32-byte sector (or of the launch), so every store fills whole sectors.
struct traj_stage {
    double* s;                    // shared, [d][SECTOR][blockDim.x]
    double* out;                  // trajectory row base of this point (coordinate 0, step 0)
    int64_t row;                  // global index of that element
    int horizon, first;           // first step staged by this launch

    SLB_DEV void put(int c, int t, double v, int last) {
        const int64_t o = row + (int64_t)c * horizon + t;
        const int slot = (int)(o & (SECTOR - 1));
        const int bs = blockDim.x;
        s[(c * SECTOR + slot) * bs + threadIdx.x] = v;
        if (slot != SECTOR - 1 && t != last) return;
        const int lo = max(0, slot - (t - first));
        double* dst = out + (int64_t)c * horizon + t - slot;
        if (lo == 0 && slot == SECTOR - 1 && (reinterpret_cast<uintptr_t>(dst) & 31) == 0) {
            const double* q = s + (c * SECTOR) * bs + threadIdx.x;
            reinterpret_cast<double2*>(dst)[0] = make_double2(q[0], q[bs]);
            reinterpret_cast<double2*>(dst)[1] = make_double2(q[2 * bs], q[3 * bs]);
        } else {
            for (int j = lo; j <= slot; ++j) dst[j] = s[(c * SECTOR + j) * bs + threadIdx.x];
        }
    }
};

// compute_roa: steps t in [t_begin, t_end) of x_t = f(x_{t-1}, pi(x_{t-1})), t >= 1.  The first
// launch (t_begin == 1) reads the start states; the last one applies the distance test
// norm(x - eq, 2) <= tol (numpy's row norm: sqrt of the sequential sum of squares).  DIN > 0: the GP
// mean's slices in dynamic shared memory (chunk_rows, nomax of bellman_stage_config), the trajectory
// staging behind them.
template <int DIN>
__global__ void __launch_bounds__(RT_MAX)
roa_chunk_kernel(const __grid_constant__ slb_bellman cfg, const double* __restrict__ states,
                 int64_t idx_begin, int64_t n, int t_begin, int t_end, int horizon,
                 const double* __restrict__ x_in, double* __restrict__ x_out, double* __restrict__ traj,
                 const roa_epilogue ep, uint8_t* __restrict__ roa, double* __restrict__ end_states,
                 int chunk_rows, int nomax) {
    extern __shared__ double s_traj[];
    const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bellman_smem S;
    double* stage = s_traj;
    if constexpr (DIN == 0) {
        if (i0 >= n) return;                              // no block barrier below
    } else {
        extern __shared__ __align__(16) unsigned char smem_raw[];
        bellman_setup<DIN>(S, smem_raw, cfg, chunk_rows, nomax);
        stage = S.P.gbuf + 2 * S.P.gstride;
    }
    const bool valid = DIN == 0 || i0 < n;
    const int64_t i = valid ? i0 : n - 1;                 // every thread stays for the block barriers
    const int d = cfg.grid.ndim;
    double z[SLB_MAX_IN];
    if (t_begin == 1) {
        load_start(cfg, states, idx_begin, i, d, z);
    } else {
        for (int c = 0; c < d; ++c) z[c] = x_in[c * n + i];
    }
    traj_stage ts;
    const bool write_traj = traj != nullptr && valid;
    if (write_traj) {
        ts.s = stage;
        ts.row = i * d * (int64_t)horizon;
        ts.out = traj + ts.row;
        ts.horizon = horizon;
        ts.first = t_begin == 1 ? 0 : t_begin;
        if (t_begin == 1)                                 // trajectories[:, :, 0] = start states
            for (int c = 0; c < d; ++c) ts.put(c, 0, z[c], t_end - 1);
    }
    for (int t = t_begin; t < t_end; ++t) {
        apply_policy(cfg, z, d);
        if constexpr (DIN == 0) apply_dynamics(cfg, z, d);
        else apply_gp_mean<DIN>(cfg, S, z, d);
        if (write_traj)
            for (int c = 0; c < d; ++c) ts.put(c, t, z[c], t_end - 1);
    }
    if (!valid) return;
    if (ep.last) {
        double ss = 0.0;
        for (int c = 0; c < d; ++c) {
            const double df = f64sub(z[c], ep.eq[c]);
            const double sq = f64mul(df, df);
            ss = c == 0 ? sq : f64add(ss, sq);
        }
        roa[i] = sqrt(ss) <= ep.tol ? 1 : 0;              // NaN / inf end states: outside
        if (end_states != nullptr)
            for (int c = 0; c < d; ++c) end_states[i * d + c] = z[c];
    } else {
        for (int c = 0; c < d; ++c) x_out[c * n + i] = z[c];
    }
}

// reward_rollout, one chunk: steps t in [chunk * RK, min((chunk + 1) * RK, horizon)) of
//   u = pi(x);  temp = discount^t * r([x, u]);  sum += temp;  x = f([x, u])
// with the per-block maximum of |temp| per step into partial[step][block].  Chunk c reads
// buf[c & 1] (chunk 0 the start states) and writes buf[(c + 1) & 1] = [x (d rows); sum] of [n].
// After the finish kernel found T* in chunk c, launch c + 1 re-runs chunk c up to T* instead.
// DIN > 0: the GP mean's slices in dynamic shared memory, as in roa_chunk_kernel.
template <int DIN>
__global__ void __launch_bounds__(RT_MAX)
reward_chunk_kernel(const __grid_constant__ slb_bellman cfg, const double* __restrict__ states,
                    int64_t idx_begin, int64_t n, int chunk, int nchunks, int horizon,
                    const double* __restrict__ discount, double* __restrict__ buf0,
                    double* __restrict__ buf1, double* __restrict__ sums,
                    uint64_t* __restrict__ partial, const roll_ctrl* __restrict__ ctrl,
                    int chunk_rows, int nomax) {
    __shared__ uint64_t s_max[RK][RT_MAX / 32];
    const int phase = ctrl->phase;                        // written by the previous finish kernel
    if (phase == 2) return;
    const bool fixup = phase == 1;
    if (!fixup && chunk >= nchunks) return;
    const int run = fixup ? chunk - 1 : chunk;
    const int t0 = run * RK;
    const int t1 = fixup ? (int)ctrl->stop + 1 : min(t0 + RK, horizon);
    bellman_smem S;
    if constexpr (DIN > 0) {
        extern __shared__ __align__(16) unsigned char smem_raw[];
        bellman_setup<DIN>(S, smem_raw, cfg, chunk_rows, nomax);
    }
    const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = i0 < n;
    const int64_t i = valid ? i0 : n - 1;                 // every thread stays for the block maxima
    const int d = cfg.grid.ndim;
    double z[SLB_MAX_IN];
    double sum = 0.0;
    if (run == 0) {
        load_start(cfg, states, idx_begin, i, d, z);
    } else {
        const double* in = (run & 1) ? buf1 : buf0;
        for (int c = 0; c < d; ++c) z[c] = in[c * n + i];
        sum = in[d * n + i];
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int t = t0; t < t1; ++t) {
        apply_policy(cfg, z, d);
        double r[SLB_MAX_OUT];
        eval_fn(cfg.reward, z, r);
        const double temp = f64mul(__ldg(discount + t), r[0]);
        sum = f64add(sum, temp);
        if constexpr (DIN == 0) apply_dynamics(cfg, z, d);
        else apply_gp_mean<DIN>(cfg, S, z, d);
        if (!fixup) {
            unsigned long long b = valid ? (unsigned long long)__double_as_longlong(fabs(temp)) : 0ull;
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) {
                const unsigned long long o = __shfl_xor_sync(0xffffffffu, b, off);
                b = o > b ? o : b;
            }
            if (lane == 0) s_max[t - t0][warp] = b;
        }
    }
    if (valid) {
        if (fixup || run == nchunks - 1) {
            sums[i] = sum;
        } else {
            double* out = (run & 1) ? buf0 : buf1;
            for (int c = 0; c < d; ++c) out[c * n + i] = z[c];
            out[d * n + i] = sum;
        }
    }
    if (fixup) return;
    __syncthreads();
    if ((int)threadIdx.x < t1 - t0) {
        uint64_t m = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) m = s_max[threadIdx.x][w] > m ? s_max[threadIdx.x][w] : m;
        partial[(int64_t)threadIdx.x * gridDim.x + blockIdx.x] = m;
    }
}

// One block: the grid-wide maximum of |temp| for every step of chunk `chunk` (one warp per step),
// then the first step below tol (as bit patterns: tol_bits = 0 when tol <= 0 or NaN).
constexpr int FIN_THREADS = 1024;
static_assert(FIN_THREADS / 32 >= RK, "one warp per step of a chunk");

__global__ void __launch_bounds__(FIN_THREADS)
reward_finish_kernel(const uint64_t* __restrict__ partial, int nblocks, int chunk, int horizon,
                     uint64_t tol_bits, roll_ctrl* __restrict__ ctrl, int64_t* __restrict__ stop_out) {
    __shared__ uint64_t s_step[RK];
    const int phase = ctrl->phase;
    if (phase != 0) {                                     // 1: the chunk kernel just ran the re-run
        if (phase == 1 && threadIdx.x == 0) ctrl->phase = 2;
        return;
    }
    const int steps = min(RK, horizon - chunk * RK);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (warp < steps) {
        const uint64_t* row = partial + (int64_t)warp * nblocks;
        unsigned long long m = 0;
        for (int j = lane; j < nblocks; j += 32) {
            const unsigned long long v = row[j];
            m = v > m ? v : m;
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const unsigned long long o = __shfl_xor_sync(0xffffffffu, m, off);
            m = o > m ? o : m;
        }
        if (lane == 0) s_step[warp] = m;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int s = 0; s < steps; ++s) {
            if (s_step[s] < tol_bits) {
                ctrl->stop = (int64_t)chunk * RK + s;
                ctrl->phase = 1;
                *stop_out = ctrl->stop;
                break;
            }
        }
    }
}

// block size: 256 threads, fewer when that leaves SMs idle (the 10^4-point rollouts of the
// notebooks are latency-bound chains; smaller blocks spread them over every SM)
int rollout_block(int64_t n) {
    int bs = RT_MAX;
    while (bs > 64 && (n + bs - 1) / bs < 2 * SLB_NUM_SMS) bs >>= 1;
    return bs;
}

// gp_mean: the dynamics are the posterior mean of cfg->gp (slb_rollout_gp_mean / slb_reward_rollout_gp_mean)
int validate_rollout(const char* who, const slb_bellman* cfg, const double* states_dev, int64_t idx_begin,
                     int64_t n, int32_t horizon, bool reward, bool gp_mean) {
    SLB_CHECK(cfg != nullptr, "%s: null config", who);
    SLB_CHECK(gp_mean || cfg->gp.num_outputs == 0,
              "%s: GP dynamics cannot be rolled out (gp.num_outputs must be 0)", who);
    SLB_CHECK(!cfg->fixed_action, "%s: a rollout follows the policy (fixed_action must be 0)", who);
    const int d = cfg->grid.ndim;
    SLB_CHECK(d >= 1 && d <= SLB_MAX_DIM, "%s: state dimension %d outside 1..%d", who, d, SLB_MAX_DIM);
    SLB_CHECK(n >= 0, "%s: negative n", who);
    SLB_CHECK(horizon >= 0, "%s: negative horizon %d", who, horizon);
    if (states_dev == nullptr) {
        if (slb_validate_grid(&cfg->grid, false)) return 1;
        if (slb_validate_range(who, idx_begin, idx_begin + n, cfg->grid.nindex)) return 1;
    }
    if (slb_validate_function(&cfg->policy, "policy", d)) return 1;
    SLB_CHECK(cfg->policy.kind != SLB_FN_NONE, "%s: a policy is required", who);
    const int m = slb_fn_columns(cfg->policy);
    SLB_CHECK(m >= 1 && d + m <= SLB_MAX_IN, "%s: state %d + action %d exceeds %d inputs", who, d, m,
              SLB_MAX_IN);
    if (gp_mean) {
        SLB_CHECK(cfg->gp.num_outputs == d, "%s: the GP stack has %d outputs but the state has %d dims",
                  who, cfg->gp.num_outputs, d);
        if (slb_validate_gp(&cfg->gp)) return 1;
        SLB_CHECK(cfg->gp.input_dim == d + m, "%s: GP input_dim %d != state %d + action %d", who,
                  cfg->gp.input_dim, d, m);
        SLB_CHECK(d + m <= 6, "%s: GP input_dim %d not compiled (1..6)", who, d + m);
        SLB_CHECK(cfg->dynamics.kind == SLB_FN_NONE,
                  "%s: the GP mean is the dynamics (dynamics.kind must be SLB_FN_NONE)", who);
        if (slb_validate_staged_tables(&cfg->gp, who)) return 1;
    } else if (slb_validate_dynamics(&cfg->dynamics, who, d, m)) {
        return 1;
    }
    if (reward) {
        if (slb_validate_function(&cfg->reward, "reward_function", d + m)) return 1;
        SLB_CHECK(cfg->reward.kind != SLB_FN_NONE, "%s: a reward function is required", who);
        SLB_CHECK(slb_fn_columns(cfg->reward) == 1, "%s: the reward must return one column", who);
    }
    return 0;
}

// Launches the chunk kernel of the dynamics' source: launch(D, smem, chunk_rows, nomax) with D = 0
// (fused dynamics, `extra` bytes of dynamic shared memory) or D = d_in of the GP stack (its pipeline,
// then `extra` bytes; the kernel `kern(D)` opts in beyond 48 KB).
template <class K, class F>
int launch_rollout(const slb_bellman& cfg, bool gp_mean, size_t extra, K&& kern, F&& launch) {
    if (!gp_mean) return launch(std::integral_constant<int, 0>{}, extra, 0, 0);
    int chunk_rows, nomax;
    const size_t smem = bellman_stage_config(cfg, cfg.gp.input_dim, &chunk_rows, &nomax) + extra;
    return slb_dispatch_dim<1, 6>(cfg.gp.input_dim, "rollout: GP input_dim", [&](auto D) {
        if (smem > 48 * 1024)
            SLB_CUDA(cudaFuncSetAttribute(kern(D), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        return launch(D, smem, chunk_rows, nomax);
    });
}

// The one-step posterior mean (slb_gp_mean): one point per thread on the Bellman sweep's pipeline.
constexpr int GM_THREADS = 256;

template <int DIN>
__global__ void __launch_bounds__(GM_THREADS, 2)
gp_mean_kernel(const __grid_constant__ slb_bellman cfg, const double* __restrict__ points, int64_t n,
               double* __restrict__ mean, int chunk_rows, int nomax) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    bellman_smem S;
    bellman_setup<DIN>(S, smem_raw, cfg, chunk_rows, nomax);
    const int64_t i0 = (int64_t)blockIdx.x * GM_THREADS + threadIdx.x;
    const bool valid = i0 < n;
    const int64_t i = valid ? i0 : n - 1;                 // every thread stays for the block barriers
    double z[SLB_MAX_IN], mu[SLB_MAX_OUT], err[SLB_MAX_OUT];
#pragma unroll
    for (int c = 0; c < DIN; ++c) z[c] = points[i * DIN + c];
    mean_pipe_start<DIN>(cfg.gp, S.P);
    gp_mean_staged<DIN, false>(cfg.gp, z, mu, err, S.tab512, S.tab64, S.P);
    if (!valid) return;
    const int D = cfg.gp.num_outputs;
    for (int o = 0; o < D; ++o) mean[i * D + o] = mu[o];
}

int64_t align256(int64_t b) { return (b + 255) & ~(int64_t)255; }

int rollout_impl(const char* who, bool gp_mean, void* stream, const slb_bellman* cfg,
                 const double* states_dev, int64_t idx_begin, int64_t n, int32_t horizon,
                 const double* equilibrium_host, double tol, uint8_t* roa_dev, double* end_states_dev,
                 double* traj_dev, void* workspace_dev) {
    if (validate_rollout(who, cfg, states_dev, idx_begin, n, horizon, false, gp_mean)) return 1;
    SLB_CHECK(traj_dev == nullptr || horizon >= 1, "%s: trajectories need horizon >= 1", who);
    if (n == 0) return 0;
    SLB_CHECK(roa_dev != nullptr, "%s: null flag output", who);
    const int d = cfg->grid.ndim;
    const int steps = horizon > 1 ? horizon - 1 : 0;         // range(1, horizon)
    const int nchunks = steps > 0 ? (steps + RK - 1) / RK : 1;
    SLB_CHECK(nchunks == 1 || workspace_dev != nullptr, "%s: null workspace", who);
    roa_epilogue ep;
    memset(&ep, 0, sizeof(ep));
    for (int c = 0; c < d; ++c) ep.eq[c] = equilibrium_host != nullptr ? equilibrium_host[c] : 0.0;
    ep.tol = tol;
    double* buf[2] = {static_cast<double*>(workspace_dev), nullptr};
    if (workspace_dev != nullptr) buf[1] = buf[0] + align256(n * d * 8) / 8;
    const int bs = rollout_block(n);
    const unsigned nb = (unsigned)((n + bs - 1) / bs);
    const size_t traj_smem = traj_dev != nullptr ? (size_t)bs * d * SECTOR * sizeof(double) : 0;
    cudaStream_t st = (cudaStream_t)stream;
    return launch_rollout(*cfg, gp_mean, traj_smem, [](auto D) { return roa_chunk_kernel<decltype(D)::value>; },
                          [&](auto D, size_t smem, int chunk_rows, int nomax) {
        for (int c = 0; c < nchunks; ++c) {
            const int t_begin = 1 + c * RK;
            const int t_end = steps > 0 ? min(t_begin + RK, horizon) : 1;
            ep.last = c == nchunks - 1;
            roa_chunk_kernel<decltype(D)::value><<<nb, bs, smem, st>>>(
                *cfg, states_dev, idx_begin, n, t_begin, t_end, horizon, buf[c & 1], buf[(c + 1) & 1], traj_dev,
                ep, roa_dev, end_states_dev, chunk_rows, nomax);
            SLB_LAUNCH_CHECK();
        }
        return 0;
    });
}

int reward_rollout_impl(const char* who, bool gp_mean, void* stream, const slb_bellman* cfg,
                        const double* states_dev, int64_t idx_begin, int64_t n, int32_t horizon,
                        const double* discount_dev, double tol, double* sums_dev, int64_t* stop_dev,
                        void* workspace_dev) {
    if (validate_rollout(who, cfg, states_dev, idx_begin, n, horizon, true, gp_mean)) return 1;
    SLB_CHECK(stop_dev != nullptr, "%s: null stop output", who);
    cudaStream_t st = (cudaStream_t)stream;
    SLB_CUDA(cudaMemsetAsync(stop_dev, 0xff, sizeof(int64_t), st));          // -1: not converged
    if (n == 0) return 0;
    SLB_CHECK(sums_dev != nullptr, "%s: null output", who);
    if (horizon == 0) {
        SLB_CUDA(cudaMemsetAsync(sums_dev, 0, (size_t)n * sizeof(double), st));
        return 0;
    }
    SLB_CHECK(discount_dev != nullptr && workspace_dev != nullptr, "%s: null discount/workspace", who);
    const int d = cfg->grid.ndim;
    const int bs = rollout_block(n);
    const int nb = (int)((n + bs - 1) / bs);
    char* w = static_cast<char*>(workspace_dev);
    double* buf0 = reinterpret_cast<double*>(w);
    double* buf1 = reinterpret_cast<double*>(w + align256(n * (d + 1) * 8));
    uint64_t* partial = reinterpret_cast<uint64_t*>(w + 2 * align256(n * (d + 1) * 8));
    roll_ctrl* ctrl = reinterpret_cast<roll_ctrl*>(reinterpret_cast<char*>(partial) + align256(RK * (int64_t)nb * 8));
    SLB_CUDA(cudaMemsetAsync(ctrl, 0, sizeof(roll_ctrl), st));
    uint64_t tol_bits = 0;                                 // max |temp| < tol: never when tol <= 0 or NaN
    if (tol > 0.0) memcpy(&tol_bits, &tol, sizeof(tol_bits));
    const int nchunks = (horizon + RK - 1) / RK;
    return launch_rollout(*cfg, gp_mean, 0, [](auto D) { return reward_chunk_kernel<decltype(D)::value>; },
                          [&](auto D, size_t smem, int chunk_rows, int nomax) {
        for (int c = 0; c <= nchunks; ++c) {               // launch nchunks: the re-run of the last chunk
            reward_chunk_kernel<decltype(D)::value><<<nb, bs, smem, st>>>(
                *cfg, states_dev, idx_begin, n, c, nchunks, horizon, discount_dev, buf0, buf1, sums_dev, partial,
                ctrl, chunk_rows, nomax);
            SLB_LAUNCH_CHECK();
            if (c == nchunks) break;
            reward_finish_kernel<<<1, FIN_THREADS, 0, st>>>(partial, nb, c, horizon, tol_bits, ctrl, stop_dev);
            SLB_LAUNCH_CHECK();
        }
        return 0;
    });
}

}  // namespace

extern "C" {

int64_t slb_rollout_workspace(const slb_bellman* cfg, int64_t n, int32_t reward) {
    if (cfg == nullptr || n <= 0) return 0;
    const int64_t d = cfg->grid.ndim;
    if (!reward) return 2 * align256(n * d * 8);
    const int64_t nb = (n + rollout_block(n) - 1) / rollout_block(n);
    return 2 * align256(n * (d + 1) * 8) + align256(RK * nb * 8) + align256(sizeof(roll_ctrl));
}

int slb_rollout(void* stream, const slb_bellman* cfg, const double* states_dev, int64_t idx_begin,
                int64_t n, int32_t horizon, const double* equilibrium_host, double tol,
                uint8_t* roa_dev, double* end_states_dev, double* traj_dev, void* workspace_dev) {
    return rollout_impl("slb_rollout", false, stream, cfg, states_dev, idx_begin, n, horizon, equilibrium_host, tol,
                   roa_dev, end_states_dev, traj_dev, workspace_dev);
}

int slb_rollout_gp_mean(void* stream, const slb_bellman* cfg, const double* states_dev, int64_t idx_begin,
                        int64_t n, int32_t horizon, const double* equilibrium_host, double tol,
                        uint8_t* roa_dev, double* end_states_dev, double* traj_dev, void* workspace_dev) {
    return rollout_impl("slb_rollout_gp_mean", true, stream, cfg, states_dev, idx_begin, n, horizon, equilibrium_host,
                   tol, roa_dev, end_states_dev, traj_dev, workspace_dev);
}

int slb_reward_rollout(void* stream, const slb_bellman* cfg, const double* states_dev, int64_t idx_begin,
                       int64_t n, int32_t horizon, const double* discount_dev, double tol,
                       double* sums_dev, int64_t* stop_dev, void* workspace_dev) {
    return reward_rollout_impl("slb_reward_rollout", false, stream, cfg, states_dev, idx_begin, n, horizon,
                          discount_dev, tol, sums_dev, stop_dev, workspace_dev);
}

int slb_reward_rollout_gp_mean(void* stream, const slb_bellman* cfg, const double* states_dev,
                               int64_t idx_begin, int64_t n, int32_t horizon, const double* discount_dev,
                               double tol, double* sums_dev, int64_t* stop_dev, void* workspace_dev) {
    return reward_rollout_impl("slb_reward_rollout_gp_mean", true, stream, cfg, states_dev, idx_begin, n, horizon,
                          discount_dev, tol, sums_dev, stop_dev, workspace_dev);
}

int slb_gp_mean(void* stream, const slb_gp_stack* gp, const double* points_dev, int64_t n, double* mean_dev) {
    SLB_CHECK(gp != nullptr, "slb_gp_mean: null gp");
    if (slb_validate_gp(gp)) return 1;
    SLB_CHECK(gp->num_outputs > 0, "slb_gp_mean: GP stack has no outputs");
    SLB_CHECK(gp->input_dim >= 1 && gp->input_dim <= 6, "slb_gp_mean: GP input_dim %d not compiled (1..6)",
              gp->input_dim);
    if (slb_validate_staged_tables(gp, "slb_gp_mean")) return 1;
    SLB_CHECK(n >= 0, "slb_gp_mean: negative n");
    SLB_CHECK(n == 0 || (points_dev != nullptr && mean_dev != nullptr), "slb_gp_mean: null buffer");
    if (n == 0) return 0;
    slb_bellman cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gp = *gp;
    int chunk_rows, nomax;
    const size_t smem = bellman_stage_config(cfg, gp->input_dim, &chunk_rows, &nomax);
    const unsigned nb = (unsigned)((n + GM_THREADS - 1) / GM_THREADS);
    return slb_dispatch_dim<1, 6>(gp->input_dim, "slb_gp_mean: GP input_dim", [&](auto D) {
        gp_mean_kernel<decltype(D)::value><<<nb, GM_THREADS, smem, (cudaStream_t)stream>>>(
            cfg, points_dev, n, mean_dev, chunk_rows, nomax);
        SLB_LAUNCH_CHECK();
        return 0;
    });
}

}  // extern "C"
