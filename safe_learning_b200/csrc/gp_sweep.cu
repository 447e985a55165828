// gp_sweep.cu -- C entry points of the GP sweep: factor packing, posterior on a point list, the
// fused Lyapunov sweep over an index range / a state list, and the refine pass of the filtered
// sweep.  The kernel itself is gp_tile.cuh, instantiated per input dimension in gp_tile_inst.cu.
#include "common.cuh"

#include <string.h>

#include "gp_args.h"

namespace {

// Packed factor: for 8-row block b and k-step PAIR kp <= b, 32 lanes x 2 doubles: lane T holds
// L^-1[8b + T/4, 8kp + T%4] and L^-1[8b + T/4, 8kp + 4 + T%4]; pair offset b(b+1)/2 + kp.
__global__ void pack_factor_kernel(const double* __restrict__ Linv, int M, int nrb,
                                   double* __restrict__ W, int64_t total) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= total) return;
    const int64_t pair = e >> 6;
    const int lane = (int)((e >> 1) & 31);
    const int half = (int)(e & 1);
    int64_t b = (int64_t)((sqrt(8.0 * (double)pair + 1.0) - 1.0) * 0.5);
    while (b * (b + 1) / 2 > pair) --b;
    while ((b + 1) * (b + 2) / 2 <= pair) ++b;
    const int64_t kp = pair - b * (b + 1) / 2;
    const int64_t row = 8 * b + (lane >> 2);
    const int64_t col = 8 * kp + 4 * half + (lane & 3);
    W[e] = (row < M && col <= row) ? Linv[row * M + col] : 0.0;
}


// slb_record_factor_dependency: an event (owned by the library, one per device) that every launch
// reading the packed factors has to wait for -- a restore of the GP tables whose large part, the
// packed L^-1, is still in flight on another stream while the filter stages, which do not read it,
// already run
cudaEvent_t g_factor_event[64] = {};
bool g_factor_pending[64] = {};

int wait_for_factors(cudaStream_t st) {
    int device = 0;
    SLB_CUDA(cudaGetDevice(&device));
    if (device < 0 || device >= 64 || !g_factor_pending[device]) return 0;
    // under stream capture the wait becomes an external-event node: every replay of the graph
    // waits for the event's latest record
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    SLB_CUDA(cudaStreamIsCapturing(st, &cs));
    SLB_CUDA(cudaStreamWaitEvent(st, g_factor_event[device],
                                 cs == cudaStreamCaptureStatusActive ? cudaEventWaitExternal : 0));
    return 0;
}

// tp: points per CTA (64 for sweeps and point lists; 32 only in the refine pass)
int dispatch_gp_tile(cudaStream_t st, const slb_sweep& cfg, const slb_gp_args& a, int tp = 64) {
    if (a.n <= 0) return 0;
    if (wait_for_factors(st)) return 1;
    SLB_CHECK(a.n <= (int64_t)0x7fffffff * tp, "too many points for one launch");
    const bool timing = a.timing != nullptr;
    bool kexpr = false;
    for (int f = 0; f < cfg.gp.num_factors; ++f) kexpr |= cfg.gp.factors[f].kernel.num_prims > 0;
    return slb_dispatch_dim<1, 6>(cfg.gp.input_dim, "GP input_dim", [&](auto D) {
        return tp == 64 ? slb_gp_tile_launch<D, 64>(st, cfg, a, kexpr, timing)
                        : slb_gp_tile_launch<D, 32>(st, cfg, a, kexpr, timing);
    });
}

}  // namespace

// for the other units whose kernels read the packed factors (gp_grad.cu)
int slb_wait_for_factors(cudaStream_t st) { return wait_for_factors(st); }

// implemented in light.cu
int slb_launch_det_sweep(cudaStream_t st, const slb_sweep& cfg, const double* states, int64_t n,
                         int64_t idx_begin, uint8_t* negative, double* values, double* decrease,
                         double* threshold, double* mean);

static long long* g_timing_buffer = nullptr;
static unsigned long long* g_refine_timing = nullptr;   // slb_debug_refine_timing

// The full posterior for the points the decision filter (filter.cu) could not decide: `list`
// holds their indices relative to idx_begin, `count` (device) how many there are.  The list is
// usually a small fraction of the grid -- too short to fill the SMs with 64-point tiles, and a
// tile's duration does not shrink with the list -- so the pass is launched once per tile size
// (32 and 64 points per CTA) and only the launch whose range holds the list length does work;
// the CTAs of the other (and those beyond the list) leave at once.
static int64_t g_refine_split = 32 * SLB_NUM_SMS;   // longest list that gets 32-point tiles

// Short lists (<= 32 points per SM) additionally split every tile's ROWS over the CTAs the grid has
// to spare (up to SLB_SPLIT_MAX groups of equal triangular area, gp_tile.cuh): the tile kernel's
// duration is set by the M^2 / 2 contraction of one tile, so a few hundred points in whole tiles keep
// a few dozen SMs busy while the rest idle; split 8 ways a 32-point tile's share is ~8 times shorter.
// mean / err: NULL, or [n_max, D] rows indexed like `negative` (slb_debug_refine); fold: see slb_fold_target;
// side / side_slot / closed: see slb_gp_args (NULL: the terms are computed from the list's indices)
int slb_launch_refine(cudaStream_t st, const slb_sweep& cfg, int64_t n_max, int64_t idx_begin,
                      const int64_t* list, const unsigned long long* count, uint8_t* negative,
                      double* values, double* mean, double* err, double* split_partial, int* split_ticket,
                      const slb_fold_target& fold, const filter_side* side, const int64_t* side_slot,
                      bool closed) {
    slb_gp_args a;
    memset(&a, 0, sizeof(a));
    a.idx_begin = idx_begin; a.mode = MODE_SWEEP_GRID;
    a.negative = negative; a.values = values;
    a.mean = mean; a.err = err;
    a.index_list = list; a.count = count;
    a.fold = fold;
    a.side = side; a.side_slot = side_slot;
    a.closed = side != nullptr && closed;
    a.timing = g_timing_buffer;            // slb_debug_phase_timing: per-warp phase clocks of the refine CTAs
    const int tps[2] = {32, 64};
    const int64_t lo[2] = {0, g_refine_split};
    const int64_t hi[2] = {g_refine_split, INT64_MAX};
    for (int v = 0; v < 2; ++v) {
        if (lo[v] >= hi[v] || lo[v] >= n_max) continue;
        a.count_min = lo[v]; a.count_max = hi[v];
        a.n = n_max < hi[v] ? n_max : hi[v];        // the grid never needs to cover more
        a.split_partial = nullptr; a.split_ticket = nullptr; a.marks = nullptr;
        if (v == 0 && split_partial != nullptr) {
            // at least one CTA per SM, so that short lists have CTAs to spread their rows over
            if (a.n < (int64_t)SLB_NUM_SMS * tps[v]) a.n = (int64_t)SLB_NUM_SMS * tps[v];
            if ((a.n + tps[v] - 1) / tps[v] <= SLB_SPLIT_ITEMS) {
                a.split_partial = split_partial; a.split_ticket = split_ticket;
                a.marks = g_refine_timing;
            }
        }
        const int rc = dispatch_gp_tile(st, cfg, a, tps[v]);
        if (rc) return rc;
    }
    return 0;
}

extern "C" {

/* diagnostics: list length up to which the refine pass uses 32-point tiles */
int slb_debug_refine_split(int64_t upto32) {
    g_refine_split = upto32 < 0 ? 0 : upto32;
    return 0;
}

int slb_restore_tables(void* dst_dev, const void* src_host, int64_t split_bytes, int64_t total_bytes,
                       void* stream, void* side_stream) {
    SLB_CHECK(dst_dev != nullptr && src_host != nullptr, "slb_restore_tables: null buffer");
    SLB_CHECK(split_bytes >= 0 && split_bytes <= total_bytes, "slb_restore_tables: split %lld outside [0, %lld]",
              (long long)split_bytes, (long long)total_bytes);
    cudaStream_t st = static_cast<cudaStream_t>(stream), side = static_cast<cudaStream_t>(side_stream);
    char* dst = static_cast<char*>(dst_dev);
    const char* src = static_cast<const char*>(src_host);
    if (split_bytes > 0) SLB_CUDA(cudaMemcpyAsync(dst, src, (size_t)split_bytes, cudaMemcpyHostToDevice, st));
    const int64_t rest = total_bytes - split_bytes;
    if (rest <= 0) return 0;
    if (side == nullptr || side == st) {
        SLB_CUDA(cudaMemcpyAsync(dst + split_bytes, src + split_bytes, (size_t)rest, cudaMemcpyHostToDevice, st));
        return 0;
    }
    // the second stream must not overtake earlier readers of the packed factors on `st`
    int device = 0;
    SLB_CUDA(cudaGetDevice(&device));
    SLB_CHECK(device >= 0 && device < 64, "slb_restore_tables: device %d unsupported", device);
    static cudaEvent_t order[64] = {};
    if (order[device] == nullptr) SLB_CUDA(cudaEventCreateWithFlags(&order[device], cudaEventDisableTiming));
    SLB_CUDA(cudaEventRecord(order[device], st));
    SLB_CUDA(cudaStreamWaitEvent(side, order[device], 0));
    SLB_CUDA(cudaMemcpyAsync(dst + split_bytes, src + split_bytes, (size_t)rest, cudaMemcpyHostToDevice, side));
    return slb_record_factor_dependency(side);
}

int slb_record_factor_dependency(void* stream) {
    int device = 0;
    SLB_CUDA(cudaGetDevice(&device));
    SLB_CHECK(device >= 0 && device < 64, "slb_record_factor_dependency: device %d unsupported", device);
    if (g_factor_event[device] == nullptr)
        SLB_CUDA(cudaEventCreateWithFlags(&g_factor_event[device], cudaEventDisableTiming));
    SLB_CUDA(cudaEventRecord(g_factor_event[device], static_cast<cudaStream_t>(stream)));
    g_factor_pending[device] = true;
    return 0;
}

int slb_debug_phase_timing(void* buffer_dev) {
    g_timing_buffer = static_cast<long long*>(buffer_dev);
    return 0;
}

int slb_debug_refine_timing(void* buffer_dev) {
    g_refine_timing = static_cast<unsigned long long*>(buffer_dev);
    return 0;
}

int64_t slb_packed_len(int32_t M) {
    if (M <= 0) return 0;
    const int64_t nrb = (M + 7) / 8;
    return nrb * (nrb + 1) * 32;
}

int slb_pack_factor(void* stream, const double* Linv_dev, int32_t M, double* Wpack_dev) {
    SLB_CHECK(Linv_dev != nullptr && Wpack_dev != nullptr, "slb_pack_factor: null pointer");
    SLB_CHECK(M > 0, "slb_pack_factor: M must be positive (got %d)", M);
    const int nrb = (M + 7) / 8;
    const int64_t total = slb_packed_len(M);
    const int threads = 256;
    const int64_t blocks = (total + threads - 1) / threads;
    pack_factor_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(Linv_dev, M, nrb,
                                                                              Wpack_dev, total);
    SLB_LAUNCH_CHECK();
    return 0;
}

int slb_gp_predict(void* stream, const slb_gp_stack* gp, const double* points_dev, int64_t n,
                   double* mean_dev, double* err_dev, int32_t want_var) {
    SLB_CHECK(gp != nullptr, "slb_gp_predict: null gp");
    if (slb_validate_gp(gp)) return 1;
    SLB_CHECK(gp->num_outputs > 0, "slb_gp_predict: GP stack has no outputs");
    SLB_CHECK(n >= 0, "slb_gp_predict: negative n");
    SLB_CHECK(n == 0 || (points_dev && mean_dev && err_dev), "slb_gp_predict: null buffer");
    slb_sweep cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gp = *gp;
    slb_gp_args a;
    memset(&a, 0, sizeof(a));
    a.points = points_dev; a.n = n; a.mode = MODE_PREDICT; a.want_var = want_var;
    a.mean = mean_dev; a.err = err_dev;
    return dispatch_gp_tile((cudaStream_t)stream, cfg, a);
}

static int sweep_common(void* stream, const slb_sweep* cfg, const double* states, int64_t n,
                        int64_t idx_begin, uint8_t* negative, double* values, double* decrease,
                        double* threshold, double* mean, double* err) {
    int m;
    if (slb_validate_sweep(cfg, states != nullptr, &m)) return 1;
    SLB_CHECK(n >= 0, "lyapunov sweep: negative point count");
    if (n == 0) return 0;
    SLB_CHECK(negative != nullptr, "lyapunov sweep: negative_dev is required");
    if (cfg->gp.num_outputs > 0) {
        slb_gp_args a;
        memset(&a, 0, sizeof(a));
        a.points = states; a.n = n; a.idx_begin = idx_begin;
        a.mode = states ? MODE_SWEEP_STATES : MODE_SWEEP_GRID;
        a.negative = negative; a.values = values; a.decrease = decrease; a.threshold = threshold;
        a.mean = mean; a.err = err;
        a.timing = g_timing_buffer;
        return dispatch_gp_tile((cudaStream_t)stream, *cfg, a);
    }
    SLB_CHECK(err == nullptr, "deterministic dynamics have no error bounds (err_dev must be NULL)");
    return slb_launch_det_sweep((cudaStream_t)stream, *cfg, states, n, idx_begin, negative, values,
                                decrease, threshold, mean);
}

int slb_lyapunov_sweep(void* stream, const slb_sweep* cfg, int64_t idx_begin, int64_t idx_end,
                       uint8_t* negative_dev, double* values_dev, double* decrease_dev,
                       double* threshold_dev, double* mean_dev, double* err_dev) {
    SLB_CHECK(cfg != nullptr, "slb_lyapunov_sweep: null config");
    if (slb_validate_range("slb_lyapunov_sweep", idx_begin, idx_end, cfg->grid.nindex)) return 1;
    return sweep_common(stream, cfg, nullptr, idx_end - idx_begin, idx_begin, negative_dev,
                        values_dev, decrease_dev, threshold_dev, mean_dev, err_dev);
}

int slb_lyapunov_points(void* stream, const slb_sweep* cfg, const double* states_dev, int64_t n,
                        uint8_t* negative_dev, double* values_dev, double* decrease_dev,
                        double* threshold_dev, double* mean_dev, double* err_dev) {
    SLB_CHECK(n == 0 || states_dev != nullptr, "slb_lyapunov_points: null states");
    return sweep_common(stream, cfg, states_dev, n, 0, negative_dev, values_dev, decrease_dev,
                        threshold_dev, mean_dev, err_dev);
}

}  // extern "C"
