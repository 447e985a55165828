// no_shrink.cu -- update_safe_set(can_shrink=False) (lyapunov.py:497-606 with :507-510, :540-582): the
// V-sorted batch loop of the reference, resolved per batch on the device.
//
// In sorted positions (order = stable sort of V), batch k is B_k = [k b, min((k+1) b, n)).  S0 / R0 are the
// previous safe set and refinement, known = negative | initial, n_req the required refinement.  The loop
// sets safe = S0 | negative on B_k and stops at the first batch where some position is not verified:
//   p_k  first position of B_k with neither S0 nor negative (end_k: the batch is safe, go on);
//   R = 1: [p_k, end_k) unsafe, refine 0, stop;
//   R > 1: h_k = first position >= p_k that is not known and whose n_req is outside [2, R] (n_req = 1
//          re-checks the centre at tau, which is `negative` and fails); the non-known positions of
//          [p_k, h_k) are the candidates of the refined check, q_k the first of them whose check fails
//          (else h_k); [p_k, q_k) is safe with refine n_req (1 where known), and if q_k < end_k the rest
//          of the batch is unsafe with refine 0 and the loop stops.
// Later batches keep S0 / R0; the initial set ends safe with refine 1.
//
// No batch after the first k with h_k < end_k can be reached, so the candidates are only marked up to
// that k (k_stop) and the caller evaluates the refined check there alone.  Four launches, each one CTA per
// batch with a strided loop inside, so any batch size works:
//   scan     p_k, h_k; integer atomicMin of k_stop          (slb_no_shrink_scan)
//   mark     candidate mask in grid order, every point written once
//   q        q_k for k <= k_stop; integer atomicMin of the stop batch k*   (slb_no_shrink_resolve)
//   apply    safe / refinement in grid order, c_max's sorted position and value
// Each minimum is one integer, so the result does not depend on the CTAs' order.
#include "common.cuh"

#include <cmath>

namespace {

constexpr int NT = 256;
constexpr unsigned long long NONE = ~0ull;   // no stopping batch

struct ns_in {
    const int64_t* order;
    const uint8_t* negative;
    const uint8_t* prev_safe;
    const uint8_t* initial;   // may be null
    const double* n_req;      // null when R == 1
    int64_t n, batch, R;
};

// workspace: [0] k_stop, [1] k* (unsigned, NONE when absent), then (p_k, h_k, q_k) per batch
__device__ __forceinline__ int64_t* batch_slot(int64_t* ws, int64_t k) { return ws + 2 + 3 * k; }

__device__ __forceinline__ bool is_known(const ns_in& a, int64_t g) {
    return a.negative[g] || (a.initial != nullptr && a.initial[g]);
}

// First position in [lo, hi) where pred holds, else hi; the same value in every thread of the CTA.
template <class Pred>
__device__ int64_t block_first(int64_t lo, int64_t hi, Pred pred) {
    __shared__ int s_warp[NT / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int64_t base = lo; base < hi; base += NT) {
        const int64_t pos = base + threadIdx.x;
        const bool hit = pos < hi && pred(pos);
        const unsigned b = __ballot_sync(0xffffffffu, hit);
        if (lane == 0) s_warp[warp] = b ? warp * 32 + __ffs(b) - 1 : NT;
        __syncthreads();
        int first = NT;
        for (int w = 0; w < NT / 32; ++w) first = min(first, s_warp[w]);
        __syncthreads();
        if (first < NT) return base + first;
    }
    return hi;
}

__global__ void __launch_bounds__(NT) ns_scan_kernel(ns_in a, int64_t* ws) {
    const int64_t k = blockIdx.x, start = k * a.batch, end = min(start + a.batch, a.n);
    const int64_t p = block_first(start, end, [&](int64_t pos) {
        const int64_t g = a.order[pos];
        return !(a.prev_safe[g] || a.negative[g]);
    });
    int64_t h = p;
    if (a.R > 1 && p < end) {
        const double R = (double)a.R;
        h = block_first(p, end, [&](int64_t pos) {
            const int64_t g = a.order[pos];
            const double r = a.n_req[g];
            return !is_known(a, g) && !(r >= 2.0 && r <= R);
        });
    }
    if (threadIdx.x == 0) {
        batch_slot(ws, k)[0] = p;
        batch_slot(ws, k)[1] = h;
        if (h < end) atomicMin((unsigned long long*)ws, (unsigned long long)k);
    }
}

__global__ void __launch_bounds__(NT) ns_mark_kernel(ns_in a, const int64_t* ws, uint8_t* cand) {
    const int64_t k = blockIdx.x, start = k * a.batch, end = min(start + a.batch, a.n);
    const bool live = (unsigned long long)k <= ((const unsigned long long*)ws)[0];
    const int64_t p = ws[2 + 3 * k], h = ws[2 + 3 * k + 1];
    for (int64_t pos = start + threadIdx.x; pos < end; pos += NT) {
        const int64_t g = a.order[pos];
        cand[g] = (uint8_t)(live && pos >= p && pos < h && !is_known(a, g));
    }
}

__global__ void __launch_bounds__(NT) ns_q_kernel(ns_in a, const uint8_t* refined, int64_t* ws) {
    const int64_t k = blockIdx.x, end = min(k * a.batch + a.batch, a.n);
    if ((unsigned long long)k > ((const unsigned long long*)ws)[0]) return;   // never reached
    int64_t* slot = batch_slot(ws, k);
    const int64_t q = block_first(slot[0], slot[1], [&](int64_t pos) {
        const int64_t g = a.order[pos];
        return !is_known(a, g) && !refined[g];
    });
    if (threadIdx.x == 0) {
        slot[2] = q;
        if (q < end) atomicMin((unsigned long long*)(ws + 1), (unsigned long long)k);
    }
}

__global__ void __launch_bounds__(NT) ns_apply_kernel(ns_in a, const double* values, const int64_t* prev_refine,
                                                      const int64_t* ws, uint8_t* safe, int64_t* refinement,
                                                      int64_t* cmax_position, double* cmax) {
    const int64_t nb = (a.n + a.batch - 1) / a.batch;
    const unsigned long long kstar = ((const unsigned long long*)ws)[1];
    const int64_t k = blockIdx.x, start = k * a.batch, end = min(start + a.batch, a.n);
    if (k < nb) {
        const bool reached = (unsigned long long)k <= kstar;
        const int64_t p = reached ? ws[2 + 3 * k] : end;
        const int64_t q = (unsigned long long)k == kstar ? ws[2 + 3 * k + 2] : end;
        for (int64_t pos = start + threadIdx.x; pos < end; pos += NT) {
            const int64_t g = a.order[pos];
            bool s;
            int64_t r;
            if (!reached) {
                s = a.prev_safe[g];
                r = prev_refine[g];
            } else if (pos < p) {
                s = true;
                r = a.negative[g] ? 1 : prev_refine[g];
            } else if (pos < q) {   // verified by the refinement: candidates hold n_req in [2, R]
                s = true;
                r = is_known(a, g) ? 1 : (int64_t)a.n_req[g];
            } else {
                s = false;
                r = 0;
            }
            if (a.initial != nullptr && a.initial[g]) {
                s = true;
                r = 1;
            }
            safe[g] = (uint8_t)s;
            refinement[g] = r;
        }
    }
    if (k == 0 && threadIdx.x == 0) {
        // start + bound + refine_bound - 1 of the last batch processed (lyapunov.py:589)
        int64_t pos = -1;
        if (kstar != NONE) {
            pos = ws[2 + 3 * (int64_t)kstar + 2] - 1;
        } else if (nb > 0) {
            const int64_t last = nb - 1;
            pos = ws[2 + 3 * last] == a.n ? last * a.batch - 1 : a.n - 1;
        }
        *cmax_position = pos;
        *cmax = a.n == 0 ? NAN : values[a.order[pos < 0 ? a.n - 1 : pos]];
    }
}

int check_common(const char* who, const int64_t* order, const uint8_t* negative, const uint8_t* prev_safe,
                 const double* n_req, int64_t n, int64_t batch, int64_t R, void* ws) {
    SLB_CHECK(n >= 0, "%s: negative n (%lld)", who, (long long)n);
    SLB_CHECK(batch >= 1, "%s: batch size %lld < 1", who, (long long)batch);
    SLB_CHECK(R >= 1, "%s: max_refinement %lld < 1", who, (long long)R);
    SLB_CHECK(ws != nullptr, "%s: null workspace", who);
    SLB_CHECK(n == 0 || (order && negative && prev_safe), "%s: null order/negative/prev_safe", who);
    SLB_CHECK(n == 0 || R == 1 || n_req, "%s: null n_req with max_refinement %lld > 1", who, (long long)R);
    SLB_CHECK((n + batch - 1) / batch <= 0x7fffffff, "%s: %lld batches exceed one launch", who,
              (long long)((n + batch - 1) / batch));
    return 0;
}

}  // namespace

extern "C" {

int64_t slb_no_shrink_workspace(int64_t n, int64_t batch) {
    if (n < 0 || batch < 1) return -1;
    return (int64_t)sizeof(int64_t) * (2 + 3 * ((n + batch - 1) / batch));
}

int slb_no_shrink_scan(void* stream, const int64_t* order_dev, const uint8_t* negative_dev,
                       const uint8_t* prev_safe_dev, const uint8_t* initial_dev, const double* n_req_dev,
                       int64_t n, int64_t batch, int64_t max_refinement, void* workspace_dev,
                       uint8_t* candidates_dev) {
    const char* who = "slb_no_shrink_scan";
    if (check_common(who, order_dev, negative_dev, prev_safe_dev, n_req_dev, n, batch, max_refinement,
                     workspace_dev))
        return 1;
    SLB_CHECK(n == 0 || candidates_dev, "%s: null candidates", who);
    cudaStream_t st = (cudaStream_t)stream;
    SLB_CUDA(cudaMemsetAsync(workspace_dev, 0xff, 2 * sizeof(int64_t), st));
    const int64_t nb = (n + batch - 1) / batch;
    if (nb == 0) return 0;
    const ns_in a{order_dev, negative_dev, prev_safe_dev, initial_dev, n_req_dev, n, batch, max_refinement};
    ns_scan_kernel<<<(unsigned)nb, NT, 0, st>>>(a, (int64_t*)workspace_dev);
    SLB_LAUNCH_CHECK();
    ns_mark_kernel<<<(unsigned)nb, NT, 0, st>>>(a, (const int64_t*)workspace_dev, candidates_dev);
    SLB_LAUNCH_CHECK();
    return 0;
}

int slb_no_shrink_resolve(void* stream, const int64_t* order_dev, const double* values_dev,
                          const uint8_t* negative_dev, const uint8_t* prev_safe_dev,
                          const int64_t* prev_refinement_dev, const uint8_t* initial_dev,
                          const double* n_req_dev, const uint8_t* refined_dev, int64_t n, int64_t batch,
                          int64_t max_refinement, void* workspace_dev, uint8_t* safe_dev,
                          int64_t* refinement_dev, int64_t* cmax_position_dev, double* cmax_dev) {
    const char* who = "slb_no_shrink_resolve";
    if (check_common(who, order_dev, negative_dev, prev_safe_dev, n_req_dev, n, batch, max_refinement,
                     workspace_dev))
        return 1;
    SLB_CHECK(n == 0 || (values_dev && prev_refinement_dev && refined_dev), "%s: null values/prev_refinement/refined",
              who);
    SLB_CHECK(n == 0 || (safe_dev && refinement_dev), "%s: null safe/refinement output", who);
    SLB_CHECK(cmax_position_dev && cmax_dev, "%s: null c_max output", who);
    cudaStream_t st = (cudaStream_t)stream;
    SLB_CUDA(cudaMemsetAsync((int64_t*)workspace_dev + 1, 0xff, sizeof(int64_t), st));
    const int64_t nb = (n + batch - 1) / batch;
    const ns_in a{order_dev, negative_dev, prev_safe_dev, initial_dev, n_req_dev, n, batch, max_refinement};
    if (nb > 0) {
        ns_q_kernel<<<(unsigned)nb, NT, 0, st>>>(a, refined_dev, (int64_t*)workspace_dev);
        SLB_LAUNCH_CHECK();
    }
    ns_apply_kernel<<<(unsigned)(nb > 0 ? nb : 1), NT, 0, st>>>(a, values_dev, prev_refinement_dev,
                                                                (const int64_t*)workspace_dev, safe_dev,
                                                                refinement_dev, cmax_position_dev, cmax_dev);
    SLB_LAUNCH_CHECK();
    return 0;
}

}  // extern "C"
