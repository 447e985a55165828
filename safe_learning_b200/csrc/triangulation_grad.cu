// triangulation_grad.cu -- the transpose of the vertex-table lookups: the gradient of tri(x) (Triangulation)
// or pwc(x) (PiecewiseConstant) with respect to the vertex values (the reference gets it from tf.gradients
// through the tf.gather of functions.py:1494-1499; trained in tests/test_rl.py:29-77 and
// examples/basic_dynamic_programming.ipynb), the rows of _Triangulation.parameter_derivative
// (functions.py:1228-1259) and GridWorld.state_to_index (functions.py:733-752).
//
// For points x_p with cotangent g [n, out], G[v, o] = sum_p sum_k [c_pk = v] w_pk g_po, where (c_pk, w_pk),
// k = 0..R-1, are the rows of the forward evaluation.  Triangulation: R = d + 1 vertices and barycentric
// weights, tri_lookup<TRI_WEIGHTS>, the same lookup and arithmetic as TRI_EVAL (projection, corner_simplex
// table and the Q6 choice included, no TRI_CELL repair).  PiecewiseConstant: R = 1, the nearest vertex
// (grid_nearest_index) with weight 1; a point with a NaN coordinate has none and its key names vertex
// nindex, which no vertex's segment reaches.  Three steps, no floating-point atomics:
//   (1) rows:  one thread per point writes w[j] and the key (c_j << jbits) | j, j = p R + k;
//   (2) sort:  cub::DeviceRadixSort over the key's vbits + jbits bits.  The keys are unique, so the
//              sorted order is the one order "by vertex, then by j" whatever the sort's stability;
//   (3) sum:   one thread per vertex binary-searches its segment and adds w_j g_{p(j), o} in ascending j,
//              from +0.0, one rounding per product and per sum: bit for bit
//              np.add.at(G, c.ravel(), (w[..., None] * g[:, None, :]).reshape(-1, out)) (for R = 1,
//              w = 1 and the product is exact: np.add.at(G, c, g)).
//              Every vertex is written (zeros included), so G needs no memset.
// A thread walks its vertex's whole segment: when all n points clip to one vertex, that thread adds
// n R terms serially (the cost of the determinism; ordinary batches spread over the table).
#include "common.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <string.h>

namespace {

constexpr int NT = 256;

int bit_width(uint64_t x) { return x == 0 ? 0 : 64 - __builtin_clzll(x); }

// rows of the point's forward lookup per point: d + 1 simplex vertices, or the one nearest vertex
int rows_per_point(const slb_function& f) { return f.kind == SLB_FN_PIECEWISE_CONSTANT ? 1 : f.grid.ndim + 1; }

__global__ void __launch_bounds__(NT) tri_rows_kernel(const __grid_constant__ slb_function f,
                                                      const double* __restrict__ x, int64_t n,
                                                      int64_t* __restrict__ cols, uint64_t* __restrict__ keys,
                                                      int jbits, double* __restrict__ weights,
                                                      double* __restrict__ out) {
    const int64_t p = (int64_t)blockIdx.x * NT + threadIdx.x;
    if (p >= n) return;
    const int d = f.grid.ndim;
    double xin[SLB_MAX_DIM], w[SLB_MAX_DIM + 1];
    for (int c = 0; c < d; ++c) xin[c] = x[p * d + c];
    if (f.kind == SLB_FN_PIECEWISE_CONSTANT) {
        const int64_t v = grid_nearest_index(f.grid, f.cparams, xin);
        if (weights != nullptr) weights[p] = 1.0;
        if (cols != nullptr) cols[p] = v;
        if (keys != nullptr) keys[p] = ((uint64_t)(v < 0 ? f.grid.nindex : v) << jbits) | (uint64_t)p;
        if (out != nullptr)                     // eval_fn's row gather
            for (int o = 0; o < f.out_dim; ++o)
                out[p * f.out_dim + o] = v < 0 ? __longlong_as_double(0x7ff8000000000000ll)
                                               : f.matrix[v * f.out_dim + o];
        return;
    }
    int64_t corner;
    int simplex;
    tri_lookup<TRI_WEIGHTS>(f, xin, w, &corner, &simplex);
    const int64_t* simp = f.unit_simplices + (size_t)simplex * (d + 1);
    for (int k = 0; k <= d; ++k) {
        const int64_t j = p * (d + 1) + k;
        const int64_t v = simp[k] + corner;
        if (weights != nullptr) weights[j] = w[k];
        if (cols != nullptr) cols[j] = v;
        if (keys != nullptr) keys[j] = ((uint64_t)v << jbits) | (uint64_t)j;
    }
    if (out != nullptr) {                       // TRI_EVAL's gather, same order and roundings
        const int od = f.out_dim;
        for (int o = 0; o < od; ++o) {
            double v = f64mul(w[0], f.matrix[(simp[0] + corner) * od + o]);
            for (int k = 1; k <= d; ++k) v = f64add(v, f64mul(w[k], f.matrix[(simp[k] + corner) * od + o]));
            out[p * od + o] = v;
        }
    }
}

__global__ void __launch_bounds__(NT) tri_sum_kernel(const uint64_t* __restrict__ keys, int64_t nkeys, int jbits,
                                                     int dp1, const double* __restrict__ weights,
                                                     const double* __restrict__ g, int od, int64_t nindex,
                                                     double* __restrict__ grad) {
    const int64_t v = (int64_t)blockIdx.x * NT + threadIdx.x;
    if (v >= nindex) return;
    const uint64_t first = (uint64_t)v << jbits, mask = (1ull << jbits) - 1;
    int64_t lo = 0, hi = nkeys;                 // first key >= first
    while (lo < hi) {
        const int64_t mid = lo + (hi - lo) / 2;
        if (keys[mid] < first) lo = mid + 1;
        else hi = mid;
    }
    for (int o = 0; o < od; ++o) {
        double acc = 0.0;
        for (int64_t i = lo; i < nkeys; ++i) {
            const uint64_t key = keys[i];
            if ((key >> jbits) != (uint64_t)v) break;
            const int64_t j = (int64_t)(key & mask);
            acc = f64add(acc, f64mul(weights[j], g[(j / dp1) * od + o]));
        }
        grad[v * od + o] = acc;
    }
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// bits of the vertex part of a key: vertices 0 .. nindex - 1, and for a PiecewiseConstant also nindex (the
// key of a point without a vertex)
int vertex_bits(const slb_function& f) {
    return bit_width((uint64_t)(f.kind == SLB_FN_PIECEWISE_CONSTANT ? f.grid.nindex : f.grid.nindex - 1));
}

// key layout: jbits low bits for j = p R + k, the vertex above them
int key_bits(const slb_function& f, int64_t n, int* jbits, const char* what) {
    const int64_t nkeys = n * rows_per_point(f);
    *jbits = bit_width((uint64_t)(nkeys - 1));
    const int vbits = vertex_bits(f);
    SLB_CHECK(*jbits + vbits <= 64,
              "%s: the sort key of %lld points on %lld vertices needs %d + %d > 64 bits (split the batch)",
              what, (long long)n, (long long)f.grid.nindex, vbits, *jbits);
    return 0;
}

// bytes of the keys (in, out), the weights and cub's scratch, in that order
int workspace_layout(int64_t nkeys, int end_bit, size_t* cub_bytes, size_t* total) {
    *cub_bytes = 0;
    SLB_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, *cub_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                                            nkeys, 0, end_bit));
    *total = 3 * align256((size_t)nkeys * 8) + align256(*cub_bytes);
    return 0;
}

}  // namespace

// ---- called by slb_function_vjp / slb_function_vjp_workspace (network_grad.cu) for SLB_FN_TRIANGULATION and
// SLB_FN_PIECEWISE_CONSTANT, after the descriptor, the flags and n >= 0 were checked
int64_t slb_triangulation_vjp_workspace(const slb_function* fn, int64_t n) {
    if (n == 0) return 0;
    int jbits;
    if (key_bits(*fn, n, &jbits, "slb_function_vjp_workspace")) return -1;
    const int end_bit = jbits + vertex_bits(*fn);
    size_t cub_bytes, total;
    if (workspace_layout(n * rows_per_point(*fn), end_bit, &cub_bytes, &total)) return -1;
    return (int64_t)total;
}

int slb_triangulation_vjp(cudaStream_t st, const slb_function* fn, const double* points_dev, int64_t n,
                          const double* grad_out_dev, double* grad_in_dev, double* grad_params_dev,
                          double* out_dev, void* workspace_dev) {
    SLB_CHECK(grad_in_dev == nullptr || fn->kind != SLB_FN_TRIANGULATION,
              "slb_function_vjp: grad_in must be NULL for a Triangulation (its point gradient is the "
              "SLB_FLAG_GRADIENT evaluation)");
    SLB_CHECK(grad_in_dev == nullptr,
              "slb_function_vjp: grad_in must be NULL for a PiecewiseConstant (its point gradient is 0)");
    const int64_t nindex = fn->grid.nindex;
    const int od = fn->out_dim, R = rows_per_point(*fn);
    if (n == 0) {
        if (grad_params_dev != nullptr)
            SLB_CUDA(cudaMemsetAsync(grad_params_dev, 0, (size_t)nindex * od * sizeof(double), st));
        return 0;
    }
    int jbits;
    if (key_bits(*fn, n, &jbits, "slb_function_vjp")) return 1;
    SLB_CHECK(grad_params_dev == nullptr || workspace_dev != nullptr,
              "slb_function_vjp: a vertex table's gradient needs slb_function_vjp_workspace bytes of workspace");
    if (grad_params_dev == nullptr && out_dev == nullptr) return 0;
    const int64_t nkeys = n * R;
    const unsigned blocks = (unsigned)((n + NT - 1) / NT);
    if (grad_params_dev == nullptr) {           // forward only
        tri_rows_kernel<<<blocks, NT, 0, st>>>(*fn, points_dev, n, nullptr, nullptr, 0, nullptr, out_dev);
        SLB_LAUNCH_CHECK();
        return 0;
    }
    const int end_bit = jbits + vertex_bits(*fn);
    size_t cub_bytes, total;
    if (workspace_layout(nkeys, end_bit, &cub_bytes, &total)) return 2;
    char* ws = (char*)workspace_dev;
    const size_t slab = align256((size_t)nkeys * 8);
    uint64_t* keys_in = (uint64_t*)ws;
    uint64_t* keys_out = (uint64_t*)(ws + slab);
    double* weights = (double*)(ws + 2 * slab);
    void* scratch = ws + 3 * slab;
    tri_rows_kernel<<<blocks, NT, 0, st>>>(*fn, points_dev, n, nullptr, keys_in, jbits, weights, out_dev);
    SLB_LAUNCH_CHECK();
    SLB_CUDA(cub::DeviceRadixSort::SortKeys(scratch, cub_bytes, keys_in, keys_out, nkeys, 0, end_bit, st));
    slb_count_launch();
    tri_sum_kernel<<<(unsigned)((nindex + NT - 1) / NT), NT, 0, st>>>(keys_out, nkeys, jbits, R, weights,
                                                                       grad_out_dev, od, nindex, grad_params_dev);
    SLB_LAUNCH_CHECK();
    return 0;
}

extern "C" int slb_triangulation_rows(void* stream, const slb_function* fn, const double* points_dev, int64_t n,
                                      int64_t* cols_dev, double* weights_dev) {
    SLB_CHECK(fn != nullptr, "slb_triangulation_rows: null function");
    SLB_CHECK(fn->kind == SLB_FN_TRIANGULATION, "slb_triangulation_rows: function kind %d is not a Triangulation",
              fn->kind);
    SLB_CHECK((fn->flags & ~SLB_FLAG_PROJECT) == 0,
              "slb_triangulation_rows: post-op flags 0x%x (only the projection applies)", fn->flags);
    if (slb_validate_function(fn, "slb_triangulation_rows", 0)) return 1;
    SLB_CHECK(n >= 0, "slb_triangulation_rows: negative n (%lld)", (long long)n);
    if (n == 0) return 0;
    SLB_CHECK(points_dev && cols_dev && weights_dev, "slb_triangulation_rows: null buffer");
    tri_rows_kernel<<<(unsigned)((n + NT - 1) / NT), NT, 0, (cudaStream_t)stream>>>(
        *fn, points_dev, n, cols_dev, nullptr, 0, weights_dev, nullptr);
    SLB_LAUNCH_CHECK();
    return 0;
}

extern "C" int slb_grid_nearest_index(void* stream, const slb_grid* grid, const double* points_dev, int64_t n,
                                      int64_t* idx_dev) {
    SLB_CHECK(grid != nullptr, "slb_grid_nearest_index: null grid");
    if (slb_validate_grid(grid, false)) return 1;
    SLB_CHECK(n >= 0, "slb_grid_nearest_index: negative n (%lld)", (long long)n);
    // the lookup of a PiecewiseConstant on this grid, with numpy's 1. / unit_maxes (IEEE division)
    slb_function f;
    memset(&f, 0, sizeof(f));
    f.kind = SLB_FN_PIECEWISE_CONSTANT;
    f.grid = *grid;
    for (int c = 0; c < grid->ndim; ++c) {
        f.cparams[c] = 1.0 / grid->unit_maxes[c];
        SLB_CHECK(f.cparams[c] > 0.0 && f.cparams[c] < INFINITY,
                  "slb_grid_nearest_index: unit_maxes[%d] = %g has no positive finite inverse", c,
                  grid->unit_maxes[c]);
    }
    if (n == 0) return 0;
    SLB_CHECK(points_dev && idx_dev, "slb_grid_nearest_index: null buffer");
    tri_rows_kernel<<<(unsigned)((n + NT - 1) / NT), NT, 0, (cudaStream_t)stream>>>(
        f, points_dev, n, idx_dev, nullptr, 0, nullptr, nullptr);
    SLB_LAUNCH_CHECK();
    return 0;
}
