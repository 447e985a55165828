/*
 * slb200.h -- C ABI of libslb200.so: the H100 (sm_90a) implementation of the
 * safe_learning region-of-attraction hot path.
 *
 * The reference (befelix/safe_learning @ f1aad5a) has no FFI: the path sits behind
 * Python classes that build a TF1 graph and call Session.run once per 10 000-point
 * batch.  The entry points below are what a binding for that path would bind; each
 * cites the reference code it replaces (paths relative to the upstream sources).  The
 * Python host side (safe_learning_b200/) loads this library with ctypes -- see
 * INTEGRATION.md for the stub a maintainer of the reference would add.
 *
 * Conventions
 *   - plain C: pointers, sizes, POD structs passed by pointer; no torch/C++ types.
 *   - every `*_dev` / `const double*` inside a struct is a DEVICE pointer (fp64,
 *     row-major, contiguous) owned by the caller; the library never allocates or frees.
 *   - `stream` is a cudaStream_t (CUstream) cast to void*; calls enqueue and return.
 *   - return 0 on success, non-zero on error; slb_last_error() gives the message.
 *     There is NO CPU fallback: without a CUDA device every compute call fails.
 *   - fp64 everywhere (safe_learning/configuration.py:16); flags are uint8; flat grid
 *     indices int64 with the last dimension fastest (functions.py:622-638).
 */
#ifndef SLB200_H
#define SLB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SLB_ABI_VERSION 6   /* 2: slb_gp_factor.kernel (covariance expressions), GRADIENT / MAXABS flags
                               3: decision filter (slb_gp_factor.Whead, slb_lyapunov_sweep_filtered),
                                  state-dependent lipschitz_dynamics, peer-memory key exchange
                                  (slb_exchange), fixed-action Bellman tables
                               4: filter tables staged by TMA bulk copies (slb_gp_factor.Xf / Xhead /
                                  head_rows / hmax, slb_gp_output.gamma_f / gamma_l1): pivoted head
                                  subset, computed error bound of the filter's mean
                               5: fp32 screening stage in front of the filter (slb_debug_screening_probe,
                                  bit 2 of slb_debug_filter_stages); no structure changed
                               6: slb_debug_refine_split takes one threshold (no 16-point tiles)    */
#define SLB_MAX_DIM 6   /* state dimension d                         */
#define SLB_MAX_IN  8   /* GP input dimension d_in = d + m           */
#define SLB_MAX_OUT 6   /* stacked one-output GPs (FunctionStack)    */
#define SLB_MAX_ACT 2   /* action dimension m                        */
#define SLB_TILE_POINTS 64  /* grid points per CTA tile of the GP kernels */
#define SLB_HEAD_RANK 64    /* size of the training subset behind the decision filter's variance bound */
#define SLB_MAX_RANKS 16    /* ranks of one peer-memory key exchange (one NVSwitch domain)       */

/* ---- GridWorld (functions.py:579-817) ------------------------------------------- */
typedef struct slb_grid {
    int32_t ndim;
    int32_t _pad;
    int64_t nindex;                    /* prod(num_points)                              */
    int64_t num_points[SLB_MAX_DIM];
    double  offset[SLB_MAX_DIM];       /* limits[:, 0]                  (:604)          */
    double  unit_maxes[SLB_MAX_DIM];   /* (hi - lo) / (n - 1)           (:605-606)      */
    double  upper[SLB_MAX_DIM];        /* limits[:, 1]                                  */
    const double* discrete_points;     /* device, concatenated np.linspace values per dim
                                          (:612-614); needed only by SLB_FN_TRIANGULATION */
} slb_grid;

/* ---- function objects fused into the kernels (functions.py, examples/utilities.py) -- */
enum slb_fn_kind {
    SLB_FN_NONE = 0,
    SLB_FN_CONSTANT = 1,       /* ConstantFunction            functions.py:241-251          */
    SLB_FN_LINEAR = 2,         /* LinearSystem  y = x A^T      functions.py:1546-1583        */
    SLB_FN_QUADRATIC = 3,      /* QuadraticFunction sum((xP)*x) functions.py:1513-1539       */
    SLB_FN_TRIANGULATION = 4,  /* Triangulation               functions.py:1103-1158,1442-1499 */
    SLB_FN_PENDULUM = 5,       /* InvertedPendulum            examples/utilities.py:144-289 */
    SLB_FN_CARTPOLE = 6,       /* CartPole                    examples/utilities.py:292-437 */
    SLB_FN_LYAPUNOV_NN = 7,    /* LyapunovNetwork             examples/utilities.py:48-104  */
    SLB_FN_MLP = 8,            /* NeuralNetwork               functions.py:1702-1729        */
    SLB_FN_VANDERPOL = 9,      /* VanDerPol (reverse time)    examples/utilities.py:440-519
                                  maps [x, y, u] (3 inputs, u ignored) to 2 columns; cparams:
                                  [0] damping, [1] dt / 10, [2] 1 if normalised, [3..4] Tx,
                                  [5..6] 1 / Tx.  The normalisation is the reference's
                                  state . diag(T): column j = s_j T_j + s_(1-j) 0, so an inf or
                                  NaN component makes the other column NaN */
    SLB_FN_PIECEWISE_CONSTANT = 10  /* PiecewiseConstant      functions.py:820-932
                                  the row of the nearest grid vertex (GridWorld.state_to_index,
                                  functions.py:733-752): clip to the limits, (x - offset) * inv,
                                  np.rint (half to even), ravel.  matrix = vertex values
                                  [nindex, out]; grid = the discretization (discrete_points not
                                  needed); in_dim = grid.ndim; cparams[0..d-1] = inv = 1. /
                                  unit_maxes as numpy computes it.  A row with a NaN coordinate
                                  gives NaN in every column (the reference raises) */
};
/* post-ops, applied in this order: saturate -> abs -> norm1 | maxabs -> out_scale */
#define SLB_FLAG_SATURATE 1u   /* Saturation  functions.py:349-354                     */
#define SLB_FLAG_ABS      2u   /* tf.abs(fun(x))     (notebook Lipschitz lambdas)      */
#define SLB_FLAG_NORM1    4u   /* tf.norm(., ord=1, axis=1, keepdims=True)             */
#define SLB_FLAG_PROJECT  8u   /* Triangulation(project=True) functions.py:1479-1485  */
#define SLB_FLAG_SCALE   16u   /* multiply by out_scale (MultipliedFunction / __neg__) */
#define SLB_FLAG_GRADIENT 32u  /* TRIANGULATION with one output column: return the d partial
                                  derivatives of the piecewise-linear interpolant instead of its
                                  value (Triangulation.gradient, functions.py:1260-1326, 1506-1510);
                                  out_dim = d.
                                  LYAPUNOV_NN, or MLP whose output width is 1: return the input
                                  gradient d f / d x (tf.gradients(V(x), x), the Lipschitz lambda of
                                  lyapunov_function_learning.ipynb cell 19), in_dim columns before
                                  any NORM1 / MAXABS / SCALE; out_dim = in_dim <= SLB_MAX_OUT.  Equal
                                  bit for bit to slb_function_vjp's grad_in for grad_out = 1, which
                                  rejects the flag (its VJP would be a Hessian-vector product) */
#define SLB_FLAG_MAXABS  64u   /* tf.reduce_max(tf.abs(.), axis=1, keepdims=True): the
                                  Lipschitz lambda of examples/inverted_pendulum.ipynb cell 14;
                                  applied after saturate, reduces to 1 column              */

typedef struct slb_function {
    int32_t kind;
    int32_t in_dim;
    int32_t out_dim;            /* before NORM1 / MAXABS (which reduce to 1 column)    */
    uint32_t flags;
    double  out_scale;
    double  lower, upper;       /* saturation bounds                                   */
    double  cparams[24];        /* CONSTANT: value; PENDULUM/CARTPOLE: plant constants
                                   (see safe_learning_b200/functions.py); LYAPUNOV_NN / MLP:
                                   [0] layers, [1+i] width of layer i (<= 64), [9+i] activation
                                   (0 tanh, 1 relu, 2 identity); MLP: [17] output_scale, [18] 1 if
                                   hidden layers carry a bias (matrix = [W_i (out x in), b_i] ...) */
    const double*  matrix;      /* LINEAR [out,in]; QUADRATIC [in,in]; TRIANGULATION and
                                   PIECEWISE_CONSTANT vertex values [nindex,out]; LYAPUNOV_NN
                                   packed kernels */
    const double*  hyperplanes; /* TRIANGULATION [nsimplex, d, d]  (functions.py:1090-1101) */
    const int64_t* unit_simplices; /* TRIANGULATION [nsimplex, d+1] (functions.py:1064-1088) */
    const int32_t* corner_simplex; /* TRIANGULATION [2^d] or NULL: Qhull's find_simplex answer for
                                      a query clipped in EVERY dimension (bit c set = clipped to
                                      the upper limit); such points sit on a unit-cell corner
                                      where several simplices meet and extrapolation differs  */
    int32_t nsimplex;
    int32_t _pad;
    slb_grid grid;              /* TRIANGULATION / PIECEWISE_CONSTANT discretization   */
} slb_function;

/* ---- covariance functions ------------------------------------------------------------------
 * The reference hands any gpflow kernel to GPRCached (functions.py:370-393) and only ever calls
 * kern.K(X), kern.K(X, Xnew) and kern.Kdiag(Xnew) on it (functions.py:399, 438, 450).  Its
 * experiments use sums of products of gpflow==0.4.0 primitives with `active_dims`
 * (examples/inverted_pendulum.ipynb cell 6, adaptive_safety_verification.ipynb cell 9,
 * 1d_region_of_attraction_estimate.ipynb cell 5):
 *     k(x, x') = sum over terms t of  prod over primitives p with p.term == t of  k_p(x, x')
 * gpflow 0.4.0 kernels.py arithmetic of the primitives (r^2 = sum_c ((x_c - x'_c) w_c)^2 with
 * w_c = 1 / lengthscale_c on active dimensions and 0 elsewhere; r = sqrt(r^2 + 1e-12)):          */
enum slb_kernel_kind {
    SLB_K_RBF = 0,        /* variance exp(-r^2 / 2)                                          */
    SLB_K_MATERN12 = 1,   /* variance exp(-r)                                                */
    SLB_K_MATERN32 = 2,   /* variance (1 + sqrt3 r) exp(-sqrt3 r)                            */
    SLB_K_MATERN52 = 3,   /* variance (1 + sqrt5 r + 5/3 r^2) exp(-sqrt5 r)                  */
    SLB_K_LINEAR = 4,     /* sum_c w_c x_c x'_c, w_c = variance_c on active dims (ARD or not) */
    SLB_K_CONSTANT = 5,   /* variance (gpflow Constant / Bias)                               */
    SLB_K_WHITE = 6       /* variance on the diagonal (Kdiag, K(X)); 0 against new points    */
};
#define SLB_MAX_KPRIM 6

typedef struct slb_kernel_prim {
    int32_t kind;               /* slb_kernel_kind                                      */
    int32_t term;               /* product term; primitives are listed in term order    */
    double  variance;           /* stationary / constant / white primitives             */
    double  w[SLB_MAX_IN];      /* per input column, see above; 0 = inactive dimension  */
} slb_kernel_prim;

typedef struct slb_kernel {
    int32_t num_prims;          /* 0 => the factor is the plain full-dimensional RBF described
                                   by slb_gp_factor.lengthscales / variance / kss (fast path)  */
    int32_t _pad;
    slb_kernel_prim prims[SLB_MAX_KPRIM];
} slb_kernel;

/* ---- GP stack: FunctionStack of GaussianProcess(GPRCached) (functions.py:254-546) ---- */
typedef struct slb_gp_factor {
    int32_t M;                  /* training points; 0 => prior only (empty data set of the
                                   notebooks before the first add_data_point)           */
    int32_t nrb;                /* ceil(M / 8) row blocks of the packed factor          */
    const double* Xs;           /* device [M, d_in]: X / lengthscales when kernel.num_prims == 0
                                   (gpflow RBF), the raw X otherwise                    */
    const double* Wpack;        /* device: L^-1 in DMMA fragment order, k-steps paired
                                   (slb_pack_factor); L = chol(scale^2 (K + noise I))
                                   functions.py:399-408 */
    double lengthscales[SLB_MAX_IN];
    double variance;            /* RBF variance (Kdiag)                                 */
    double scale;               /* GPRCached _scale                functions.py:392     */
    double kss;                 /* (scale**2) * variance           functions.py:450     */
    slb_kernel kernel;          /* general covariance expression (num_prims > 0)        */
    /* ---- tables of the decision filter (slb_lyapunov_sweep_filtered); may be NULL / 0 if that
       call is not used.  The posterior variance given ANY subset S of the training set is an upper
       bound of the full posterior variance; the host picks up to SLB_HEAD_RANK points in pivoted-
       Cholesky (greedy max-variance) order and factors them on their own:                        */
    const double* Whead;        /* device [SLB_HEAD_RANK, SLB_HEAD_RANK], COLUMN-major, zero padded:
                                   Whead[j * SLB_HEAD_RANK + i] = L_S^-1[i, j], L_S = chol(scale^2
                                   (K(X_S) + noise I))                                   */
    const double* Wheadp;       /* device, 16-byte aligned: the same L_S^-1 (zero padded to SLB_HEAD_RANK^2) in
                                   DMMA.8x8x4 A-fragment order: for row block b (8 rows) and k-step s
                                   (4 columns) 32 doubles, lane T <-> L_S^-1[8b + T/4, 4s + T%4], block
                                   offset (b * (SLB_HEAD_RANK / 4) + s) * 32                */
    const double* Xhead;        /* device [SLB_HEAD_RANK, d_in], zero padded: the subset's inputs,
                                   scaled like Xs                                        */
    int32_t head_rows;          /* |S| = min(M, SLB_HEAD_RANK)                           */
    int32_t _pad2;
    const double* Xf;           /* device [8 ceil(M/8), w], zero padded, 16-byte aligned (TMA bulk
                                   copies): kernel.num_prims == 0: w = d_in + 1, row j =
                                   (Xs[j, :], -|Xs[j, :]|^2 / 2); otherwise w = d_in, the raw X  */
    double hmax;                /* max_j |Xs[j, :]|^2 / 2 (rounding bound of the expanded distance) */
} slb_gp_factor;

typedef struct slb_gp_output {
    int32_t factor;             /* index into factors[] (outputs sharing X, kernel and
                                   noise share one factor)                              */
    int32_t _pad;
    double  beta;               /* GaussianProcess.beta            functions.py:487,514 */
    const double* alpha;        /* device [8*nrb]: L^-1 scale (Y - m(X)), zero padded
                                                                    functions.py:405-409 */
    const double* gamma;        /* device [M]: L^-T alpha (mean-only Bellman path)      */
    const double* prior_mean;   /* device [d_in] linear prior-mean row, or NULL         */
    const double* gamma_f;      /* device [8 ceil(M/8)], zero padded, 16-byte aligned: the filter's
                                   mean weights, scale^2 gamma (times the RBF variance when
                                   kernel.num_prims == 0, whose kernel values are then <= 1)   */
    double gamma_l1;            /* >= sum_i (|L^-1|^T |alpha|)_i in the units of gamma_f: bounds the
                                   rounding error of every way of summing the mean (filter)    */
} slb_gp_output;

typedef struct slb_gp_stack {
    int32_t num_outputs;        /* D; 0 => dynamics are deterministic                   */
    int32_t num_factors;        /* D' distinct Cholesky factors                         */
    int32_t input_dim;          /* d_in                                                 */
    int32_t _pad;
    slb_gp_factor factors[SLB_MAX_OUT];
    slb_gp_output outputs[SLB_MAX_OUT];
} slb_gp_stack;

/* ---- one Lyapunov sweep: the graph of lyapunov.py:433-441 -----------------------------
 * Shapes.  A function's COLUMNS are what it returns after its post-ops: out_dim, except 1 for
 * QUADRATIC and LYAPUNOV_NN, 2 for PENDULUM and VANDERPOL, 4 for CARTPOLE, in_dim for a network gradient
 * (SLB_FLAG_GRADIENT on LYAPUNOV_NN / MLP with out_dim = in_dim), and 1 after NORM1 or MAXABS.  With
 * d = grid.ndim and m = the policy's columns:
 *   policy        d inputs, m = 1..SLB_MAX_ACT columns
 *   dynamics      d + m inputs, d columns                   (gp.num_outputs == 0)
 *   gp            d outputs, input_dim = d + m              (gp.num_outputs > 0)
 *   lyapunov      d inputs
 *   lipschitz_v   d inputs, 1 or d columns                  (or kind NONE)
 *   lipschitz_f   d inputs; L_f is its first column         (or kind NONE)
 * Every sweep entry point rejects a descriptor that breaks them, also for an empty index range. */
typedef struct slb_sweep {
    slb_grid     grid;          /* discretization                                       */
    slb_function policy;        /* x -> u                       lyapunov.py:436         */
    slb_function dynamics;      /* deterministic [x,u] -> x+ when gp.num_outputs == 0   */
    slb_gp_stack gp;            /* uncertain dynamics           lyapunov.py:437         */
    slb_function lyapunov;      /* V                            lyapunov.py:351-352     */
    slb_function lipschitz_v;   /* L_V(.) as a function, or kind NONE => lv_const       */
    double lv_const;            /* scalar lipschitz_lyapunov    lyapunov.py:246-263     */
    double lf_const;            /* scalar lipschitz_dynamics    lyapunov.py:227-244     */
    double tau;                 /* discretization constant      lyapunov.py:195         */
    slb_function lipschitz_f;   /* state-dependent L_f(x) as a fused function (first column), or
                                   kind NONE                    lyapunov.py:227-244, 287 */
    const double* lf_values;    /* device, or NULL: L_f tabulated per flat grid index (an arbitrary
                                   Python callable evaluated once by the host); entry for grid
                                   index i is lf_values[i - lf_index_base].  Index-range sweeps only.
                                   Precedence: lf_values, lipschitz_f, lf_const            */
    int64_t lf_index_base;
} slb_sweep;

/* ---- one Bellman sweep: PolicyIteration.future_values (reinforcement_learning.py:65-114)
 * Shapes (columns as for slb_sweep), with d = grid.ndim and m = the policy's columns, or
 * m = policy.out_dim with fixed_action (the action dimension; the rest of the policy is ignored):
 *   policy        d inputs, m = 1..SLB_MAX_ACT columns
 *   dynamics      d + m inputs, d columns                   (gp.num_outputs == 0)
 *   gp            d outputs, input_dim = d + m              (gp.num_outputs > 0)
 *   reward        d + m inputs, 1 column
 *   value         d inputs, 1 column
 * slb_bellman_sweep, slb_bellman_argmax and slb_value_operator reject a descriptor that breaks them
 * before any work.  The rollouts check their own subset (see slb_rollout). */
typedef struct slb_bellman {
    slb_grid     grid;          /* value_function.discretization (state space, :58-59)  */
    slb_function policy;        /* ignored when fixed_action != 0                       */
    slb_function dynamics;      /* deterministic dynamics when gp.num_outputs == 0      */
    slb_gp_stack gp;            /* GP dynamics: mean only               (:98-99)        */
    slb_function reward;        /* r([x,u])                             (:95)           */
    slb_function value;         /* V as Triangulation or PiecewiseConstant (vertex table =
                                   `matrix`)                           (:101)           */
    double gamma;               /*                                      (:104)          */
    int32_t fixed_action;       /* 1 => use `action` for every state (:266-270)         */
    int32_t _pad;
    double action[SLB_MAX_ACT];
} slb_bellman;


/* ---- result of the first-fail reduction (sort-free form of lyapunov.py:512-587) ------- */
typedef struct slb_fail_key {
    uint64_t key_value;   /* order-preserving bits of V at the first failing point in stable
                             V-order, or UINT64_MAX if no point fails                     */
    int64_t  key_index;   /* its flat grid index, or INT64_MAX                            */
    int64_t  n_ok;        /* number of points with negative | initial                     */
    int64_t  _pad;
} slb_fail_key;

typedef struct slb_prefix_stats {
    int64_t  n_safe;        /* |{key < k*} U initial|                                     */
    int64_t  n_below;       /* |{key < k*}| = sorted position p* of the first failure     */
    uint64_t max_below;     /* order-preserving bits of max{V_i : key_i < k*} (0 if none) */
    uint64_t max_all;       /* order-preserving bits of max V over the range              */
} slb_prefix_stats;

/* ---- per-sweep key exchange between the ranks of one NVLink domain without a collective call:
 *      every rank owns `slots` = slb_fail_key[2][world] in peer-mapped (symmetric) memory; after its
 *      first-fail reduction a rank STORES its key into slot [parity][rank] of every peer (P2P
 *      writes through NVLink) with the sweep's sequence number as the release flag, and the prefix
 *      kernel of every rank waits for the `world` flags of the current sweep in its own copy.
 *      Ranks must issue the same sequence of sweeps (like any collective).                        */
typedef struct slb_exchange {
    int32_t world;
    int32_t rank;
    slb_fail_key* slots[SLB_MAX_RANKS];  /* slots[r]: rank r's slot array as mapped in THIS process */
    int64_t* seq_dev;                    /* local device int64 (zero-initialised): sweeps issued  */
} slb_exchange;

/* ---- library ---------------------------------------------------------------------------- */
int         slb_abi_version(void);
const char* slb_last_error(void);
/* number of CUDA devices visible, or <0 with slb_last_error set */
int         slb_device_count(void);
/* sizeof() of the ABI structs in declaration order (grid, function, gp_factor, gp_output,
   gp_stack, sweep, bellman, fail_key, prefix_stats, exchange); returns how many there are */
int         slb_struct_sizes(int64_t* out, int32_t n);
/* kernels this library has launched since load (bench.py's gpu_launches) */
int64_t     slb_launch_count(void);
/* a caller that replays a CUDA graph captured around `kernels` launches of this library reports
   each replay here so that slb_launch_count stays truthful */
void        slb_note_graph_replay(int64_t kernels);

/* diagnostics: when buffer_dev != NULL, every later Lyapunov sweep writes int64 cycle counts
 * [tile][warp(8)][8] = {k-row generation, DMMA contraction, panel epilogues, whole tile}, the
 * %globaltimer (ns) at tile start / end, cycles spent waiting at block barriers, 0;
 * pass NULL to switch it off (default) */
int         slb_debug_phase_timing(void* buffer_dev);
/* diagnostics: when buffer_dev != NULL (uint64 [133][8], zeroed by the caller), every later filtered
 * sweep raises entry [c][m] to the %globaltimer (ns) at which the last warp of head-stage CTA c passed
 * mark m = {entry, head tables landed, bound of factor 0, bound of every factor, screened decision,
 * fp64 means of the round, final decision, exit}, and [132][0] to the time the last warp of the first
 * stage left (tools/head_stage_timeline.py); pass NULL to switch it off (default) */
int         slb_debug_head_timing(void* buffer_dev);
/* diagnostics: when buffer_dev != NULL (uint64 [tiles][8], zeroed by the caller; tiles = the launch's
 * 16 x 16 tiles), every later filtered sweep whose stage 1 runs the factored grid mean raises entry [t][m]
 * to the %globaltimer (ns) at which the last warp of tile t's CTA passed mark m = {entry, prologue done,
 * work items 0, 1, 2 and 3 (and later) done, means done, exit} (tools/stage1_timeline.py); pass NULL to
 * switch it off (default) */
int         slb_debug_stage1_timing(void* buffer_dev);
/* diagnostics: when buffer_dev != NULL (uint64 [512][16], zeroed by the caller), every later filtered sweep
 * whose refine pass runs row-split 32-point tiles raises entry [c][m] to the %globaltimer (ns) at which the
 * last warp of its CTA c passed mark m = {entry, prologue done, j-panel 0, 1, 2, 3 (and later) generated,
 * j-panel 0, 1, 2, 3 (and later) contracted, partial sums written, ticket taken, factor epilogues done,
 * decision and fold done, exit}, and sets [c][15] = 1 in the CTAs that finished a tile
 * (tools/refine_timeline.py); pass NULL to switch it off (default) */
int         slb_debug_refine_timing(void* buffer_dev);
/* Records an event (owned by the library, one per device) on `stream` that every later launch reading
 * the packed factors (slb_gp_factor.Wpack: the full posterior of slb_gp_predict / slb_lyapunov_sweep /
 * slb_lyapunov_points and the refine pass of slb_lyapunov_sweep_filtered) waits for on ITS stream.  A
 * caller that restores the GP tables from the host copies the packed factors -- 90% of the bytes -- on a
 * second stream, calls this behind the copy, and enqueues the sweep at once: the filter stages do not
 * read the packed factors and overlap the copy.  Under stream capture the wait is an external-event
 * node (re-evaluated at every replay).  Single-threaded use like the other setters. */
int         slb_record_factor_dependency(void* stream);
/* Restore of a packed table arena (safe_learning_b200.functions.PackedCache: every cached GP table of a
 * stack in one device buffer, mirrored by one page-locked host buffer, the packed factors last) in one
 * call: bytes [0, split_bytes) are copied host -> device on `stream`, bytes [split_bytes, total_bytes)
 * -- the packed factors -- on `side_stream` behind everything enqueued on `stream` so far, followed by
 * slb_record_factor_dependency(side_stream).  side_stream NULL (or == stream): one stream, no event. */
int         slb_restore_tables(void* dst_dev, const void* src_host, int64_t split_bytes, int64_t total_bytes,
                               void* stream, void* side_stream);
/* diagnostics (timing of the individual stages of slb_lyapunov_sweep_filtered; the flags are only
 * complete with bits 0 and 1 set -- 3, the default, or 7): bit 0 runs the head stage, bit 1 the
 * refine pass; bit 2 forces the fp64 mean stage where the fp32 screening stage would run; bit 3
 * forces the head stage's split schedule (a warp per group and factor, means on the spare warps),
 * bit 4 its round loop (a warp per group), which it otherwise chooses from the list length; bit 5
 * forces the fp32 screening kernel where the factored grid mean would run (slb_filter_mean_scheme) */
int         slb_debug_filter_stages(int32_t mask);
/* diagnostics: while both pointers are non-NULL, the fp32 screening stage (or the factored grid mean) of
 * slb_lyapunov_sweep_filtered also writes, for every point of the swept range (row = index relative to
 * idx_begin of the LAST pass), its screened mean [n, D] and the certified bound of its error [n, D]
 * (+inf where the point is left to the fp64 stages); tests hold |mean - fp64 mean| <= bound */
int         slb_debug_screening_probe(double* mu_dev, double* dm_dev);
/* diagnostics: deterministic-dynamics sweeps of the LQR composition (d = 2, saturated linear policy,
 * linear dynamics, quadratic V, constant / abs-linear L_V) take a specialised register-resident
 * kernel; 0 switches back to the generic interpreter (A/B timing, parity tests). */
int         slb_debug_det_fast(int32_t enable);
/* diagnostics: the refine pass of slb_lyapunov_sweep_filtered uses 32-point tiles for lists of up
 * to `upto32` points and 64-point tiles beyond (default 32 points per SM, 32 * 132); with 32-point
 * tiles the rows of a tile are additionally split over the CTAs a one-per-SM grid has to spare (up
 * to 8 per tile) */
int         slb_debug_refine_split(int64_t upto32);

/* ---- GP factor packing (after GPRCached.update_cache, functions.py:395-415) ------------ */
/* doubles needed for the packed L^-1 of an M-point GP */
int64_t slb_packed_len(int32_t M);
/* Linv_dev [M,M] row-major lower-triangular -> Wpack_dev (slb_packed_len(M) doubles) */
int slb_pack_factor(void* stream, const double* Linv_dev, int32_t M, double* Wpack_dev);

/* head subset of the decision filter: the first r <= min(M, SLB_HEAD_RANK) pivots of the pivoted
 * Cholesky factorisation of the symmetric positive semi-definite kernel_dev [M, M] (greedy: the
 * training point with the largest variance given those already chosen; ties: lowest index)
 * -> picks_dev [r] (int64).  scratch_dev: M * (r + 1) doubles. */
int slb_pivoted_subset(void* stream, const double* kernel_dev, int32_t M, int32_t r,
                       int64_t* picks_dev, double* scratch_dev);

/* ---- GP posterior on an explicit point list: GaussianProcess.__call__ / FunctionStack
 *      (functions.py:278-291, 417-458, 507-515).  points_dev [n, d_in] (already [x,u]
 *      concatenated, utilities.py:143); mean_dev, err_dev [n, D];
 *      err = beta*sqrt(var) (want_var == 0) or the latent variance (want_var != 0). ------- */
int slb_gp_predict(void* stream, const slb_gp_stack* gp, const double* points_dev, int64_t n,
                   double* mean_dev, double* err_dev, int32_t want_var);
/* ---- reverse mode of slb_gp_predict (want_var == 0), the reference's tf.gradients through the GP
 *      posterior (examples/inverted_pendulum.ipynb cells 9, 17):
 *        grad_points_dev [n, d_in] = grad_mean^T d mean / d points + grad_err^T d (beta sigma) / d points,
 *      OVERWRITTEN; grad_mean_dev / grad_err_dev [n, D], either may be NULL (not both).  With grad_err NULL
 *      the call does no O(M^2) work: the mean gradient needs only slb_gp_output.gamma, O(M d_in) per point.
 *      Where a variance is 0 the err gradient follows torch's sqrt backward (division by 2 sqrt(var) = 0:
 *      inf or NaN).  Every sum runs in a fixed order without atomics: two calls give bit-identical results.
 *      n == 0 launches nothing.  workspace_dev: >= slb_gp_vjp_workspace(gp, n) bytes (0 for every stack
 *      here); the size function returns -1 for a stack it rejects. */
/* ---- posterior mean only (GaussianProcess.to_mean_function(), DESIGN.md §3.16): mean_dev [n, D] of the
 *      stack at points_dev [n, d_in], d_in = 1..6, one point per thread on the Bellman sweep's staged
 *      pipeline (slb_gp_factor.Xf and slb_gp_output.gamma_f, which must be present and 16-byte aligned
 *      wherever a factor has data):  mean_o = (sum_j k_j gamma_f[o][j] + scale m_o(z)) / scale.
 *      This is a different fp64 form from the full posterior's  a^T alpha  (the mean of the predict entry
 *      point above): the two agree within the mean's rounding bound (DESIGN.md §3.16), not bit for bit.
 *      A point's mean depends only on the training rows' order: not on n, the block or the slice size.
 *      The closed-loop rollouts of the mean (slb_rollout_gp_mean) evaluate exactly this form.
 *      Host checks (before any launch): the stack, its staged tables, n >= 0, non-null buffers. */
int slb_gp_mean(void* stream, const slb_gp_stack* gp, const double* points_dev, int64_t n, double* mean_dev);
int64_t slb_gp_vjp_workspace(const slb_gp_stack* gp, int64_t n);
int slb_gp_vjp(void* stream, const slb_gp_stack* gp, const double* points_dev, int64_t n,
               const double* grad_mean_dev, const double* grad_err_dev, double* grad_points_dev,
               void* workspace_dev);

/* ---- gradient of the GP log marginal likelihood with respect to the hyper-parameters (gpflow 0.4.0
 *      GPR.build_likelihood): with K = kern.K(X) + noise I, alpha = K^-1 (Y - m(X)), W = alpha alpha^T - K^-1,
 *        d LML / d theta = 1/2 sum_ij W_ij d K_ij / d theta,     d LML / d noise = 1/2 tr W,
 *      for every slot of the covariance expression kern (num_prims >= 1; GPRCached.scale does not enter).
 *      X_dev [M, d_in] raw inputs, Kinv_dev [M, M] = K^-1 (row-major, both triangles), alpha_dev [M];
 *      grad_dev [SLB_GP_HYPER_SLOTS] (device) receives, for primitive p, d / d prims[p].variance at
 *      [p * (1 + SLB_MAX_IN)] and d / d prims[p].w[c] at [p * (1 + SLB_MAX_IN) + 1 + c] (w = 1 / lengthscale
 *      for the stationary kinds, the per-column variance for LINEAR; slots of absent primitives and columns
 *      are 0), and d / d noise last.  WHITE is K(X)'s form: its variance counts on the diagonal i == j only.
 *      One pass over the lower triangle in tiles of SLB_GP_HYPER_TILE x SLB_GP_HYPER_TILE pairs; per-tile
 *      sums go to workspace_dev (>= slb_gp_lml_grad_workspace(M) bytes) and are added in tile order: two
 *      calls give bit-identical results.  M == 0 returns before any CUDA call (grad_dev is not written). */
#define SLB_GP_HYPER_TILE 64
#define SLB_GP_HYPER_SLOTS (SLB_MAX_KPRIM * (1 + SLB_MAX_IN) + 1)
int64_t slb_gp_lml_grad_workspace(int32_t M);
int slb_gp_lml_grad(void* stream, const double* X_dev, int32_t M, int32_t d_in, const slb_kernel* kern,
                    const double* Kinv_dev, const double* alpha_dev, double* grad_dev, void* workspace_dev);
/* ---- the same gradient for a GP with k = 1..SLB_MAX_OUT target columns sharing one kernel and noise (gpflow's
 *      GPR with Y [M, k]): alpha_dev [M, k] row-major = K^-1 (Y - m(X)) and W = sum_c alpha_c alpha_c^T - k K^-1,
 *      formed per pair as w = -k Kinv_ij, then w = fma(alpha_ic, alpha_jc, w) for c = 0 .. k-1.  Still one pass
 *      over the lower triangle (each pair's d K / d theta evaluated once) with the same workspace.  k = 1 is
 *      fma(alpha_i, alpha_j, -Kinv_ij): slb_gp_lml_grad is this call with k = 1, bit for bit.  Host checks
 *      (before any launch): those of slb_gp_lml_grad and 1 <= k <= SLB_MAX_OUT. */
int slb_gp_lml_grad_cols(void* stream, const double* X_dev, int32_t M, int32_t d_in, const slb_kernel* kern,
                         const double* Kinv_dev, const double* alpha_dev, int32_t k, double* grad_dev,
                         void* workspace_dev);

/* ---- the fused Lyapunov sweep over flat grid indices [idx_begin, idx_end):
 *      index -> x (functions.py:714-731) -> u = policy(x) -> [x,u] -> GP mean / beta*sigma
 *      (or deterministic dynamics) -> V(x), V(mu), L_V(mu) . e -> decrease < threshold
 *      (lyapunov.py:265-288, 324-376, 436-441).  Outputs are arrays of length
 *      idx_end - idx_begin; any of values/decrease/threshold/mean/err may be NULL. -------- */
int slb_lyapunov_sweep(void* stream, const slb_sweep* cfg, int64_t idx_begin, int64_t idx_end,
                       uint8_t* negative_dev, double* values_dev, double* decrease_dev,
                       double* threshold_dev, double* mean_dev, double* err_dev);
/* The same decision flags (and V) with a certified filter in front of the O(M^2) posterior:
 * a thread-per-point kernel computes the GP mean (k . L^-T alpha, with a computed error bound),
 * V(mu), L_V(mu) and an UPPER bound of every output's standard deviation -- first the prior's,
 * then (one warp per remaining point) the posterior given only a head subset of at most
 * SLB_HEAD_RANK training points (factor.Whead / Xhead) -- and decides every point whose
 * comparison `decrease < threshold` has the same outcome for all sigma in [0, bound] (guard band:
 * 1e-6 relative + the mean's error bound); the remaining points are compacted and go through the
 * full fp64 posterior (the kernel of slb_lyapunov_sweep).  Every flag equals the exact outcome wherever
 * the decrease is farther from the threshold than the full kernel's certified error; with the refine
 * pass's unsplit tiles the flags are identical to slb_lyapunov_sweep's, while tiles whose rows are split
 * over several CTAs (slb_debug_refine_split) sum in another order and may differ from them within that
 * error.
 * workspace_dev: >= slb_filter_workspace(n) bytes.  stats_dev: NULL or 4 int64 (device):
 * {decided by mean + prior bound, decided by the head-rank bound, refined by the full posterior,
 * points} accumulated over calls (the caller zeroes it). */
int64_t slb_filter_workspace(int64_t n);
/* diagnostics: where a filtered sweep of n <= 2^22 points (one pass) leaves its lists in workspace_dev,
 * as byte offsets: offsets[0] the counters (uint64 [3]: entries of list A, entries of list B, list A entries
 * of the factored grid mean without an fp64-class mean), offsets[1] list A (int64 [n]: the points stage 1 left
 * undecided), offsets[2] list B (int64 [n]: the points the head stage left to the full posterior).  Indices
 * are relative to idx_begin, in no particular order; only the first counters[0] / counters[1] entries are
 * written.  The lists describe the LAST pass of the last call only.  Returns non-zero for n < 0,
 * n > 2^22 or a NULL offsets. */
int slb_debug_filter_lists(int64_t n, int64_t* offsets);
/* which first stage slb_lyapunov_sweep_filtered runs for this configuration: 32 = the fp32 screening
 * kernel (plain RBF factors, quadratic V on at most four outputs, constant / abs-linear L_V, tables fit
 * the head stage's shared memory) with an fp64 mean only for the points its error box leaves open;
 * 64 = the fp64 mean kernel; 0 = no GP */
int slb_filter_stage1(const slb_sweep* cfg);
/* how that first stage computes the mean: SLB_MEAN_FP64 per point (the fp64 mean kernel);
 * SLB_MEAN_FP32_SCREENED per point in fp32 with a certified bound (stage 1 = 32); SLB_MEAN_GRID_FACTORED
 * (also stage 1 = 32: the same screened list entries) per tile of a 2-D grid from per-axis tables of
 * kernel values contracted in fp64, with an fp64-class certified bound -- plain RBF factors on
 * [x0, x1, u] and a LINEAR one-output policy with at most SATURATE and SCALE; bit 5 of
 * slb_debug_filter_stages forces the fp32 screening kernel instead.  SLB_MEAN_NONE: no GP. */
#define SLB_MEAN_NONE 0
#define SLB_MEAN_FP64 1
#define SLB_MEAN_FP32_SCREENED 2
#define SLB_MEAN_GRID_FACTORED 3
int slb_filter_mean_scheme(const slb_sweep* cfg);
int slb_lyapunov_sweep_filtered(void* stream, const slb_sweep* cfg, int64_t idx_begin,
                                int64_t idx_end, uint8_t* negative_dev, double* values_dev,
                                void* workspace_dev, int64_t* stats_dev);
/* one step of update_safe_set on a single process: the filtered sweep of [idx_begin, idx_end) (arguments
 * as slb_lyapunov_sweep_filtered, its flags into negative_dev) whose decision kernels fold the first-fail
 * key as they decide each point, then the prefix rule on that key -- what slb_first_fail followed by
 * slb_apply_prefix compute on the sweep's flags, with the same key_dev, safe_dev and prefix_stats_dev.
 * values_dev [n]: V over the range (read only); initial_dev may be NULL. */
int slb_safe_set_step(void* stream, const slb_sweep* cfg, int64_t idx_begin, int64_t idx_end,
                      uint8_t* negative_dev, const double* values_dev, const uint8_t* initial_dev,
                      void* workspace_dev, int64_t* stats_dev, slb_fail_key* key_dev, uint8_t* safe_dev,
                      slb_prefix_stats* prefix_stats_dev);
/* diagnostics: the refine pass of slb_lyapunov_sweep_filtered alone, on a caller's point list:
 * list_dev [*count_dev] (device) holds indices relative to idx_begin, each in [0, n_max), and
 * 0 <= n_max <= the pass length of slb_filter_workspace.  Both tile-size launches, the row / factor
 * split and its workspace run exactly as in the filtered sweep (the split tickets are zeroed first).
 * At the listed points it writes negative and values (NULL: not written) as slb_lyapunov_sweep would,
 * and, unless NULL, mean_dev / err_dev [n_max, D] (err = beta sigma); every other entry is untouched.
 * workspace_dev: >= slb_filter_workspace(n_max) bytes. */
int slb_debug_refine(void* stream, const slb_sweep* cfg, int64_t idx_begin, int64_t n_max,
                     const int64_t* list_dev, const unsigned long long* count_dev,
                     uint8_t* negative_dev, double* values_dev, double* mean_dev, double* err_dev,
                     void* workspace_dev);
/* same on an explicit state list states_dev [n, d] (get_safe_sample-style callers) */
int slb_lyapunov_points(void* stream, const slb_sweep* cfg, const double* states_dev, int64_t n,
                        uint8_t* negative_dev, double* values_dev, double* decrease_dev,
                        double* threshold_dev, double* mean_dev, double* err_dev);

/* ---- prefix rule without sorting (lyapunov.py:500-606, SURVEY.md Q1/Q4):
 *      k* = min over failing points of key (V_i, i); safe_i = key_i < k* | initial_i.
 *      workspace_dev: >= slb_first_fail_workspace(n) bytes.  result_dev: one slb_fail_key
 *      in device memory (the caller all-reduces it across ranks, then applies).           */
int64_t slb_first_fail_workspace(int64_t n);
int slb_first_fail(void* stream, const double* values_dev, const uint8_t* negative_dev,
                   const uint8_t* initial_dev /* may be NULL */, int64_t n, int64_t idx_begin,
                   void* workspace_dev, slb_fail_key* result_dev);
/* sharded form with the exchange fused into the two kernels: slb_first_fail_x pushes this rank's
 * key to every peer, slb_apply_prefix_x waits for all keys of the sweep, reduces them (writing the
 * winner to key_out_dev) and applies the prefix rule -- no collective call, no host round trip */
int slb_first_fail_x(void* stream, const double* values_dev, const uint8_t* negative_dev,
                     const uint8_t* initial_dev, int64_t n, int64_t idx_begin, void* workspace_dev,
                     slb_fail_key* result_dev, const slb_exchange* xchg);
int slb_apply_prefix_x(void* stream, const double* values_dev, const uint8_t* initial_dev,
                       int64_t n, int64_t idx_begin, slb_fail_key* key_out_dev, uint8_t* safe_dev,
                       void* workspace_dev, slb_prefix_stats* stats_dev, const slb_exchange* xchg);
/* multi-GPU: lexicographic min (and n_ok sum) over `world` keys all-gathered by the caller
 * (the one collective of a sweep, SURVEY.md section 8e) -> out_dev; may alias gathered_dev[0] */
int slb_combine_fail_keys(void* stream, const slb_fail_key* gathered_dev, int32_t world,
                          slb_fail_key* out_dev);
int slb_apply_prefix(void* stream, const double* values_dev, const uint8_t* initial_dev,
                     int64_t n, int64_t idx_begin, const slb_fail_key* key_dev,
                     uint8_t* safe_dev, void* workspace_dev, slb_prefix_stats* stats_dev);

/* ---- update_safe_set(can_shrink=False) (lyapunov.py:497-606 with :507-510, :540-582): the V-sorted
 *      batch loop resolved per batch on the device, single process.  order_dev [n]: stable sort of V
 *      (sorted position -> grid index); batch = config.gp_batch_size >= 1; max_refinement R >= 1
 *      (1: the plain branch).  negative_dev, prev_safe_dev [n]: the sweep's flags and the current safe
 *      set; initial_dev may be NULL; n_req_dev [n] = ceil(max(s thr / dec, 0)), NaN -> 0, may be NULL
 *      only when R == 1.  All arrays are in grid order.
 *      slb_no_shrink_scan writes candidates_dev [n]: 1 where the refined check (tau / n_req on the
 *      cell's mesh) can decide the result.  The caller writes that check into refined_dev [n]
 *      (1 = verified; read at candidates only), then slb_no_shrink_resolve writes safe_dev and
 *      refinement_dev [n], c_max's sorted position (-1: the largest V) and c_max.
 *      workspace_dev: >= slb_no_shrink_workspace(n, batch) bytes, kept between the two calls.      */
int64_t slb_no_shrink_workspace(int64_t n, int64_t batch);
int slb_no_shrink_scan(void* stream, const int64_t* order_dev, const uint8_t* negative_dev,
                       const uint8_t* prev_safe_dev, const uint8_t* initial_dev, const double* n_req_dev,
                       int64_t n, int64_t batch, int64_t max_refinement, void* workspace_dev,
                       uint8_t* candidates_dev);
int slb_no_shrink_resolve(void* stream, const int64_t* order_dev, const double* values_dev,
                          const uint8_t* negative_dev, const uint8_t* prev_safe_dev,
                          const int64_t* prev_refinement_dev, const uint8_t* initial_dev,
                          const double* n_req_dev, const uint8_t* refined_dev, int64_t n, int64_t batch,
                          int64_t max_refinement, void* workspace_dev, uint8_t* safe_dev,
                          int64_t* refinement_dev, int64_t* cmax_position_dev, double* cmax_dev);

/* ---- generic evaluation of a fused function object on explicit points:
 *      DeterministicFunction.__call__, Lyapunov.update_values (lyapunov.py:305-322).
 *      points_dev [n, fn->in_dim] -> out_dev [n, out columns]. ---------------------------- */
int slb_eval_function(void* stream, const slb_function* fn, const double* points_dev, int64_t n,
                      double* out_dev);
/* fn's COLUMNS (see slb_sweep), the width of slb_eval_function's out_dev; -1 for a NULL fn.  The
 * descriptor is not validated otherwise. */
int slb_function_columns(const slb_function* fn);
/* grid coordinates for flat indices [idx_begin, idx_end): GridWorld.index_to_state */
int slb_index_to_state(void* stream, const slb_grid* grid, int64_t idx_begin, int64_t idx_end,
                       double* states_dev);

/* ---- Bellman sweep (reinforcement_learning.py:65-114, 135-140, 213-279) ---------------- */
/* out_dev[i] = r(x_i,u_i) + gamma * V(mean f(x_i,u_i)) for flat indices [idx_begin, idx_end) */
int slb_bellman_sweep(void* stream, const slb_bellman* cfg, int64_t idx_begin, int64_t idx_end,
                      double* out_dev);
/* discrete_policy_optimization: actions_dev [n_actions, m]; constraint_dev [n_actions, n] or
 * NULL (value < 0 => -inf, :272-275); best_dev[i] = first argmax over actions (:278, NaN counts as
 * the maximum like np.argmax).  workspace_dev: NULL, or >= slb_bellman_argmax_workspace bytes: with
 * GP dynamics on plain RBF factors and a state dimension of 1 or 2 (n_actions >= 2) the action
 * is then factored out of the exponent (one kernel
 * row per STATE, an [n_actions x M] x [M x states] fp64 tensor-core contraction per output)
 * instead of n_actions sweeps; the workspace size is 0 when that path does not apply. */
int64_t slb_bellman_argmax_workspace(const slb_bellman* cfg, int32_t n_actions);
int slb_bellman_argmax(void* stream, const slb_bellman* cfg, int64_t idx_begin, int64_t idx_end,
                       const double* actions_dev, int32_t n_actions, const double* constraint_dev,
                       int32_t* best_dev, double* best_value_dev, void* workspace_dev);
/* max_i |a_i - b_i| into result_dev[0] (value-iteration convergence test, test_rl.py:66-69) */
int slb_max_abs_diff(void* stream, const double* a_dev, const double* b_dev, int64_t n,
                     double* result_dev);

/* ---- closed-loop rollouts x <- f(x, pi(x)) (examples/utilities.py:654-686 compute_roa,
 *      :522-545 reward_rollout).  The slb_bellman descriptor carries the closed loop: `policy`,
 *      deterministic `dynamics` (gp.num_outputs must be 0; the _gp_mean forms below take the GP mean),
 *      and `reward` for slb_reward_rollout;
 *      `value`, `gamma` and `action` are ignored, fixed_action must be 0.  The state dimension d is
 *      grid.ndim.  Start states: the device array states_dev [n, d], or, when states_dev is NULL,
 *      the grid points of flat indices [idx_begin, idx_begin + n).
 *      workspace_dev: >= slb_rollout_workspace(cfg, n, reward) bytes (reward = 1 for
 *      slb_reward_rollout); slb_rollout needs none when horizon <= 33. ---------------------------- */
int64_t slb_rollout_workspace(const slb_bellman* cfg, int64_t n, int32_t reward);
/* compute_roa: applies the closed loop horizon - 1 times (none for horizon <= 1);
 * roa_dev[i] = ||x_end - equilibrium||_2 <= tol (numpy's row norm; NaN / inf end states give 0).
 * equilibrium_host: HOST array of d doubles, or NULL for the origin.  end_states_dev [n, d] may be
 * NULL; traj_dev NULL or [n, d, horizon] (trajectory[:, :, 0] = start states, horizon >= 1). */
int slb_rollout(void* stream, const slb_bellman* cfg, const double* states_dev, int64_t idx_begin,
                int64_t n, int32_t horizon, const double* equilibrium_host, double tol,
                uint8_t* roa_dev, double* end_states_dev, double* traj_dev, void* workspace_dev);
/* reward_rollout: for t = 0 .. horizon - 1:  temp = discount_dev[t] * r(x_t, pi(x_t)),
 * sums_dev[i] += temp, stop after the first t with max_i |temp_i| < tol (a NaN anywhere: not below),
 * x_{t+1} = f(x_t, pi(x_t)).  discount_dev [horizon] = discount ** t as computed by the caller.
 * stop_dev (device int64) receives that first t, or -1 when the sums did not converge. */
int slb_reward_rollout(void* stream, const slb_bellman* cfg, const double* states_dev, int64_t idx_begin,
                       int64_t n, int32_t horizon, const double* discount_dev, double tol,
                       double* sums_dev, int64_t* stop_dev, void* workspace_dev);
/* The same two rollouts with the GP posterior mean as the dynamics: cfg->gp holds the stack with
 * num_outputs == d and input_dim == d + m (at most 6), cfg->dynamics.kind must be SLB_FN_NONE and the
 * staged tables present (as for slb_gp_mean).  Every step evaluates slb_gp_mean's form, so a rollout of
 * h steps is bit-identical to h compositions of the policy's evaluation and slb_gp_mean.  Workspace:
 * slb_rollout_workspace, as above. */
int slb_rollout_gp_mean(void* stream, const slb_bellman* cfg, const double* states_dev, int64_t idx_begin,
                        int64_t n, int32_t horizon, const double* equilibrium_host, double tol,
                        uint8_t* roa_dev, double* end_states_dev, double* traj_dev, void* workspace_dev);
int slb_reward_rollout_gp_mean(void* stream, const slb_bellman* cfg, const double* states_dev,
                               int64_t idx_begin, int64_t n, int32_t horizon, const double* discount_dev,
                               double tol, double* sums_dev, int64_t* stop_dev, void* workspace_dev);

/* ---- exact policy evaluation (reinforcement_learning.py:142-211 optimize_value_function): the
 *      fixed point of  v = r + gamma T v,  T = the value table's rows at the mean next states
 *      (DESIGN.md §3.9, §3.15).  Row i of T has ncols entries: cols_dev[i * ncols + j] (int32, or int64
 *      when the value grid has more than 2^31 - 1 vertices), weights_dev[i * ncols + j] (fp64).  A
 *      Triangulation gives ncols = d + 1 barycentric weights, d = the value grid's dimension; a
 *      PiecewiseConstant gives ncols = 2: the next state's nearest vertex with weight 1, then the same
 *      vertex with weight 0 (slb_value_solve's narrowest row; a NaN next state: vertex 0 with weights NaN,
 *      0).  stats_dev: SLB_VALUE_STATS uint64 slots:
 *        [0] ~key(min weight)  (order-preserving key of the smallest weight, complemented)
 *        [1] rho = max_i sum_j |w_ij|, fp64 bits     [2] rows re-searched (grid-line lookups, Q6)
 *        [3] rows with a NaN next state / reward     [4] iterations   [5] last ||dv||_inf, fp64 bits
 *        [6] certified bound, fp64 bits              [7] status (SLB_VALUE_*)   [8] solver tier (1, 2)
 *      The assembly entry points write [0..3]; slb_value_solve writes [0, 1] and [4..8]. ---------- */
#define SLB_VALUE_STATS 16
#define SLB_VALUE_CONVERGED 0
#define SLB_VALUE_MAX_ITERS 1
#define SLB_VALUE_NEGATIVE_WEIGHT 2
#define SLB_VALUE_NOT_CONTRACTIVE 3
#define SLB_VALUE_NAN 4
/* fused assembly for flat indices [idx_begin, idx_end): u = policy(x), x+ = mean dynamics(x, u)
 * (deterministic function or GP stack), rewards_dev[i] = reward(x, u); cfg->value is a one-output
 * Triangulation (projection allowed) or PiecewiseConstant, without post-op flags; fixed_action must be 0 */
int slb_value_operator(void* stream, const slb_bellman* cfg, int64_t idx_begin, int64_t idx_end,
                       void* cols_dev, double* weights_dev, double* rewards_dev, uint64_t* stats_dev);
/* composed assembly: the rows of next_states_dev [n, d] */
int slb_value_operator_points(void* stream, const slb_function* value, const double* next_states_dev,
                              int64_t n, void* cols_dev, double* weights_dev, uint64_t* stats_dev);
/* bytes of workspace slb_value_solve needs: 0 when n <= 12288 (one-CTA tier), else n doubles + 128 */
int64_t slb_value_solve_workspace(int64_t n, int32_t ncols);
/* iterate v <- r + gamma T v from v_inout_dev [n] until gamma rho / (1 - gamma rho) ||dv||_inf <=
 * tol max(1, ||v||_inf), then write v to v_inout_dev.  The status (stats slot 7) says why it stopped;
 * v_inout_dev is left unchanged when the operator has a weight < -1e-12, gamma rho >= 1, or a NaN in a
 * weight, a reward or v_inout_dev itself. */
int slb_value_solve(void* stream, int64_t n, int32_t ncols, const void* cols_dev, const double* weights_dev,
                    const double* rewards_dev, double gamma, double tol, int64_t max_iters,
                    double* v_inout_dev, void* workspace_dev, uint64_t* stats_dev);

/* ---- reverse mode of the fused networks and plants (the reference's tf.gradients through
 *      NeuralNetwork functions.py:1702-1729, LyapunovNetwork and the plants examples/utilities.py:48-104,
 *      242-289, 387-437): for a cotangent grad_out_dev [n, out] (out = 1 for LYAPUNOV_NN)
 *        grad_in_dev     [n, in]  = grad_out^T d out / d points               (or NULL)
 *        grad_params_dev          = sum over the n points of grad_out^T d out / d params, OVERWRITTEN,
 *                                   in the layout of fn->matrix (MLP: packed weights and biases; LYAPUNOV_NN:
 *                                   the packed layer kernels [W^T W + eps I; W_extra]); NULL, and NULL for
 *                                   the plants, which have no parameters
 *        out_dev         [n, out] = the forward pass recomputed by the gradient kernel, bit-identical to
 *                                   slb_eval_function (or NULL)
 *      Kinds MLP, LYAPUNOV_NN, PENDULUM, CARTPOLE and VANDERPOL (and TRIANGULATION, PIECEWISE_CONSTANT, below) without post-op
 *      flags; VANDERPOL's action column gets a zero gradient.  Gradient conventions: ReLU' = 0
 *      at 0, tanh' = 1 - tanh^2.  The parameter gradient is reduced in a fixed order without atomics: two
 *      calls with the same inputs give bit-identical results.  n == 0 zeroes grad_params and launches
 *      nothing.  workspace_dev: >= slb_function_vjp_workspace(fn, n) bytes when grad_params_dev is
 *      given (0 for the plants and for n <= 32); the size function returns -1 for a descriptor it rejects. */
int64_t slb_function_vjp_workspace(const slb_function* fn, int64_t n);
int slb_function_vjp(void* stream, const slb_function* fn, const double* points_dev, int64_t n,
                     const double* grad_out_dev, double* grad_in_dev, double* grad_params_dev,
                     double* out_dev, void* workspace_dev);
/* ---- SLB_FN_TRIANGULATION in slb_function_vjp (the tf.gather of functions.py:1494-1499 under
 *      tf.gradients): grad_params_dev [nindex, out] = sum over the points p and simplex vertices k of
 *      w_pk grad_out[p] scattered to vertex c_pk, OVERWRITTEN; (c_pk, w_pk) are the vertices and barycentric
 *      weights of the forward evaluation (slb_triangulation_rows).  Each entry is summed sequentially in
 *      ascending j = p (d + 1) + k from +0.0, without atomics: bit for bit np.add.at over the rows, and two
 *      calls give identical results.  grad_in_dev must be NULL (the point gradient is the SLB_FLAG_GRADIENT
 *      evaluation); out_dev [n, out] is the forward, bit-identical to slb_eval_function.  No post-op flags
 *      (SLB_FLAG_PROJECT applies).  n == 0 zeroes grad_params.  The workspace (rows, sort keys, sort scratch)
 *      is needed when grad_params_dev is given and n > 0; a batch whose sort key (bits of nindex - 1 plus
 *      bits of n (d + 1) - 1) exceeds 64 bits is rejected.  One thread sums each vertex, so a batch whose
 *      points all land on one vertex costs n (d + 1) serial additions. */
/* ---- SLB_FN_PIECEWISE_CONSTANT in slb_function_vjp: the same transpose with one row per point, its
 *      nearest vertex with weight 1: grad_params_dev [nindex, out] = sum over the points p of grad_out[p]
 *      scattered to that vertex, OVERWRITTEN, summed in ascending p from +0.0 without atomics (bit for bit
 *      np.add.at(G, idx, grad_out)).  A point with a NaN coordinate (NaN forward, no vertex) adds nothing.
 *      grad_in_dev must be NULL (the point gradient is 0); no flags; workspace and key limit as above. */
/* GridWorld.state_to_index (functions.py:733-752) on the device, the lookup of SLB_FN_PIECEWISE_CONSTANT:
 * idx_dev [n] (int64) = the flat index of the nearest vertex of points_dev [n, grid->ndim], or -1 for a
 * row with a NaN coordinate (PiecewiseConstant.parameter_derivative, functions.py:889-913) */
int slb_grid_nearest_index(void* stream, const slb_grid* grid, const double* points_dev, int64_t n,
                           int64_t* idx_dev);
/* the rows of _Triangulation.parameter_derivative (functions.py:1228-1259) at points_dev [n, d]:
 * cols_dev int64 [n, d + 1] vertex indices and weights_dev [n, d + 1] barycentric weights of the forward
 * evaluation (projection, corner table and simplex choice included) */
int slb_triangulation_rows(void* stream, const slb_function* fn, const double* points_dev, int64_t n,
                           int64_t* cols_dev, double* weights_dev);

#ifdef __cplusplus
}
#endif
#endif /* SLB200_H */
