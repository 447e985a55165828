"""ctypes binding of ``libslb200.so`` (C ABI declared in ``include/slb200.h``).

There is NO CPU fallback: if the shared library is missing, or a compute entry point
is called without a CUDA device, an exception is raised.  The structures below mirror
``include/slb200.h`` field for field; ``_check_layout`` verifies the sizes against
``slb_struct_sizes`` at load time.
"""

from __future__ import annotations

import ctypes as C
import os

SLB_MAX_DIM = 6
SLB_MAX_IN = 8
SLB_MAX_OUT = 6
SLB_MAX_ACT = 2
SLB_TILE_POINTS = 64
SLB_HEAD_RANK = 64
SLB_MAX_RANKS = 16

FN_NONE, FN_CONSTANT, FN_LINEAR, FN_QUADRATIC, FN_TRIANGULATION, FN_PENDULUM, FN_CARTPOLE, \
    FN_LYAPUNOV_NN, FN_MLP, FN_VANDERPOL, FN_PIECEWISE_CONSTANT = range(11)
FLAG_SATURATE, FLAG_ABS, FLAG_NORM1, FLAG_PROJECT, FLAG_SCALE, FLAG_GRADIENT, FLAG_MAXABS = \
    1, 2, 4, 8, 16, 32, 64
K_RBF, K_MATERN12, K_MATERN32, K_MATERN52, K_LINEAR, K_CONSTANT, K_WHITE = range(7)
SLB_MAX_KPRIM = 6
# slb_gp_lml_grad: tile edge and gradient slots [prim][variance, w[0..SLB_MAX_IN)] + noise (include/slb200.h)
SLB_GP_HYPER_TILE = 64
SLB_GP_HYPER_SLOTS = SLB_MAX_KPRIM * (1 + SLB_MAX_IN) + 1
ABI_VERSION = 6
# slb_value_solve: stats slots and status codes (include/slb200.h)
VALUE_STATS = 16
VALUE_CONVERGED, VALUE_MAX_ITERS, VALUE_NEGATIVE_WEIGHT, VALUE_NOT_CONTRACTIVE, VALUE_NAN = range(5)
# slb_filter_mean_scheme: how stage 1 of the filtered sweep computes the GP mean (include/slb200.h)
MEAN_NONE, MEAN_FP64, MEAN_FP32_SCREENED, MEAN_GRID_FACTORED = range(4)

UINT64_MAX = (1 << 64) - 1
INT64_MAX = (1 << 63) - 1


class NativeLibraryError(RuntimeError):
    """libslb200 is missing, mismatched, or reported an error."""


class SlbGrid(C.Structure):
    _fields_ = [("ndim", C.c_int32), ("_pad", C.c_int32), ("nindex", C.c_int64),
                ("num_points", C.c_int64 * SLB_MAX_DIM), ("offset", C.c_double * SLB_MAX_DIM),
                ("unit_maxes", C.c_double * SLB_MAX_DIM), ("upper", C.c_double * SLB_MAX_DIM),
                ("discrete_points", C.c_void_p)]


class SlbFunction(C.Structure):
    _fields_ = [("kind", C.c_int32), ("in_dim", C.c_int32), ("out_dim", C.c_int32),
                ("flags", C.c_uint32), ("out_scale", C.c_double), ("lower", C.c_double),
                ("upper", C.c_double), ("cparams", C.c_double * 24), ("matrix", C.c_void_p),
                ("hyperplanes", C.c_void_p), ("unit_simplices", C.c_void_p),
                ("corner_simplex", C.c_void_p), ("nsimplex", C.c_int32), ("_pad", C.c_int32), ("grid", SlbGrid)]


class SlbKernelPrim(C.Structure):
    _fields_ = [("kind", C.c_int32), ("term", C.c_int32), ("variance", C.c_double),
                ("w", C.c_double * SLB_MAX_IN)]


class SlbKernel(C.Structure):
    _fields_ = [("num_prims", C.c_int32), ("_pad", C.c_int32),
                ("prims", SlbKernelPrim * SLB_MAX_KPRIM)]


class SlbGpFactor(C.Structure):
    _fields_ = [("M", C.c_int32), ("nrb", C.c_int32), ("Xs", C.c_void_p), ("Wpack", C.c_void_p),
                ("lengthscales", C.c_double * SLB_MAX_IN), ("variance", C.c_double),
                ("scale", C.c_double), ("kss", C.c_double), ("kernel", SlbKernel),
                ("Whead", C.c_void_p), ("Wheadp", C.c_void_p), ("Xhead", C.c_void_p),
                ("head_rows", C.c_int32),
                ("_pad2", C.c_int32), ("Xf", C.c_void_p), ("hmax", C.c_double)]


class SlbGpOutput(C.Structure):
    _fields_ = [("factor", C.c_int32), ("_pad", C.c_int32), ("beta", C.c_double),
                ("alpha", C.c_void_p), ("gamma", C.c_void_p), ("prior_mean", C.c_void_p),
                ("gamma_f", C.c_void_p), ("gamma_l1", C.c_double)]


class SlbGpStack(C.Structure):
    _fields_ = [("num_outputs", C.c_int32), ("num_factors", C.c_int32),
                ("input_dim", C.c_int32), ("_pad", C.c_int32),
                ("factors", SlbGpFactor * SLB_MAX_OUT), ("outputs", SlbGpOutput * SLB_MAX_OUT)]


class SlbSweep(C.Structure):
    _fields_ = [("grid", SlbGrid), ("policy", SlbFunction), ("dynamics", SlbFunction),
                ("gp", SlbGpStack), ("lyapunov", SlbFunction), ("lipschitz_v", SlbFunction),
                ("lv_const", C.c_double), ("lf_const", C.c_double), ("tau", C.c_double),
                ("lipschitz_f", SlbFunction), ("lf_values", C.c_void_p),
                ("lf_index_base", C.c_int64)]


class SlbBellman(C.Structure):
    _fields_ = [("grid", SlbGrid), ("policy", SlbFunction), ("dynamics", SlbFunction),
                ("gp", SlbGpStack), ("reward", SlbFunction), ("value", SlbFunction),
                ("gamma", C.c_double), ("fixed_action", C.c_int32), ("_pad", C.c_int32),
                ("action", C.c_double * SLB_MAX_ACT)]


class SlbFailKey(C.Structure):
    _fields_ = [("key_value", C.c_uint64), ("key_index", C.c_int64), ("n_ok", C.c_int64),
                ("_pad", C.c_int64)]


class SlbPrefixStats(C.Structure):
    _fields_ = [("n_safe", C.c_int64), ("n_below", C.c_int64), ("max_below", C.c_uint64),
                ("max_all", C.c_uint64)]


class SlbExchange(C.Structure):
    _fields_ = [("world", C.c_int32), ("rank", C.c_int32),
                ("slots", C.c_void_p * SLB_MAX_RANKS), ("seq_dev", C.c_void_p)]


_STRUCTS = (SlbGrid, SlbFunction, SlbGpFactor, SlbGpOutput, SlbGpStack, SlbSweep, SlbBellman,
            SlbFailKey, SlbPrefixStats, SlbExchange)

LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "libslb200.so")

_vp, _i64, _i32, _dp = C.c_void_p, C.c_int64, C.c_int32, C.c_void_p

# name -> (restype, argtypes): every symbol include/slb200.h declares
SIGNATURES = {
    "slb_abi_version": (C.c_int, []),
    "slb_last_error": (C.c_char_p, []),
    "slb_device_count": (C.c_int, []),
    "slb_struct_sizes": (C.c_int, [C.POINTER(C.c_int64), _i32]),
    "slb_launch_count": (C.c_int64, []),
    "slb_note_graph_replay": (None, [_i64]),
    "slb_debug_phase_timing": (C.c_int, [_vp]),
    "slb_debug_head_timing": (C.c_int, [_vp]),
    "slb_debug_stage1_timing": (C.c_int, [_vp]),
    "slb_debug_refine_timing": (C.c_int, [_vp]),
    "slb_record_factor_dependency": (C.c_int, [_vp]),
    "slb_restore_tables": (C.c_int, [_vp, _vp, _i64, _i64, _vp, _vp]),
    "slb_debug_refine_split": (C.c_int, [_i64]),
    "slb_debug_det_fast": (C.c_int, [_i32]),
    "slb_debug_filter_stages": (C.c_int, [_i32]),
    "slb_debug_screening_probe": (C.c_int, [_dp, _dp]),
    "slb_filter_stage1": (C.c_int, [C.POINTER(SlbSweep)]),
    "slb_filter_mean_scheme": (C.c_int, [C.POINTER(SlbSweep)]),
    "slb_packed_len": (C.c_int64, [_i32]),
    "slb_pack_factor": (C.c_int, [_vp, _dp, _i32, _dp]),
    "slb_pivoted_subset": (C.c_int, [_vp, _dp, _i32, _i32, _vp, _dp]),
    "slb_gp_predict": (C.c_int, [_vp, C.POINTER(SlbGpStack), _dp, _i64, _dp, _dp, _i32]),
    "slb_lyapunov_sweep": (C.c_int, [_vp, C.POINTER(SlbSweep), _i64, _i64, _dp, _dp, _dp, _dp,
                                     _dp, _dp]),
    "slb_lyapunov_points": (C.c_int, [_vp, C.POINTER(SlbSweep), _dp, _i64, _dp, _dp, _dp, _dp,
                                      _dp, _dp]),
    "slb_filter_workspace": (C.c_int64, [_i64]),
    "slb_debug_filter_lists": (C.c_int, [_i64, C.POINTER(C.c_int64)]),
    "slb_lyapunov_sweep_filtered": (C.c_int, [_vp, C.POINTER(SlbSweep), _i64, _i64, _dp, _dp, _vp,
                                              _vp]),
    "slb_safe_set_step": (C.c_int, [_vp, C.POINTER(SlbSweep), _i64, _i64, _dp, _dp, _dp, _vp, _vp, _vp,
                                    _dp, _vp]),
    "slb_debug_refine": (C.c_int, [_vp, C.POINTER(SlbSweep), _i64, _i64, _vp, _vp, _vp, _dp, _dp, _dp,
                                   _vp]),
    "slb_first_fail_workspace": (C.c_int64, [_i64]),
    "slb_first_fail_x": (C.c_int, [_vp, _dp, _dp, _dp, _i64, _i64, _vp, _vp,
                                   C.POINTER(SlbExchange)]),
    "slb_apply_prefix_x": (C.c_int, [_vp, _dp, _dp, _i64, _i64, _vp, _dp, _vp, _vp,
                                     C.POINTER(SlbExchange)]),
    "slb_first_fail": (C.c_int, [_vp, _dp, _dp, _dp, _i64, _i64, _vp, _vp]),
    "slb_combine_fail_keys": (C.c_int, [_vp, _vp, _i32, _vp]),
    "slb_apply_prefix": (C.c_int, [_vp, _dp, _dp, _i64, _i64, _vp, _dp, _vp, _vp]),
    "slb_no_shrink_workspace": (C.c_int64, [_i64, _i64]),
    "slb_no_shrink_scan": (C.c_int, [_vp, _dp, _dp, _dp, _dp, _dp, _i64, _i64, _i64, _vp, _dp]),
    "slb_no_shrink_resolve": (C.c_int, [_vp, _dp, _dp, _dp, _dp, _dp, _dp, _dp, _dp, _i64, _i64, _i64,
                                        _vp, _dp, _dp, _dp, _dp]),
    "slb_eval_function": (C.c_int, [_vp, C.POINTER(SlbFunction), _dp, _i64, _dp]),
    "slb_function_columns": (C.c_int, [C.POINTER(SlbFunction)]),
    "slb_index_to_state": (C.c_int, [_vp, C.POINTER(SlbGrid), _i64, _i64, _dp]),
    "slb_bellman_sweep": (C.c_int, [_vp, C.POINTER(SlbBellman), _i64, _i64, _dp]),
    "slb_bellman_argmax_workspace": (C.c_int64, [C.POINTER(SlbBellman), _i32]),
    "slb_bellman_argmax": (C.c_int, [_vp, C.POINTER(SlbBellman), _i64, _i64, _dp, _i32, _dp, _dp,
                                     _dp, _vp]),
    "slb_max_abs_diff": (C.c_int, [_vp, _dp, _dp, _i64, _dp]),
    "slb_rollout_workspace": (C.c_int64, [C.POINTER(SlbBellman), _i64, _i32]),
    "slb_rollout": (C.c_int, [_vp, C.POINTER(SlbBellman), _dp, _i64, _i64, _i32, _dp, C.c_double,
                              _vp, _dp, _dp, _vp]),
    "slb_reward_rollout": (C.c_int, [_vp, C.POINTER(SlbBellman), _dp, _i64, _i64, _i32, _dp,
                                     C.c_double, _dp, _vp, _vp]),
    "slb_rollout_gp_mean": (C.c_int, [_vp, C.POINTER(SlbBellman), _dp, _i64, _i64, _i32, _dp, C.c_double,
                                      _vp, _dp, _dp, _vp]),
    "slb_reward_rollout_gp_mean": (C.c_int, [_vp, C.POINTER(SlbBellman), _dp, _i64, _i64, _i32, _dp,
                                             C.c_double, _dp, _vp, _vp]),
    "slb_value_operator": (C.c_int, [_vp, C.POINTER(SlbBellman), _i64, _i64, _vp, _dp, _dp, _vp]),
    "slb_value_operator_points": (C.c_int, [_vp, C.POINTER(SlbFunction), _dp, _i64, _vp, _dp, _vp]),
    "slb_value_solve_workspace": (C.c_int64, [_i64, _i32]),
    "slb_value_solve": (C.c_int, [_vp, _i64, _i32, _vp, _dp, _dp, C.c_double, C.c_double, _i64, _dp,
                                  _vp, _vp]),
    "slb_function_vjp_workspace": (C.c_int64, [C.POINTER(SlbFunction), _i64]),
    "slb_function_vjp": (C.c_int, [_vp, C.POINTER(SlbFunction), _dp, _i64, _dp, _dp, _dp, _dp, _vp]),
    "slb_triangulation_rows": (C.c_int, [_vp, C.POINTER(SlbFunction), _dp, _i64, _vp, _dp]),
    "slb_grid_nearest_index": (C.c_int, [_vp, C.POINTER(SlbGrid), _dp, _i64, _vp]),
    "slb_gp_mean": (C.c_int, [_vp, C.POINTER(SlbGpStack), _dp, _i64, _dp]),
    "slb_gp_vjp_workspace": (C.c_int64, [C.POINTER(SlbGpStack), _i64]),
    "slb_gp_vjp": (C.c_int, [_vp, C.POINTER(SlbGpStack), _dp, _i64, _dp, _dp, _dp, _vp]),
    "slb_gp_lml_grad_workspace": (C.c_int64, [_i32]),
    "slb_gp_lml_grad": (C.c_int, [_vp, _dp, _i32, _i32, C.POINTER(SlbKernel), _dp, _dp, _dp, _vp]),
    "slb_gp_lml_grad_cols": (C.c_int, [_vp, _dp, _i32, _i32, C.POINTER(SlbKernel), _dp, _dp, _i32, _dp, _vp]),
}

_lib = None


def load():
    """Load libslb200.so (once). Raises NativeLibraryError if it is missing or mismatched."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeLibraryError(
            "%s not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). safe_learning_b200 has no CPU fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if lib.slb_abi_version() != ABI_VERSION:
        raise NativeLibraryError("libslb200 ABI version %d != %d (rebuild: python -c 'import "
                                 "__graft_entry__ as g; g.build()')"
                                 % (lib.slb_abi_version(), ABI_VERSION))
    _check_layout(lib)
    _lib = lib
    return lib


def _check_layout(lib):
    sizes = (C.c_int64 * len(_STRUCTS))()
    n = lib.slb_struct_sizes(sizes, len(_STRUCTS))
    if n != len(_STRUCTS):
        raise NativeLibraryError("libslb200 reports %d ABI structs, binding has %d"
                                 % (n, len(_STRUCTS)))
    for st, size in zip(_STRUCTS, sizes):
        if C.sizeof(st) != size:
            raise NativeLibraryError("layout mismatch for %s: ctypes %d bytes, C %d bytes"
                                     % (st.__name__, C.sizeof(st), size))


def last_error():
    return load().slb_last_error().decode("utf-8", "replace")


def check(rc, what):
    """Turn a non-zero return code into an exception carrying slb_last_error()."""
    if rc != 0:
        raise NativeLibraryError("%s failed (rc=%d): %s" % (what, rc, last_error()))


def require_device():
    """Fail loudly when there is no CUDA device (no CPU fallback exists)."""
    lib = load()
    n = lib.slb_device_count()
    if n <= 0:
        raise NativeLibraryError("no CUDA device available: %s" % (last_error() or "count=0"))
    return n


def launch_count():
    return int(load().slb_launch_count())
