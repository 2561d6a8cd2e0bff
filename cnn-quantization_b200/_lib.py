"""ctypes binding of the C ABI declared in include/fqb200.h (libfqb200.so, built by build.py).

There is no CPU fallback: if the library is missing the import of any compute entry point raises.
"""
import ctypes
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("FQB200_LIB") or os.path.join(HERE, "libfqb200.so")  # env override: A/B builds in development

OK, ERR_INVALID, ERR_WORKSPACE, ERR_CUDA, ERR_UNSUPPORTED = 0, 1, 2, 3, 4
SCOPE_GROUP, SCOPE_GROUP_MEAN, SCOPE_TENSOR = 0, 1, 2
RANGE_MINMAX, RANGE_LAPLACE, RANGE_GAUS, RANGE_KSTD, RANGE_GIVEN = 0, 1, 2, 3, 4
LEAF_TORCH, LEAF_COMPILED, LEAF_MIDTREAD = 0, 1, 2
PRIOR_STD, PRIOR_B = 0, 1
STATS_STRIDE = 12
STAT_COLUMNS = ("min", "max", "mean", "b", "std", "delta", "offset", "bits", "scale", "zero_point", "qmax", "flags")

ABI_VERSION = 3


class Desc(ctypes.Structure):
    """struct fqb200_desc (include/fqb200.h)."""
    _fields_ = [
        ("outer", ctypes.c_int64), ("groups", ctypes.c_int64), ("inner", ctypes.c_int64),
        ("scope", ctypes.c_int32), ("range_mode", ctypes.c_int32), ("leaf", ctypes.c_int32),
        ("num_bits", ctypes.c_int32), ("positive", ctypes.c_int32), ("solve_f64", ctypes.c_int32),
        ("clip_k", ctypes.c_float),
        ("bit_alloc", ctypes.c_int32), ("bit_alloc_prior", ctypes.c_int32), ("bit_alloc_round", ctypes.c_int32),
        ("bit_alloc_target", ctypes.c_float),
        ("mt_target", ctypes.c_float), ("mt_clip", ctypes.c_int32),
        ("bias_corr", ctypes.c_int32), ("var_corr", ctypes.c_int32), ("stats_only", ctypes.c_int32),
        ("out_stats", ctypes.c_void_p),
        ("bias", ctypes.c_void_p),
        ("bias_period", ctypes.c_int64),
        ("channels_last", ctypes.c_int32),
        ("out_hist", ctypes.c_void_p),
        ("hist_bins", ctypes.c_int32), ("hist_offset", ctypes.c_int32),
        ("out_hist_clamped", ctypes.c_void_p),
        ("relu_passthrough", ctypes.c_int32),
        ("residual", ctypes.c_void_p), ("residual_relu", ctypes.c_int32),
        ("residual_stats", ctypes.c_void_p), ("residual_bias", ctypes.c_void_p),
        ("pool", ctypes.c_int32), ("pool_h", ctypes.c_int64), ("pool_w", ctypes.c_int64), ("pool_out", ctypes.c_void_p),
        ("given_delta", ctypes.c_void_p), ("given_offset", ctypes.c_void_p), ("given_bits", ctypes.c_void_p),
        ("debug_stamps", ctypes.c_void_p),
    ]


_vp, _i64, _i32, _f32, _sz, _desc = (ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_float, ctypes.c_size_t,
                                      ctypes.POINTER(Desc))
# name -> (restype, argtypes) of every function include/fqb200.h declares (tests check the export table against this)
PROTOTYPES = {
    "fqb200_abi_version": (_i32, []),
    "fqb200_last_error": (ctypes.c_char_p, []),
    "fqb200_resident_ctas": (_i32, []),
    "fqb200_plan_info": (_i32, [_desc, ctypes.POINTER(ctypes.c_int64)]),
    "fqb200_selftest_division": (_i32, [_vp, _vp, _vp, _vp, _i64, _vp]),
    "fqb200_workspace_bytes": (_sz, [_desc]),
    "fqb200_workspace_init": (_i32, [_vp, _sz, _vp]),
    "fqb200_float2gemmlowp": (_i32, [_vp, _vp, _i64, _f32, _f32, _i32, _i32, _i32, _vp, _vp]),
    "fqb200_quantize1": (_i32, [_vp, _vp, _vp, _i64, _i64, _i64, _vp, _vp, _vp, _i32, _i32, _vp, _i32, _vp]),
    "fqb200_quantize1_bca": (_i32, [_vp, _vp, _i64, _i64, _i64, _vp, _vp, _vp, _i32, _i32, _vp, _i32, _vp, _vp, _sz, _vp]),
    "fqb200_fused": (_i32, [_desc, _vp, _vp, _vp, _sz, _vp]),
    "fqb200_fused_into": (_i32, [_desc, _vp, _vp, _i64, _vp, _sz, _vp]),
    "fqb200_add_relu": (_i32, [_vp, _vp, _vp, _i64, _vp]),
    "fqb200_maxpool2d_nhwc": (_i32, [_vp, _vp, _i64, _i64, _i64, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _vp]),
    "fqb200_maxpool2d_nhwc_into": (_i32, [_vp, _vp, _i64, _i64, _i64, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _i64, _vp]),
    "fqb200_kld_threshold": (_i32, [_vp, _i64, _i64, _i32, _i32, _vp, _vp, _vp, _vp, _sz, _vp]),
    "fqb200_kld_workspace_bytes": (_sz, [_i64, _i32]),
    "fqb200_sample_sumsq": (_i32, [_vp, _i64, _i64, _vp, _vp, _sz, _vp]),
    "fqb200_sample_sumsq_workspace_bytes": (_sz, [_i64, _i64]),
    "fqb200_clip_error": (_i32, [_vp, _i64, _i64, _i64, _i32, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _sz, _i32, _vp]),
    "fqb200_clip_error_workspace_bytes": (_sz, [_i64, _i64, _i64, _i32]),
    "fqb200_clip_mse": (_i32, [_vp, _i64, _i64, _i64, _i32, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _i32, _vp, _vp, _vp, _sz,
                               _i32, _vp]),
    "fqb200_clip_mse_widths": (_i32, [_vp, _i64, _i64, _i64, _i32, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _vp, _i32, _vp, _vp,
                                      _vp, _sz, _i32, _vp]),
    "fqb200_clip_mse_select": (_i32, [_vp, _i64, _i64, _i64, _i32, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _i32, _vp, _vp,
                                      _vp, _vp, _vp, _vp, _sz, _i32, _vp]),
    "fqb200_clip_mse_workspace_bytes": (_sz, [_i64, _i64, _i64, _i32, _i32]),
    "fqb200_clip_mse_grid": (_i32, [_vp, _i64, _i64, _i64, _i32, _vp, _i32, _i32, _i32, _i32, _i32, _vp, _i32, _vp, _i32, _vp,
                                    _vp, _vp, _sz, _i32, _vp]),
    "fqb200_clip_mse_grid_workspace_bytes": (_sz, [_i64, _i64, _i64, _i32, _i32, _i32]),
    "fqb200_kmeans1d": (_i32, [_vp, _i64, _i32, _i64, _vp, _i32, _vp, _i32, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz,
                               _i32, _vp]),
    "fqb200_kmeans1d_workspace_bytes": (_sz, [_i64, _i32]),
    "fqb200_sample_angles": (_i32, [_vp, _i64, _i64, _vp, _vp, _vp, _sz, _i32, _vp]),
    "fqb200_sample_angles_workspace_bytes": (_sz, [_i64, _i64]),
    "fqb200_sample_noise": (_i32, [_vp, _vp, _vp, _i64, _i64, _i64, _vp, _vp, _sz, _i32, _vp]),
    "fqb200_sample_noise_workspace_bytes": (_sz, [_i64, _i64]),
    "fqb200_quantize_weights_given": (_i32, [_vp, _vp, _i64, _i64, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _sz, _vp]),
    "fqb200_quantize_weights_given_workspace_bytes": (_sz, [_i64, _i64, _i32, _i32, _i32, _i32]),
    "fqb200_allocate_widths": (_i32, [_vp, _i64, ctypes.c_double, _vp, _vp, _vp, _sz, _vp]),
    "fqb200_allocate_widths_workspace_bytes": (_sz, [_i64, ctypes.c_double]),
    "fqb200_allocate_select": (_i32, [_vp, _vp, _vp, _i32, _vp, _i64, ctypes.c_double, _vp, _vp, _vp, _vp, _vp, _vp, _sz,
                                      _vp]),
    "fqb200_allocate_select_workspace_bytes": (_sz, [_i64, ctypes.c_double]),
}
SYMBOLS = tuple(PROTOTYPES)


class FqError(RuntimeError):
    pass


_lib = None


def load():
    """Load libfqb200.so (once) and declare the prototypes.  Raises if the library has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise FqError("libfqb200.so is not built (run `python cnn-quantization_b200/build.py` or "
                      "__graft_entry__.build()); there is no CPU fallback for the fake-quantization path")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (restype, argtypes) in PROTOTYPES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    if lib.fqb200_abi_version() != ABI_VERSION:
        raise FqError("libfqb200.so ABI version mismatch")
    _lib = lib
    return lib


def check(rc):
    if rc != OK:
        raise FqError("fqb200 error %d: %s" % (rc, load().fqb200_last_error().decode()))
