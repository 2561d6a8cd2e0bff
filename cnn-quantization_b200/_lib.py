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

# every symbol include/fqb200.h declares (tests check the export table against this)
SYMBOLS = ("fqb200_abi_version", "fqb200_last_error", "fqb200_resident_ctas", "fqb200_plan_info",
           "fqb200_selftest_division", "fqb200_workspace_bytes", "fqb200_workspace_init", "fqb200_float2gemmlowp",
           "fqb200_quantize1", "fqb200_quantize1_bca", "fqb200_fused", "fqb200_fused_into", "fqb200_add_relu",
           "fqb200_maxpool2d_nhwc", "fqb200_maxpool2d_nhwc_into",
           "fqb200_kld_threshold", "fqb200_kld_workspace_bytes", "fqb200_sample_sumsq",
           "fqb200_sample_sumsq_workspace_bytes", "fqb200_clip_error", "fqb200_clip_error_workspace_bytes",
           "fqb200_kmeans1d", "fqb200_kmeans1d_workspace_bytes", "fqb200_sample_angles",
           "fqb200_sample_angles_workspace_bytes")
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
    vp, i64, i32, f32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_float
    lib.fqb200_abi_version.restype = i32
    lib.fqb200_abi_version.argtypes = []
    lib.fqb200_last_error.restype = ctypes.c_char_p
    lib.fqb200_last_error.argtypes = []
    lib.fqb200_resident_ctas.restype = i32
    lib.fqb200_resident_ctas.argtypes = []
    lib.fqb200_workspace_bytes.restype = ctypes.c_size_t
    lib.fqb200_workspace_bytes.argtypes = [ctypes.POINTER(Desc)]
    lib.fqb200_workspace_init.restype = i32
    lib.fqb200_workspace_init.argtypes = [vp, ctypes.c_size_t, vp]
    lib.fqb200_float2gemmlowp.restype = i32
    lib.fqb200_float2gemmlowp.argtypes = [vp, vp, i64, f32, f32, i32, i32, i32, vp, vp]
    lib.fqb200_quantize1.restype = i32
    lib.fqb200_quantize1.argtypes = [vp, vp, vp, i64, i64, i64, vp, vp, vp, i32, i32, vp, i32, vp]
    lib.fqb200_fused.restype = i32
    lib.fqb200_fused.argtypes = [ctypes.POINTER(Desc), vp, vp, vp, ctypes.c_size_t, vp]
    lib.fqb200_fused_into.restype = i32
    lib.fqb200_fused_into.argtypes = [ctypes.POINTER(Desc), vp, vp, i64, vp, ctypes.c_size_t, vp]
    lib.fqb200_quantize1_bca.restype = i32
    lib.fqb200_quantize1_bca.argtypes = [vp, vp, i64, i64, i64, vp, vp, vp, i32, i32, vp, i32, vp, vp, ctypes.c_size_t, vp]
    lib.fqb200_maxpool2d_nhwc.restype = i32
    lib.fqb200_maxpool2d_nhwc.argtypes = [vp, vp, i64, i64, i64, i64, i32, i32, i32, i32, i32, i32, vp]
    lib.fqb200_maxpool2d_nhwc_into.restype = i32
    lib.fqb200_maxpool2d_nhwc_into.argtypes = [vp, vp, i64, i64, i64, i64, i32, i32, i32, i32, i32, i32, i64, vp]
    lib.fqb200_add_relu.restype = i32
    lib.fqb200_add_relu.argtypes = [vp, vp, vp, i64, vp]
    lib.fqb200_selftest_division.restype = i32
    lib.fqb200_selftest_division.argtypes = [vp, vp, vp, vp, i64, vp]
    lib.fqb200_kld_threshold.restype = i32
    lib.fqb200_kld_threshold.argtypes = [vp, i64, i64, i32, i32, vp, vp, vp, vp, ctypes.c_size_t, vp]
    lib.fqb200_kld_workspace_bytes.restype = ctypes.c_size_t
    lib.fqb200_kld_workspace_bytes.argtypes = [i64, i32]
    lib.fqb200_sample_sumsq.restype = i32
    lib.fqb200_sample_sumsq.argtypes = [vp, i64, i64, vp, vp, ctypes.c_size_t, vp]
    lib.fqb200_sample_sumsq_workspace_bytes.restype = ctypes.c_size_t
    lib.fqb200_sample_sumsq_workspace_bytes.argtypes = [i64, i64]
    lib.fqb200_sample_angles.restype = i32
    lib.fqb200_sample_angles.argtypes = [vp, i64, i64, vp, vp, vp, ctypes.c_size_t, i32, vp]
    lib.fqb200_sample_angles_workspace_bytes.restype = ctypes.c_size_t
    lib.fqb200_sample_angles_workspace_bytes.argtypes = [i64, i64]
    lib.fqb200_clip_error.restype = i32
    lib.fqb200_clip_error.argtypes = [vp, i64, i64, i64, i32, vp, i32, i32, i32, i32, vp, vp, vp, ctypes.c_size_t, i32, vp]
    lib.fqb200_clip_error_workspace_bytes.restype = ctypes.c_size_t
    lib.fqb200_clip_error_workspace_bytes.argtypes = [i64, i64, i64, i32]
    lib.fqb200_kmeans1d.restype = i32
    lib.fqb200_kmeans1d.argtypes = [vp, i64, i32, i64, vp, i32, vp, i32, i64, vp, vp, vp, vp, vp, vp, vp, vp, ctypes.c_size_t,
                                    i32, vp]
    lib.fqb200_kmeans1d_workspace_bytes.restype = ctypes.c_size_t
    lib.fqb200_kmeans1d_workspace_bytes.argtypes = [i64, i32]
    lib.fqb200_plan_info.restype = i32
    lib.fqb200_plan_info.argtypes = [ctypes.POINTER(Desc), ctypes.POINTER(ctypes.c_int64)]
    if lib.fqb200_abi_version() != ABI_VERSION:
        raise FqError("libfqb200.so ABI version mismatch")
    _lib = lib
    return lib


def check(rc):
    if rc != OK:
        raise FqError("fqb200 error %d: %s" % (rc, load().fqb200_last_error().decode()))
