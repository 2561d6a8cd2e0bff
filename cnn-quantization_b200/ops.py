"""Tensor-level wrappers over the C ABI: device pointers and the current stream come from torch, the
arithmetic all happens in libfqb200.so.  Nothing here synchronises with the host."""
import collections
import ctypes

import numpy as np
import torch

from . import _lib as L

_workspaces = {}  # (device index, stream handle) -> uint8 tensor

# ---- optional per-launch timing (bench.py): CUDA events recorded on the launching stream around each call --------
_prof = {"on": False, "records": [], "launches": 0}


def profile_reset(enable):
    _prof["on"] = bool(enable)
    _prof["records"] = []
    _prof["launches"] = 0


def profile_collect():
    """Synchronise and return {'launches': n, 'modes': {mode: {launches, elems, bytes, ms}}}.  Modes by algorithmic
    traffic: 'D' two statistics passes + apply (16 B/elem), 'B' one statistics pass + apply (12), 'A' apply only (8),
    'S' statistics only; 'K' the KLD calibration (ops.kld_threshold), 'M' the activation norm measurement
    (ops.sample_sumsq), 'G' the sample-angle measurement (ops.sample_angles), 'N' the quantization-noise measurement
    (ops.sample_noise), 'E' the clipping-error measurement (ops.clip_error), 'R' the clipping-MSE curves (ops.clip_mse,
    and with the choice of each group's clipping value ops.clip_mse_select) and 'C' the k-means clustering of a weight tensor (ops.kmeans1d), which quantize nothing; 'W' the given-parameter
    weight launch with its corrections (ops.quantize_weights_given) and 'L' the width allocation (ops.allocate_widths,
    and from a call site's error sums to its parameters ops.allocate_select)."""
    torch.cuda.synchronize()
    modes, shapes = {}, {}
    for mode, elems, nbytes, e0, e1, tag in _prof["records"]:
        ms = e0.elapsed_time(e1)
        for table, key in ((modes, mode), (shapes, "%s %s" % (mode, tag))):
            m = table.setdefault(key, {"launches": 0, "elems": 0, "bytes": 0, "ms": 0.0})
            m["launches"] += 1
            m["elems"] += elems
            m["bytes"] += nbytes
            m["ms"] += ms
    return {"launches": _prof["launches"], "modes": modes, "shapes": shapes}


class _Timed(object):
    def __init__(self, mode, elems, bytes_per_elem, tag=""):
        self.args = (mode, elems, elems * bytes_per_elem)
        self.tag = tag

    def __enter__(self):
        _prof["launches"] += 1
        if _prof["on"]:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e1 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def __exit__(self, *exc):
        if _prof["on"]:
            self.e1.record()
            _prof["records"].append(self.args + (self.e0, self.e1, self.tag))


def _stream_handle(device):
    return torch.cuda.current_stream(device).cuda_stream


def _require_cuda_f32(t, name):
    if not isinstance(t, torch.Tensor):
        raise TypeError("%s must be a torch.Tensor" % name)
    if not t.is_cuda:
        raise L.FqError("%s must live on a CUDA device: the fake-quantization path has no CPU implementation" % name)
    if t.dtype != torch.float32:
        raise TypeError("%s must be float32, got %s" % (name, t.dtype))


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _launch(dev, timed, fn, *args):
    """``fn(*args, stream)`` on the current stream of ``dev``, recorded in the launch profile by ``timed`` (a ``_Timed``);
    raises on an error code."""
    with torch.cuda.device(dev), timed:
        L.check(fn(*args, _stream_handle(dev)))


def _workspace(device, stream, nbytes):
    key = (device.index, stream)
    ws = _workspaces.get(key)
    if ws is None or ws.numel() < nbytes:
        size = max(int(nbytes), 1 << 20)
        ws = torch.empty(size, dtype=torch.uint8, device=device)
        L.check(L.load().fqb200_workspace_init(ws.data_ptr(), ws.numel(), stream))
        _workspaces[key] = ws
    return ws


def _own_workspace(device, need, required=True):
    """A workspace for one launch that zeroes or fills it itself (the shared ``_workspace`` keeps the fused kernels'
    barriers): ``need`` bytes as the entry point's sizer reports them, None for 0.  ``required``: 0 is the sizer refusing
    the arguments; raise its error."""
    if not need and required:
        L.check(L.ERR_INVALID)
    return torch.empty(need, dtype=torch.uint8, device=device) if need else None


def _samples(x, what):
    """(x, rows, row_len) of a float32 CUDA tensor read sample by sample (dim 0).  A sample is contiguous in NCHW and in
    channels-last memory; anything else is copied."""
    _require_cuda_f32(x, "tensor")
    if x.dim() == 0:
        raise ValueError("%s needs a tensor with a sample dimension" % what)
    if not dense(x):
        x = x.contiguous()
    rows = x.shape[0]
    return x, rows, (x.numel() // rows if rows else 0)


def nhwc(x):
    """True when ``x`` is 4-D and stored channels-last without also being NCHW-contiguous (C == 1, H == W == 1)."""
    return x.dim() == 4 and not x.is_contiguous() and x.is_contiguous(memory_format=torch.channels_last)


def dense(t):
    return t.is_contiguous() or nhwc(t)


def cl_channels_ok(c):
    """Channel counts the channels-last kernels take (flat_eligible in fqb200.cu)."""
    return c % 4 == 0 and 4 <= c <= 2048


def cl_eligible(x, layout=None):
    """True when ``x`` is an NCHW-shaped activation stored channels-last that the flat-stream kernels take as it is:
    C % 4 == 0, C <= 2048, 16-byte aligned (``layout``, when given, must be its (N, C, H*W) view)."""
    if not nhwc(x):
        return False
    n, c = x.shape[0], x.shape[1]
    if layout is not None and tuple(int(v) for v in layout) != (n, c, x.numel() // (n * c)):
        return False
    return cl_channels_ok(c) and x.data_ptr() % 16 == 0


def slice_pitch(out):
    """Floats between two pixels of ``out`` when it is an [N, C, H, W] channel slice of a wider channels-last tensor (channel
    stride 1, rows and images packed at that pixel pitch), else 0."""
    if out.dim() != 4 or out.stride(1) != 1:
        return 0
    p = out.stride(3)
    return p if out.stride(2) == out.shape[3] * p and out.stride(0) == out.shape[2] * out.shape[3] * p else 0


def _overlaps(x, out, pitch):
    pixels = out.numel() // max(out.shape[1], 1)
    x0, o0 = x.data_ptr(), out.data_ptr()
    return o0 < x0 + 4 * x.numel() and x0 < o0 + 4 * ((pixels - 1) * pitch + out.shape[1])


def slice_eligible(x, out, channels_last=True, stats_only=False, pool=None, residual=None, bias_period=0):
    """True when a launch of ``fused`` on ``x`` writes ``out``, a channel slice of a wider channels-last tensor
    (``slice_pitch``), in place (C ABI fqb200_fused_into; the library applies the same rules): a channels-last apply launch,
    or a per-sample / per-tensor min-max launch (``channels_last=False``) that knows C from its channel-fastest bias
    (``bias_period`` = -C, at most 4096 samples), without pooling or residual on a ``cl_eligible`` x, the pixel pitch >= C
    and a multiple of 4, ``out`` 16-byte aligned, not overlapping x."""
    rows_cl = not channels_last and bias_period < 0 and -bias_period == x.shape[1] and x.shape[0] <= 4096
    if (not (channels_last or rows_cl) or stats_only or pool is not None or residual is not None or not cl_eligible(x)
            or tuple(out.shape) != tuple(x.shape)):
        return False
    p = slice_pitch(out)
    return (p >= x.shape[1] and p % 4 == 0 and out.data_ptr() % 16 == 0 and not _overlaps(x, out, p)
            and (out.numel() // x.shape[1]) * p // 4 < 2 ** 32)


def rows_eligible(x, other=None):
    """True when the per-sample / per-tensor min-max kernel takes the 4-D ``x`` (and ``other``, an operand read alongside)
    as it is: dense, N <= 4096 samples of a multiple of 4 elements, 16-byte aligned (rows_supported in fqb200.cu)."""
    if x.dim() != 4 or not dense(x):
        return False
    n = x.shape[0]
    return n <= 4096 and (x.numel() // n) % 4 == 0 and x.data_ptr() % 16 == 0 and (other is None or other.data_ptr() % 16 == 0)


# 3x3 pooling: one tile reads three input rows of at least 3 pixels, 9 * C/4 vectors, from one ring stage.  This mirrors
# the tile-width search of fqb200_fused, which would take a few channels more (C <= 908 with the default stage size).
POOL3_MAX_CHANNELS = 896


def pool_request_ok(x, pool, nhwc_launch, stats_only=False, residual=None, hist=None):
    """True when ``fused`` accepts ``pool``: (2, 2) or (3, 3) on a launch that reads channels-last memory (``nhwc_launch``: a
    channels_last launch, or a rows launch told C by a channel-fastest bias), no residual / histogram, W even (3x3: H too)."""
    return (tuple(pool) in ((2, 2), (3, 3)) and nhwc_launch and not stats_only and residual is None and hist is None
            and x.shape[3] % 2 == 0 and (pool[0] == 2 or x.shape[2] % 2 == 0))


def pool_tile_fits(x, kind):
    """True when the library finds a pooling tile for the channels-last [N, C, H, W] ``x`` (``kind`` 2 or 3)."""
    return x.shape[2] >= 2 and x.shape[3] >= 2 and (kind == 2 or x.shape[1] <= POOL3_MAX_CHANNELS)


def _resolve_out(x, out):
    """(tensor the kernel writes, tensor the caller gets back).  ``x`` is the tensor handed to the kernel, i.e. AFTER any
    ``.contiguous()`` re-layout; ``out`` is the caller's output tensor or None.  The kernels write linearly in the memory
    order of ``x``, so the caller's tensor is used directly only when it has exactly that memory order (same strides);
    otherwise (e.g. an NHWC-strided ``out`` while the kernel runs on an NCHW copy) the result is produced in a scratch
    tensor and copied back element for element."""
    if out is None:
        return torch.empty_like(x), None
    if out.shape != x.shape:
        raise ValueError("out must have the shape of the input, got %r vs %r" % (tuple(out.shape), tuple(x.shape)))
    _require_cuda_f32(out, "out")
    if out.stride() == x.stride():
        return out, None
    return torch.empty_like(x), out


def _finish_out(kernel_out, user_out):
    if user_out is None:
        return kernel_out
    user_out.copy_(kernel_out)
    return user_out


def resident_ctas():
    return L.load().fqb200_resident_ctas()


def float2gemmlowp(x, range_, offset, num_bits, int_exp, enforce_true_zero, noise=None, out=None):
    """C ABI fqb200_float2gemmlowp on torch tensors (scalars by value, like the reference's pybind call)."""
    _require_cuda_f32(x, "in")
    lib = L.load()
    if noise is not None:
        _require_cuda_f32(noise, "noise")
        if noise.shape != x.shape:
            raise ValueError("noise must have the shape of the input")
    # one parameter set for the whole tensor: any dense memory order will do (no copy for channels-last activations)
    if not dense(x) or (noise is not None and noise.stride() != x.stride()):
        x = x.contiguous()
        noise = noise.contiguous() if noise is not None else None
    kout, uout = _resolve_out(x, out)
    _launch(x.device, _Timed("A", x.numel(), 8), lib.fqb200_float2gemmlowp, x.data_ptr(), kout.data_ptr(), x.numel(),
            float(range_), float(offset), int(num_bits), int(bool(int_exp)), int(bool(enforce_true_zero)), _ptr(noise))
    return _finish_out(kout, uout)


def quantize1(x, delta, offset, num_bits, bits=None, layout=None, want_grid=False, out=None, bias=None):
    """C ABI fqb200_quantize1.  ``layout`` = (outer, groups, inner); default: [R, K] rows with per-row
    parameters when ``delta`` has R elements, else one parameter set for the whole tensor."""
    _require_cuda_f32(x, "tensor")
    lib = L.load()
    dev = x.device
    delta = torch.as_tensor(delta, dtype=torch.float32, device=dev).contiguous()
    offset = torch.as_tensor(offset, dtype=torch.float32, device=dev).contiguous()
    per_group = delta.numel() > 1 or (bits is not None)
    # channels-last activations with per-channel parameters run on the NHWC memory as it is (layout = (N, C, H*W));
    # one parameter set for the whole tensor does not care about the memory order at all
    cl = bool(per_group and layout is not None and cl_eligible(x, layout))
    if not cl and (per_group or not dense(x)):
        x = x.contiguous()
    if layout is None:
        layout = (1, x.shape[0], x.numel() // x.shape[0]) if per_group else (1, 1, x.numel())
    outer, groups, inner = layout
    if per_group:
        if delta.numel() == 1:
            delta = delta.reshape(1).expand(groups).contiguous()
        if offset.numel() == 1:
            offset = offset.reshape(1).expand(groups).contiguous()
        if delta.numel() != groups or offset.numel() != groups:
            raise ValueError("per-group parameters must have %d elements" % groups)
    if bits is not None:
        bits = torch.as_tensor(bits, dtype=torch.float32, device=dev).contiguous()
        if bits.numel() != groups:
            raise ValueError("bit_alloc must have %d elements" % groups)
    if bias is not None:
        _require_cuda_f32(bias, "bias")
        bias = bias.contiguous()
        if bias.numel() != groups:
            raise ValueError("bias must have one element per group (%d)" % groups)
    kout, uout = _resolve_out(x, out)
    grid = torch.empty_like(x) if want_grid else None
    _launch(dev, _Timed("A", x.numel(), 8, "%dx%dx%d" % (outer, groups, inner)), lib.fqb200_quantize1, x.data_ptr(),
            kout.data_ptr(), _ptr(grid), outer, groups, inner, delta.data_ptr(), offset.data_ptr(), _ptr(bits),
            int(per_group), int(num_bits), _ptr(bias), int(cl))
    out = _finish_out(kout, uout)
    return (out, grid) if want_grid else out


def quantize1_bca(x, delta, offset, num_bits, bits=None, bias=None, relu_first=False, out=None, want_qbias=False):
    """C ABI fqb200_quantize1_bca: given-parameter quantization of a channels-last [N, C, H, W] activation with the
    reference's activation bias correction (`-bca`, inference_quantization_manager.py:180-196) in the same launch.
    ``x`` must satisfy ``cl_eligible``.  Returns the corrected quantized tensor (and the [C] corrections)."""
    _require_cuda_f32(x, "tensor")
    if not cl_eligible(x):
        raise ValueError("quantize1_bca needs a channels-last activation with C % 4 == 0, C <= 2048")
    lib = L.load()
    dev = x.device
    n, c = x.shape[0], x.shape[1]
    inner = x.numel() // (n * c)
    delta = torch.as_tensor(delta, dtype=torch.float32, device=dev).contiguous()
    offset = torch.as_tensor(offset, dtype=torch.float32, device=dev).contiguous()
    per_group = delta.numel() > 1 or bits is not None
    if per_group:
        delta = delta.reshape(-1).expand(c).contiguous() if delta.numel() == 1 else delta
        offset = offset.reshape(-1).expand(c).contiguous() if offset.numel() == 1 else offset
    if bits is not None:
        bits = torch.as_tensor(bits, dtype=torch.float32, device=dev).contiguous()
    if bias is not None:
        _require_cuda_f32(bias, "bias")
        bias = bias.contiguous()
    kout, uout = _resolve_out(x, out)
    qb = torch.empty(c, dtype=torch.float32, device=dev) if want_qbias else None
    d = L.Desc()
    d.outer, d.groups, d.inner, d.num_bits, d.channels_last = n, c, inner, 8, 1
    with torch.cuda.device(dev):
        ws = _workspace(dev, _stream_handle(dev), lib.fqb200_workspace_bytes(ctypes.byref(d)))
    _launch(dev, _Timed("C", x.numel(), 12, "%dx%dx%d" % (n, c, inner)), lib.fqb200_quantize1_bca, x.data_ptr(),
            kout.data_ptr(), n, c, inner, delta.data_ptr(), offset.data_ptr(), _ptr(bits), int(per_group), int(num_bits),
            _ptr(bias), int(bool(relu_first)), _ptr(qb), ws.data_ptr(), ws.numel())
    res = _finish_out(kout, uout)
    return (res, qb) if want_qbias else res


def fused(x, layout, *, scope=L.SCOPE_GROUP, range_mode=L.RANGE_MINMAX, leaf=L.LEAF_TORCH, num_bits=8,
          positive=False, solve_f64=False, clip_k=0.0, bit_alloc=False, bit_alloc_prior=L.PRIOR_STD,
          bit_alloc_round=True, bit_alloc_target=None, mt_target=0.0, mt_clip=False, bias_corr=False,
          var_corr=False, stats_only=False, want_stats=False, out=None, bias=None, bias_period=0, hist=None,
          channels_last=False, any_dense_format=False, debug_stamps=None, relu_passthrough=False, hist_offset=0,
          hist_clamped=None, residual=None, residual_relu=False, residual_stats=None, residual_bias=None, pool=None, given=None):
    """C ABI fqb200_fused: statistics -> parameters -> quantize/dequantize in one launch.

    Returns ``out`` (or ``(out, stats)`` with ``want_stats``; ``stats`` alone with ``stats_only``), where
    ``stats`` is a [groups, 12] tensor with columns ``_lib.STAT_COLUMNS``.  A channels-last launch, or a per-sample /
    per-tensor min-max launch on channels-last memory with a channel-fastest bias (``bias_period`` = -C), writes an ``out``
    that is a channel slice of a wider channels-last tensor directly (``slice_eligible``; profile mode suffix "i")."""
    _require_cuda_f32(x, "tensor")
    lib = L.load()
    is_cl = x.dim() == 4 and x.is_contiguous(memory_format=torch.channels_last)
    if channels_last:
        # layout = (N, C, H*W) of a tensor stored [N][H*W][C]
        if not is_cl:
            raise ValueError("channels_last=True needs a channels-last contiguous 4-D tensor")
    elif not (any_dense_format and is_cl):
        # any_dense_format: the layout does not care about the order inside a sample (per-tensor / per-sample min-max)
        x = x.contiguous()
    dev = x.device
    outer, groups, inner = (int(v) for v in layout)
    if outer * groups * inner != x.numel():
        raise ValueError("layout %r does not cover %d elements" % (layout, x.numel()))
    d = L.Desc()
    d.outer, d.groups, d.inner = outer, groups, inner
    d.scope, d.range_mode, d.leaf = scope, range_mode, leaf
    d.num_bits, d.positive, d.solve_f64 = int(num_bits), int(bool(positive)), int(bool(solve_f64))
    d.clip_k = float(clip_k)
    d.bit_alloc, d.bit_alloc_prior, d.bit_alloc_round = int(bool(bit_alloc)), bit_alloc_prior, int(bool(bit_alloc_round))
    d.bit_alloc_target = float(bit_alloc_target if bit_alloc_target is not None else num_bits)
    d.mt_target, d.mt_clip = float(mt_target), int(bool(mt_clip))
    d.bias_corr, d.var_corr, d.stats_only = int(bool(bias_corr)), int(bool(var_corr)), int(bool(stats_only))
    d.channels_last = int(bool(channels_last))
    if bias is not None:
        _require_cuda_f32(bias, "bias")
        bias = bias.contiguous()
        want = (inner // bias_period if bias_period > 0 else -bias_period) if bias_period else groups
        if bias.numel() != want:
            raise ValueError("bias must have %d elements" % want)
        d.bias = bias.data_ptr()
        d.bias_period = int(bias_period)
    else:
        d.bias = None
        d.bias_period = 0
    d.hist_bins, d.hist_offset, d.out_hist_clamped = 0, 0, None
    if hist is not None:
        if hist.dtype != torch.int64 or not hist.is_cuda or not hist.is_contiguous() or not (1 <= hist.numel() <= 8192):
            raise ValueError("hist must be a contiguous CUDA int64 tensor of at most 8192 counters")
        d.out_hist = hist.data_ptr()
        d.hist_bins, d.hist_offset = hist.numel(), int(hist_offset)
        if hist_clamped is not None:
            if hist_clamped.dtype != torch.int64 or not hist_clamped.is_cuda or hist_clamped.numel() != 2 * groups:
                raise ValueError("hist_clamped must be a CUDA int64 tensor [groups, 2]")
            d.out_hist_clamped = hist_clamped.data_ptr()
    else:
        d.out_hist = None
    d.debug_stamps = debug_stamps.data_ptr() if debug_stamps is not None else None
    d.relu_passthrough = int(bool(relu_passthrough))
    d.residual, d.residual_relu = None, 0
    if residual is not None:
        _require_cuda_f32(residual, "residual")
        if residual.shape != x.shape or residual.stride() != x.stride():
            raise ValueError("residual needs a tensor with the input's shape and strides")
        d.residual, d.residual_relu = residual.data_ptr(), int(bool(residual_relu))
    d.residual_stats, d.residual_bias = None, None
    if residual_stats is not None:
        # the [groups, 12] table a stats_only launch exported for the residual tensor: it is quantized on the fly
        if residual is None or residual_stats.dtype != torch.float32 or not residual_stats.is_cuda or not residual_stats.is_contiguous() \
                or residual_stats.dim() != 2 or residual_stats.shape[1] != L.STATS_STRIDE:
            raise ValueError("residual_stats: the contiguous CUDA [groups, %d] table of a stats_only launch, with a residual" % L.STATS_STRIDE)
        d.residual_stats = residual_stats.data_ptr()
        if residual_bias is not None:
            _require_cuda_f32(residual_bias, "residual_bias")
            residual_bias = residual_bias.contiguous()
            if bias is None or residual_bias.numel() != bias.numel():
                raise ValueError("residual_bias must have the form of `bias`")
            d.residual_bias = residual_bias.data_ptr()
    elif residual_bias is not None:
        raise ValueError("residual_bias needs residual_stats")
    d.given_delta, d.given_offset, d.given_bits = None, None, None
    if range_mode == L.RANGE_GIVEN:
        # parameters from the caller (`-sm use`): per-group delta / offset (/ bits) device vectors, no statistics phases
        if given is None or not channels_last or stats_only or want_stats:
            raise ValueError("RANGE_GIVEN needs given=(delta, offset, bits), channels_last=True and no statistics outputs")
        gd, go, gb = given
        keep = []
        for name, v in (("delta", gd), ("offset", go), ("bits", gb)):
            if v is None:
                keep.append(None)
                continue
            _require_cuda_f32(v, "given " + name)
            v = v.contiguous()
            if v.numel() != groups:
                raise ValueError("given %s must have %d elements" % (name, groups))
            keep.append(v)
        if keep[0] is None or keep[1] is None:
            raise ValueError("RANGE_GIVEN needs delta and offset")
        d.given_delta, d.given_offset = keep[0].data_ptr(), keep[1].data_ptr()
        d.given_bits = keep[2].data_ptr() if keep[2] is not None else None
    d.pool, d.pool_h, d.pool_w, d.pool_out = 0, 0, 0, None
    pooled = None
    if pool is not None:
        # a 2x2 / stride-2 max pooling (floor mode) follows and is the only consumer: computed inside the apply phase
        # ((3, 3): stride 2, padding 1, H and W even - the ResNet stem)
        rows_cl = any_dense_format and is_cl and bias is not None and bias_period < 0
        if not pool_request_ok(x, pool, channels_last or rows_cl, stats_only, residual, hist):
            raise ValueError("pool=(2, 2) / (3, 3) needs a channels-last launch with an even W (3x3: and H) and no residual / histogram")
        n_, c_, h_, w_ = x.shape
        pooled = torch.empty((n_, c_, h_ // 2, w_ // 2), dtype=x.dtype, device=dev, memory_format=torch.channels_last)
        d.pool, d.pool_h, d.pool_w, d.pool_out = int(pool[0]), h_, w_, pooled.data_ptr()
    stats = None
    if want_stats or stats_only:
        stats = torch.zeros((groups, L.STATS_STRIDE), dtype=torch.float32, device=dev)
        d.out_stats = stats.data_ptr()
    else:
        d.out_stats = None
    if x.numel() == 0:
        res = pooled if pooled is not None else x.clone()
        return stats if stats_only else ((res, stats) if want_stats else res)
    pitch = 0
    if stats_only or pooled is not None:
        kout, uout = None, None
    elif out is not None and out.stride() != x.stride() and slice_eligible(
            x, out, channels_last, residual=residual, bias_period=bias_period if bias is not None and is_cl else 0):
        _require_cuda_f32(out, "out")
        kout, uout, pitch = out, None, slice_pitch(out)
    else:
        kout, uout = _resolve_out(x, out)
    with torch.cuda.device(dev):
        need = lib.fqb200_workspace_bytes(ctypes.byref(d))
        if need == 0:
            L.check(L.ERR_INVALID)
        ws = _workspace(dev, _stream_handle(dev), need)
    two_pass = (range_mode != L.RANGE_MINMAX or leaf == L.LEAF_MIDTREAD or var_corr or stats_only or
                (bit_alloc and num_bits <= 4 and scope == L.SCOPE_GROUP))
    mode = "S" if stats_only else ("D" if two_pass else "B")
    bpe = (8 if two_pass else 4) + (0 if stats_only else 8)
    if range_mode == L.RANGE_GIVEN:
        mode, bpe = "A", 8
    if residual is not None:   # + the residual read of the fused block epilogue (the write is the apply's own)
        mode, bpe = mode + "r", bpe + 4
    if pooled is not None:     # the apply phase reads x (3x3: rows twice, the second time mostly out of L2) and writes a quarter
        mode, bpe = mode + "p", bpe - 3
    if pitch:                  # written into a channel slice of a wider tensor
        mode += "i"
    _launch(dev, _Timed(mode, x.numel(), bpe, "%dx%dx%d" % (outer, groups, inner)), lib.fqb200_fused_into, ctypes.byref(d),
            x.data_ptr(), _ptr(kout), pitch, ws.data_ptr(), ws.numel())
    if stats_only:
        return stats
    if pooled is not None:
        return (pooled, stats) if want_stats else pooled
    out = _finish_out(kout, uout)
    return (out, stats) if want_stats else out


def kld_threshold(x, num_bins=2001, num_quantized_bins=15, return_hist=False):
    """C ABI fqb200_kld_threshold: the KL-divergence threshold of every sample (dim 0) of ``x``, as the reference's
    kld_threshold._get_optimal_threshold computes it per sample (numpy 1.x histogram edges, divergence in float64).
    Returns device tensors ``(th[N], div[N], idx[N])``: the threshold, its divergence and its position in the search
    (int32); a sample holding NaN / Inf gets NaN, NaN, -1.  With ``return_hist`` the [N, num_bins] int32 bin counts come
    fourth (a view of the workspace).  Recorded in the launch profile under mode 'K' (two reads of the tensor), apart from
    the quantization launches."""
    x, rows, row_len = _samples(x, "kld_threshold")
    lib = L.load()
    dev = x.device
    th = torch.empty(rows, dtype=torch.float32, device=dev)
    div = torch.empty(rows, dtype=torch.float32, device=dev)
    idx = torch.empty(rows, dtype=torch.int32, device=dev)
    if rows == 0:
        return (th, div, idx, torch.zeros((0, num_bins), dtype=torch.int32, device=dev)) if return_hist else (th, div, idx)
    ws = _own_workspace(dev, lib.fqb200_kld_workspace_bytes(rows, int(num_bins)))
    _launch(dev, _Timed("K", x.numel(), 8, "%dx%d" % (rows, row_len)), lib.fqb200_kld_threshold, x.data_ptr(), rows, row_len,
            int(num_bins), int(num_quantized_bins), th.data_ptr(), div.data_ptr(), idx.data_ptr(), ws.data_ptr(), ws.numel())
    if not return_hist:
        return th, div, idx
    head = (rows * 4 + 255) // 256 * 256   # the counters follow the rows' max |x| words (fqb200_kld_threshold)
    return th, div, idx, ws[head:head + rows * num_bins * 4].view(torch.int32).view(rows, num_bins)


def _sample_sums(entry, x, rows, row_len, shape, mode, bytes_per_elem, head, tail=()):
    """The float64 ``shape`` device tensor the per-sample sums entry point ``entry`` writes for ``x`` (rows x row_len, from
    ``_samples``), called as entry(*head, rows, row_len, out, workspace, workspace_bytes, *tail, stream) and recorded in
    the launch profile under ``mode``."""
    dev = x.device
    if rows == 0 or x.numel() == 0:
        return torch.zeros(shape, dtype=torch.float64, device=dev)   # empty samples sum to 0, as in torch
    lib = L.load()
    out = torch.empty(shape, dtype=torch.float64, device=dev)
    need = getattr(lib, entry + "_workspace_bytes")(rows, row_len)
    ws = _own_workspace(dev, need, required=False)
    _launch(dev, _Timed(mode, x.numel(), bytes_per_elem, "%dx%d" % (rows, row_len)), getattr(lib, entry), *head, rows,
            row_len, out.data_ptr(), _ptr(ws), need, *tail)
    return out


def sample_sumsq(x):
    """C ABI fqb200_sample_sumsq: ``x.double().pow(2).sum()`` of every sample (dim 0) of ``x`` as a float64 [N] device
    tensor - the activation norm `-ms` records (distance_stats.py:27-28).  Deterministic (fixed chunks, fixed summation
    order), no host synchronisation.  Recorded in the launch profile under mode 'M' (one read of the tensor), apart from
    the quantization launches."""
    x, rows, row_len = _samples(x, "sample_sumsq")
    return _sample_sums("fqb200_sample_sumsq", x, rows, row_len, (rows,), "M", 4, (x.data_ptr(),))


def sample_angles(x, return_gram=False, max_ctas=0):
    """C ABI fqb200_sample_angles: the pairwise angles between the samples (dim 0) of ``x`` as a float32 [N, N] device
    tensor - ``acos(cos_sim(x[i], x[j]))`` for j > i and 0 on and below the diagonal, the matrix the reference's angle
    measurement records (angle_stats.py:29-37).  The cosine comes from the float64 Gram matrix (FP64 tensor cores), is
    clamped to [-1, 1] (the reference's fp32 cosine can step over 1 and give NaN) and is NaN where it is not finite (a zero
    sample, NaN / Inf input).  With ``return_gram`` also returns the float64 [N, N] Gram matrix (valid for j >= i).
    Deterministic (the bits depend neither on the run nor on ``max_ctas``), no host synchronisation.  Recorded in the launch
    profile under mode 'G' (one read of the tensor)."""
    x, rows, row_len = _samples(x, "sample_angles")
    dev = x.device
    angles = torch.empty((rows, rows), dtype=torch.float32, device=dev)
    gram = torch.empty((rows, rows), dtype=torch.float64, device=dev) if return_gram else None
    if rows > 0:
        if x.numel() == 0:
            raise ValueError("sample_angles needs samples of at least one element")
        lib = L.load()
        need = lib.fqb200_sample_angles_workspace_bytes(rows, row_len)
        ws = _own_workspace(dev, need, required=False)
        _launch(dev, _Timed("G", x.numel(), 4, "%dx%d" % (rows, row_len)), lib.fqb200_sample_angles, x.data_ptr(), rows,
                row_len, angles.data_ptr(), _ptr(gram), _ptr(ws), need, int(max_ctas))
    return (angles, gram) if return_gram else angles


NOISE_SUMS = ("y", "y2", "q", "q2", "yq", "e", "e2")


def sample_noise(y, q=None, bias=None, bias_period=0, max_ctas=0):
    """C ABI fqb200_sample_noise: per sample (dim 0) of ``y`` the float64 sums behind the quantization-noise measurement
    (measure_statistics.py:19-99) as a float64 [N, 7] device tensor, columns ``NOISE_SUMS``: sum y, y^2, q, q^2, y*q, e, e^2
    with e = y - q in float64; without ``q`` the [N, 2] sums of y and y^2 (a layer input; a weight as one row).  ``q`` has
    y's shape (read in y's memory order; copied when its strides differ).  ``bias`` (float32 [C]) is added to y first, as
    the single fp32 add of a quantization launch with a convolution bias: ``bias_period`` H*W for an NCHW ``y``, -C for a
    channels-last one.  Deterministic (the bits depend neither on the run nor on ``max_ctas``), no host synchronisation.
    Recorded in the launch profile under mode 'N' (one read of y and q: 8 B/element, 4 without q)."""
    y, rows, row_len = _samples(y, "sample_noise")
    if q is not None:
        _require_cuda_f32(q, "q")
        if q.shape != y.shape:
            raise ValueError("sample_noise: q has shape %s, y %s" % (tuple(q.shape), tuple(y.shape)))
        if q.stride() != y.stride():
            q = torch.empty_like(y).copy_(q)   # y's dense memory order
    if bias is not None:
        _require_cuda_f32(bias, "bias")
        bias = bias.contiguous()
        c, period = bias.numel(), int(bias_period)
        if not ((period > 0 and c * period == row_len) or (period < 0 and c == -period and row_len % c == 0)):
            raise ValueError("sample_noise: a bias of %d values on rows of %d elements needs bias_period %d (NCHW) or "
                             "%d (channels-last), got %d" % (c, row_len, row_len // max(c, 1), -c, period))
    shape = (rows, len(NOISE_SUMS) if q is not None else 2)
    return _sample_sums("fqb200_sample_noise", y, rows, row_len, shape, "N", 8 if q is not None else 4,
                        (y.data_ptr(), _ptr(q), _ptr(bias), int(bias_period)), (int(max_ctas),))


CLIP_ERROR_CANDIDATES = ("lowp", "gaus", "laplace")


def clip_error(x, table, layout, channels_last, num_bits, positive, bit_alloc=False, solve_f64=None, want_params=False,
               max_ctas=0):
    """C ABI fqb200_clip_error: per group of ``layout`` = (outer, groups, inner), the float64 sums behind the mse_* / cos_*
    statistics of the three candidates ``CLIP_ERROR_CANDIDATES`` of `-c mix`, as a [groups, 10] device tensor: column 0
    sum x^2, 1 + k sum (x - q_k)^2, 4 + k sum x * q_k, 7 + k sum q_k^2.  ``table`` is the [groups, 12] table of a
    ``fused(..., stats_only=True)`` launch on the same tensor and layout (with ``bit_alloc``, one configured with the same
    bit allocation: its column 7 holds the widths); the candidates' parameters are solved from it on the device, in float64
    when ``solve_f64`` (default: a single group) else fp32.  ``channels_last``: per-channel groups of an ``cl_eligible``
    tensor, read in place; other per-channel tensors are read as NCHW (copied when not contiguous).  Deterministic, no
    host synchronisation; with ``want_params`` also returns the [groups, 3, 6] candidate parameters (delta, offset, bits,
    scale, zero point, qmax).  Recorded in the launch profile under mode 'E' (one read of the tensor)."""
    x, table, _, (outer, groups, inner), solve_f64, out, params = _clip_io(
        "clip_error", x, table, layout, channels_last, solve_f64, want_params, 3, sums=3)
    if x.numel():
        lib = L.load()
        ws = _own_workspace(x.device, lib.fqb200_clip_error_workspace_bytes(outer, groups, inner, int(bool(channels_last))))
        _launch(x.device, _Timed("E", x.numel(), 4, "%dx%dx%d" % (outer, groups, inner)), lib.fqb200_clip_error,
                x.data_ptr(), outer, groups, inner, int(bool(channels_last)), table.data_ptr(), int(num_bits),
                int(bool(positive)), int(bool(bit_alloc)), int(bool(solve_f64)), out.data_ptr(), _ptr(params),
                ws.data_ptr(), ws.numel(), int(max_ctas))
    return (out, params) if want_params else out


def _clip_io(name, x, table, layout, channels_last, solve_f64, want_params, candidates, multipliers=None, bad_prior=None,
             sums=1):
    """The checks and outputs of clip_error, clip_mse and clip_mse_grid: (x in the memory order the launch reads, table,
    float32 device ``multipliers`` or None, layout, ``solve_f64`` (default: one group), float64 [groups, 1 + n * ``sums``]
    output, zero for an empty x, and [groups, n, 6] parameters or None), n = ``candidates`` (per multiplier when given).
    ``bad_prior``, when not false, is the ValueError of an unusable prior."""
    _require_cuda_f32(x, "tensor")
    outer, groups, inner = (int(v) for v in layout)
    if outer * groups * inner != x.numel():
        raise ValueError("layout %r does not cover %d elements" % (layout, x.numel()))
    if bad_prior:
        raise ValueError(bad_prior)
    if channels_last:
        if not cl_eligible(x, layout):
            raise ValueError("channels_last=True needs a channels-last activation that cl_eligible takes, with layout (N, C, H*W)")
    elif not (outer == 1 and groups == 1 and dense(x)):
        x = x.contiguous()   # one group: any dense memory order; per channel: NCHW order
    if (not isinstance(table, torch.Tensor) or table.dtype != torch.float32 or table.device != x.device
            or tuple(table.shape) != (groups, L.STATS_STRIDE)):
        raise ValueError("table must be the float32 [%d, %d] statistics table on the tensor's device" % (groups, L.STATS_STRIDE))
    mult = None
    if multipliers is not None:
        mult = torch.as_tensor(multipliers, dtype=torch.float32).reshape(-1).to(x.device).contiguous()
        if not 1 <= mult.numel() <= 256:
            raise ValueError("%s takes 1..256 multipliers, got %d" % (name, mult.numel()))
        candidates *= mult.numel()
    out = torch.empty((groups, 1 + candidates * sums), dtype=torch.float64, device=x.device)
    if x.numel() == 0:
        out.zero_()
    params = torch.empty((groups, candidates, 6), dtype=torch.float32, device=x.device) if want_params else None
    return x, table.contiguous(), mult, (outer, groups, inner), groups == 1 if solve_f64 is None else solve_f64, out, params


CLIP_MSE_PRIORS = {"laplace": 0, "gaus": 1, "minmax": 2}


def clip_mse(x, table, layout, channels_last, num_bits, positive, multipliers, prior="laplace", bit_alloc=False,
             solve_f64=None, want_params=False, max_ctas=0, widths=None):
    """C ABI fqb200_clip_mse: per group of ``layout`` = (outer, groups, inner), the clipping-MSE curve of the quantizer
    ``clip_error`` describes, over K = len(``multipliers``) (1..256) clipping values alpha_k = multipliers[k] * b
    (``prior`` "laplace") or * std ("gaus"), as a [groups, K + 1] float64 device tensor: column 0 sum x^2, column 1 + k
    sum (x - q_k)^2.  ``table``, ``channels_last``, ``bit_alloc`` and ``solve_f64`` as in ``clip_error``; a multiplier equal
    to the ACIQ Laplace factor of the width gives its Laplace candidate.  ``multipliers``: a sequence of floats or a
    float32 tensor (rounded to float32).  ``widths`` (fqb200_clip_mse_widths): K ints in 0..8, candidate k's bit width
    instead of ``num_bits`` (not with ``bit_alloc``); only then ``prior`` may also be "minmax", the table's min/max range
    (0 as the lower bound when ``positive``), which ignores the multipliers.  Deterministic, no host synchronisation; with
    ``want_params`` also returns the [groups, K, 6] candidate parameters (delta, offset, bits, scale, zero point, qmax).
    Recorded in the launch profile under mode 'R' (one read of the tensor)."""
    bad_prior = prior not in CLIP_MSE_PRIORS or (prior == "minmax" and widths is None)
    x, table, mult, (outer, groups, inner), solve_f64, out, params = _clip_io(
        "clip_mse", x, table, layout, channels_last, solve_f64, want_params, 1, multipliers,
        bad_prior and "prior must be one of %s (minmax with widths only), got %r" % (sorted(CLIP_MSE_PRIORS), prior))
    k = mult.numel()
    if widths is not None:
        widths = np.ascontiguousarray(widths, dtype=np.int32).reshape(-1)   # host values, validated by the library
        if widths.size != k:
            raise ValueError("clip_mse: %d widths for %d multipliers" % (widths.size, k))
    if x.numel():
        lib = L.load()
        ws = _own_workspace(x.device, lib.fqb200_clip_mse_workspace_bytes(outer, groups, inner, int(bool(channels_last)), k))
        head = (x.data_ptr(), outer, groups, inner, int(bool(channels_last)), table.data_ptr(), int(num_bits),
                int(bool(positive)), int(bool(bit_alloc)), int(bool(solve_f64)), CLIP_MSE_PRIORS[prior], mult.data_ptr())
        tail = (k, out.data_ptr(), _ptr(params), ws.data_ptr(), ws.numel(), int(max_ctas))
        timed = _Timed("R", x.numel(), 4, "%dx%dx%d" % (outer, groups, inner))
        if widths is None:
            _launch(x.device, timed, lib.fqb200_clip_mse, *head, *tail)
        else:
            _launch(x.device, timed, lib.fqb200_clip_mse_widths, *head, widths.ctypes.data, *tail)
    return (out, params) if want_params else out


def clip_mse_select(x, table, layout, channels_last, num_bits, positive, multipliers, prior="laplace", bit_alloc=False,
                    solve_f64=None, max_ctas=0):
    """C ABI fqb200_clip_mse_select: ``clip_mse`` (same arguments, prior "laplace" or "gaus") together with each group's
    choice, made on the device without a host round trip - `-c mse` on the fly.  Returns (sums, choice, given, table):
    the [groups, K + 1] float64 sums of ``clip_mse``, bit for bit; the int32 [groups] column of the least error in
    statistics.best_columns' order (ties: the smaller multiplier; NaN never wins); the float32 [3, groups] delta, offset
    and bits of that candidate, bit for bit ``clip_mse``'s parameters at that column; and the float32 [groups, 12]
    parameter table (``_lib.STAT_COLUMNS``: ``table``'s statistics, then the chosen candidate's parameters and torch
    leaf).  Recorded in the launch profile under mode 'R' (one read of the tensor)."""
    x, table, mult, (outer, groups, inner), solve_f64, out, _ = _clip_io(
        "clip_mse_select", x, table, layout, channels_last, solve_f64, False, 1, multipliers,
        prior not in ("laplace", "gaus") and "clip_mse_select: prior must be 'laplace' or 'gaus', got %r" % (prior,))
    k = mult.numel()
    choice = torch.empty(groups, dtype=torch.int32, device=x.device)
    given = torch.empty((3, groups), dtype=torch.float32, device=x.device)
    chosen = torch.empty((groups, L.STATS_STRIDE), dtype=torch.float32, device=x.device)
    lib = L.load()
    ws = _own_workspace(x.device, lib.fqb200_clip_mse_workspace_bytes(outer, groups, inner, int(bool(channels_last)), k))
    _launch(x.device, _Timed("R", x.numel(), 4, "%dx%dx%d" % (outer, groups, inner)), lib.fqb200_clip_mse_select,
            x.data_ptr(), outer, groups, inner, int(bool(channels_last)), table.data_ptr(), int(num_bits), int(bool(positive)),
            int(bool(bit_alloc)), int(bool(solve_f64)), CLIP_MSE_PRIORS[prior], mult.data_ptr(), k, out.data_ptr(), None,
            choice.data_ptr(), given.data_ptr(), chosen.data_ptr(), ws.data_ptr(), ws.numel(), int(max_ctas))
    return out, choice, given, chosen


def clip_mse_grid(x, table, layout, channels_last, num_bits, positive, multipliers, widths, prior="laplace", solve_f64=None,
                  want_params=False, max_ctas=0):
    """C ABI fqb200_clip_mse_grid: ``clip_mse`` over every pair of W = len(``widths``) (1..9 distinct values in 0..8) bit
    widths and M = len(``multipliers``) (1..256) clipping values, the joint width-and-clip tables of `-c mse -bap mse`, as
    a [groups, 1 + W * M] float64 device tensor: column 0 sum x^2, column 1 + i * M + k the sum of candidate (widths[i],
    multipliers[k]) - bit for bit ``clip_mse(..., [multipliers[k]], widths=[widths[i]])``.  ``prior`` "laplace" or "gaus"
    (min/max ignores the multipliers); the other arguments as in ``clip_mse``.  With ``want_params`` also returns the
    [groups, W * M, 6] candidate parameters.  Recorded in the launch profile under mode 'R'."""
    widths = np.ascontiguousarray(widths, dtype=np.int32).reshape(-1)   # host values, validated by the library
    x, table, mult, (outer, groups, inner), solve_f64, out, params = _clip_io(
        "clip_mse_grid", x, table, layout, channels_last, solve_f64, want_params, widths.size, multipliers,
        prior not in ("laplace", "gaus") and "clip_mse_grid: prior must be 'laplace' or 'gaus', got %r" % (prior,))
    if not 1 <= widths.size <= 9:
        raise ValueError("clip_mse_grid takes 1..9 widths, got %d" % widths.size)
    if x.numel():
        lib = L.load()
        m = mult.numel()
        ws = _own_workspace(x.device, lib.fqb200_clip_mse_grid_workspace_bytes(outer, groups, inner, int(bool(channels_last)),
                                                                               m, widths.size))
        _launch(x.device, _Timed("R", x.numel(), 4, "%dx%dx%d" % (outer, groups, inner)), lib.fqb200_clip_mse_grid,
                x.data_ptr(), outer, groups, inner, int(bool(channels_last)), table.data_ptr(), int(num_bits),
                int(bool(positive)), 0, int(bool(solve_f64)), CLIP_MSE_PRIORS[prior], mult.data_ptr(), m,
                widths.ctypes.data, widths.size, out.data_ptr(), _ptr(params), ws.data_ptr(), ws.numel(), int(max_ctas))
    return (out, params) if want_params else out


def quantize_weights_given(w, delta, offset, num_bits, bits=None, bias_corr=False, var_corr=False, hist=None):
    """C ABI fqb200_quantize_weights_given: per-output-channel quantization of a weight ([O, ...], read in NCHW order,
    copied when not contiguous) with given float32 [O] device ``delta`` / ``offset`` / ``bits`` (None: ``num_bits``) and the
    `-vcw` / `-bcw` corrections of the RANGE_MINMAX weight launch, in one launch.  ``hist``: 256 int64 counters of the
    integer grid (`-me`), accumulated.  Returns the contiguous result.  Recorded in the launch profile under mode 'W'."""
    _require_cuda_f32(w, "weight")
    lib = L.load()
    w = w.contiguous()
    dev = w.device
    groups = w.shape[0]
    inner = w.numel() // groups if groups else 0
    vecs = []
    for name, v in (("delta", delta), ("offset", offset), ("bits", bits)):
        if v is not None:
            _require_cuda_f32(v, name)
            v = v.contiguous()
            if v.numel() != groups:
                raise ValueError("%s must have %d elements" % (name, groups))
        vecs.append(v)
    if hist is not None and (hist.dtype != torch.int64 or not hist.is_cuda or not hist.is_contiguous() or hist.numel() != 256):
        raise ValueError("hist must be a contiguous CUDA int64 tensor of 256 counters")
    out = torch.empty_like(w)
    if w.numel() == 0:
        return out
    with torch.cuda.device(dev):
        need = lib.fqb200_quantize_weights_given_workspace_bytes(groups, inner, int(num_bits), int(bits is not None),
                                                                 int(bool(bias_corr)), int(bool(var_corr)))
        if need == 0:
            L.check(L.ERR_INVALID)
        ws = _workspace(dev, _stream_handle(dev), need)
    _launch(dev, _Timed("W", w.numel(), 16 if var_corr else 12, "%dx%d" % (groups, inner)),
            lib.fqb200_quantize_weights_given, w.data_ptr(), out.data_ptr(), groups, inner, vecs[0].data_ptr(),
            vecs[1].data_ptr(), _ptr(vecs[2]), int(num_bits), int(bool(bias_corr)), int(bool(var_corr)), _ptr(hist),
            ws.data_ptr(), ws.numel())
    return out


def allocate_widths(sse, target, status=None):
    """C ABI fqb200_allocate_widths: float32 [G] device widths in 0..8 that minimise the sum of the float64 [G, 9] device
    table ``sse`` for the budget of ``target`` bits per channel - bit_alloc.allocate's result, bit for bit, without a host
    round trip.  ``status``: an int32 device tensor set to 1 when ``sse`` holds a non-finite value (never cleared)."""
    if not (isinstance(sse, torch.Tensor) and sse.is_cuda and sse.dtype == torch.float64 and sse.dim() == 2
            and sse.shape[1] == 9):
        raise ValueError("allocate_widths needs a float64 [G, 9] CUDA table")
    if status is not None and (status.dtype != torch.int32 or status.device != sse.device):
        raise ValueError("status must be an int32 tensor on the table's device")
    lib = L.load()
    sse = sse.contiguous()
    groups = sse.shape[0]
    ws = _own_workspace(sse.device, lib.fqb200_allocate_widths_workspace_bytes(groups, float(target)))
    out = torch.empty(groups, dtype=torch.float32, device=sse.device)
    _launch(sse.device, _Timed("L", groups, 72), lib.fqb200_allocate_widths, sse.data_ptr(), groups, float(target),
            out.data_ptr(), _ptr(status), ws.data_ptr(), ws.numel())
    return out


def allocate_select(sums, params, stats, target, multipliers=None, status=None):
    """C ABI fqb200_allocate_select: measured bit allocation from one call site's error sums to its apply parameters on the
    device, without a host round trip (`-baa -bap mse` on the fly).  ``sums`` / ``params``: the float64 [G, 1 + 9 M] sums
    and [G, 9 M, 6] parameters of ``clip_mse(..., widths=range(9), want_params=True)`` (M = 1) or of ``clip_mse_grid`` over
    widths 0..8 and the M ``multipliers`` (float32 device tensor, required when M > 1); ``stats``: the float32 [G, 12]
    table the candidates were solved from.  Per channel and width the least column in statistics.best_columns' order, then
    ``allocate_widths`` over those sums for ``target`` bits per channel.  Returns (widths, choice, given, table): float32 [G]
    widths; int32 [G] column of the chosen width (None when M = 1); float32 [3, G] delta, offset and bits, bit for bit
    ``params`` at the chosen (width, column); the float32 [G, 12] parameter table of ``clip_mse_select``.  ``status``: an
    int32 device tensor set to 1 on a non-finite per-width sum.  Recorded in the launch profile under mode 'L'."""
    if not (isinstance(sums, torch.Tensor) and sums.is_cuda and sums.dtype == torch.float64 and sums.dim() == 2
            and sums.shape[1] > 1 and (sums.shape[1] - 1) % 9 == 0):
        raise ValueError("allocate_select needs float64 [G, 1 + 9 M] CUDA sums")
    groups, m = sums.shape[0], (sums.shape[1] - 1) // 9
    dev = sums.device
    if not (isinstance(params, torch.Tensor) and params.dtype == torch.float32 and params.device == dev
            and tuple(params.shape) == (groups, 9 * m, 6)):
        raise ValueError("params must be the float32 [%d, %d, 6] candidate parameters on the sums' device" % (groups, 9 * m))
    if not (isinstance(stats, torch.Tensor) and stats.dtype == torch.float32 and stats.device == dev
            and tuple(stats.shape) == (groups, L.STATS_STRIDE)):
        raise ValueError("stats must be the float32 [%d, %d] statistics table on the sums' device" % (groups, L.STATS_STRIDE))
    mult = None
    if m > 1:
        if not (isinstance(multipliers, torch.Tensor) and multipliers.dtype == torch.float32 and multipliers.device == dev
                and multipliers.numel() == m):
            raise ValueError("allocate_select: %d columns per width need the %d float32 multipliers on the sums' device"
                             % (m, m))
        mult = multipliers.contiguous()
    if status is not None and (status.dtype != torch.int32 or status.device != dev):
        raise ValueError("status must be an int32 tensor on the sums' device")
    lib = L.load()
    sums, params, stats = sums.contiguous(), params.contiguous(), stats.contiguous()
    ws = _own_workspace(dev, lib.fqb200_allocate_select_workspace_bytes(groups, float(target)))
    widths = torch.empty(groups, dtype=torch.float32, device=dev)
    choice = torch.empty(groups, dtype=torch.int32, device=dev) if m > 1 else None
    given = torch.empty((3, groups), dtype=torch.float32, device=dev)
    table = torch.empty((groups, L.STATS_STRIDE), dtype=torch.float32, device=dev)
    _launch(dev, _Timed("L", groups, 72 * m), lib.fqb200_allocate_select, sums.data_ptr(), params.data_ptr(), _ptr(mult),
            m, stats.data_ptr(), groups, float(target), widths.data_ptr(), _ptr(choice), given.data_ptr(), table.data_ptr(),
            _ptr(status), ws.data_ptr(), ws.numel())
    return widths, choice, given, table


KMeans1d =collections.namedtuple("KMeans1d", "labels centres inertia n_iter init_ids out out_bcorr")
KMEANS_TASKS = {None: 0, "quantize": 1, "clip": 2}


def kmeans_trials(k):
    """scikit-learn's number of k-means++ local trials: 2 + int(log k)."""
    return 2 + int(np.log(k))


def kmeans_draws(n, k, seed):
    """The random draws of scikit-learn's k-means++ (_kmeans_plusplus) on ``np.random.RandomState(seed)``, in its order: the
    first centre ``choice(n, p=w / w.sum())`` with float32 unit weights, then ``uniform(size=n_local_trials)`` for every
    further centre.  They do not depend on the data.  Returns (first index, float64 [k - 1, n_local_trials])."""
    rs = np.random.RandomState(seed)
    w = np.ones(n, dtype=np.float32)
    first = int(rs.choice(n, p=w / w.sum()))
    del w
    t = kmeans_trials(k)
    u = np.stack([rs.uniform(size=t) for _ in range(k - 1)]) if k > 1 else np.zeros((0, t))
    return first, u


def kmeans1d(x, num_bits, seed=0, task=None, init=None, rows=None, max_ctas=0):
    """C ABI fqb200_kmeans1d: scikit-learn's ``KMeans(n_clusters=2**num_bits, random_state=seed).fit`` on the values of the
    dense tensor ``x`` in memory order (kmeans_quantization.py:14-30), in one launch.  ``task`` 'quantize' also returns
    ``out`` = each value replaced by its centre, 'clip' returns ``x`` clipped to [min, max] of the centres; ``rows`` (with a
    task) adds ``out_bcorr``, the per-output-channel bias correction of kmeans_quantization.py:86-88 over ``rows`` rows
    (float64 row means, rounded to fp32 once).  ``init``: initial centres (k values in the data's units, scikit-learn's
    ``init=``) instead of k-means++.  Returns a ``KMeans1d`` of device tensors: labels (uint8, x's shape), centres (float32
    [k], centre + mean like ``cluster_centers_``), inertia (float64 scalar), n_iter (int32 scalar), init_ids (int64 [k], the
    k-means++ sample indices; -1 with ``init``), out and out_bcorr (x's shape and strides, or None).  Non-finite input raises
    ValueError, as scikit-learn does (one host synchronisation for that check); otherwise the launch does not synchronise.
    Deterministic: the bits depend neither on the run nor on ``max_ctas``.  Recorded in the launch profile under mode
    'C'."""
    _require_cuda_f32(x, "tensor")
    if task not in KMEANS_TASKS:
        raise ValueError("task must be None, 'quantize' or 'clip'")
    num_bits = int(num_bits)
    if not 1 <= num_bits <= 8:
        raise ValueError("num_bits must be in 1..8")
    k = 1 << num_bits
    if not dense(x):
        x = x.contiguous()
    n = x.numel()
    if n < k:
        raise ValueError("n_samples=%d should be >= n_clusters=%d." % (n, k))
    if not bool(torch.isfinite(x).all()):
        raise ValueError("Input contains NaN or infinity.")
    rows = int(rows or 0)
    if rows and (task is None or n % rows):
        raise ValueError("rows needs a task and must divide the number of elements")
    lib = L.load()
    dev = x.device
    labels = torch.empty_like(x, dtype=torch.uint8)
    centres = torch.empty(k, dtype=torch.float32, device=dev)
    inertia = torch.empty((), dtype=torch.float64, device=dev)
    n_iter = torch.empty((), dtype=torch.int32, device=dev)
    init_ids = torch.empty(k, dtype=torch.int64, device=dev)
    out = torch.empty_like(x) if task else None
    out_bcorr = torch.empty_like(x) if rows else None
    first, draws, init_t = 0, None, None
    if init is None:
        first, u = kmeans_draws(n, k, seed)
        draws = torch.from_numpy(np.ascontiguousarray(u, dtype=np.float64)).to(dev)
    else:
        init_t = torch.as_tensor(init, dtype=torch.float64).reshape(-1).to(dev).contiguous()
        if init_t.numel() != k:
            raise ValueError("init must hold %d centres" % k)
    ws = _own_workspace(dev, lib.fqb200_kmeans1d_workspace_bytes(n, k))
    _launch(dev, _Timed("C", n, 4, "%d k=%d" % (n, k)), lib.fqb200_kmeans1d, x.data_ptr(), n, num_bits, first, _ptr(draws),
            kmeans_trials(k), _ptr(init_t), KMEANS_TASKS[task], rows, labels.data_ptr(), centres.data_ptr(),
            inertia.data_ptr(), n_iter.data_ptr(), init_ids.data_ptr(), _ptr(out), _ptr(out_bcorr), ws.data_ptr(),
            ws.numel(), int(max_ctas))
    return KMeans1d(labels, centres, inertia, n_iter, init_ids, out, out_bcorr)


def add_relu_(a, b):
    """``a += b; relu_(a)`` in one pass (C ABI fqb200_add_relu, 12 instead of 20 bytes per element).  Both tensors must be
    dense with identical strides (any memory format); returns ``a``.  Bit-identical to the two torch ops."""
    _require_cuda_f32(a, "a")
    _require_cuda_f32(b, "b")
    if a.shape != b.shape or a.stride() != b.stride() or not dense(a):
        raise ValueError("add_relu_ needs two dense tensors of identical shape and strides")
    _launch(a.device, _Timed("E", a.numel(), 12), L.load().fqb200_add_relu, a.data_ptr(), b.data_ptr(), a.data_ptr(), a.numel())
    return a


def maxpool2d_cl(x, kernel_size, stride, padding, out=None):
    """``F.max_pool2d(x, kernel_size, stride, padding)`` for a channels-last fp32 activation with C % 4 == 0 (C ABI
    fqb200_maxpool2d_nhwc_into); the result is channels-last as well.  Bit-identical to torch.  ``out``: where to write it,
    directly when it is a channel slice of a wider channels-last tensor (profile mode "Pi"), else through a copy."""
    _require_cuda_f32(x, "input")
    if x.dim() != 4 or not x.is_contiguous(memory_format=torch.channels_last) or x.shape[1] % 4 != 0:
        raise ValueError("maxpool2d_cl needs a channels-last [N, C, H, W] tensor with C % 4 == 0")
    kh, kw = (kernel_size, kernel_size) if isinstance(kernel_size, int) else kernel_size
    sh, sw = (stride, stride) if isinstance(stride, int) else stride
    ph, pw = (padding, padding) if isinstance(padding, int) else padding
    n, c, h, w = x.shape
    oh, ow = (h + 2 * ph - kh) // sh + 1, (w + 2 * pw - kw) // sw + 1
    user = out
    if user is not None:
        _require_cuda_f32(user, "out")
        if tuple(user.shape) != (n, c, oh, ow):
            raise ValueError("out must have the pooled shape %r, got %r" % ((n, c, oh, ow), tuple(user.shape)))
    pitch = slice_pitch(user) if user is not None else 0
    direct = pitch >= c and pitch % 4 == 0 and user.data_ptr() % 16 == 0 and not _overlaps(x, user, pitch)
    kout = user if direct else torch.empty((n, c, oh, ow), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
    _launch(x.device, _Timed("Pi" if direct and pitch != c else "P", kout.numel(), 4 + 4 * sh * sw),
            L.load().fqb200_maxpool2d_nhwc_into, x.data_ptr(), kout.data_ptr(), n, h, w, c, kh, kw, sh, sw, ph, pw,
            pitch if direct else c)
    return _finish_out(kout, None if direct else user)


def _test_division(a, b):
    """(fast, ieee) quotients from the device: the 3-instruction exact division next to __fdiv_rn."""
    lib = L.load()
    fast, ieee = torch.empty_like(a), torch.empty_like(a)
    with torch.cuda.device(a.device):
        L.check(lib.fqb200_selftest_division(a.data_ptr(), b.data_ptr(), fast.data_ptr(), ieee.data_ptr(), a.numel(),
                                         _stream_handle(a.device)))
    return fast, ieee
