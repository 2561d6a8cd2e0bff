/*
 * fqb200 - H100-native (sm_90a) fake-quantization library: C ABI.
 *
 * Drop-in boundary for the fake-quantization hot path of submission2019/cnn-quantization
 * (SURVEY.md section 8).  Plain C: device pointers, sizes, a stream handle; no torch types.
 * Every entry point returns 0 (FQB200_OK) or an FQB200_ERR_* code; nothing throws.  The only process
 * state is the per-device set-up (kernel attributes, occupancy, constant tables), done once under
 * std::call_once - entry points may be called concurrently from several host threads (one device each,
 * like torch.nn.DataParallel's workers), and the last-error text is per thread.  All tensors are fp32, contiguous,
 * resident on the current CUDA device.  `stream` is a cudaStream_t passed as void*.
 *
 * Reference interfaces replaced (paths relative to the reference repository):
 *   fqb200_float2gemmlowp   <- kernels/int_quantization.cpp:6-12 + kernels/gemmlowp.cu:8-45
 *                              (`int_quantization.float2gemmlowp`, the only compiled symbol)
 *   fqb200_quantize1        <- pytorch_quantizer/quantization/qtypes/int_quantizer.py:557-603
 *                              (`IntQuantizer.__gemmlowpQuantize1__`, parameters given)
 *   fqb200_fused            <- int_quantizer.py:327-359 (gemmlowpClippingQuantize), :409-451
 *                              (gemmlowpQuantizeActivationPerChannel), :453-476
 *                              (gemmlowpQuantizeWeightsPerChannel), :361-379 + :605-614
 *                              (gemmlowpMinMaxQuantize -> __gemmlowpQuantize__), :147-225 (mid-tread),
 *                              with :507-555 (statistics), :227-325 (ACIQ alpha), :381-407 (bit
 *                              allocation) and inference_quantization_manager.py:374-391 (weight
 *                              bias / variance correction) fused into ONE kernel launch.
 */
#ifndef FQB200_H_
#define FQB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FQB200_ABI_VERSION 3

/* ---- return codes ------------------------------------------------------------------------- */
#define FQB200_OK 0
#define FQB200_ERR_INVALID 1     /* bad argument (null pointer, non-positive size, bad enum) */
#define FQB200_ERR_WORKSPACE 2   /* workspace missing or smaller than fqb200_workspace_bytes() */
#define FQB200_ERR_CUDA 3        /* CUDA runtime error; text via fqb200_last_error() */
#define FQB200_ERR_UNSUPPORTED 4 /* valid request this build does not implement */

/* ---- enums (plain ints in the struct) ------------------------------------------------------- */
/* how statistics map to quantization parameters */
#define FQB200_SCOPE_GROUP 0      /* one parameter set per group (per channel / per output row) */
#define FQB200_SCOPE_GROUP_MEAN 1 /* statistics per group, averaged over groups -> ONE parameter set
                                     (the reference's avg_over_batch min/max, int_quantizer.py:372,:525-526) */
#define FQB200_SCOPE_TENSOR 2     /* min of the group minima / max of the group maxima -> ONE parameter set, while
                                     `groups` keeps its meaning for the per-row weight correction (per-tensor
                                     weight quantization + -bcw, inference_quantization_manager.py:374-391) */
/* where (delta, offset) come from */
#define FQB200_RANGE_MINMAX 0  /* delta = max - min, offset = min (0 if positive) */
#define FQB200_RANGE_LAPLACE 1 /* ACIQ Laplace: alpha = F[bits] * b          (int_quantizer.py:227-253) */
#define FQB200_RANGE_GAUS 2    /* ACIQ Gauss:   alpha = F[bits] * std        (:255-264) */
#define FQB200_RANGE_KSTD 3    /* alpha = clip_k * std ('2std')              (:266-275) */
#define FQB200_RANGE_GIVEN 4   /* no statistics: per-group delta / offset (/ bits) from the caller (`-sm use`, the a3 leaf of
                                  fqb200_quantize1) - through this descriptor so that the launch can also take bias,
                                  residual (+ residual_stats) and pool; channels_last, torch leaf, scope GROUP only */
/* which leaf arithmetic */
#define FQB200_LEAF_TORCH 0    /* __gemmlowpQuantize1__: round-half-even, scale floor 1e-8, true zero */
#define FQB200_LEAF_COMPILED 1 /* float2gemmlowp: roundf (half away), no floor, preserve_zero rule */
#define FQB200_LEAF_MIDTREAD 2 /* mid_tread_quantization (bin allocation), int_quantizer.py:185-225 */
/* bit-allocation prior */
#define FQB200_PRIOR_STD 0
#define FQB200_PRIOR_B 1

/* number of floats written per group into fqb200_desc.out_stats */
#define FQB200_STATS_STRIDE 12
/* out_stats[g*12 + k]: 0 min, 1 max, 2 mean, 3 b, 4 std, 5 delta, 6 offset, 7 bits, 8 scale, 9 zero_point,
 * 10 qmax, 11 flags (bit0: passthrough, bit1: true-zero form) */

/*
 * One hooked tensor = one descriptor = one kernel launch.
 * The tensor is viewed as [outer][groups][inner], contiguous fp32:
 *   per-channel activation [N,C,H,W]      outer=N  groups=C    inner=H*W
 *   per-output-channel weight [O,I,k,k]   outer=1  groups=O    inner=I*k*k
 *   per-tensor                            outer=1  groups=1    inner=numel
 *   per-sample averaged min/max           outer=1  groups=N    inner=C*H*W, scope=GROUP_MEAN
 *   per-channel activation stored NHWC    outer=N  groups=C    inner=H*W, channels_last=1 (memory [N][H*W][C])
 */
typedef struct fqb200_desc {
  int64_t outer, groups, inner;
  int32_t scope;      /* FQB200_SCOPE_* */
  int32_t range_mode; /* FQB200_RANGE_* */
  int32_t leaf;       /* FQB200_LEAF_* */
  int32_t num_bits;   /* 1..8 (ignored by the mid-tread leaf) */
  int32_t positive;   /* force_positive or half_range: range starts at 0, one-sided ACIQ tables */
  int32_t solve_f64;  /* parameter arithmetic in float64, rounded to fp32 at the end: the reference's
                         per-tensor clipping branch (int_quantizer.py:354-357) */
  float clip_k;       /* FQB200_RANGE_KSTD multiplier */
  /* per-group bit allocation (int_quantizer.py:381-407); only honoured when num_bits <= 4, like the reference */
  int32_t bit_alloc;
  int32_t bit_alloc_prior; /* FQB200_PRIOR_* */
  int32_t bit_alloc_round; /* 1: round, 0: ceil */
  float bit_alloc_target;  /* mean bits per group to hit (the reference defaults it to num_bits) */
  /* mid-tread leaf */
  float mt_target; /* log2 of the mean number of bins per group */
  int32_t mt_clip; /* 1: Laplace clipping around the mean (activations), 0: min/max range (weights) */
  /* weight post-processing (inference_quantization_manager.py:374-391) */
  int32_t bias_corr; /* w_q <- w_q - mean(w_q) + mean(w) per group */
  int32_t var_corr;  /* w_q <- (w_q - mean(w_q)) * std(w)/(std(w_q)+1e-8) + mean(w_q), before bias_corr */
  int32_t stats_only; /* 1: compute statistics/parameters into out_stats, do not touch `out` */
  float* out_stats;   /* optional device buffer, groups * FQB200_STATS_STRIDE floats (rows beyond the first are
                         left untouched when the parameters are per tensor) */
  const float* bias;  /* optional device vector of `groups` floats added to every element of its group before
                         anything else (x + bias[g], one fp32 rounding): the folded-BN convolution bias, so the
                         caller can run its convolution bias-free and skip a full read+write pass over the
                         activation.  NULL = none. */
  int64_t bias_period; /* 0: bias[g] (groups are channels).  > 0: the row of a group holds inner / bias_period channels
                          of bias_period floats each and element i of the row gets bias[i / bias_period] - the
                          per-tensor and per-sample layouts of an NCHW activation (bias_period = H*W).  Needs
                          bias_period % 4 == 0 on the 128-bit path.  < 0: element i of the row gets bias[i % -bias_period] -
                          the same layouts of a CHANNELS-LAST activation (bias_period = -C; C % 4 == 0, C <= 2048). */
  int32_t channels_last; /* 1: the tensor is [outer][inner][groups] in memory (groups fastest), i.e. an NCHW-shaped
                          activation stored channels-last (NHWC).  Per-channel scope with the torch / mid-tread leaves;
                          needs groups % 4 == 0 and groups <= 2048.  Sums of different CTAs meet in float64 atomics:
                          statistics are reproducible to fp32 rounding, not bit for bit.  The standard deviation comes
                          from the first pass (shifted sums; SURVEY.md 8d "single-pass" option). */
  unsigned long long* out_hist; /* optional device array of hist_bins counters: the launch ADDS the histogram of the integer
                          grid q to it (bin = clamp(q + hist_offset, 0, hist_bins - 1)) - what the reference's `-me`
                          entropy measurement needs (utils/entropy.py:6-17; int_quantizer.py:586-587, :216-221) without
                          torch.unique over the tensor.  Torch leaf: q in [0, 255], hist_bins 256, hist_offset 0.
                          Mid-tread leaf (channels_last only): q is clamped to per-channel, generally fractional bounds;
                          elements ON a bound are counted in out_hist_clamped instead. */
  int32_t hist_bins;   /* 0 = 256; at most 8192 (channels_last), 256 otherwise */
  int32_t hist_offset; /* added to q before binning (mid-tread grids are signed) */
  unsigned long long* out_hist_clamped; /* mid-tread: optional [groups][2] counters, elements on c_min / c_max of the group */
  int32_t relu_passthrough; /* 1: the caller has fused the ReLU that follows this quantizer away (a positive range starts at
                          zero with zero point 0, so the quantized tensor is >= 0 already).  The one case where that is
                          not true - the compiled leaf handing its input back because the range is empty (range <= 0,
                          gemmlowp.cu:31-32) - then returns max(x, 0) instead of x, so quantizer + ReLU stay exact. */
  const float* residual; /* channels_last launches and the per-sample / per-tensor min-max launches on the compiled leaf
                          (outer = 1, rows = samples); NULL = none: a tensor of the same shape and memory order that is ADDED to the
                          quantized values in the apply phase, out = quantize(x + bias) + residual, and with residual_relu
                          followed by max(., 0): the `out += identity; out = relu(out)` that closes a ResNet block
                          (torchvision resnet.py), fused into the launch that quantizes the block's last convolution
                          (8 B/element less traffic than a separate add + ReLU pass).  Must not alias `out`. */
  int32_t residual_relu;
  const float* residual_stats; /* NULL: the residual is added as it is.  Else the [groups][FQB200_STATS_STRIDE] table
                          (channels_last) or the one row (per-sample / per-tensor min-max) that a stats_only launch with the
                          same leaf exported for the residual tensor: the residual is QUANTIZED with those parameters on the
                          fly (columns scale, zero_point, qmax, flags) before the add - the shortcut branch of a
                          down-sampling ResNet block never makes a round trip through memory as a quantized tensor
                          (stats_only 8 B/element + 4 B/element here instead of 16 + 4) */
  const float* residual_bias; /* optional bias of the residual tensor, added before its quantization; same form as `bias`
                          (per channel; channel-fastest on the min-max launches) */
  int32_t pool;           /* 0 = none; 2 = a 2x2 / stride-2 max pooling (floor mode, no padding), 3 = a 3x3 / stride-2 / padding-1
                          max pooling (H and W even: the ResNet stem) follows this quantizer and is its only consumer: channels_last launches compute it INSIDE the apply phase (the leaf is monotone:
                          quantize(max) == max(quantize), bit for bit) and write only the pooled tensor - `out` is not
                          touched; statistics are those of the full tensor.  Saves the write of the quantized tensor and
                          the pooling kernel's read: 8 of 21 B/element (VGG-16: every convolution in front of a pooling) */
  int64_t pool_h, pool_w; /* the H and W behind `inner` = H * W (W even; pool = 3: H even too) */
  float* pool_out;        /* [outer][H/2][W/2][groups], 16-byte aligned */
  const float* given_delta;  /* FQB200_RANGE_GIVEN: [groups] device vectors (delta, offset as in fqb200_quantize1) ... */
  const float* given_offset;
  const float* given_bits;   /* ... and optional per-group bit widths (NULL: num_bits) */
  unsigned long long* debug_stamps; /* diagnostics, NULL = off: device array of 16 counters that receives %globaltimer
                          (ns) at the phase boundaries of this launch (slot 0: start, 1 / 5: statistics phases combined,
                          4 / 8: past the grid barriers, 7: parameters ready, 9: apply done; tools/phasebench.py) */
} fqb200_desc;

/* ---- library ---------------------------------------------------------------------------------- */
int fqb200_abi_version(void);
/* text of the last error on the calling thread ("" if none) */
const char* fqb200_last_error(void);
/* number of CTAs the fused kernel keeps resident on the current device (132 SMs x 2 on an H100) */
int fqb200_resident_ctas(void);

/* What a launch of `d` would look like on the current device (introspection for tools and tests), 8 values:
 * channels_last, and the per-sample / per-tensor min-max layouts ({3, ...}) on the bulk-copy engine:
 *                {2, grid, units, stages per unit, vectors per stage, consumer stride, ring stages, phases};
 * otherwise:     {access mode 4|1|8, grid, units, parts per group, vectors per part, stride, ring depth, leader lanes}. */
int fqb200_plan_info(const fqb200_desc* d, int64_t* out8);
/* Self-test hook: fast[i] = the kernels' 3-instruction exact division a[i] / b[i], ieee[i] = IEEE a[i] / b[i]
 * (tests/test_gpu_parity.py::test_division_is_ieee).  Device pointers. */
int fqb200_selftest_division(const float* a, const float* b, float* fast, float* ieee, int64_t n, void* stream);

/* Scratch the fused kernel needs for `d` (partials, per-group results, grid-barrier words). */
size_t fqb200_workspace_bytes(const fqb200_desc* d);
/* Zero the barrier words once after allocating a workspace (kernels leave them zeroed). */
int fqb200_workspace_init(void* workspace, size_t bytes, void* stream);

/*
 * a1 - `int_quantization.float2gemmlowp(in, range, offset, num_bits, int_exp, enforce_true_zero, noise)`.
 * range <= 0 copies `in` to `out` (the reference returns its input).  `noise` may be NULL (= zeros).
 * `out` may alias `in`.
 */
int fqb200_float2gemmlowp(const float* in, float* out, int64_t n, float range, float offset, int num_bits,
                          int int_exp, int enforce_true_zero, const float* noise, void* stream);

/*
 * a3 - `IntQuantizer.__gemmlowpQuantize1__(tensor, delta, offset, bit_alloc)`, parameters on the device:
 * `delta`/`offset` hold `groups` floats (per_group=1) or one float (per_group=0); `bits` is NULL or
 * `groups` floats (per-row bit widths).  Tensor viewed [outer][groups][inner] (a [R,K] matrix is
 * outer=1, groups=R, inner=K).  Optional `grid` receives the integer grid q (fp32 integers).  Optional `bias`
 * (`groups` floats) is added to every element of its group first, like fqb200_desc.bias.  `out` may alias `in`.
 * channels_last = 1: the tensor is [outer][inner][groups] in memory (an NCHW-shaped activation stored NHWC; needs
 * groups % 4 == 0, groups <= 2048, 16-byte aligned pointers) - `-sm use` on channels-last models without a copy.
 */
int fqb200_quantize1(const float* in, float* out, float* grid, int64_t outer, int64_t groups, int64_t inner,
                     const float* delta, const float* offset, const float* bits, int per_group, int num_bits,
                     const float* bias, int channels_last, void* stream);

/*
 * `-bca` - a3 with the activation bias correction of Conv2dWithId.forward (inference_quantization_manager.py:180-196) in the
 * same launch: y = quantize1(x + bias); per group q_bias = (sum r - sum y) / (#(r > 0) + 1e-8), r = x + bias (rectified
 * first when relu_first, i.e. when a ReLU follows the convolution); out = y + q_bias where y > 0.  The tensor must be
 * channels-last ([outer][inner][groups] in memory, groups % 4 == 0, groups <= 2048).  Optional out_qbias receives the
 * `groups` corrections.  Workspace as for fqb200_fused (fqb200_workspace_bytes of any channels_last descriptor with the
 * same `groups`).  `out` may alias `in`.
 */
int fqb200_quantize1_bca(const float* in, float* out, int64_t outer, int64_t groups, int64_t inner, const float* delta,
                         const float* offset, const float* bits, int per_group, int num_bits, const float* bias, int relu_first,
                         float* out_qbias, void* workspace, size_t workspace_bytes, void* stream);

/*
 * Max pooling of a channels-last activation ([n][h][w][c] in memory, c % 4 == 0; dilation 1, floor mode) - the operator in
 * front of the `activation_pooling` quantization call site (MaxPool2dWithId.forward, inference_quantization_manager.py:
 * 58-74).  out is [n][oh][ow][c], oh = (h + 2 ph - kh) / sh + 1.  Bit-identical to torch.nn.functional.max_pool2d
 * (NaN in a window wins).
 */
int fqb200_maxpool2d_nhwc(const float* in, float* out, int64_t n, int64_t h, int64_t w, int64_t c, int kh, int kw, int sh, int sw,
                          int ph, int pw, void* stream);

/*
 * out[i] = max(a[i] + b[i], 0) - the residual add + ReLU between two hooked convolutions of a ResNet block (the call
 * sites' surroundings, SURVEY.md 8f rank 4: torchvision's `out += identity; out = relu(out)`), one pass instead of two
 * torch kernels; bit-identical to them.  `out` may alias `a` or `b`.
 */
int fqb200_add_relu(const float* a, const float* b, float* out, int64_t n, void* stream);

/*
 * a4/a5/a6/a11/a12(+a7-a10, a13) - statistics -> parameters -> quantize-dequantize (-> weight
 * correction) in ONE cooperative kernel launch.  `out` may alias `in`.
 */
int fqb200_fused(const fqb200_desc* d, const float* in, float* out, void* workspace, size_t workspace_bytes,
                 void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FQB200_H_ */
