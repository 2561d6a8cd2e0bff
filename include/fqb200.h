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

/* The launch fqb200_fused makes for `d` with 16-byte-aligned tensors on the current device (an H100 when there is none),
 * or the code and message with which it refuses `d` (introspection for tools and tests), 8 values:
 * channels_last, and the per-sample / per-tensor min-max layouts ({3, ...}) on the bulk-copy engine:
 *                {2, grid, units, stages per unit, vectors per stage, consumer stride, ring stages, phases}
 *                (phases: 1 for FQB200_RANGE_GIVEN, which only applies);
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
 * same `groups`, 16-byte aligned; FQB200_ERR_WORKSPACE otherwise, checked before any device call).  `out` may alias `in`.
 */
int fqb200_quantize1_bca(const float* in, float* out, int64_t outer, int64_t groups, int64_t inner, const float* delta,
                         const float* offset, const float* bits, int per_group, int num_bits, const float* bias, int relu_first,
                         float* out_qbias, void* workspace, size_t workspace_bytes, void* stream);

/*
 * Max pooling of a channels-last activation ([n][h][w][c] in memory, c % 4 == 0; dilation 1, floor mode) - the operator in
 * front of the `activation_pooling` quantization call site (MaxPool2dWithId.forward, inference_quantization_manager.py:
 * 58-74).  out is [n][oh][ow][c], oh = (h + 2 ph - kh) / sh + 1, and must not overlap in (FQB200_ERR_INVALID).
 * Bit-identical to torch.nn.functional.max_pool2d (NaN in a window wins).
 */
int fqb200_maxpool2d_nhwc(const float* in, float* out, int64_t n, int64_t h, int64_t w, int64_t c, int kh, int kw, int sh, int sw,
                          int ph, int pw, void* stream);
/*
 * fqb200_maxpool2d_nhwc writing a channel slice of a wider channels-last tensor: pixel p of the result goes to
 * out + p * out_pixel_stride (out points at the slice's first channel); the other channels of every pixel are left
 * untouched (the max-pool branch of an Inception block).  out_pixel_stride >= c and a multiple of 4, out 16-byte aligned
 * (FQB200_ERR_UNSUPPORTED otherwise); out must not overlap in (FQB200_ERR_INVALID).  fqb200_maxpool2d_nhwc is the case
 * out_pixel_stride = c, so it refuses overlapping tensors as well.
 */
int fqb200_maxpool2d_nhwc_into(const float* in, float* out, int64_t n, int64_t h, int64_t w, int64_t c, int kh, int kw,
                               int sh, int sw, int ph, int pw, int64_t out_pixel_stride, void* stream);

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
/*
 * fqb200_fused writing its result into a channel slice of a wider channels-last tensor
 * [pixels][out_pixel_stride]: pixel p of the result goes to out + p * out_pixel_stride (out points at the slice's
 * first channel); the other channels of every pixel are left untouched.  A branch of an Inception block writes its part
 * of the concatenation this way, bit for bit what fqb200_fused followed by a copy would give.
 * Two kinds of apply launch take a pitch, C being the channels of a pixel:
 *   - channels-last launches (on-the-fly statistics, RANGE_GIVEN, torch and mid-tread leaves): C = groups, pixels =
 *     outer * inner;
 *   - per-sample / per-tensor min-max launches (compiled leaf, outer = 1, groups = samples) on channels-last memory with a
 *     channel-fastest bias: C = -bias_period, element (n, pixel, c) goes to out + (n * H*W + pixel) * out_pixel_stride + c.
 *     Without such a bias the launch does not know C and takes no pitch.
 * FQB200_ERR_UNSUPPORTED: stats_only, pool, residual, out_hist or any other descriptor; out_pixel_stride < C or not
 * a multiple of 4; a misaligned in / out.  out_pixel_stride = C is the dense case, where `out` may alias `in`; with
 * any other pitch an `out` overlapping `in` returns FQB200_ERR_INVALID.  These rules are checked before any device call.
 * fqb200_fused(d, ...) is fqb200_fused_into(d, ..., 0, ...): a dense `out` for any descriptor.
 */
int fqb200_fused_into(const fqb200_desc* d, const float* in, float* out, int64_t out_pixel_stride, void* workspace,
                      size_t workspace_bytes, void* stream);

/*
 * KL-divergence calibration (`-kld` collect, statistic_manager.py:80-82 -> kld_threshold.py:15-80): for each of `rows`
 * contiguous rows of `row_len` floats (one sample; any dense memory order of it), th = max |x| and a histogram of
 * `num_bins` bins over (-th, th) with numpy 1.x's edges (float32 of the float64 linspace; th == 0 -> (-0.5, 0.5)), then
 * the threshold search over the candidates i = num_quantized_bins/2 .. num_bins/2 with the divergence in float64.
 * Writes per row the threshold out_th = edge[num_bins/2 + 1 + i], its divergence out_div, and out_idx = the candidate's
 * position in the search (i - num_quantized_bins/2; np.argmin rules: the first NaN, else the first minimum).  A row with a
 * NaN or Inf gets th = div = NaN and idx = -1.  num_bins odd, 3 .. 8001; num_quantized_bins odd, 3 .. num_bins; row_len
 * < 2^31.  Three kernel launches on `stream`, no host synchronisation.  The workspace (fqb200_kld_workspace_bytes, 16-byte
 * aligned) is private to the call: it is zeroed and filled with counters, so it must not be a fqb200_fused workspace.
 * After the call it holds the histograms: uint32 counts [rows][num_bins] from byte offset (rows * 4 rounded up to 256).
 */
int fqb200_kld_threshold(const float* in, int64_t rows, int64_t row_len, int num_bins, int num_quantized_bins, float* out_th,
                         float* out_div, int32_t* out_idx, void* workspace, size_t workspace_bytes, void* stream);
/* Workspace of fqb200_kld_threshold: rows x num_bins counters and rows words (0 and fqb200_last_error() on bad arguments). */
size_t fqb200_kld_workspace_bytes(int64_t rows, int num_bins);

/*
 * Activation norm measurement (`-ms`, distance_stats.py:22-33): out[r] = the float64 sum of x * x over row r, for `rows`
 * contiguous rows of `row_len` floats (one sample; any dense memory order of it).  Work units are (row, chunk) with a
 * chunk length that depends on row_len only; each unit's partial goes to the workspace and a row's partials are added in
 * chunk order, so the result has the same bits on every run.  NaN and Inf propagate; rows == 0 launches nothing.  One
 * read of the tensor plus, when a row spans several chunks, a small second launch, on `stream`; no host synchronisation.
 * The workspace (fqb200_sample_sumsq_workspace_bytes, 16-byte aligned; may be null when that is 0) is private to the call.
 */
int fqb200_sample_sumsq(const float* in, int64_t rows, int64_t row_len, double* out, void* workspace, size_t workspace_bytes,
                        void* stream);
/* Workspace of fqb200_sample_sumsq in bytes (0 and fqb200_last_error() on bad arguments: rows < 0, row_len <= 0). */
size_t fqb200_sample_sumsq_workspace_bytes(int64_t rows, int64_t row_len);

/*
 * Sample-angle measurement (angle_stats.py:17-44): for `rows` contiguous rows of `row_len` floats (one sample; any dense
 * memory order of it), the float64 Gram matrix G = X X^T on the FP64 tensor cores (fp32 products are exact in float64,
 * accumulation in float64) and the pairwise angles.  Outputs, row-major [rows][rows]:
 *   out_angles (float32): float(acos(c_ij)) for j > i with c_ij = G_ij / sqrt(G_ii * G_jj) in float64, clamped to
 *     [-1, 1]; 0 on and below the diagonal.  A pair whose cosine is not finite is NaN: a zero sample (0 / 0, as in the
 *     reference) and a sample holding NaN or Inf.  The clamp differs from the reference on purpose: its fp32 cosine can
 *     land a rounding step above 1 for nearly parallel samples and give NaN.  A duplicated sample gives exactly 0 and a
 *     negated one exactly float(pi).
 *   out_gram (float64, may be null): G_ij for j >= i; the entries below the diagonal are unspecified.
 * At least one of the two outputs must be given.  rows <= 8192 (FQB200_ERR_UNSUPPORTED above); rows == 0 launches nothing.
 * The reduction is cut into K slices whose count depends on (rows, row_len) only; each (64 x 64 tile pair, slice) unit
 * writes its partial to its own workspace slot and a second launch adds them in slice order, so the bits do not depend on
 * the run or on max_ctas (0: the default grid, else at most that many CTAs).  Two launches on `stream`, no host
 * synchronisation.  The workspace (fqb200_sample_angles_workspace_bytes, 16-byte aligned; at most (P + 1024) * 32 KB
 * with P = T (T + 1) / 2 tile pairs, T = ceil(rows / 64): 34 MB at rows = 512) is private to the call.
 * FQB200_ERR_INVALID: rows < 0, row_len <= 0, max_ctas < 0, `in` or both outputs null; FQB200_ERR_WORKSPACE: a workspace
 * that is missing, too small or misaligned.
 */
int fqb200_sample_angles(const float* in, int64_t rows, int64_t row_len, float* out_angles, double* out_gram,
                         void* workspace, size_t workspace_bytes, int32_t max_ctas, void* stream);
/* Workspace of fqb200_sample_angles in bytes (0 and fqb200_last_error() on bad arguments: rows < 0, row_len <= 0,
 * rows > 8192). */
size_t fqb200_sample_angles_workspace_bytes(int64_t rows, int64_t row_len);

/*
 * Quantization-noise measurement (measure_statistics.py:19-99): for `rows` contiguous rows of `row_len` floats (one
 * sample; any dense memory order of it, the same for y and q), the float64 sums of y and of its quantized form q:
 *   q != NULL: out[r * 7 + k], k = 0 sum y, 1 sum y^2, 2 sum q, 3 sum q^2, 4 sum y*q, 5 sum e, 6 sum e^2 with e = y - q
 *              formed in float64;
 *   q == NULL: out[r * 2 + k], k = 0 sum y, 1 sum y^2 (the layer input, or a weight as one row).
 * `bias` (optional) is added to y first, as the single fp32 add of a quantization launch with fqb200_desc.bias, in its
 * row convention: bias_period > 0 gives element i of a row bias[i / bias_period] (NCHW, bias_period = H*W), < 0
 * bias[i % -bias_period] (channels-last, -C); |bias_period| must divide row_len, and rows with a bias hold fewer than 2^32
 * elements (FQB200_ERR_UNSUPPORTED).  bias_period is ignored without a bias.  Work units are (row, chunk) with a chunk
 * length that depends on row_len only; each unit's partials go to the workspace and a row's partials are added in chunk
 * order, so the bits do not depend on the run or on max_ctas (0: the default grid, else at most that many CTAs).  One
 * read of y and q (16-byte loads where rows are 16-byte aligned, scalar loads otherwise) plus, when a row spans several
 * chunks, a small second launch, on `stream`; no host synchronisation.  NaN and Inf propagate; rows == 0 launches nothing.
 * The workspace (fqb200_sample_noise_workspace_bytes, 16-byte aligned; may be null when that is 0) is private to the call.
 * FQB200_ERR_INVALID: rows < 0, row_len <= 0, max_ctas < 0, y or out null, a bias with a bias_period that does not fit;
 * FQB200_ERR_WORKSPACE: a workspace that is missing, too small or misaligned.
 */
int fqb200_sample_noise(const float* y, const float* q, const float* bias, int64_t bias_period, int64_t rows, int64_t row_len,
                        double* out, void* workspace, size_t workspace_bytes, int32_t max_ctas, void* stream);
/* Workspace of fqb200_sample_noise in bytes, with or without q (0 and fqb200_last_error() on bad arguments: rows < 0,
 * row_len <= 0). */
size_t fqb200_sample_noise_workspace_bytes(int64_t rows, int64_t row_len);

/*
 * Clipping-error measurement (the mse_* / cos_* columns of `-sm collect`, statistic_manager.py:83-111): for every group g
 * of x (layout as fqb200_desc: outer x groups x inner, NCHW order; or channels_last != 0: [outer][inner][groups] memory,
 * groups % 4 == 0, 4 <= groups <= 2048) and the three candidate quantizers of get_alpha(clip_type='mix')
 * (int_quantizer.py:310-323; k = 0 lowp: alpha = (max - min) / 2, 1 gaus, 2 laplace), out[g * 10 + j] =
 *   j = 0: sum x^2;  j = 1 + k: sum (x - q_k)^2;  j = 4 + k: sum x * q_k;  j = 7 + k: sum q_k^2     (float64)
 * where q_k is the torch leaf (FQB200_LEAF_TORCH) with candidate k's parameters, solved on the device from `stats`, the
 * [groups][FQB200_STATS_STRIDE] table of a stats_only fqb200_fused launch on the same x: alpha2DeltaOffset in float64
 * when solve_f64 (per tensor) else fp32, the positive range when `positive`, num_bits (1..8) or, with bit_alloc
 * (num_bits <= 4), the table's allocated widths (column 7) - exactly the parameters the on-the-fly quantizer of each clip
 * type computes from that table.  out_params (optional, [groups][3][6] floats): per candidate delta, offset, bits, scale,
 * zero point, qmax.  An NCHW group with outer > 1 must hold fewer than 2^32 elements.  One read of x (4 B/element) and a
 * small second launch on `stream`; nothing else is written, no host synchronisation.  Work units and summation order
 * are fixed (no atomics on values): the bits do not depend on the run or on max_ctas (0: the default grid, else at most
 * that many CTAs).  The workspace (fqb200_clip_error_workspace_bytes, 16-byte aligned) is private to the call.
 */
int fqb200_clip_error(const float* in, int64_t outer, int64_t groups, int64_t inner, int32_t channels_last, const float* stats,
                      int32_t num_bits, int32_t positive, int32_t bit_alloc, int32_t solve_f64, double* out, float* out_params,
                      void* workspace, size_t workspace_bytes, int32_t max_ctas, void* stream);
/* Workspace of fqb200_clip_error in bytes (0 and fqb200_last_error() on a layout it does not take). */
size_t fqb200_clip_error_workspace_bytes(int64_t outer, int64_t groups, int64_t inner, int32_t channels_last);

/*
 * Clipping-MSE curves (the simulation of the reference's mse_analysis.py, eq. 6 of the paper, on real tensors): for every
 * group g of x (layouts as fqb200_clip_error) and K = num_multipliers (1..256) candidate quantizers that differ only in
 * their clipping value, out[g * (K + 1) + j] =
 *   j = 0: sum x^2;  j = 1 + k: sum (x - q_k)^2     (float64, x - q_k formed in float64)
 * where candidate k clips at alpha = multipliers[k] * b (prior 0, the Laplace scale, column 3 of `stats`) or
 * multipliers[k] * std (prior 1, Gauss, column 4), one fp32 multiply, and q_k is the torch leaf with the parameters
 * solve_range gives that alpha from `stats` (a stats_only fqb200_fused table on the same x), exactly as fqb200_clip_error
 * solves its candidates: float64 alpha2DeltaOffset when solve_f64, else fp32; the positive range when `positive`; num_bits
 * (1..8) or, with bit_alloc (num_bits <= 4), the table's allocated widths.  A multiplier equal to the ACIQ Laplace factor of
 * the width gives fqb200_clip_error's Laplace candidate.  `multipliers` is a device array of K floats.  out_params
 * (optional, [groups][K][6] floats): per candidate delta, offset, bits, scale, zero point, qmax.  One read of x
 * (4 B/element) and a small second launch on `stream`; nothing else is written, no host synchronisation.  Work units and
 * summation order are fixed (no atomics on values): the bits do not depend on the run or on max_ctas (0: the default
 * grid, else at most that many CTAs).  NaN propagates.  The workspace (fqb200_clip_mse_workspace_bytes, 16-byte aligned)
 * is private to the call.  FQB200_ERR_INVALID: a layout fqb200_clip_error does not take, K outside 1..256, prior not 0 or
 * 1, a null x, stats, multipliers or out, bad num_bits / bit_alloc, max_ctas < 0; FQB200_ERR_WORKSPACE: a workspace that
 * is missing, too small or misaligned.
 */
int fqb200_clip_mse(const float* in, int64_t outer, int64_t groups, int64_t inner, int32_t channels_last, const float* stats,
                    int32_t num_bits, int32_t positive, int32_t bit_alloc, int32_t solve_f64, int32_t prior,
                    const float* multipliers, int32_t num_multipliers, double* out, float* out_params, void* workspace,
                    size_t workspace_bytes, int32_t max_ctas, void* stream);
/*
 * fqb200_clip_mse with a bit width per candidate (the per-channel error tables of `-bap mse`): candidate k quantizes at
 * widths[k] instead of num_bits, everything else as fqb200_clip_mse.  `widths` is a host array of K values in 0..8 (read
 * before the call returns; width 0 is the torch leaf with qmax 0); NULL is fqb200_clip_mse.  With widths, prior 2 is the
 * min/max range (FQB200_RANGE_MINMAX from the table's min and max, 0 as the lower bound when `positive`), which ignores
 * the multipliers.  The workspace is fqb200_clip_mse_workspace_bytes.  FQB200_ERR_INVALID, before any CUDA call, also on:
 * a width outside 0..8, widths together with bit_alloc (two sources of widths), prior 2 without widths, prior outside 0..2.
 */
int fqb200_clip_mse_widths(const float* in, int64_t outer, int64_t groups, int64_t inner, int32_t channels_last,
                           const float* stats, int32_t num_bits, int32_t positive, int32_t bit_alloc, int32_t solve_f64,
                           int32_t prior, const float* multipliers, const int32_t* widths, int32_t num_multipliers,
                           double* out, float* out_params, void* workspace, size_t workspace_bytes, int32_t max_ctas,
                           void* stream);
/*
 * fqb200_clip_mse with the choice of each group's clipping value on the device (`-c mse` on the fly): the same `out`
 * sums, bit for bit, and then, in the second launch once a group's sums are final, per group g:
 *   choice[g]   (int32) the column k of the least sum (x - q_k)^2 in statistics.best_columns' order: ties go to the
 *               smaller multiplier, then the earlier column; NaN never wins, so a row of NaN takes the smallest multiplier
 *   given[g], given[groups + g], given[2 * groups + g]   (float32) that candidate's delta, offset and bits, bit for bit
 *               out_params' values at column k
 *   out_table (optional, [groups][FQB200_STATS_STRIDE] floats): columns 0..4 copied from `stats`, 5..10 the chosen
 *               delta, offset, bits, scale, zero point and qmax of the torch leaf, 11 its flags - the table a deferred
 *               shortcut hands to the launch that quantizes it.
 * No atomics and no host synchronisation.  The arguments of fqb200_clip_mse (prior 0 or 1, no widths) and its workspace
 * (fqb200_clip_mse_workspace_bytes).  FQB200_ERR_INVALID, before any CUDA call: fqb200_clip_mse's argument errors and a
 * null choice or given.
 */
int fqb200_clip_mse_select(const float* in, int64_t outer, int64_t groups, int64_t inner, int32_t channels_last,
                           const float* stats, int32_t num_bits, int32_t positive, int32_t bit_alloc, int32_t solve_f64,
                           int32_t prior, const float* multipliers, int32_t num_multipliers, double* out, float* out_params,
                           int32_t* choice, float* given, float* out_table, void* workspace, size_t workspace_bytes,
                           int32_t max_ctas, void* stream);
/* Workspace of fqb200_clip_mse, fqb200_clip_mse_widths and fqb200_clip_mse_select in bytes (0 and fqb200_last_error() on
 * a layout or K it does not take). */
size_t fqb200_clip_mse_workspace_bytes(int64_t outer, int64_t groups, int64_t inner, int32_t channels_last,
                                       int32_t num_multipliers);
/*
 * The joint width-and-clip tables of `-c mse -bap mse`: fqb200_clip_mse over every pair of W = num_widths (1..9) distinct
 * widths (0..8) and M = num_multipliers (1..256) multipliers in one launch.  Candidate j = i * M + k quantizes at
 * widths[i] and clips at alpha = multipliers[k] * b (prior 0) or * std (prior 1):
 *   out[g * (1 + W * M) + 0] = sum x^2;  out[g * (1 + W * M) + 1 + j] = sum (x - q_j)^2
 * and every column has the bits of fqb200_clip_mse_widths on the same (width, multiplier) pair, on every run and for
 * every max_ctas.  `widths` is a host array (read before the call returns), `multipliers` a device array; the other
 * arguments as in fqb200_clip_mse_widths.  out_params (optional): [groups][W * M][6].  Each work unit runs one width's M
 * candidates, so a unit's shared memory is that of an M-candidate launch; x is read from HBM once per chunk and from L2
 * by the chunk's other W - 1 units.  Workspace (fqb200_clip_mse_grid_workspace_bytes): groups x chunks x (1 + W * M) x 8
 * bytes, computed from the shapes - e.g. 64 x 784 x 1126 x 8 = 452 MB for a channels-last 512 x 64 x 112 x 112 tensor at
 * 9 x 125 candidates.  FQB200_ERR_INVALID, before any CUDA call: the layout errors of fqb200_clip_error, M outside
 * 1..256, W outside 1..9, a width outside 0..8 or repeated, prior other than 0 or 1 (min/max ignores the multipliers: it
 * has no grid), bit_alloc set, a null x, stats, multipliers, widths or out, bad num_bits, max_ctas < 0.
 */
int fqb200_clip_mse_grid(const float* in, int64_t outer, int64_t groups, int64_t inner, int32_t channels_last,
                         const float* stats, int32_t num_bits, int32_t positive, int32_t bit_alloc, int32_t solve_f64,
                         int32_t prior, const float* multipliers, int32_t num_multipliers, const int32_t* widths,
                         int32_t num_widths, double* out, float* out_params, void* workspace, size_t workspace_bytes,
                         int32_t max_ctas, void* stream);
/* Workspace of fqb200_clip_mse_grid in bytes (0 and fqb200_last_error() on a layout, M or W it does not take). */
size_t fqb200_clip_mse_grid_workspace_bytes(int64_t outer, int64_t groups, int64_t inner, int32_t channels_last,
                                            int32_t num_multipliers, int32_t num_widths);

/*
 * 1-D k-means quantization of one weight tensor (pytorch_quantizer/quantization/kmeans_quantization.py:14-30): scikit-learn
 * 1.9's KMeans(n_clusters=k, random_state=seed).fit on the n floats of `in` in memory order (k = 2^num_bits, num_bits 1..8,
 * k <= n < 2^40): the data centred on its mean, one k-means++ init, Lloyd with max_iter 300 and tol = var(in) * 1e-4,
 * empty clusters relocated to the farthest points, all in float64 with fixed summation orders (fq_kmeans.cuh).
 *   k-means++: first_id (0 .. n - 1) is the first centre and draws[(c - 1) * n_trials + t] (device, float64) the uniforms of
 *   step c = 1 .. k - 1, trial t (n_trials = 2 + int(log k)) - the host's np.random.RandomState(seed).choice / .uniform
 *   calls in scikit-learn's order; the draws do not depend on the data.  init != NULL (device, k float64 centres in the
 *   data's units, scikit-learn's init= array) replaces k-means++; first_id, draws and n_trials are then ignored.
 * Writes out_labels[n] (nearest centre, ties to the lowest index), out_centres[k] (float32 of centre + mean, like
 * cluster_centers_), out_inertia (float64, about the centred data), out_n_iter, and out_init_ids[k] (the k-means++ sample
 * indices; -1 with init; may be NULL).  task FQB200_KMEANS_QUANTIZE writes out[i] = out_centres[label[i]], FQB200_KMEANS_CLIP
 * writes in clipped to [min, max] of out_centres, FQB200_KMEANS_NONE writes no tensor (out may be NULL).  rows > 0 (with a
 * task; n % rows == 0) also writes out_bcorr = fp32(out - (mean_row(out) - mean_row(in))) over `rows` rows of n / rows
 * (kmeans_quantization.py:86-88; the row means in float64).  `out` and `out_bcorr` must not alias `in`.
 * One cooperative launch on `stream` (and two small memsets); no host synchronisation.  No atomics on values: the bits do not
 * depend on the run or on max_ctas (0: every resident CTA, else at most that many).  The workspace
 * (fqb200_kmeans1d_workspace_bytes, 16-byte aligned) is private to the call; it needs no initialisation.
 */
#define FQB200_KMEANS_NONE 0
#define FQB200_KMEANS_QUANTIZE 1
#define FQB200_KMEANS_CLIP 2
int fqb200_kmeans1d(const float* in, int64_t n, int32_t num_bits, int64_t first_id, const double* draws, int32_t n_trials,
                    const double* init, int32_t task, int64_t rows, uint8_t* out_labels, float* out_centres,
                    double* out_inertia, int32_t* out_n_iter, int64_t* out_init_ids, float* out, float* out_bcorr,
                    void* workspace, size_t workspace_bytes, int32_t max_ctas, void* stream);
/* Workspace of fqb200_kmeans1d in bytes for n elements and k clusters (0 and fqb200_last_error() when k is not a power of
 * two in 2 .. 256 or n < k). */
size_t fqb200_kmeans1d_workspace_bytes(int64_t n, int32_t k);

/*
 * Per-channel weight quantization with given parameters and the weight corrections (`clip_weight="mse"`): the rows
 * [groups][inner] of a contiguous NCHW-ordered weight ([O][I*k*k]) through the torch leaf with the caller's per-row device
 * vectors delta, offset and (optional, NULL = num_bits everywhere) bits, then the correction phases of the FQB200_RANGE_MINMAX
 * weight launch of fqb200_fused: var_corr (`-vcw`) first, then bias_corr (`-bcw`), from the float64 row means and stds of
 * `in`.  hist (optional): 256 int64 counters of the integer grid, accumulated (`-me`).  It runs that launch's plan
 * (bits given = its bit allocation), with the solve replaced by the given parameters, so given the delta, offset and bits
 * columns (5, 6, 7) a RANGE_MINMAX weight launch reports in its statistics table, `out` has that launch's bits, with or
 * without corrections, bit allocation and histogram.  One cooperative launch on `stream`, no host synchronisation.  The
 * workspace (fqb200_quantize_weights_given_workspace_bytes, the same for any `bits` pointer of the same nullness) is the
 * shared one of fqb200_fused (fqb200_workspace_init).  FQB200_ERR_INVALID, before any CUDA call: negative extents,
 * num_bits outside 1..8, a null in, out, delta or offset.
 */
int fqb200_quantize_weights_given(const float* in, float* out, int64_t groups, int64_t inner, const float* delta,
                                  const float* offset, const float* bits, int32_t num_bits, int32_t bias_corr,
                                  int32_t var_corr, unsigned long long* hist, void* workspace, size_t workspace_bytes,
                                  void* stream);
/* Workspace of fqb200_quantize_weights_given in bytes (0 and fqb200_last_error() on arguments it does not take). */
size_t fqb200_quantize_weights_given_workspace_bytes(int64_t groups, int64_t inner, int32_t num_bits, int32_t has_bits,
                                                     int32_t bias_corr, int32_t var_corr);
/*
 * Exact per-channel bit allocation on the device, the result of bit_alloc.allocate bit for bit: the float32 widths_out[G]
 * in 0..8 minimising sum_g sse[g][w_g] (sse: device float64 [G][9], the error of channel g at width w) subject to
 * sum_g w_g <= min(floor(target * G), 8 G); among minimisers the lexicographically smallest width vector.  The same
 * dynamic programme from the last channel to the first, with the same float64 sums in the same order and the strict `<`
 * per width in increasing width order, in one CTA (fq_alloc.cuh).  The host function refuses non-finite errors; here NaN
 * never wins a comparison and any non-finite entry sets *status (optional, device int32) to 1 - it is never cleared, so
 * one flag can collect a whole model.  One launch on `stream`, no host synchronisation.  Workspace
 * (fqb200_allocate_widths_workspace_bytes, private to the call, no initialisation): the uint8 choice table G x (budget +
 * 1), plus the two float64 best[] rows when they exceed 227 KB of shared memory.  FQB200_ERR_INVALID, before any CUDA call:
 * G outside 1..2^20, a negative or NaN budget, a null sse or widths_out; FQB200_ERR_WORKSPACE: a workspace that is missing,
 * too small or misaligned.
 */
int fqb200_allocate_widths(const double* sse, int64_t groups, double target, float* widths_out, int32_t* status,
                           void* workspace, size_t workspace_bytes, void* stream);
/* Workspace of fqb200_allocate_widths in bytes (0 and fqb200_last_error() on arguments it does not take). */
size_t fqb200_allocate_widths_workspace_bytes(int64_t groups, double target);
/*
 * Measured bit allocation on the fly (`-baa -bap mse` with `-sm no`): from the error sums of one call site to the
 * parameters its apply launch takes, in one launch and without host synchronisation.  `sums` (device float64
 * [G][1 + 9 M]) and `out_params` ([G][9 M][6]) are what fqb200_clip_mse_widths (M = 1, widths 0..8) or
 * fqb200_clip_mse_grid (widths 0..8 times M multipliers) write: column 1 + w * M + k is width w at multiplier k.
 *   1. per channel g and width w, the column k of the least sum in statistics.best_columns' order over `multipliers`
 *      (device, M floats, read only when M > 1): ties go to the smaller multiplier, then the earlier column; NaN never wins
 *   2. the widths of fqb200_allocate_widths over those per-width sums (the same programme, bit for bit bit_alloc.allocate),
 *      written to widths_out[G] (float32); *status (optional) is set to 1 on a non-finite per-width sum
 *   3. per channel, for its width w and that width's column k: choice_out[g] = k (optional, int32); given[g],
 *      given[G + g], given[2 G + g] the delta, offset and bits of out_params at (g, w * M + k), bit for bit; out_table
 *      (optional, [G][FQB200_STATS_STRIDE]) columns 0..4 copied from `stats` ([G][FQB200_STATS_STRIDE]), 5..10 that
 *      delta, offset, bits, scale, zero point and qmax of the torch leaf, 11 its flags, as fqb200_clip_mse_select writes it.
 * No atomics.  Workspace (fqb200_allocate_select_workspace_bytes, private to the call, no initialisation).
 * FQB200_ERR_INVALID, before any CUDA call: fqb200_allocate_widths' argument errors, M outside 1..256, a null sums,
 * out_params, widths_out or given, a null multipliers with M > 1, a null stats with out_table.
 */
int fqb200_allocate_select(const double* sums, const float* out_params, const float* multipliers, int32_t num_multipliers,
                           const float* stats, int64_t groups, double target, float* widths_out, int32_t* choice_out,
                           float* given, float* out_table, int32_t* status, void* workspace, size_t workspace_bytes,
                           void* stream);
/* Workspace of fqb200_allocate_select in bytes (0 and fqb200_last_error() on arguments it does not take). */
size_t fqb200_allocate_select_workspace_bytes(int64_t groups, double target);

#ifdef __cplusplus
}
#endif
#endif /* FQB200_H_ */
