// fqb200: fused fake-quantization kernels for H100 (sm_90a) + the C ABI of include/fqb200.h.
//
// One hooked tensor = one launch of fq_fused_kernel, a persistent cooperative kernel:
//
//   phase S1  read x          per-item min / max / sum            -> grid barrier, leader: per-group finalize
//   phase S2  read x          per-item sum|x-mu|, sum (x-mu)^2    -> grid barrier, leader: bit allocation,
//             (only when b or std is needed)                         ACIQ alpha, (delta, offset), scale/zero-point
//   phase A   read x, write y quantize - clip - dequantize with the per-group parameters
//   phase C   (weights only)  mean / variance correction of y
//
// Work item = (group g, part p): a contiguous share of the N*H*W elements of channel g, walked with 128-bit
// loads directly on the NCHW layout (no transposes).  Items are assigned round-robin to the resident CTAs and
// walked in opposite directions in consecutive phases so the tail of one phase is still in L2 for the next.
//
// Reference semantics (file:line in /root/reference) are cited at each device function; the CPU restatement
// they are tested against lives in oracle/fq_oracle.py.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/fqb200.h"
#include "fq_device.cuh"
#include "fq_bulk.cuh"

namespace fqb {

// ACIQ multipliers, int_quantizer.py:81-85.  Index = bit width (0..8).
__constant__ float kGaus[9] = {0.f, 1.24f, 1.71f, 2.15f, 2.55f, 2.93f, 3.28f, 3.61f, 3.92f};
__constant__ float kGausPos[9] = {0.f, 1.71f, 2.15f, 2.55f, 2.93f, 3.28f, 3.61f, 3.92f, 4.2f};
__constant__ float kLaplace[9] = {1.05f, 1.86f, 2.83f, 3.89f, 5.03f, 6.2f, 7.41f, 8.64f, 9.89f};
__constant__ float kLaplacePos[9] = {1.86f, 2.83f, 3.89f, 5.02f, 6.2f, 7.41f, 8.64f, 9.89f, 11.16f};
// mid-tread: optimal Laplace clipping multiplier vs number of bins, int_quantizer.py:41-51 (filled by the host)
constexpr int kTable = 101;
__constant__ double kOmegaTable[kTable];
__constant__ double kAlphaTable[kTable];

enum : int { FLAG_PASSTHROUGH = 1, FLAG_TRUE_ZERO = 2, FLAG_RELU = 4 };

// Per-group (or per-tensor) leaf parameters as the apply phase consumes them.
//   torch leaf:     a = scale, b = zero_point,            c = qmax
//   compiled leaf:  a = scale, b = shift (zp or -offset),  c = qmax, flags
//   mid-tread leaf: a = Delta, b = c_min,                  c = c_max
struct alignas(16) LeafParam {
  float a, b, c;
  int flags;
};

struct FusedArgs {
  Geometry geo;
  FlatGeo flat;        // channels-last / flat-stream kernels (fq_cl.cuh)
  RowsGeo rows;        // ... row structure of the per-sample min-max kernel
  const float* in;
  float* out;
  unsigned out_pad_v;     // channels-last apply: a channel slice of a wider tensor is written, (pixel pitch - C) / 4 vectors
                          // skipped after every pixel (fqb200_fused_into); 0: `out` is dense like `in`
  const float* residual;  // channels-last kernel: optional tensor added to the quantized values (fqb200_desc.residual)
  int residual_relu;      // ... followed by max(., 0)
  PoolGeo pool;           // channels-last kernel: 2x2 / stride-2 max pooling inside the apply phase (pool.tiles != 0) ...
  float* pool_out;        // ... into this [N][H/2][W/2][C] tensor (`out` is not written)
  const float* residual_stats;  // ... quantized on the fly with the parameters of this exported table first
  const float* residual_bias;   // ... after this bias has been added to it
  const float* bias;   // optional per-group addend applied to x before everything else (folded-BN conv bias)
  unsigned long long bias_magic;  // 0: bias[g];  else ceil(2^40 / period_v): bias[(j * magic) >> 40], j = column in vectors
                                  // (per-tensor / per-sample layouts, where a row holds C channels of period_v vectors each)
  float* grid_out;     // optional integer grid (quantize1)
  // configuration (mirrors fqb200_desc)
  int scope, range_mode, leaf, num_bits, positive, solve_f64;
  float clip_k;
  int bit_alloc, prior, ba_round;
  float ba_target;
  float mt_target;
  int mt_clip;
  int bias_corr, var_corr, stats_only;
  int relu_passthrough;  // fqb200_desc.relu_passthrough
  int need_dev;      // phase S2 required (b and/or std)
  const float *g_delta, *g_offset, *g_bits;
  int given_per_group;
  unsigned inner;      // floats per channel row (bundled layouts locate channel boundaries with it)
  double n_per_group;  // outer * inner
  float* out_stats;
  unsigned long long* hist_clamped;  // mid-tread `-me`: [channels][2] elements on the lower / upper clamp bound
  int hist_bins, hist_offset;        // integer-grid histogram: bin = clamp(q + hist_offset, 0, hist_bins - 1)
  unsigned long long* hist;  // optional histogram of the integer grid (entropy measurement, `-me`), accumulated
  unsigned long long* dbg;   // fqb200_desc.debug_stamps: %globaltimer at the phase boundaries (NULL: off)
  // workspace
  GridSync* sync;
  float *pmin, *pmax;                   // [items]
  double *psum, *pabs, *psq;            // [items]
  float *gmin, *gmax, *gmean, *gb, *gstd, *gbits, *gprior;  // [G]
  double* gmean_d;                      // [G]
  float *gdelta, *goffset;              // [G]
  LeafParam* lp;                        // [G] (entry 0 when the parameters are per tensor)
  float *cq, *co, *ck;                  // [G] weight correction: mean(w_q), mean(w), variance factor
  // channels-last kernels: per-channel accumulators combined with atomics, zero between launches (fixed place in
  // the workspace, right after the barrier words)
  unsigned *amin_inv, *amax;            // max of ~enc(x) (= min) and of enc(x), enc = order-preserving uint encoding
  double *asum, *aabs, *asq;
  unsigned nhwc_rep;                    // replicas of the accumulators (CTA b adds into replica b % nhwc_rep): one
                                        // address per channel for the whole grid serialises in L2; rep * C <= 4096
};

constexpr unsigned kMaxNhwcChannels = 4096;

__device__ __forceinline__ void stamp(const FusedArgs& A, int slot) {
  if (A.dbg && threadIdx.x == 0) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    A.dbg[slot] = t;
  }
}

// ------------------------------------------------------------------------------------------------
// leader-section helpers (run by ONE CTA between phases)
// ------------------------------------------------------------------------------------------------
struct LeaderSmem {
  double d[kWarps];
  float f[kWarps];
  int i[kWarps];
  int flag;
};

// Reduce the P per-unit partials of every group in a fixed order (slot p * G + g: coalesced over g).
// `red_lanes` lanes cooperate on one group; kThreads / red_lanes groups are finished per sweep.  Up to three arrays
// are reduced in one sweep so their (independent) L2 round trips overlap.
template <typename T0, typename Op0, typename T1, typename Op1, typename T2, typename Op2>
__device__ __forceinline__ void reduce_partials3(const Geometry& geo, const T0* p0, T0* o0, T0 id0, Op0 op0, const T1* p1,
                                                 T1* o1, T1 id1, Op1 op1, const T2* p2, T2* o2, T2 id2, Op2 op2) {
  const unsigned L = geo.red_lanes;
  const unsigned sub = threadIdx.x % L;
  const unsigned per_sweep = kThreads / L;
  for (unsigned g0 = 0; g0 < geo.channels; g0 += per_sweep) {
    const unsigned g = g0 + threadIdx.x / L;
    T0 a0 = id0;
    T1 a1 = id1;
    T2 a2 = id2;
    if (g < geo.channels) {
#pragma unroll 4
      for (unsigned p = sub; p < geo.parts; p += L) {
        const size_t slot = static_cast<size_t>(p) * geo.channels + g;
        if (p0) a0 = op0(a0, ld_ws(p0 + slot));
        if (p1) a1 = op1(a1, ld_ws(p1 + slot));
        if (p2) a2 = op2(a2, ld_ws(p2 + slot));
      }
    }
    for (unsigned o = L >> 1; o > 0; o >>= 1) {
      a0 = op0(a0, __shfl_xor_sync(0xffffffffu, a0, o));
      a1 = op1(a1, __shfl_xor_sync(0xffffffffu, a1, o));
      a2 = op2(a2, __shfl_xor_sync(0xffffffffu, a2, o));
    }
    if (g < geo.channels && sub == 0) {
      if (p0) o0[g] = a0;
      if (p1) o1[g] = a1;
      if (p2) o2[g] = a2;
    }
  }
}

// per-group bit allocation, int_quantizer.py:381-407 (get_bits_alloc_fixed_target).  All threads of the CTA.
__device__ __noinline__ void solve_bit_alloc(const FusedArgs& A, LeaderSmem& sm) {
  const unsigned G = A.geo.channels;
  const float* prior = (A.prior == FQB200_PRIOR_STD) ? A.gstd : A.gb;
  // p = alpha^(2/3)  (torch.pow with a python-float exponent -> fp32 powf).  Up to kRegGroups groups per thread stay
  // in registers across the iterations (G <= 2048: every CNN layer); larger G falls back to the workspace arrays.
  constexpr unsigned kRegGroups = 4;
  const bool in_regs = G <= kRegGroups * kThreads;
  float pr[kRegGroups], bt[kRegGroups];
  double local = 0.0;
#pragma unroll
  for (unsigned k = 0; k < kRegGroups; ++k) {
    pr[k] = 0.f;
    bt[k] = 0.f;
  }
  if (in_regs) {
#pragma unroll
    for (unsigned k = 0; k < kRegGroups; ++k) {
      const unsigned g = threadIdx.x + k * kThreads;
      if (g < G) {
        pr[k] = powf(prior[g], 0.6666666666666666f);
        local += static_cast<double>(pr[k]);
      }
    }
  } else {
    for (unsigned g = threadIdx.x; g < G; g += kThreads) {
      float p = powf(prior[g], 0.6666666666666666f);
      A.gprior[g] = p;
      local += static_cast<double>(p);
    }
  }
  const float psum = static_cast<float>(block_reduce(local, OpAdd(), sm.d));
  stamp(A, 15);
  const float goal = A.ba_target;
  double m = static_cast<double>(A.ba_target);
  float half_gap = 1.0f;
  const float inv_g = 1.0f / static_cast<float>(G);  // torch's CUDA mean multiplies by fl(1/N)
  int it = 0;
  __shared__ int warp_bits[2][kWarps];
  auto bits_of = [&](float p, float budget) {
    const float bins = __fdiv_rn(__fmul_rn(budget, p), psum);
    const float lg = log2f(bins);
    float bits = A.ba_round ? rintf(lg) : ceilf(lg);
    if (!(bits >= 0.f)) bits = 0.f;
    if (bits > 8.f) bits = 8.f;
    return bits;
  };
  while (fabsf(2.0f * half_gap) > 0.01f && it < 10) {
    const float budget = static_cast<float>(static_cast<double>(G) * exp2(m));
    int sum_bits = 0;
    if (in_regs) {
#pragma unroll
      for (unsigned k = 0; k < kRegGroups; ++k) {
        if (threadIdx.x + k * kThreads < G) {
          bt[k] = bits_of(pr[k], budget);
          sum_bits += static_cast<int>(bt[k]);
        }
      }
    } else {
      for (unsigned g = threadIdx.x; g < G; g += kThreads) {
        const float bits = bits_of(A.gprior[g], budget);
        A.gbits[g] = bits;
        sum_bits += static_cast<int>(bits);
      }
    }
    // exact integer sum: one REDUX per warp, one barrier per iteration (buffers alternate)
    sum_bits = __reduce_add_sync(0xffffffffu, sum_bits);
    if ((threadIdx.x & 31) == 0) warp_bits[it & 1][threadIdx.x >> 5] = sum_bits;
    cta_sync();
    int total = 0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) total += warp_bits[it & 1][w];
    ++it;
    const float mean = __fmul_rn(static_cast<float>(total), inv_g);
    half_gap = __fmul_rn(__fsub_rn(goal, mean), 0.5f);
    m += static_cast<double>(half_gap);
  }
  stamp(A, 11);
  if (in_regs) {
#pragma unroll
    for (unsigned k = 0; k < kRegGroups; ++k) {
      const unsigned g = threadIdx.x + k * kThreads;
      if (g < G) A.gbits[g] = bt[k];
    }
  }
  cta_sync();
}

// Internal range rule of the clipping-error candidates (fq_cliperr.cuh), not a public FQB200_RANGE_* value: the `lowp`
// alpha of get_alpha(clip_type='mix'), (max - min) / 2 (int_quantizer.py:320), through alpha2DeltaOffset like the others.
constexpr int kRangeLowp = -1;

// (delta, offset) of one group/tensor from its statistics: int_quantizer.py:284-300 (alpha2DeltaOffset),
// :227-275 (alpha), :348-352 / :354-357 (fp32 per-channel vs float64 per-tensor arithmetic), :361-379, :409-424.
__device__ __forceinline__ void solve_range(int range_mode, bool positive, int num_bits, float clip_k, bool solve_f64,
                                            float mn, float mx, float mean, float b, float sd, float bits, float& delta,
                                            float& offset) {
  if (range_mode == FQB200_RANGE_MINMAX) {
    offset = positive ? 0.f : mn;
    delta = __fsub_rn(mx, offset);
    return;
  }
  float alpha;
  const int bi = static_cast<int>(bits);
  if (range_mode == FQB200_RANGE_LAPLACE) {
    alpha = __fmul_rn(b, positive ? kLaplacePos[bi] : kLaplace[bi]);
  } else if (range_mode == FQB200_RANGE_GAUS) {
    alpha = __fmul_rn(sd, positive ? kGausPos[num_bits] : kGaus[num_bits]);
  } else if (range_mode == kRangeLowp) {
    alpha = __fmul_rn(__fsub_rn(mx, mn), 0.5f);   // = RN((mx - mn) / 2)
  } else {
    alpha = __fmul_rn(clip_k, sd);
  }
  if (solve_f64) {
    const double al = alpha, me = mean;
    double dl, of;
    if (positive) {
      dl = fmax(me, 0.0) + al;
      of = 0.0;
    } else {
      dl = 2.0 * al;
      of = fmax(static_cast<double>(mn), me - al);
    }
    delta = static_cast<float>(dl);
    offset = static_cast<float>(of);
  } else {
    if (positive) {
      delta = __fadd_rn(fmaxf(mean, 0.f), alpha);
      offset = 0.f;
    } else {
      const float rng = __fmul_rn(2.f, alpha);
      offset = fmaxf(mn, __fsub_rn(mean, alpha));
      // the reference forms max_ = offset + range and later max_ - offset (:351, :447)
      delta = __fsub_rn(__fadd_rn(offset, rng), offset);
    }
  }
}
__device__ __forceinline__ void solve_range(const FusedArgs& A, float mn, float mx, float mean, float b, float sd,
                                            float bits, float& delta, float& offset) {
  solve_range(A.range_mode, A.positive != 0, A.num_bits, A.clip_k, A.solve_f64 != 0, mn, mx, mean, b, sd, bits, delta,
              offset);
}

// leaf parameters from (delta, offset, bits)
__device__ __forceinline__ LeafParam make_leaf_param(int leaf, float delta, float offset, float bits, bool relu = false) {
  LeafParam q;
  q.flags = 0;
  if (leaf == FQB200_LEAF_TORCH) {
    // int_quantizer.py:557-572
    const float qmax = static_cast<float>((1 << static_cast<int>(bits)) - 1);
    float scale = (qmax > 0.f) ? __fdiv_rn(delta, qmax) : 0.f;
    scale = fmaxf(scale, 1e-8f);
    q.a = scale;
    q.b = rintf(__fsub_rn(0.f, __fdiv_rn(offset, scale)));
    q.c = qmax;
    q.flags = FLAG_TRUE_ZERO;
  } else {
    // gemmlowp.cu:30-41 with int_quantizer.py:613 (preserve_zero)
    if (!(delta > 0.f)) {
      q.a = 1.f;
      q.b = 0.f;
      q.c = 0.f;
      q.flags = FLAG_PASSTHROUGH | (relu ? FLAG_RELU : 0);
      return q;
    }
    const float qmax = static_cast<float>((1 << static_cast<int>(bits)) - 1);
    const float scale = __fdiv_rn(delta, qmax);
    const bool tz = (__fadd_rn(offset, delta) > 0.f) && (offset < 0.f);
    q.a = scale;
    q.b = tz ? roundf(__fdiv_rn(-offset, scale)) : -offset;
    q.c = qmax;
    q.flags = tz ? FLAG_TRUE_ZERO : 0;
  }
  return q;
}

__device__ __forceinline__ void export_stats(const FusedArgs& A, unsigned g, float mn, float mx, float mean, float b,
                                             float sd, float delta, float offset, float bits, const LeafParam& q) {
  if (!A.out_stats) return;
  float* o = A.out_stats + static_cast<size_t>(g) * FQB200_STATS_STRIDE;
  o[0] = mn; o[1] = mx; o[2] = mean; o[3] = b; o[4] = sd; o[5] = delta; o[6] = offset; o[7] = bits;
  o[8] = q.a; o[9] = q.b; o[10] = q.c; o[11] = static_cast<float>(q.flags);
}

// mid-tread parameters, int_quantizer.py:185-214 (+ :128-145)
__device__ __noinline__ void solve_mid_tread(const FusedArgs& A, LeaderSmem& sm) {
  const unsigned G = A.geo.channels;
  double local = 0.0;
  for (unsigned g = threadIdx.x; g < G; g += kThreads) {
    float p = powf(A.gstd[g], 0.6666666666666666f);
    A.gprior[g] = p;
    local += static_cast<double>(p);
  }
  const float psum = static_cast<float>(block_reduce(local, OpAdd(), sm.d));
  const float budget = static_cast<float>(static_cast<double>(G) * exp2(static_cast<double>(A.mt_target)));
  const bool sym = !A.positive;
  for (unsigned g = threadIdx.x; g < G; g += kThreads) {
    const float omega = rintf(__fdiv_rn(__fmul_rn(budget, A.gprior[g]), psum));
    const float mn = A.gmin[g], mx = A.gmax[g], mu = A.gmean[g], b = A.gb[g];
    float rng;
    if (A.mt_clip) {
      // alpha multiplier: linear interpolation in the (omega, alpha) table, float64, one-sided uses 2*omega
      double om = sym ? static_cast<double>(omega) : 2.0 * static_cast<double>(omega);
      int i = 0;
      while (i < kTable - 1 && kOmegaTable[i] < om) ++i;  // searchsorted(side='left'), clamped to the table
      double am;
      if (i == 0) {
        am = kAlphaTable[0];
      } else {
        const double inc = (kAlphaTable[i] - kAlphaTable[i - 1]) / (kOmegaTable[i] - kOmegaTable[i - 1]);
        am = kAlphaTable[i] - inc * (kOmegaTable[i] - om);
      }
      const float amf = static_cast<float>(am);
      rng = sym ? __fmul_rn(__fmul_rn(2.f, amf), b) : __fadd_rn(fmaxf(mu, 0.f), __fmul_rn(amf, b));
    } else {
      rng = sym ? __fsub_rn(mx, mn) : mx;
    }
    const float step = (omega > 0.f) ? __fdiv_rn(rng, omega) : 3.402823466e+38f;
    LeafParam q;
    q.a = step;
    q.flags = 0;
    if (A.mt_clip) {
      const float mu_q = sym ? __fdiv_rn(mu, step) : __fdiv_rn(fmaxf(mu, 0.f), step);
      q.c = __fadd_rn(mu_q, sym ? __fmul_rn(omega, 0.5f) : omega);
      q.b = sym ? __fsub_rn(mu_q, __fmul_rn(omega, 0.5f)) : 0.f;
    } else {
      q.b = -INFINITY;
      q.c = INFINITY;
    }
    A.lp[g] = q;
    export_stats(A, g, mn, mx, mu, b, A.gstd[g], rng, 0.f, omega, q);
  }
}

// The parameter solve: runs once per launch, after the last statistics phase.
__device__ __noinline__ void solve_params(const FusedArgs& A, LeaderSmem& sm) {
  const unsigned G = A.geo.channels;
  if (A.leaf == FQB200_LEAF_MIDTREAD) {
    solve_mid_tread(A, sm);
    return;
  }
  if (A.g_delta) {
    // fqb200_quantize_weights_given: the caller's per-row (delta, offset, bits) stand in for the solve; the statistics
    // phases ran only for the corrections
    for (unsigned g = threadIdx.x; g < G; g += kThreads) {
      const float delta = A.g_delta[g], offset = A.g_offset[g];
      const float bits = A.g_bits ? A.g_bits[g] : static_cast<float>(A.num_bits);
      A.lp[g] = make_leaf_param(A.leaf, delta, offset, bits);
      A.gdelta[g] = delta;
      A.goffset[g] = offset;
    }
    return;
  }
  const bool alloc = A.bit_alloc && A.num_bits <= 4 && A.scope == FQB200_SCOPE_GROUP;
  if (alloc) solve_bit_alloc(A, sm);
  stamp(A, 12);
  if (A.scope != FQB200_SCOPE_GROUP) {
    // GROUP_MEAN: batch average of the per-sample min / max (int_quantizer.py:372, :525-526);
    // TENSOR: global min / max assembled from the per-row ones.  Either way ONE parameter set.
    float mn, mx;
    if (A.scope == FQB200_SCOPE_GROUP_MEAN) {
      double smin = 0.0, smax = 0.0;
      for (unsigned g = threadIdx.x; g < G; g += kThreads) {
        smin += static_cast<double>(A.gmin[g]);
        smax += static_cast<double>(A.gmax[g]);
      }
      smin = block_reduce(smin, OpAdd(), sm.d);
      smax = block_reduce(smax, OpAdd(), sm.d);
      mn = static_cast<float>(smin / G);
      mx = static_cast<float>(smax / G);
    } else {
      float lmin = INFINITY, lmax = -INFINITY;
      for (unsigned g = threadIdx.x; g < G; g += kThreads) {
        lmin = fminf(lmin, A.gmin[g]);
        lmax = fmaxf(lmax, A.gmax[g]);
      }
      mn = block_reduce(lmin, OpMin(), sm.f);
      mx = block_reduce(lmax, OpMax(), sm.f);
    }
    if (threadIdx.x == 0) {
      float delta, offset;
      solve_range(A, mn, mx, 0.f, 0.f, 0.f, static_cast<float>(A.num_bits), delta, offset);
      const LeafParam q = make_leaf_param(A.leaf, delta, offset, static_cast<float>(A.num_bits), A.relu_passthrough != 0);
      A.lp[0] = q;
      A.gdelta[0] = delta;
      A.goffset[0] = offset;
      export_stats(A, 0, mn, mx, 0.f, 0.f, 0.f, delta, offset, static_cast<float>(A.num_bits), q);
    }
    return;
  }
  for (unsigned g = threadIdx.x; g < G; g += kThreads) {
    const float bits = alloc ? A.gbits[g] : static_cast<float>(A.num_bits);
    const float mn = A.gmin[g], mx = A.gmax[g], mean = A.gmean[g];
    const float b = A.need_dev ? A.gb[g] : 0.f, sd = A.need_dev ? A.gstd[g] : 0.f;
    float delta, offset;
    solve_range(A, mn, mx, mean, b, sd, bits, delta, offset);
    const LeafParam q = make_leaf_param(A.leaf, delta, offset, bits, A.relu_passthrough != 0);
    A.lp[g] = q;
    A.gdelta[g] = delta;
    A.goffset[g] = offset;
    export_stats(A, g, mn, mx, mean, b, sd, delta, offset, bits, q);
  }
}

// ------------------------------------------------------------------------------------------------
// streaming phases
// ------------------------------------------------------------------------------------------------
struct PhaseSmem {
  float f0[kWarps], f1[kWarps];
  double d0[kWarps], d1[kWarps];
  // bundled layouts: one row per channel of the bundle
  float bf0[4][kWarps], bf1[4][kWarps];
  double bd0[4][kWarps], bd1[4][kWarps];
  // `-me`: per-warp histograms of the integer grid (the grid of the torch leaf lives in [0, 255])
  unsigned hist[kWarps][256];
};

__device__ __forceinline__ void hist_clear(PhaseSmem& sm) {
  for (unsigned i = threadIdx.x; i < kWarps * 256u; i += kThreads) (&sm.hist[0][0])[i] = 0u;
  cta_sync();
}
__device__ __forceinline__ void hist_add(PhaseSmem& sm, float q) {
  if (q >= 0.f && q <= 255.f) atomicAdd(&sm.hist[threadIdx.x >> 5][static_cast<unsigned>(q)], 1u);  // NaN falls through
}
__device__ __forceinline__ void hist_flush(PhaseSmem& sm, unsigned long long* out) {
  cta_sync();
  for (unsigned b = threadIdx.x; b < 256u; b += kThreads) {
    unsigned long long c = 0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) c += sm.hist[w][b];
    if (c) atomicAdd(out + b, c);
  }
}

#ifndef FQB_USTATS
#define FQB_USTATS 4
#endif
#ifndef FQB_UAPPLY
#define FQB_UAPPLY 4
#endif
// CTA-wide sums of up to two doubles and min/max of two floats, result valid in thread 0.  Two barriers.
__device__ __forceinline__ void block_combine(PhaseSmem& sm, float& mn, float& mx, double& s0, double& s1, bool use_f,
                                              bool use_d1) {
  if (use_f) {
    mn = warp_reduce(mn, OpMin());
    mx = warp_reduce(mx, OpMax());
  }
  s0 = warp_reduce(s0, OpAdd());
  if (use_d1) s1 = warp_reduce(s1, OpAdd());
  cta_sync();
  const unsigned w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) {
    sm.f0[w] = mn;
    sm.f1[w] = mx;
    sm.d0[w] = s0;
    sm.d1[w] = s1;
  }
  cta_sync();
  if (w == 0) {
    float a = (l < kWarps) ? sm.f0[l] : INFINITY, b = (l < kWarps) ? sm.f1[l] : -INFINITY;
    double c = (l < kWarps) ? sm.d0[l] : 0.0, d = (l < kWarps) ? sm.d1[l] : 0.0;
#pragma unroll
    for (int o = kWarps / 2; o > 0; o >>= 1) {
      a = fminf(a, __shfl_xor_sync(0xffffffffu, a, o));
      b = fmaxf(b, __shfl_xor_sync(0xffffffffu, b, o));
      c += __shfl_xor_sync(0xffffffffu, c, o);
      d += __shfl_xor_sync(0xffffffffu, d, o);
    }
    mn = a;
    mx = b;
    s0 = c;
    s1 = d;
  }
}

// the bias addend of a vector: per group, or per channel inside the row (bias_magic != 0)
// BIASJ is a compile-time switch: the column j is dead code (and with it the consume-side cursor of the statistics
// phases) in every kernel that does not need it.
template <bool BIASJ>
__device__ __forceinline__ float bias_at(const FusedArgs& A, float group_bias, unsigned j) {
  if (!BIASJ) return group_bias;
  return __ldg(A.bias + static_cast<unsigned>((static_cast<unsigned long long>(j) * A.bias_magic) >> 40));
}

// S1: min / max / sum per unit  (int_quantizer.py:541-546)
template <int VEC, bool BIASJ = false>
struct AccStats1 {
  const FusedArgs& A;
  PhaseSmem& sm;
  float mn, mx, bias;
  double s;
  __device__ __forceinline__ void begin(const UnitInfo& ui) {
    mn = INFINITY;
    mx = -INFINITY;
    s = 0.0;
    bias = (A.bias && !BIASJ) ? __ldg(A.bias + ui.g) : 0.f;  // x + 0 when there is none
  }
  __device__ __forceinline__ void consume(const float4& v, unsigned, unsigned j) {
    const float bj = bias_at<BIASJ>(A, bias, j);
    const float x0 = __fadd_rn(v.x, bj), x1 = __fadd_rn(v.y, bj), x2 = __fadd_rn(v.z, bj), x3 = __fadd_rn(v.w, bj);
    mn = fminf(mn, fminf(fminf(x0, x1), fminf(x2, x3)));
    mx = fmaxf(mx, fmaxf(fmaxf(x0, x1), fmaxf(x2, x3)));
    s += static_cast<double>(__fadd_rn(__fadd_rn(x0, x1), __fadd_rn(x2, x3)));
  }
  __device__ __forceinline__ void consume(const float& v, unsigned, unsigned j) {
    const float x = __fadd_rn(v, bias_at<BIASJ>(A, bias, j));
    mn = fminf(mn, x);
    mx = fmaxf(mx, x);
    s += static_cast<double>(x);
  }
  __device__ __forceinline__ void end(const UnitInfo& ui) {
    double unused = 0.0;
    block_combine(sm, mn, mx, s, unused, true, false);
    if (threadIdx.x == 0) {
      const size_t u = static_cast<size_t>(ui.p) * A.geo.channels + ui.g;
      st_ws(A.pmin + u, mn);
      st_ws(A.pmax + u, mx);
      st_ws(A.psum + u, s);
    }
  }
};

// S2: sum |x - mu| and sum (x - mu)^2 per unit, mu = fp32 group mean  (int_quantizer.py:547-550).
// Also used on the quantized weights for the variance correction (then without the bias addend).
template <int VEC>
struct AccStats2 {
  const FusedArgs& A;
  PhaseSmem& sm;
  const float* mean;
  bool with_bias;
  double* out_abs;
  double* out_sq;
  float mu, bias;
  double sa, sq;
  __device__ __forceinline__ void begin(const UnitInfo& ui) {
    mu = ld_ws(mean + ui.g);
    bias = (with_bias && A.bias) ? __ldg(A.bias + ui.g) : 0.f;
    sa = 0.0;
    sq = 0.0;
  }
  __device__ __forceinline__ void consume(const float4& v, unsigned, unsigned j) {
    const float d0 = __fsub_rn(__fadd_rn(v.x, bias), mu), d1 = __fsub_rn(__fadd_rn(v.y, bias), mu);
    const float d2 = __fsub_rn(__fadd_rn(v.z, bias), mu), d3 = __fsub_rn(__fadd_rn(v.w, bias), mu);
    sa += static_cast<double>(__fadd_rn(__fadd_rn(fabsf(d0), fabsf(d1)), __fadd_rn(fabsf(d2), fabsf(d3))));
    sq += static_cast<double>(__fmaf_rn(d3, d3, __fmaf_rn(d2, d2, __fmaf_rn(d1, d1, __fmul_rn(d0, d0)))));
  }
  __device__ __forceinline__ void consume(const float& v, unsigned, unsigned j) {
    const float d = __fsub_rn(__fadd_rn(v, bias), mu);
    sa += static_cast<double>(fabsf(d));
    sq += static_cast<double>(__fmul_rn(d, d));
  }
  __device__ __forceinline__ void end(const UnitInfo& ui) {
    float f0 = 0.f, f1 = 0.f;
    block_combine(sm, f0, f1, sa, sq, false, true);
    if (threadIdx.x == 0) {
      const size_t u = static_cast<size_t>(ui.p) * A.geo.channels + ui.g;
      if (out_abs) st_ws(out_abs + u, sa);
      st_ws(out_sq + u, sq);
    }
  }
};

// one element through the leaf
template <int LEAF, bool FAST, bool NOISE = false>
__device__ __forceinline__ float leaf_apply(float x, const LeafParam& q, const Divisor& dv, float noise, float& grid) {
  if constexpr (LEAF == FQB200_LEAF_TORCH) {
    // int_quantizer.py:573-592: o = x/scale + zp; clamp [0, qmax]; round-half-even; (o - zp) * scale
    float t = __fadd_rn(div_exact<FAST>(x, dv), q.b);
    t = max_nan(min_nan(t, q.c), 0.f);
    t = rint_small_nonneg(t);
    grid = t;
    return __fmul_rn(__fsub_rn(t, q.b), q.a);
  } else if constexpr (LEAF == FQB200_LEAF_COMPILED) {
    // gemmlowp.cu:10-24
    if (q.flags & FLAG_PASSTHROUGH) {
      grid = x;
      return ((q.flags & FLAG_RELU) && x < 0.f) ? 0.f : x;  // the caller fused the ReLU that follows away
    }
    float t;
    if (q.flags & FLAG_TRUE_ZERO)
      t = __fadd_rn(div_exact<FAST>(x, dv), q.b);
    else
      t = div_exact<FAST>(__fadd_rn(x, q.b), dv);
    if (NOISE) t = __fadd_rn(t, noise);
    t = fmaxf(fminf(t, q.c), 0.f);
    t = roundf(t);
    grid = t;
    if (q.flags & FLAG_TRUE_ZERO) return __fmul_rn(__fsub_rn(t, q.b), q.a);
    return __fmaf_rn(t, q.a, -q.b);  // single FFMA in the reference's nvcc build (DESIGN.md, "a1 contraction")
  } else {
    // int_quantizer.py:202-224: round(x/Delta), clamp to [c_min, c_max], * Delta
    float t = rintf(div_exact<FAST>(x, dv));
    t = max_nan(min_nan(t, q.c), q.b);
    grid = t;
    return __fmul_rn(t, q.a);
  }
}

// ------------------------------------------------------------------------------------------------
// bundled layouts (inner % 4 != 0): every thread sits on a fixed column of the bundle row, so its four floats always
// belong to channel cA (the first `split` of them) and, when the vector straddles a row end, channel cA + 1.
// ------------------------------------------------------------------------------------------------
struct Column {
  unsigned chA;    // global channel of the first element
  unsigned split;  // 1..4 elements belong to chA, the rest to chA + 1
};
__device__ __forceinline__ Column column_of(const FusedArgs& A, const UnitInfo& ui) {
  const unsigned inner = A.inner;  // floats per channel row
  const unsigned e0 = 4u * ui.start.j;
  const unsigned cA = e0 / inner;
  Column c;
  c.chA = ui.g * A.geo.bundle + cA;
  c.split = min(4u, inner - (e0 - cA * inner));
  return c;
}

// CTA-wide per-channel combine for one bundle: thread values (A-part for channel cA, B-part for cA+1) -> one result
// per channel of the bundle, valid in thread 0 (arrays indexed by channel within the bundle).  Two barriers.
template <bool USE_F, bool USE_D1>
__device__ __forceinline__ void bundle_combine(PhaseSmem& sm, unsigned bundle, unsigned cA, bool hasB, float fA0, float fA1,
                                               double dA0, double dA1, float fB0, float fB1, double dB0, double dB1,
                                               float (&rf0)[4], float (&rf1)[4], double (&rd0)[4], double (&rd1)[4]) {
  const unsigned w = threadIdx.x >> 5, l = threadIdx.x & 31;
  cta_sync();  // previous unit's readers are done with sm
  for (unsigned ch = 0; ch < bundle; ++ch) {
    const bool a = (cA == ch), b = hasB && (cA + 1u == ch);
    float v0 = a ? fA0 : INFINITY, v1 = a ? fA1 : -INFINITY;
    double s0 = a ? dA0 : 0.0, s1 = a ? dA1 : 0.0;
    if (b) {
      v0 = fminf(v0, fB0);
      v1 = fmaxf(v1, fB1);
      s0 += dB0;
      s1 += dB1;
    }
    if (USE_F) {
      v0 = warp_reduce(v0, OpMin());
      v1 = warp_reduce(v1, OpMax());
    }
    s0 = warp_reduce(s0, OpAdd());
    if (USE_D1) s1 = warp_reduce(s1, OpAdd());
    if (l == 0) {
      sm.bf0[ch][w] = v0;
      sm.bf1[ch][w] = v1;
      sm.bd0[ch][w] = s0;
      sm.bd1[ch][w] = s1;
    }
  }
  cta_sync();
  if (w == 0) {
    for (unsigned ch = 0; ch < bundle; ++ch) {
      float a = (l < kWarps) ? sm.bf0[ch][l] : INFINITY, b = (l < kWarps) ? sm.bf1[ch][l] : -INFINITY;
      double c = (l < kWarps) ? sm.bd0[ch][l] : 0.0, d = (l < kWarps) ? sm.bd1[ch][l] : 0.0;
#pragma unroll
      for (int o = kWarps / 2; o > 0; o >>= 1) {
        a = fminf(a, __shfl_xor_sync(0xffffffffu, a, o));
        b = fmaxf(b, __shfl_xor_sync(0xffffffffu, b, o));
        c += __shfl_xor_sync(0xffffffffu, c, o);
        d += __shfl_xor_sync(0xffffffffu, d, o);
      }
      rf0[ch] = a;
      rf1[ch] = b;
      rd0[ch] = c;
      rd1[ch] = d;
    }
  }
}

struct AccStats1B {
  const FusedArgs& A;
  PhaseSmem& sm;
  Column col;
  float mnA, mxA, mnB, mxB, biasA, biasB;
  double sA, sB;
  __device__ __forceinline__ void begin(const UnitInfo& ui) {
    col = column_of(A, ui);
    mnA = mnB = INFINITY;
    mxA = mxB = -INFINITY;
    sA = sB = 0.0;
    biasA = A.bias ? __ldg(A.bias + col.chA) : 0.f;
    biasB = (A.bias && col.split < 4u) ? __ldg(A.bias + col.chA + 1u) : 0.f;
  }
  __device__ __forceinline__ void consume(const float4& v, unsigned, unsigned j) {
    const unsigned sp = col.split;
    const float x0 = __fadd_rn(v.x, biasA);
    const float x1 = __fadd_rn(v.y, sp > 1u ? biasA : biasB);
    const float x2 = __fadd_rn(v.z, sp > 2u ? biasA : biasB);
    const float x3 = __fadd_rn(v.w, sp > 3u ? biasA : biasB);
    // A part
    mnA = fminf(mnA, fminf(fminf(x0, sp > 1u ? x1 : INFINITY), fminf(sp > 2u ? x2 : INFINITY, sp > 3u ? x3 : INFINITY)));
    mxA = fmaxf(mxA, fmaxf(fmaxf(x0, sp > 1u ? x1 : -INFINITY), fmaxf(sp > 2u ? x2 : -INFINITY, sp > 3u ? x3 : -INFINITY)));
    sA += static_cast<double>(__fadd_rn(__fadd_rn(x0, sp > 1u ? x1 : 0.f), __fadd_rn(sp > 2u ? x2 : 0.f, sp > 3u ? x3 : 0.f)));
    if (sp < 4u) {  // per-thread constant: only the few columns that straddle a row end come here
      mnB = fminf(mnB, fminf(fminf(sp > 1u ? INFINITY : x1, sp > 2u ? INFINITY : x2), x3));
      mxB = fmaxf(mxB, fmaxf(fmaxf(sp > 1u ? -INFINITY : x1, sp > 2u ? -INFINITY : x2), x3));
      sB += static_cast<double>(__fadd_rn(__fadd_rn(sp > 1u ? 0.f : x1, sp > 2u ? 0.f : x2), x3));
    }
  }
  __device__ __forceinline__ void end(const UnitInfo& ui) {
    float r0[4], r1[4];
    double d0[4], d1[4];
    const unsigned base = ui.g * A.geo.bundle;
    bundle_combine<true, false>(sm, A.geo.bundle, col.chA - base, col.split < 4u, mnA, mxA, sA, 0.0, mnB, mxB, sB, 0.0, r0, r1, d0, d1);
    if (threadIdx.x == 0) {
      for (unsigned ch = 0; ch < A.geo.bundle; ++ch) {
        const size_t u = static_cast<size_t>(ui.p) * A.geo.channels + base + ch;
        st_ws(A.pmin + u, r0[ch]);
        st_ws(A.pmax + u, r1[ch]);
        st_ws(A.psum + u, d0[ch]);
      }
    }
  }
};

struct AccStats2B {
  const FusedArgs& A;
  PhaseSmem& sm;
  Column col;
  float muA, muB, biasA, biasB;
  double saA, sqA, saB, sqB;
  __device__ __forceinline__ void begin(const UnitInfo& ui) {
    col = column_of(A, ui);
    const bool hasB = col.split < 4u;
    muA = ld_ws(A.gmean + col.chA);
    muB = hasB ? ld_ws(A.gmean + col.chA + 1u) : 0.f;
    biasA = A.bias ? __ldg(A.bias + col.chA) : 0.f;
    biasB = (A.bias && hasB) ? __ldg(A.bias + col.chA + 1u) : 0.f;
    saA = sqA = saB = sqB = 0.0;
  }
  __device__ __forceinline__ void consume(const float4& v, unsigned, unsigned j) {
    const unsigned sp = col.split;
    const float d0 = __fsub_rn(__fadd_rn(v.x, biasA), muA);
    const float d1 = __fsub_rn(__fadd_rn(v.y, sp > 1u ? biasA : biasB), sp > 1u ? muA : muB);
    const float d2 = __fsub_rn(__fadd_rn(v.z, sp > 2u ? biasA : biasB), sp > 2u ? muA : muB);
    const float d3 = __fsub_rn(__fadd_rn(v.w, sp > 3u ? biasA : biasB), sp > 3u ? muA : muB);
    const float a1 = sp > 1u ? d1 : 0.f, a2 = sp > 2u ? d2 : 0.f, a3 = sp > 3u ? d3 : 0.f;
    saA += static_cast<double>(__fadd_rn(__fadd_rn(fabsf(d0), fabsf(a1)), __fadd_rn(fabsf(a2), fabsf(a3))));
    sqA += static_cast<double>(__fmaf_rn(a3, a3, __fmaf_rn(a2, a2, __fmaf_rn(a1, a1, __fmul_rn(d0, d0)))));
    if (sp < 4u) {
      const float b1 = sp > 1u ? 0.f : d1, b2 = sp > 2u ? 0.f : d2;
      saB += static_cast<double>(__fadd_rn(__fadd_rn(fabsf(b1), fabsf(b2)), fabsf(d3)));
      sqB += static_cast<double>(__fmaf_rn(d3, d3, __fmaf_rn(b2, b2, __fmul_rn(b1, b1))));
    }
  }
  __device__ __forceinline__ void end(const UnitInfo& ui) {
    float r0[4], r1[4];
    double d0[4], d1[4];
    const unsigned base = ui.g * A.geo.bundle;
    bundle_combine<false, true>(sm, A.geo.bundle, col.chA - base, col.split < 4u, 0.f, 0.f, saA, sqA, 0.f, 0.f, saB, sqB, r0, r1, d0, d1);
    if (threadIdx.x == 0) {
      for (unsigned ch = 0; ch < A.geo.bundle; ++ch) {
        const size_t u = static_cast<size_t>(ui.p) * A.geo.channels + base + ch;
        st_ws(A.pabs + u, d0[ch]);
        st_ws(A.psq + u, d1[ch]);
      }
    }
  }
};

__device__ __forceinline__ LeafParam load_leaf_param(const LeafParam* lp, unsigned idx) {
  const float4 raw = ld_ws(reinterpret_cast<const float4*>(lp) + idx);
  LeafParam q;
  q.a = raw.x;
  q.b = raw.y;
  q.c = raw.z;
  q.flags = __float_as_int(raw.w);
  return q;
}

// A: quantize - clip - dequantize one unit with its group's (or the tensor's) parameters held in registers.
// ACC: also accumulate sum(y) (weight bias correction); GRID: also store the integer grid; GIVEN: derive the leaf
// parameters from caller-provided delta / offset / bits instead of the solved table.
template <int VEC, int LEAF, bool ACC, bool GRID, bool GIVEN, bool BIASJ = false>
struct AccApply {
  const FusedArgs& A;
  PhaseSmem& sm;
  LeafParam q;
  Divisor dv;
  float bias;
  double sy;
  __device__ __forceinline__ void begin(const UnitInfo& ui) {
    const unsigned g = ui.g;
    if (GIVEN) {
      const unsigned pi = A.given_per_group ? g : 0u;
      const float bits = A.g_bits ? __ldg(A.g_bits + g) : static_cast<float>(A.num_bits);
      q = make_leaf_param(LEAF, __ldg(A.g_delta + pi), __ldg(A.g_offset + pi), bits);
    } else {
      q = load_leaf_param(A.lp, (A.scope == FQB200_SCOPE_GROUP) ? g : 0u);
    }
    dv = make_divisor(q.a);
    bias = (A.bias && !BIASJ) ? __ldg(A.bias + g) : 0.f;
    sy = 0.0;
  }
  template <bool FAST>
  __device__ __forceinline__ void one(const float4& x, unsigned off, float bias) {
    float4 y, gq;
    y.x = leaf_apply<LEAF, FAST>(__fadd_rn(x.x, bias), q, dv, 0.f, gq.x);
    y.y = leaf_apply<LEAF, FAST>(__fadd_rn(x.y, bias), q, dv, 0.f, gq.y);
    y.z = leaf_apply<LEAF, FAST>(__fadd_rn(x.z, bias), q, dv, 0.f, gq.z);
    y.w = leaf_apply<LEAF, FAST>(__fadd_rn(x.w, bias), q, dv, 0.f, gq.w);
    st_tensor(reinterpret_cast<float4*>(A.out) + off, y);
    if (GRID) st_tensor(reinterpret_cast<float4*>(A.grid_out) + off, gq);
    if (ACC) sy += static_cast<double>(__fadd_rn(__fadd_rn(y.x, y.y), __fadd_rn(y.z, y.w)));
    if (LEAF == FQB200_LEAF_TORCH && A.hist) {  // launch-uniform
      hist_add(sm, gq.x);
      hist_add(sm, gq.y);
      hist_add(sm, gq.z);
      hist_add(sm, gq.w);
    }
  }
  template <bool FAST>
  __device__ __forceinline__ void one(const float& x, unsigned off, float bias) {
    float gq;
    const float y = leaf_apply<LEAF, FAST>(__fadd_rn(x, bias), q, dv, 0.f, gq);
    st_tensor(A.out + off, y);
    if (GRID) st_tensor(A.grid_out + off, gq);
    if (ACC) sy += static_cast<double>(y);
    if (LEAF == FQB200_LEAF_TORCH && A.hist) hist_add(sm, gq);
  }
  template <typename V>
  __device__ __forceinline__ void consume(const V& x, unsigned off, unsigned j) {
    const float bj = bias_at<BIASJ>(A, bias, j);
    if (dv.fast)  // CTA-uniform
      one<true>(x, off, bj);
    else
      one<false>(x, off, bj);
  }
  __device__ __forceinline__ void end(const UnitInfo& ui) {
    if (ACC) {
      float f0 = 0.f, f1 = 0.f;
      double unused = 0.0;
      block_combine(sm, f0, f1, sy, unused, false, false);
      if (threadIdx.x == 0) st_ws(A.psum + static_cast<size_t>(ui.p) * A.geo.channels + ui.g, sy);
    } else {
      cta_sync();  // the engine publishes the next unit ids at this barrier
    }
  }
};

// C1: y <- (y - m_q) * k + m_q  (variance), then y <- y - m_q + m_o  (mean); inference_quantization_manager.py:386-391
template <int VEC>
struct AccCorr {
  const FusedArgs& A;
  float mq, mo, kv;
  bool vc, bc;
  __device__ __forceinline__ void begin(const UnitInfo& ui) {
    const unsigned g = ui.g;
    mq = ld_ws(A.cq + g);
    mo = ld_ws(A.co + g);
    kv = A.var_corr ? ld_ws(A.ck + g) : 1.f;
    vc = A.var_corr != 0;
    bc = A.bias_corr != 0;
  }
  __device__ __forceinline__ float fix(float y) const {
    if (vc) y = __fadd_rn(__fmul_rn(__fsub_rn(y, mq), kv), mq);
    if (bc) y = __fadd_rn(__fsub_rn(y, mq), mo);
    return y;
  }
  __device__ __forceinline__ void consume(const float4& y, unsigned off, unsigned) {
    st_tensor(reinterpret_cast<float4*>(A.out) + off, make_float4(fix(y.x), fix(y.y), fix(y.z), fix(y.w)));
  }
  __device__ __forceinline__ void consume(const float& y, unsigned off, unsigned) { st_tensor(A.out + off, fix(y)); }
  __device__ __forceinline__ void end(const UnitInfo&) { cta_sync(); }
};

template <int LEAF>
struct AccApplyB {
  const FusedArgs& A;
  PhaseSmem& sm;
  Column col;
  LeafParam qA, qB;
  Divisor dvA, dvB;
  float biasA, biasB;
  __device__ __forceinline__ void begin(const UnitInfo& ui) {
    col = column_of(A, ui);
    const bool hasB = col.split < 4u;
    const bool per_group = (A.scope == FQB200_SCOPE_GROUP);
    qA = load_leaf_param(A.lp, per_group ? col.chA : 0u);
    qB = hasB ? load_leaf_param(A.lp, per_group ? col.chA + 1u : 0u) : qA;
    dvA = make_divisor(qA.a);
    dvB = make_divisor(qB.a);
    biasA = A.bias ? __ldg(A.bias + col.chA) : 0.f;
    biasB = (A.bias && hasB) ? __ldg(A.bias + col.chA + 1u) : biasA;
  }
  template <bool FAST>
  __device__ __forceinline__ float elem(float x, bool inA) {
    LeafParam q;
    Divisor dv;
    q.a = inA ? qA.a : qB.a;
    q.b = inA ? qA.b : qB.b;
    q.c = inA ? qA.c : qB.c;
    q.flags = inA ? qA.flags : qB.flags;
    dv.s = q.a;
    dv.r = inA ? dvA.r : dvB.r;
    dv.fast = FAST;
    float gq;
    const float y = leaf_apply<LEAF, FAST>(__fadd_rn(x, inA ? biasA : biasB), q, dv, 0.f, gq);
    if (LEAF == FQB200_LEAF_TORCH && A.hist) hist_add(sm, gq);
    return y;
  }
  template <bool FAST>
  __device__ __forceinline__ void one(const float4& x, unsigned off) {
    const unsigned sp = col.split;
    float4 y;
    y.x = elem<FAST>(x.x, true);
    y.y = elem<FAST>(x.y, sp > 1u);
    y.z = elem<FAST>(x.z, sp > 2u);
    y.w = elem<FAST>(x.w, sp > 3u);
    st_tensor(reinterpret_cast<float4*>(A.out) + off, y);
  }
  __device__ __forceinline__ void consume(const float4& x, unsigned off, unsigned) {
    if (dvA.fast && dvB.fast)
      one<true>(x, off);
    else
      one<false>(x, off);
  }
  __device__ __forceinline__ void end(const UnitInfo&) { cta_sync(); }
};

// ------------------------------------------------------------------------------------------------
// the fused persistent kernel (cooperative launch: every CTA is resident)
// ------------------------------------------------------------------------------------------------
// One instantiation per (vector width, leaf, second statistics pass?, weight correction?) so that each kernel holds
// only the loops it runs.  Phase directions: S1 forward, S2 backward, A forward again (backward when there is no S2):
// each phase starts on the bytes the previous one touched last, which are still in L2.
// MODE: 4 = 128-bit path, 1 = scalar path, 8 = bundled 128-bit path (inner % 4 != 0, see Geometry)
// BIASJ: the bias is indexed by the channel inside the row (fqb200_desc.bias_period); instantiated for the one
// configuration that uses it (128-bit path, min/max range, compiled leaf: the per-tensor / per-sample activations).
template <int MODE, int LEAF, bool DEV, bool CORR, bool BIASJ = false>
__global__ void __launch_bounds__(kThreads, kCtasPerSm) fq_fused_kernel(const __grid_constant__ FusedArgs A) {
  constexpr int VEC = (MODE == 1) ? 1 : 4;
  constexpr bool BUNDLED = (MODE == 8);
  static_assert(!(BUNDLED && CORR), "weight correction runs on the plain layouts");
  static_assert(!BIASJ || (MODE == 4 && !DEV && !CORR), "bias_period: 128-bit path, one statistics pass, no correction");
  __shared__ PhaseSmem psm;
  __shared__ LeaderSmem lsm;
  __shared__ StreamSmem ssm;
  unsigned epoch = 0;
  const Geometry& geo = A.geo;
  const double n = A.n_per_group;

  // ---- S1
  if (blockIdx.x == 0) stamp(A, 0);
  if constexpr (BUNDLED) {
    AccStats1B acc{A, psm};
    stream_units<4, false>(geo, A.in, &A.sync->unit_counter[0], ssm, acc);
  } else {
    AccStats1<VEC, BIASJ> acc{A, psm};
    stream_units<VEC, false>(geo, A.in, &A.sync->unit_counter[0], ssm, acc);
  }
  if (blockIdx.x == 0) stamp(A, 1);
  if (grid_arrive(A.sync, epoch, &lsm.flag)) {
    stamp(A, 2);
    reduce_partials3(geo, A.pmin, A.gmin, INFINITY, OpMin(), A.pmax, A.gmax, -INFINITY, OpMax(), A.psum, A.gmean_d, 0.0, OpAdd());
    cta_sync();
    for (unsigned g = threadIdx.x; g < geo.channels; g += kThreads) {
      const double m = A.gmean_d[g] / n;
      A.gmean_d[g] = m;
      A.gmean[g] = static_cast<float>(m);
    }
    cta_sync();
    if (!DEV) solve_params(A, lsm);
    stamp(A, 3);
    grid_release(A.sync, epoch);
  }
  if (blockIdx.x == 0) stamp(A, 4);

  // ---- S2
  if constexpr (DEV) {
    if constexpr (BUNDLED) {
      AccStats2B acc{A, psm};
      stream_units<4, true>(geo, A.in, &A.sync->unit_counter[1], ssm, acc);
    } else {
      AccStats2<VEC> acc{A, psm, A.gmean, true, A.pabs, A.psq};
      stream_units<VEC, true>(geo, A.in, &A.sync->unit_counter[1], ssm, acc);
    }
    if (blockIdx.x == 0) stamp(A, 5);
    if (grid_arrive(A.sync, epoch, &lsm.flag)) {
      stamp(A, 6);
      double* tabs = A.psum;              // [>= G] free now
      double* tsq = A.psum + geo.channels;  // psum holds slots + 2G doubles
      reduce_partials3(geo, A.pabs, tabs, 0.0, OpAdd(), A.psq, tsq, 0.0, OpAdd(), static_cast<const double*>(nullptr),
                       static_cast<double*>(nullptr), 0.0, OpAdd());
      cta_sync();
      stamp(A, 10);
      for (unsigned g = threadIdx.x; g < geo.channels; g += kThreads) {
        A.gb[g] = static_cast<float>(tabs[g] / n);
        // sum (x - mu32)^2 -> sum (x - mu)^2 with the exact mean; unbiased (torch.std default)
        const double dm = A.gmean_d[g] - static_cast<double>(A.gmean[g]);
        double ss = tsq[g] - n * dm * dm;
        if (ss < 0.0) ss = 0.0;
        A.gstd[g] = static_cast<float>(sqrt(ss / (n - 1.0)));
      }
      cta_sync();
      stamp(A, 11);
      solve_params(A, lsm);
      stamp(A, 7);
      grid_release(A.sync, epoch);
    }
    if (blockIdx.x == 0) stamp(A, 8);
  }

  // ---- A (+ C)
  if (!A.stats_only) {
    if (LEAF == FQB200_LEAF_TORCH && A.hist) hist_clear(psm);
    if constexpr (BUNDLED) {
      AccApplyB<LEAF> acc{A, psm};
      stream_units<4, !DEV>(geo, A.in, &A.sync->unit_counter[2], ssm, acc);
    } else {
      AccApply<VEC, LEAF, CORR, false, false, BIASJ> acc{A, psm};
      stream_units<VEC, !DEV>(geo, A.in, &A.sync->unit_counter[2], ssm, acc);
    }
    if (LEAF == FQB200_LEAF_TORCH && A.hist) hist_flush(psm, A.hist);
    if (blockIdx.x == 0) stamp(A, 9);
    if constexpr (CORR) {
      if (grid_arrive(A.sync, epoch, &lsm.flag)) {
        double* tmp = A.pabs;
        reduce_partials3(geo, A.psum, tmp, 0.0, OpAdd(), static_cast<const double*>(nullptr), static_cast<double*>(nullptr), 0.0,
                         OpAdd(), static_cast<const double*>(nullptr), static_cast<double*>(nullptr), 0.0, OpAdd());
        cta_sync();
        for (unsigned g = threadIdx.x; g < geo.channels; g += kThreads) {
          A.cq[g] = static_cast<float>(tmp[g] / n);
          A.co[g] = A.gmean[g];
        }
        grid_release(A.sync, epoch);
      }
      if (A.var_corr) {
        {
          AccStats2<VEC> acc{A, psm, A.cq, false, nullptr, A.psq};
          stream_units<VEC, false>(geo, A.out, &A.sync->unit_counter[3], ssm, acc);
        }
        if (grid_arrive(A.sync, epoch, &lsm.flag)) {
          double* tmp = A.pabs;
          reduce_partials3(geo, A.psq, tmp, 0.0, OpAdd(), static_cast<const double*>(nullptr), static_cast<double*>(nullptr), 0.0,
                           OpAdd(), static_cast<const double*>(nullptr), static_cast<double*>(nullptr), 0.0, OpAdd());
          cta_sync();
          for (unsigned g = threadIdx.x; g < geo.channels; g += kThreads) {
            // tmp = sum (y - fl32(mean_q))^2 ; fl32(mean_q) stands in for the mean (error O(ulp^2))
            const float sdq = static_cast<float>(sqrt(tmp[g] / (n - 1.0)));
            A.ck[g] = __fdiv_rn(A.gstd[g], __fadd_rn(sdq, 1e-8f));
          }
          grid_release(A.sync, epoch);
        }
      }
      {
        AccCorr<VEC> acc{A};
        stream_units<VEC, false>(geo, A.out, &A.sync->unit_counter[4], ssm, acc);
      }
    }
  }
  grid_exit(A.sync);
}

}  // namespace fqb
#include "fq_cl.cuh"
#include "fq_kld.cuh"
#include "fq_cliperr.cuh"
#include "fq_clipmse.cuh"
#include "fq_kmeans.cuh"
#include "fq_angle.cuh"
#include "fq_sample_sums.cuh"
#include "fq_alloc.cuh"
namespace fqb {

// Standalone a1 with host-side scalars (gemmlowp.cu:30-45): flat grid-stride, parameters by value.
template <int VEC, bool NOISE, bool FAST>
__global__ void __launch_bounds__(kThreads, kCtasPerSm)
    fq_leaf_kernel(const float* __restrict__ in, float* __restrict__ out, const float* __restrict__ noise,
                   unsigned long long nvec, LeafParam q) {
  using V = typename VecT<VEC>::type;
  const Divisor dv = make_divisor(q.a);
  const unsigned long long stride = static_cast<unsigned long long>(gridDim.x) * kThreads;
  unsigned long long i = static_cast<unsigned long long>(blockIdx.x) * kThreads + threadIdx.x;
  constexpr int U = 4;
  for (; i < nvec; i += U * stride) {
    V x[U], nz[U];
    bool ok[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      ok[u] = i + u * stride < nvec;
      if (ok[u]) {
        x[u] = ld_tensor(reinterpret_cast<const V*>(in) + i + u * stride);
        if (NOISE) nz[u] = ld_tensor(reinterpret_cast<const V*>(noise) + i + u * stride);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (!ok[u]) continue;
      float gq;
      if constexpr (VEC == 4) {
        float4 y;
        y.x = leaf_apply<FQB200_LEAF_COMPILED, FAST, NOISE>(x[u].x, q, dv, NOISE ? nz[u].x : 0.f, gq);
        y.y = leaf_apply<FQB200_LEAF_COMPILED, FAST, NOISE>(x[u].y, q, dv, NOISE ? nz[u].y : 0.f, gq);
        y.z = leaf_apply<FQB200_LEAF_COMPILED, FAST, NOISE>(x[u].z, q, dv, NOISE ? nz[u].z : 0.f, gq);
        y.w = leaf_apply<FQB200_LEAF_COMPILED, FAST, NOISE>(x[u].w, q, dv, NOISE ? nz[u].w : 0.f, gq);
        st_tensor(reinterpret_cast<float4*>(out) + i + u * stride, y);
      } else {
        st_tensor(out + i + u * stride, leaf_apply<FQB200_LEAF_COMPILED, FAST, NOISE>(x[u], q, dv, NOISE ? nz[u] : 0.f, gq));
      }
    }
  }
}

// Mode A (parameters given by the caller, int_quantizer.py:557-603 called directly): no statistics, no grid
// barrier, ordinary launch.  Leaf parameters are derived per item from the device-resident delta/offset/bits
// (a few CTA-uniform flops), so nothing is synchronised with the host.
template <int VEC, int LEAF, bool GRID>
__global__ void __launch_bounds__(kThreads, kCtasPerSm) fq_given_kernel(const __grid_constant__ FusedArgs A) {
  __shared__ PhaseSmem psm;
  __shared__ StreamSmem ssm;
  AccApply<VEC, LEAF, false, GRID, true> acc{A, psm};
  stream_units<VEC, false>(A.geo, A.in, nullptr, ssm, acc);
}

// y = max(a + b, 0): the residual add + ReLU that closes every ResNet block, one pass (2 reads + 1 write) instead of torch's
// add_ (2R + 1W) and relu_ (1R + 1W).  fl(a + b) then the clamp: bit-identical to the two torch kernels.  NaN propagates
// like torch.relu (x < 0 ? 0 : x).
template <int VEC>
__global__ void __launch_bounds__(kThreads, kCtasPerSm)
    fq_add_relu_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, unsigned long long nvec) {
  using V = typename VecT<VEC>::type;
  const unsigned long long stride = static_cast<unsigned long long>(gridDim.x) * kThreads;
  unsigned long long i = static_cast<unsigned long long>(blockIdx.x) * kThreads + threadIdx.x;
  constexpr int U = 4;
  auto f = [](float x, float y) {
    const float s = __fadd_rn(x, y);
    return s < 0.f ? 0.f : s;
  };
  for (; i < nvec; i += U * stride) {
    V x[U], y[U];
    bool ok[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      ok[u] = i + u * stride < nvec;
      if (ok[u]) {
        x[u] = ld_tensor(reinterpret_cast<const V*>(a) + i + u * stride);
        y[u] = ld_tensor(reinterpret_cast<const V*>(b) + i + u * stride);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (!ok[u]) continue;
      if constexpr (VEC == 4) {
        st_tensor(reinterpret_cast<float4*>(out) + i + u * stride,
                  make_float4(f(x[u].x, y[u].x), f(x[u].y, y[u].y), f(x[u].z, y[u].z), f(x[u].w, y[u].w)));
      } else {
        st_tensor(out + i + u * stride, f(x[u], y[u]));
      }
    }
  }
}

// Max pooling on channels-last memory ([N][H][W][C], C % 4 == 0): the operator in front of the `activation_pooling`
// quantization call site (MaxPool2dWithId.forward, inference_quantization_manager.py:58-74), in place of torch's NHWC
// kernel; this one is a plain gather of k*k 128-bit vectors per output vector - neighbouring windows overlap in L1 / L2 - with torch's
// NaN rule (a NaN in the window wins).  Results are bit-identical (max is exact).
struct PoolArgs {
  const float* in;
  float* out;
  unsigned long long out_pv;  // output pixel pitch in vectors (cv: dense)
  unsigned n, h, w, cv, oh, ow;
  int kh, kw, sh, sw, ph, pw;
  unsigned long long total;  // output vectors
};
__global__ void __launch_bounds__(256, 4) fq_maxpool_nhwc_kernel(const __grid_constant__ PoolArgs P) {
  const unsigned long long stride = static_cast<unsigned long long>(gridDim.x) * blockDim.x;
  const float4* in = reinterpret_cast<const float4*>(P.in);
  float4* out = reinterpret_cast<float4*>(P.out);
  auto upd = [](float& m, float v) { m = (v > m || v != v) ? v : m; };
  for (unsigned long long i = static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < P.total; i += stride) {
    const unsigned c = static_cast<unsigned>(i % P.cv);
    const unsigned long long pixel = i / P.cv;
    unsigned long long r = pixel;
    const unsigned ow = static_cast<unsigned>(r % P.ow);
    r /= P.ow;
    const unsigned oh = static_cast<unsigned>(r % P.oh);
    const unsigned n = static_cast<unsigned>(r / P.oh);
    const int h0 = static_cast<int>(oh) * P.sh - P.ph, w0 = static_cast<int>(ow) * P.sw - P.pw;
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    for (int dy = 0; dy < P.kh; ++dy) {
      const int y = h0 + dy;
      if (y < 0 || y >= static_cast<int>(P.h)) continue;
      const float4* row = in + (static_cast<unsigned long long>(n) * P.h + y) * P.w * P.cv + c;
#pragma unroll 3
      for (int dx = 0; dx < P.kw; ++dx) {
        const int x = w0 + dx;
        if (x < 0 || x >= static_cast<int>(P.w)) continue;
        const float4 v = __ldg(row + static_cast<unsigned long long>(x) * P.cv);
        upd(m.x, v.x);
        upd(m.y, v.y);
        upd(m.z, v.z);
        upd(m.w, v.w);
      }
    }
    __stcs(out + pixel * P.out_pv + c, m);
  }
}

// test hook: q[i] = div_exact(a[i], b[i]) next to IEEE a[i]/b[i]
__global__ void fq_divtest_kernel(const float* a, const float* b, float* fast, float* ieee, unsigned long long n) {
  const unsigned long long stride = static_cast<unsigned long long>(gridDim.x) * blockDim.x;
  for (unsigned long long i = static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const Divisor dv = make_divisor(b[i]);
    fast[i] = dv.fast ? div_exact<true>(a[i], dv) : div_exact<false>(a[i], dv);
    ieee[i] = __fdiv_rn(a[i], b[i]);
  }
}

}  // namespace fqb

// ================================================================================================
// host side: geometry, workspace carving, launches, C ABI
// ================================================================================================
#include <mutex>

namespace {

thread_local char g_err[512] = "";

int fail(int code, const char* fmt, const char* detail = "", const char* detail2 = "") {
  snprintf(g_err, sizeof(g_err), fmt, detail, detail2);
  return code;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// `need` bytes of caller workspace, as `sizer`() reports them (none: anything goes)
int check_workspace(const void* ws, size_t bytes, size_t need, const char* sizer) {
  if (need && (!ws || bytes < need || !aligned16(ws)))
    return fail(FQB200_ERR_WORKSPACE, "workspace smaller than %s() or not 16-byte aligned", sizer);
  return FQB200_OK;
}

// the error of the launches just queued, if any
int launched(const char* what) {
  const cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) return FQB200_OK;
  return fail(FQB200_ERR_CUDA, *what ? "launch %s: %s" : "launch%s: %s", what, cudaGetErrorString(e));
}

// one CTA per work unit, at most `cap`, or at most `max_ctas` when the caller sets it
int grid_for(unsigned long long units, unsigned long long cap, int max_ctas = 0) {
  if (max_ctas > 0) cap = static_cast<unsigned long long>(max_ctas);
  return static_cast<int>(units < cap ? units : cap);
}

// allow `fn` `smem` bytes of dynamic shared memory; with `per_sm`, also count its CTAs of `threads` that fit on an SM
template <class F>
cudaError_t setup(F fn, int threads, size_t smem, int* per_sm = nullptr) {
  const void* f = reinterpret_cast<const void*>(fn);
  cudaError_t e = cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (e == cudaSuccess && per_sm) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(per_sm, f, threads, smem);
  return e;
}

// channels-last kernel variants: leaf (torch / mid-tread) x second statistics pass x histogram
const void* cl_kernel_ptr(int leaf, bool dev, bool hist) {
#define FQB_CL(L, D, H) reinterpret_cast<const void*>(fqb::fq_cl_kernel<L, D, H>)
  if (leaf == FQB200_LEAF_MIDTREAD) {
    if (hist) return dev ? FQB_CL(FQB200_LEAF_MIDTREAD, true, true) : FQB_CL(FQB200_LEAF_MIDTREAD, false, true);
    return dev ? FQB_CL(FQB200_LEAF_MIDTREAD, true, false) : FQB_CL(FQB200_LEAF_MIDTREAD, false, false);
  }
  if (hist) return dev ? FQB_CL(FQB200_LEAF_TORCH, true, true) : FQB_CL(FQB200_LEAF_TORCH, false, true);
  return dev ? FQB_CL(FQB200_LEAF_TORCH, true, false) : FQB_CL(FQB200_LEAF_TORCH, false, false);
#undef FQB_CL
}
size_t cl_smem(bool /*hist*/) {  // (the histogram variants borrow the last ring stage)
  return static_cast<size_t>(fqb::kStages) * fqb::kStageBytes + fqb::kClCombineBytes;
}
size_t cl_given_smem() { return static_cast<size_t>(fqb::kStages) * fqb::kStageBytes; }

struct DeviceInfo {
  int rc = FQB200_OK;      // result of the one-time initialisation
  char err[256] = "";
  int sms = 0;
  int resident = 0;        // CTAs of the cp.async-ring fused kernels (512 threads) that fit at once
  int resident_cl[2] = {0, 0};  // channels-last kernels without / with the histogram
  int resident_bca = 0;         // fq_cl_bca_kernel
  int resident_rows = 0;        // fq_rows_kernel
  int resident_angle[2] = {0, 0};  // fq_gram_partial_kernel<1>, <4>
};
constexpr int kMaxDevices = 64;
constexpr int kAssumedSms = 132;  // H100 SXM: the SM count plans assume when no device is present
DeviceInfo g_dev[kMaxDevices];
std::once_flag g_dev_once[kMaxDevices];

// dynamic shared memory of a launch: the cp.async ring of the 128-bit path
size_t dyn_smem(int vec) { return static_cast<size_t>(vec == 4 ? fqb::ring_bytes<4>() : fqb::ring_bytes<1>()); }

// the instantiations of the fused kernel: (mode 4 | 1 | 8) x (leaf 0..2) x (second statistics pass) x (weight correction;
// not for the bundled mode)
template <int MODE, int LEAF>
const void* fused_ptr2(bool dev, bool corr) {
  if constexpr (MODE == 8) {
    return dev ? reinterpret_cast<const void*>(fqb::fq_fused_kernel<8, LEAF, true, false>)
               : reinterpret_cast<const void*>(fqb::fq_fused_kernel<8, LEAF, false, false>);
  } else {
    if (dev) return corr ? reinterpret_cast<const void*>(fqb::fq_fused_kernel<MODE, LEAF, true, true>)
                         : reinterpret_cast<const void*>(fqb::fq_fused_kernel<MODE, LEAF, true, false>);
    return corr ? reinterpret_cast<const void*>(fqb::fq_fused_kernel<MODE, LEAF, false, true>)
                : reinterpret_cast<const void*>(fqb::fq_fused_kernel<MODE, LEAF, false, false>);
  }
}
template <int MODE>
const void* fused_ptr1(int leaf, bool dev, bool corr) {
  if (leaf == FQB200_LEAF_TORCH) return fused_ptr2<MODE, FQB200_LEAF_TORCH>(dev, corr);
  if (leaf == FQB200_LEAF_COMPILED) return fused_ptr2<MODE, FQB200_LEAF_COMPILED>(dev, corr);
  return fused_ptr2<MODE, FQB200_LEAF_MIDTREAD>(dev, corr);
}
const void* fused_kernel_ptr(int mode, int leaf, bool dev, bool corr) {
  if (mode == 4) return fused_ptr1<4>(leaf, dev, corr);
  if (mode == 8) return fused_ptr1<8>(leaf, dev, corr);
  return fused_ptr1<1>(leaf, dev, corr);
}

// optimum of 2*exp(-a) + a^2/(3 w^2): a*exp(a) = 3 w^2 (Lambert W), Newton in float64.  The reference gets the
// same numbers from scipy's Brent minimiser (int_quantizer.py:48) to ~1e-8.
double laplace_opt_alpha(double w) {
  const double c = 3.0 * w * w;
  double a = (c < 1.0) ? c : log(c);
  if (a <= 0) a = 1e-3;
  for (int i = 0; i < 100; ++i) {
    const double e = exp(a), f = a * e - c, fp = e * (a + 1.0);
    const double na = a - f / fp;
    if (fabs(na - a) <= 1e-16 * fabs(na)) {
      a = na;
      break;
    }
    a = na;
  }
  return a;
}

// KLD kernels (fq_kld.cuh): shared-memory histogram replicas, and the dynamic shared memory of the histogram and search
// kernels
constexpr int kKldMaxBins = 8001;
int kld_replicas(int num_bins) {
  const int rep = 65536 / (num_bins * 4);
  return rep < 1 ? 1 : (rep > fqb::kKldMaxReplicas ? fqb::kKldMaxReplicas : rep);
}
size_t kld_hist_smem(int num_bins) { return static_cast<size_t>(kld_replicas(num_bins) + 1) * num_bins * 4 + 4; }
size_t kld_search_smem(int num_bins) {
  return static_cast<size_t>((2 * (num_bins + 1) + 1) & ~1) * 4 + static_cast<size_t>(num_bins / 2 + 1) * 8;
}

size_t kmeans_smem(int k) {
  const size_t stage = static_cast<size_t>(fqb::kKmMaxT) * fqb::kKmBlk * 8;
  const size_t acc = static_cast<size_t>(fqb::kWarps) * k * 12;
  const size_t tot = static_cast<size_t>(fqb::kThreads) * 16;
  return stage > acc ? (stage > tot ? stage : tot) : (acc > tot ? acc : tot);
}

// One-time, per-device set-up (kernel attributes, occupancy, constant tables).  Runs under std::call_once: the reference's
// callers include torch.nn.DataParallel worker threads, one per device (SURVEY 8b).
void init_device(int dev) {
  DeviceInfo& d = g_dev[dev];
  auto bad = [&](const char* what, cudaError_t e) {
    d.rc = FQB200_ERR_CUDA;
    snprintf(d.err, sizeof(d.err), "%s: %s", what, cudaGetErrorString(e));
  };
  int sms = 0, per_sm = 1 << 20;
  cudaError_t e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (e != cudaSuccess) return bad("cudaDeviceGetAttribute", e);
  const int modes[3] = {4, 1, 8};
  for (int mi = 0; mi < 3; ++mi)
    for (int leaf = 0; leaf < 3; ++leaf)
      for (int dv = 0; dv < 2; ++dv)
        for (int cr = 0; cr < 2; ++cr) {
          if (modes[mi] == 8 && cr) continue;
          int n = 0;
          e = setup(fused_kernel_ptr(modes[mi], leaf, dv != 0, cr != 0), fqb::kThreads, dyn_smem(modes[mi] == 1 ? 1 : 4), &n);
          if (e != cudaSuccess) return bad("fused kernel setup", e);
          if (n < per_sm) per_sm = n;
        }
  {
    int n = 0;
    e = setup(fqb::fq_fused_kernel<4, FQB200_LEAF_COMPILED, false, false, true>, fqb::kThreads, dyn_smem(4), &n);
    if (e != cudaSuccess) return bad("bias-period kernel setup", e);
    if (n < per_sm) per_sm = n;
  }
  if (per_sm < 1) {
    d.rc = FQB200_ERR_CUDA;
    snprintf(d.err, sizeof(d.err), "fused kernel does not fit on an SM");
    return;
  }
  for (int hist = 0; hist < 2; ++hist) {
    int worst = 1 << 20;
    for (int leaf = 0; leaf < 3; leaf += 2)
      for (int dv = 0; dv < 2; ++dv) {
        int n = 0;
        e = setup(cl_kernel_ptr(leaf, dv != 0, hist != 0), fqb::kBulkThreads, cl_smem(hist != 0), &n);
        if (e != cudaSuccess && hist) {  // the histogram variant may not fit next to an enlarged ring (development builds)
          (void)cudaGetLastError();
          n = 0;
          e = cudaSuccess;
        }
        if (e != cudaSuccess) return bad("channels-last kernel setup", e);
        if (n < worst) worst = n;
      }
    if (worst < 1 && hist) {
      d.resident_cl[1] = 0;
      continue;
    }
    if (worst < 1) {
      d.rc = FQB200_ERR_CUDA;
      snprintf(d.err, sizeof(d.err), "channels-last kernel does not fit on an SM");
      return;
    }
    d.resident_cl[hist] = sms * worst;
  }
  int n = 0;
  e = setup(fqb::fq_cl_bca_kernel, fqb::kBulkThreads, cl_smem(false), &n);
  if (e != cudaSuccess || n < 1) return bad("bias-correction kernel setup", e);
  d.resident_bca = sms * n;
  e = setup(fqb::fq_rows_kernel, fqb::kBulkThreads, cl_given_smem(), &n);
  if (e != cudaSuccess || n < 1) return bad("row kernel setup", e);
  d.resident_rows = sms * n;
  for (int v = 0; v < 2; ++v) {
    e = setup(v ? fqb::fq_gram_partial_kernel<4> : fqb::fq_gram_partial_kernel<1>, fqb::kAngThreads, fqb::kAngSmemBytes, &n);
    if (e != cudaSuccess || n < 1) return bad("Gram kernel setup", e);
    d.resident_angle[v] = sms * n;
  }
  if ((e = setup(fqb::fq_given_kernel<4, FQB200_LEAF_TORCH, false>, fqb::kThreads, dyn_smem(4))) != cudaSuccess ||
      (e = setup(fqb::fq_given_kernel<4, FQB200_LEAF_TORCH, true>, fqb::kThreads, dyn_smem(4))) != cudaSuccess ||
      (e = setup(fqb::fq_cl_given_kernel<false>, fqb::kBulkThreads, cl_given_smem())) != cudaSuccess ||
      (e = setup(fqb::fq_cl_given_kernel<true>, fqb::kBulkThreads, cl_given_smem())) != cudaSuccess)
    return bad("given-parameter kernel setup", e);
  e = setup(fqb::fq_cl_given_fused_kernel, fqb::kBulkThreads, cl_given_smem());
  if (e != cudaSuccess) return bad("given-parameter fused kernel setup", e);
  if ((e = setup(fqb::fq_leaf_bulk_kernel<false>, fqb::kBulkThreads, cl_given_smem())) != cudaSuccess ||
      (e = setup(fqb::fq_leaf_bulk_kernel<true>, fqb::kBulkThreads, cl_given_smem())) != cudaSuccess)
    return bad("a1 bulk kernel setup", e);
  // the KLD and k-means launches size their shared memory by argument: allow the largest any accepted argument needs
  if ((e = setup(fqb::fq_kld_hist_kernel<1>, fqb::kKldThreads, kld_hist_smem(kKldMaxBins))) != cudaSuccess ||
      (e = setup(fqb::fq_kld_hist_kernel<4>, fqb::kKldThreads, kld_hist_smem(kKldMaxBins))) != cudaSuccess ||
      (e = setup(fqb::fq_kld_search_kernel, fqb::kKldThreads, kld_search_smem(kKldMaxBins))) != cudaSuccess)
    return bad("KLD kernel setup", e);
  e = setup(fqb::fq_kmeans_kernel, fqb::kThreads, kmeans_smem(fqb::kKmMaxK));
  if (e != cudaSuccess) return bad("k-means kernel setup", e);
  if ((e = setup(fqb::fq_clipmse_partial_kernel<0>, fqb::kCmThreads, fqb::cm_smem_bytes(fqb::kCmMaxK, 1))) != cudaSuccess ||
      (e = setup(fqb::fq_clipmse_partial_kernel<1>, fqb::kCmThreads, fqb::cm_smem_bytes(fqb::kCmMaxK, 1))) != cudaSuccess ||
      (e = setup(fqb::fq_clipmse_partial_kernel<2>, fqb::kCmThreads, fqb::cm_smem_bytes(fqb::kCmMaxK, fqb::kCmSlab))) != cudaSuccess)
    return bad("clipping-MSE kernel setup", e);
  // mid-tread table (int_quantizer.py:41-51): omega grid = 5 decades x 20 steps, leading 0
  double om[fqb::kTable], al[fqb::kTable];
  om[0] = 0.0;
  al[0] = 0.0;
  const double lo[5] = {0.01, 0.1, 1, 10, 100}, hi[5] = {0.1, 1, 10, 100, 1000};
  for (int dcd = 0; dcd < 5; ++dcd)
    for (int k = 0; k < 20; ++k) {
      const double w = lo[dcd] + (hi[dcd] - lo[dcd]) * k / 20.0;
      om[1 + dcd * 20 + k] = w;
      al[1 + dcd * 20 + k] = laplace_opt_alpha(w);
    }
  e = cudaMemcpyToSymbol(fqb::kOmegaTable, om, sizeof(om));
  if (e == cudaSuccess) e = cudaMemcpyToSymbol(fqb::kAlphaTable, al, sizeof(al));
  if (e != cudaSuccess) return bad("table upload", e);
  d.sms = sms;
  d.resident = sms * per_sm;
}

int get_device(DeviceInfo** out) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return fail(FQB200_ERR_CUDA, "cudaGetDevice: %s", cudaGetErrorString(e));
  if (dev < 0 || dev >= kMaxDevices) return fail(FQB200_ERR_UNSUPPORTED, "device index out of range%s");
  std::call_once(g_dev_once[dev], init_device, dev);
  DeviceInfo& d = g_dev[dev];
  if (d.rc != FQB200_OK) return fail(d.rc, "device set-up failed: %s", d.err);
  *out = &d;
  return FQB200_OK;
}

struct Plan {
  fqb::Geometry geo;
  fqb::FlatGeo flat;
  int vec;   // 4 or 1: floats per access
  int mode;  // 4, 1, 8 (bundled 128-bit path) or 2 (flat stream on the bulk-copy engine)
  int grid;
};

constexpr uint64_t kUnitsPerCta = 8;  // dynamic work units per resident CTA

// Choose the access mode (128-bit, bundled 128-bit, scalar), the number of parts per group (unit size) and the grid
// size; fill the geometry.
int make_plan(int64_t outer, int64_t groups, int64_t inner, bool can_vec, bool allow_bundle, int max_ctas, Plan* pl) {
  if (outer <= 0 || groups <= 0 || inner <= 0) return fail(FQB200_ERR_INVALID, "non-positive tensor extent%s");
  if (groups > 0x3fffffffLL || outer > 0x7fffffffLL || inner > 0x7fffffffLL * 4LL)
    return fail(FQB200_ERR_UNSUPPORTED, "tensor extent exceeds 2^31%s");
  int vec = (can_vec && inner % 4 == 0) ? 4 : 1;
  int mode = vec;
  uint64_t bundle = 1;
  if (vec == 1 && can_vec && allow_bundle && inner >= 4) {
    const uint64_t b = (inner % 2 == 0) ? 2 : 4;
    const uint64_t row_v = b * static_cast<uint64_t>(inner) / 4;
    if (groups % b == 0 && row_v <= static_cast<uint64_t>(fqb::kThreads)) {
      bundle = b;
      vec = 4;
      mode = 8;
    }
  }
  const uint64_t G = static_cast<uint64_t>(groups) / bundle;                // streaming groups
  const uint64_t inner_v = bundle * static_cast<uint64_t>(inner) / vec;       // vectors per streaming-group row
  if (inner_v > 0xffffffffULL) return fail(FQB200_ERR_UNSUPPORTED, "row too long%s");
  const uint64_t stride = (mode == 8) ? (fqb::kThreads / inner_v) * inner_v : fqb::kThreads;
  const uint64_t group_v = static_cast<uint64_t>(outer) * inner_v;
  const uint64_t total_v = group_v * G;
  if (total_v >= (1ULL << 32)) return fail(FQB200_ERR_UNSUPPORTED, "tensors of 2^32 vectors (64 GB) and more are not supported%s");
  const uint64_t ctas = static_cast<uint64_t>(max_ctas);
  // Units: about kUnitsPerCta per CTA so that dynamic assignment can even out the CTAs' unequal speeds, but no
  // smaller than one full ring (kRingDepth sweeps of the CTA) when the group allows it.
  const uint64_t min_unit_v = static_cast<uint64_t>(fqb::kRingDepth) * stride;
  uint64_t parts = (kUnitsPerCta * ctas + G - 1) / G;
  const uint64_t max_parts = group_v / min_unit_v > 0 ? group_v / min_unit_v : 1;
  if (parts > max_parts) parts = max_parts;
  if (parts < 1) parts = 1;
  while ((group_v + parts - 1) / parts >= 0x7fffffffULL) ++parts;  // unit lengths are 32-bit
  uint64_t part_v = (group_v + parts - 1) / parts;
  if (mode == 8) part_v = (part_v + inner_v - 1) / inner_v * inner_v;  // whole rows: every thread keeps its column
  parts = (group_v + part_v - 1) / part_v;  // no empty trailing part
  if (parts * G >= 0xfffffff0ULL) return fail(FQB200_ERR_UNSUPPORTED, "too many work units%s");
  const uint64_t units = parts * G;
  // leader reductions: cover all channels in one sweep when possible (kThreads / lanes >= channels), never more lanes than parts
  unsigned lanes = 32;
  while (lanes > 1 && (static_cast<uint64_t>(fqb::kThreads / lanes) < static_cast<uint64_t>(groups) || (lanes >> 1) >= parts)) lanes >>= 1;
  fqb::Geometry& g = pl->geo;
  g.groups = static_cast<unsigned>(G);
  g.channels = static_cast<unsigned>(groups);
  g.bundle = static_cast<unsigned>(bundle);
  g.stride = static_cast<unsigned>(stride);
  g.parts = static_cast<unsigned>(parts);
  g.units = static_cast<unsigned>(units);
  g.inner_v = static_cast<unsigned>(inner_v);
  g.step_q = static_cast<unsigned>(stride / inner_v);
  g.step_r = static_cast<unsigned>(stride % inner_v);
  g.red_lanes = lanes;
  g.part_v = static_cast<unsigned>(part_v);
  g.group_v = group_v;
  g.row_pitch = G * inner_v;
  pl->vec = vec;
  pl->mode = mode;
  pl->grid = grid_for(units, ctas);
  return FQB200_OK;
}

// flat-stream plan (bulk-copy engine): `elems` contiguous floats, channel period `channels` (0: no per-channel state).
// A stage is kStageVec * stride vectors with stride the largest multiple of channels/4 that fits in the 512 consumer
// threads, so that a thread always sees the same four channels; units are runs of stages, about kUnitsPerCta per CTA.
bool flat_eligible(int64_t channels) { return channels % 4 == 0 && channels / 4 >= 1 && channels / 4 <= fqb::kConsumers; }

int make_plan_flat(uint64_t elems, int64_t channels, int max_ctas, Plan* pl) {
  if (elems == 0 || elems % 4 != 0) return fail(FQB200_ERR_UNSUPPORTED, "flat stream needs a multiple of 4 elements%s");
  const uint64_t total_v = elems / 4;
  if (total_v >= (1ULL << 32)) return fail(FQB200_ERR_UNSUPPORTED, "tensors of 2^32 vectors (64 GB) and more are not supported%s");
  const uint64_t cv = channels > 0 ? static_cast<uint64_t>(channels) / 4 : 1;
  if (channels > 0 && !flat_eligible(channels)) return fail(FQB200_ERR_UNSUPPORTED, "channels-last needs C %% 4 == 0 and C <= 2048%s");
  const uint64_t stride = (fqb::kConsumers / cv) * cv;
  const uint64_t stage_v = static_cast<uint64_t>(fqb::kStageVec) * stride;
  const uint64_t n_stages = (total_v + stage_v - 1) / stage_v;
  const uint64_t ctas = static_cast<uint64_t>(max_ctas);
  uint64_t unit_stages = n_stages / (kUnitsPerCta * ctas);
  if (unit_stages < 2) unit_stages = 2;   // a ticket (one atomic round trip) per >= 32 KB
  if (unit_stages > 64) unit_stages = 64;
  const uint64_t units = (n_stages + unit_stages - 1) / unit_stages;
  fqb::FlatGeo& g = pl->flat;
  g.total_v = static_cast<unsigned>(total_v);
  g.stride = static_cast<unsigned>(stride);
  g.stage_v = static_cast<unsigned>(stage_v);
  g.n_stages = static_cast<unsigned>(n_stages);
  g.unit_stages = static_cast<unsigned>(unit_stages);
  g.units = static_cast<unsigned>(units);
  g.channels = static_cast<unsigned>(channels > 0 ? channels : 0);
  g.cv = static_cast<unsigned>(cv);
  memset(&pl->geo, 0, sizeof(pl->geo));
  pl->geo.channels = g.channels;  // solve_bit_alloc reads the channel count here
  pl->vec = 4;
  pl->mode = 2;
  pl->grid = grid_for(units, ctas);
  return FQB200_OK;
}

// row-structured plan (fq_rows_kernel): `rows` rows of `row_elems` contiguous floats; channel period `channels` as in
// make_plan_flat (0: none).  Units are runs of stages inside one row.
int make_plan_rows(uint64_t rows, uint64_t row_elems, int64_t channels, int max_ctas, Plan* pl, fqb::RowsGeo* rg) {
  if (rows == 0 || row_elems == 0 || row_elems % 4 != 0 || rows > fqb::kMaxNhwcChannels)
    return fail(FQB200_ERR_UNSUPPORTED, "row stream needs rows <= 4096 of a multiple of 4 elements%s");
  const uint64_t row_v = row_elems / 4;
  if (rows * row_v >= (1ULL << 32)) return fail(FQB200_ERR_UNSUPPORTED, "tensors of 2^32 vectors (64 GB) and more are not supported%s");
  const uint64_t cv = channels > 0 ? static_cast<uint64_t>(channels) / 4 : 1;
  if (channels > 0 && (!flat_eligible(channels) || row_v % cv != 0)) return fail(FQB200_ERR_UNSUPPORTED, "bias period does not fit the rows%s");
  const uint64_t stride = (fqb::kConsumers / cv) * cv;
  const uint64_t stage_v = static_cast<uint64_t>(fqb::kStageVec) * stride;
  const uint64_t spr = (row_v + stage_v - 1) / stage_v;
  const uint64_t ctas = static_cast<uint64_t>(max_ctas);
  uint64_t unit_stages = rows * spr / (kUnitsPerCta * ctas);
  if (unit_stages < 1) unit_stages = 1;
  if (unit_stages > 64) unit_stages = 64;
  if (unit_stages > spr) unit_stages = spr;
  const uint64_t upr = (spr + unit_stages - 1) / unit_stages;
  const uint64_t units = rows * upr;
  if (units >= 0xfffffff0ULL) return fail(FQB200_ERR_UNSUPPORTED, "too many work units%s");
  fqb::FlatGeo& g = pl->flat;
  g.total_v = static_cast<unsigned>(rows * row_v);
  g.stride = static_cast<unsigned>(stride);
  g.stage_v = static_cast<unsigned>(stage_v);
  g.n_stages = static_cast<unsigned>(rows * spr);
  g.unit_stages = static_cast<unsigned>(unit_stages);
  g.units = static_cast<unsigned>(units);
  g.channels = static_cast<unsigned>(channels > 0 ? channels : 0);
  g.cv = static_cast<unsigned>(cv);
  rg->rows = static_cast<unsigned>(rows);
  rg->row_v = static_cast<unsigned>(row_v);
  rg->stages_per_row = static_cast<unsigned>(spr);
  rg->units_per_row = static_cast<unsigned>(upr);
  memset(&pl->geo, 0, sizeof(pl->geo));
  pl->geo.channels = static_cast<unsigned>(rows);
  pl->vec = 4;
  pl->mode = 3;
  pl->grid = grid_for(units, ctas);
  return FQB200_OK;
}

// what fq_rows_kernel takes: one min/max parameter set from per-row (per-sample) statistics, compiled-leaf arithmetic
bool rows_supported(const fqb200_desc* d, bool can_vec) {
  if (d->leaf != FQB200_LEAF_COMPILED || d->range_mode != FQB200_RANGE_MINMAX || d->bias_corr || d->var_corr || d->channels_last ||
      d->out_hist || !can_vec || d->outer != 1 || d->inner % 4 != 0 || d->groups > static_cast<int64_t>(fqb::kMaxNhwcChannels))
    return false;
  if (!(d->scope == FQB200_SCOPE_GROUP_MEAN || d->scope == FQB200_SCOPE_TENSOR || d->groups == 1)) return false;
  if (d->bias) {  // only the channel-fastest form (bias_period = -C): a per-thread constant
    if (d->bias_period >= 0) return false;
    const int64_t c = -d->bias_period;
    if (!flat_eligible(c) || d->inner % c != 0) return false;
  }
  return true;
}

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// KLD workspace: [rows] max |x| words, then [rows][num_bins] bin counters (fq_kld.cuh)
size_t kld_workspace(int64_t rows, int num_bins) {
  return align_up(static_cast<size_t>(rows) * 4, 256) + static_cast<size_t>(rows) * static_cast<size_t>(num_bins) * 4;
}

// per-sample sums workspace: `sums` float64 partials per (row, chunk) unit when a row spans several chunks
// (fq_sample_sums.cuh)
size_t sums_workspace(int64_t rows, int64_t row_len, int sums) {
  const unsigned long long chunk = fqb::sums_chunk(static_cast<unsigned long long>(row_len));
  const unsigned long long chunks = (static_cast<unsigned long long>(row_len) + chunk - 1) / chunk;
  return chunks > 1 ? static_cast<size_t>(rows) * static_cast<size_t>(chunks) * static_cast<size_t>(sums) * 8 : 0;
}

// fq_sums_partial_kernel<VEC, S, BIAS>, then, when a row spans several chunks, fq_sums_finish_kernel<S>: the per-sample
// sums of sum set S (1, 2 or 7) over rows x row_len; `what` names the launch in an error message
template <int S>
int launch_sums(const float* y, const float* q, const float* bias, int64_t bias_period, int64_t rows, int64_t row_len,
                double* out, void* workspace, int32_t max_ctas, void* stream, const char* what) {
  using namespace fqb;
  DeviceInfo* di = nullptr;
  const int rc = get_device(&di);
  if (rc != FQB200_OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  SumsArgs A;
  memset(&A, 0, sizeof(A));
  A.y = y;
  A.q = q;
  A.bias = bias;
  A.period = static_cast<unsigned>(bias_period < 0 ? 0ull - static_cast<unsigned long long>(bias_period)
                                                   : static_cast<unsigned long long>(bias_period));
  A.rows = static_cast<unsigned long long>(rows);
  A.row_len = static_cast<unsigned long long>(row_len);
  A.chunk = sums_chunk(A.row_len);
  A.chunks = (A.row_len + A.chunk - 1) / A.chunk;
  A.partial = static_cast<double*>(workspace);
  A.out = out;
  const int grid = grid_for(A.rows * A.chunks, di->sms * (2048ull / kSumsThreads), max_ctas);
  const bool vec = row_len % 4 == 0 && aligned16(y) && (!q || aligned16(q));
#define FQB_LAUNCH_SUMS(B)                                                          \
  do {                                                                              \
    if (vec) fq_sums_partial_kernel<4, S, B><<<grid, kSumsThreads, 0, st>>>(A);     \
    else     fq_sums_partial_kernel<1, S, B><<<grid, kSumsThreads, 0, st>>>(A);     \
  } while (0)
  if constexpr (S == 1) FQB_LAUNCH_SUMS(kSumsBiasNone);   // the activation norm takes no bias
  else if (!bias) FQB_LAUNCH_SUMS(kSumsBiasNone);
  else if (bias_period > 0) FQB_LAUNCH_SUMS(kSumsBiasNchw);
  else FQB_LAUNCH_SUMS(kSumsBiasCl);
#undef FQB_LAUNCH_SUMS
  if (A.chunks > 1) {
    const unsigned long long blocks = (A.rows * S + kSumsThreads - 1) / kSumsThreads;
    fq_sums_finish_kernel<S><<<static_cast<unsigned>(blocks), kSumsThreads, 0, st>>>(A);
  }
  return launched(what);
}

// sample-angle workspace: one 64 x 64 float64 block per (tile pair, slice) unit (fq_angle.cuh)
size_t angle_workspace(int64_t rows, int64_t row_len) {
  const fqb::AngleSplit s = fqb::angle_split(static_cast<unsigned long long>(rows), static_cast<unsigned long long>(row_len));
  return static_cast<size_t>(s.pairs * s.slices) * fqb::kAngTile * fqb::kAngTile * 8;
}

// clipping-error workspace: kCeSums float64 partials per (group, unit) (fq_cliperr.cuh)
unsigned long long cliperr_units_per_group(int64_t outer, int64_t inner, int channels_last) {
  const unsigned long long n = static_cast<unsigned long long>(outer) * static_cast<unsigned long long>(inner);
  const unsigned long long per = channels_last ? fqb::kCeClRows : fqb::kCeChunk;
  return (n + per - 1) / per;
}
size_t cliperr_workspace(int64_t outer, int64_t groups, int64_t inner, int channels_last) {
  return static_cast<size_t>(groups) * static_cast<size_t>(cliperr_units_per_group(outer, inner, channels_last)) * fqb::kCeSums * 8;
}

// clipping-MSE workspace: k + 1 float64 partials per (group, chunk), k = nw * K candidates (fq_clipmse.cuh)
unsigned long long clipmse_units_per_group(int64_t outer, int64_t inner, int channels_last) {
  const unsigned long long n = static_cast<unsigned long long>(outer) * static_cast<unsigned long long>(inner);
  const unsigned long long per = channels_last ? fqb::kCmClRows : fqb::kCmChunk;
  return (n + per - 1) / per;
}
size_t clipmse_workspace(int64_t outer, int64_t groups, int64_t inner, int channels_last, int k) {
  return static_cast<size_t>(groups) * static_cast<size_t>(clipmse_units_per_group(outer, inner, channels_last)) *
         static_cast<size_t>(k + 1) * 8;
}

// k-means workspace (fq_kmeans.cuh): barrier words, control block, per-block / per-superblock column sums, Lloyd unit
// partials, relocation candidates.  Fills A's pointers when base != nullptr.
size_t kmeans_carve(char* base, unsigned long long n, int k, fqb::KmArgs* A) {
  const unsigned long long nb = (n + fqb::kKmBlk - 1) / fqb::kKmBlk, nsb = (nb + fqb::kKmSuper - 1) / fqb::kKmSuper;
  const unsigned long long per = fqb::kWarps * ((nb + fqb::kWarps * fqb::kKmMaxUnits - 1) / (fqb::kWarps * fqb::kKmMaxUnits));
  const unsigned long long units = (nb + per - 1) / per;
  size_t off = 0;
  auto take = [&](size_t bytes) {
    char* p = base ? base + off : nullptr;
    off = align_up(off + bytes, 256);
    return p;
  };
  char* sync = take(sizeof(fqb::GridSync));
  char* ctrl = take(sizeof(fqb::KmCtrl));
  char* col = take(static_cast<size_t>(fqb::kKmMaxT) * nb * 8);
  char* sup = take(static_cast<size_t>(fqb::kKmMaxT) * nsb * 8);
  char* usum = take(static_cast<size_t>(units) * k * 8);
  char* ucnt = take(static_cast<size_t>(units) * k * 4);
  char* rbd = take(static_cast<size_t>(nb) * 8);
  char* rbi = take(static_cast<size_t>(nb) * 8);
  char* far = take(static_cast<size_t>(k) * 8);
  if (A) {
    A->n = n; A->nb = nb; A->nsb = nsb; A->k = k;
    A->unit_blocks = per; A->units = units;
    A->sync = reinterpret_cast<fqb::GridSync*>(sync);
    A->ctrl = reinterpret_cast<fqb::KmCtrl*>(ctrl);
    A->col = reinterpret_cast<double*>(col);
    A->sup = reinterpret_cast<double*>(sup);
    A->usum = reinterpret_cast<double*>(usum);
    A->ucnt = reinterpret_cast<unsigned*>(ucnt);
    A->rbd = reinterpret_cast<double*>(rbd);
    A->rbi = reinterpret_cast<long long*>(rbi);
    A->far = reinterpret_cast<long long*>(far);
  }
  return off;
}
// workspace layout; returns total bytes, fills pointers when base != nullptr.  Partials: one slot per unit.
size_t carve(char* base, uint64_t slots, uint64_t groups, fqb::FusedArgs* A) {
  size_t off = 0;
  auto take = [&](size_t bytes) {
    char* p = base ? base + off : nullptr;
    off = align_up(off + bytes, 256);
    return p;
  };
  char* sync = take(sizeof(fqb::GridSync));
  // channels-last accumulators, two banks (fq_cl.cuh): fixed place and size, zero between launches
  char* acc_u = take(2 * fqb::kAccU * sizeof(unsigned));
  char* acc_d = take(2 * fqb::kAccD * sizeof(double));
  char* pmin = take(slots * sizeof(float));
  char* pmax = take(slots * sizeof(float));
  char* psum = take((slots + 2 * groups) * sizeof(double));
  char* pabs = take((slots + 2 * groups) * sizeof(double));
  char* psq = take((slots + 2 * groups) * sizeof(double));
  char* gf = take(groups * sizeof(float) * 12);
  char* gd = take(groups * sizeof(double));
  char* lp = take(groups * sizeof(fqb::LeafParam));
  if (A) {
    A->sync = reinterpret_cast<fqb::GridSync*>(sync);
    A->pmin = reinterpret_cast<float*>(pmin);
    A->pmax = reinterpret_cast<float*>(pmax);
    A->psum = reinterpret_cast<double*>(psum);
    A->pabs = reinterpret_cast<double*>(pabs);
    A->psq = reinterpret_cast<double*>(psq);
    float* f = reinterpret_cast<float*>(gf);
    A->gmin = f + 0 * groups;
    A->gmax = f + 1 * groups;
    A->gmean = f + 2 * groups;
    A->gb = f + 3 * groups;
    A->gstd = f + 4 * groups;
    A->gbits = f + 5 * groups;
    A->gprior = f + 6 * groups;
    A->gdelta = f + 7 * groups;
    A->goffset = f + 8 * groups;
    A->cq = f + 9 * groups;
    A->co = f + 10 * groups;
    A->ck = f + 11 * groups;
    A->gmean_d = reinterpret_cast<double*>(gd);
    A->lp = reinterpret_cast<fqb::LeafParam*>(lp);
    A->amin_inv = reinterpret_cast<unsigned*>(acc_u);  // bank 0; bank b at + b * kAccU (fq_cl.cuh: cl_view)
    A->amax = nullptr;
    A->asum = reinterpret_cast<double*>(acc_d);        // bank 0; bank b at + b * kAccD
    A->aabs = nullptr;
    A->asq = nullptr;
  }
  return off;
}

int check_desc(const fqb200_desc* d) {
  if (!d) return fail(FQB200_ERR_INVALID, "null descriptor%s");
  if (d->scope < FQB200_SCOPE_GROUP || d->scope > FQB200_SCOPE_TENSOR) return fail(FQB200_ERR_INVALID, "bad scope%s");
  if (d->range_mode < FQB200_RANGE_MINMAX || d->range_mode > FQB200_RANGE_GIVEN) return fail(FQB200_ERR_INVALID, "bad range_mode%s");
  if (d->range_mode == FQB200_RANGE_GIVEN &&
      (!d->channels_last || d->leaf != FQB200_LEAF_TORCH || d->scope != FQB200_SCOPE_GROUP || d->stats_only || d->out_stats || d->out_hist ||
       d->bias_corr || d->var_corr || d->bit_alloc || !d->given_delta || !d->given_offset))
    return fail(FQB200_ERR_UNSUPPORTED, "RANGE_GIVEN: channels_last, torch leaf, scope GROUP, given_delta / given_offset, no statistics outputs%s");
  if (d->leaf < FQB200_LEAF_TORCH || d->leaf > FQB200_LEAF_MIDTREAD) return fail(FQB200_ERR_INVALID, "bad leaf%s");
  if (d->leaf != FQB200_LEAF_MIDTREAD && (d->num_bits < 1 || d->num_bits > 8))
    return fail(FQB200_ERR_INVALID, "num_bits must be in 1..8%s");
  if (d->scope != FQB200_SCOPE_GROUP && (d->range_mode != FQB200_RANGE_MINMAX || d->leaf == FQB200_LEAF_MIDTREAD))
    return fail(FQB200_ERR_UNSUPPORTED, "group-mean / tensor scopes are defined for min/max ranges only%s");
  if (d->bit_alloc && !(d->bit_alloc_target > 0.f)) return fail(FQB200_ERR_INVALID, "bit_alloc_target must be > 0%s");
  if ((d->bias_corr || d->var_corr) && d->scope == FQB200_SCOPE_GROUP_MEAN)
    return fail(FQB200_ERR_UNSUPPORTED, "weight correction is per row (scope GROUP or TENSOR)%s");
  return FQB200_OK;
}

// Widest pooling tile (pixels) whose row pieces fit a ring stage, 0 if none.  2x2: a tile is 2 rows x wt input pixels,
// two row pieces in the two halves of a stage, (wt / 2) * cv output vectors.  3x3: a tile is 1 output row x wt output
// pixels, three row pieces of 2 * wt + 1 input pixels in three regions of a stage.
unsigned pool_tile_width(int kind, int64_t w, const fqb::FlatGeo& f) {
  const unsigned cv = f.cv, stage_v = fqb::kStageVec * fqb::kConsumers;
  if (kind == 2) {
    for (int64_t cand = w; cand >= 2; cand -= 2)
      if (w % cand == 0 && static_cast<uint64_t>(cand) * cv <= stage_v / 2u && static_cast<uint64_t>(cand / 2) * cv <= f.stride)
        return static_cast<unsigned>(cand);
  } else {
    const int64_t ow = w / 2;
    for (int64_t cand = ow; cand >= 1; --cand)
      if (ow % cand == 0 && 3ull * static_cast<uint64_t>(2 * cand + 1) * cv <= stage_v && static_cast<uint64_t>(cand) * cv <= f.stride)
        return static_cast<unsigned>(cand);
  }
  return 0;
}

// The channel count C of a launch whose apply phase can write a channel slice of a wider channels-last tensor: a
// channels-last launch's groups, or the period of the channel-fastest bias (bias_period = -C) of a per-sample / per-tensor
// min-max launch, which reads channels-last memory as rows of samples and learns C from that bias as its in-launch pooling
// does.  0: the launch cannot write a slice.
int64_t slice_channels(const fqb200_desc* d) {
  if (d->channels_last) return d->groups;
  if (d->bias && d->bias_period < 0 && rows_supported(d, true)) return -d->bias_period;
  return 0;
}

// What a pitched `out` (fqb200_fused_into, `pitch` floats between two pixels) needs beyond the descriptor's own route: the
// apply phase of a launch with a slice_channels() C, without pooling / residual, is the only store that can skip the other
// channels of a pixel; a 16-byte aligned `out` (`can_vec`); and 32-bit vector offsets.  No CUDA calls: fqb200_fused_into
// checks it before any device call, plan_fused again for the plan it makes.
int pitch_rules(const fqb200_desc* d, bool can_vec, int64_t pitch) {
  const int64_t c = slice_channels(d);
  if (!c || d->stats_only || d->pool || d->residual)
    return fail(FQB200_ERR_UNSUPPORTED, "out_pixel_stride: channels-last apply launches, or per-sample / per-tensor min-max apply "
                                        "launches with a channel-fastest bias, without pooling / residual only%s");
  if (pitch < c || pitch % 4 != 0)
    return fail(FQB200_ERR_UNSUPPORTED, "out_pixel_stride must be >= C and a multiple of 4%s");
  if (!can_vec) return fail(FQB200_ERR_UNSUPPORTED, "out_pixel_stride needs 16-byte aligned tensors%s");
  const uint64_t pixels = static_cast<uint64_t>(d->outer) * static_cast<uint64_t>(d->groups) * static_cast<uint64_t>(d->inner) /
                          static_cast<uint64_t>(c);
  if (pixels * static_cast<uint64_t>(pitch) / 4 >= (1ull << 32))
    return fail(FQB200_ERR_UNSUPPORTED, "out_pixel_stride: outputs of 2^32 vectors and more are not supported%s");
  return FQB200_OK;
}

// One fqb200_fused launch: route, geometry, kernel and its arguments, all but in / out and the workspace pointers.
struct FusedPlan {
  Plan pl;                    // mode 2: channels-last flat stream, 3: rows, 4 / 1 / 8: fq_fused_kernel
  fqb::FusedArgs A;
  uint64_t slots;             // per-unit partial slots in the workspace
  size_t workspace;           // bytes the launch needs (0: none)
  const void* kernel;
  unsigned block;
  size_t smem;
  bool coop;
  const char* name;
};

// The single place where a fused descriptor's route is decided and refused.  `d` passed check_desc; `can_vec`: in / out
// are 16-byte aligned; `out_pitch`: floats between two pixels of `out` when it is a channel slice of a wider channels-last
// tensor (fqb200_fused_into), 0 when `out` is dense; `r` holds the resident-CTA counts the grids are sized for.  No CUDA calls.
int plan_fused(const fqb200_desc* d, bool can_vec, int64_t out_pitch, const DeviceInfo& r, FusedPlan* fp) {
  memset(fp, 0, sizeof(*fp));
  Plan& pl = fp->pl;
  fqb::FusedArgs& A = fp->A;
  if (d->outer <= 0 || d->groups <= 0 || d->inner <= 0) return fail(FQB200_ERR_INVALID, "non-positive tensor extent%s");
  if (d->bias && d->bias_period == 0 && d->scope == FQB200_SCOPE_GROUP_MEAN)
    return fail(FQB200_ERR_UNSUPPORTED, "a per-group bias needs groups = channels (scope GROUP or TENSOR); use bias_period%s");
  const bool given = d->range_mode == FQB200_RANGE_GIVEN;
  int rc;
  if (d->channels_last) {
    // what the channels-last kernel can take (everything else with channels_last set is an error: the caller re-lays out)
    if (!can_vec || d->scope != FQB200_SCOPE_GROUP || d->leaf == FQB200_LEAF_COMPILED || d->bias_corr || d->var_corr ||
        d->bias_period > 0 || !flat_eligible(d->groups))
      return fail(FQB200_ERR_UNSUPPORTED, "channels_last: per-channel torch / mid-tread leaves on 16-byte aligned tensors, C %% 4 == 0, C <= 2048%s");
    rc = make_plan_flat(static_cast<uint64_t>(d->outer) * d->groups * d->inner, d->groups,
                        given ? r.resident_cl[0] * 2 : r.resident_cl[d->out_hist ? 1 : 0], &pl);
  } else if (rows_supported(d, can_vec)) {
    rc = make_plan_rows(static_cast<uint64_t>(d->groups), static_cast<uint64_t>(d->inner), d->bias ? -d->bias_period : 0,
                        r.resident_rows, &pl, &A.rows);
  } else if (d->bias && d->bias_period < 0) {
    return fail(FQB200_ERR_UNSUPPORTED, "a channel-fastest bias (bias_period < 0) needs the per-sample / per-tensor min-max layout%s");
  } else {
    rc = make_plan(d->outer, d->groups, d->inner, can_vec, !(d->bias_corr || d->var_corr), r.resident, &pl);
  }
  if (rc != FQB200_OK) return rc;
  if (out_pitch) {
    rc = pitch_rules(d, can_vec, out_pitch);
    if (rc != FQB200_OK) return rc;
    A.out_pad_v = static_cast<unsigned>((out_pitch - slice_channels(d)) / 4);
  }
  if ((d->residual_stats || d->residual_bias) && !d->residual)
    return fail(FQB200_ERR_INVALID, "residual_stats / residual_bias without a residual%s");
  if (d->residual_bias && !d->residual_stats)
    return fail(FQB200_ERR_INVALID, "residual_bias needs residual_stats (a bias on a plain addend can be folded by the caller)%s");
  if (d->residual && ((!d->channels_last && pl.mode != 3) || d->stats_only || !aligned16(d->residual)))
    return fail(FQB200_ERR_UNSUPPORTED, "residual: channels-last or per-sample / per-tensor min-max apply launches, 16-byte aligned%s");
  if (d->pool) {
    // channels-last per-channel launches, or the per-sample / per-tensor min-max launches (rows = samples) on channels-last
    // memory, which know the channel count from their channel-fastest bias
    const bool rows_cl = pl.mode == 3 && d->bias && d->bias_period < 0;
    if ((d->pool != 2 && d->pool != 3) || !(d->channels_last || rows_cl) || d->stats_only || d->residual || d->out_hist || !d->pool_out ||
        !aligned16(d->pool_out))
      return fail(FQB200_ERR_UNSUPPORTED, "pool: 2 (2x2 stride 2) or 3 (3x3 stride 2 padding 1) on channels-last apply launches without residual / histogram, 16-byte aligned pool_out%s");
    const int64_t h = d->pool_h, w = d->pool_w;
    const int64_t hw = rows_cl ? d->inner / -d->bias_period : d->inner;
    const int64_t images = rows_cl ? d->groups : d->outer;
    if (h < 2 || w < 2 || w % 2 != 0 || h * w != hw || (d->pool == 3 && h % 2 != 0))
      return fail(FQB200_ERR_UNSUPPORTED, "pool: pool_h * pool_w must be H * W of the tensor, W even (3x3: H even too)%s");
    const unsigned wt = pool_tile_width(d->pool, w, pl.flat);
    if (!wt) return fail(FQB200_ERR_UNSUPPORTED, "pool: no tile width fits%s");
    const int64_t tiles_per_row = (d->pool == 2 ? w : w / 2) / wt;
    const uint64_t tiles = static_cast<uint64_t>(images) * static_cast<uint64_t>(h / 2) * static_cast<uint64_t>(tiles_per_row);
    if (tiles >= 0xfffffff0ull) return fail(FQB200_ERR_UNSUPPORTED, "pool: too many tiles%s");
    uint64_t unit_tiles = tiles / (kUnitsPerCta * static_cast<uint64_t>(pl.grid));
    if (unit_tiles < 2) unit_tiles = 2;
    if (unit_tiles > 64) unit_tiles = 64;
    A.pool.h = static_cast<unsigned>(h);
    A.pool.w = static_cast<unsigned>(w);
    A.pool.wt = wt;
    A.pool.tiles_per_row = static_cast<unsigned>(tiles_per_row);
    A.pool.row_pairs = static_cast<unsigned>(h / 2);
    A.pool.tiles = static_cast<unsigned>(tiles);
    A.pool.unit_tiles = static_cast<unsigned>(unit_tiles);
    A.pool.units = static_cast<unsigned>((tiles + unit_tiles - 1) / unit_tiles);
    A.pool.ow = static_cast<unsigned>(w / 2);
    A.pool.kind = static_cast<unsigned>(d->pool);
    A.pool_out = d->pool_out;
  }
  A.hist_bins = d->out_hist ? (d->hist_bins > 0 ? d->hist_bins : 256) : 0;
  if (d->out_hist && d->leaf != FQB200_LEAF_TORCH && !d->channels_last)
    return fail(FQB200_ERR_UNSUPPORTED, "out_hist: torch leaf, or the mid-tread leaf on channels-last tensors%s");
  if (d->out_hist && (A.hist_bins > static_cast<int>(fqb::kHistWords) || (!d->channels_last && A.hist_bins != 256)))
    return fail(FQB200_ERR_UNSUPPORTED, "hist_bins: 256 (default), up to 8192 on channels-last tensors%s");
  A.geo = pl.geo;
  A.flat = pl.flat;
  A.scope = d->scope;
  A.range_mode = d->range_mode;
  A.leaf = d->leaf;
  A.num_bits = d->num_bits;
  A.positive = d->positive;
  A.solve_f64 = d->solve_f64;
  A.clip_k = d->clip_k;
  A.bit_alloc = d->bit_alloc;
  A.prior = d->bit_alloc_prior;
  A.ba_round = d->bit_alloc_round;
  A.ba_target = d->bit_alloc_target;
  A.mt_target = d->mt_target;
  A.mt_clip = d->mt_clip;
  A.bias_corr = d->bias_corr;
  A.var_corr = d->var_corr;
  A.stats_only = d->stats_only;
  A.relu_passthrough = d->relu_passthrough;
  A.residual = d->residual;
  A.residual_relu = d->residual_relu;
  A.residual_stats = d->residual_stats;
  A.residual_bias = d->residual_bias;
  A.out_stats = d->out_stats;
  A.bias = d->bias;
  A.hist = d->out_hist;
  A.hist_offset = d->hist_offset;
  A.hist_clamped = d->out_hist_clamped;
  A.dbg = d->debug_stamps;
  fp->block = fqb::kBulkThreads;
  fp->coop = !given;
  if (given) {  // no statistics, no barrier: no workspace
    A.g_delta = d->given_delta;
    A.g_offset = d->given_offset;
    A.g_bits = d->given_bits;
    A.given_per_group = 1;
    fp->kernel = reinterpret_cast<const void*>(fqb::fq_cl_given_fused_kernel);
    fp->smem = cl_given_smem();
    fp->name = "fq_cl_given_fused_kernel";
    return FQB200_OK;
  }
  if (pl.mode == 3) {
    if (d->scope == FQB200_SCOPE_GROUP) A.scope = FQB200_SCOPE_TENSOR;  // one row
    A.n_per_group = static_cast<double>(d->inner);
    fp->kernel = reinterpret_cast<const void*>(fqb::fq_rows_kernel);
    fp->smem = cl_given_smem();
    fp->name = "fq_rows_kernel";
  } else {
    if (d->bias && d->bias_period > 0) {
      // bias indexed by the channel inside the row: needs whole vectors per channel and an exact magic division
      const uint64_t pv = static_cast<uint64_t>(d->bias_period) / pl.vec;
      if (pl.mode != 4 || d->leaf != FQB200_LEAF_COMPILED || d->range_mode != FQB200_RANGE_MINMAX || d->bias_corr || d->var_corr ||
          d->stats_only || d->bias_period % pl.vec != 0 || d->inner % d->bias_period != 0 || pv == 0 ||
          static_cast<uint64_t>(pl.geo.inner_v) * pv >= (1ull << 40) || pl.geo.inner_v >= (1u << 24))
        return fail(FQB200_ERR_UNSUPPORTED, "bias_period does not fit this layout%s");
      A.bias_magic = ((1ull << 40) + pv - 1) / pv;
    }
    A.inner = static_cast<unsigned>(d->inner);
    A.n_per_group = static_cast<double>(d->outer) * static_cast<double>(d->inner);
    const bool alloc = d->bit_alloc && d->num_bits <= 4 && d->scope == FQB200_SCOPE_GROUP && d->leaf != FQB200_LEAF_MIDTREAD;
    if (pl.mode == 2) {
      // replicas of the per-channel accumulators: CTA b adds into replica b % rep (same-address atomics serialise in L2)
      const unsigned rep = fqb::kMaxNhwcChannels / static_cast<unsigned>(d->groups);
      A.nhwc_rep = rep < 1u ? 1u : (rep > 8u ? 8u : rep);
      // phase S2 (sum |x - mean|) of the channels-last kernel: only where the Laplace b is consumed
      A.need_dev = d->range_mode == FQB200_RANGE_LAPLACE || (d->leaf == FQB200_LEAF_MIDTREAD && d->mt_clip) ||
                   (alloc && d->bit_alloc_prior == FQB200_PRIOR_B) || d->stats_only || d->out_stats != nullptr;
      fp->kernel = cl_kernel_ptr(d->leaf, A.need_dev != 0, d->out_hist != nullptr);
      fp->smem = cl_smem(d->out_hist != nullptr);
      fp->name = "fq_cl_kernel";
    } else {
      A.nhwc_rep = 1;
      A.need_dev = (d->range_mode != FQB200_RANGE_MINMAX) || alloc || d->var_corr || d->leaf == FQB200_LEAF_MIDTREAD || d->stats_only;
      fp->slots = static_cast<uint64_t>(pl.geo.parts) * pl.geo.channels;  // the channels-last kernels use the accumulators
      fp->kernel = A.bias_magic ? reinterpret_cast<const void*>(fqb::fq_fused_kernel<4, FQB200_LEAF_COMPILED, false, false, true>)
                                : fused_kernel_ptr(pl.mode, d->leaf, A.need_dev != 0, d->bias_corr || d->var_corr);
      fp->block = fqb::kThreads;
      fp->smem = dyn_smem(pl.vec);
      fp->name = "fq_fused_kernel";
    }
  }
  fp->workspace = carve(nullptr, fp->slots, pl.geo.channels, nullptr);
  return FQB200_OK;
}

// the resident-CTA counts plans are made for without a launch: the current device's, or, when there is none, an H100's
// at each kernel family's __launch_bounds__ residency
DeviceInfo plan_residency() {
  DeviceInfo* di = nullptr;
  if (get_device(&di) == FQB200_OK) return *di;
  DeviceInfo h;
  h.resident = kAssumedSms * fqb::kCtasPerSm;
  h.resident_cl[0] = h.resident_cl[1] = h.resident_rows = kAssumedSms * fqb::kBulkCtasPerSm;
  return h;
}

}  // namespace

extern "C" {

int fqb200_abi_version(void) { return FQB200_ABI_VERSION; }

const char* fqb200_last_error(void) { return g_err; }

int fqb200_resident_ctas(void) {
  DeviceInfo* di = nullptr;
  if (get_device(&di) != FQB200_OK) return -1;
  return di->resident;
}

size_t fqb200_workspace_bytes(const fqb200_desc* d) {
  if (check_desc(d) != FQB200_OK) return 0;
  if (d->outer == 0 || d->groups == 0 || d->inner == 0) return 256;
  const DeviceInfo r = plan_residency();
  size_t bytes = 0;
  for (bool can_vec : {false, true}) {  // the aligned plan last: its message stands when both refuse
    FusedPlan fp;
    if (plan_fused(d, can_vec, 0, r, &fp) != FQB200_OK) continue;
    const size_t need = fp.workspace ? fp.workspace : 256;  // RANGE_GIVEN uses none; non-zero = "descriptor accepted"
    if (need > bytes) bytes = need;
  }
  return bytes;
}

int fqb200_workspace_init(void* workspace, size_t bytes, void* stream) {
  const size_t head = carve(nullptr, 0, 0, nullptr);  // barrier words + channels-last accumulator banks
  if (!workspace || bytes < head) return fail(FQB200_ERR_WORKSPACE, "workspace too small%s");
  cudaError_t e = cudaMemsetAsync(workspace, 0, head, static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return fail(FQB200_ERR_CUDA, "cudaMemsetAsync: %s", cudaGetErrorString(e));
  return FQB200_OK;
}

int fqb200_plan_info(const fqb200_desc* d, int64_t* out8) {
  g_err[0] = 0;
  int rc = check_desc(d);
  if (rc != FQB200_OK) return rc;
  if (!out8) return fail(FQB200_ERR_INVALID, "null output%s");
  FusedPlan fp;
  rc = plan_fused(d, true, 0, plan_residency(), &fp);
  if (rc != FQB200_OK) return rc;
  const Plan& pl = fp.pl;
  if (pl.mode == 2 || pl.mode == 3) {  // phases: apply only (RANGE_GIVEN), statistics + apply, + the second statistics pass
    out8[0] = pl.mode; out8[1] = pl.grid; out8[2] = pl.flat.units; out8[3] = pl.flat.unit_stages; out8[4] = pl.flat.stage_v;
    out8[5] = pl.flat.stride; out8[6] = fqb::kStages; out8[7] = d->range_mode == FQB200_RANGE_GIVEN ? 1 : 2 + fp.A.need_dev;
    return FQB200_OK;
  }
  out8[0] = pl.mode; out8[1] = pl.grid; out8[2] = pl.geo.units; out8[3] = pl.geo.parts; out8[4] = pl.geo.part_v;
  out8[5] = pl.geo.stride; out8[6] = fqb::kRingDepth; out8[7] = pl.geo.red_lanes;
  return FQB200_OK;
}

int fqb200_float2gemmlowp(const float* in, float* out, int64_t n, float range, float offset, int num_bits, int int_exp,
                          int enforce_true_zero, const float* noise, void* stream) {
  g_err[0] = 0;
  if (n < 0 || num_bits < 1 || num_bits > 30) return fail(FQB200_ERR_INVALID, "bad n / num_bits%s");
  if (n == 0) return FQB200_OK;
  if (!in || !out) return fail(FQB200_ERR_INVALID, "null tensor pointer%s");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (range <= 0) {  // gemmlowp.cu:31-32: the reference hands back its input
    if (in != out) {
      cudaError_t e = cudaMemcpyAsync(out, in, static_cast<size_t>(n) * sizeof(float), cudaMemcpyDeviceToDevice, st);
      if (e != cudaSuccess) return fail(FQB200_ERR_CUDA, "cudaMemcpyAsync: %s", cudaGetErrorString(e));
    }
    return FQB200_OK;
  }
  DeviceInfo* di = nullptr;
  int rc = get_device(&di);
  if (rc != FQB200_OK) return rc;
  // host wrapper arithmetic, gemmlowp.cu:36-41 (fp32, one rounding per operator)
  const long long qmax_i = (1ll << num_bits) - 1;
  volatile float scale = range / static_cast<float>(qmax_i);
  if (int_exp) scale = powf(2.f, static_cast<float>(static_cast<int>(ceilf(log2f(scale)))));
  volatile float zr = -offset / scale;
  const float zero_point = roundf(zr);
  fqb::LeafParam q;
  q.a = scale;
  q.b = enforce_true_zero ? zero_point : -offset;
  q.c = static_cast<float>(qmax_i);
  q.flags = enforce_true_zero ? fqb::FLAG_TRUE_ZERO : 0;
  const bool vec = (n % 4 == 0) && aligned16(in) && aligned16(out) && (!noise || aligned16(noise));
  // the streaming case (16-byte aligned, a multiple of 4 elements, at least a few stages per SM): bulk-copy ring
  if (vec && static_cast<uint64_t>(n) >= (1ull << 20) && static_cast<uint64_t>(n) / 4 < (1ull << 32)) {
    Plan pl;
    rc = make_plan_flat(static_cast<uint64_t>(n), 0, di->resident_cl[0] * 2, &pl);
    if (rc != FQB200_OK) return rc;
    fqb::LeafBulkArgs B;
    B.flat = pl.flat;
    B.in = in;
    B.out = out;
    B.noise = noise;
    B.q = q;
    if (noise) fqb::fq_leaf_bulk_kernel<true><<<pl.grid, fqb::kBulkThreads, cl_given_smem(), st>>>(B);
    else       fqb::fq_leaf_bulk_kernel<false><<<pl.grid, fqb::kBulkThreads, cl_given_smem(), st>>>(B);
    return launched("fq_leaf_bulk_kernel");
  }
  const unsigned long long nvec = vec ? static_cast<unsigned long long>(n / 4) : static_cast<unsigned long long>(n);
  const int grid = grid_for((nvec + fqb::kThreads * 4ull - 1) / (fqb::kThreads * 4ull), di->resident * 2ull);
  const float as = fabsf(q.a);
  const bool fast = (as > 1e-30f) && (as < 1e30f);
#define FQB_LAUNCH_LEAF(V, N, F) fqb::fq_leaf_kernel<V, N, F><<<grid, fqb::kThreads, 0, st>>>(in, out, noise, nvec, q)
  if (vec) {
    if (noise) { if (fast) FQB_LAUNCH_LEAF(4, true, true); else FQB_LAUNCH_LEAF(4, true, false); }
    else       { if (fast) FQB_LAUNCH_LEAF(4, false, true); else FQB_LAUNCH_LEAF(4, false, false); }
  } else {
    if (noise) { if (fast) FQB_LAUNCH_LEAF(1, true, true); else FQB_LAUNCH_LEAF(1, true, false); }
    else       { if (fast) FQB_LAUNCH_LEAF(1, false, true); else FQB_LAUNCH_LEAF(1, false, false); }
  }
#undef FQB_LAUNCH_LEAF
  return launched("fq_leaf_kernel");
}

int fqb200_quantize1(const float* in, float* out, float* grid, int64_t outer, int64_t groups, int64_t inner,
                     const float* delta, const float* offset, const float* bits, int per_group, int num_bits,
                     const float* bias, int channels_last, void* stream) {
  g_err[0] = 0;
  if (outer == 0 || groups == 0 || inner == 0) return FQB200_OK;
  if (!in || !out || !delta || !offset) return fail(FQB200_ERR_INVALID, "null pointer%s");
  if (num_bits < 1 || num_bits > 8) {
    if (!bits) return fail(FQB200_ERR_INVALID, "num_bits must be in 1..8%s");
  }
  if (bits && !per_group) return fail(FQB200_ERR_INVALID, "per-row bit widths need per-group parameters%s");
  DeviceInfo* di = nullptr;
  int rc = get_device(&di);
  if (rc != FQB200_OK) return rc;
  Plan pl;
  const bool can_vec = aligned16(in) && aligned16(out) && (!grid || aligned16(grid));
  fqb::FusedArgs A;
  memset(&A, 0, sizeof(A));
  A.in = in;
  A.out = out;
  A.grid_out = grid;
  A.leaf = FQB200_LEAF_TORCH;
  A.num_bits = num_bits;
  A.g_delta = delta;
  A.g_offset = offset;
  A.g_bits = bits;
  A.given_per_group = per_group;
  A.bias = bias;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const uint64_t elems = static_cast<uint64_t>(outer) * static_cast<uint64_t>(groups) * static_cast<uint64_t>(inner);
  // flat streams on the bulk-copy engine: channels-last per-channel parameters, or one parameter set for the whole tensor
  const bool flat_cl = channels_last && per_group;
  const bool flat_tensor = !per_group && !bias;
  if (channels_last && !per_group && bias) return fail(FQB200_ERR_UNSUPPORTED, "channels_last with one parameter set takes no bias%s");
  if (flat_cl && !(can_vec && flat_eligible(groups)))
    return fail(FQB200_ERR_UNSUPPORTED, "channels_last needs 16-byte aligned tensors, C %% 4 == 0 and C <= 2048%s");
  if (flat_cl || (flat_tensor && can_vec && elems % 4 == 0)) {
    rc = make_plan_flat(elems, flat_cl ? groups : 0, di->resident_cl[0] * 2, &pl);
    if (rc != FQB200_OK) return rc;
    A.flat = pl.flat;
    if (grid) fqb::fq_cl_given_kernel<true><<<pl.grid, fqb::kBulkThreads, cl_given_smem(), st>>>(A);
    else      fqb::fq_cl_given_kernel<false><<<pl.grid, fqb::kBulkThreads, cl_given_smem(), st>>>(A);
    return launched("fq_cl_given_kernel");
  }
  rc = make_plan(outer, groups, inner, can_vec, false, di->resident * 2, &pl);
  if (rc != FQB200_OK) return rc;
  A.geo = pl.geo;
  if (pl.vec == 4) {
    if (grid) fqb::fq_given_kernel<4, FQB200_LEAF_TORCH, true><<<pl.grid, fqb::kThreads, dyn_smem(4), st>>>(A);
    else      fqb::fq_given_kernel<4, FQB200_LEAF_TORCH, false><<<pl.grid, fqb::kThreads, dyn_smem(4), st>>>(A);
  } else {
    if (grid) fqb::fq_given_kernel<1, FQB200_LEAF_TORCH, true><<<pl.grid, fqb::kThreads, dyn_smem(1), st>>>(A);
    else      fqb::fq_given_kernel<1, FQB200_LEAF_TORCH, false><<<pl.grid, fqb::kThreads, dyn_smem(1), st>>>(A);
  }
  return launched("fq_given_kernel");
}

int fqb200_fused(const fqb200_desc* d, const float* in, float* out, void* workspace, size_t workspace_bytes,
                 void* stream) {
  return fqb200_fused_into(d, in, out, 0, workspace, workspace_bytes, stream);
}

int fqb200_fused_into(const fqb200_desc* d, const float* in, float* out, int64_t out_pixel_stride, void* workspace,
                      size_t workspace_bytes, void* stream) {
  g_err[0] = 0;
  int rc = check_desc(d);
  if (rc != FQB200_OK) return rc;
  if (d->outer == 0 || d->groups == 0 || d->inner == 0) return FQB200_OK;
  if (!in) return fail(FQB200_ERR_INVALID, "null input%s");
  if (!out && !d->stats_only && !d->pool) return fail(FQB200_ERR_INVALID, "null output%s");
  if (d->stats_only && !d->out_stats) return fail(FQB200_ERR_INVALID, "stats_only needs out_stats%s");
  const bool can_vec = aligned16(in) && (d->stats_only || d->pool || aligned16(out));
  int64_t c = 0;   // channels of a pixel (slice_channels), when `out` is pitched
  if (out_pixel_stride != 0) {   // 0: fqb200_fused, a dense `out`
    if (out_pixel_stride < 0) return fail(FQB200_ERR_INVALID, "negative out_pixel_stride%s");
    rc = pitch_rules(d, can_vec, out_pixel_stride);
    if (rc != FQB200_OK) return rc;
    c = slice_channels(d);
    const uint64_t elems = static_cast<uint64_t>(d->outer) * static_cast<uint64_t>(d->groups) * static_cast<uint64_t>(d->inner);
    const uint64_t pixels = elems / static_cast<uint64_t>(c);
    const uintptr_t i0 = reinterpret_cast<uintptr_t>(in), i1 = i0 + elems * sizeof(float);
    const uintptr_t o0 = reinterpret_cast<uintptr_t>(out),
                    o1 = o0 + ((pixels - 1) * out_pixel_stride + c) * sizeof(float);
    if (out_pixel_stride != c && o0 < i1 && i0 < o1)   // (the dense case may work in place)
      return fail(FQB200_ERR_INVALID, "out_pixel_stride: out overlaps in%s");
  }
  DeviceInfo* di = nullptr;
  rc = get_device(&di);
  if (rc != FQB200_OK) return rc;
  FusedPlan fp;
  rc = plan_fused(d, can_vec, out_pixel_stride == c ? 0 : out_pixel_stride, *di, &fp);   // pitch C: dense
  if (rc != FQB200_OK) return rc;
  rc = check_workspace(workspace, workspace_bytes, fp.workspace, "fqb200_workspace_bytes");
  if (rc != FQB200_OK) return rc;
  if (fp.workspace) carve(static_cast<char*>(workspace), fp.slots, fp.pl.geo.channels, &fp.A);
  fp.A.in = in;
  fp.A.out = out;
  void* args[] = {&fp.A};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // (the cooperative launch guarantees the co-residency the grid barriers need)
  const cudaError_t e = fp.coop ? cudaLaunchCooperativeKernel(fp.kernel, dim3(fp.pl.grid), dim3(fp.block), args, fp.smem, st)
                                : cudaLaunchKernel(fp.kernel, dim3(fp.pl.grid), dim3(fp.block), args, fp.smem, st);
  if (e != cudaSuccess) return fail(FQB200_ERR_CUDA, fp.coop ? "cooperative launch %s: %s" : "launch %s: %s", fp.name, cudaGetErrorString(e));
  return FQB200_OK;
}

int fqb200_quantize1_bca(const float* in, float* out, int64_t outer, int64_t groups, int64_t inner, const float* delta,
                         const float* offset, const float* bits, int per_group, int num_bits, const float* bias, int relu_first,
                         float* out_qbias, void* workspace, size_t workspace_bytes, void* stream) {
  g_err[0] = 0;
  if (outer == 0 || groups == 0 || inner == 0) return FQB200_OK;
  if (!in || !out || !delta || !offset) return fail(FQB200_ERR_INVALID, "null pointer%s");
  if ((num_bits < 1 || num_bits > 8) && !bits) return fail(FQB200_ERR_INVALID, "num_bits must be in 1..8%s");
  if (bits && !per_group) return fail(FQB200_ERR_INVALID, "per-row bit widths need per-group parameters%s");
  if (!(aligned16(in) && aligned16(out) && flat_eligible(groups)))
    return fail(FQB200_ERR_UNSUPPORTED, "bias-corrected quantization runs on channels-last tensors: 16-byte aligned, C %% 4 == 0, C <= 2048%s");
  int rc = check_workspace(workspace, workspace_bytes, carve(nullptr, 0, static_cast<uint64_t>(groups), nullptr),
                           "fqb200_workspace_bytes");
  if (rc != FQB200_OK) return rc;
  DeviceInfo* di = nullptr;
  rc = get_device(&di);
  if (rc != FQB200_OK) return rc;
  Plan pl;
  rc = make_plan_flat(static_cast<uint64_t>(outer) * groups * inner, groups, di->resident_bca, &pl);
  if (rc != FQB200_OK) return rc;
  fqb::FusedArgs A;
  memset(&A, 0, sizeof(A));
  carve(static_cast<char*>(workspace), 0, static_cast<uint64_t>(groups), &A);
  A.flat = pl.flat;
  A.geo = pl.geo;
  A.in = in;
  A.out = out;
  A.leaf = FQB200_LEAF_TORCH;
  A.num_bits = num_bits;
  A.g_delta = delta;
  A.g_offset = offset;
  A.g_bits = bits;
  A.given_per_group = per_group;
  A.bias = bias;
  A.relu_passthrough = relu_first;
  A.out_stats = out_qbias;
  const unsigned r = fqb::kMaxNhwcChannels / static_cast<unsigned>(groups);
  A.nhwc_rep = r < 1u ? 1u : (r > 8u ? 8u : r);
  void* args[] = {&A};
  cudaError_t e = cudaLaunchCooperativeKernel(reinterpret_cast<const void*>(fqb::fq_cl_bca_kernel), dim3(pl.grid),
                                              dim3(fqb::kBulkThreads), args, cl_smem(false), static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return fail(FQB200_ERR_CUDA, "cooperative launch fq_cl_bca_kernel: %s", cudaGetErrorString(e));
  return FQB200_OK;
}

int fqb200_maxpool2d_nhwc(const float* in, float* out, int64_t n, int64_t h, int64_t w, int64_t c, int kh, int kw, int sh, int sw,
                          int ph, int pw, void* stream) {
  return fqb200_maxpool2d_nhwc_into(in, out, n, h, w, c, kh, kw, sh, sw, ph, pw, c, stream);
}

int fqb200_maxpool2d_nhwc_into(const float* in, float* out, int64_t n, int64_t h, int64_t w, int64_t c, int kh, int kw, int sh,
                               int sw, int ph, int pw, int64_t out_pixel_stride, void* stream) {
  g_err[0] = 0;
  if (n < 0 || h <= 0 || w <= 0 || c <= 0 || kh <= 0 || kw <= 0 || sh <= 0 || sw <= 0 || ph < 0 || pw < 0 || 2 * ph > kh || 2 * pw > kw)
    return fail(FQB200_ERR_INVALID, "bad pooling geometry%s");
  if (n == 0) return FQB200_OK;
  if (!in || !out) return fail(FQB200_ERR_INVALID, "null tensor pointer%s");
  if (c % 4 != 0 || !aligned16(in) || !aligned16(out)) return fail(FQB200_ERR_UNSUPPORTED, "channels-last pooling needs C %% 4 == 0 and 16-byte aligned tensors%s");
  if (out_pixel_stride < c || out_pixel_stride % 4 != 0)
    return fail(FQB200_ERR_UNSUPPORTED, "out_pixel_stride must be >= C and a multiple of 4%s");
  const int64_t oh = (h + 2 * ph - kh) / sh + 1, ow = (w + 2 * pw - kw) / sw + 1;
  if (oh <= 0 || ow <= 0 || h >= (1ll << 31) || w >= (1ll << 31) || n >= (1ll << 31)) return fail(FQB200_ERR_INVALID, "bad pooling geometry%s");
  const uintptr_t i0 = reinterpret_cast<uintptr_t>(in), i1 = i0 + static_cast<uint64_t>(n * h * w * c) * sizeof(float);
  const uintptr_t o0 = reinterpret_cast<uintptr_t>(out),
                  o1 = o0 + static_cast<uint64_t>((n * oh * ow - 1) * out_pixel_stride + c) * sizeof(float);
  if (o0 < i1 && i0 < o1) return fail(FQB200_ERR_INVALID, "out overlaps in%s");
  DeviceInfo* di = nullptr;
  int rc = get_device(&di);
  if (rc != FQB200_OK) return rc;
  fqb::PoolArgs P;
  P.in = in; P.out = out; P.out_pv = static_cast<unsigned long long>(out_pixel_stride / 4);
  P.n = static_cast<unsigned>(n); P.h = static_cast<unsigned>(h); P.w = static_cast<unsigned>(w); P.cv = static_cast<unsigned>(c / 4);
  P.oh = static_cast<unsigned>(oh); P.ow = static_cast<unsigned>(ow);
  P.kh = kh; P.kw = kw; P.sh = sh; P.sw = sw; P.ph = ph; P.pw = pw;
  P.total = static_cast<unsigned long long>(n) * oh * ow * (c / 4);
  const int grid = grid_for((P.total + 255ull) / 256ull, di->sms * 32ull);
  fqb::fq_maxpool_nhwc_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(P);
  return launched("fq_maxpool_nhwc_kernel");
}

int fqb200_add_relu(const float* a, const float* b, float* out, int64_t n, void* stream) {
  g_err[0] = 0;
  if (n < 0) return fail(FQB200_ERR_INVALID, "negative size%s");
  if (n == 0) return FQB200_OK;
  if (!a || !b || !out) return fail(FQB200_ERR_INVALID, "null tensor pointer%s");
  DeviceInfo* di = nullptr;
  int rc = get_device(&di);
  if (rc != FQB200_OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool vec = (n % 4 == 0) && aligned16(a) && aligned16(b) && aligned16(out);
  const unsigned long long nvec = vec ? static_cast<unsigned long long>(n / 4) : static_cast<unsigned long long>(n);
  const int grid = grid_for((nvec + fqb::kThreads * 4ull - 1) / (fqb::kThreads * 4ull), di->resident * 4ull);
  if (vec) fqb::fq_add_relu_kernel<4><<<grid, fqb::kThreads, 0, st>>>(a, b, out, nvec);
  else     fqb::fq_add_relu_kernel<1><<<grid, fqb::kThreads, 0, st>>>(a, b, out, nvec);
  return launched("fq_add_relu_kernel");
}

size_t fqb200_kld_workspace_bytes(int64_t rows, int num_bins) {
  g_err[0] = 0;
  if (rows <= 0 || rows > (1ll << 31) - 1) return fail(FQB200_ERR_INVALID, "rows must be in 1 .. 2^31 - 1%s"), 0;
  if (num_bins < 3 || num_bins > kKldMaxBins || num_bins % 2 == 0) return fail(FQB200_ERR_INVALID, "num_bins must be odd, 3 .. 8001%s"), 0;
  return kld_workspace(rows, num_bins);
}

int fqb200_kld_threshold(const float* in, int64_t rows, int64_t row_len, int num_bins, int num_quantized_bins, float* out_th,
                         float* out_div, int32_t* out_idx, void* workspace, size_t workspace_bytes, void* stream) {
  g_err[0] = 0;
  if (num_bins < 3 || num_bins > kKldMaxBins || num_bins % 2 == 0) return fail(FQB200_ERR_INVALID, "num_bins must be odd, 3 .. 8001%s");
  if (num_quantized_bins < 3 || num_quantized_bins > num_bins || num_quantized_bins % 2 == 0)
    return fail(FQB200_ERR_INVALID, "num_quantized_bins must be odd, 3 .. num_bins%s");
  if (rows <= 0 || row_len <= 0 || rows > (1ll << 31) - 1) return fail(FQB200_ERR_INVALID, "rows / row_len must be positive (rows < 2^31)%s");
  if (row_len > (1ll << 31) - 1) return fail(FQB200_ERR_UNSUPPORTED, "rows of 2^31 elements and more (int32 bin counts)%s");
  if (!in || !out_th || !out_div || !out_idx) return fail(FQB200_ERR_INVALID, "null pointer%s");
  const size_t need = kld_workspace(rows, num_bins);
  int rc = check_workspace(workspace, workspace_bytes, need, "fqb200_kld_workspace_bytes");
  if (rc != FQB200_OK) return rc;
  DeviceInfo* di = nullptr;
  rc = get_device(&di);
  if (rc != FQB200_OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  fqb::KldArgs A;
  memset(&A, 0, sizeof(A));
  A.in = in;
  A.rows = static_cast<unsigned long long>(rows);
  A.row_len = static_cast<unsigned long long>(row_len);
  // fill the GPU with (row, chunk) units but keep them long: every unit flushes up to num_bins counters
  const unsigned long long want = static_cast<unsigned long long>(di->sms) * 4ull;
  unsigned long long chunks = (want + A.rows - 1) / A.rows;
  const unsigned long long max_chunks = (A.row_len + 4095ull) / 4096ull;
  chunks = chunks < max_chunks ? chunks : max_chunks;
  A.chunk = ((A.row_len + chunks - 1) / chunks + 3ull) / 4ull * 4ull;
  A.chunks = (A.row_len + A.chunk - 1) / A.chunk;
  A.absmax = static_cast<unsigned*>(workspace);
  A.hist = reinterpret_cast<unsigned*>(static_cast<char*>(workspace) + align_up(static_cast<size_t>(rows) * 4, 256));
  A.nb = num_bins;
  A.nq = num_quantized_bins;
  A.replicas = kld_replicas(num_bins);
  A.out_th = out_th;
  A.out_div = out_div;
  A.out_idx = out_idx;
  const size_t hist_smem = kld_hist_smem(num_bins), search_smem = kld_search_smem(num_bins);
  const bool vec = row_len % 4 == 0 && aligned16(in);
  const cudaError_t e = cudaMemsetAsync(workspace, 0, need, st);
  if (e != cudaSuccess) return fail(FQB200_ERR_CUDA, "cudaMemsetAsync: %s", cudaGetErrorString(e));
  const int grid = grid_for(A.rows * A.chunks, want);
  if (vec) {
    fqb::fq_kld_absmax_kernel<4><<<grid, fqb::kKldThreads, 0, st>>>(A);
    fqb::fq_kld_hist_kernel<4><<<grid, fqb::kKldThreads, hist_smem, st>>>(A);
  } else {
    fqb::fq_kld_absmax_kernel<1><<<grid, fqb::kKldThreads, 0, st>>>(A);
    fqb::fq_kld_hist_kernel<1><<<grid, fqb::kKldThreads, hist_smem, st>>>(A);
  }
  fqb::fq_kld_search_kernel<<<static_cast<unsigned>(rows), fqb::kKldThreads, search_smem, st>>>(A);
  return launched("KLD kernels");
}

size_t fqb200_sample_sumsq_workspace_bytes(int64_t rows, int64_t row_len) {
  g_err[0] = 0;
  if (rows < 0 || row_len <= 0) return fail(FQB200_ERR_INVALID, "rows must be >= 0 and row_len > 0%s"), 0;
  return sums_workspace(rows, row_len, 1);
}

int fqb200_sample_sumsq(const float* in, int64_t rows, int64_t row_len, double* out, void* workspace, size_t workspace_bytes,
                        void* stream) {
  g_err[0] = 0;
  if (rows < 0 || row_len <= 0) return fail(FQB200_ERR_INVALID, "rows must be >= 0 and row_len > 0%s");
  if (!in || !out) return fail(FQB200_ERR_INVALID, "null pointer%s");
  const int rc = check_workspace(workspace, workspace_bytes, sums_workspace(rows, row_len, 1),
                                 "fqb200_sample_sumsq_workspace_bytes");
  if (rc != FQB200_OK) return rc;
  if (rows == 0) return FQB200_OK;
  return launch_sums<1>(in, nullptr, nullptr, 0, rows, row_len, out, workspace, 0, stream, "sum-of-squares kernels");
}

// the requests fqb200_sample_angles takes (FQB200_OK, or the code with the message in fqb200_last_error())
static int angle_bad_args(int64_t rows, int64_t row_len) {
  if (rows < 0 || row_len <= 0) return fail(FQB200_ERR_INVALID, "rows must be >= 0 and row_len > 0%s");
  if (rows > fqb::kAngMaxRows) return fail(FQB200_ERR_UNSUPPORTED, "rows must be <= 8192%s");
  return FQB200_OK;
}

size_t fqb200_sample_angles_workspace_bytes(int64_t rows, int64_t row_len) {
  g_err[0] = 0;
  if (angle_bad_args(rows, row_len) != FQB200_OK) return 0;
  return angle_workspace(rows, row_len);
}

int fqb200_sample_angles(const float* in, int64_t rows, int64_t row_len, float* out_angles, double* out_gram,
                         void* workspace, size_t workspace_bytes, int32_t max_ctas, void* stream) {
  g_err[0] = 0;
  int rc = angle_bad_args(rows, row_len);
  if (rc != FQB200_OK) return rc;
  if (!out_angles && !out_gram) return fail(FQB200_ERR_INVALID, "null pointer: out_angles and out_gram%s");
  if (!in) return fail(FQB200_ERR_INVALID, "null pointer%s");
  if (max_ctas < 0) return fail(FQB200_ERR_INVALID, "max_ctas must be >= 0%s");
  rc = check_workspace(workspace, workspace_bytes, angle_workspace(rows, row_len), "fqb200_sample_angles_workspace_bytes");
  if (rc != FQB200_OK) return rc;
  if (rows == 0) return FQB200_OK;
  DeviceInfo* di = nullptr;
  rc = get_device(&di);
  if (rc != FQB200_OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const fqb::AngleSplit sp = fqb::angle_split(static_cast<unsigned long long>(rows), static_cast<unsigned long long>(row_len));
  fqb::AngleArgs A;
  memset(&A, 0, sizeof(A));
  A.in = in;
  A.rows = static_cast<unsigned long long>(rows);
  A.row_len = static_cast<unsigned long long>(row_len);
  A.tiles = sp.tiles;
  A.pairs = sp.pairs;
  A.slices = sp.slices;
  A.slice_steps = sp.slice_steps;
  A.partial = static_cast<double*>(workspace);
  A.angles = out_angles;
  A.gram = out_gram;
  const bool vec = row_len % 4 == 0 && aligned16(in);
  const int grid = grid_for(A.pairs * A.slices, di->resident_angle[vec ? 1 : 0], max_ctas);
  if (vec) fqb::fq_gram_partial_kernel<4><<<grid, fqb::kAngThreads, fqb::kAngSmemBytes, st>>>(A);
  else     fqb::fq_gram_partial_kernel<1><<<grid, fqb::kAngThreads, fqb::kAngSmemBytes, st>>>(A);
  const dim3 fgrid(fqb::kAngTile * fqb::kAngTile / fqb::kAngFinishThreads, static_cast<unsigned>(A.pairs));
  fqb::fq_gram_finish_kernel<<<fgrid, fqb::kAngFinishThreads, 0, st>>>(A);
  return launched("Gram kernels");
}

size_t fqb200_sample_noise_workspace_bytes(int64_t rows, int64_t row_len) {
  g_err[0] = 0;
  if (rows < 0 || row_len <= 0) return fail(FQB200_ERR_INVALID, "rows must be >= 0 and row_len > 0%s"), 0;
  return sums_workspace(rows, row_len, fqb::kSumsMax);   // enough for the two sums of a call without q too
}

int fqb200_sample_noise(const float* y, const float* q, const float* bias, int64_t bias_period, int64_t rows, int64_t row_len,
                        double* out, void* workspace, size_t workspace_bytes, int32_t max_ctas, void* stream) {
  g_err[0] = 0;
  if (rows < 0 || row_len <= 0) return fail(FQB200_ERR_INVALID, "rows must be >= 0 and row_len > 0%s");
  if (!y || !out) return fail(FQB200_ERR_INVALID, "null pointer%s");
  if (max_ctas < 0) return fail(FQB200_ERR_INVALID, "max_ctas must be >= 0%s");
  const unsigned long long period = bias_period < 0 ? 0ull - static_cast<unsigned long long>(bias_period)
                                                    : static_cast<unsigned long long>(bias_period);
  if (bias) {
    if (period == 0 || static_cast<unsigned long long>(row_len) % period != 0)
      return fail(FQB200_ERR_INVALID, "a bias needs a bias_period != 0 whose magnitude divides row_len%s");
    if (static_cast<unsigned long long>(row_len) > 0xffffffffull)
      return fail(FQB200_ERR_UNSUPPORTED, "rows of 2^32 elements and more take no bias%s");
  }
  const int rc = check_workspace(workspace, workspace_bytes, sums_workspace(rows, row_len, fqb::kSumsMax),
                                 "fqb200_sample_noise_workspace_bytes");
  if (rc != FQB200_OK) return rc;
  if (rows == 0) return FQB200_OK;
  const char* what = "quantization-noise kernels";
  if (q) return launch_sums<fqb::kSumsMax>(y, q, bias, bias_period, rows, row_len, out, workspace, max_ctas, stream, what);
  return launch_sums<2>(y, nullptr, bias, bias_period, rows, row_len, out, workspace, max_ctas, stream, what);
}

// the layouts fqb200_clip_error takes (argument errors as a message, nullptr when they are fine)
static const char* cliperr_bad_args(int64_t outer, int64_t groups, int64_t inner, int channels_last) {
  if (outer <= 0 || groups <= 0 || inner <= 0) return "outer, groups and inner must be > 0%s";
  if (channels_last && !flat_eligible(groups)) return "channels_last needs C %% 4 == 0 and 4 <= C <= 2048%s";
  if (!channels_last && outer > 1 && static_cast<unsigned long long>(outer) * static_cast<unsigned long long>(inner) >= (1ull << 32))
    return "a group of an NCHW layout must hold fewer than 2^32 elements%s";
  return nullptr;
}

size_t fqb200_clip_error_workspace_bytes(int64_t outer, int64_t groups, int64_t inner, int32_t channels_last) {
  g_err[0] = 0;
  const char* bad = cliperr_bad_args(outer, groups, inner, channels_last);
  if (bad) return fail(FQB200_ERR_INVALID, bad), 0;
  return cliperr_workspace(outer, groups, inner, channels_last);
}

int fqb200_clip_error(const float* in, int64_t outer, int64_t groups, int64_t inner, int32_t channels_last, const float* stats,
                      int32_t num_bits, int32_t positive, int32_t bit_alloc, int32_t solve_f64, double* out, float* out_params,
                      void* workspace, size_t workspace_bytes, int32_t max_ctas, void* stream) {
  g_err[0] = 0;
  const char* bad = cliperr_bad_args(outer, groups, inner, channels_last);
  if (bad) return fail(FQB200_ERR_INVALID, bad);
  if (!in || !stats || !out) return fail(FQB200_ERR_INVALID, "null pointer%s");
  if (num_bits < 1 || num_bits > 8) return fail(FQB200_ERR_INVALID, "num_bits must be in 1..8%s");
  if (bit_alloc && num_bits > 4) return fail(FQB200_ERR_INVALID, "bit_alloc applies to num_bits <= 4 only%s");
  if (max_ctas < 0) return fail(FQB200_ERR_INVALID, "max_ctas must be >= 0%s");
  int rc = check_workspace(workspace, workspace_bytes, cliperr_workspace(outer, groups, inner, channels_last),
                           "fqb200_clip_error_workspace_bytes");
  if (rc != FQB200_OK) return rc;
  DeviceInfo* di = nullptr;
  rc = get_device(&di);
  if (rc != FQB200_OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  fqb::ClipErrArgs A;
  memset(&A, 0, sizeof(A));
  A.in = in;
  A.stats = stats;
  A.outer = static_cast<unsigned long long>(outer);
  A.groups = static_cast<unsigned long long>(groups);
  A.inner = static_cast<unsigned long long>(inner);
  A.channels_last = channels_last ? 1 : 0;
  A.num_bits = num_bits;
  A.positive = positive ? 1 : 0;
  A.bit_alloc = bit_alloc ? 1 : 0;
  A.solve_f64 = solve_f64 ? 1 : 0;
  A.units_per_group = cliperr_units_per_group(outer, inner, channels_last);
  A.units = A.units_per_group * (channels_last ? (A.groups + fqb::kCeSlab - 1) / fqb::kCeSlab : A.groups);
  A.partial = static_cast<double*>(workspace);
  A.out = out;
  A.params = out_params;
  const int grid = grid_for(A.units, di->sms * (2048ull / fqb::kCeThreads), max_ctas);
  if (!channels_last && inner % 4 == 0 && aligned16(in)) fqb::fq_cliperr_partial_kernel<4><<<grid, fqb::kCeThreads, 0, st>>>(A);
  else                                                   fqb::fq_cliperr_partial_kernel<1><<<grid, fqb::kCeThreads, 0, st>>>(A);
  fqb::fq_cliperr_finish_kernel<<<static_cast<unsigned>(groups), fqb::kCeThreads, 0, st>>>(A);
  return launched("clipping-error kernels");
}

// the layouts and candidate counts fqb200_clip_mse takes (argument errors as a message, nullptr when they are fine)
static const char* clipmse_bad_args(int64_t outer, int64_t groups, int64_t inner, int channels_last, int32_t k) {
  const char* bad = cliperr_bad_args(outer, groups, inner, channels_last);
  if (bad) return bad;
  if (k < 1 || k > fqb::kCmMaxK) return "num_multipliers must be in 1..256%s";
  return nullptr;
}

size_t fqb200_clip_mse_workspace_bytes(int64_t outer, int64_t groups, int64_t inner, int32_t channels_last,
                                       int32_t num_multipliers) {
  g_err[0] = 0;
  const char* bad = clipmse_bad_args(outer, groups, inner, channels_last, num_multipliers);
  if (bad) return fail(FQB200_ERR_INVALID, bad), 0;
  return clipmse_workspace(outer, groups, inner, channels_last, num_multipliers);
}

int fqb200_clip_mse(const float* in, int64_t outer, int64_t groups, int64_t inner, int32_t channels_last, const float* stats,
                    int32_t num_bits, int32_t positive, int32_t bit_alloc, int32_t solve_f64, int32_t prior,
                    const float* multipliers, int32_t num_multipliers, double* out, float* out_params, void* workspace,
                    size_t workspace_bytes, int32_t max_ctas, void* stream) {
  return fqb200_clip_mse_widths(in, outer, groups, inner, channels_last, stats, num_bits, positive, bit_alloc, solve_f64, prior,
                                multipliers, nullptr, num_multipliers, out, out_params, workspace, workspace_bytes, max_ctas,
                                stream);
}

// the launch of fqb200_clip_mse_widths, fqb200_clip_mse_select and fqb200_clip_mse_grid after their argument checks: K
// candidates per unit, nw units per (group, chunk) - nw widths[i] of a grid launch, else 1 (widths, when given, one per
// candidate); with `choice`, the finish kernel also selects each group's candidate
static int clipmse_launch(const float* in, int64_t outer, int64_t groups, int64_t inner, int32_t channels_last,
                          const float* stats, int32_t num_bits, int32_t positive, int32_t bit_alloc, int32_t solve_f64,
                          int32_t prior, const float* multipliers, int32_t K, const int32_t* widths, int32_t nw, bool grid,
                          double* out, float* out_params, int32_t* choice, float* given, float* out_table,
                          void* workspace, size_t workspace_bytes, int32_t max_ctas, void* stream, const char* sizer) {
  int rc = check_workspace(workspace, workspace_bytes, clipmse_workspace(outer, groups, inner, channels_last, nw * K), sizer);
  if (rc != FQB200_OK) return rc;
  DeviceInfo* di = nullptr;
  rc = get_device(&di);
  if (rc != FQB200_OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  fqb::ClipMseArgs A;
  memset(&A, 0, sizeof(A));
  A.in = in;
  A.stats = stats;
  A.mult = multipliers;
  A.outer = static_cast<unsigned long long>(outer);
  A.groups = static_cast<unsigned long long>(groups);
  A.inner = static_cast<unsigned long long>(inner);
  A.channels_last = channels_last ? 1 : 0;
  A.num_bits = num_bits;
  A.positive = positive ? 1 : 0;
  A.bit_alloc = bit_alloc ? 1 : 0;
  A.solve_f64 = solve_f64 ? 1 : 0;
  A.prior = prior;
  A.K = K;
  A.Kpad = (K + fqb::kCmTile - 1) / fqb::kCmTile * fqb::kCmTile;
  A.has_widths = widths && !grid ? 1 : 0;
  A.grid = grid ? 1 : 0;
  A.nw = nw;
  for (int k = 0; widths && k < (grid ? nw : K); ++k) A.widths[k] = static_cast<unsigned char>(widths[k]);
  A.units_per_group = clipmse_units_per_group(outer, inner, channels_last);
  A.units = A.units_per_group * (channels_last ? (A.groups + fqb::kCmSlab - 1) / fqb::kCmSlab : A.groups) *
            static_cast<unsigned long long>(nw);
  A.partial = static_cast<double*>(workspace);
  A.out = out;
  A.params = out_params;
  A.choice = choice;
  A.given = given;
  A.table = out_table;
  const int grid_ctas = grid_for(A.units, di->sms * 2ull, max_ctas);
  if (channels_last) {
    fqb::fq_clipmse_partial_kernel<2><<<grid_ctas, fqb::kCmThreads, fqb::cm_smem_bytes(A.K, fqb::kCmSlab), st>>>(A);
  } else if (inner % 4 == 0 && aligned16(in)) {
    fqb::fq_clipmse_partial_kernel<1><<<grid_ctas, fqb::kCmThreads, fqb::cm_smem_bytes(A.K, 1), st>>>(A);
  } else {
    fqb::fq_clipmse_partial_kernel<0><<<grid_ctas, fqb::kCmThreads, fqb::cm_smem_bytes(A.K, 1), st>>>(A);
  }
  fqb::fq_clipmse_finish_kernel<<<static_cast<unsigned>(groups), fqb::kCmThreads, 0, st>>>(A);
  return launched("clipping-MSE kernels");
}

// fqb200_clip_mse_widths' argument checks, then its launch (with a selection when `choice` is given)
static int clipmse_checked(const float* in, int64_t outer, int64_t groups, int64_t inner, int32_t channels_last,
                           const float* stats, int32_t num_bits, int32_t positive, int32_t bit_alloc, int32_t solve_f64,
                           int32_t prior, const float* multipliers, const int32_t* widths, int32_t num_multipliers,
                           double* out, float* out_params, int32_t* choice, float* given, float* out_table, void* workspace,
                           size_t workspace_bytes, int32_t max_ctas, void* stream) {
  const char* bad = clipmse_bad_args(outer, groups, inner, channels_last, num_multipliers);
  if (bad) return fail(FQB200_ERR_INVALID, bad);
  if (!in || !stats || !multipliers || !out) return fail(FQB200_ERR_INVALID, "null pointer%s");
  if (num_bits < 1 || num_bits > 8) return fail(FQB200_ERR_INVALID, "num_bits must be in 1..8%s");
  if (bit_alloc && num_bits > 4) return fail(FQB200_ERR_INVALID, "bit_alloc applies to num_bits <= 4 only%s");
  if (widths) {
    if (prior < 0 || prior > 2) return fail(FQB200_ERR_INVALID, "prior must be 0 (Laplace b), 1 (Gauss std) or 2 (min/max)%s");
    if (bit_alloc) return fail(FQB200_ERR_INVALID, "widths and bit_alloc are two sources of widths: pass one%s");
    for (int k = 0; k < num_multipliers; ++k)
      if (widths[k] < 0 || widths[k] > 8) return fail(FQB200_ERR_INVALID, "widths must be in 0..8%s");
  } else {
    if (prior == 2) return fail(FQB200_ERR_INVALID, "prior 2 (min/max) ignores the multipliers: it needs widths%s");
    if (prior != 0 && prior != 1) return fail(FQB200_ERR_INVALID, "prior must be 0 (Laplace b) or 1 (Gauss std)%s");
  }
  if (max_ctas < 0) return fail(FQB200_ERR_INVALID, "max_ctas must be >= 0%s");
  return clipmse_launch(in, outer, groups, inner, channels_last, stats, num_bits, positive, bit_alloc, solve_f64, prior,
                        multipliers, num_multipliers, widths, 1, false, out, out_params, choice, given, out_table, workspace,
                        workspace_bytes, max_ctas, stream, "fqb200_clip_mse_workspace_bytes");
}

int fqb200_clip_mse_widths(const float* in, int64_t outer, int64_t groups, int64_t inner, int32_t channels_last,
                           const float* stats, int32_t num_bits, int32_t positive, int32_t bit_alloc, int32_t solve_f64,
                           int32_t prior, const float* multipliers, const int32_t* widths, int32_t num_multipliers,
                           double* out, float* out_params, void* workspace, size_t workspace_bytes, int32_t max_ctas,
                           void* stream) {
  g_err[0] = 0;
  return clipmse_checked(in, outer, groups, inner, channels_last, stats, num_bits, positive, bit_alloc, solve_f64, prior,
                         multipliers, widths, num_multipliers, out, out_params, nullptr, nullptr, nullptr, workspace,
                         workspace_bytes, max_ctas, stream);
}

int fqb200_clip_mse_select(const float* in, int64_t outer, int64_t groups, int64_t inner, int32_t channels_last,
                           const float* stats, int32_t num_bits, int32_t positive, int32_t bit_alloc, int32_t solve_f64,
                           int32_t prior, const float* multipliers, int32_t num_multipliers, double* out, float* out_params,
                           int32_t* choice, float* given, float* out_table, void* workspace, size_t workspace_bytes,
                           int32_t max_ctas, void* stream) {
  g_err[0] = 0;
  if (!choice || !given) return fail(FQB200_ERR_INVALID, "null pointer%s");
  return clipmse_checked(in, outer, groups, inner, channels_last, stats, num_bits, positive, bit_alloc, solve_f64, prior,
                         multipliers, nullptr, num_multipliers, out, out_params, choice, given, out_table, workspace,
                         workspace_bytes, max_ctas, stream);
}

// the layouts, multiplier and width counts fqb200_clip_mse_grid takes (argument errors as a message, nullptr when fine)
static const char* clipmse_grid_bad_args(int64_t outer, int64_t groups, int64_t inner, int channels_last, int32_t m,
                                         int32_t w) {
  const char* bad = clipmse_bad_args(outer, groups, inner, channels_last, m);
  if (bad) return bad;
  if (w < 1 || w > 9) return "num_widths must be in 1..9%s";
  return nullptr;
}

size_t fqb200_clip_mse_grid_workspace_bytes(int64_t outer, int64_t groups, int64_t inner, int32_t channels_last,
                                            int32_t num_multipliers, int32_t num_widths) {
  g_err[0] = 0;
  const char* bad = clipmse_grid_bad_args(outer, groups, inner, channels_last, num_multipliers, num_widths);
  if (bad) return fail(FQB200_ERR_INVALID, bad), 0;
  return clipmse_workspace(outer, groups, inner, channels_last, num_widths * num_multipliers);
}

int fqb200_clip_mse_grid(const float* in, int64_t outer, int64_t groups, int64_t inner, int32_t channels_last,
                         const float* stats, int32_t num_bits, int32_t positive, int32_t bit_alloc, int32_t solve_f64,
                         int32_t prior, const float* multipliers, int32_t num_multipliers, const int32_t* widths,
                         int32_t num_widths, double* out, float* out_params, void* workspace, size_t workspace_bytes,
                         int32_t max_ctas, void* stream) {
  g_err[0] = 0;
  const char* bad = clipmse_grid_bad_args(outer, groups, inner, channels_last, num_multipliers, num_widths);
  if (bad) return fail(FQB200_ERR_INVALID, bad);
  if (!in || !stats || !multipliers || !widths || !out) return fail(FQB200_ERR_INVALID, "null pointer%s");
  if (num_bits < 1 || num_bits > 8) return fail(FQB200_ERR_INVALID, "num_bits must be in 1..8%s");
  if (bit_alloc) return fail(FQB200_ERR_INVALID, "widths and bit_alloc are two sources of widths: pass one%s");
  if (prior != 0 && prior != 1)
    return fail(FQB200_ERR_INVALID, "prior must be 0 (Laplace b) or 1 (Gauss std): min/max ignores the multipliers%s");
  unsigned seen = 0;
  for (int i = 0; i < num_widths; ++i) {
    if (widths[i] < 0 || widths[i] > 8) return fail(FQB200_ERR_INVALID, "widths must be in 0..8%s");
    if (seen & (1u << widths[i])) return fail(FQB200_ERR_INVALID, "widths must be distinct%s");
    seen |= 1u << widths[i];
  }
  if (max_ctas < 0) return fail(FQB200_ERR_INVALID, "max_ctas must be >= 0%s");
  return clipmse_launch(in, outer, groups, inner, channels_last, stats, num_bits, positive, 0, solve_f64, prior,
                        multipliers, num_multipliers, widths, num_widths, true, out, out_params, nullptr, nullptr, nullptr,
                        workspace, workspace_bytes, max_ctas, stream, "fqb200_clip_mse_grid_workspace_bytes");
}

// the requests fqb200_kmeans1d takes (argument errors as a message, nullptr when they are fine)
static const char* kmeans_bad_args(int64_t n, int32_t k) {
  if (k < 2 || k > fqb::kKmMaxK || (k & (k - 1))) return "k must be a power of two, 2 .. 256%s";
  if (n < k) return "n must be >= k (scikit-learn raises for fewer samples than clusters)%s";
  if (n >= (1ll << 40)) return "n must be < 2^40%s";
  return nullptr;
}

size_t fqb200_kmeans1d_workspace_bytes(int64_t n, int32_t k) {
  g_err[0] = 0;
  const char* bad = kmeans_bad_args(n, k);
  if (bad) return fail(FQB200_ERR_INVALID, bad), 0;
  return kmeans_carve(nullptr, static_cast<unsigned long long>(n), k, nullptr);
}

int fqb200_kmeans1d(const float* in, int64_t n, int32_t num_bits, int64_t first_id, const double* draws, int32_t n_trials,
                    const double* init, int32_t task, int64_t rows, uint8_t* out_labels, float* out_centres,
                    double* out_inertia, int32_t* out_n_iter, int64_t* out_init_ids, float* out, float* out_bcorr,
                    void* workspace, size_t workspace_bytes, int32_t max_ctas, void* stream) {
  g_err[0] = 0;
  if (num_bits < 1 || num_bits > 8) return fail(FQB200_ERR_INVALID, "num_bits must be in 1..8%s");
  const int k = 1 << num_bits;
  const char* bad = kmeans_bad_args(n, k);
  if (bad) return fail(FQB200_ERR_INVALID, bad);
  if (!in || !out_labels || !out_centres || !out_inertia || !out_n_iter) return fail(FQB200_ERR_INVALID, "null pointer%s");
  if (task != FQB200_KMEANS_NONE && task != FQB200_KMEANS_QUANTIZE && task != FQB200_KMEANS_CLIP)
    return fail(FQB200_ERR_INVALID, "task must be FQB200_KMEANS_NONE, _QUANTIZE or _CLIP%s");
  if (task != FQB200_KMEANS_NONE && !out) return fail(FQB200_ERR_INVALID, "a task needs `out`%s");
  if (rows < 0) return fail(FQB200_ERR_INVALID, "rows must be >= 0%s");
  if (rows > 0 && (task == FQB200_KMEANS_NONE || !out_bcorr || n % rows != 0))
    return fail(FQB200_ERR_INVALID, "rows > 0 needs a task, out_bcorr and n %% rows == 0%s");
  if (!init) {
    if (!draws) return fail(FQB200_ERR_INVALID, "k-means++ needs the draws (or pass init)%s");
    if (first_id < 0 || first_id >= n) return fail(FQB200_ERR_INVALID, "first_id must be in 0 .. n - 1%s");
    if (n_trials < 1 || n_trials > 7) return fail(FQB200_ERR_INVALID, "n_trials must be in 1..7%s");
  }
  if (max_ctas < 0) return fail(FQB200_ERR_INVALID, "max_ctas must be >= 0%s");
  fqb::KmArgs A;
  memset(&A, 0, sizeof(A));
  const size_t need = kmeans_carve(static_cast<char*>(workspace), static_cast<unsigned long long>(n), k, &A);
  int rc = check_workspace(workspace, workspace_bytes, need, "fqb200_kmeans1d_workspace_bytes");
  if (rc != FQB200_OK) return rc;
  DeviceInfo* di = nullptr;
  rc = get_device(&di);
  if (rc != FQB200_OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  A.in = in;
  A.T = init ? 1 : n_trials;
  A.task = task;
  A.given = init ? 1 : 0;
  A.first_id = init ? 0 : first_id;
  A.draws = draws;
  A.init = init;
  A.rows = static_cast<unsigned long long>(rows);
  A.labels = out_labels;
  A.centres = out_centres;
  A.inertia = out_inertia;
  A.n_iter = out_n_iter;
  A.init_ids = init ? nullptr : reinterpret_cast<long long*>(out_init_ids);
  A.out = out;
  A.out_bcorr = out_bcorr;
  const void* fn = reinterpret_cast<const void*>(fqb::fq_kmeans_kernel);
  const size_t smem = kmeans_smem(k);
  int per_sm = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, fqb::kThreads, smem);
  if (e != cudaSuccess || per_sm < 1) return fail(FQB200_ERR_CUDA, "k-means kernel setup: %s", cudaGetErrorString(e));
  const unsigned long long resident = static_cast<unsigned long long>(di->sms) * per_sm;
  const int grid = grid_for(resident, resident, max_ctas);
  // barrier words and control block start at zero
  e = cudaMemsetAsync(workspace, 0, reinterpret_cast<char*>(A.col) - static_cast<char*>(workspace), st);
  if (e == cudaSuccess && init && out_init_ids) e = cudaMemsetAsync(out_init_ids, 0xff, static_cast<size_t>(k) * 8, st);
  if (e != cudaSuccess) return fail(FQB200_ERR_CUDA, "cudaMemsetAsync: %s", cudaGetErrorString(e));
  void* args[] = {&A};
  e = cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(fqb::kThreads), args, smem, st);
  if (e != cudaSuccess) return fail(FQB200_ERR_CUDA, "cooperative launch fq_kmeans_kernel: %s", cudaGetErrorString(e));
  return FQB200_OK;
}

// The descriptor of the RANGE_MINMAX weight launch whose plan fqb200_quantize_weights_given runs: bits given = that
// launch with bit allocation (prior std), so the phases, their walking directions and the workspace are the same.
static fqb200_desc weights_given_desc(int64_t groups, int64_t inner, int32_t num_bits, bool has_bits, int32_t bias_corr,
                                      int32_t var_corr, unsigned long long* hist) {
  fqb200_desc d;
  memset(&d, 0, sizeof(d));
  d.outer = 1;
  d.groups = groups;
  d.inner = inner;
  d.scope = FQB200_SCOPE_GROUP;
  d.range_mode = FQB200_RANGE_MINMAX;
  d.leaf = FQB200_LEAF_TORCH;
  d.num_bits = num_bits;
  d.bit_alloc = has_bits ? 1 : 0;
  d.bit_alloc_prior = FQB200_PRIOR_STD;
  d.bit_alloc_round = 1;
  d.bit_alloc_target = static_cast<float>(num_bits);
  d.bias_corr = bias_corr ? 1 : 0;
  d.var_corr = var_corr ? 1 : 0;
  d.out_hist = hist;
  return d;
}

static const char* weights_given_bad_args(int64_t groups, int64_t inner, int32_t num_bits) {
  if (groups < 0 || inner < 0) return "negative extent%s";
  if (num_bits < 1 || num_bits > 8) return "num_bits must be in 1..8%s";
  return nullptr;
}

size_t fqb200_quantize_weights_given_workspace_bytes(int64_t groups, int64_t inner, int32_t num_bits, int32_t has_bits,
                                                     int32_t bias_corr, int32_t var_corr) {
  g_err[0] = 0;
  const char* bad = weights_given_bad_args(groups, inner, num_bits);
  if (bad) return fail(FQB200_ERR_INVALID, bad), 0;
  const fqb200_desc d = weights_given_desc(groups, inner, num_bits, has_bits != 0, bias_corr, var_corr, nullptr);
  return fqb200_workspace_bytes(&d);
}

int fqb200_quantize_weights_given(const float* in, float* out, int64_t groups, int64_t inner, const float* delta,
                                  const float* offset, const float* bits, int32_t num_bits, int32_t bias_corr,
                                  int32_t var_corr, unsigned long long* hist, void* workspace, size_t workspace_bytes,
                                  void* stream) {
  g_err[0] = 0;
  const char* bad = weights_given_bad_args(groups, inner, num_bits);
  if (bad) return fail(FQB200_ERR_INVALID, bad);
  if (!in || !out || !delta || !offset) return fail(FQB200_ERR_INVALID, "null pointer%s");
  if (groups == 0 || inner == 0) return FQB200_OK;
  const fqb200_desc d = weights_given_desc(groups, inner, num_bits, bits != nullptr, bias_corr, var_corr, hist);
  DeviceInfo* di = nullptr;
  int rc = get_device(&di);
  if (rc != FQB200_OK) return rc;
  FusedPlan fp;
  rc = plan_fused(&d, aligned16(in) && aligned16(out), 0, *di, &fp);
  if (rc != FQB200_OK) return rc;
  rc = check_workspace(workspace, workspace_bytes, fp.workspace, "fqb200_quantize_weights_given_workspace_bytes");
  if (rc != FQB200_OK) return rc;
  carve(static_cast<char*>(workspace), fp.slots, fp.pl.geo.channels, &fp.A);
  fp.A.in = in;
  fp.A.out = out;
  fp.A.g_delta = delta;
  fp.A.g_offset = offset;
  fp.A.g_bits = bits;
  fp.A.given_per_group = 1;
  void* args[] = {&fp.A};
  const cudaError_t e = cudaLaunchCooperativeKernel(fp.kernel, dim3(fp.pl.grid), dim3(fp.block), args, fp.smem,
                                                    static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return fail(FQB200_ERR_CUDA, "cooperative launch %s: %s", fp.name, cudaGetErrorString(e));
  return FQB200_OK;
}

// bit_alloc.allocate's budget: min(floor(target * G), 8 G); -1 when it is negative or not a number
static int64_t alloc_budget(int64_t groups, double target) {
  const double b = floor(target * static_cast<double>(groups));
  if (!(b >= 0.0)) return -1;
  return b < 8.0 * static_cast<double>(groups) ? static_cast<int64_t>(b) : 8 * groups;
}

static const char* alloc_bad_args(int64_t groups, double target) {
  if (groups < 1 || groups > fqb::kAllocMaxGroups) return "groups must be in 1..2^20%s";
  if (alloc_budget(groups, target) < 0) return "target gives a negative budget%s";
  return nullptr;
}

// choice table G x (budget + 1) bytes, then the two best[] rows when they do not fit in shared memory
static size_t alloc_choice_bytes(int64_t groups, int64_t budget) {
  return (static_cast<size_t>(groups) * static_cast<size_t>(budget + 1) + 15u) & ~static_cast<size_t>(15u);
}
static bool alloc_rows_in_smem(int64_t budget) { return 2u * static_cast<size_t>(budget + 1) * sizeof(double) <= fqb::kAllocMaxSmem; }

size_t fqb200_allocate_widths_workspace_bytes(int64_t groups, double target) {
  g_err[0] = 0;
  const char* bad = alloc_bad_args(groups, target);
  if (bad) return fail(FQB200_ERR_INVALID, bad), 0;
  const int64_t budget = alloc_budget(groups, target);
  return alloc_choice_bytes(groups, budget) + (alloc_rows_in_smem(budget) ? 0u : 2u * static_cast<size_t>(budget + 1) * sizeof(double));
}

int fqb200_allocate_widths(const double* sse, int64_t groups, double target, float* widths_out, int32_t* status,
                           void* workspace, size_t workspace_bytes, void* stream) {
  g_err[0] = 0;
  const char* bad = alloc_bad_args(groups, target);
  if (bad) return fail(FQB200_ERR_INVALID, bad);
  if (!sse || !widths_out) return fail(FQB200_ERR_INVALID, "null pointer%s");
  const int64_t budget = alloc_budget(groups, target);
  const bool in_smem = alloc_rows_in_smem(budget);
  const size_t choice = alloc_choice_bytes(groups, budget);
  int rc = check_workspace(workspace, workspace_bytes, fqb200_allocate_widths_workspace_bytes(groups, target),
                           "fqb200_allocate_widths_workspace_bytes");
  if (rc != FQB200_OK) return rc;
  const size_t smem = in_smem ? 2u * static_cast<size_t>(budget + 1) * sizeof(double) : 0u;
  cudaError_t e = setup(fqb::fq_allocate_widths_kernel, fqb::kAllocThreads, smem);
  if (e != cudaSuccess) return fail(FQB200_ERR_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
  unsigned char* ws = static_cast<unsigned char*>(workspace);
  double* rows = in_smem ? nullptr : reinterpret_cast<double*>(ws + choice);
  fqb::fq_allocate_widths_kernel<<<1, fqb::kAllocThreads, smem, static_cast<cudaStream_t>(stream)>>>(
      sse, static_cast<unsigned>(groups), static_cast<unsigned>(budget), ws, rows, widths_out, status);
  return launched("fq_allocate_widths_kernel");
}

int fqb200_selftest_division(const float* a, const float* b, float* fast, float* ieee, int64_t n, void* stream) {
  if (n <= 0) return FQB200_OK;
  fqb::fq_divtest_kernel<<<296, 256, 0, static_cast<cudaStream_t>(stream)>>>(a, b, fast, ieee, static_cast<unsigned long long>(n));
  return launched("");
}

}  // extern "C"
