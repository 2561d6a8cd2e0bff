// Channels-last (NHWC) activations: ONE cooperative launch per hooked tensor on the bulk-copy engine of fq_bulk.cuh.
// Included by fqb200.cu after FusedArgs / the solve_* helpers / leaf_apply (namespace fqb).
//
// [N][H*W][C] in memory, the channel is the fastest dimension: the tensor is one flat stream of N*H*W*C/4 vectors and,
// because the consumer stride is a multiple of C/4, thread t always holds the same four channels (4 * (t mod C/4)).
// Per-channel accumulators and leaf parameters therefore live in registers for a whole phase.
//
//   S1   read x         per channel min, max, S = sum (x - k), Q = sum (x - k)^2 with the common shift k = the channel's
//                       value at pixel 0 (exact for constant channels, well conditioned otherwise): mean AND std from
//                       one pass (SURVEY 8d allows it; the reference's second std pass is not reproduced)
//   S2   read x         sum |x - mean32|  (only when the Laplace b is needed)
//   A    read x, write  quantize - clip - dequantize
//
// No leader sections on the critical path (they cost time on every launch, mostly cold instruction fetch of code that
// ONE CTA ran once): CTAs meet in replicated per-channel accumulators (atomics), a plain grid barrier
// follows, and then every CTA derives what it needs for ITS channels itself.  The one global computation - bit
// allocation / mid-tread bin allocation, which needs the std of every channel - runs in CTA 0 while the other CTAs
// stream phase S2, and is published before CTA 0 arrives at the second barrier.
//
// Accumulators are double-banked by launch parity: a launch uses the bank the previous launch of this workspace left
// zeroed and zeroes the other one in passing, so nothing on the critical path re-arms them.
#pragma once

namespace fqb {

__device__ __forceinline__ unsigned enc_ordered(float x) {
  const unsigned b = __float_as_uint(x);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float dec_ordered(unsigned e) {
  return __uint_as_float((e & 0x80000000u) ? (e & 0x7fffffffu) : ~e);
}

// accumulator bank layout (element offsets into A.acc_u / A.acc_d of one bank)
constexpr unsigned kAccU = 2u * kMaxNhwcChannels;  // min (inverted encoding), max
constexpr unsigned kAccD = 3u * kMaxNhwcChannels;  // S, Q, sum |x - mean|

struct ClView {
  unsigned* amin_inv;
  unsigned* amax;
  double* asum;
  double* asq;
  double* aabs;
};
__device__ __forceinline__ ClView cl_view(const FusedArgs& A, unsigned bank) {
  ClView v;
  v.amin_inv = A.amin_inv + bank * kAccU;
  v.amax = v.amin_inv + kMaxNhwcChannels;
  v.asum = A.asum + bank * kAccD;
  v.asq = v.asum + kMaxNhwcChannels;
  v.aabs = v.asq + kMaxNhwcChannels;
  return v;
}

// fire-and-forget reductions on global memory (no generic-address fallback, no return value)
__device__ __forceinline__ void red_add_f64(double* p, double v) {
  asm volatile("red.global.add.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}
__device__ __forceinline__ void red_max_u32(unsigned* p, unsigned v) {
  asm volatile("red.global.max.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// plain grid barrier over the consumer threads of every CTA: the last CTA to arrive releases the others
// Split in two so that a CTA can do useful (instruction-cache warming) work between posting its arrival and waiting.
// Memory ordering: release / acquire at GPU scope on the arrival counter and the release word (cumulative over the CTA
// barrier in front), NOT __threadfence(): that is fence.sc.gpu, and a sequentially-consistent fence issued while the other
// CTAs stream at full bandwidth waits for their traffic (debug stamps "aux: iterations" -> "aux solved").
__device__ __noinline__ void grid_arrive_cl(GridSync* gs, unsigned& epoch) {
  ++epoch;
  consumer_sync();
  if (threadIdx.x == 0) {
    unsigned prev;
    asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], 1;" : "=r"(prev) : "l"(&gs->arrive) : "memory");
    if (prev + 1u == epoch * gridDim.x) st_release_u32(&gs->release, epoch);
  }
}
__device__ __noinline__ void grid_wait_cl(GridSync* gs, unsigned epoch) {
  if (threadIdx.x == 0) {
    while (ld_acquire_u32(&gs->release) < epoch) __nanosleep(32);
  }
  consumer_sync();
}
__device__ __forceinline__ void grid_barrier_cl(GridSync* gs, unsigned& epoch) {
  grid_arrive_cl(gs, epoch);
  grid_wait_cl(gs, epoch);
}
__device__ __forceinline__ void grid_exit_cl(GridSync* gs) {
  consumer_sync();
  if (threadIdx.x == 0) {
    const unsigned prev = atomicAdd(&gs->exited, 1u);
    if (prev + 1u == gridDim.x) {
      gs->arrive = 0u;
      gs->release = 0u;
      for (int i = 0; i < 8; ++i) gs->unit_counter[i] = 0u;
      gs->launch_count = gs->launch_count + 1u;  // flips the accumulator bank, retires aux_ready
      __threadfence();
      gs->exited = 0u;
    }
  }
}

// ---- per-phase accumulators ---------------------------------------------------------------------------------------------
// Stages summed in fp32 before folding into float64: ONE.  A thread reads the same vectors of a stage in the same order
// whichever CTA consumes it, so a one-stage chunk is a fixed set of elements summed in a fixed order; chunks spanning two
// stages would pair whatever stages the dynamic work assignment gave a CTA, and the fp32 rounding of the pair (~1e-7)
// would differ from run to run - enough to move a bit width that sits on its rounding boundary.  What remains
// order-dependent is the float64 accumulation of the chunks (~1e-16 relative), far below fp32 resolution.
constexpr unsigned kClChunkStages = 1;

// S1 runs on the RAW values (the bias is a per-channel constant): min / max of x + bias are (min x) + bias and
// (max x) + bias exactly (rounding is monotone), and mean / std of fl(x + bias) equal mean(x) + bias / std(x) up to the
// rounding of single elements (~1e-8 relative, far inside the fp32 statistics of the reference itself).  That saves four
// registers and one instruction per element in the phase that reads HBM.
struct ClStats1 {
  float mn[4], mx[4], k[4], fs[4], fq[4];
  double s[4], q[4];
  unsigned cnt;
  __device__ __forceinline__ void init(const FusedArgs& A, unsigned c0, bool active) {
    // common shift: the channel's value at pixel 0, the same bits in every thread of every CTA
    float4 first = make_float4(0.f, 0.f, 0.f, 0.f);
    if (active) first = ld_tensor(reinterpret_cast<const float4*>(A.in) + (c0 >> 2));
    k[0] = first.x;
    k[1] = first.y;
    k[2] = first.z;
    k[3] = first.w;
    cnt = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      mn[i] = INFINITY;
      mx[i] = -INFINITY;
      fs[i] = 0.f;
      fq[i] = 0.f;
      s[i] = 0.0;
      q[i] = 0.0;
    }
  }
  __device__ __forceinline__ void flush() {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      s[i] += static_cast<double>(fs[i]);
      q[i] += static_cast<double>(fq[i]);
      fs[i] = 0.f;
      fq[i] = 0.f;
    }
    cnt = 0;
  }
  __device__ __forceinline__ void consume(const float4& v, unsigned) {
    const float x[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float d = __fsub_rn(x[i], k[i]);
      mn[i] = fminf(mn[i], x[i]);
      mx[i] = fmaxf(mx[i], x[i]);
      fs[i] = __fadd_rn(fs[i], d);
      fq[i] = __fmaf_rn(d, d, fq[i]);
    }
  }
  __device__ __forceinline__ void stage_end(const StageMeta&) {
    if (++cnt == kClChunkStages) flush();
  }
};

struct ClStats2 {
  float mu[4], bias[4], fa[4];
  double sa[4];
  unsigned cnt;
  __device__ __forceinline__ void init(const FusedArgs& A, unsigned c0, bool active, const float (&mean)[4]) {
    cnt = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      bias[i] = (A.bias && active) ? __ldg(A.bias + c0 + i) : 0.f;
      mu[i] = mean[i];
      fa[i] = 0.f;
      sa[i] = 0.0;
    }
  }
  __device__ __forceinline__ void flush() {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      sa[i] += static_cast<double>(fa[i]);
      fa[i] = 0.f;
    }
    cnt = 0;
  }
  __device__ __forceinline__ void consume(const float4& v, unsigned) {
    const float x[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) fa[i] = __fadd_rn(fa[i], fabsf(__fsub_rn(__fadd_rn(x[i], bias[i]), mu[i])));
  }
  __device__ __forceinline__ void stage_end(const StageMeta&) {
    if (++cnt == kClChunkStages) flush();
  }
};

// `-me` (entropy of the integer grid, utils/entropy.py:6-17): the apply phase histograms the grid into shared memory.
// kHistWords counters per CTA, organised as `copies` replicas of `bins` counters (warp w uses replica w % copies): 16
// replicas of the torch leaf's 256 levels, fewer of the wider mid-tread grids.  Mid-tread grids are clamped to the
// per-channel, generally fractional bounds c_min / c_max (int_quantizer.py:207-214); elements sitting on a bound are
// counted per channel (they are distinct symbols for torch.unique) instead of in the integer histogram.
constexpr unsigned kHistWords = 8192;
static_assert(kHistWords * 4u <= kStageBytes, "the histogram borrows one ring stage");

template <int LEAF, bool HIST>
struct ClApply {
  const FusedArgs& A;
  unsigned* hist;  // [kHistWords] in shared memory (HIST)
  LeafParam q[4];
  float r[4], bias[4];
  unsigned nlo[4], nhi[4];  // HIST, mid-tread: elements on the lower / upper clamp bound of each channel
  unsigned hbase;           // this warp's replica
  bool fast;
  // the residual operand of the fused block epilogue, when it is quantized on the fly (fqb200_desc.residual_stats)
  LeafParam rq[4];
  float rr[4], rbias[4];
  bool rquant;
  __device__ __forceinline__ void init(unsigned c0, bool active, const LeafParam (&lp)[4]) {
    fast = true;
    rquant = A.residual != nullptr && A.residual_stats != nullptr;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      rq[i].a = 1.f;
      rq[i].b = 0.f;
      rq[i].c = 0.f;
      rq[i].flags = 0;
      rr[i] = 1.f;
      rbias[i] = 0.f;
      if (rquant && active) {
        const float* row = A.residual_stats + static_cast<size_t>(c0 + i) * FQB200_STATS_STRIDE;
        rq[i].a = __ldg(row + 8);
        rq[i].b = __ldg(row + 9);
        rq[i].c = __ldg(row + 10);
        rq[i].flags = static_cast<int>(__ldg(row + 11));
        const Divisor dr = make_divisor(rq[i].a);
        rr[i] = dr.r;
        fast = fast && dr.fast;
        if (A.residual_bias) rbias[i] = __ldg(A.residual_bias + c0 + i);
      }
    }
    const unsigned copies = max(1u, min(static_cast<unsigned>(kWarps), kHistWords / static_cast<unsigned>(max(A.hist_bins, 1))));
    hbase = ((threadIdx.x >> 5) % copies) * static_cast<unsigned>(A.hist_bins);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      q[i] = lp[i];
      const Divisor dv = make_divisor(q[i].a);
      r[i] = dv.r;
      fast = fast && dv.fast;
      bias[i] = (A.bias && active) ? __ldg(A.bias + c0 + i) : 0.f;
      nlo[i] = 0u;
      nhi[i] = 0u;
    }
  }
  __device__ __forceinline__ void count(int i, float gq) {
    if (LEAF == FQB200_LEAF_MIDTREAD) {
      if (gq == q[i].c) {
        ++nhi[i];
        return;
      }
      if (gq == q[i].b) {
        ++nlo[i];
        return;
      }
    }
    if (gq == gq) {  // NaN is not a symbol of the grid
      const float v = fminf(fmaxf(gq + static_cast<float>(A.hist_offset), 0.f), static_cast<float>(A.hist_bins - 1));
      atomicAdd(hist + hbase + static_cast<unsigned>(v), 1u);
    }
  }
  template <bool FAST, bool PAIR, bool RQ = false>
  __device__ __forceinline__ void one(const float4& v, const float4& rv, unsigned off) {
    const float x[4] = {v.x, v.y, v.z, v.w};
    float y[4], gq[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      Divisor dv;
      dv.s = q[i].a;
      dv.r = r[i];
      dv.fast = FAST;
      y[i] = leaf_apply<LEAF, FAST>(__fadd_rn(x[i], bias[i]), q[i], dv, 0.f, gq[i]);
    }
    if (PAIR) {  // the residual add (+ ReLU) that closes a ResNet block, on the quantized values
      float res[4] = {rv.x, rv.y, rv.z, rv.w};
      if (RQ) {  // the shortcut of a down-sampling block arrives raw: quantize it with its own parameters first
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          Divisor dr;
          dr.s = rq[i].a;
          dr.r = rr[i];
          dr.fast = FAST;
          float g2;
          res[i] = leaf_apply<LEAF, FAST>(__fadd_rn(res[i], rbias[i]), rq[i], dr, 0.f, g2);
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        y[i] = __fadd_rn(y[i], res[i]);
        if (A.residual_relu) y[i] = y[i] < 0.f ? 0.f : y[i];
      }
    }
    // a channel slice of a wider tensor (out_pad_v): `off` counts cv vectors per pixel, the output out_pad_v more
    const unsigned o = A.out_pad_v ? off + (off / A.flat.cv) * A.out_pad_v : off;
    st_tensor(reinterpret_cast<float4*>(A.out) + o, make_float4(y[0], y[1], y[2], y[3]));
    if (HIST) {
#pragma unroll
      for (int i = 0; i < 4; ++i) count(i, gq[i]);
    }
  }
  __device__ __forceinline__ void consume(const float4& v, unsigned off) {
    if (fast)
      one<true, false>(v, v, off);
    else
      one<false, false>(v, v, off);
  }
  // 2x2 max pooling in front of the leaf (consume_pool_phase): the leaf is monotone, so quantize(max) == max(quantize);
  // torch's NaN rule (a NaN in the window wins); the bias is a per-channel constant and commutes with the max as well
  template <bool FAST>
  __device__ __forceinline__ void pooled_one(const float4& a0, const float4& a1, const float4& b0, const float4& b1, unsigned off) {
    auto mx = [](float p, float q) { return (q > p || q != q) ? q : p; };
    const float m[4] = {mx(mx(mx(a0.x, a1.x), b0.x), b1.x), mx(mx(mx(a0.y, a1.y), b0.y), b1.y),
                        mx(mx(mx(a0.z, a1.z), b0.z), b1.z), mx(mx(mx(a0.w, a1.w), b0.w), b1.w)};
    float y[4], gq;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      Divisor dv;
      dv.s = q[i].a;
      dv.r = r[i];
      dv.fast = FAST;
      y[i] = leaf_apply<LEAF, FAST>(__fadd_rn(m[i], bias[i]), q[i], dv, 0.f, gq);
    }
    st_tensor(reinterpret_cast<float4*>(A.pool_out) + off, make_float4(y[0], y[1], y[2], y[3]));
  }
  __device__ __forceinline__ void pooled(const float4& a0, const float4& a1, const float4& b0, const float4& b1, unsigned off) {
    if (fast)
      pooled_one<true>(a0, a1, b0, b1, off);
    else
      pooled_one<false>(a0, a1, b0, b1, off);
  }
  // the same tap by tap (consume_pool3_phase: windows at the image border have fewer taps)
  float pm[4];
  __device__ __forceinline__ void pool_begin() {
#pragma unroll
    for (int i = 0; i < 4; ++i) pm[i] = -INFINITY;
  }
  __device__ __forceinline__ void pool_tap(const float4& v) {
    auto mx = [](float p, float q) { return (q > p || q != q) ? q : p; };
    pm[0] = mx(pm[0], v.x);
    pm[1] = mx(pm[1], v.y);
    pm[2] = mx(pm[2], v.z);
    pm[3] = mx(pm[3], v.w);
  }
  template <bool FAST>
  __device__ __forceinline__ void pool_end_one(unsigned off) {
    float y[4], gq;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      Divisor dv;
      dv.s = q[i].a;
      dv.r = r[i];
      dv.fast = FAST;
      y[i] = leaf_apply<LEAF, FAST>(__fadd_rn(pm[i], bias[i]), q[i], dv, 0.f, gq);
    }
    st_tensor(reinterpret_cast<float4*>(A.pool_out) + off, make_float4(y[0], y[1], y[2], y[3]));
  }
  __device__ __forceinline__ void pool_end(unsigned off) {
    if (fast)
      pool_end_one<true>(off);
    else
      pool_end_one<false>(off);
  }
  // the residual comes through the ring next to x (consume_pair_phase)
  __device__ __forceinline__ void consume2(const float4& v, const float4& rv, unsigned off) {
    if (rquant) {
      if (fast)
        one<true, true, true>(v, rv, off);
      else
        one<false, true, true>(v, rv, off);
    } else if (fast) {
      one<true, true>(v, rv, off);
    } else {
      one<false, true>(v, rv, off);
    }
  }
  __device__ __forceinline__ void stage_end(const StageMeta&) {}
};

// ---- CTA-wide combine of per-thread channel partials, then one reduction per channel into the replicated accumulators ----
// buf: 16 KB of shared memory.  Threads sharing a column (t, t + cv, ...) are reduced by the column's owner items
// (item it -> column it % cv, channel-in-column it / cv; <= 4 items per thread since 4 * cv <= 2048).  The staging rounds
// keep their results in registers and ALL the global reductions are issued at the very end: a CTA barrier behind a batch
// of `red.global` waits for them (every round would pay that wait with the reductions inside the rounds).
constexpr unsigned kClItems = 4;

template <typename T, typename Op>
__device__ __forceinline__ void cl_stage_round(unsigned char* buf, unsigned cv, unsigned stride, const T (&v)[4], T identity, Op op,
                                               T (&res)[kClItems]) {
  T* st = reinterpret_cast<T*>(buf);  // [4][kConsumers]
  consumer_sync();
#pragma unroll
  for (int i = 0; i < 4; ++i) st[i * kConsumers + threadIdx.x] = (threadIdx.x < stride) ? v[i] : identity;
  consumer_sync();
#pragma unroll
  for (unsigned k = 0; k < kClItems; ++k) {
    const unsigned it = threadIdx.x + k * kConsumers;
    T a = identity;
    if (it < 4u * cv) {
      const unsigned col = it % cv, i = it / cv;
      for (unsigned t = col; t < stride; t += cv) a = op(a, st[i * kConsumers + t]);
    }
    res[k] = a;
  }
}

// S1: (min, max) as one uint2 round, S and Q one round each, then the reductions
__device__ __noinline__ void cl_combine_s1(unsigned char* buf, unsigned cv, unsigned stride, const unsigned (&umn)[4],
                                           const unsigned (&umx)[4], const double (&s)[4], const double (&q)[4], unsigned* dmn,
                                           unsigned* dmx, double* ds, double* dq) {
  if (cv == stride) {  // every active thread owns its column alone (C = 2048 with 512 threads): no staging
    if (threadIdx.x < stride) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const unsigned c = 4u * threadIdx.x + i;
        red_max_u32(dmn + c, umn[i]);
        red_max_u32(dmx + c, umx[i]);
        red_add_f64(ds + c, s[i]);
        red_add_f64(dq + c, q[i]);
      }
    }
    return;
  }
  uint2 mm[4], rmm[kClItems];
#pragma unroll
  for (int i = 0; i < 4; ++i) mm[i] = make_uint2(umn[i], umx[i]);
  auto max2 = [](uint2 a, uint2 b) { return make_uint2(a.x > b.x ? a.x : b.x, a.y > b.y ? a.y : b.y); };
  double rs[kClItems], rq[kClItems];
  cl_stage_round(buf, cv, stride, mm, make_uint2(0u, 0u), max2, rmm);
  cl_stage_round(buf, cv, stride, s, 0.0, OpAdd(), rs);
  cl_stage_round(buf, cv, stride, q, 0.0, OpAdd(), rq);
#pragma unroll
  for (unsigned k = 0; k < kClItems; ++k) {
    const unsigned it = threadIdx.x + k * kConsumers;
    if (it < 4u * cv) {
      const unsigned c = 4u * (it % cv) + it / cv;
      red_max_u32(dmn + c, rmm[k].x);
      red_max_u32(dmx + c, rmm[k].y);
      red_add_f64(ds + c, rs[k]);
      red_add_f64(dq + c, rq[k]);
    }
  }
}
// up to three float64 sums (S2: one, `-bca`: three)
__device__ __noinline__ void cl_combine_add_f64(unsigned char* buf, unsigned cv, unsigned stride, const double (&v0)[4], double* d0,
                                                const double (&v1)[4], double* d1, const double (&v2)[4], double* d2) {
  if (cv == stride) {
    if (threadIdx.x < stride) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const unsigned c = 4u * threadIdx.x + i;
        red_add_f64(d0 + c, v0[i]);
        if (d1) red_add_f64(d1 + c, v1[i]);
        if (d2) red_add_f64(d2 + c, v2[i]);
      }
    }
    return;
  }
  double r0[kClItems], r1[kClItems], r2[kClItems];
  cl_stage_round(buf, cv, stride, v0, 0.0, OpAdd(), r0);
  if (d1) cl_stage_round(buf, cv, stride, v1, 0.0, OpAdd(), r1);
  if (d2) cl_stage_round(buf, cv, stride, v2, 0.0, OpAdd(), r2);
#pragma unroll
  for (unsigned k = 0; k < kClItems; ++k) {
    const unsigned it = threadIdx.x + k * kConsumers;
    if (it < 4u * cv) {
      const unsigned c = 4u * (it % cv) + it / cv;
      red_add_f64(d0 + c, r0[k]);
      if (d1) red_add_f64(d1 + c, r1[k]);
      if (d2) red_add_f64(d2 + c, r2[k]);
    }
  }
}

// sum over the (<= 8) replicas of one accumulator entry: all loads issued before the first add (they are slow L2 round
// trips while the other CTAs stream)
template <typename T, typename Op>
__device__ __forceinline__ T cl_rep_reduce(const T* p, unsigned rep, unsigned C, unsigned c, T identity, Op op) {
  T v[8];
#pragma unroll
  for (unsigned r = 0; r < 8u; ++r) v[r] = (r < rep) ? ld_ws(p + r * C + c) : identity;
  return op(op(op(v[0], v[1]), op(v[2], v[3])), op(op(v[4], v[5]), op(v[6], v[7])));
}
__device__ __forceinline__ double cl_mean(const ClView& acc, unsigned rep, unsigned C, unsigned c, float k, float bias, double n) {
  const double s = cl_rep_reduce(acc.asum, rep, C, c, 0.0, OpAdd());
  return static_cast<double>(k) + static_cast<double>(bias) + s / n;
}
// unbiased std of channel c: sqrt((Q - S^2 / n) / (n - 1))
__device__ __forceinline__ float cl_std(const ClView& acc, unsigned rep, unsigned C, unsigned c, double n) {
  const double s = cl_rep_reduce(acc.asum, rep, C, c, 0.0, OpAdd());
  const double q = cl_rep_reduce(acc.asq, rep, C, c, 0.0, OpAdd());
  double m2 = q - s * s / n;
  if (m2 < 0.0) m2 = 0.0;
  return static_cast<float>(sqrt(m2 / (n - 1.0)));
}

// mid-tread parameters of one channel from its bin count omega: int_quantizer.py:185-214 (+ :137-145)
__device__ __forceinline__ LeafParam mid_tread_param(const FusedArgs& A, float omega, float mn, float mx, float mu, float b,
                                                     float& rng) {
  const bool sym = !A.positive;
  if (A.mt_clip) {
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
  return q;
}

// CTA 0, all consumer threads: the one computation that needs every channel - per-channel bit widths (int_quantizer.py:
// 381-407) or mid-tread bin counts (:128-135) from the per-channel std (prior 'gaus') or b (prior 'laplace') - into
// A.gbits, then the aux_ready flag.
__device__ __noinline__ void cl_solve_aux(const FusedArgs& A, const ClView& acc, LeaderSmem& sm, unsigned tag, bool have_b,
                                          bool publish) {
  const unsigned C = A.flat.channels;
  const double n = A.n_per_group;
  const bool prior_b = (A.leaf != FQB200_LEAF_MIDTREAD) && A.prior == FQB200_PRIOR_B;
  for (unsigned c = threadIdx.x; c < C; c += kConsumers) {
    if (prior_b) {
      const double sa = have_b ? cl_rep_reduce(acc.aabs, A.nhwc_rep, C, c, 0.0, OpAdd()) : 0.0;
      A.gb[c] = static_cast<float>(sa / n);
    } else {
      A.gstd[c] = cl_std(acc, A.nhwc_rep, C, c, n);
    }
  }
  consumer_sync();
  stamp(A, 10);
  if (A.leaf == FQB200_LEAF_MIDTREAD) {
    double local = 0.0;
    for (unsigned c = threadIdx.x; c < C; c += kConsumers) {
      const float p = powf(A.gstd[c], 0.6666666666666666f);
      A.gprior[c] = p;
      local += static_cast<double>(p);
    }
    const float psum = static_cast<float>(block_reduce(local, OpAdd(), sm.d));
    const float budget = static_cast<float>(static_cast<double>(C) * exp2(static_cast<double>(A.mt_target)));
    for (unsigned c = threadIdx.x; c < C; c += kConsumers) A.gbits[c] = rintf(__fdiv_rn(__fmul_rn(budget, A.gprior[c]), psum));
  } else {
    solve_bit_alloc(A, sm);
  }
  consumer_sync();
  // `publish`: the result is needed before this CTA reaches another grid barrier (no S2 phase to hide behind); otherwise
  // CTA 0's arrival at barrier 2 (release) publishes A.gbits along with everything else
  if (publish && threadIdx.x == 0) st_release_u32(&A.sync->aux_ready, tag);
}

// leaf parameters of channel c from the reduced accumulators (what the leader section of the NCHW kernel computes, here for
// one channel at a time): min / max / b over the replicas, std when a range mode or the export needs it, the channel's bit
// width (or mid-tread bin count) published by CTA 0, then int_quantizer.py:284-300 + :557-572 (or :185-214).
template <int LEAF, bool DEV>
__device__ __noinline__ LeafParam cl_channel_param(const FusedArgs& A, const ClView& acc, unsigned rep, unsigned C, unsigned c,
                                                   float mu, double n, bool alloc, bool do_export) {
  auto umax = [](unsigned a, unsigned b) { return a > b ? a : b; };
  const unsigned lo = cl_rep_reduce(acc.amin_inv, rep, C, c, 0u, umax);
  const unsigned hi = cl_rep_reduce(acc.amax, rep, C, c, 0u, umax);
  const double sa = DEV ? cl_rep_reduce(acc.aabs, rep, C, c, 0.0, OpAdd()) : 0.0;
  const float cb = A.bias ? __ldg(A.bias + c) : 0.f;  // S1 ran on the raw values: min / max shift by the bias exactly
  const float mn = __fadd_rn(dec_ordered(~lo), cb), mx = __fadd_rn(dec_ordered(hi), cb);
  const float b = DEV ? static_cast<float>(sa / n) : 0.f;
  const bool need_sd = A.range_mode == FQB200_RANGE_GAUS || A.range_mode == FQB200_RANGE_KSTD || do_export;
  const float sd = need_sd ? cl_std(acc, rep, C, c, n) : 0.f;
  const float aux = alloc ? ld_ws(A.gbits + c) : static_cast<float>(A.num_bits);
  LeafParam q;
  if constexpr (LEAF == FQB200_LEAF_MIDTREAD) {
    float rng;
    q = mid_tread_param(A, aux, mn, mx, mu, b, rng);
    if (do_export) export_stats(A, c, mn, mx, mu, b, sd, rng, 0.f, aux, q);
  } else {
    float delta, offset;
    solve_range(A, mn, mx, mu, b, sd, aux, delta, offset);
    q = make_leaf_param(LEAF, delta, offset, aux);
    if (do_export) export_stats(A, c, mn, mx, mu, b, sd, delta, offset, aux, q);
  }
  return q;
}

// ---- the streaming phases as separate (non-inlined) functions: each gets the whole register budget for its hot loop ----
struct ClCtx {
  const FlatGeo* g;
  BulkRing* ring;
  unsigned char* stages;
  unsigned char* cbuf;
  RingPos pos;
  ClView acc;
  unsigned rep_base, c0;
  bool active;
};

__device__ __noinline__ void cl_phase_s1(const FusedArgs& A, ClCtx& cx, float (&kshift)[4]) {
  const FlatGeo& g = *cx.g;
  ClStats1 s1;
  s1.init(A, cx.c0, cx.active);
#pragma unroll
  for (int i = 0; i < 4; ++i) kshift[i] = s1.k[i];
  RingPos pos = cx.pos;
  consume_phase(g, *cx.ring, cx.stages, pos, s1);
  cx.pos = pos;
  s1.flush();
  if (blockIdx.x == 0) stamp(A, 13);
  unsigned umn[4], umx[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    umn[i] = ~enc_ordered(s1.mn[i]);
    umx[i] = enc_ordered(s1.mx[i]);
  }
  const ClView& acc = cx.acc;
  const unsigned rb = cx.rep_base;
  cl_combine_s1(cx.cbuf, g.cv, g.stride, umn, umx, s1.s, s1.q, acc.amin_inv + rb, acc.amax + rb, acc.asum + rb, acc.asq + rb);
}

__device__ __noinline__ void cl_phase_s2(const FusedArgs& A, ClCtx& cx, const float (&mean)[4]) {
  const FlatGeo& g = *cx.g;
  ClStats2 s2;
  s2.init(A, cx.c0, cx.active, mean);
  RingPos pos = cx.pos;
  consume_phase(g, *cx.ring, cx.stages, pos, s2);
  cx.pos = pos;
  s2.flush();
  if (blockIdx.x == 0) stamp(A, 14);
  const ClView& acc = cx.acc;
  const unsigned rb = cx.rep_base;
  cl_combine_add_f64(cx.cbuf, g.cv, g.stride, s2.sa, acc.aabs + rb, s2.sa, nullptr, s2.sa, nullptr);
}

template <int LEAF, bool HIST>
__device__ __noinline__ void cl_phase_apply(const FusedArgs& A, ClCtx& cx, const LeafParam (&lp)[4], unsigned* hist) {
  const FlatGeo& g = *cx.g;
  const unsigned t = threadIdx.x;
  if (HIST) {
    for (unsigned i = t; i < kHistWords; i += kConsumers) hist[i] = 0u;
    consumer_sync();
  }
  ClApply<LEAF, HIST> ap{A, hist};
  ap.init(cx.c0, cx.active, lp);
  RingPos pos = cx.pos;
  if (A.pool.tiles) {
    if (A.pool.kind == 3u)
      consume_pool3_phase(g, A.pool, *cx.ring, cx.stages, pos, ap);
    else
      consume_pool_phase(g, A.pool, *cx.ring, cx.stages, pos, ap);
  } else if (A.residual) {
    const FlatGeo h = half_geo(g);
    consume_pair_phase(h, *cx.ring, cx.stages, pos, ap);
  } else {
    consume_phase(g, *cx.ring, cx.stages, pos, ap);
  }
  cx.pos = pos;
  if (HIST) {
    consumer_sync();
    const unsigned bins = static_cast<unsigned>(A.hist_bins);
    const unsigned copies = max(1u, min(static_cast<unsigned>(kWarps), kHistWords / bins));
    for (unsigned b = t; b < bins; b += kConsumers) {
      unsigned long long cnt = 0;
      for (unsigned w = 0; w < copies; ++w) cnt += hist[w * bins + b];
      if (cnt) atomicAdd(A.hist + b, cnt);
    }
    if (LEAF == FQB200_LEAF_MIDTREAD && A.hist_clamped && cx.active) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (ap.nlo[i]) atomicAdd(A.hist_clamped + 2u * (cx.c0 + i), static_cast<unsigned long long>(ap.nlo[i]));
        if (ap.nhi[i]) atomicAdd(A.hist_clamped + 2u * (cx.c0 + i) + 1u, static_cast<unsigned long long>(ap.nhi[i]));
      }
    }
  }
}

// ---- the kernel -----------------------------------------------------------------------------------------------------------
// LEAF: torch or mid-tread.  DEV: phase S2 (the Laplace b) is needed.  HIST: histogram of the integer grid (`-me`).
// Dynamic shared memory: [kStages stages][16 KB combine staging / parameter table][4 KB mean table]; HIST: the last stage
// holds the histograms and the ring runs with kStages - 1.
constexpr unsigned kClStagingBytes = 4u * kConsumers * 8u;          // 16 KB
constexpr unsigned kClTableChannels = 1024;                          // channel tables live in shared memory up to here
constexpr unsigned kClCombineBytes = kClStagingBytes + kClTableChannels * 4u;

template <int LEAF, bool DEV, bool HIST>
__global__ void __launch_bounds__(kBulkThreads, kBulkCtasPerSm) fq_cl_kernel(const __grid_constant__ FusedArgs A) {
  extern __shared__ __align__(128) unsigned char fq_dyn[];
  unsigned char* stages = fq_dyn;
  unsigned char* cbuf = fq_dyn + kStages * kStageBytes;
  float* tab_mean = reinterpret_cast<float*>(cbuf + kClStagingBytes);
  unsigned* hist = reinterpret_cast<unsigned*>(stages + (kStages - 1) * kStageBytes);  // HIST: the ring runs one stage short
  __shared__ BulkRing ring;
  __shared__ LeaderSmem lsm;
  __shared__ alignas(8) unsigned long long solver_done;  // mbarrier: CTA 0's consumers are back from the global solve
  const FlatGeo& g = A.flat;
  const unsigned C = g.channels, cv = g.cv;
  const unsigned launch = ld_ws(&A.sync->launch_count);
  const unsigned bank = launch & 1u;
  const unsigned tag = launch + 1u;
  const bool alloc = (LEAF == FQB200_LEAF_MIDTREAD) || (A.bit_alloc && A.num_bits <= 4);
  const bool aux_needs_b = alloc && LEAF != FQB200_LEAF_MIDTREAD && A.prior == FQB200_PRIOR_B;
  // CTA 0 computes the bit widths while the others stream S2: it takes no static S2 tickets and starts pulling dynamic
  // ones only when its consumers are back (it would sit on them otherwise)
  const bool solver_in_s2 = alloc && !aux_needs_b && DEV && gridDim.x > 1u;
  // the producer starts a phase's loads when the consumers are through the previous phase's combine: its reductions
  // (a few thousand fire-and-forget atomics) queue behind 192 KB of bulk loads otherwise
  __shared__ alignas(8) unsigned long long phase_go[2];
  if (threadIdx.x == 0) {
    mbar_init(smem_u32(&solver_done), 1u);
    mbar_init(smem_u32(&phase_go[0]), 1u);
    mbar_init(smem_u32(&phase_go[1]), 1u);
  }
  const unsigned nstages = HIST ? kStages - 1u : kStages;  // the histogram lives in the last stage's memory
  ring_init(ring, nstages);

  // ================================ producer warp ================================
  if (threadIdx.x >= kConsumers) {
    if (threadIdx.x == kConsumers) {
      RingPos pos;
      pos.init(nstages);
      const float4* src = reinterpret_cast<const float4*>(A.in);
      const TicketPlan all = {2u, blockIdx.x, gridDim.x, 2u * gridDim.x};
      // the phase in which CTA 0's consumers are busy with the global solve: no static tickets for it, and its producer
      // pulls dynamic ones only when they are back
      const TicketPlan no0 = {blockIdx.x == 0 ? 0u : 2u, blockIdx.x - 1u, gridDim.x - 1u, 2u * (gridDim.x - 1u)};
      produce_phase<false>(g, src, &A.sync->unit_counter[0], all, ring, stages, pos);
      if (DEV) {
        mbar_wait(smem_u32(&phase_go[0]), 0u);
        if (solver_in_s2 && blockIdx.x == 0) mbar_wait(smem_u32(&solver_done), 0u);
        produce_phase<true>(g, src, &A.sync->unit_counter[1], solver_in_s2 ? no0 : all, ring, stages, pos);
      }
      if (!A.stats_only) {
        mbar_wait(smem_u32(&phase_go[1]), 0u);
        if (A.pool.tiles && A.pool.kind == 3u)
          produce_pool3_phase(g, A.pool, src, &A.sync->unit_counter[2], all, ring, stages, pos);
        else if (A.pool.tiles)
          produce_pool_phase(g, A.pool, src, &A.sync->unit_counter[2], all, ring, stages, pos);
        else if (A.residual)
          produce_phase<!DEV, true>(half_geo(g), src, &A.sync->unit_counter[2], all, ring, stages, pos,
                                    reinterpret_cast<const float4*>(A.residual));
        else
          produce_phase<!DEV>(g, src, &A.sync->unit_counter[2], all, ring, stages, pos);
      }
    }
    return;
  }

  // ================================ consumers ================================
  const unsigned t = threadIdx.x;
  const bool active = t < g.stride;
  const bool direct = cv == g.stride;  // every active thread is the only one on its column: no shared-memory tables
  const unsigned col = active ? t % cv : 0u;
  const unsigned c0 = 4u * col;
  const double n = A.n_per_group;
  const ClView acc = cl_view(A, bank);
  const unsigned rep = A.nhwc_rep;
  const unsigned rep_base = (blockIdx.x % rep) * C;
  unsigned epoch = 0;
  if (blockIdx.x == 0) stamp(A, 0);

  // the bank the previous launch used: zero it for the next one (off the critical path)
  if (blockIdx.x == gridDim.x - 1u) {
    const ClView other = cl_view(A, bank ^ 1u);
    uint4* zu = reinterpret_cast<uint4*>(other.amin_inv);
    uint4* zd = reinterpret_cast<uint4*>(other.asum);
    const uint4 z = make_uint4(0u, 0u, 0u, 0u);
    for (unsigned i = t; i < kAccU / 4u; i += kConsumers) zu[i] = z;
    for (unsigned i = t; i < kAccD / 2u; i += kConsumers) zd[i] = z;
  }

  // ---- S1
  ClCtx cx;
  cx.g = &g;
  cx.ring = &ring;
  cx.stages = stages;
  cx.cbuf = cbuf;
  cx.pos.init(nstages);
  cx.acc = acc;
  cx.rep_base = rep_base;
  cx.c0 = c0;
  cx.active = active;
  float kshift[4];
  cl_phase_s1(A, cx, kshift);
  if (t == 0) mbar_arrive(smem_u32(&phase_go[DEV ? 0 : 1]));
  if (blockIdx.x == 0) stamp(A, 1);
  grid_barrier_cl(A.sync, epoch);
  if (blockIdx.x == 0) stamp(A, 4);

  // ---- the mean of every channel: each accumulator value is read once per CTA
  float mean[4];
  if (direct) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
      mean[i] = static_cast<float>(cl_mean(acc, rep, C, c0 + i, kshift[i], (A.bias && active) ? __ldg(A.bias + c0 + i) : 0.f, n));
  } else {
    for (unsigned c = t; c < C; c += kConsumers)
      tab_mean[c] = static_cast<float>(cl_mean(acc, rep, C, c, ld_tensor(A.in + c), A.bias ? __ldg(A.bias + c) : 0.f, n));
    consumer_sync();
#pragma unroll
    for (int i = 0; i < 4; ++i) mean[i] = tab_mean[c0 + i];
  }

  // ---- the global solve, where it can overlap with S2
  if (alloc && !aux_needs_b && blockIdx.x == 0) {
    cl_solve_aux(A, acc, lsm, tag, false, !solver_in_s2);
    stamp(A, 12);
    if (t == 0) mbar_arrive(smem_u32(&solver_done));
  }

  // ---- S2
  if constexpr (DEV) {
    cl_phase_s2(A, cx, mean);
    if (t == 0) mbar_arrive(smem_u32(&phase_go[1]));
    if (blockIdx.x == 0) stamp(A, 5);
    grid_barrier_cl(A.sync, epoch);
    if (blockIdx.x == 0) stamp(A, 8);
    if (aux_needs_b && blockIdx.x == 0) cl_solve_aux(A, acc, lsm, tag, true, true);
  }
  if (alloc && !solver_in_s2) {  // (overlapped with S2, CTA 0's arrival at barrier 2 has published the bit widths already)
    if (t == 0)
      while (ld_acquire_u32(&A.sync->aux_ready) != tag) __nanosleep(40);
    consumer_sync();
  }

  // ---- leaf parameters of every channel, again each accumulator value read once per CTA
  LeafParam lp[4];
  const bool do_export = A.out_stats != nullptr && blockIdx.x == 0;
  if (direct) {
#pragma unroll
    for (int i = 0; i < 4; ++i) lp[i] = cl_channel_param<LEAF, DEV>(A, acc, rep, C, c0 + i, mean[i], n, alloc, do_export && active);
  } else {
    LeafParam* tab_lp = reinterpret_cast<LeafParam*>(cbuf);
    consumer_sync();  // the combine staging is free
    for (unsigned c = t; c < C; c += kConsumers) tab_lp[c] = cl_channel_param<LEAF, DEV>(A, acc, rep, C, c, tab_mean[c], n, alloc, do_export);
    consumer_sync();
#pragma unroll
    for (int i = 0; i < 4; ++i) lp[i] = tab_lp[c0 + i];
  }
  if (blockIdx.x == 0) stamp(A, 7);

  // ---- A
  if (!A.stats_only) {
    cl_phase_apply<LEAF, HIST>(A, cx, lp, hist);
    if (blockIdx.x == 0) stamp(A, 9);
  }
  grid_exit_cl(A.sync);
}

// ---- mode A on channels-last memory: parameters given, no statistics, no barrier (ordinary launch) ---------------------------
// Static round-robin units; leaf parameters derived per thread from the caller's delta / offset / bits of its 4 channels
// (per_group) or of the whole tensor.
template <bool GRID>
struct ClGiven {
  const FusedArgs& A;
  LeafParam q[4];
  float r[4], bias[4];
  bool fast;
  template <bool FAST>
  __device__ __forceinline__ void one(const float4& v, unsigned off) {
    const float x[4] = {v.x, v.y, v.z, v.w};
    float y[4], gq[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      Divisor dv;
      dv.s = q[i].a;
      dv.r = r[i];
      dv.fast = FAST;
      y[i] = leaf_apply<FQB200_LEAF_TORCH, FAST>(__fadd_rn(x[i], bias[i]), q[i], dv, 0.f, gq[i]);
    }
    st_tensor(reinterpret_cast<float4*>(A.out) + off, make_float4(y[0], y[1], y[2], y[3]));
    if (GRID) st_tensor(reinterpret_cast<float4*>(A.grid_out) + off, make_float4(gq[0], gq[1], gq[2], gq[3]));
  }
  __device__ __forceinline__ void consume(const float4& v, unsigned off) {
    if (fast)
      one<true>(v, off);
    else
      one<false>(v, off);
  }
  __device__ __forceinline__ void stage_end(const StageMeta&) {}
};

template <bool GRID>
__global__ void __launch_bounds__(kBulkThreads, kBulkCtasPerSm) fq_cl_given_kernel(const __grid_constant__ FusedArgs A) {
  extern __shared__ __align__(128) unsigned char fq_dyn[];
  __shared__ BulkRing ring;
  const FlatGeo& g = A.flat;
  ring_init(ring);
  if (threadIdx.x >= kConsumers) {
    if (threadIdx.x == kConsumers) {
      RingPos pos;
      pos.init();
      // static assignment: ticket k of CTA b = b + k * grid (no workspace, no counter)
      const TicketPlan tp = {0xffffffffu, blockIdx.x, gridDim.x, 0u};
      produce_phase<false>(g, reinterpret_cast<const float4*>(A.in), nullptr, tp, ring, fq_dyn, pos);
    }
    return;
  }
  const unsigned t = threadIdx.x;
  const bool active = t < g.stride;
  const unsigned c0 = active ? 4u * (t % g.cv) : 0u;
  ClGiven<GRID> ap{A};
  ap.fast = true;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const unsigned c = c0 + i;
    const unsigned pi = A.given_per_group ? c : 0u;
    const float bits = A.g_bits ? __ldg(A.g_bits + c) : static_cast<float>(A.num_bits);
    ap.q[i] = make_leaf_param(FQB200_LEAF_TORCH, __ldg(A.g_delta + pi), __ldg(A.g_offset + pi), bits);
    const Divisor dv = make_divisor(ap.q[i].a);
    ap.r[i] = dv.r;
    ap.fast = ap.fast && dv.fast;
    ap.bias[i] = (A.bias && active) ? __ldg(A.bias + c) : 0.f;
  }
  RingPos pos;
  pos.init();
  consume_phase(g, ring, fq_dyn, pos, ap);
}

// ---- mode A with everything the apply phase can carry (FQB200_RANGE_GIVEN through fqb200_fused): bias, the block epilogue
// (residual, raw or quantized on the fly), max pooling.  Same apply code as fq_cl_kernel (ClApply), no statistics, no barrier,
// ordinary launch, static round-robin units.
__global__ void __launch_bounds__(kBulkThreads, kBulkCtasPerSm) fq_cl_given_fused_kernel(const __grid_constant__ FusedArgs A) {
  extern __shared__ __align__(128) unsigned char fq_dyn[];
  __shared__ BulkRing ring;
  const FlatGeo& g = A.flat;
  ring_init(ring);
  if (threadIdx.x >= kConsumers) {
    if (threadIdx.x == kConsumers) {
      RingPos pos;
      pos.init();
      const float4* src = reinterpret_cast<const float4*>(A.in);
      const TicketPlan tp = {0xffffffffu, blockIdx.x, gridDim.x, 0u};
      if (A.pool.tiles && A.pool.kind == 3u)
        produce_pool3_phase(g, A.pool, src, nullptr, tp, ring, fq_dyn, pos);
      else if (A.pool.tiles)
        produce_pool_phase(g, A.pool, src, nullptr, tp, ring, fq_dyn, pos);
      else if (A.residual)
        produce_phase<false, true>(half_geo(g), src, nullptr, tp, ring, fq_dyn, pos, reinterpret_cast<const float4*>(A.residual));
      else
        produce_phase<false>(g, src, nullptr, tp, ring, fq_dyn, pos);
    }
    return;
  }
  const unsigned t = threadIdx.x;
  const bool active = t < g.stride;
  const unsigned c0 = active ? 4u * (t % g.cv) : 0u;
  LeafParam lp[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const unsigned c = c0 + i;
    const float bits = A.g_bits ? __ldg(A.g_bits + c) : static_cast<float>(A.num_bits);
    lp[i] = make_leaf_param(FQB200_LEAF_TORCH, __ldg(A.g_delta + c), __ldg(A.g_offset + c), bits);
  }
  ClApply<FQB200_LEAF_TORCH, false> ap{A, nullptr};
  ap.init(c0, active, lp);
  RingPos pos;
  pos.init();
  if (A.pool.tiles && A.pool.kind == 3u)
    consume_pool3_phase(g, A.pool, ring, fq_dyn, pos, ap);
  else if (A.pool.tiles)
    consume_pool_phase(g, A.pool, ring, fq_dyn, pos, ap);
  else if (A.residual)
    consume_pair_phase(half_geo(g), ring, fq_dyn, pos, ap);
  else
    consume_phase(g, ring, fq_dyn, pos, ap);
}

// ---- a1, the drop-in of the reference's compiled kernel (kernels/gemmlowp.cu:8-45), on the bulk-copy ring -------------------
// One parameter set, compiled-leaf arithmetic (roundf), optional noise tensor: it rides through the ring next to x (pair
// stages).  Ordinary launch, static round-robin units.
struct LeafBulkArgs {
  FlatGeo flat;
  const float* in;
  float* out;
  const float* noise;
  LeafParam q;
};

template <bool NOISE>
struct LeafBulk {
  const LeafBulkArgs& A;
  Divisor dv;
  template <bool FAST>
  __device__ __forceinline__ void one(const float4& v, const float4& nz, unsigned off) {
    float gq;
    float4 y;
    y.x = leaf_apply<FQB200_LEAF_COMPILED, FAST, NOISE>(v.x, A.q, dv, NOISE ? nz.x : 0.f, gq);
    y.y = leaf_apply<FQB200_LEAF_COMPILED, FAST, NOISE>(v.y, A.q, dv, NOISE ? nz.y : 0.f, gq);
    y.z = leaf_apply<FQB200_LEAF_COMPILED, FAST, NOISE>(v.z, A.q, dv, NOISE ? nz.z : 0.f, gq);
    y.w = leaf_apply<FQB200_LEAF_COMPILED, FAST, NOISE>(v.w, A.q, dv, NOISE ? nz.w : 0.f, gq);
    st_tensor(reinterpret_cast<float4*>(A.out) + off, y);
  }
  __device__ __forceinline__ void consume(const float4& v, unsigned off) {
    if (dv.fast)
      one<true>(v, v, off);
    else
      one<false>(v, v, off);
  }
  __device__ __forceinline__ void consume2(const float4& v, const float4& nz, unsigned off) {
    if (dv.fast)
      one<true>(v, nz, off);
    else
      one<false>(v, nz, off);
  }
  __device__ __forceinline__ void stage_end(const StageMeta&) {}
};

template <bool NOISE>
__global__ void __launch_bounds__(kBulkThreads, kBulkCtasPerSm) fq_leaf_bulk_kernel(const __grid_constant__ LeafBulkArgs A) {
  extern __shared__ __align__(128) unsigned char fq_dyn[];
  __shared__ BulkRing ring;
  const FlatGeo g = NOISE ? half_geo(A.flat) : A.flat;
  ring_init(ring);
  if (threadIdx.x >= kConsumers) {
    if (threadIdx.x == kConsumers) {
      RingPos pos;
      pos.init();
      const TicketPlan tp = {0xffffffffu, blockIdx.x, gridDim.x, 0u};
      produce_phase<false, NOISE>(g, reinterpret_cast<const float4*>(A.in), nullptr, tp, ring, fq_dyn, pos,
                                  reinterpret_cast<const float4*>(A.noise));
    }
    return;
  }
  LeafBulk<NOISE> ap{A, make_divisor(A.q.a)};
  RingPos pos;
  pos.init();
  if (NOISE)
    consume_pair_phase(g, ring, fq_dyn, pos, ap);
  else
    consume_phase(g, ring, fq_dyn, pos, ap);
}

// ---- `-bca`: given-parameter quantization with activation bias correction (inference_quantization_manager.py:180-196) -----
// Per channel: q_bias = (sum r - sum y) / (#(r > 0) + 1e-8) with y the quantized activation and r the activation itself
// (rectified first when a ReLU follows), added back where y > 0.  Two passes over x (both recompute y), one write:
// 12 B/element where the reference makes three transposed copies, three reductions and three elementwise passes.
struct ClBca1 {
  const FusedArgs& A;
  LeafParam q[4];
  float r[4], bias[4], fr[4], fy[4];
  double sr[4], sy[4];
  unsigned cnt[4], n;
  bool fast;
  __device__ __forceinline__ void flush() {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      sr[i] += static_cast<double>(fr[i]);
      sy[i] += static_cast<double>(fy[i]);
      fr[i] = 0.f;
      fy[i] = 0.f;
    }
    n = 0;
  }
  template <bool FAST>
  __device__ __forceinline__ void one(const float4& v) {
    const float x[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      Divisor dv;
      dv.s = q[i].a;
      dv.r = r[i];
      dv.fast = FAST;
      float gq;
      const float xb = __fadd_rn(x[i], bias[i]);
      const float y = leaf_apply<FQB200_LEAF_TORCH, FAST>(xb, q[i], dv, 0.f, gq);
      const float rr = (A.relu_passthrough && xb < 0.f) ? 0.f : xb;
      fr[i] = __fadd_rn(fr[i], rr);
      fy[i] = __fadd_rn(fy[i], y);
      cnt[i] += rr > 0.f ? 1u : 0u;
    }
  }
  __device__ __forceinline__ void consume(const float4& v, unsigned) {
    if (fast)
      one<true>(v);
    else
      one<false>(v);
  }
  __device__ __forceinline__ void stage_end(const StageMeta&) {
    if (++n == kClChunkStages) flush();
  }
};

struct ClBca2 {
  const FusedArgs& A;
  LeafParam q[4];
  float r[4], bias[4], qb[4];
  bool fast;
  template <bool FAST>
  __device__ __forceinline__ void one(const float4& v, unsigned off) {
    const float x[4] = {v.x, v.y, v.z, v.w};
    float y[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      Divisor dv;
      dv.s = q[i].a;
      dv.r = r[i];
      dv.fast = FAST;
      float gq;
      y[i] = leaf_apply<FQB200_LEAF_TORCH, FAST>(__fadd_rn(x[i], bias[i]), q[i], dv, 0.f, gq);
      if (y[i] > 0.f) y[i] = __fadd_rn(y[i], qb[i]);
    }
    st_tensor(reinterpret_cast<float4*>(A.out) + off, make_float4(y[0], y[1], y[2], y[3]));
  }
  __device__ __forceinline__ void consume(const float4& v, unsigned off) {
    if (fast)
      one<true>(v, off);
    else
      one<false>(v, off);
  }
  __device__ __forceinline__ void stage_end(const StageMeta&) {}
};

__global__ void __launch_bounds__(kBulkThreads, kBulkCtasPerSm) fq_cl_bca_kernel(const __grid_constant__ FusedArgs A) {
  extern __shared__ __align__(128) unsigned char fq_dyn[];
  unsigned char* stages = fq_dyn;
  unsigned char* cbuf = fq_dyn + kStages * kStageBytes;
  __shared__ BulkRing ring;
  const FlatGeo& g = A.flat;
  const unsigned C = g.channels, cv = g.cv;
  const unsigned bank = ld_ws(&A.sync->launch_count) & 1u;
  ring_init(ring);
  if (threadIdx.x >= kConsumers) {
    if (threadIdx.x == kConsumers) {
      RingPos pos;
      pos.init();
      const float4* src = reinterpret_cast<const float4*>(A.in);
      const TicketPlan all = {2u, blockIdx.x, gridDim.x, 2u * gridDim.x};
      produce_phase<false>(g, src, &A.sync->unit_counter[0], all, ring, stages, pos);
      produce_phase<true>(g, src, &A.sync->unit_counter[1], all, ring, stages, pos);
    }
    return;
  }
  const unsigned t = threadIdx.x;
  const bool active = t < g.stride;
  const unsigned c0 = active ? 4u * (t % cv) : 0u;
  const ClView acc = cl_view(A, bank);
  const unsigned rep = A.nhwc_rep;
  const unsigned rep_base = (blockIdx.x % rep) * C;
  unsigned epoch = 0;
  RingPos pos;
  pos.init();
  if (blockIdx.x == gridDim.x - 1u) {  // zero the bank of the previous launch
    const ClView other = cl_view(A, bank ^ 1u);
    uint4* zu = reinterpret_cast<uint4*>(other.amin_inv);
    uint4* zd = reinterpret_cast<uint4*>(other.asum);
    const uint4 z = make_uint4(0u, 0u, 0u, 0u);
    for (unsigned i = t; i < kAccU / 4u; i += kConsumers) zu[i] = z;
    for (unsigned i = t; i < kAccD / 2u; i += kConsumers) zd[i] = z;
  }
  ClBca1 p1{A};
  p1.fast = true;
  p1.n = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const unsigned c = c0 + i;
    const unsigned pi = A.given_per_group ? c : 0u;
    const float bits = A.g_bits ? __ldg(A.g_bits + c) : static_cast<float>(A.num_bits);
    p1.q[i] = make_leaf_param(FQB200_LEAF_TORCH, __ldg(A.g_delta + pi), __ldg(A.g_offset + pi), bits);
    const Divisor dv = make_divisor(p1.q[i].a);
    p1.r[i] = dv.r;
    p1.fast = p1.fast && dv.fast;
    p1.bias[i] = (A.bias && active) ? __ldg(A.bias + c) : 0.f;
    p1.fr[i] = p1.fy[i] = 0.f;
    p1.sr[i] = p1.sy[i] = 0.0;
    p1.cnt[i] = 0u;
  }
  consume_phase(g, ring, stages, pos, p1);
  p1.flush();
  double dc[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) dc[i] = static_cast<double>(p1.cnt[i]);
  cl_combine_add_f64(cbuf, cv, g.stride, p1.sr, acc.asum + rep_base, p1.sy, acc.asq + rep_base, dc, acc.aabs + rep_base);
  grid_barrier_cl(A.sync, epoch);
  // q_bias of every channel, each accumulator value read once per CTA (table in shared memory; direct when cv == stride)
  auto qbias_of = [&](unsigned c) {
    double a = 0.0, b = 0.0, n = 0.0;
    for (unsigned r = 0; r < rep; ++r) {
      a += ld_ws(acc.asum + r * C + c);
      b += ld_ws(acc.asq + r * C + c);
      n += ld_ws(acc.aabs + r * C + c);
    }
    // fp32 like the reference: (sum r - sum y) / (count + 1e-8)
    return __fdiv_rn(__fsub_rn(static_cast<float>(a), static_cast<float>(b)), __fadd_rn(static_cast<float>(n), 1e-8f));
  };
  ClBca2 p2{A};
  p2.fast = p1.fast;
  if (cv == g.stride) {
#pragma unroll
    for (int i = 0; i < 4; ++i) p2.qb[i] = qbias_of(c0 + i);
  } else {
    float* tab = reinterpret_cast<float*>(cbuf);
    consumer_sync();
    for (unsigned c = t; c < C; c += kConsumers) tab[c] = qbias_of(c);
    consumer_sync();
#pragma unroll
    for (int i = 0; i < 4; ++i) p2.qb[i] = tab[c0 + i];
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    p2.q[i] = p1.q[i];
    p2.r[i] = p1.r[i];
    p2.bias[i] = p1.bias[i];
    if (A.out_stats && blockIdx.x == 0 && t < cv) A.out_stats[c0 + i] = p2.qb[i];  // diagnostics: the correction applied
  }
  consume_phase(g, ring, stages, pos, p2);
  grid_exit_cl(A.sync);
}

// ---- per-sample / per-tensor min-max ranges with the compiled-leaf arithmetic on the bulk engine -------------------------------
// gemmlowpMinMaxQuantize (int_quantizer.py:361-379 + :605-614): every tensor of BASELINE configs[1] (W8A8) and the int8
// pooling / classifier tensors of every other config.  Rows = samples (contiguous in NCHW and in channels-last memory);
// S1: min / max of every row (units never straddle rows; one CTA-wide combine + two atomics per unit), grid barrier, then
// EVERY CTA derives the one parameter set itself from the <= 4096 row results (scope GROUP_MEAN: batch average of the
// per-sample min / max, :372; scope TENSOR / one row: global min / max), A: apply.  The optional per-channel bias (folded
// BN) is a per-thread constant on channels-last memory, where a vector's channels are (index mod C/4); with it the apply
// phase can also write a channel slice of a wider channels-last tensor (FusedArgs::out_pad_v, fqb200_fused_into).
struct RowsStats {
  const FusedArgs& A;
  float* scratch;  // [2][kWarps] floats in shared memory
  const ClView& acc;
  float bias[4];
  float mn, mx;
  __device__ __forceinline__ void consume(const float4& v, unsigned) {
    const float x0 = __fadd_rn(v.x, bias[0]), x1 = __fadd_rn(v.y, bias[1]), x2 = __fadd_rn(v.z, bias[2]), x3 = __fadd_rn(v.w, bias[3]);
    mn = fminf(mn, fminf(fminf(x0, x1), fminf(x2, x3)));
    mx = fmaxf(mx, fmaxf(fmaxf(x0, x1), fmaxf(x2, x3)));
  }
  __device__ __forceinline__ void stage_end(const StageMeta& m) {
    if (!(m.tag & 0x80000000u)) return;  // CTA-uniform: the unit goes on
    const float a = warp_reduce(mn, OpMin()), b = warp_reduce(mx, OpMax());
    const unsigned w = threadIdx.x >> 5, l = threadIdx.x & 31u;
    consumer_sync();
    if (l == 0) {
      scratch[w] = a;
      scratch[kWarps + w] = b;
    }
    consumer_sync();
    if (w == 0) {
      float c = (l < kWarps) ? scratch[l] : INFINITY, d = (l < kWarps) ? scratch[kWarps + l] : -INFINITY;
#pragma unroll
      for (int o = kWarps / 2; o > 0; o >>= 1) {
        c = fminf(c, __shfl_xor_sync(0xffffffffu, c, o));
        d = fmaxf(d, __shfl_xor_sync(0xffffffffu, d, o));
      }
      if (l == 0) {
        const unsigned row = m.tag & 0x7fffffffu;
        red_max_u32(acc.amin_inv + row, ~enc_ordered(c));
        red_max_u32(acc.amax + row, enc_ordered(d));
      }
    }
    mn = INFINITY;
    mx = -INFINITY;
  }
};

struct RowsApply {
  const FusedArgs& A;
  LeafParam q;
  Divisor dv;
  float bias[4];
  // the residual operand, when it is quantized on the fly (fqb200_desc.residual_stats: one row, compiled leaf)
  LeafParam rq;
  Divisor rdv;
  float rbias[4];
  bool rquant;
  __device__ __forceinline__ void init_residual(unsigned c0, bool active) {
    rquant = A.residual != nullptr && A.residual_stats != nullptr;
    rq.a = 1.f;
    rq.b = 0.f;
    rq.c = 0.f;
    rq.flags = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) rbias[i] = 0.f;
    if (rquant) {
      rq.a = __ldg(A.residual_stats + 8);
      rq.b = __ldg(A.residual_stats + 9);
      rq.c = __ldg(A.residual_stats + 10);
      rq.flags = static_cast<int>(__ldg(A.residual_stats + 11));
      if (A.residual_bias && active) {
#pragma unroll
        for (int i = 0; i < 4; ++i) rbias[i] = __ldg(A.residual_bias + c0 + i);
      }
    }
    rdv = make_divisor(rq.a);
    if (rquant && !rdv.fast) dv.fast = false;  // one flag selects the division for both operands
    rdv.fast = dv.fast;
  }
  template <bool FAST, bool PAIR>
  __device__ __forceinline__ void one(const float4& v, const float4& r0, unsigned off) {
    float gq;
    float4 y;
    float4 r = r0;
    if (PAIR && rquant) {
      r.x = leaf_apply<FQB200_LEAF_COMPILED, FAST>(__fadd_rn(r0.x, rbias[0]), rq, rdv, 0.f, gq);
      r.y = leaf_apply<FQB200_LEAF_COMPILED, FAST>(__fadd_rn(r0.y, rbias[1]), rq, rdv, 0.f, gq);
      r.z = leaf_apply<FQB200_LEAF_COMPILED, FAST>(__fadd_rn(r0.z, rbias[2]), rq, rdv, 0.f, gq);
      r.w = leaf_apply<FQB200_LEAF_COMPILED, FAST>(__fadd_rn(r0.w, rbias[3]), rq, rdv, 0.f, gq);
    }
    y.x = leaf_apply<FQB200_LEAF_COMPILED, FAST>(__fadd_rn(v.x, bias[0]), q, dv, 0.f, gq);
    y.y = leaf_apply<FQB200_LEAF_COMPILED, FAST>(__fadd_rn(v.y, bias[1]), q, dv, 0.f, gq);
    y.z = leaf_apply<FQB200_LEAF_COMPILED, FAST>(__fadd_rn(v.z, bias[2]), q, dv, 0.f, gq);
    y.w = leaf_apply<FQB200_LEAF_COMPILED, FAST>(__fadd_rn(v.w, bias[3]), q, dv, 0.f, gq);
    if (PAIR) {  // the residual add (+ ReLU) that closes a ResNet block, on the quantized values
      y.x = __fadd_rn(y.x, r.x);
      y.y = __fadd_rn(y.y, r.y);
      y.z = __fadd_rn(y.z, r.z);
      y.w = __fadd_rn(y.w, r.w);
      if (A.residual_relu) {
        y.x = y.x < 0.f ? 0.f : y.x;
        y.y = y.y < 0.f ? 0.f : y.y;
        y.z = y.z < 0.f ? 0.f : y.z;
        y.w = y.w < 0.f ? 0.f : y.w;
      }
    }
    // a channel slice of a wider channels-last tensor (out_pad_v, launches with a channel-fastest bias only): `off` counts
    // cv = C/4 vectors per pixel, the output out_pad_v more
    const unsigned o = A.out_pad_v ? off + (off / A.flat.cv) * A.out_pad_v : off;
    st_tensor(reinterpret_cast<float4*>(A.out) + o, y);
  }
  __device__ __forceinline__ void consume(const float4& v, unsigned off) {
    if (dv.fast)
      one<true, false>(v, v, off);
    else
      one<false, false>(v, v, off);
  }
  __device__ __forceinline__ void consume2(const float4& v, const float4& r, unsigned off) {
    if (dv.fast)
      one<true, true>(v, r, off);
    else
      one<false, true>(v, r, off);
  }
  __device__ __forceinline__ void stage_end(const StageMeta&) {}
  // max pooling in front of the (monotone) leaf, see ClApply
  float pm[4];
  __device__ __forceinline__ void pool_begin() {
#pragma unroll
    for (int i = 0; i < 4; ++i) pm[i] = -INFINITY;
  }
  __device__ __forceinline__ void pool_tap(const float4& v) {
    auto mx = [](float p, float q) { return (q > p || q != q) ? q : p; };
    pm[0] = mx(pm[0], v.x);
    pm[1] = mx(pm[1], v.y);
    pm[2] = mx(pm[2], v.z);
    pm[3] = mx(pm[3], v.w);
  }
  __device__ __forceinline__ void pool_end(unsigned off) {
    float gq;
    float4 y;
    if (dv.fast) {
      y.x = leaf_apply<FQB200_LEAF_COMPILED, true>(__fadd_rn(pm[0], bias[0]), q, dv, 0.f, gq);
      y.y = leaf_apply<FQB200_LEAF_COMPILED, true>(__fadd_rn(pm[1], bias[1]), q, dv, 0.f, gq);
      y.z = leaf_apply<FQB200_LEAF_COMPILED, true>(__fadd_rn(pm[2], bias[2]), q, dv, 0.f, gq);
      y.w = leaf_apply<FQB200_LEAF_COMPILED, true>(__fadd_rn(pm[3], bias[3]), q, dv, 0.f, gq);
    } else {
      y.x = leaf_apply<FQB200_LEAF_COMPILED, false>(__fadd_rn(pm[0], bias[0]), q, dv, 0.f, gq);
      y.y = leaf_apply<FQB200_LEAF_COMPILED, false>(__fadd_rn(pm[1], bias[1]), q, dv, 0.f, gq);
      y.z = leaf_apply<FQB200_LEAF_COMPILED, false>(__fadd_rn(pm[2], bias[2]), q, dv, 0.f, gq);
      y.w = leaf_apply<FQB200_LEAF_COMPILED, false>(__fadd_rn(pm[3], bias[3]), q, dv, 0.f, gq);
    }
    st_tensor(reinterpret_cast<float4*>(A.pool_out) + off, y);
  }
  __device__ __forceinline__ void pooled(const float4& a0, const float4& a1, const float4& b0, const float4& b1, unsigned off) {
    pool_begin();
    pool_tap(a0);
    pool_tap(a1);
    pool_tap(b0);
    pool_tap(b1);
    pool_end(off);
  }
};

__global__ void __launch_bounds__(kBulkThreads, kBulkCtasPerSm) fq_rows_kernel(const __grid_constant__ FusedArgs A) {
  extern __shared__ __align__(128) unsigned char fq_dyn[];
  __shared__ BulkRing ring;
  __shared__ LeaderSmem lsm;
  __shared__ float scratch[2 * kWarps];
  const FlatGeo& g = A.flat;
  const RowsGeo& rg = A.rows;
  const unsigned bank = ld_ws(&A.sync->launch_count) & 1u;
  ring_init(ring);
  if (threadIdx.x >= kConsumers) {
    if (threadIdx.x == kConsumers) {
      RingPos pos;
      pos.init();
      const float4* src = reinterpret_cast<const float4*>(A.in);
      const TicketPlan all = {2u, blockIdx.x, gridDim.x, 2u * gridDim.x};
      produce_rows_phase<false>(g, rg, src, &A.sync->unit_counter[0], all, ring, fq_dyn, pos);
      if (!A.stats_only) {
        if (A.pool.tiles && A.pool.kind == 3u) {
          produce_pool3_phase(g, A.pool, src, &A.sync->unit_counter[2], all, ring, fq_dyn, pos);
        } else if (A.pool.tiles) {
          produce_pool_phase(g, A.pool, src, &A.sync->unit_counter[2], all, ring, fq_dyn, pos);
        } else if (A.residual) {
          const FlatGeo h = half_geo(g);
          produce_rows_phase<true, true>(h, half_rows(h, rg), src, &A.sync->unit_counter[2], all, ring, fq_dyn, pos,
                                         reinterpret_cast<const float4*>(A.residual));
        } else {
          produce_rows_phase<true>(g, rg, src, &A.sync->unit_counter[2], all, ring, fq_dyn, pos);
        }
      }
    }
    return;
  }
  const unsigned t = threadIdx.x;
  const bool active = t < g.stride;
  const unsigned c0 = active ? 4u * (t % g.cv) : 0u;
  const ClView acc = cl_view(A, bank);
  unsigned epoch = 0;
  RingPos pos;
  pos.init();
  if (blockIdx.x == 0) stamp(A, 0);
  if (blockIdx.x == gridDim.x - 1u) {  // zero the bank of the previous launch
    const ClView other = cl_view(A, bank ^ 1u);
    uint4* zu = reinterpret_cast<uint4*>(other.amin_inv);
    uint4* zd = reinterpret_cast<uint4*>(other.asum);
    const uint4 z = make_uint4(0u, 0u, 0u, 0u);
    for (unsigned i = t; i < kAccU / 4u; i += kConsumers) zu[i] = z;
    for (unsigned i = t; i < kAccD / 2u; i += kConsumers) zd[i] = z;
  }
  float bias[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) bias[i] = (A.bias && active) ? __ldg(A.bias + c0 + i) : 0.f;
  {
    RowsStats s1{A, scratch, acc, {bias[0], bias[1], bias[2], bias[3]}, INFINITY, -INFINITY};
    consume_phase(g, ring, fq_dyn, pos, s1);
  }
  if (blockIdx.x == 0) stamp(A, 1);
  grid_barrier_cl(A.sync, epoch);
  if (blockIdx.x == 0) stamp(A, 4);
  // the one parameter set, computed by every CTA from the row results
  const unsigned R = rg.rows;
  float mn, mx;
  if (A.scope == FQB200_SCOPE_GROUP_MEAN) {
    double smin = 0.0, smax = 0.0;
    for (unsigned r = t; r < R; r += kConsumers) {
      smin += static_cast<double>(dec_ordered(~ld_ws(acc.amin_inv + r)));
      smax += static_cast<double>(dec_ordered(ld_ws(acc.amax + r)));
    }
    smin = block_reduce(smin, OpAdd(), lsm.d);
    smax = block_reduce(smax, OpAdd(), lsm.d);
    mn = static_cast<float>(smin / R);
    mx = static_cast<float>(smax / R);
  } else {
    float lmin = INFINITY, lmax = -INFINITY;
    for (unsigned r = t; r < R; r += kConsumers) {
      lmin = fminf(lmin, dec_ordered(~ld_ws(acc.amin_inv + r)));
      lmax = fmaxf(lmax, dec_ordered(ld_ws(acc.amax + r)));
    }
    mn = block_reduce(lmin, OpMin(), lsm.f);
    mx = block_reduce(lmax, OpMax(), lsm.f);
  }
  float delta, offset;
  solve_range(A, mn, mx, 0.f, 0.f, 0.f, static_cast<float>(A.num_bits), delta, offset);
  const LeafParam q = make_leaf_param(FQB200_LEAF_COMPILED, delta, offset, static_cast<float>(A.num_bits), A.relu_passthrough != 0);
  if (blockIdx.x == 0 && t == 0) export_stats(A, 0, mn, mx, 0.f, 0.f, 0.f, delta, offset, static_cast<float>(A.num_bits), q);
  if (blockIdx.x == 0) stamp(A, 7);
  if (!A.stats_only) {
    RowsApply ap{A, q, make_divisor(q.a), {bias[0], bias[1], bias[2], bias[3]}};
    ap.init_residual(c0, active);
    if (A.pool.tiles && A.pool.kind == 3u)
      consume_pool3_phase(g, A.pool, ring, fq_dyn, pos, ap);
    else if (A.pool.tiles)
      consume_pool_phase(g, A.pool, ring, fq_dyn, pos, ap);
    else if (A.residual)
      consume_pair_phase(half_geo(g), ring, fq_dyn, pos, ap);
    else
      consume_phase(g, ring, fq_dyn, pos, ap);
    if (blockIdx.x == 0) stamp(A, 9);
  }
  grid_exit_cl(A.sync);
}

}  // namespace fqb
