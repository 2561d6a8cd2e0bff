// Clipping-error measurement (`-sm collect` with collect_err; statistic_manager.py:83-111,
// statistic_manager_perchannel.py:80-116): per group, the float64 sums behind the mse_* / cos_* columns for the three
// candidate quantizers get_alpha(clip_type='mix') chooses between (int_quantizer.py:310-323), in one read of x and
// without writing any quantized tensor.  Included by fqb200.cu after solve_range / make_leaf_param / leaf_apply.
//
//   candidate k   0 lowp: alpha = (max - min) / 2    1 gaus: std * F_gaus[num_bits]    2 laplace: b * F_laplace[bits]
//   each through solve_range (alpha2DeltaOffset: float64 per tensor, fp32 per channel) and make_leaf_param(LEAF_TORCH),
//   with the statistics of the [groups][FQB200_STATS_STRIDE] table of a stats_only fqb200_fused launch on the same
//   tensor (bits = that table's allocated width with bit_alloc), so each candidate is the leaf the on-the-fly
//   quantizer of that clip type applies to the tensor.
//
//   sums[g] = { sum x^2,  sum (x - q_k)^2 (k = 0..2),  sum x * q_k (k = 0..2),  sum q_k^2 (k = 0..2) }
//
//   fq_cliperr_partial_kernel  read x (4 B/element)  fixed work units: (group, chunk of kCeChunk elements) on NCHW /
//                                                    per-tensor layouts (128-bit loads when inner % 4 == 0 and x is
//                                                    16-byte aligned), (32-channel slab, kCeClRows pixels) on channels-last
//                                                    [N][HW][C] memory (one channel per lane, coalesced 4-byte loads).
//                                                    Every element is summed in float64 by a fixed thread in a fixed order,
//                                                    then a fixed warp / CTA tree; each unit writes its own workspace slot.
//   fq_cliperr_finish_kernel   one CTA per group     adds the group's unit partials (fixed per-thread stride, fixed tree),
//                                                    writes sums[g] and, optionally, the candidates' parameters.
//
// No atomics touch the values: the result has the same bits on every run and for every grid size.  x - q, x * q and q * q
// are exact or correctly rounded in float64; NaN propagates.
namespace fqb {

constexpr int kCeThreads = 256;
constexpr int kCeWarps = kCeThreads / 32;
constexpr int kCeSums = 10;
constexpr int kCeParams = 6;                     // per candidate: delta, offset, bits, scale, zero point, qmax
constexpr unsigned long long kCeChunk = 16384;   // NCHW / per tensor: elements of one group per unit (a multiple of 4)
constexpr unsigned long long kCeClRows = 512;    // channels-last: pixels per unit
constexpr unsigned kCeSlab = 32;                 // channels-last: channels per unit (one per lane)

struct ClipErrArgs {
  const float* in;
  const float* stats;                  // [groups][FQB200_STATS_STRIDE]
  unsigned long long outer, groups, inner;
  int channels_last, num_bits, positive, bit_alloc, solve_f64;
  unsigned long long units_per_group;  // NCHW: chunks of one group; channels-last: pixel chunks (of every slab)
  unsigned long long units;
  double* partial;                     // [groups][units_per_group][kCeSums]
  double* out;                         // [groups][kCeSums]
  float* params;                       // optional [groups][3][kCeParams]
};

// candidate k of group g: (delta, offset, bits) by the on-the-fly solve, then the torch leaf's parameters
__device__ __forceinline__ LeafParam ce_candidate(const ClipErrArgs& A, unsigned long long g, int k, float& delta, float& offset,
                                                  float& bits) {
  const float* t = A.stats + g * FQB200_STATS_STRIDE;
  bits = A.bit_alloc ? __ldg(t + 7) : static_cast<float>(A.num_bits);
  const int mode = k == 0 ? kRangeLowp : (k == 1 ? FQB200_RANGE_GAUS : FQB200_RANGE_LAPLACE);
  solve_range(mode, A.positive != 0, A.num_bits, 0.f, A.solve_f64 != 0, __ldg(t + 0), __ldg(t + 1), __ldg(t + 2),
              __ldg(t + 3), __ldg(t + 4), bits, delta, offset);
  return make_leaf_param(FQB200_LEAF_TORCH, delta, offset, bits);
}

struct CeCands {
  LeafParam q[3];
  Divisor dv[3];
  bool fast;   // all three divisors take the exact 3-instruction division
};

__device__ __forceinline__ CeCands ce_cands(const ClipErrArgs& A, unsigned long long g) {
  CeCands c;
  c.fast = true;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    float d, o, b;
    c.q[k] = ce_candidate(A, g, k, d, o, b);
    c.dv[k] = make_divisor(c.q[k].a);
    c.fast = c.fast && c.dv[k].fast;
  }
  return c;
}

template <bool FAST>
__device__ __forceinline__ void ce_add(double (&s)[kCeSums], float x, const CeCands& c) {
  const double xd = static_cast<double>(x);
  s[0] = __fma_rn(xd, xd, s[0]);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    float grid;
    const double qd = static_cast<double>(leaf_apply<FQB200_LEAF_TORCH, FAST>(x, c.q[k], c.dv[k], 0.f, grid));
    const double d = __dsub_rn(xd, qd);
    s[1 + k] = __fma_rn(d, d, s[1 + k]);
    s[4 + k] = __fma_rn(xd, qd, s[4 + k]);
    s[7 + k] = __fma_rn(qd, qd, s[7 + k]);
  }
}

template <bool FAST>
__device__ __forceinline__ void ce_add4(double (&s)[kCeSums], const float4& v, const CeCands& c) {
  ce_add<FAST>(s, v.x, c);
  ce_add<FAST>(s, v.y, c);
  ce_add<FAST>(s, v.z, c);
  ce_add<FAST>(s, v.w, c);
}

// one (group, chunk) unit of an NCHW / per-tensor layout: logical index k = o * inner + i of the group's outer * inner
// elements, at offset (o * groups + g) * inner + i.  The host guarantees outer * inner < 2^32 when outer > 1.
template <int VEC, bool FAST>
__device__ __forceinline__ void ce_unit_nchw(const ClipErrArgs& A, unsigned long long g, unsigned long long k0,
                                             unsigned long long k1, const CeCands& c, double (&s)[kCeSums]) {
  const unsigned inner32 = static_cast<unsigned>(A.inner);
  auto offset = [&](unsigned long long k) -> unsigned long long {
    if (A.outer == 1) return g * A.inner + k;
    const unsigned kk = static_cast<unsigned>(k);
    const unsigned o = kk / inner32;
    return (static_cast<unsigned long long>(o) * A.groups + g) * A.inner + (kk - o * inner32);
  };
  constexpr unsigned long long step = static_cast<unsigned long long>(VEC) * kCeThreads;
  unsigned long long k = k0 + static_cast<unsigned long long>(VEC) * threadIdx.x;
  if constexpr (VEC == 4) {
    // four independent 128-bit loads in flight per thread (inner % 4 == 0: a vector never straddles a row)
    for (; k + 3 * step < k1; k += 4 * step) {
      float4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = __ldg(reinterpret_cast<const float4*>(A.in + offset(k + u * step)));
#pragma unroll
      for (int u = 0; u < 4; ++u) ce_add4<FAST>(s, v[u], c);
    }
    for (; k < k1; k += step) ce_add4<FAST>(s, __ldg(reinterpret_cast<const float4*>(A.in + offset(k))), c);
  } else {
    for (; k + 3 * step < k1; k += 4 * step) {
      float v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = __ldg(A.in + offset(k + u * step));
#pragma unroll
      for (int u = 0; u < 4; ++u) ce_add<FAST>(s, v[u], c);
    }
    for (; k < k1; k += step) ce_add<FAST>(s, __ldg(A.in + offset(k)), c);
  }
}

// one (slab, pixel chunk) unit of a channels-last layout: lane = channel of the slab, warp w takes pixels r0 + w + 8 j
template <bool FAST>
__device__ __forceinline__ void ce_unit_cl(const ClipErrArgs& A, unsigned long long c, unsigned long long r0,
                                           unsigned long long r1, const CeCands& cand, double (&s)[kCeSums]) {
  if (c >= A.groups) return;
  const unsigned long long w = threadIdx.x >> 5;
  unsigned long long r = r0 + w;
  for (; r + 3 * kCeWarps < r1; r += 4 * kCeWarps) {
    float v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u] = __ldg(A.in + (r + u * kCeWarps) * A.groups + c);
#pragma unroll
    for (int u = 0; u < 4; ++u) ce_add<FAST>(s, v[u], cand);
  }
  for (; r < r1; r += kCeWarps) ce_add<FAST>(s, __ldg(A.in + r * A.groups + c), cand);
}

template <int VEC>
__global__ void __launch_bounds__(kCeThreads) fq_cliperr_partial_kernel(const __grid_constant__ ClipErrArgs A) {
  __shared__ double red[kCeWarps][32][kCeSums];
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (unsigned long long u = blockIdx.x; u < A.units; u += gridDim.x) {
    double s[kCeSums];
#pragma unroll
    for (int k = 0; k < kCeSums; ++k) s[k] = 0.0;
    const unsigned long long slab_or_g = u / A.units_per_group, chunk = u % A.units_per_group;
    if (A.channels_last) {
      const unsigned long long c = slab_or_g * kCeSlab + lane;
      const CeCands cand = ce_cands(A, c < A.groups ? c : A.groups - 1);
      const bool fast = __syncthreads_and(cand.fast) != 0;   // the same slab in every warp: uniform over the CTA
      const unsigned long long rows = A.outer * A.inner, r0 = chunk * kCeClRows;
      const unsigned long long r1 = r0 + kCeClRows < rows ? r0 + kCeClRows : rows;
      if (fast) ce_unit_cl<true>(A, c, r0, r1, cand, s);
      else      ce_unit_cl<false>(A, c, r0, r1, cand, s);
    } else {
      const unsigned long long g = slab_or_g, n = A.outer * A.inner, k0 = chunk * kCeChunk;
      const unsigned long long k1 = k0 + kCeChunk < n ? k0 + kCeChunk : n;
      const CeCands cand = ce_cands(A, g);
      if (cand.fast) ce_unit_nchw<VEC, true>(A, g, k0, k1, cand, s);
      else           ce_unit_nchw<VEC, false>(A, g, k0, k1, cand, s);
      // every thread holds a share of the same group: a fixed xor tree over the warp first
#pragma unroll
      for (int k = 0; k < kCeSums; ++k)
        for (int o = 16; o; o >>= 1) s[k] = __dadd_rn(s[k], __shfl_xor_sync(0xffffffffu, s[k], o));
    }
#pragma unroll
    for (int k = 0; k < kCeSums; ++k) red[warp][lane][k] = s[k];
    __syncthreads();
    if (A.channels_last) {
      // per channel (lane of every warp): warps added in order
      for (unsigned i = threadIdx.x; i < 32u * kCeSums; i += kCeThreads) {
        const unsigned l = i / kCeSums, k = i % kCeSums;
        const unsigned long long c = slab_or_g * kCeSlab + l;
        if (c >= A.groups) continue;
        double t = red[0][l][k];
        for (int w2 = 1; w2 < kCeWarps; ++w2) t = __dadd_rn(t, red[w2][l][k]);
        A.partial[(c * A.units_per_group + chunk) * kCeSums + k] = t;
      }
    } else if (threadIdx.x < kCeSums) {
      double t = red[0][0][threadIdx.x];
      for (int w2 = 1; w2 < kCeWarps; ++w2) t = __dadd_rn(t, red[w2][0][threadIdx.x]);
      A.partial[u * kCeSums + threadIdx.x] = t;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kCeThreads) fq_cliperr_finish_kernel(const __grid_constant__ ClipErrArgs A) {
  __shared__ double red[kCeWarps][kCeSums];
  const unsigned long long g = blockIdx.x;
  const double* p = A.partial + g * A.units_per_group * kCeSums;
  double s[kCeSums];
#pragma unroll
  for (int k = 0; k < kCeSums; ++k) s[k] = 0.0;
  for (unsigned long long u = threadIdx.x; u < A.units_per_group; u += kCeThreads) {
#pragma unroll
    for (int k = 0; k < kCeSums; ++k) s[k] = __dadd_rn(s[k], p[u * kCeSums + k]);
  }
#pragma unroll
  for (int k = 0; k < kCeSums; ++k)
    for (int o = 16; o; o >>= 1) s[k] = __dadd_rn(s[k], __shfl_xor_sync(0xffffffffu, s[k], o));
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int k = 0; k < kCeSums; ++k) red[threadIdx.x >> 5][k] = s[k];
  }
  __syncthreads();
  if (threadIdx.x < kCeSums) {
    double t = red[0][threadIdx.x];
    for (int w = 1; w < kCeWarps; ++w) t = __dadd_rn(t, red[w][threadIdx.x]);
    A.out[g * kCeSums + threadIdx.x] = t;
  }
  if (A.params && threadIdx.x < 3) {
    float d, o, b;
    const LeafParam q = ce_candidate(A, g, threadIdx.x, d, o, b);
    float* dst = A.params + (g * 3 + threadIdx.x) * kCeParams;
    dst[0] = d; dst[1] = o; dst[2] = b; dst[3] = q.a; dst[4] = q.b; dst[5] = q.c;
  }
}

}  // namespace fqb
