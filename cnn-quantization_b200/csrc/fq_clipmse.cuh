// Clipping-MSE curves (`-sm collect` with collect_mse; the simulation half of the reference's mse_analysis.py, eq. 6 of
// the paper, run on real activations with the quantizer this library applies): per group, the float64 sum of the squared
// error of K candidate quantizers that differ only in their clipping value, in one read of x and without writing any
// quantized tensor.  Included by fqb200.cu after solve_range / make_leaf_param / leaf_apply.
//
//   candidate k   alpha = m_k * b (prior 0, Laplace) or m_k * std (prior 1, Gauss), one fp32 multiply like the Laplace
//                 rule's b * F[bits]; then solve_range (alpha2DeltaOffset: float64 when solve_f64, else fp32) and
//                 make_leaf_param(LEAF_TORCH) with the statistics of the [groups][FQB200_STATS_STRIDE] table of a stats_only
//                 fqb200_fused launch on the same tensor (bits = that table's allocated width with bit_alloc), as
//                 ce_candidate does for the three fixed candidates of fq_cliperr.cuh.  Prior 2 is the min/max range
//                 (FQB200_RANGE_MINMAX, lower bound 0 when positive) and ignores m_k.
//                 With per-candidate widths (`-bap mse`'s bit-allocation tables) candidate k quantizes at widths[k]
//                 (0..8) instead, so one launch measures a channel's error at every width.
//   grid launch   (fqb200_clip_mse_grid, the joint width-and-clip tables of `-c mse -bap mse`): nw widths times K
//                 multipliers; candidate j = i * K + k quantizes at widths[i] and clips at mult[k].  The width is one
//                 more unit dimension, so a unit runs one width's K candidates with one qmax, in the shared memory of a
//                 K-candidate launch, and every column has the bits of the per-candidate-width launch on that pair.
//
//   out[g] = { sum x^2,  sum (x - q_j)^2 (j = 0 .. nw*K-1) }      d = x - q_j formed in float64 as in ce_add
//
//   fq_clipmse_partial_kernel  fixed work units: (group, chunk of kCmChunk elements) on NCHW / per-tensor layouts (128-bit
//                              loads when inner % 4 == 0 and x is 16-byte aligned), (32-channel slab, kCmClRows pixels) on
//                              channels-last [N][HW][C] memory (one channel per lane), times the nw widths of a grid
//                              launch (adjacent units, so the chunk's other reads hit L2).  A unit first solves its candidates'
//                              parameters and divisors into shared memory.  It then walks its chunk in pieces of kCmPer
//                              elements per thread, each loaded once from global memory into registers; every candidate
//                              tile of kCmTile float64 accumulators runs over the piece in registers, and a fixed
//                              warp / CTA tree adds the tile into the unit's shared-memory sums.  Each unit writes its own
//                              workspace slot; sum x^2 comes from the units of width 0 only.
//   fq_clipmse_finish_kernel   one CTA per group: adds the group's unit partials in chunk order, writes out[g] and,
//                              optionally, the candidates' parameters.  A select launch (fqb200_clip_mse_select, `-c mse`
//                              on the fly) then picks the group's column in statistics.best_columns' order (cm_before)
//                              with one warp over the final sums, and writes that candidate's parameters.
//
// No atomics touch the values: the result has the same bits on every run and for every grid size.  NaN propagates.
namespace fqb {

constexpr int kCmThreads = 256;
constexpr int kCmWarps = kCmThreads / 32;
constexpr int kCmMaxK = 256;
constexpr int kCmTile = 8;    // candidates per register tile (float64 accumulators)
constexpr int kCmPer = 32;    // elements per thread per piece
constexpr unsigned long long kCmPiece = static_cast<unsigned long long>(kCmPer) * kCmThreads;   // NCHW: elements per piece
constexpr unsigned long long kCmChunk = 32 * kCmPiece;                                           // NCHW: elements per unit
constexpr unsigned long long kCmClPiece = static_cast<unsigned long long>(kCmPer) * kCmWarps;   // channels-last: pixels per piece
constexpr unsigned long long kCmClRows = 32 * kCmClPiece;                                        // channels-last: pixels per unit
constexpr unsigned kCmSlab = 32;
static_assert(kCmTile == kCmWarps, "the channels-last fold gives each warp one candidate of the tile");

struct ClipMseArgs {
  const float* in;
  const float* stats;                  // [groups][FQB200_STATS_STRIDE]
  const float* mult;                   // [K] clipping multipliers
  unsigned long long outer, groups, inner;
  int channels_last, num_bits, positive, bit_alloc, solve_f64, prior, K, Kpad;
  int has_widths;                      // widths[k] is candidate k's width (else num_bits or the table's column 7)
  int grid;                            // grid launch: widths[i] is the width of unit width index i (has_widths is 0)
  int nw;                              // widths per (group, chunk): nw of a grid launch, else 1
  unsigned char widths[kCmMaxK];
  unsigned long long units_per_group;  // NCHW: chunks of one group; channels-last: pixel chunks (of every slab)
  unsigned long long units;
  double* partial;                     // [groups][units_per_group][nw * K + 1]
  double* out;                         // [groups][nw * K + 1]
  float* params;                       // optional [groups][nw * K][kCeParams]
  int* choice;                         // select launch: [groups] chosen column (nullptr: no selection)
  float* given;                        // select launch: [3][groups] chosen delta, offset, bits
  float* table;                        // select launch, optional: [groups][FQB200_STATS_STRIDE] parameter table
};

// candidate k (of width index wi in a grid launch) of group g: alpha = mult[k] * (b or std) - solve_range's k-std rule
// with the prior's scale in the std slot - or, prior 2, the min/max range
__device__ __forceinline__ LeafParam cm_candidate(const ClipMseArgs& A, unsigned long long g, int k, int wi, float& delta,
                                                  float& offset, float& bits) {
  const float* t = A.stats + g * FQB200_STATS_STRIDE;
  bits = A.grid         ? static_cast<float>(A.widths[wi])
         : A.has_widths ? static_cast<float>(A.widths[k])
         : A.bit_alloc  ? __ldg(t + 7)
                        : static_cast<float>(A.num_bits);
  solve_range(A.prior == 2 ? FQB200_RANGE_MINMAX : FQB200_RANGE_KSTD, A.positive != 0, A.num_bits, __ldg(A.mult + k),
              A.solve_f64 != 0, __ldg(t + 0), __ldg(t + 1), __ldg(t + 2), __ldg(t + 3), __ldg(t + (A.prior ? 4 : 3)), bits,
              delta, offset);
  return make_leaf_param(FQB200_LEAF_TORCH, delta, offset, bits);
}

// dynamic shared memory of a unit with S groups side by side (1 on NCHW, kCmSlab on channels-last)
struct CmSmem {
  double* acc;                // [K + 1][S]: sum x^2, then the candidates' sums
  double* red;                // [2][kCmWarps][kCmTile][S]: fold buffers, alternating
  float *scale, *zp, *rcp;    // [Kpad][S]: the candidates' leaf parameters and reciprocals (Kpad - K copies of the last)
  float* qmax;                // [S]; with per-candidate widths qmax = 2^w - 1 comes from the width instead
};
__host__ __device__ inline size_t cm_smem_bytes(int K, int S) {
  const int kpad = (K + kCmTile - 1) / kCmTile * kCmTile;
  return (static_cast<size_t>(K + 1) * S + 2ull * kCmWarps * kCmTile * S) * 8 + (3ull * kpad * S + S) * 4;
}
__device__ __forceinline__ CmSmem cm_carve(unsigned char* raw, int K, int Kpad, int S) {
  CmSmem s;
  s.acc = reinterpret_cast<double*>(raw);
  s.red = s.acc + (K + 1) * S;
  s.scale = reinterpret_cast<float*>(s.red + 2 * kCmWarps * kCmTile * S);
  s.zp = s.scale + Kpad * S;
  s.rcp = s.zp + Kpad * S;
  s.qmax = s.rcp + Kpad * S;
  return s;
}

// add a tile's per-thread sums s[0 .. n-1] into acc[k0 + c]: NCHW, every thread holds a share of the one group (xor
// tree over the warp, then the warps in order); channels-last, lane = channel (the warps in order, per channel).
template <bool CL>
__device__ __forceinline__ void cm_fold(const CmSmem& sm, double (&s)[kCmTile], int buf, int k0, int n) {
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if constexpr (CL) {
    double* red = sm.red + buf * (kCmWarps * kCmTile * kCmSlab);
#pragma unroll
    for (int c = 0; c < kCmTile; ++c) red[(warp * kCmTile + c) * kCmSlab + lane] = s[c];
    __syncthreads();
    const int c = static_cast<int>(warp);
    if (c < n) {
      double t = red[c * kCmSlab + lane];
      for (int w = 1; w < kCmWarps; ++w) t = __dadd_rn(t, red[(w * kCmTile + c) * kCmSlab + lane]);
      double* a = sm.acc + (k0 + c) * kCmSlab + lane;
      *a = __dadd_rn(*a, t);
    }
  } else {
    double* red = sm.red + buf * (kCmWarps * kCmTile);
#pragma unroll
    for (int c = 0; c < kCmTile; ++c)
      for (int o = 16; o; o >>= 1) s[c] = __dadd_rn(s[c], __shfl_xor_sync(0xffffffffu, s[c], o));
    if (lane == 0) {
#pragma unroll
      for (int c = 0; c < kCmTile; ++c) red[warp * kCmTile + c] = s[c];
    }
    __syncthreads();
    const int c = static_cast<int>(threadIdx.x);
    if (c < n) {
      double t = red[c];
      for (int w = 1; w < kCmWarps; ++w) t = __dadd_rn(t, red[w * kCmTile + c]);
      sm.acc[k0 + c] = __dadd_rn(sm.acc[k0 + c], t);
    }
  }
}

// element offset of logical index k = o * inner + i of NCHW group g (outer * inner < 2^32 when outer > 1)
__device__ __forceinline__ unsigned long long cm_nchw_offset(const ClipMseArgs& A, unsigned long long g, unsigned long long k) {
  if (A.outer == 1) return g * A.inner + k;
  const unsigned kk = static_cast<unsigned>(k), inner32 = static_cast<unsigned>(A.inner);
  const unsigned o = kk / inner32;
  return (static_cast<unsigned long long>(o) * A.groups + g) * A.inner + (kk - o * inner32);
}

// one unit: LAY 0 NCHW scalar loads, 1 NCHW float4 loads, 2 channels-last
template <int LAY, bool FAST>
__device__ __forceinline__ void cm_unit(const ClipMseArgs& A, const CmSmem& sm, unsigned long long sg, unsigned long long chunk) {
  constexpr bool CL = LAY == 2;
  constexpr int S = CL ? static_cast<int>(kCmSlab) : 1;
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned slot = CL ? lane : 0;
  const unsigned long long n = A.outer * A.inner, per = CL ? kCmClRows : kCmChunk, piece = CL ? kCmClPiece : kCmPiece;
  const unsigned long long begin = chunk * per, end = begin + per < n ? begin + per : n;
  const unsigned long long c = sg * kCmSlab + lane;   // channels-last: this lane's channel
  const bool live = !CL || c < A.groups;
  double sx = 0.0;
  int buf = 0;
  for (unsigned long long p0 = begin; p0 < end; p0 += piece) {
    float xv[kCmPer];
    int nv = 0;   // the valid elements of this thread are a prefix of xv
    if constexpr (LAY == 1) {
#pragma unroll
      for (int v = 0; v < kCmPer / 4; ++v) {
        const unsigned long long k = p0 + 4ull * threadIdx.x + 4ull * kCmThreads * v;
        float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k < end) {
          t = __ldg(reinterpret_cast<const float4*>(A.in + cm_nchw_offset(A, sg, k)));
          nv = 4 * v + 4;
        }
        xv[4 * v] = t.x; xv[4 * v + 1] = t.y; xv[4 * v + 2] = t.z; xv[4 * v + 3] = t.w;
      }
    } else {
#pragma unroll
      for (int j = 0; j < kCmPer; ++j) {
        const unsigned long long k = p0 + (CL ? warp : threadIdx.x) + static_cast<unsigned long long>(CL ? kCmWarps : kCmThreads) * j;
        xv[j] = 0.f;
        if (k < end && live) {
          xv[j] = __ldg(A.in + (CL ? k * A.groups + c : cm_nchw_offset(A, sg, k)));
          nv = j + 1;
        }
      }
    }
#pragma unroll
    for (int j = 0; j < kCmPer; ++j) {
      if (j < nv) {
        const double xd = static_cast<double>(xv[j]);
        sx = __fma_rn(xd, xd, sx);
      }
    }
    for (int k0 = 0; k0 < A.K; k0 += kCmTile) {
      LeafParam q[kCmTile];
      Divisor dv[kCmTile];
      const float qmax = sm.qmax[slot];
#pragma unroll
      for (int t = 0; t < kCmTile; ++t) {
        const int i = (k0 + t) * S + slot;
        q[t].a = sm.scale[i];
        q[t].b = sm.zp[i];
        q[t].c = A.has_widths ? static_cast<float>((1 << A.widths[min(k0 + t, A.K - 1)]) - 1) : qmax;
        q[t].flags = FLAG_TRUE_ZERO;
        dv[t].s = q[t].a;
        dv[t].r = sm.rcp[i];
        dv[t].fast = FAST;
      }
      double s[kCmTile];
#pragma unroll
      for (int t = 0; t < kCmTile; ++t) s[t] = 0.0;
#pragma unroll
      for (int j = 0; j < kCmPer; ++j) {
        if (j < nv) {
          const double xd = static_cast<double>(xv[j]);
#pragma unroll
          for (int t = 0; t < kCmTile; ++t) {
            float grid;
            const double qd = static_cast<double>(leaf_apply<FQB200_LEAF_TORCH, FAST>(xv[j], q[t], dv[t], 0.f, grid));
            const double d = __dsub_rn(xd, qd);
            s[t] = __fma_rn(d, d, s[t]);
          }
        }
      }
      cm_fold<CL>(sm, s, buf, 1 + k0, A.K - k0 < kCmTile ? A.K - k0 : kCmTile);
      buf ^= 1;
    }
  }
  double s[kCmTile];
#pragma unroll
  for (int t = 0; t < kCmTile; ++t) s[t] = t == 0 ? sx : 0.0;
  cm_fold<CL>(sm, s, buf, 0, 1);
}

template <int LAY>
__global__ void __launch_bounds__(kCmThreads, 2) fq_clipmse_partial_kernel(const __grid_constant__ ClipMseArgs A) {
  extern __shared__ __align__(16) unsigned char cm_raw[];
  constexpr int S = LAY == 2 ? static_cast<int>(kCmSlab) : 1;
  const CmSmem sm = cm_carve(cm_raw, A.K, A.Kpad, S);
  const int W = A.K + 1;
  for (unsigned long long u = blockIdx.x; u < A.units; u += gridDim.x) {
    const unsigned long long cu = u / static_cast<unsigned>(A.nw);   // unit = (group or slab, chunk, width index)
    const unsigned long long sg = cu / A.units_per_group, chunk = cu % A.units_per_group;
    const int wi = static_cast<int>(u - cu * static_cast<unsigned>(A.nw));
    bool fast = true;
    for (int i = threadIdx.x; i < A.Kpad * S; i += kCmThreads) {
      const int slot = i % S, k = i / S;
      unsigned long long g = LAY == 2 ? sg * kCmSlab + slot : sg;
      if (g >= A.groups) g = A.groups - 1;
      float d, o, b;
      const LeafParam q = cm_candidate(A, g, k < A.K ? k : A.K - 1, wi, d, o, b);
      const Divisor dv = make_divisor(q.a);
      sm.scale[i] = q.a;
      sm.zp[i] = q.b;
      sm.rcp[i] = dv.r;
      if (k == 0) sm.qmax[slot] = q.c;
      fast = fast && dv.fast;
    }
    for (int i = threadIdx.x; i < W * S; i += kCmThreads) sm.acc[i] = 0.0;
    if (__syncthreads_and(fast)) cm_unit<LAY, true>(A, sm, sg, chunk);
    else                         cm_unit<LAY, false>(A, sm, sg, chunk);
    __syncthreads();
    const int wi2 = static_cast<int>(u % static_cast<unsigned>(A.nw)), row = A.nw * A.K + 1;
    for (int i = threadIdx.x; i < W * S; i += kCmThreads) {
      const int slot = i % S, k = i / S;
      const unsigned long long g = LAY == 2 ? sg * kCmSlab + slot : sg;
      if (g < A.groups && (k > 0 || wi2 == 0)) A.partial[(g * A.units_per_group + chunk) * row + (k ? wi2 * A.K + k : 0)] = sm.acc[i];
    }
    __syncthreads();
  }
}

// one candidate in the selection: its error (NaN read as +inf, so it never wins), multiplier and column (-1: none)
struct CmPick {
  double e;
  float m;
  int k;
};
// true when a goes before b in statistics.best_columns' order: the smaller error, then the smaller multiplier (NaN
// last, as np.argsort puts it), then the earlier column.  A total order, so the warp's tree gives the same pick as a scan.
__device__ __forceinline__ bool cm_before(const CmPick& a, const CmPick& b) {
  if (a.k < 0 || b.k < 0) return b.k < 0 && a.k >= 0;
  if (a.e != b.e) return a.e < b.e;
  const bool an = isnan(a.m), bn = isnan(b.m);
  if (an != bn) return bn;
  if (!an && a.m != b.m) return a.m < b.m;
  return a.k < b.k;
}

// the select launch's tail, warp 0 of group g's finish CTA once out[g] is final: the chosen column and its candidate's
// (delta, offset, bits) and leaf, exactly as cm_candidate gives them to out_params
__device__ __forceinline__ void cm_select(const ClipMseArgs& A, unsigned long long g) {
  const double* e = A.out + g * (A.K + 1) + 1;
  CmPick p{0.0, 0.f, -1};
  for (int k = threadIdx.x; k < A.K; k += 32) {
    const double ek = e[k];
    const CmPick c{isnan(ek) ? static_cast<double>(INFINITY) : ek, __ldg(A.mult + k), k};
    if (cm_before(c, p)) p = c;
  }
  for (int o = 16; o; o >>= 1) {
    const CmPick c{__shfl_xor_sync(0xffffffffu, p.e, o), __shfl_xor_sync(0xffffffffu, p.m, o),
                   __shfl_xor_sync(0xffffffffu, p.k, o)};
    if (cm_before(c, p)) p = c;
  }
  if (threadIdx.x != 0) return;
  float d, o, b;
  const LeafParam q = cm_candidate(A, g, p.k, 0, d, o, b);
  A.choice[g] = p.k;
  A.given[g] = d;
  A.given[A.groups + g] = o;
  A.given[2 * A.groups + g] = b;
  if (A.table) {
    const float* t = A.stats + g * FQB200_STATS_STRIDE;
    float* dst = A.table + g * FQB200_STATS_STRIDE;
    for (int c = 0; c < 5; ++c) dst[c] = t[c];
    dst[5] = d; dst[6] = o; dst[7] = b; dst[8] = q.a; dst[9] = q.b; dst[10] = q.c; dst[11] = static_cast<float>(q.flags);
  }
}

__global__ void __launch_bounds__(kCmThreads) fq_clipmse_finish_kernel(const __grid_constant__ ClipMseArgs A) {
  const unsigned long long g = blockIdx.x;
  const int n = A.nw * A.K, W = n + 1;
  const double* p = A.partial + g * A.units_per_group * W;
  for (int k = threadIdx.x; k < W; k += kCmThreads) {
    double t = p[k];
    for (unsigned long long u = 1; u < A.units_per_group; ++u) t = __dadd_rn(t, p[u * W + k]);
    A.out[g * W + k] = t;
  }
  if (A.params) {
    for (int j = threadIdx.x; j < n; j += kCmThreads) {
      float d, o, b;
      const int wi = j / A.K;
      const LeafParam q = cm_candidate(A, g, j - wi * A.K, wi, d, o, b);
      float* dst = A.params + (g * n + j) * kCeParams;
      dst[0] = d; dst[1] = o; dst[2] = b; dst[3] = q.a; dst[4] = q.b; dst[5] = q.c;
    }
  }
  if (A.choice) {
    __syncthreads();   // the group's sums in out[g] are final and visible to the CTA
    if (threadIdx.x < 32) cm_select(A, g);
  }
}

}  // namespace fqb
