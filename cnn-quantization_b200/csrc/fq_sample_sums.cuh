// Per-sample float64 sums over every contiguous row (one sample, in NCHW and channels-last memory alike) of a tensor y, for
// the activation norm measurement (`-ms`, distance_stats.py:22-33) and the quantization-noise measurement (`-ms` with
// measure_stats_kind="noise", measure_statistics.py:19-99).  The sum set S is a template parameter:
//
//   S = 1   out[r]           sum y^2                                       (the activation norm)
//   S = 2   out[r * 2 + k]   k = 0 sum y   1 sum y^2                       (noise: the layer input, the weight)
//   S = 7   out[r * 7 + k]   k = 0 sum y   1 sum y^2   2 sum q   3 sum q^2   4 sum y * q   5 sum e   6 sum e^2
//
// y may carry the convolution bias the quantization launch adds, as the same single fp32 add; q is y's quantized form and
// e = y - q.  fp32 values are exact in float64, so are their products, and e is formed in float64.  Two launches, no host
// synchronisation, no atomics on the values:
//
//   fq_sums_partial_kernel  read y (and q)         one (row, chunk) unit per CTA iteration: each thread sums its strided
//                                                  elements, then a fixed warp / CTA tree; the unit's partials go to their
//                                                  own workspace slots (or straight to out when a row is one chunk)
//   fq_sums_finish_kernel   one thread per output  adds a row's partials in chunk order
//
// The chunk length depends on row_len only and every unit is reduced in a fixed order by whichever CTA takes it, so the
// result has the same bits on every run and for every grid size.  NaN and Inf propagate.
namespace fqb {

constexpr int kSumsThreads = 256;
constexpr int kSumsMax = 7;                        // the largest sum set: S = 7
constexpr unsigned long long kSumsChunk = 16384;   // elements per work unit (64 KB of y), a multiple of 4
enum { kSumsBiasNone = 0, kSumsBiasNchw = 1, kSumsBiasCl = 2 };

struct SumsArgs {
  const float* y;
  const float* q;                    // S = 7 only
  const float* bias;                 // BIAS != none: element i of a row gets bias[i / period] (NCHW) or bias[i % period]
  unsigned period;                   // H*W (NCHW) or C (channels-last)
  unsigned long long rows, row_len;  // row r is [r * row_len, (r + 1) * row_len)
  unsigned long long chunk;          // elements per unit (a multiple of 4 when the row is longer than one unit)
  unsigned long long chunks;         // units per row
  double* partial;                   // [rows][chunks][S] (chunks > 1)
  double* out;                       // [rows][S]
};

__host__ __device__ inline unsigned long long sums_chunk(unsigned long long row_len) {
  return row_len <= kSumsChunk ? row_len : kSumsChunk;
}

template <int S>
__device__ __forceinline__ void sums_acc(double (&s)[S], float yv, float qv) {
  static_assert(S == 1 || S == 2 || S == kSumsMax, "sum sets: {y^2}, {y, y^2}, {y, y^2, q, q^2, yq, e, e^2}");
  const double y = static_cast<double>(yv);
  if constexpr (S == 1) {
    s[0] = __fma_rn(y, y, s[0]);
  } else {
    s[0] = __dadd_rn(s[0], y);
    s[1] = __fma_rn(y, y, s[1]);
  }
  if constexpr (S == kSumsMax) {
    const double q = static_cast<double>(qv);
    const double e = __dsub_rn(y, q);
    s[2] = __dadd_rn(s[2], q);
    s[3] = __fma_rn(q, q, s[3]);
    s[4] = __fma_rn(y, q, s[4]);
    s[5] = __dadd_rn(s[5], e);
    s[6] = __fma_rn(e, e, s[6]);
  }
}

// the bias of element i of a row (i < 2^32: the host refuses longer rows with a bias)
template <int BIAS>
__device__ __forceinline__ float sums_bias(const SumsArgs& A, unsigned i) {
  if constexpr (BIAS == kSumsBiasNchw) return __ldg(A.bias + i / A.period);
  else if constexpr (BIAS == kSumsBiasCl) return __ldg(A.bias + i % A.period);
  else return 0.f;
}

// one vector of VEC elements starting at row element i: y (+ bias, one fp32 add as the quantization launch does) and q
template <int VEC, int S, int BIAS>
__device__ __forceinline__ void sums_vec(const SumsArgs& A, double (&s)[S], typename VecT<VEC>::type yv,
                                         typename VecT<VEC>::type qv, unsigned i) {
  constexpr bool Q = S == kSumsMax;
  if constexpr (VEC == 4) {
    float b[4] = {0.f, 0.f, 0.f, 0.f};
    if constexpr (BIAS == kSumsBiasNchw) {   // one division per vector, then step through the channel boundary
      unsigned c = i / A.period, r = i - c * A.period;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        b[k] = __ldg(A.bias + c);
        if (++r == A.period && k < 3) { r = 0; ++c; }
      }
    } else if constexpr (BIAS == kSumsBiasCl) {
      unsigned c = i % A.period;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        b[k] = __ldg(A.bias + c);
        if (++c == A.period) c = 0;
      }
    }
    const float y0 = BIAS ? __fadd_rn(yv.x, b[0]) : yv.x, y1 = BIAS ? __fadd_rn(yv.y, b[1]) : yv.y;
    const float y2 = BIAS ? __fadd_rn(yv.z, b[2]) : yv.z, y3 = BIAS ? __fadd_rn(yv.w, b[3]) : yv.w;
    sums_acc<S>(s, y0, Q ? qv.x : 0.f);
    sums_acc<S>(s, y1, Q ? qv.y : 0.f);
    sums_acc<S>(s, y2, Q ? qv.z : 0.f);
    sums_acc<S>(s, y3, Q ? qv.w : 0.f);
  } else {
    sums_acc<S>(s, BIAS ? __fadd_rn(yv, sums_bias<BIAS>(A, i)) : yv, Q ? qv : 0.f);
  }
}

template <int VEC, int S, int BIAS>
__global__ void __launch_bounds__(kSumsThreads) fq_sums_partial_kernel(const __grid_constant__ SumsArgs A) {
  using V = typename VecT<VEC>::type;
  constexpr bool Q = S == kSumsMax;
  __shared__ double red[S][kSumsThreads / 32];
  const unsigned long long units = A.rows * A.chunks;
  for (unsigned long long u = blockIdx.x; u < units; u += gridDim.x) {
    const unsigned long long row = u / A.chunks, c = u % A.chunks;
    const unsigned long long e0 = c * A.chunk;
    const unsigned long long e1 = e0 + A.chunk < A.row_len ? e0 + A.chunk : A.row_len;
    const V* py = reinterpret_cast<const V*>(A.y + row * A.row_len);
    const V* pq = reinterpret_cast<const V*>(Q ? A.q + row * A.row_len : A.y);
    const unsigned long long v0 = e0 / VEC, v1 = e1 / VEC;
    double s[S];
#pragma unroll
    for (int k = 0; k < S; ++k) s[k] = 0.0;
    unsigned long long v = v0 + threadIdx.x;
    // four independent vector pairs in flight per thread, summed in index order
    for (; v + 3ull * kSumsThreads < v1; v += 4ull * kSumsThreads) {
      V y[4], q[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        y[k] = __ldg(py + v + k * kSumsThreads);
        if constexpr (Q) q[k] = __ldg(pq + v + k * kSumsThreads);
        else q[k] = y[k];
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) sums_vec<VEC, S, BIAS>(A, s, y[k], q[k], static_cast<unsigned>((v + k * kSumsThreads) * VEC));
    }
    for (; v < v1; v += kSumsThreads) {
      const V y = __ldg(py + v);
      const V q = Q ? __ldg(pq + v) : y;
      sums_vec<VEC, S, BIAS>(A, s, y, q, static_cast<unsigned>(v * VEC));
    }
#pragma unroll
    for (int k = 0; k < S; ++k) {
      for (int o = 16; o; o >>= 1) s[k] = __dadd_rn(s[k], __shfl_xor_sync(0xffffffffu, s[k], o));
      if ((threadIdx.x & 31) == 0) red[k][threadIdx.x >> 5] = s[k];
    }
    __syncthreads();
    if (threadIdx.x < S) {
      const int k = threadIdx.x;
      double t = red[k][0];
      for (int w = 1; w < kSumsThreads / 32; ++w) t = __dadd_rn(t, red[k][w]);
      if (A.chunks == 1) A.out[row * S + k] = t;
      else A.partial[u * S + k] = t;
    }
    __syncthreads();
  }
}

template <int S>
__global__ void __launch_bounds__(kSumsThreads) fq_sums_finish_kernel(const __grid_constant__ SumsArgs A) {
  const unsigned long long i = static_cast<unsigned long long>(blockIdx.x) * kSumsThreads + threadIdx.x;
  if (i >= A.rows * S) return;
  const unsigned long long row = i / S, k = i % S;
  const double* p = A.partial + row * A.chunks * S + k;
  double t = p[0];
  for (unsigned long long c = 1; c < A.chunks; ++c) t = __dadd_rn(t, p[c * S]);
  A.out[i] = t;
}

}  // namespace fqb
