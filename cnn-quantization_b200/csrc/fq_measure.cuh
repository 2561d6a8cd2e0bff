// Activation norm measurement (`-ms`, distance_stats.py:22-33): the float64 sum of x * x over every contiguous row (one
// sample, in NCHW and channels-last memory alike).  Two launches, no host synchronisation, no atomics on the values:
//
//   fq_sumsq_partial_kernel  read x (4 B/element)  one (row, chunk) unit per CTA iteration: each thread sums its strided
//                                                  elements in float64, then a fixed warp / CTA tree; the unit's partial
//                                                  goes to its own workspace slot (or straight to out when a row is one
//                                                  chunk)
//   fq_sumsq_finish_kernel   one thread per row    adds the row's partials in chunk order
//
// The chunk length depends on row_len only and every unit is reduced in a fixed order by whichever CTA takes it, so the
// result has the same bits on every run and for every grid size.  x * x is exact in float64; NaN and Inf propagate.
namespace fqb {

constexpr int kSumsqThreads = 256;
constexpr unsigned long long kSumsqChunk = 16384;   // elements per work unit (64 KB), a multiple of 4

struct SumsqArgs {
  const float* in;
  unsigned long long rows, row_len;  // row r is in[r * row_len, (r + 1) * row_len)
  unsigned long long chunk;          // elements per unit (a multiple of 4 when the row is longer than one unit)
  unsigned long long chunks;         // units per row
  double* partial;                   // [rows][chunks] (chunks > 1)
  double* out;                       // [rows]
};

__host__ __device__ inline unsigned long long sumsq_chunk(unsigned long long row_len) {
  return row_len <= kSumsqChunk ? row_len : kSumsqChunk;
}

template <int VEC>
__global__ void __launch_bounds__(kSumsqThreads) fq_sumsq_partial_kernel(const __grid_constant__ SumsqArgs A) {
  using V = typename VecT<VEC>::type;
  __shared__ double red[kSumsqThreads / 32];
  const unsigned long long units = A.rows * A.chunks;
  for (unsigned long long u = blockIdx.x; u < units; u += gridDim.x) {
    const unsigned long long row = u / A.chunks, c = u % A.chunks;
    const unsigned long long e0 = c * A.chunk;
    const unsigned long long e1 = e0 + A.chunk < A.row_len ? e0 + A.chunk : A.row_len;
    const V* p = reinterpret_cast<const V*>(A.in + row * A.row_len);
    const unsigned long long v0 = e0 / VEC, v1 = e1 / VEC;
    double s = 0.0;
    unsigned long long v = v0 + threadIdx.x;
    // four independent loads in flight per thread, summed in index order
    for (; v + 3ull * kSumsqThreads < v1; v += 4ull * kSumsqThreads) {
      V x[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) x[k] = __ldg(p + v + k * kSumsqThreads);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if constexpr (VEC == 4) {
          s = __fma_rn(static_cast<double>(x[k].x), static_cast<double>(x[k].x), s);
          s = __fma_rn(static_cast<double>(x[k].y), static_cast<double>(x[k].y), s);
          s = __fma_rn(static_cast<double>(x[k].z), static_cast<double>(x[k].z), s);
          s = __fma_rn(static_cast<double>(x[k].w), static_cast<double>(x[k].w), s);
        } else {
          s = __fma_rn(static_cast<double>(x[k]), static_cast<double>(x[k]), s);
        }
      }
    }
    for (; v < v1; v += kSumsqThreads) {
      const V x = __ldg(p + v);
      if constexpr (VEC == 4) {
        s = __fma_rn(static_cast<double>(x.x), static_cast<double>(x.x), s);
        s = __fma_rn(static_cast<double>(x.y), static_cast<double>(x.y), s);
        s = __fma_rn(static_cast<double>(x.z), static_cast<double>(x.z), s);
        s = __fma_rn(static_cast<double>(x.w), static_cast<double>(x.w), s);
      } else {
        s = __fma_rn(static_cast<double>(x), static_cast<double>(x), s);
      }
    }
    for (int o = 16; o; o >>= 1) s = __dadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = red[0];
      for (int w = 1; w < kSumsqThreads / 32; ++w) t = __dadd_rn(t, red[w]);
      if (A.chunks == 1) A.out[row] = t;
      else A.partial[u] = t;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kSumsqThreads) fq_sumsq_finish_kernel(const __grid_constant__ SumsqArgs A) {
  const unsigned long long row = static_cast<unsigned long long>(blockIdx.x) * kSumsqThreads + threadIdx.x;
  if (row >= A.rows) return;
  const double* p = A.partial + row * A.chunks;
  double t = p[0];
  for (unsigned long long c = 1; c < A.chunks; ++c) t = __dadd_rn(t, p[c]);
  A.out[row] = t;
}

}  // namespace fqb
