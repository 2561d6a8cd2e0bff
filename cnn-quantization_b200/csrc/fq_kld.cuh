// KL-divergence calibration (`-kld`, statistic_manager.py:80-82 -> kld_threshold.py:15-80): per sample row, a histogram of
// num_bins bins over (-th, th), th = max |x|, then the MXNet / TensorRT threshold search over the candidates
// i = num_quantized_bins/2 .. num_bins/2.  Three launches, no host synchronisation:
//
//   fq_kld_absmax_kernel  read x (4 B/element)  per-row max |x| as float bits, atomicMax into the workspace
//   fq_kld_hist_kernel    read x (4 B/element)  per-CTA shared-memory histograms against the fp32 edges, flushed with one
//                                               red.global per non-zero bin into rows x num_bins counters
//   fq_kld_search_kernel  one CTA per row       prefix sums of counts and non-zero flags in shared memory; one warp per
//                                               candidate, divergence in float64; argmin with numpy's rules
//
// The edges are those numpy 1.x computed: float32(linspace(-th, th, num_bins + 1)) evaluated in float64 (k * step + lo,
// last edge = hi), a degenerate range (th == 0) widened to (-0.5, 0.5).  A bin holds e_k <= x < e_{k+1}, the last one is
// closed, so the counts are exactly numpy's.  Rows whose max |x| is not finite (NaN / Inf inside) get th = div = NaN and
// idx = -1; the reference raises on them.
namespace fqb {

constexpr int kKldThreads = 512;
constexpr int kKldMaxReplicas = 4;

struct KldArgs {
  const float* in;
  unsigned long long rows, row_len;  // row r is in[r * row_len, (r + 1) * row_len)
  unsigned long long chunk;          // elements per histogram work unit (a multiple of 4)
  unsigned long long chunks;         // units per row
  unsigned* absmax;                  // [rows] float bits of max |x|
  unsigned* hist;                    // [rows][nb]
  int nb, nq, replicas;
  float* out_th;
  float* out_div;
  int* out_idx;
};

// numpy.linspace(lo, hi, nb + 1)[k] in float64 (y = k * step; y += lo; y[-1] = hi), rounded to float32
__host__ __device__ inline float kld_edge(double lo, double hi, int nb, int k) {
  if (k >= nb) return static_cast<float>(hi);
#ifdef __CUDA_ARCH__
  const double step = __ddiv_rn(__dsub_rn(hi, lo), static_cast<double>(nb));
  return __double2float_rn(__dadd_rn(__dmul_rn(static_cast<double>(k), step), lo));
#else
  const double step = (hi - lo) / nb;
  return static_cast<float>(static_cast<double>(k) * step + lo);
#endif
}

__device__ inline bool kld_range(const KldArgs& A, unsigned long long row, double* lo, double* hi) {
  const float th = __uint_as_float(A.absmax[row]);
  if (!(th <= 3.402823466e38f)) return false;  // NaN / Inf in the row
  *lo = -static_cast<double>(th);
  *hi = static_cast<double>(th);
  if (th == 0.f) *lo = -0.5, *hi = 0.5;
  return true;
}

template <int VEC>
__device__ inline void kld_unit(const KldArgs& A, unsigned long long unit, unsigned long long* row,
                                unsigned long long* v0, unsigned long long* v1) {
  *row = unit / A.chunks;
  const unsigned long long c = unit % A.chunks;
  const unsigned long long e0 = c * A.chunk;
  const unsigned long long e1 = e0 + A.chunk < A.row_len ? e0 + A.chunk : A.row_len;
  *v0 = e0 / VEC;
  *v1 = e1 / VEC;
}

template <int VEC>
__global__ void __launch_bounds__(kKldThreads) fq_kld_absmax_kernel(const __grid_constant__ KldArgs A) {
  using V = typename VecT<VEC>::type;
  __shared__ unsigned red[kKldThreads / 32];
  const unsigned long long units = A.rows * A.chunks;
  for (unsigned long long u = blockIdx.x; u < units; u += gridDim.x) {
    unsigned long long row, v0, v1;
    kld_unit<VEC>(A, u, &row, &v0, &v1);
    const V* p = reinterpret_cast<const V*>(A.in + row * A.row_len);
    unsigned m = 0;   // |x| as bits: the order of non-negative floats, NaN above Inf
    for (unsigned long long v = v0 + threadIdx.x; v < v1; v += kKldThreads) {
      const V x = __ldg(p + v);
      if constexpr (VEC == 4) {
        m = max(m, max(max(__float_as_uint(fabsf(x.x)), __float_as_uint(fabsf(x.y))),
                       max(__float_as_uint(fabsf(x.z)), __float_as_uint(fabsf(x.w)))));
      } else {
        m = max(m, __float_as_uint(fabsf(x)));
      }
    }
    for (int o = 16; o; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x < 32) {
      m = threadIdx.x < kKldThreads / 32 ? red[threadIdx.x] : 0u;
      for (int o = 16; o; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
      if (threadIdx.x == 0) atomicMax(A.absmax + row, m);
    }
    __syncthreads();
  }
}

// bin of x: the estimate from the value, corrected against the fp32 edges (e[k] <= x < e[k+1], last bin closed)
__device__ inline int kld_bin(float x, float lo, float scale, const float* __restrict__ e, int nb) {
  int k = static_cast<int>(floorf(__fmul_rn(__fsub_rn(x, lo), scale)));
  k = k < 0 ? 0 : (k > nb - 1 ? nb - 1 : k);
  while (k > 0 && x < e[k]) --k;
  while (k < nb - 1 && x >= e[k + 1]) ++k;
  return k;
}

// Shared-memory layout: `replicas` histograms of nb counters (warp w counts into replica w % replicas), then nb + 1 edges.
// Runs of one bin (zeros after a ReLU, a constant row) are counted in a register and added once.
template <int VEC>
__global__ void __launch_bounds__(kKldThreads) fq_kld_hist_kernel(const __grid_constant__ KldArgs A) {
  using V = typename VecT<VEC>::type;
  extern __shared__ unsigned kld_smem[];
  const int nb = A.nb;
  unsigned* sh = kld_smem;
  float* e = reinterpret_cast<float*>(kld_smem + A.replicas * nb);
  unsigned* mine = sh + ((threadIdx.x >> 5) % A.replicas) * nb;
  const unsigned long long units = A.rows * A.chunks;
  for (unsigned long long u = blockIdx.x; u < units; u += gridDim.x) {
    unsigned long long row, v0, v1;
    kld_unit<VEC>(A, u, &row, &v0, &v1);
    double lo, hi;
    if (!kld_range(A, row, &lo, &hi)) continue;   // uniform over the CTA
    for (int k = threadIdx.x; k < A.replicas * nb; k += kKldThreads) sh[k] = 0;
    for (int k = threadIdx.x; k <= nb; k += kKldThreads) e[k] = kld_edge(lo, hi, nb, k);
    __syncthreads();
    const float lof = static_cast<float>(lo);
    const float scale = static_cast<float>(static_cast<double>(nb) / (hi - lo));
    const V* p = reinterpret_cast<const V*>(A.in + row * A.row_len);
    int run_bin = -1;
    unsigned run = 0;
    auto add = [&](float x) {
      const int k = kld_bin(x, lof, scale, e, nb);
      if (k == run_bin) {
        ++run;
      } else {
        if (run) atomicAdd(mine + run_bin, run);
        run_bin = k;
        run = 1;
      }
    };
    for (unsigned long long v = v0 + threadIdx.x; v < v1; v += kKldThreads) {
      const V x = __ldg(p + v);
      if constexpr (VEC == 4) {
        add(x.x);
        add(x.y);
        add(x.z);
        add(x.w);
      } else {
        add(x);
      }
    }
    if (run) atomicAdd(mine + run_bin, run);
    __syncthreads();
    unsigned* g = A.hist + row * static_cast<unsigned long long>(nb);
    for (int k = threadIdx.x; k < nb; k += kKldThreads) {
      unsigned s = 0;
      for (int r = 0; r < A.replicas; ++r) s += sh[r * nb + k];
      if (s) atomicAdd(g + k, s);   // result unused: compiled to red.global.add
    }
    __syncthreads();
  }
}

// inclusive block scan of two counters per element, in place: a[1..n], b[1..n] (a[0] = b[0] = 0)
__device__ inline void kld_scan2(unsigned* a, unsigned* b, int n) {
  __shared__ unsigned wa[kKldThreads / 32], wb[kKldThreads / 32];
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  const int seg = (n + kKldThreads - 1) / kKldThreads;
  const int k0 = 1 + t * seg, k1 = min(n + 1, k0 + seg);
  unsigned sa = 0, sb = 0;
  for (int k = k0; k < k1; ++k) sa += a[k], sb += b[k];
  unsigned ia = sa, ib = sb;   // inclusive warp scan of the per-thread sums
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned xa = __shfl_up_sync(0xffffffffu, ia, o), xb = __shfl_up_sync(0xffffffffu, ib, o);
    if (lane >= o) ia += xa, ib += xb;
  }
  if (lane == 31) wa[w] = ia, wb[w] = ib;
  __syncthreads();
  unsigned pa = ia - sa, pb = ib - sb;
  for (int i = 0; i < w; ++i) pa += wa[i], pb += wb[i];
  for (int k = k0; k < k1; ++k) {
    pa += a[k];
    pb += b[k];
    a[k] = pa;
    b[k] = pb;
  }
  __syncthreads();
}

// first NaN, else first minimum (np.argmin)
__device__ inline void kld_better(double& v, int& i, double v2, int i2) {
  const bool n1 = v != v, n2 = v2 != v2;
  bool take;
  if (n1 != n2) take = n2;
  else if (n1) take = i2 < i;
  else take = v2 < v || (v2 == v && i2 < i);
  if (take) v = v2, i = i2;
}

// Shared memory: cnt[nb + 1] and nz[nb + 1] (prefix sums of the counts and of the non-zero flags), then the divergence of
// every candidate (double).  Candidate c is i = c + nq/2: the 2i + 1 bins around the zero bin z = nb/2.
__global__ void __launch_bounds__(kKldThreads) fq_kld_search_kernel(const __grid_constant__ KldArgs A) {
  extern __shared__ unsigned kld_smem[];
  const int nb = A.nb, nq = A.nq, z = nb / 2, half_q = nq / 2;
  const int ncand = nb / 2 + 1 - half_q;
  unsigned* cnt = kld_smem;
  unsigned* nz = cnt + nb + 1;
  double* div = reinterpret_cast<double*>(kld_smem + ((2 * (nb + 1) + 1) & ~1));
  const unsigned long long row = blockIdx.x;
  double lo, hi;
  if (!kld_range(A, row, &lo, &hi)) {
    if (threadIdx.x == 0) A.out_th[row] = A.out_div[row] = __int_as_float(0x7fc00000), A.out_idx[row] = -1;
    return;
  }
  const unsigned* g = A.hist + row * static_cast<unsigned long long>(nb);
  for (int k = threadIdx.x; k < nb; k += kKldThreads) {
    const unsigned h = g[k];
    cnt[k + 1] = h;
    nz[k + 1] = h != 0;
  }
  if (threadIdx.x == 0) cnt[0] = nz[0] = 0;
  __syncthreads();
  kld_scan2(cnt, nz, nb);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const double eps = 0.0001, log_eps = log(eps);
  const unsigned total = cnt[nb];
  const double sp = static_cast<double>(total);
  for (int c = warp; c < ncand; c += kKldThreads / 32) {
    const int i = c + half_q, n = 2 * i + 1, s = z - i, m = n / nq;
    const unsigned left = cnt[s], right = total - cnt[s + n];
    const unsigned h0 = cnt[s + 1] - cnt[s], hl = cnt[s + n] - cnt[s + n - 1];
    // p = sliced histogram with the outliers added to its ends; q = the merged bins expanded over the non-zero bins of
    // their slice (the last slice stops at n - 1: q[n-1] stays 0), so q > 0 exactly on the non-zero bins 0 .. n-2
    const int nnz_p = static_cast<int>(nz[s + n] - nz[s]) - (h0 != 0) - (hl != 0) + (h0 + left != 0) + (hl + right != 0);
    const int nnz_q = static_cast<int>(nz[s + n - 1] - nz[s]);
    const double eps1_p = eps * static_cast<double>(n - nnz_p) / static_cast<double>(nnz_p);
    const double eps1_q = nnz_q ? eps * static_cast<double>(n - nnz_q) / static_cast<double>(nnz_q) : 0.0;
    auto bin_q = [&](int j, unsigned* norm_out) {   // q value of merged bin j (float32, as the reference's q array)
      const int b0 = j * m;
      const int b1 = j == nq - 1 ? n : b0 + m;
      const int stop = j == nq - 1 ? n - 1 : b0 + m;
      const unsigned norm = stop > b0 ? nz[s + stop] - nz[s + b0] : 0u;
      *norm_out = norm;
      return norm ? static_cast<double>(static_cast<float>(static_cast<double>(cnt[s + b1] - cnt[s + b0]) / static_cast<double>(norm)))
                  : 0.0;
    };
    double sq = 0.0;
    for (int j = lane; j < nq; j += 32) {
      unsigned norm;
      const double q = bin_q(j, &norm);
      sq += q * static_cast<double>(norm);
    }
    double acc = 0.0;
    int cj = -1;
    double lqj = 0.0;
    for (int k = lane; k < n; k += 32) {
      const unsigned hk = cnt[s + k + 1] - cnt[s + k];
      const unsigned pk = hk + (k == 0 ? left : 0u) + (k == n - 1 ? right : 0u);
      const bool qnz = hk != 0 && k != n - 1;
      if (pk == 0 && !qnz) continue;   // eps * log(eps / eps) = 0
      const double ps = pk ? static_cast<double>(pk) - eps1_p : eps;
      double lq = log_eps;
      if (qnz) {
        const int j = min(k / m, nq - 1);
        if (j != cj) {
          unsigned norm;
          lqj = log(bin_q(j, &norm) - eps1_q);
          cj = j;
        }
        lq = lqj;
      }
      acc += ps * (log(ps) - lq);
    }
    for (int o = 16; o; o >>= 1) {
      acc += __shfl_xor_sync(0xffffffffu, acc, o);
      sq += __shfl_xor_sync(0xffffffffu, sq, o);
    }
    if (lane == 0) {
      // smoothing conserves mass: sum(p_s) = sp, sum(q_s) = sq; KL(p_s/sp || q_s/sq) = acc/sp + log(sq/sp).
      // All-zero q: the reference's entropy(p, q) divides 0 by 0 -> NaN.
      div[c] = nnz_q ? acc / sp + log(sq / sp) : __longlong_as_double(0x7ff8000000000000ll);
    }
  }
  __syncthreads();
  double bv = __longlong_as_double(0x7ff0000000000000ll);
  int bi = 0x7fffffff;
  for (int c = threadIdx.x; c < ncand; c += kKldThreads) kld_better(bv, bi, div[c], c);
  for (int o = 16; o; o >>= 1) {
    const double v2 = __shfl_xor_sync(0xffffffffu, bv, o);
    const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
    kld_better(bv, bi, v2, i2);
  }
  __shared__ double wv[kKldThreads / 32];
  __shared__ int wi[kKldThreads / 32];
  if (lane == 0) wv[warp] = bv, wi[warp] = bi;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kKldThreads / 32; ++w) kld_better(bv, bi, wv[w], wi[w]);
    A.out_idx[row] = bi;
    A.out_div[row] = static_cast<float>(bv);
    A.out_th[row] = kld_edge(lo, hi, nb, z + 1 + half_q + bi);
  }
}

}  // namespace fqb
