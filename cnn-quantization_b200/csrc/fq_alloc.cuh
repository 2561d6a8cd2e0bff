// Exact per-channel bit allocation on the device (fqb200_allocate_widths): the dynamic programme of bit_alloc.allocate,
//
//   minimise  sum_g sse[g][w_g]   subject to   sum_g w_g <= budget,   w_g in 0..8
//
// run from the last channel to the first with the same float64 sums in the same order.  One CTA: best[b] is the least
// error of the channels after the current one with at most b bits; for every b one thread tries w = 0, 1, .. in
// increasing order and keeps a candidate only when it is strictly smaller (a tie keeps the smaller width), writing the
// winner into a uint8 choice table [G][budget + 1].  The two best[] rows live in shared memory when they fit, else in the
// workspace (L2).  Thread 0 then walks the choice table from channel 0 with the whole budget: among minimisers this is the
// lexicographically smallest width vector, the host function's tie rule.  NaN never wins a comparison (a channel whose
// candidates are all NaN keeps width 0); any non-finite entry sets *status to 1.
namespace fqb {

constexpr int kAllocThreads = 1024;
constexpr int64_t kAllocMaxGroups = 1 << 20;
constexpr size_t kAllocMaxSmem = 227u * 1024u;  // the two best[] rows in shared memory up to this size (H100: 227 KB per CTA)

__global__ void __launch_bounds__(kAllocThreads, 1)
    fq_allocate_widths_kernel(const double* __restrict__ sse, unsigned groups, unsigned budget, unsigned char* __restrict__ choice,
                              double* rows, float* __restrict__ widths, int* __restrict__ status) {
  extern __shared__ __align__(16) double fq_alloc_rows[];
  const unsigned n = budget + 1u;
  double* best = rows ? rows : fq_alloc_rows;
  double* next = best + n;
  bool bad = false;
  for (unsigned i = threadIdx.x; i < groups * 9u; i += blockDim.x) bad |= !isfinite(sse[i]);
  if (__syncthreads_or(bad) && threadIdx.x == 0 && status) *status = 1;
  for (unsigned b = threadIdx.x; b < n; b += blockDim.x) best[b] = 0.0;
  __syncthreads();
  const unsigned wmax = budget < 8u ? budget : 8u;
  for (unsigned c = groups; c-- > 0;) {
    double e[9];
#pragma unroll
    for (int w = 0; w < 9; ++w) e[w] = __ldg(sse + static_cast<size_t>(c) * 9u + w);
    unsigned char* pick = choice + static_cast<size_t>(c) * n;
    for (unsigned b = threadIdx.x; b < n; b += blockDim.x) {
      double cur = INFINITY;
      unsigned char p = 0;
#pragma unroll
      for (unsigned w = 0; w < 9u; ++w) {
        if (w > wmax || w > b) break;
        const double cand = __dadd_rn(e[w], best[b - w]);
        if (cand < cur) {
          cur = cand;
          p = static_cast<unsigned char>(w);
        }
      }
      next[b] = cur;
      pick[b] = p;
    }
    __syncthreads();
    double* t = best;
    best = next;
    next = t;
  }
  if (threadIdx.x == 0) {
    unsigned b = budget;
    for (unsigned c = 0; c < groups; ++c) {
      const unsigned w = choice[static_cast<size_t>(c) * n + b];
      widths[c] = static_cast<float>(w);
      b -= w;
    }
  }
}

}  // namespace fqb
