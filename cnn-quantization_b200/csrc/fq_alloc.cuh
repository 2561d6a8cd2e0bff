// Exact per-channel bit allocation on the device (fqb200_allocate_widths, fqb200_allocate_select): the dynamic programme
// of bit_alloc.allocate,
//
//   minimise  sum_g sse[g][w_g]   subject to   sum_g w_g <= B = min(floor(target * G), 8 G),   w_g in 0..8
//
// run from the last channel to the first with the same float64 sums in the same order.  One CTA: best[b] is the least
// error of the channels after the current one with at most b bits; for every b one thread tries w = 0, 1, .. in
// increasing order and keeps a candidate only when it is strictly smaller (a tie keeps the smaller width), writing the
// winner into a uint8 choice table [G][B + 1].  The two best[] rows live in shared memory when they fit, else in the
// workspace (L2).  Thread 0 then walks the choice table from channel 0 with the whole budget: among minimisers this is the
// lexicographically smallest width vector, the host function's tie rule.  NaN never wins a comparison (a channel whose
// candidates are all NaN keeps width 0); any non-finite entry sets *status to 1.
//
// Banding (exact): channel c is computed only for b in [max(0, B - 8c), min(B, 8(G - c))].  The walk from channel 0 never
// holds fewer than B - 8c bits at channel c, and over the k = G - c channels c..G-1 every b >= 8k has the candidates of
// b = 8k (each reads the same entry, clamped), so its best value and pick are those of 8k, bit for bit; reads above the
// previous band's top are clamped to it, and the walk reads choice[c][min(b, 8(G - c))].  At target 4 that is about 2 G^2
// states instead of 4 G^2.
//
// Register window: a thread takes kAllocRun adjacent states, so their 9 reads each come from kAllocRun + 8 loads of
// best[]; kAllocRun is odd, so the lanes' float64 loads (stride kAllocRun) fall in distinct shared-memory banks.  The next
// channel's nine errors are loaded while the current one is computed.
//
// fqb200_allocate_select runs the same programme over a table it first builds in the workspace: per (channel, width) the
// least of the M multiplier columns of a clip_mse_widths / clip_mse_grid launch (cm_before, statistics.best_columns'
// order), and ends with the chosen candidate's parameters.
namespace fqb {

constexpr int kAllocThreads = 512;
constexpr int kAllocRun = 9;   // adjacent states per thread (odd: conflict-free float64 loads)
constexpr int64_t kAllocMaxGroups = 1 << 20;
constexpr size_t kAllocMaxSmem = 227u * 1024u;  // the two best[] rows in shared memory up to this size (H100: 227 KB per CTA)

// the programme over sse[g * 9 + w]; thread 0 writes widths[] (visible to the CTA after the caller's __syncthreads)
__device__ __forceinline__ void alloc_dp(const double* sse, unsigned groups, unsigned budget, unsigned char* choice,
                                         double* rows, float* widths, int* status) {
  extern __shared__ __align__(16) double fq_alloc_rows[];
  const unsigned n = budget + 1u;
  double* best = rows ? rows : fq_alloc_rows;
  double* next = best + n;
  bool bad = false;
  for (unsigned i = threadIdx.x; i < groups * 9u; i += blockDim.x) bad |= !isfinite(sse[i]);
  if (__syncthreads_or(bad) && threadIdx.x == 0 && status) *status = 1;
  if (threadIdx.x == 0) best[0] = 0.0;   // no channel after the last: best[] is 0, its band is {0}
  __syncthreads();
  const unsigned wmax = budget < 8u ? budget : 8u;
  double en[9];
#pragma unroll
  for (int w = 0; w < 9; ++w) en[w] = sse[static_cast<size_t>(groups - 1u) * 9u + w];
  for (unsigned c = groups; c-- > 0;) {
    double e[9];
#pragma unroll
    for (int w = 0; w < 9; ++w) e[w] = en[w];
    if (c > 0) {
#pragma unroll
      for (int w = 0; w < 9; ++w) en[w] = sse[static_cast<size_t>(c - 1u) * 9u + w];
    }
    const unsigned k = groups - c;
    const unsigned lo = budget > 8u * c ? budget - 8u * c : 0u;
    const unsigned hi = budget < 8u * k ? budget : 8u * k;
    const unsigned top = budget < 8u * (k - 1u) ? budget : 8u * (k - 1u);   // best[] is defined up to here
    unsigned char* pick = choice + static_cast<size_t>(c) * n;
    for (unsigned b0 = lo + threadIdx.x * kAllocRun; b0 <= hi; b0 += blockDim.x * kAllocRun) {
      double win[kAllocRun + 8];   // win[i] = best[b0 - 8 + i] (clamped to top; entries below 0 are never read)
#pragma unroll
      for (int i = 0; i < kAllocRun + 8; ++i) {
        const int j = static_cast<int>(b0) - 8 + i;
        win[i] = j >= 0 ? best[static_cast<unsigned>(j) < top ? static_cast<unsigned>(j) : top] : 0.0;
      }
#pragma unroll
      for (int r = 0; r < kAllocRun; ++r) {
        const unsigned b = b0 + r;
        double cur = INFINITY;
        unsigned char p = 0;
#pragma unroll
        for (unsigned w = 0; w < 9u; ++w) {
          if (w > wmax || w > b) break;
          const double cand = __dadd_rn(e[w], win[r + 8 - w]);
          if (cand < cur) {
            cur = cand;
            p = static_cast<unsigned char>(w);
          }
        }
        if (b <= hi) {
          next[b] = cur;
          pick[b] = p;
        }
      }
    }
    __syncthreads();
    double* t = best;
    best = next;
    next = t;
  }
  if (threadIdx.x == 0) {
    unsigned b = budget;
    for (unsigned c = 0; c < groups; ++c) {
      const unsigned cap = 8u * (groups - c);
      const unsigned w = choice[static_cast<size_t>(c) * n + (b < cap ? b : cap)];
      widths[c] = static_cast<float>(w);
      b -= w;
    }
  }
}

__global__ void __launch_bounds__(kAllocThreads, 1)
    fq_allocate_widths_kernel(const double* __restrict__ sse, unsigned groups, unsigned budget, unsigned char* __restrict__ choice,
                              double* rows, float* __restrict__ widths, int* __restrict__ status) {
  alloc_dp(sse, groups, budget, choice, rows, widths, status);
}

struct AllocSelectArgs {
  const double* sums;        // [groups][1 + 9 M]: sum x^2, then width w, multiplier k at column 1 + w * M + k
  const float* params;       // [groups][9 M][kCeParams]
  const float* mult;         // [M] (read when M > 1)
  const float* stats;        // [groups][FQB200_STATS_STRIDE]
  unsigned groups, budget;
  int M;
  double* least;             // workspace [groups][9]: the sum at each width's chosen column
  unsigned char* column;     // workspace [groups][9]: that column (M > 1)
  unsigned char* choice;     // workspace: the programme's choice table
  double* rows;              // workspace rows, or nullptr: shared memory
  float* widths;             // [groups]
  int* chosen;               // optional [groups]: the chosen width's column (M > 1)
  float* given;              // [3][groups]: delta, offset, bits
  float* table;              // optional [groups][FQB200_STATS_STRIDE]
  int* status;
};

__global__ void __launch_bounds__(kAllocThreads, 1) fq_allocate_select_kernel(const __grid_constant__ AllocSelectArgs A) {
  const unsigned row = 1u + 9u * static_cast<unsigned>(A.M);
  for (unsigned i = threadIdx.x; i < A.groups * 9u; i += blockDim.x) {
    const unsigned g = i / 9u, w = i - 9u * g;
    const double* e = A.sums + static_cast<size_t>(g) * row + 1u + w * static_cast<unsigned>(A.M);
    CmPick p{0.0, 0.f, -1};
    for (int k = 0; k < A.M; ++k) {
      const double ek = e[k];
      const CmPick c{isnan(ek) ? static_cast<double>(INFINITY) : ek, A.M > 1 ? __ldg(A.mult + k) : 0.f, k};
      if (cm_before(c, p)) p = c;
    }
    A.least[i] = e[p.k];   // NaN stays NaN: the programme's status flag sees it
    A.column[i] = static_cast<unsigned char>(p.k);
  }
  __syncthreads();
  alloc_dp(A.least, A.groups, A.budget, A.choice, A.rows, A.widths, A.status);
  __syncthreads();   // thread 0's widths are visible to the CTA
  for (unsigned g = threadIdx.x; g < A.groups; g += blockDim.x) {
    const unsigned w = static_cast<unsigned>(A.widths[g]);
    const unsigned k = A.column[g * 9u + w];
    const float* src = A.params + (static_cast<size_t>(g) * (row - 1u) + w * static_cast<unsigned>(A.M) + k) * kCeParams;
    const float d = src[0], o = src[1], b = src[2];
    if (A.chosen) A.chosen[g] = static_cast<int>(k);
    A.given[g] = d;
    A.given[A.groups + g] = o;
    A.given[2u * A.groups + g] = b;
    if (A.table) {
      const LeafParam q = make_leaf_param(FQB200_LEAF_TORCH, d, o, b);
      const float* t = A.stats + static_cast<size_t>(g) * FQB200_STATS_STRIDE;
      float* dst = A.table + static_cast<size_t>(g) * FQB200_STATS_STRIDE;
      for (int c = 0; c < 5; ++c) dst[c] = t[c];
      dst[5] = d; dst[6] = o; dst[7] = b; dst[8] = q.a; dst[9] = q.b; dst[10] = q.c; dst[11] = static_cast<float>(q.flags);
    }
  }
}

}  // namespace fqb
