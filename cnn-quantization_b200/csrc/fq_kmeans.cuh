// 1-D k-means weight quantization (pytorch_quantizer/quantization/kmeans_quantization.py:14-30): scikit-learn 1.9's
// KMeans(n_clusters=k, random_state=seed) on the n values of one tensor - one k-means++ init (n_init='auto'), Lloyd with
// max_iter=300 and tol=1e-4 - in ONE cooperative launch of fq_kmeans_kernel.  Included by fqb200.cu after fq_device.cuh.
//
// Everything runs in float64 on the centred values xc = x - mean (scikit-learn's `fit` centres the data first).  Every sum
// is taken in one fixed order, so the result has the same bits on every run and for every grid size, and
// tests/golden/kmeans_oracle.py restates each of them with numpy:
//
//   block       kKmBlk = 512 consecutive elements, one warp: lane l adds elements l, l + 32, ... (16 rows) in order, then
//               an xor butterfly over the lanes (offsets 16, 8, 4, 2, 1)
//   superblock  32 consecutive blocks: the same butterfly over their block sums
//   total       the superblock sums added one after the other
//
// k-means++ (sklearn _kmeans_plusplus): the random draws are the host's (they do not depend on the data); step c
// evaluates the candidates t, each a column of per-block sums of min(d_i, (xc_i - xc_cand)^2), where d_i is the distance
// to the nearest centre chosen so far (binary search over the sorted centres in shared memory: nothing is stored per
// element).  The leader CTA of the step's grid barrier totals the columns, keeps the first minimum, and draws the next
// step's candidates: v = u * pot, then searchsorted(cumsum, v, side='left') with the cumsum of the hierarchy above - the
// first superblock whose running total reaches v, the first of its blocks whose running total (from the superblock's
// start) reaches v, and the first element of that block whose running total (from the block's start) does; the last
// block / element when rounding leaves none, n - 1 when no superblock does.
//
// Lloyd (sklearn _kmeans_single_lloyd): per iteration one pass - nearest centre by binary search, ties to the lowest
// index; per-cluster float64 sums and counts of fixed work units (kWarps * mult blocks) in per-warp shared accumulators,
// lanes of one cluster combined with __match_any_sync in lane order, warps folded in order - and one grid barrier whose
// leader folds the unit partials in a fixed order, relocates empty clusters (_relocate_empty_clusters_dense: the
// farthest points, one grid-wide argmax pass per empty cluster; farthest first, ties to the lowest index), averages
// (_average_centers, including its placement of clusters left empty) and tests convergence: labels unchanged (strict),
// or the sum over clusters of (c_new - c_old)^2 <= tol = var(x) * 1e-4.  Without strict convergence a last pass
// reassigns the labels.  The last pass also sums the inertia and writes the task's tensor; an optional row pass adds the
// per-output-channel bias correction (kmeans_quantization.py:78-88) with float64 row means.
//
// No atomics touch a value (the only atomics are the grid barrier's and one integer "labels changed" flag).
namespace fqb {

constexpr int kKmBlk = 512;                 // elements per block (16 rows of 32 lanes)
constexpr int kKmRows = kKmBlk / 32;
constexpr int kKmSuper = 32;                // blocks per superblock
constexpr int kKmMaxK = 256;
constexpr int kKmMaxT = 8;                  // k-means++ local trials: 2 + int(log k) <= 7
constexpr int kKmMaxIter = 300;
constexpr unsigned long long kKmMaxUnits = 16384;

struct KmCtrl {
  double mean, tol, inertia, pad0;
  double cent[kKmMaxK];        // centred centres by index (k-means++: the ones chosen so far)
  double cval[kKmMaxT];        // k-means++: the centred values of this step's candidates
  double pot[kKmMaxT];
  long long cand[kKmMaxT];
  double tsum[kKmMaxK];        // Lloyd: per-cluster sums and counts of the iteration, for a relocating leader
  unsigned long long tcnt[kKmMaxK];
  double reloc_d;              // relocation: the last point picked (distance, index)
  long long reloc_i;
  int n_chosen, n_cand, changed, stop, strict, n_iter, reloc, n_empty;
};

struct KmArgs {
  const float* in;
  unsigned long long n, nb, nsb;   // elements, blocks, superblocks
  int k, T, task, given;
  long long first_id;
  const double* draws;             // [k - 1][T] uniforms
  const double* init;              // optional [k] initial centres (not centred)
  unsigned long long unit_blocks, units;
  unsigned long long rows;
  GridSync* sync;
  KmCtrl* ctrl;
  double* col;                     // [kKmMaxT][nb] per-block sums
  double* sup;                     // [kKmMaxT][nsb] per-superblock sums
  double* usum;                    // [units][k]
  unsigned* ucnt;                  // [units][k]
  double* rbd;                     // [nb] relocation: per-block farthest distance ...
  long long* rbi;                  // ... and its index
  long long* far;                  // [k]
  unsigned char* labels;
  float* centres;
  double* inertia;
  int* n_iter;
  long long* init_ids;
  float* out;
  float* out_bcorr;
};

__device__ __forceinline__ double km_d2(double a, double b) {
  const double t = __dsub_rn(a, b);
  return __dmul_rn(t, t);
}

__device__ __forceinline__ double km_xc(const KmArgs& A, unsigned long long i, double mean) {
  return __dsub_rn(static_cast<double>(__ldg(A.in + i)), mean);
}

// first position of the sorted centres holding a value > x
__device__ __forceinline__ int km_upper(const double* sc, int m, double x) {
  int lo = 0, hi = m;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (sc[mid] > x) hi = mid;
    else lo = mid + 1;
  }
  return lo;
}

// squared distance to the nearest of the m sorted centres (+inf when m == 0): rounding is monotone, so it is one of the
// two neighbours of x in sorted order
__device__ __forceinline__ double km_nearest_d(const double* sc, int m, double x) {
  const int p = km_upper(sc, m, x);
  double d = __longlong_as_double(0x7ff0000000000000ll);
  if (p > 0) d = km_d2(x, sc[p - 1]);
  if (p < m) d = fmin(d, km_d2(x, sc[p]));
  return d;
}

// np.argmin over j of (x - c_j)^2: the lowest index among the centres at the minimal distance, which are contiguous in
// sorted order around the neighbours of x
__device__ __forceinline__ int km_label(const double* sc, const int* si, int m, double x, double& dmin) {
  const int p = km_upper(sc, m, x);
  double d = __longlong_as_double(0x7ff0000000000000ll);
  if (p > 0) d = km_d2(x, sc[p - 1]);
  if (p < m) d = fmin(d, km_d2(x, sc[p]));
  int lab = 1 << 30;
  for (int j = p - 1; j >= 0 && km_d2(x, sc[j]) == d; --j) lab = min(lab, si[j]);
  for (int j = p; j < m && km_d2(x, sc[j]) == d; ++j) lab = min(lab, si[j]);
  dmin = d;
  return lab;
}

// relocation order: farther first, then the lower index (i < 0: nothing)
__device__ __forceinline__ bool km_better(double d, long long i, double bd, long long bi) {
  return i >= 0 && (bi < 0 || d > bd || (d == bd && i < bi));
}

// leader CTA, after the per-cluster totals are in tsum / tcnt (shared): relocation of empty clusters, averaging (with
// _average_centers' placement of clusters still empty), shift, convergence; publishes the new centres
__device__ void km_finish(const KmArgs& A, KmCtrl* C, double* tsum, unsigned long long* tcnt, const double* cv, int k,
                          double mean) {
  if (threadIdx.x == 0) {
    if (__ldcg(&C->reloc)) {
      // the empty clusters as they were before any relocation (a far point's own cluster may empty on the way; it is
      // left to the averaging below, as in _relocate_empty_clusters_dense): far[0 .. n_empty) pair with them in order
      unsigned empty[kKmMaxK / 32];
      for (int w = 0; w < kKmMaxK / 32; ++w) empty[w] = 0u;
      for (int j = 0; j < k; ++j) if (tcnt[j] == 0) empty[j >> 5] |= 1u << (j & 31);
      const int n_empty = __ldcg(&C->n_empty);
      int r = 0;
      for (int j = 0; j < k && r < n_empty; ++j) {
        if (!(empty[j >> 5] >> (j & 31) & 1u)) continue;
        const long long f = __ldcg(A.far + r++);
        const int old = __ldcg(A.labels + f);
        const double xf = __dsub_rn(static_cast<double>(A.in[f]), mean);
        tsum[old] = __dsub_rn(tsum[old], xf);
        tsum[j] = xf;
        tcnt[j] = 1;
        tcnt[old] -= 1;
      }
    }
    int amax = 0;
    for (int j = 1; j < k; ++j) if (tcnt[j] > tcnt[amax]) amax = j;
    for (int j = 0; j < k; ++j) {
      if (tcnt[j] > 0) tsum[j] = __dmul_rn(tsum[j], 1.0 / static_cast<double>(tcnt[j]));
      else tsum[j] = tsum[amax];
    }
    double shift = 0.0;
    for (int j = 0; j < k; ++j) shift = __dadd_rn(shift, km_d2(tsum[j], cv[j]));
    C->stop = C->strict || shift <= C->tol;
  }
  __syncthreads();
  if (threadIdx.x < static_cast<unsigned>(k)) C->cent[threadIdx.x] = tsum[threadIdx.x];
}

__device__ __forceinline__ double km_butterfly(double v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// sorted copy (value, then index) of cent[0..m) in shared memory: rank sort, one thread per centre
__device__ __forceinline__ void km_sort(const KmCtrl* C, int m, double* cv, double* sc, int* si) {
  if (threadIdx.x < static_cast<unsigned>(m)) cv[threadIdx.x] = __ldcg(C->cent + threadIdx.x);
  __syncthreads();
  if (threadIdx.x < static_cast<unsigned>(m)) {
    const int j = threadIdx.x;
    const double v = cv[j];
    int r = 0;
    for (int i = 0; i < m; ++i) r += (cv[i] < v) || (cv[i] == v && i < j);
    sc[r] = v;
    si[r] = j;
  }
  __syncthreads();
}

// column c of the per-block sums -> superblock sums (one warp), and their sequential total
__device__ double km_total(const KmArgs& A, int c) {
  const unsigned lane = threadIdx.x & 31;
  const double* col = A.col + static_cast<unsigned long long>(c) * A.nb;
  double* sup = A.sup + static_cast<unsigned long long>(c) * A.nsb;
  double tot = 0.0;
  for (unsigned long long g0 = 0; g0 < A.nsb; g0 += 32) {
    double mine = 0.0;
    for (int u = 0; u < 32 && g0 + u < A.nsb; ++u) {
      const unsigned long long b = (g0 + u) * kKmSuper + lane;
      const double s = km_butterfly(b < A.nb ? __ldcg(col + b) : 0.0);
      if (lane == static_cast<unsigned>(u)) mine = s;
    }
    if (g0 + lane < A.nsb) sup[g0 + lane] = mine;
    for (int u = 0; u < 32 && g0 + u < A.nsb; ++u) tot = __dadd_rn(tot, __shfl_sync(0xffffffffu, mine, u));
  }
  return tot;
}

// searchsorted(cumsum, v, 'left') over column c, clipped to n - 1 (one warp; `stage` holds kKmBlk doubles).  The element
// values of the chosen block are recomputed: min(nearest distance over the m sorted centres, distance to xcand).
__device__ long long km_search(const KmArgs& A, int c, double v, const double* sc, int m, double xcand, double mean,
                               double* stage) {
  const unsigned lane = threadIdx.x & 31;
  const double* col = A.col + static_cast<unsigned long long>(c) * A.nb;
  const double* sup = A.sup + static_cast<unsigned long long>(c) * A.nsb;
  double q = 0.0;
  long long gsel = -1;
  for (unsigned long long g0 = 0; g0 < A.nsb && gsel < 0; g0 += 32) {
    const double s = g0 + lane < A.nsb ? __ldcg(sup + g0 + lane) : 0.0;
    for (int u = 0; u < 32 && g0 + u < A.nsb; ++u) {
      const double qn = __dadd_rn(q, __shfl_sync(0xffffffffu, s, u));
      if (qn >= v) { gsel = static_cast<long long>(g0 + u); break; }
      q = qn;
    }
  }
  if (gsel < 0) return static_cast<long long>(A.n - 1);
  const unsigned long long b0 = static_cast<unsigned long long>(gsel) * kKmSuper;
  const unsigned long long b1 = b0 + kKmSuper < A.nb ? b0 + kKmSuper : A.nb;
  const double sb = b0 + lane < b1 ? __ldcg(col + b0 + lane) : 0.0;
  unsigned long long bsel = b1 - 1;
  double r = q;
  for (unsigned long long b = b0; b < b1; ++b) {
    const double rn = __dadd_rn(r, __shfl_sync(0xffffffffu, sb, static_cast<int>(b - b0)));
    if (rn >= v || b + 1 == b1) { bsel = b; break; }
    r = rn;
  }
  const unsigned long long e0 = bsel * kKmBlk, e1 = e0 + kKmBlk < A.n ? e0 + kKmBlk : A.n;
  for (unsigned long long i = e0 + lane; i < e1; i += 32) {
    const double x = km_xc(A, i, mean);
    stage[i - e0] = fmin(km_nearest_d(sc, m, x), km_d2(x, xcand));
  }
  __syncwarp();
  long long sel = static_cast<long long>(e1 - 1);
  if (lane == 0) {
    double cs = r;
    for (unsigned long long i = e0; i < e1; ++i) {
      cs = __dadd_rn(cs, stage[i - e0]);
      if (cs >= v) { sel = static_cast<long long>(i); break; }
    }
  }
  __syncwarp();
  return __shfl_sync(0xffffffffu, sel, 0);
}

// one warp, block b: lane-sequential sums of f(i, xc) over the rows, butterfly; every lane gets the block sum(s)
template <int NT, class F>
__device__ __forceinline__ void km_block_sums(const KmArgs& A, unsigned long long b, double mean, F f, double (&s)[NT]) {
  const unsigned lane = threadIdx.x & 31;
#pragma unroll
  for (int t = 0; t < NT; ++t) s[t] = 0.0;
  const unsigned long long e0 = b * kKmBlk + lane;
#pragma unroll 4
  for (int r = 0; r < kKmRows; ++r) {
    const unsigned long long i = e0 + static_cast<unsigned long long>(r) * 32;
    if (i < A.n) f(i, km_xc(A, i, mean), s);
  }
#pragma unroll
  for (int t = 0; t < NT; ++t) s[t] = km_butterfly(s[t]);
}

__global__ void __launch_bounds__(kThreads, kCtasPerSm) fq_kmeans_kernel(const __grid_constant__ KmArgs A) {
  extern __shared__ __align__(16) unsigned char km_smem[];
  __shared__ double cv[kKmMaxK], sc[kKmMaxK], pot_s[kKmMaxT];
  __shared__ int si[kKmMaxK];
  __shared__ int flag_s;
  __shared__ double red_d[kWarps];
  __shared__ long long red_i[kWarps];
  KmCtrl* C = A.ctrl;
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned long long gwarp = static_cast<unsigned long long>(blockIdx.x) * kWarps + warp;
  const unsigned long long nwarps = static_cast<unsigned long long>(gridDim.x) * kWarps;
  const int k = A.k;
  unsigned epoch = 0;
  const double inf = __longlong_as_double(0x7ff0000000000000ll);

  // ---- mean and variance ----------------------------------------------------------------------------------------------
  for (int pass = 0; pass < 2; ++pass) {
    const double mean = pass ? __ldcg(&C->mean) : 0.0;
    for (unsigned long long b = gwarp; b < A.nb; b += nwarps) {
      double s[1];
      km_block_sums<1>(A, b, mean, [&](unsigned long long, double x, double (&a)[1]) {
        a[0] = __dadd_rn(a[0], pass ? __dmul_rn(x, x) : x);
      }, s);
      if (lane == 0) A.col[b] = s[0];
    }
    if (grid_arrive(A.sync, epoch, &flag_s)) {
      if (warp == 0) {
        const double tot = km_total(A, 0);
        if (lane == 0) {
          if (pass == 0) {
            C->mean = tot / static_cast<double>(A.n);
          } else {
            C->tol = tot / static_cast<double>(A.n) * 1e-4;
            if (A.given)
              for (int j = 0; j < k; ++j) C->cent[j] = __dsub_rn(A.init[j], C->mean);
            C->n_chosen = 0;
            C->n_cand = 1;
            C->cand[0] = A.first_id;
            C->cval[0] = __dsub_rn(static_cast<double>(A.in[A.first_id]), C->mean);
          }
        }
      }
      grid_release(A.sync, epoch);
    }
  }
  const double mean = __ldcg(&C->mean);

  // ---- k-means++ ------------------------------------------------------------------------------------------------------
  if (!A.given) {
    for (int c = 0; c < k; ++c) {
      const int m = c;
      km_sort(C, m, cv, sc, si);
      const int T = c == 0 ? 1 : A.T;
      double xcand[kKmMaxT];
#pragma unroll
      for (int t = 0; t < kKmMaxT; ++t) xcand[t] = t < T ? __ldcg(C->cval + t) : 0.0;
      for (unsigned long long b = gwarp; b < A.nb; b += nwarps) {
        double s[kKmMaxT];
        km_block_sums<kKmMaxT>(A, b, mean, [&](unsigned long long, double x, double (&a)[kKmMaxT]) {
          const double d = km_nearest_d(sc, m, x);
#pragma unroll
          for (int t = 0; t < kKmMaxT; ++t)
            if (t < T) a[t] = __dadd_rn(a[t], fmin(d, km_d2(x, xcand[t])));
        }, s);
        if (lane < static_cast<unsigned>(T)) {
          double mine = s[0];
#pragma unroll
          for (int t = 1; t < kKmMaxT; ++t) if (lane == static_cast<unsigned>(t)) mine = s[t];
          A.col[static_cast<unsigned long long>(lane) * A.nb + b] = mine;
        }
      }
      if (grid_arrive(A.sync, epoch, &flag_s)) {
        if (warp < static_cast<unsigned>(T)) {
          const double p = km_total(A, warp);
          if (lane == 0) pot_s[warp] = p;
        }
        __syncthreads();
        int best = 0;
        for (int t = 1; t < T; ++t) if (pot_s[t] < pot_s[best]) best = t;
        const double xb = __ldcg(C->cval + best);
        if (threadIdx.x == 0) {
          C->cent[c] = xb;
          C->n_chosen = c + 1;
          if (A.init_ids) A.init_ids[c] = __ldcg(C->cand + best);
        }
        if (c + 1 < k) {
          // the next step's candidates, searched on the best column with the updated centres
          __syncthreads();
          if (threadIdx.x == 0) {   // insert xb into this CTA's sorted list (indices are not needed here)
            int p = km_upper(sc, m, xb);
            for (int i = m; i > p; --i) sc[i] = sc[i - 1];
            sc[p] = xb;
          }
          __syncthreads();
          double* stage = reinterpret_cast<double*>(km_smem) + static_cast<size_t>(warp) * kKmBlk;
          if (warp < static_cast<unsigned>(A.T)) {
            const double v = __dmul_rn(__ldg(A.draws + static_cast<size_t>(c) * A.T + warp), pot_s[best]);
            const long long id = km_search(A, best, v, sc, m + 1, xb, mean, stage);
            if (lane == 0) {
              C->cand[warp] = id;
              C->cval[warp] = __dsub_rn(static_cast<double>(A.in[id]), mean);
            }
          }
        }
        grid_release(A.sync, epoch);
      }
    }
  }

  // ---- Lloyd ----------------------------------------------------------------------------------------------------------
  double* wsum = reinterpret_cast<double*>(km_smem);                         // [kWarps][k]
  unsigned* wcnt = reinterpret_cast<unsigned*>(wsum + static_cast<size_t>(kWarps) * k);
  bool strict = false;
  int it = 0;
  for (; it < kKmMaxIter; ++it) {
    // (the accumulators share shared memory with the leader's totals)
    for (int i = threadIdx.x; i < kWarps * k; i += kThreads) { wsum[i] = 0.0; wcnt[i] = 0u; }
    km_sort(C, k, cv, sc, si);
    bool changed = false;
    for (unsigned long long u = blockIdx.x; u < A.units; u += gridDim.x) {
      for (unsigned long long b = u * A.unit_blocks + warp; b < (u + 1) * A.unit_blocks && b < A.nb; b += kWarps) {
        for (int r = 0; r < kKmRows; ++r) {
          const unsigned long long i = b * kKmBlk + static_cast<unsigned long long>(r) * 32 + lane;
          const bool valid = i < A.n;
          const unsigned vmask = __ballot_sync(0xffffffffu, valid);
          if (!valid) continue;
          const double x = km_xc(A, i, mean);
          double dmin;
          const int lab = km_label(sc, si, k, x, dmin);
          if (it == 0 || A.labels[i] != lab) changed = true;
          A.labels[i] = static_cast<unsigned char>(lab);
          const unsigned peers = __match_any_sync(vmask, lab);
          double s = 0.0;
          for (unsigned mm = peers; mm; mm &= mm - 1) s = __dadd_rn(s, __shfl_sync(peers, x, __ffs(mm) - 1));
          if (lane == static_cast<unsigned>(__ffs(peers) - 1)) {
            wsum[warp * k + lab] = __dadd_rn(wsum[warp * k + lab], s);
            wcnt[warp * k + lab] += __popc(peers);
          }
        }
      }
      __syncthreads();
      if (threadIdx.x < static_cast<unsigned>(k)) {
        const int j = threadIdx.x;
        double s = 0.0;
        unsigned cnt = 0;
        for (int w = 0; w < kWarps; ++w) {
          s = __dadd_rn(s, wsum[w * k + j]);
          cnt += wcnt[w * k + j];
          wsum[w * k + j] = 0.0;
          wcnt[w * k + j] = 0u;
        }
        A.usum[u * k + j] = s;
        A.ucnt[u * k + j] = cnt;
      }
      __syncthreads();
    }
    changed = __syncthreads_or(changed) != 0;
    if (changed && threadIdx.x == 0) atomicOr(&C->changed, 1);

    // leader: per-cluster totals (units in order; P = kThreads / k interleaved parts folded in order)
    double* tsum = reinterpret_cast<double*>(km_smem);        // [kThreads] then [k]
    unsigned long long* tcnt = reinterpret_cast<unsigned long long*>(tsum + kThreads);
    if (grid_arrive(A.sync, epoch, &flag_s)) {
      const int P = kThreads / k;
      {
        const int j = threadIdx.x % k, p = threadIdx.x / k;
        double s = 0.0;
        unsigned long long cnt = 0;
        if (p < P)
          for (unsigned long long u = p; u < A.units; u += P) {
            s = __dadd_rn(s, __ldcg(A.usum + u * k + j));
            cnt += __ldcg(A.ucnt + u * k + j);
          }
        __syncthreads();
        tsum[threadIdx.x] = s;
        tcnt[threadIdx.x] = cnt;
        __syncthreads();
        if (threadIdx.x < static_cast<unsigned>(k)) {
          for (int q = 1; q < P; ++q) {
            s = __dadd_rn(s, tsum[q * k + j]);
            cnt += tcnt[q * k + j];
          }
        }
        __syncthreads();
        if (threadIdx.x < static_cast<unsigned>(k)) { tsum[j] = s; tcnt[j] = cnt; }
        __syncthreads();
      }
      if (threadIdx.x == 0) {
        int n_empty = 0;
        for (int j = 0; j < k; ++j) n_empty += tcnt[j] == 0;
        C->n_empty = n_empty;
        C->reloc = n_empty > 0;
        C->reloc_d = inf;
        C->reloc_i = -1;
        C->strict = __ldcg(&C->changed) == 0;
        C->changed = 0;
        flag_s = n_empty;
      }
      __syncthreads();
      if (flag_s == 0) {
        km_finish(A, C, tsum, tcnt, cv, k, mean);
      } else if (threadIdx.x < static_cast<unsigned>(k)) {   // the relocating leader may be another CTA
        C->tsum[threadIdx.x] = tsum[threadIdx.x];
        C->tcnt[threadIdx.x] = tcnt[threadIdx.x];
      }
      grid_release(A.sync, epoch);
    }
    const int n_empty = __ldcg(&C->n_empty);
    if (n_empty > 0) {
      // the n_empty farthest points from their centres (by the labels just assigned), one grid-wide argmax per point
      for (int r = 0; r < n_empty; ++r) {
        const double pd = __ldcg(&C->reloc_d);
        const long long pi = __ldcg(&C->reloc_i);
        for (unsigned long long b = gwarp; b < A.nb; b += nwarps) {
          double bd = -1.0;
          long long bi = -1;
          for (int rr = 0; rr < kKmRows; ++rr) {
            const unsigned long long i = b * kKmBlk + static_cast<unsigned long long>(rr) * 32 + lane;
            if (i >= A.n) continue;
            const double d = km_d2(km_xc(A, i, mean), cv[A.labels[i]]);
            const long long ii = static_cast<long long>(i);
            if ((d < pd || (d == pd && ii > pi)) && km_better(d, ii, bd, bi)) { bd = d; bi = ii; }
          }
          for (int o = 16; o; o >>= 1) {
            const double od = __shfl_xor_sync(0xffffffffu, bd, o);
            const long long oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (km_better(od, oi, bd, bi)) { bd = od; bi = oi; }
          }
          if (lane == 0) { A.rbd[b] = bd; A.rbi[b] = bi; }
        }
        if (grid_arrive(A.sync, epoch, &flag_s)) {
          double bd = -1.0;
          long long bi = -1;
          for (unsigned long long b = threadIdx.x; b < A.nb; b += kThreads) {
            const double d = __ldcg(A.rbd + b);
            const long long ii = __ldcg(A.rbi + b);
            if (km_better(d, ii, bd, bi)) { bd = d; bi = ii; }
          }
          for (int o = 16; o; o >>= 1) {
            const double od = __shfl_xor_sync(0xffffffffu, bd, o);
            const long long oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (km_better(od, oi, bd, bi)) { bd = od; bi = oi; }
          }
          if (lane == 0) { red_d[warp] = bd; red_i[warp] = bi; }
          __syncthreads();
          if (threadIdx.x == 0) {
            for (int w = 0; w < kWarps; ++w)
              if (km_better(red_d[w], red_i[w], bd, bi)) { bd = red_d[w]; bi = red_i[w]; }
            // scikit-learn relocates nothing when every point sits on its centre
            if (r == 0 && !(bd > 0.0)) C->reloc = 0;
            A.far[r] = bi;
            C->reloc_d = bd;
            C->reloc_i = bi;
          }
          grid_release(A.sync, epoch);
        }
        if (!__ldcg(&C->reloc)) break;
      }
      // leader: relocation, averaging, shift, convergence
      if (grid_arrive(A.sync, epoch, &flag_s)) {
        if (threadIdx.x < static_cast<unsigned>(k)) {
          tsum[threadIdx.x] = __ldcg(C->tsum + threadIdx.x);
          tcnt[threadIdx.x] = __ldcg(C->tcnt + threadIdx.x);
        }
        __syncthreads();
        km_finish(A, C, tsum, tcnt, cv, k, mean);
        grid_release(A.sync, epoch);
      }
    }
    if (__ldcg(&C->stop)) {
      strict = __ldcg(&C->strict) != 0;
      break;
    }
  }
  const int n_iter = it < kKmMaxIter ? it + 1 : kKmMaxIter;

  // ---- last pass: labels (without strict convergence), inertia, the task's tensor -------------------------------------
  km_sort(C, k, cv, sc, si);
  __shared__ float cf[kKmMaxK];
  __shared__ float clo, chi;
  if (threadIdx.x < static_cast<unsigned>(k)) cf[threadIdx.x] = static_cast<float>(__dadd_rn(cv[threadIdx.x], mean));
  __syncthreads();
  if (threadIdx.x == 0) {
    float lo = cf[0], hi = cf[0];
    for (int j = 1; j < k; ++j) { lo = fminf(lo, cf[j]); hi = fmaxf(hi, cf[j]); }
    clo = lo;
    chi = hi;
  }
  __syncthreads();
  for (unsigned long long b = gwarp; b < A.nb; b += nwarps) {
    double s[1];
    km_block_sums<1>(A, b, mean, [&](unsigned long long i, double x, double (&a)[1]) {
      int lab;
      if (strict) {
        lab = A.labels[i];
      } else {
        double dmin;
        lab = km_label(sc, si, k, x, dmin);
        A.labels[i] = static_cast<unsigned char>(lab);
      }
      a[0] = __dadd_rn(a[0], km_d2(x, cv[lab]));
      if (A.task == 1) A.out[i] = cf[lab];
      else if (A.task == 2) A.out[i] = fminf(fmaxf(__ldg(A.in + i), clo), chi);
    }, s);
    if (lane == 0) A.col[b] = s[0];
  }
  if (grid_arrive(A.sync, epoch, &flag_s)) {
    if (warp == 0) {
      const double tot = km_total(A, 0);
      if (lane == 0) {
        *A.inertia = tot;
        *A.n_iter = n_iter;
      }
    }
    if (threadIdx.x < static_cast<unsigned>(k)) A.centres[threadIdx.x] = cf[threadIdx.x];
    grid_release(A.sync, epoch);
  }

  // ---- per-row bias correction: out_bcorr = fp32(out - (mean_row(out) - mean_row(x))), float64 row means --------------
  if (A.rows) {
    const unsigned long long len = A.n / A.rows;
    for (unsigned long long r = gwarp; r < A.rows; r += nwarps) {
      double sw = 0.0, sq = 0.0;
      for (unsigned long long i = r * len + lane; i < (r + 1) * len; i += 32) {
        sw = __dadd_rn(sw, static_cast<double>(__ldg(A.in + i)));
        sq = __dadd_rn(sq, static_cast<double>(__ldcg(A.out + i)));
      }
      sw = km_butterfly(sw);
      sq = km_butterfly(sq);
      const double delta = __dsub_rn(sq / static_cast<double>(len), sw / static_cast<double>(len));
      for (unsigned long long i = r * len + lane; i < (r + 1) * len; i += 32)
        A.out_bcorr[i] = static_cast<float>(__dsub_rn(static_cast<double>(__ldcg(A.out + i)), delta));
    }
  }
  grid_exit(A.sync);
}

}  // namespace fqb
