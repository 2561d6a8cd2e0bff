// Sample-angle measurement (angle_stats.py:17-44): for `rows` contiguous samples of `row_len` floats (X, [rows, row_len];
// a sample is contiguous in NCHW and channels-last memory alike), the float64 Gram matrix G = X X^T and the angles
// acos(G_ij / sqrt(G_ii * G_jj)).  Two launches, no host synchronisation, no atomics on the values:
//
//   fq_gram_partial_kernel  FP64 tensor cores (mma.sync m16n8k16 f64)  one (tile pair, K slice) unit per CTA iteration:
//                                                  64x64 block (bi, bj), bi <= bj, of the Gram matrix over one slice of
//                                                  the samples; fp32 tiles staged through a cp.async ring in shared
//                                                  memory, converted to f64 when the fragments are built; the unit's
//                                                  partial block goes to its own workspace slot
//   fq_gram_finish_kernel   one thread per element of a tile pair       adds the element's partials in slice order,
//                                                  writes G (j >= i), the angle (j > i) and the zeros on and below the
//                                                  diagonal (a pair (bi, bj) also zeroes its mirror block (bj, bi))
//
// Determinism.  The slice count depends on (rows, row_len) only (kAngUnitTarget units, at least kAngMinSteps k-steps a
// slice), never on the device or the grid; every unit runs the same fixed sequence of MMAs whichever CTA takes it, and
// the finish adds slices in order, so the bits do not depend on the run or on max_ctas.  fp32 x fp32 products are exact
// in float64, and each element of G sees the same products in the same order wherever it sits in the matrix: a
// duplicated sample gives G_ij == G_ii == G_jj bit for bit, so cos = G_ij / sqrt(G_ii * G_jj) is exactly 1 (and exactly -1
// for a negated one).
//
// Workspace: pairs * slices * 64 * 64 float64, with pairs = T (T + 1) / 2, T = ceil(rows / 64), and
// slices <= ceil(kAngUnitTarget / pairs): at most (pairs + kAngUnitTarget) * 32 KB (34 MB at rows = 512, 297 MB at the
// limit of kAngMaxRows = 8192).
namespace fqb {

constexpr int kAngTile = 64;      // rows (samples) per tile
constexpr int kAngBK = 32;        // k elements per ring stage (two m16n8k16 steps)
constexpr int kAngPitch = 36;     // floats per shared-memory tile row: fragment reads hit 32 distinct banks
constexpr int kAngStages = 3;     // cp.async ring depth
constexpr int kAngThreads = 128;  // 4 warps, each a 32 x 32 quarter of the 64 x 64 block
constexpr int kAngFinishThreads = 256;
constexpr unsigned long long kAngUnitTarget = 1024;  // (tile pair, slice) units aimed at when there are fewer pairs
constexpr unsigned long long kAngMinSteps = 8;       // k-steps (of kAngBK) a slice holds at least
constexpr long long kAngMaxRows = 8192;
constexpr size_t kAngSmemBytes = static_cast<size_t>(kAngStages) * 2 * kAngTile * kAngPitch * sizeof(float);

struct AngleArgs {
  const float* in;
  unsigned long long rows, row_len;  // sample r is in[r * row_len, (r + 1) * row_len)
  unsigned long long tiles, pairs;   // T = ceil(rows / 64); pairs = T (T + 1) / 2, (bi, bj) with bi <= bj, row-major
  unsigned long long slices;         // K slices per pair
  unsigned long long slice_steps;    // kAngBK steps per slice (the last slice may hold fewer)
  double* partial;                   // [pairs][slices][64][64]
  float* angles;                     // [rows][rows] or null
  double* gram;                      // [rows][rows] or null
};

// the slice count of (rows, row_len): a function of the shape alone
struct AngleSplit {
  unsigned long long tiles, pairs, slices, slice_steps;
};
__host__ __device__ inline AngleSplit angle_split(unsigned long long rows, unsigned long long row_len) {
  AngleSplit s;
  s.tiles = (rows + kAngTile - 1) / kAngTile;
  s.pairs = s.tiles * (s.tiles + 1) / 2;
  const unsigned long long steps = (row_len + kAngBK - 1) / kAngBK;
  unsigned long long want = s.pairs ? (kAngUnitTarget + s.pairs - 1) / s.pairs : 1;
  const unsigned long long most = (steps + kAngMinSteps - 1) / kAngMinSteps;
  if (want > most) want = most;
  if (want < 1) want = 1;
  s.slice_steps = (steps + want - 1) / want;
  s.slices = (steps + s.slice_steps - 1) / s.slice_steps;
  return s;
}

// pair index p -> (bi, bj), row-major over bi <= bj
__device__ __forceinline__ void angle_pair(unsigned long long p, unsigned long long tiles, unsigned& bi, unsigned& bj) {
  unsigned long long b = 0;
  while (p >= tiles - b) {
    p -= tiles - b;
    ++b;
  }
  bi = static_cast<unsigned>(b);
  bj = static_cast<unsigned>(b + p);
}
__device__ __forceinline__ unsigned long long angle_pair_index(unsigned long long bi, unsigned long long bj,
                                                               unsigned long long tiles) {
  return bi * tiles - bi * (bi - 1) / 2 + (bj - bi);
}

// cp.async with zero fill: src_bytes = 0 writes zeros (rows past `rows`, k past the slice)
__device__ __forceinline__ void ang_cp16(unsigned dst, const float* src, unsigned src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void ang_cp4(unsigned dst, const float* src, unsigned src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}

// D += A B with A 16x16 (row), B 16x8 (col), f64.  Fragments (groupID g = lane / 4, t = lane % 4):
// a[2q] = A[g][t + 4q], a[2q + 1] = A[g + 8][t + 4q]; b[q] = B[t + 4q][g]; c = C[g][2t], C[g][2t + 1], C[g + 8][2t],
// C[g + 8][2t + 1].
__device__ __forceinline__ void dmma16816(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
  asm("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
      "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
      : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
        "d"(b[2]), "d"(b[3]));
}

// VEC = 4: 16-byte copies (row_len % 4 == 0 and a 16-byte aligned base); VEC = 1: 4-byte copies
template <int VEC>
__global__ void __launch_bounds__(kAngThreads) fq_gram_partial_kernel(const __grid_constant__ AngleArgs A) {
  extern __shared__ __align__(16) float ang_smem[];
  constexpr int kTileFloats = kAngTile * kAngPitch;
  constexpr int kChunksPerRow = kAngBK / VEC;
  constexpr int kCopies = kAngTile * kChunksPerRow / kAngThreads;  // per thread and tile
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;
  const unsigned smem0 = static_cast<unsigned>(__cvta_generic_to_shared(ang_smem));
  const unsigned long long units = A.pairs * A.slices;
  for (unsigned long long u = blockIdx.x; u < units; u += gridDim.x) {
    const unsigned long long pair = u / A.slices, slice = u % A.slices;
    unsigned bi, bj;
    angle_pair(pair, A.tiles, bi, bj);
    const bool diag = bi == bj;
    const unsigned long long k0 = slice * A.slice_steps * kAngBK;
    const unsigned long long k1 = k0 + A.slice_steps * kAngBK < A.row_len ? k0 + A.slice_steps * kAngBK : A.row_len;
    const int nsteps = static_cast<int>((k1 - k0 + kAngBK - 1) / kAngBK);

    // stage s holds tile bi's rows, then (off the diagonal) tile bj's rows, each [64][kAngPitch] over k0 + step * kAngBK
    auto load = [&](int step, int s) {
      const unsigned long long kb = k0 + static_cast<unsigned long long>(step) * kAngBK;
#pragma unroll
      for (int op = 0; op < 2; ++op) {
        if (op == 1 && diag) break;
        const unsigned long long r0 = static_cast<unsigned long long>(op ? bj : bi) * kAngTile;
#pragma unroll
        for (int i = 0; i < kCopies; ++i) {
          const int c = threadIdx.x + i * kAngThreads;
          const int rr = c / kChunksPerRow, kk = (c % kChunksPerRow) * VEC;
          const unsigned long long r = r0 + rr, k = kb + kk;
          const bool in = r < A.rows && k < k1;
          const float* src = in ? A.in + r * A.row_len + k : A.in;
          const unsigned dst = smem0 + static_cast<unsigned>(((s * 2 + op) * kTileFloats + rr * kAngPitch + kk) * 4);
          if constexpr (VEC == 4) ang_cp16(dst, src, in ? 16u : 0u);
          else                    ang_cp4(dst, src, in ? 4u : 0u);
        }
      }
    };

    double acc[2][4][4];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 4; ++ni)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[mi][ni][q] = 0.0;

#pragma unroll
    for (int s = 0; s < kAngStages - 1; ++s) {
      if (s < nsteps) load(s, s);
      cp_async_commit();
    }
    for (int step = 0; step < nsteps; ++step) {
      cp_async_wait<kAngStages - 2>();
      __syncthreads();  // stage `step` has landed for every thread; stage `step - 1` is free again
      const int nxt = step + kAngStages - 1;
      if (nxt < nsteps) load(nxt, nxt % kAngStages);
      cp_async_commit();
      const float* sa = ang_smem + (step % kAngStages) * 2 * kTileFloats;
      const float* sb = diag ? sa : sa + kTileFloats;
#pragma unroll
      for (int kk = 0; kk < kAngBK; kk += 16) {
        double a[2][8], b[4][4];
#pragma unroll
        for (int mi = 0; mi < 2; ++mi) {
          const float* p = sa + (wm + mi * 16 + g) * kAngPitch + kk + t;
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            a[mi][2 * q] = static_cast<double>(p[4 * q]);
            a[mi][2 * q + 1] = static_cast<double>(p[8 * kAngPitch + 4 * q]);
          }
        }
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) {
          const float* p = sb + (wn + ni * 8 + g) * kAngPitch + kk + t;
#pragma unroll
          for (int q = 0; q < 4; ++q) b[ni][q] = static_cast<double>(p[4 * q]);
        }
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
          for (int ni = 0; ni < 4; ++ni) dmma16816(acc[mi][ni], a[mi], b[ni]);
      }
    }
    cp_async_wait<0>();
    __syncthreads();  // the ring is reused by the next unit

    double* out = A.partial + u * (kAngTile * kAngTile);
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 4; ++ni) {
        const int r = wm + mi * 16 + g, c = wn + ni * 8 + 2 * t;
        __stcg(reinterpret_cast<double2*>(out + r * kAngTile + c), make_double2(acc[mi][ni][0], acc[mi][ni][1]));
        __stcg(reinterpret_cast<double2*>(out + (r + 8) * kAngTile + c), make_double2(acc[mi][ni][2], acc[mi][ni][3]));
      }
  }
}

// one block of the grid's x dimension covers kAngFinishThreads elements of the 64 x 64 tile pair blockIdx.y
__global__ void __launch_bounds__(kAngFinishThreads) fq_gram_finish_kernel(const __grid_constant__ AngleArgs A) {
  const unsigned long long pair = blockIdx.y;
  unsigned bi, bj;
  angle_pair(pair, A.tiles, bi, bj);
  const int e = blockIdx.x * kAngFinishThreads + threadIdx.x;
  const int ii = e / kAngTile, jj = e % kAngTile;
  const unsigned long long i = static_cast<unsigned long long>(bi) * kAngTile + ii;
  const unsigned long long j = static_cast<unsigned long long>(bj) * kAngTile + jj;
  if (bi != bj && A.angles) {  // the mirror block (bj, bi) lies below the diagonal: zeros
    const unsigned long long mi = static_cast<unsigned long long>(bj) * kAngTile + ii;
    const unsigned long long mj = static_cast<unsigned long long>(bi) * kAngTile + jj;
    if (mi < A.rows && mj < A.rows) A.angles[mi * A.rows + mj] = 0.0f;
  }
  if (i >= A.rows || j >= A.rows) return;
  constexpr int kBlock = kAngTile * kAngTile;
  const double* p = A.partial + pair * A.slices * kBlock;
  double gij = __ldcg(p + e);
  for (unsigned long long s = 1; s < A.slices; ++s) gij = __dadd_rn(gij, __ldcg(p + s * kBlock + e));
  if (A.gram && j >= i) A.gram[i * A.rows + j] = gij;
  if (!A.angles) return;
  if (j <= i) {
    A.angles[i * A.rows + j] = 0.0f;
    return;
  }
  // G_ii and G_jj from the diagonal blocks, summed in the same slice order as every other element
  const double* pi = A.partial + angle_pair_index(bi, bi, A.tiles) * A.slices * kBlock + ii * (kAngTile + 1);
  const double* pj = A.partial + angle_pair_index(bj, bj, A.tiles) * A.slices * kBlock + jj * (kAngTile + 1);
  double gii = __ldcg(pi), gjj = __ldcg(pj);
  for (unsigned long long s = 1; s < A.slices; ++s) {
    gii = __dadd_rn(gii, __ldcg(pi + s * kBlock));
    gjj = __dadd_rn(gjj, __ldcg(pj + s * kBlock));
  }
  // one sqrt of the product: a duplicated sample (G_ij == G_ii == G_jj) gives exactly 1.  The clamp keeps a cosine a
  // rounding step outside [-1, 1] a real angle; a cosine that is not finite (a zero sample: 0 / 0; NaN / Inf input) is NaN.
  const double d = __dmul_rn(gii, gjj);
  const double c = __ddiv_rn(gij, __dsqrt_rn(d));
  float th;
  if (isfinite(gij) && isfinite(d) && isfinite(c)) th = static_cast<float>(acos(fmin(fmax(c, -1.0), 1.0)));
  else th = __int_as_float(0x7fffffff);
  A.angles[i * A.rows + j] = th;
}

}  // namespace fqb
