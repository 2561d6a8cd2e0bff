// fqb200 bulk-copy streaming engine (sm_90a): flat tensors through a ring of shared-memory stages filled by the TMA unit.
//
// Why: the per-thread cp.async ring of fq_device.cuh spends most of its thread instructions per 128-bit vector on cursor /
// ring bookkeeping, and the phases of L2-resident tensors were issue-bound.  Here ONE elected thread of a dedicated producer warp issues
// `cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes` (1-D TMA, SASS UBLKCP) for a whole 16 KB stage;
// the 512 consumer threads wait on the stage's `full` mbarrier, read their vectors with LDS.128 and hand the stage back
// through its `empty` mbarrier (one arrival per consumer warp).  No per-vector address arithmetic, no cp.async groups.
//
// The producer never waits at the grid barriers between the phases of a fused launch: while the consumers combine their
// statistics and wait for the other CTAs, the ring is already being filled with the first stages of the next phase.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "fq_device.cuh"

namespace fqb {

constexpr int kConsumers = kThreads;             // 512 consumer threads (16 warps)
constexpr int kBulkThreads = kConsumers + 32;    // + one producer warp
constexpr int kConsumerWarps = kConsumers / 32;
// Ring shape: ONE CTA per SM with six 32 KB stages (192 KB of the 227 KB an H100 block may use).  A bulk request should
// be large, and one CTA per SM halves the barrier arrivals, atomics and tickets of two.  tools/build_variants.sh builds
// the other shapes (the macros below) for A/B runs.
#ifndef FQB_STAGE_VEC
#define FQB_STAGE_VEC 4
#endif
#ifndef FQB_STAGES
#define FQB_STAGES 6
#endif
#ifndef FQB_BULK_CTAS
#define FQB_BULK_CTAS 1
#endif
constexpr int kBulkCtasPerSm = FQB_BULK_CTAS;    // resident CTAs per SM of the bulk-ring kernels
constexpr int kStageVec = FQB_STAGE_VEC;         // vectors per consumer thread per stage
constexpr int kStages = FQB_STAGES;              // ring depth
constexpr unsigned kStageBytes = kStageVec * kConsumers * 16u;
#ifndef FQB_BULK_SPLIT
#define FQB_BULK_SPLIT 1
#endif
constexpr unsigned kBulkSplit = FQB_BULK_SPLIT;  // bulk copies per stage (all complete on the stage's one mbarrier)

// consumer-only CTA barrier (the producer warp never joins): named barrier 1 over the 512 consumer threads.  The
// 512-thread kernels of fq_device.cuh can use it as well (there it is equivalent to __syncthreads()).
__device__ __forceinline__ void consumer_sync() { cta_sync(); }

// ---- mbarrier / bulk-copy primitives --------------------------------------------------------------------------------
__device__ __forceinline__ unsigned smem_u32(const void* p) { return static_cast<unsigned>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(unsigned bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(unsigned bar) {
  asm volatile("{ .reg .b64 st; mbarrier.arrive.shared::cta.b64 st, [%0]; }" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned bar, unsigned bytes) {
  asm volatile("{ .reg .b64 st; mbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1; }" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned bar, unsigned parity) {
  unsigned ok;
  asm volatile(
      "{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// 1-D bulk copy global -> shared, completion counted in bytes on `bar`.  bytes % 16 == 0, both addresses 16-byte aligned.
__device__ __forceinline__ void bulk_load_one(unsigned dst_smem, const void* src, unsigned bytes, unsigned bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void bulk_load(unsigned dst_smem, const void* src, unsigned bytes, unsigned bar) {
  if (kBulkSplit == 1u) {
    bulk_load_one(dst_smem, src, bytes, bar);
    return;
  }
  constexpr unsigned piece = kStageBytes / kBulkSplit;
  for (unsigned off = 0; off < bytes; off += piece)
    bulk_load_one(dst_smem + off, static_cast<const unsigned char*>(src) + off, min(piece, bytes - off), bar);
}

// ---- geometry of a flat stream ---------------------------------------------------------------------------------------
// The tensor is ONE contiguous run of total_v vectors (channels-last activations; per-tensor views).  A stage is
// stage_v = kStageVec * stride consecutive vectors; consumer thread t reads vectors t, t + stride, ... of the stage
// (threads >= stride idle: stride is the largest multiple of the channel period cv = C/4 below 512, so that a thread
// always sees the same four channels).  A UNIT is unit_stages consecutive stages and is what CTAs pull dynamically.
struct FlatGeo {
  unsigned total_v;      // vectors in the tensor (< 2^32)
  unsigned stride;       // consumer threads that take part (<= 512), multiple of cv
  unsigned stage_v;      // kStageVec * stride
  unsigned n_stages;     // ceil(total_v / stage_v)
  unsigned unit_stages;  // stages per unit
  unsigned units;        // ceil(n_stages / unit_stages)
  unsigned channels;     // C (0 for per-tensor streams)
  unsigned cv;           // C / 4 (1 for per-tensor streams)
};

struct StageMeta {
  unsigned start;  // first vector of the stage
  unsigned count;  // valid vectors; 0 = end of phase
  unsigned tag;    // row-structured streams: row index | (last stage of its unit) << 31
  unsigned pad;
};

struct BulkRing {
  alignas(8) unsigned long long full[kStages];
  alignas(8) unsigned long long empty[kStages];
  StageMeta meta[kStages];
  unsigned nstages;  // stages in use (<= kStages; the histogram variants lend the last one to the histogram)
};

// position in the ring sequence: both sides count every stage AND every end-of-phase marker
struct RingPos {
  unsigned slot, parity, n;
  __device__ __forceinline__ void init(unsigned nstages = kStages) {
    slot = 0;
    parity = 0;
    n = nstages;
  }
  __device__ __forceinline__ void next() {
    if (++slot == n) {
      slot = 0;
      parity ^= 1u;
    }
  }
};

__device__ __forceinline__ void ring_init(BulkRing& r, unsigned nstages = kStages) {
  if (threadIdx.x == 0) {
    r.nstages = nstages;
#pragma unroll
    for (int s = 0; s < kStages; ++s) {
      mbar_init(smem_u32(&r.full[s]), 1u);                 // the producer's arrive(.expect_tx)
      mbar_init(smem_u32(&r.empty[s]), kConsumerWarps);    // one arrival per consumer warp
    }
    mbar_fence_init();
  }
  __syncthreads();  // all 544 threads, once
}

// ---- producer side (one thread) ----------------------------------------------------------------------------------------
// Ticket k of this CTA: static for the first `nstatic` (id = first + k * step; no atomic in front of the first loads),
// then from the phase's atomic counter (offset by `dyn_base`, the number of statically dealt units).  REV walks the
// units and the stages inside a unit backwards so that a phase starts on what the previous one touched last.
struct TicketPlan {
  unsigned nstatic;    // static tickets of this CTA (0..2)
  unsigned first, step;
  unsigned dyn_base;   // units dealt statically over the whole grid
};

// PAIR: a second tensor of the same shape (`src2`, the residual of a fused block epilogue) rides along: the stage holds
// stage_v vectors of src in its lower half and the same vectors of src2 in its upper half (g is then half_geo()).
constexpr unsigned kPairOffset = kStageBytes / 2u;

__device__ __forceinline__ FlatGeo half_geo(const FlatGeo& g) {
  FlatGeo h = g;
  h.stage_v = (kStageVec / 2u) * g.stride;
  h.n_stages = (g.total_v + h.stage_v - 1u) / h.stage_v;
  h.unit_stages = 2u * g.unit_stages;  // the units (and the tickets) stay the same
  return h;
}

template <bool REV, bool PAIR = false>
__device__ __forceinline__ void produce_phase(const FlatGeo& g, const float4* src, unsigned* counter, const TicketPlan tp,
                                              BulkRing& r, unsigned char* stage_base, RingPos& pos,
                                              const float4* src2 = nullptr) {
  const unsigned total = g.units;
  unsigned k = 0;
  auto fetch = [&]() -> unsigned {
    unsigned long long t;
    if (k < tp.nstatic)
      t = tp.first + static_cast<unsigned long long>(k) * tp.step;
    else
      t = static_cast<unsigned long long>(tp.dyn_base) + atomicAdd(counter, 1u);
    ++k;
    return t < total ? static_cast<unsigned>(t) : 0xffffffffu;
  };
  // two tickets ahead: the atomic's round trip (long under contention) must not sit in front of a unit's loads
  unsigned cur = fetch();
  unsigned nxt = (cur != 0xffffffffu) ? fetch() : 0xffffffffu;
  while (cur != 0xffffffffu) {
    const unsigned nxt2 = (nxt != 0xffffffffu) ? fetch() : 0xffffffffu;
    const unsigned u = REV ? total - 1u - cur : cur;
    const unsigned g0 = u * g.unit_stages;
    const unsigned g1 = min(g0 + g.unit_stages, g.n_stages);
    for (unsigned i = g0; i < g1; ++i) {
      const unsigned st = REV ? g1 - 1u - (i - g0) : i;
      const unsigned start = st * g.stage_v;
      const unsigned count = min(g.stage_v, g.total_v - start);
      mbar_wait(smem_u32(&r.empty[pos.slot]), pos.parity ^ 1u);
      r.meta[pos.slot].start = start;
      r.meta[pos.slot].count = count;
      r.meta[pos.slot].tag = 0u;
      const unsigned bar = smem_u32(&r.full[pos.slot]);
      mbar_arrive_expect_tx(bar, PAIR ? count * 32u : count * 16u);
      bulk_load(smem_u32(stage_base + pos.slot * kStageBytes), src + start, count * 16u, bar);
      if (PAIR) bulk_load(smem_u32(stage_base + pos.slot * kStageBytes + kPairOffset), src2 + start, count * 16u, bar);
      pos.next();
    }
    cur = nxt;
    nxt = nxt2;
  }
  // end-of-phase marker
  mbar_wait(smem_u32(&r.empty[pos.slot]), pos.parity ^ 1u);
  r.meta[pos.slot].start = 0u;
  r.meta[pos.slot].count = 0u;
  mbar_arrive(smem_u32(&r.full[pos.slot]));
  pos.next();
}

// Row-structured streams (per-sample statistics): `rows` rows of row_v vectors; a unit is a run of stages INSIDE one row
// (the last stage of a row is short), so that per-row partial results can be combined at unit ends.
struct RowsGeo {
  unsigned rows, row_v;
  unsigned stages_per_row;  // ceil(row_v / stage_v)
  unsigned units_per_row;   // ceil(stages_per_row / unit_stages)
};

// the row geometry of pair stages (g = half_geo() of the launch's geometry): the units stay the same
__device__ __forceinline__ RowsGeo half_rows(const FlatGeo& h, const RowsGeo& rg) {
  RowsGeo r = rg;
  r.stages_per_row = (rg.row_v + h.stage_v - 1u) / h.stage_v;
  r.units_per_row = (r.stages_per_row + h.unit_stages - 1u) / h.unit_stages;
  return r;
}

template <bool REV, bool PAIR = false>
__device__ __forceinline__ void produce_rows_phase(const FlatGeo& g, const RowsGeo& rg, const float4* src, unsigned* counter,
                                                   const TicketPlan tp, BulkRing& r, unsigned char* stage_base, RingPos& pos,
                                                   const float4* src2 = nullptr) {
  const unsigned total = g.units;  // rows * units_per_row
  unsigned k = 0;
  auto fetch = [&]() -> unsigned {
    unsigned long long t;
    if (k < tp.nstatic)
      t = tp.first + static_cast<unsigned long long>(k) * tp.step;
    else
      t = static_cast<unsigned long long>(tp.dyn_base) + atomicAdd(counter, 1u);
    ++k;
    return t < total ? static_cast<unsigned>(t) : 0xffffffffu;
  };
  unsigned cur = fetch();
  unsigned nxt = (cur != 0xffffffffu) ? fetch() : 0xffffffffu;
  while (cur != 0xffffffffu) {
    const unsigned nxt2 = (nxt != 0xffffffffu) ? fetch() : 0xffffffffu;
    const unsigned u = REV ? total - 1u - cur : cur;
    const unsigned row = u / rg.units_per_row;
    const unsigned part = u - row * rg.units_per_row;
    const unsigned s0 = part * g.unit_stages;
    const unsigned s1 = min(s0 + g.unit_stages, rg.stages_per_row);
    for (unsigned i = s0; i < s1; ++i) {
      const unsigned st = REV ? s1 - 1u - (i - s0) : i;
      const unsigned off = st * g.stage_v;
      const unsigned start = row * rg.row_v + off;
      const unsigned count = min(g.stage_v, rg.row_v - off);
      mbar_wait(smem_u32(&r.empty[pos.slot]), pos.parity ^ 1u);
      r.meta[pos.slot].start = start;
      r.meta[pos.slot].count = count;
      r.meta[pos.slot].tag = row | (i + 1u == s1 ? 0x80000000u : 0u);
      const unsigned bar = smem_u32(&r.full[pos.slot]);
      mbar_arrive_expect_tx(bar, PAIR ? count * 32u : count * 16u);
      bulk_load(smem_u32(stage_base + pos.slot * kStageBytes), src + start, count * 16u, bar);
      if (PAIR) bulk_load(smem_u32(stage_base + pos.slot * kStageBytes + kPairOffset), src2 + start, count * 16u, bar);
      pos.next();
    }
    cur = nxt;
    nxt = nxt2;
  }
  mbar_wait(smem_u32(&r.empty[pos.slot]), pos.parity ^ 1u);
  r.meta[pos.slot].start = 0u;
  r.meta[pos.slot].count = 0u;
  r.meta[pos.slot].tag = 0u;
  mbar_arrive(smem_u32(&r.full[pos.slot]));
  pos.next();
}

// ---- 2x2 / stride-2 max pooling inside the apply phase (channels-last) -------------------------------------------------------
// A TILE is two vertically adjacent input rows x `wt` pixels (wt even, wt * cv <= 1024 vectors): the two row pieces are two
// contiguous runs of the stream and land in the two halves of a stage (pair layout); thread o < (wt / 2) * cv produces output
// vector o of the tile: pixel pair j = o / cv, channel column o % cv (the same four channels the thread holds in the
// statistics phases, since the stride of those is a multiple of cv).  Units are runs of `unit_tiles` tiles.
struct PoolGeo {
  unsigned h, w;           // input rows / pixels per row
  unsigned wt;             // tile width in pixels
  unsigned tiles_per_row;  // w / wt
  unsigned row_pairs;      // h / 2 (a last odd row is dropped, like torch's floor mode)
  unsigned tiles;          // n * row_pairs * tiles_per_row
  unsigned unit_tiles, units;
  unsigned ow;             // w / 2
  unsigned kind;           // 2: 2x2 / stride 2 (above); 3: 3x3 / stride 2 / padding 1 (below)
};

// kind 3 (the ResNet stem): a tile is ONE output row x `wt` OUTPUT pixels; it needs the three input rows 2*oh-1 .. 2*oh+1
// from input pixel 2*ow0-1 on, 2*wt+1 pixels each: three bulk copies into three regions of region_v = (2*wt+1)*cv vectors
// (3 * region_v <= one stage).  The row above the image and the pixel left of it do not exist: those copies are skipped /
// start one pixel later (at the same place in the region) and the tag tells the consumer (bit 0: top row present, bit 1:
// left pixel present).  H and W are even, so the bottom row and the right pixel always exist.  Neighbouring tiles and rows
// overlap by one pixel / one row: 1.5 reads per element, most of them L2 hits.
constexpr unsigned kPoolTop = 1u, kPoolLeft = 2u;

__device__ __forceinline__ void produce_pool3_phase(const FlatGeo& g, const PoolGeo& pg, const float4* src, unsigned* counter,
                                                    const TicketPlan tp, BulkRing& r, unsigned char* stage_base, RingPos& pos) {
  const unsigned total = pg.units;
  unsigned k = 0;
  auto fetch = [&]() -> unsigned {
    unsigned long long t;
    if (k < tp.nstatic)
      t = tp.first + static_cast<unsigned long long>(k) * tp.step;
    else
      t = static_cast<unsigned long long>(tp.dyn_base) + atomicAdd(counter, 1u);
    ++k;
    return t < total ? static_cast<unsigned>(t) : 0xffffffffu;
  };
  const unsigned row_v = pg.w * g.cv;
  const unsigned region_v = (2u * pg.wt + 1u) * g.cv;
  const unsigned per_img = pg.row_pairs * pg.tiles_per_row;   // row_pairs = output rows
  unsigned cur = fetch();
  unsigned nxt = (cur != 0xffffffffu) ? fetch() : 0xffffffffu;
  while (cur != 0xffffffffu) {
    const unsigned nxt2 = (nxt != 0xffffffffu) ? fetch() : 0xffffffffu;
    const unsigned t0 = cur * pg.unit_tiles;
    const unsigned t1 = min(t0 + pg.unit_tiles, pg.tiles);
    for (unsigned tile = t0; tile < t1; ++tile) {
      const unsigned n = tile / per_img;
      const unsigned rem = tile - n * per_img;
      const unsigned oh = rem / pg.tiles_per_row;
      const unsigned wi = rem - oh * pg.tiles_per_row;
      const bool top = oh > 0u, left = wi > 0u;
      const unsigned skip = left ? 0u : g.cv;                      // vectors of the missing left pixel
      const unsigned count = region_v - skip;                       // vectors per row piece
      // first vector of the middle row's piece (input row 2*oh, input pixel 2*wi*wt - 1, clipped)
      const unsigned mid = (n * pg.h + 2u * oh) * row_v + (2u * wi * pg.wt) * g.cv - (left ? g.cv : 0u);
      const unsigned o = ((n * pg.row_pairs + oh) * pg.ow + wi * pg.wt) * g.cv;
      mbar_wait(smem_u32(&r.empty[pos.slot]), pos.parity ^ 1u);
      r.meta[pos.slot].start = o;
      r.meta[pos.slot].count = count;
      r.meta[pos.slot].tag = (top ? kPoolTop : 0u) | (left ? kPoolLeft : 0u);
      const unsigned bar = smem_u32(&r.full[pos.slot]);
      mbar_arrive_expect_tx(bar, count * 16u * (top ? 3u : 2u));
      const unsigned dst = smem_u32(stage_base + pos.slot * kStageBytes) + skip * 16u;
      if (top) bulk_load(dst, src + mid - row_v, count * 16u, bar);
      bulk_load(dst + region_v * 16u, src + mid, count * 16u, bar);
      bulk_load(dst + 2u * region_v * 16u, src + mid + row_v, count * 16u, bar);
      pos.next();
    }
    cur = nxt;
    nxt = nxt2;
  }
  mbar_wait(smem_u32(&r.empty[pos.slot]), pos.parity ^ 1u);
  r.meta[pos.slot].start = 0u;
  r.meta[pos.slot].count = 0u;
  r.meta[pos.slot].tag = 0u;
  mbar_arrive(smem_u32(&r.full[pos.slot]));
  pos.next();
}

// acc.pool_begin(); acc.pool_tap(v) for every tap of the window that exists, in torch's order (rows, then pixels);
// acc.pool_end(out_vector)
template <typename Acc>
__device__ __forceinline__ void consume_pool3_phase(const FlatGeo& g, const PoolGeo& pg, BulkRing& r, const unsigned char* stage_base,
                                                    RingPos& pos, Acc& acc) {
  const unsigned t = threadIdx.x;
  const bool lane0 = (t & 31u) == 0u;
  const bool mine = t < pg.wt * g.cv;
  const unsigned j = t / g.cv, col = t - j * g.cv;
  const unsigned region = (2u * pg.wt + 1u) * g.cv * 16u;
  const unsigned my = smem_u32(stage_base) + ((2u * j) * g.cv + col) * 16u;   // tap (dy = 0, dx = 0)
  const unsigned nxt = g.cv * 16u;
  for (;;) {
    mbar_wait(smem_u32(&r.full[pos.slot]), pos.parity);
    const StageMeta m = r.meta[pos.slot];
    if (m.count != 0u && mine) {
      const unsigned addr = my + pos.slot * kStageBytes;
      const bool first = (j != 0u) || (m.tag & kPoolLeft);   // the window's left pixel exists
      acc.pool_begin();
#pragma unroll
      for (int dy = 0; dy < 3; ++dy) {
        if (dy == 0 && !(m.tag & kPoolTop)) continue;
        const unsigned row = addr + dy * region;
        float4 v;
        if (first) {
          lds_vec(row, v);
          acc.pool_tap(v);
        }
        lds_vec(row + nxt, v);
        acc.pool_tap(v);
        lds_vec(row + 2u * nxt, v);
        acc.pool_tap(v);
      }
      acc.pool_end(m.start + t);
    }
    __syncwarp();
    if (lane0) mbar_arrive(smem_u32(&r.empty[pos.slot]));
    pos.next();
    if (m.count == 0u) break;
  }
}

__device__ __forceinline__ void produce_pool_phase(const FlatGeo& g, const PoolGeo& pg, const float4* src, unsigned* counter,
                                                   const TicketPlan tp, BulkRing& r, unsigned char* stage_base, RingPos& pos) {
  const unsigned total = pg.units;
  unsigned k = 0;
  auto fetch = [&]() -> unsigned {
    unsigned long long t;
    if (k < tp.nstatic)
      t = tp.first + static_cast<unsigned long long>(k) * tp.step;
    else
      t = static_cast<unsigned long long>(tp.dyn_base) + atomicAdd(counter, 1u);
    ++k;
    return t < total ? static_cast<unsigned>(t) : 0xffffffffu;
  };
  const unsigned row_v = pg.w * g.cv;      // vectors per input row
  const unsigned count = pg.wt * g.cv;     // vectors per row piece
  const unsigned per_img = pg.row_pairs * pg.tiles_per_row;
  unsigned cur = fetch();
  unsigned nxt = (cur != 0xffffffffu) ? fetch() : 0xffffffffu;
  while (cur != 0xffffffffu) {
    const unsigned nxt2 = (nxt != 0xffffffffu) ? fetch() : 0xffffffffu;
    const unsigned t0 = cur * pg.unit_tiles;
    const unsigned t1 = min(t0 + pg.unit_tiles, pg.tiles);
    for (unsigned tile = t0; tile < t1; ++tile) {
      const unsigned n = tile / per_img;
      const unsigned rem = tile - n * per_img;
      const unsigned hp = rem / pg.tiles_per_row;
      const unsigned wi = rem - hp * pg.tiles_per_row;
      const unsigned a = (n * pg.h + 2u * hp) * row_v + wi * count;   // < total_v < 2^32
      const unsigned o = ((n * pg.row_pairs + hp) * pg.ow + wi * (pg.wt / 2u)) * g.cv;
      mbar_wait(smem_u32(&r.empty[pos.slot]), pos.parity ^ 1u);
      r.meta[pos.slot].start = o;      // first OUTPUT vector of the tile
      r.meta[pos.slot].count = count;
      r.meta[pos.slot].tag = 0u;
      const unsigned bar = smem_u32(&r.full[pos.slot]);
      mbar_arrive_expect_tx(bar, count * 32u);
      bulk_load(smem_u32(stage_base + pos.slot * kStageBytes), src + a, count * 16u, bar);
      bulk_load(smem_u32(stage_base + pos.slot * kStageBytes + kPairOffset), src + a + row_v, count * 16u, bar);
      pos.next();
    }
    cur = nxt;
    nxt = nxt2;
  }
  mbar_wait(smem_u32(&r.empty[pos.slot]), pos.parity ^ 1u);
  r.meta[pos.slot].start = 0u;
  r.meta[pos.slot].count = 0u;
  r.meta[pos.slot].tag = 0u;
  mbar_arrive(smem_u32(&r.full[pos.slot]));
  pos.next();
}

// acc.pooled(a0, a1, b0, b1, out_vector) for the one output vector this thread owns in every tile
template <typename Acc>
__device__ __forceinline__ void consume_pool_phase(const FlatGeo& g, const PoolGeo& pg, BulkRing& r, const unsigned char* stage_base,
                                                   RingPos& pos, Acc& acc) {
  const unsigned t = threadIdx.x;
  const bool lane0 = (t & 31u) == 0u;
  const bool mine = t < (pg.wt / 2u) * g.cv;
  const unsigned j = t / g.cv, col = t - j * g.cv;
  const unsigned my = smem_u32(stage_base) + ((2u * j) * g.cv + col) * 16u;
  const unsigned nxt = g.cv * 16u;
  for (;;) {
    mbar_wait(smem_u32(&r.full[pos.slot]), pos.parity);
    const StageMeta m = r.meta[pos.slot];
    if (m.count != 0u && mine) {
      const unsigned addr = my + pos.slot * kStageBytes;
      float4 a0, a1, b0, b1;
      lds_vec(addr, a0);
      lds_vec(addr + nxt, a1);
      lds_vec(addr + kPairOffset, b0);
      lds_vec(addr + kPairOffset + nxt, b1);
      acc.pooled(a0, a1, b0, b1, m.start + t);
    }
    __syncwarp();
    if (lane0) mbar_arrive(smem_u32(&r.empty[pos.slot]));
    pos.next();
    if (m.count == 0u) break;
  }
}

// ---- consumer side (512 threads) -----------------------------------------------------------------------------------------
// acc.consume(x, v) for every vector this thread owns (v = its index from the tensor base) and acc.stage_end(meta) once per
// stage (where accumulators fold their fp32 partial sums into float64 every few stages), until the end marker.
template <typename Acc>
__device__ __forceinline__ void consume_phase(const FlatGeo& g, BulkRing& r, const unsigned char* stage_base, RingPos& pos,
                                              Acc& acc) {
  const unsigned t = threadIdx.x;
  const bool lane0 = (t & 31u) == 0u;
  const unsigned my = smem_u32(stage_base) + t * 16u;
  const unsigned step = g.stride * 16u;
  for (;;) {
    mbar_wait(smem_u32(&r.full[pos.slot]), pos.parity);
    const StageMeta m = r.meta[pos.slot];
    const unsigned addr = my + pos.slot * kStageBytes;
    if (m.count == g.stage_v) {  // whole stage (CTA-uniform): no guards
      if (t < g.stride) {
        float4 x[kStageVec];
#pragma unroll
        for (int i = 0; i < kStageVec; ++i) lds_vec(addr + i * step, x[i]);
#pragma unroll
        for (int i = 0; i < kStageVec; ++i) acc.consume(x[i], m.start + t + i * g.stride);
      }
    } else if (m.count != 0u) {
#pragma unroll
      for (int i = 0; i < kStageVec; ++i) {
        const unsigned idx = t + i * g.stride;
        if (t < g.stride && idx < m.count) {
          float4 x;
          lds_vec(addr + i * step, x);
          acc.consume(x, m.start + idx);
        }
      }
    }
    acc.stage_end(m);
    __syncwarp();
    if (lane0) mbar_arrive(smem_u32(&r.empty[pos.slot]));
    pos.next();
    if (m.count == 0u) break;
  }
}

// PAIR streams (see produce_phase): acc.consume2(x, r, v) with r the vector of the second tensor at the same index.
template <typename Acc>
__device__ __forceinline__ void consume_pair_phase(const FlatGeo& g, BulkRing& r, const unsigned char* stage_base, RingPos& pos,
                                                   Acc& acc) {
  static_assert(kStageVec % 2u == 0u, "a pair stage is split in two halves");
  constexpr int kHalf = kStageVec / 2;
  const unsigned t = threadIdx.x;
  const bool lane0 = (t & 31u) == 0u;
  const unsigned my = smem_u32(stage_base) + t * 16u;
  const unsigned step = g.stride * 16u;
  for (;;) {
    mbar_wait(smem_u32(&r.full[pos.slot]), pos.parity);
    const StageMeta m = r.meta[pos.slot];
    const unsigned addr = my + pos.slot * kStageBytes;
    if (m.count == g.stage_v) {
      if (t < g.stride) {
        float4 x[kHalf], y[kHalf];
#pragma unroll
        for (int i = 0; i < kHalf; ++i) {
          lds_vec(addr + i * step, x[i]);
          lds_vec(addr + kPairOffset + i * step, y[i]);
        }
#pragma unroll
        for (int i = 0; i < kHalf; ++i) acc.consume2(x[i], y[i], m.start + t + i * g.stride);
      }
    } else if (m.count != 0u) {
#pragma unroll
      for (int i = 0; i < kHalf; ++i) {
        const unsigned idx = t + i * g.stride;
        if (t < g.stride && idx < m.count) {
          float4 x, y;
          lds_vec(addr + i * step, x);
          lds_vec(addr + kPairOffset + i * step, y);
          acc.consume2(x, y, m.start + idx);
        }
      }
    }
    acc.stage_end(m);
    __syncwarp();
    if (lane0) mbar_arrive(smem_u32(&r.empty[pos.slot]));
    pos.next();
    if (m.count == 0u) break;
  }
}

}  // namespace fqb
