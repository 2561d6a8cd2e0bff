// fqb200 device-side building blocks (sm_90a).  Header-only, included by fqb200.cu.
//
// Design notes (see DESIGN.md):
//  * the hot path is HBM-bound elementwise + reduction work on fp32 NCHW tensors: no tensor cores.
//  * every global access to the tensor is a 128-bit vector (scalar only when H*W is not a multiple of 4),
//    issued UNROLL-deep per thread so ~64 KB per SM are in flight.
//  * one persistent cooperative kernel walks the tensor up to three times (statistics, deviations, apply);
//    phases are separated by a hand-written grid barrier whose last-arriving CTA runs the O(C) parameter solve.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace fqb {

constexpr int kThreads = 512;           // CTA size of every kernel here
constexpr int kWarps = kThreads / 32;
constexpr int kCtasPerSm = 2;           // __launch_bounds__(512, 2): <= 64 registers per thread
constexpr int kUnroll = 4;              // independent 128-bit loads in flight per thread

// CTA-wide barrier over the kThreads = 512 worker threads: named barrier 1 with an explicit count, so that kernels which
// add a producer warp (fq_bulk.cuh: 544 threads) can share every helper below - the producer warp never joins.  In the
// plain 512-thread kernels it is equivalent to __syncthreads().
__device__ __forceinline__ void cta_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kThreads) : "memory"); }

// ------------------------------------------------------------------------------------------------
// global memory access
// ------------------------------------------------------------------------------------------------
// Tensor reads: coherent (the buffer may be written in place later in the same launch), no L1 allocation
// (each byte is used once per phase; L2 - 50 MB on an H100 - is what carries reuse between phases).
__device__ __forceinline__ float4 ld_tensor(const float4* p) {
  float4 v;
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p));
  return v;
}
__device__ __forceinline__ float ld_tensor(const float* p) {
  float v;
  asm volatile("ld.global.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}
// Tensor writes: streaming (evict-first) so the output does not push the input out of L2.
__device__ __forceinline__ void st_tensor(float4* p, const float4& v) { __stcs(p, v); }
__device__ __forceinline__ void st_tensor(float* p, float v) { __stcs(p, v); }

// Workspace traffic between CTAs goes through L2 only.
template <typename T>
__device__ __forceinline__ T ld_ws(const T* p) { return __ldcg(p); }
template <typename T>
__device__ __forceinline__ void st_ws(T* p, T v) { __stcg(p, v); }

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_u32(unsigned* p, unsigned v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// ------------------------------------------------------------------------------------------------
// NaN-propagating min / max (torch.clamp / torch.min / torch.max semantics) and C fminf/fmaxf
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float min_nan(float a, float b) {
  float r;
  asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ float max_nan(float a, float b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

// ------------------------------------------------------------------------------------------------
// exact fp32 division by a CTA-uniform divisor
// ------------------------------------------------------------------------------------------------
// q = RN(x / s) with r = RN(1/s) precomputed once per item: one FMUL + two FFMA instead of the ~10
// instruction MUFU.RCP/Newton/FCHK sequence nvcc emits per element.  (Markstein: with r the correctly
// rounded reciprocal and the remainder formed exactly by FMA, the corrected quotient is the correctly
// rounded one; tests/test_gpu_parity.py::test_division_is_ieee checks it against __fdiv_rn on 2^28 pairs.)
// Outside the exponent window where the remainder is exact (huge / inf / NaN quotients) the value is
// clamped away by the caller, so the uncorrected product is returned.
struct Divisor {
  float s;     // divisor
  float r;     // RN(1/s)
  bool fast;   // s in a range where the 3-instruction sequence is exact
};
__device__ __forceinline__ Divisor make_divisor(float s) {
  Divisor d;
  d.s = s;
  d.r = __frcp_rn(s);
  float a = fabsf(s);
  d.fast = (a > 1e-30f) && (a < 1e30f);
  return d;
}
// FAST is the hoisted, CTA-uniform `d.fast`: the caller picks the loop version once per segment.
template <bool FAST>
__device__ __forceinline__ float div_exact(float x, const Divisor& d) {
  if (!FAST) return __fdiv_rn(x, d.s);
  float q0 = __fmul_rn(x, d.r);
  float rem = __fmaf_rn(-q0, d.s, x);
  float q = __fmaf_rn(rem, d.r, q0);
  // |q0| tiny: rem may have underflowed, but then |x/s| << 0.5 and any value that small rounds the same way
  // after "+ zero_point"; |q0| huge or non-finite: clamped by the caller.
  return (fabsf(q0) < 1e30f) ? q : q0;
}

// round-half-even of t in [0, 2^22): two full-rate FADDs instead of FRND
__device__ __forceinline__ float rint_small_nonneg(float t) {
  const float magic = 8388608.0f;  // 2^23
  return __fsub_rn(__fadd_rn(t, magic), magic);
}

// ------------------------------------------------------------------------------------------------
// reductions
// ------------------------------------------------------------------------------------------------
template <typename T, typename Op>
__device__ __forceinline__ T warp_reduce(T v, Op op) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
struct OpAdd {
  template <typename T>
  __device__ __forceinline__ T operator()(T a, T b) const { return a + b; }
};
struct OpMin {
  __device__ __forceinline__ float operator()(float a, float b) const { return fminf(a, b); }
};
struct OpMax {
  __device__ __forceinline__ float operator()(float a, float b) const { return fmaxf(a, b); }
};

// Block-wide reduction, result broadcast to every thread; fixed combination order (deterministic).
// `scratch` holds kWarps elements of T in shared memory.
template <typename T, typename Op>
__device__ __forceinline__ T block_reduce(T v, Op op, T* scratch) {
  v = warp_reduce(v, op);
  cta_sync();
  if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = v;
  cta_sync();
  T r = scratch[0];
#pragma unroll
  for (int w = 1; w < kWarps; ++w) r = op(r, scratch[w]);
  return r;
}

// ------------------------------------------------------------------------------------------------
// grid barrier with a leader section
// ------------------------------------------------------------------------------------------------
// Three words in the workspace, zero between launches.  `arrive` counts CTA arrivals monotonically
// (epoch e completes at e*gridDim.x), `release` publishes the last completed epoch, `exited` lets the
// last CTA to leave zero all three again.  Co-residency comes from cudaLaunchCooperativeKernel.
struct GridSync {
  unsigned arrive;
  unsigned release;
  unsigned exited;
  unsigned launch_count;     // channels-last kernels: completed launches (accumulator bank = parity; tag of aux_ready)
  unsigned unit_counter[8];  // one dynamic work counter per streaming phase
  unsigned aux_ready;        // channels-last kernels: CTA 0 published the per-channel bit widths of launch `aux_ready`
  unsigned pad[3];
};

// All threads of all CTAs call this.  Returns true in exactly one CTA (the last to arrive) WITHOUT
// waiting: that CTA runs the serial section and then calls grid_release().  Every other CTA returns
// false only after the leader has released the epoch.
__device__ __forceinline__ bool grid_arrive(GridSync* gs, unsigned& epoch, int* sh_flag) {
  ++epoch;
  cta_sync();
  if (threadIdx.x == 0) {
    __threadfence();  // publish this CTA's workspace writes (cumulative over the bar.sync above)
    unsigned prev = atomicAdd(&gs->arrive, 1u);
    *sh_flag = (prev + 1u == epoch * gridDim.x) ? 1 : 0;
  }
  cta_sync();
  const bool lead = (*sh_flag != 0);
  if (lead) {
    __threadfence();  // acquire side: see every other CTA's writes
  } else {
    if (threadIdx.x == 0) {
      while (ld_acquire_u32(&gs->release) < epoch) __nanosleep(100);
      __threadfence();
    }
    cta_sync();
  }
  return lead;
}
__device__ __forceinline__ void grid_release(GridSync* gs, unsigned epoch) {
  cta_sync();
  if (threadIdx.x == 0) {
    __threadfence();
    st_release_u32(&gs->release, epoch);
  }
}
__device__ __forceinline__ void grid_exit(GridSync* gs) {
  cta_sync();
  if (threadIdx.x == 0) {
    unsigned prev = atomicAdd(&gs->exited, 1u);
    if (prev + 1u == gridDim.x) {  // everyone is past the last wait: safe to re-arm
      gs->arrive = 0u;
      gs->release = 0u;
      for (int i = 0; i < 8; ++i) gs->unit_counter[i] = 0u;
      __threadfence();
      gs->exited = 0u;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// geometry: the tensor as [outer][groups][inner], cut into work units handed out dynamically
// ------------------------------------------------------------------------------------------------
// The vectors of every group are enumerated in (outer, inner) order: v in [0, group_v).  A work UNIT is the p-th
// 1/P share of one group: unit u = p * G + g covers v in [group_v*p/P, group_v*(p+1)/P) of group g.  Units are
// statically defined (so every partial result is reproducible bit for bit) but DYNAMICALLY assigned: CTAs pull the
// next unit id from an atomic counter.  With equal static shares the CTAs of a bandwidth-bound phase finish at
// visibly different times (memory arbitration is not fair), and the tail runs at a fraction of the HBM bandwidth;
// pulling small units instead ends every phase within one unit time.
// Consecutive ids are neighbouring channels of the same batch slab, so what the CTAs touch concurrently is a
// nearly contiguous window of memory.  Every unit leaves one partial at slot u.
//
// Rows whose length is not a multiple of 4 floats (7x7 feature maps: 49) are walked with 128-bit accesses as well:
// `bundle` (2 or 4) consecutive channels form one streaming group whose row IS 16-byte aligned (4 x 49 floats =
// 49 vectors), and the CTA stride is cut down to the largest multiple of that row length, so that every thread
// always sits on the same column of the row: the channel(s) its four floats belong to never change.
struct Geometry {
  unsigned groups;          // streaming groups: channels / bundle
  unsigned channels;        // G of the descriptor (what the statistics / parameters are indexed by)
  unsigned bundle;          // channels per streaming group: 1, or 2 / 4 when inner % 4 != 0
  unsigned stride;          // threads that walk a unit: kThreads, or the largest multiple of inner_v below it (bundled)
  unsigned parts;           // P
  unsigned units;           // P * groups
  unsigned inner_v;         // vectors per row of a streaming group
  unsigned step_q, step_r;  // stride / inner_v, stride % inner_v
  unsigned red_lanes;       // lanes per group in the leader's partial reductions (power of two <= 32)
  unsigned part_v;          // vectors per part: ceil(group_v / P) (the last part of a group may be shorter)
  unsigned long long group_v;    // outer * inner_v: vectors per group (< 2^32, checked by the host)
  unsigned long long row_pitch;  // groups * inner_v: vectors between consecutive outer slices of a group
};

template <int VEC> struct VecT;
template <> struct VecT<4> { using type = float4; };
template <> struct VecT<1> { using type = float; };

// ------------------------------------------------------------------------------------------------
// the streaming engine: dynamic units through a per-thread ring of cp.async (LDGSTS) copies
// ------------------------------------------------------------------------------------------------
// Registers cap how many loads a thread can keep in flight (64 registers -> 4 x 128 bit).  cp.async writes the
// loaded vector straight into shared memory, so the ring can be D deep at no register cost: with D = 8 and 32 warps
// per SM, 128 KB per SM are in flight.  Every thread reads back only its own slots, so the ring itself needs no CTA
// barrier; completion is tracked with cp.async groups (exactly one group per ring step, in order).
//
// The ring does not drain at unit boundaries: the issue side runs ahead into the next unit while the consume side
// finishes the current one, so the only per-unit cost is the CTA-wide combine of the accumulators.  Unit ids are
// fetched two units ahead by thread 0 (atomicAdd; the reply is only consumed at the end of the unit, so its latency
// is hidden) and published through shared memory at the per-unit barrier.
constexpr int kRingDepth = 8;
template <int VEC>
constexpr int ring_bytes() { return kRingDepth * kThreads * 4 * VEC; }  // dynamic shared memory per CTA

__device__ __forceinline__ void cp_async_vec(unsigned smem_addr, const float4* gptr) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_addr), "l"(gptr) : "memory");
}
__device__ __forceinline__ void cp_async_vec(unsigned smem_addr, const float* gptr) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_addr), "l"(gptr) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void lds_vec(unsigned smem_addr, float4& v) {
  asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(smem_addr) : "memory");
}
__device__ __forceinline__ void lds_vec(unsigned smem_addr, float& v) {
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(smem_addr) : "memory");
}

struct StreamSmem {
  unsigned ids[4];  // unit-id queue, indexed by (sequence number of the unit within this CTA) % 4
};

// (row, column) cursor over the vectors thread t visits in a unit: t, t+S, t+2S, ... (REV: from the end backwards)
struct Cursor {
  unsigned j, off;
};
template <bool REV>
__device__ __forceinline__ void cursor_step(const Geometry& geo, Cursor& c) {
  const unsigned adv = static_cast<unsigned>(geo.step_q * geo.row_pitch + geo.step_r);
  const unsigned wrap = static_cast<unsigned>(geo.row_pitch - geo.inner_v);
  if (!REV) {
    c.j += geo.step_r;
    c.off += adv;
    if (c.j >= geo.inner_v) {
      c.j -= geo.inner_v;
      c.off += wrap;
    }
  } else {
    c.off -= adv;
    if (c.j < geo.step_r) {
      c.j += geo.inner_v;
      c.off -= wrap;
    }
    c.j -= geo.step_r;
  }
}

struct UnitInfo {
  unsigned g;      // streaming group
  unsigned p;      // part
  unsigned mine;   // vectors this thread visits
  unsigned trips;  // ring steps of this thread's WARP (= `mine` of its first lane): warp-uniform loop count
  Cursor start;    // this thread's first vector
};
template <bool REV>
__device__ __forceinline__ UnitInfo unit_info(const Geometry& geo, unsigned u) {
  UnitInfo ui;
  ui.p = u / geo.groups;
  ui.g = u - ui.p * geo.groups;
  const unsigned gv = static_cast<unsigned>(geo.group_v);
  const unsigned vb = ui.p * geo.part_v;  // 32-bit: group_v < 2^32
  const unsigned len = min(geo.part_v, gv - vb);
  const unsigned S = geo.stride;
  const unsigned t = threadIdx.x, t0 = threadIdx.x & ~31u;
  ui.mine = (t < len && t < S) ? (len - t + S - 1u) / S : 0u;
  ui.trips = (t0 < len && t0 < S) ? (len - t0 + S - 1u) / S : 0u;
  const unsigned v0 = (ui.mine == 0) ? vb : (REV ? vb + (len - 1u - t) : vb + t);
  const unsigned a0 = v0 / geo.inner_v;
  ui.start.j = v0 - a0 * geo.inner_v;
  ui.start.off = static_cast<unsigned>(a0 * geo.row_pitch) + ui.g * geo.inner_v + ui.start.j;
  return ui;
}

// Stream every unit this CTA manages to pull through `acc`:
//   acc.begin(ui)           unit starts (load per-group constants, reset accumulators); ui.start.j is the thread's column
//   acc.consume(x, off, j)  one vector (off = its index from the tensor base, j = its column in the row, in vectors)
//   acc.end(ui)             unit done: CTA-wide combine + partial store; MUST contain at least one __syncthreads()
// `counter` is this phase's unit counter in the workspace (zero at launch), or nullptr for a static round-robin
// assignment (ticket k of CTA b = b + k * gridDim.x; used by the workspace-free given-parameter kernel).
// REV walks ids and vectors backwards.
template <int VEC, bool REV, typename Acc>
__device__ __forceinline__ void stream_units(const Geometry& geo, const float* base, unsigned* counter, StreamSmem& ss,
                                             Acc& acc) {
  using V = typename VecT<VEC>::type;
  constexpr int D = kRingDepth;
  constexpr unsigned kSlot = kThreads * 4u * VEC;  // bytes between consecutive ring slots of one thread
  const V* src = reinterpret_cast<const V*>(base);
  extern __shared__ __align__(16) unsigned char fq_ring[];
  const unsigned ring = static_cast<unsigned>(__cvta_generic_to_shared(fq_ring)) + threadIdx.x * (4u * VEC);
  const unsigned total = geo.units;
  auto unit_of = [&](unsigned ticket) { return REV ? total - 1u - ticket : ticket; };
  unsigned fetched = 0;  // thread 0: tickets taken so far (static mode)
  // the first two tickets of every CTA are static (b, b + grid): no atomic round trips before the first load;
  // from the third on they come from the phase counter (offset by the 2 * grid tickets dealt statically)
  auto take_ticket = [&]() -> unsigned {
    const unsigned k = fetched++;
    if (counter && k >= 2u) {
      const unsigned long long t = 2ull * gridDim.x + atomicAdd(counter, 1u);
      return t < total ? static_cast<unsigned>(t) : 0xffffffffu;
    }
    const unsigned long long t = blockIdx.x + static_cast<unsigned long long>(k) * gridDim.x;
    return t < total ? static_cast<unsigned>(t) : 0xffffffffu;
  };

  cta_sync();  // ss.ids may still be read by stragglers of a previous phase
  if (threadIdx.x == 0) {
    ss.ids[0] = take_ticket();
    ss.ids[1] = take_ticket();
  }
  cta_sync();
  unsigned seq = 0;  // sequence number (within this CTA) of the unit being consumed
  unsigned ticket = ss.ids[0];
  if (ticket >= total) return;

  // consume side
  UnitInfo cu = unit_info<REV>(geo, unit_of(ticket));
  Cursor cc = cu.start;
  unsigned cdone = 0;  // ring steps done in the consumed unit
  acc.begin(cu);
  // issue side (at most one unit ahead: that is as far as ss.ids is guaranteed visible)
  unsigned iseq = 0;
  UnitInfo iu = cu;
  UnitInfo ahead = cu;  // the unit the issue side entered last (handed to the consume side when it gets there)
  Cursor ic = cu.start;
  unsigned idone = 0;
  bool iexhausted = false;
  unsigned bubbles = 0;  // bit d: ring slot d carries no ring step (the issue side could not advance)
  unsigned pending = 0;  // thread 0: ticket fetched during this unit, published at its end

  // one ring step into `slot`; returns false when it had to leave a bubble
  auto issue_step = [&](unsigned slot) -> bool {
    while (!iexhausted && idone == iu.trips) {
      if (iseq > seq) break;
      const unsigned t = ss.ids[(iseq + 1u) & 3u];
      if (t >= total) {
        iexhausted = true;
        break;
      }
      ++iseq;
      iu = unit_info<REV>(geo, unit_of(t));
      ahead = iu;
      ic = iu.start;
      idone = 0;
    }
    bool real = false;
    if (!iexhausted && idone < iu.trips) {
      if (idone < iu.mine) {
        cp_async_vec(ring + slot * kSlot, src + ic.off);
        cursor_step<REV>(geo, ic);
      }
      ++idone;
      real = true;
    }
    cp_async_commit();  // exactly one group per ring step, empty or not
    return real;
  };

  // prologue: fill the ring
#pragma unroll
  for (int d = 0; d < D; ++d)
    if (!issue_step(d)) bubbles |= 1u << d;
  unsigned head = 0;
  if (threadIdx.x == 0) pending = take_ticket();

  for (;;) {
    if (cdone == cu.trips) {
      // ---- unit boundary
      if (threadIdx.x == 0) ss.ids[(seq + 2u) & 3u] = pending;  // visible after the barrier inside end()
      acc.end(cu);
      ++seq;
      ticket = ss.ids[seq & 3u];
      if (ticket >= total) break;
      if (threadIdx.x == 0) pending = take_ticket();
      cu = (iseq == seq) ? ahead : unit_info<REV>(geo, unit_of(ticket));  // usually the issue side is already there
      cc = cu.start;
      cdone = 0;
      acc.begin(cu);
      continue;
    }
    // ---- steady state: for the next n ring steps every lane of this warp both consumes and issues a real vector
    // and no slot is a bubble, so none of the bookkeeping below is needed (the loop is issue-bound: DESIGN.md).
    // All the quantities involved are warp-uniform except `mine`, hence the warp-wide minimum.
    if (bubbles == 0u && !iexhausted) {
      const unsigned nc = cu.mine > cdone ? cu.mine - cdone : 0u;
      const unsigned ni = iu.mine > idone ? iu.mine - idone : 0u;
      const unsigned n = __reduce_min_sync(0xffffffffu, min(nc, ni));
      if (n >= 2u) {
        for (unsigned k = 0; k < n; ++k) {
          cp_async_wait<D - 1>();
          V x;
          lds_vec(ring + head * kSlot, x);
          cp_async_vec(ring + head * kSlot, src + ic.off);
          cp_async_commit();
          cursor_step<REV>(geo, ic);
          head = (head + 1u) & (D - 1u);
          acc.consume(x, cc.off, cc.j);
          cursor_step<REV>(geo, cc);
        }
        cdone += n;
        idone += n;
        continue;
      }
    }
    cp_async_wait<D - 1>();  // the oldest group (slot `head`) has landed
    const bool bubble = (bubbles >> head) & 1u;
    const bool active = !bubble && cdone < cu.mine;
    V x;
    if (active) lds_vec(ring + head * kSlot, x);
    if (issue_step(head))
      bubbles &= ~(1u << head);
    else
      bubbles |= 1u << head;
    head = (head + 1u) & (D - 1u);
    if (active) {
      acc.consume(x, cc.off, cc.j);
      cursor_step<REV>(geo, cc);
    }
    if (!bubble) ++cdone;
  }
  cp_async_wait<0>();
}

}  // namespace fqb
