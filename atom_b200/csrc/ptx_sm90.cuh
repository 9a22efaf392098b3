// ptx_sm90.cuh -- thin inline-PTX wrappers for the sm_90a features the kernels use:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (INT8, A from registers), clusters.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace atom {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// try_wait with a suspend-time hint: the thread sleeps in hardware until the phase completes (or ~the hint elapses)
// instead of burning issue slots in a software spin loop.  kCluster: acquire at cluster scope, for a phase completed by
// other CTAs of the cluster (st.async into this CTA's shared memory).
template <bool kCluster = false>
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  if constexpr (kCluster) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity), "r"(20000u)
        : "memory");
  } else {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity), "r"(20000u)
        : "memory");
  }
  return ok != 0;
}
// A pipeline bug must not hang the GPU: after ~4 s the waiting thread traps, turning a deadlock into a launch error.  The
// clock is only consulted every 64 unsuccessful probes.  -DATOM_MBAR_DEBUG adds a diagnostic message for debugging.
#ifndef ATOM_MBAR_TIMEOUT_CYCLES
#define ATOM_MBAR_TIMEOUT_CYCLES (8000000000ll)
#endif
#ifdef ATOM_MBAR_DEBUG
__device__ __noinline__ void mbar_timeout(uint64_t* bar, uint32_t parity) {
  printf("atom_b200: mbarrier wait timed out: block (%d,%d,%d) thread %d smem 0x%x parity %u\n", blockIdx.x, blockIdx.y,
         blockIdx.z, threadIdx.x, smem_u32(bar), parity);
  __trap();
}
#else
__device__ __forceinline__ void mbar_timeout(uint64_t*, uint32_t) { asm volatile("trap;"); }
#endif
template <bool kCluster = false>
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait<kCluster>(bar, parity)) return;
  long long t0 = 0;
  uint32_t spins = 0;
  while (!mbar_try_wait<kCluster>(bar, parity)) {
    if ((++spins & 63u) == 0) {
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > ATOM_MBAR_TIMEOUT_CYCLES) mbar_timeout(bar, parity);
    }
  }
}

// ------------------------------------------------------------------ proxies / fences
// generic-proxy smem writes -> visible to the async proxy (TMA, wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ------------------------------------------------------------------ TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tile load global -> this CTA's smem, completion signalled on `bar` (complete_tx::bytes)
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// ------------------------------------------------------------------ wgmma (warpgroup MMA)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D[regs] (+)= A[regs] * B[smem desc], INT8 x INT8 -> INT32, one warpgroup, tile 64 x N x 32.  A is the m16n8k32 fragment of
// each warp's 16 rows (a0: row g, k 4q..4q+3; a1: row g+8; a2 / a3: the same rows, k + 16; g = lane / 4, q = lane % 4);
// D[4j + {0,1}] = (row g, columns 8j + 2q + {0,1}), D[4j + {2,3}] = row g + 8.  One overload per N (= 2 x registers of D).
__device__ __forceinline__ void wgmma_s8_rs(uint32_t (&d)[8], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %13, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k32.s32.s8.s8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, "
      "{%8, %9, %10, %11}, %12, p;\n\t}"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(desc_b), "r"(accumulate)
      : "memory");
}
__device__ __forceinline__ void wgmma_s8_rs(uint32_t (&d)[16], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "{%16, %17, %18, %19}, %20, p;\n\t}"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(desc_b), "r"(accumulate)
      : "memory");
}
__device__ __forceinline__ void wgmma_s8_rs(uint32_t (&d)[32], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, p;\n\t}"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(desc_b), "r"(accumulate)
      : "memory");
}
__device__ __forceinline__ void wgmma_s8_rs(uint32_t (&d)[64], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "{%64, %65, %66, %67}, %68, p;\n\t}"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(desc_b), "r"(accumulate)
      : "memory");
}

// K-major, SWIZZLE_128B operand descriptor: start>>4 [0,14) | LBO>>4 [16,30) (=1, unused for swizzled K-major) |
// SBO>>4 [32,46) (=1024 B between 8-row atoms) | swizzle mode [62,64) = 1 (128 B).  Tiles are 1024-B aligned (base offset 0).
__device__ __forceinline__ uint64_t wgmma_desc_k_sw128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}

// ------------------------------------------------------------------ clusters / DSMEM
__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ uint32_t cluster_nctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_arrive_relaxed() { asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ uint32_t mapa_shared(uint32_t addr, uint32_t rank) {
  uint32_t r; asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank)); return r;
}
__device__ __forceinline__ float4 ld_dsmem_v4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
}
// 8 bytes from registers into a cluster CTA's shared memory at `addr`; the write completes 8 bytes of transaction count on
// that CTA's mbarrier `bar` (both addresses from mapa_shared).  Nothing of the sender's shared memory is read.
__device__ __forceinline__ void st_async_v2(uint32_t addr, float x, float y, uint32_t bar) {
  asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.v2.f32 [%0], {%1, %2}, [%3];"
               ::"r"(addr), "f"(x), "f"(y), "r"(bar) : "memory");
}
__device__ __forceinline__ float2 ld_dsmem_v2(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared::cluster.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr) : "memory");
  return v;
}

// ------------------------------------------------------------------ programmatic dependent launch (PDL)
// launch_dependents: the next kernel in the stream (if it was launched with the programmatic-serialization attribute) may
// start its prologue once every CTA of this grid has executed this (or exited).  wait: blocks until the preceding grid has
// completed and its memory operations are visible; without a programmatic dependency both are no-ops.
__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ------------------------------------------------------------------ misc
// L2-coherent loads (bypass L1) for data written by the PRECEDING kernel: under programmatic dependent launch this
// kernel's CTAs share an SM (and its L1) with CTAs that were running before that data was produced
__device__ __forceinline__ uint4 ld_cg_v4(const void* p) {
  uint4 v;
  asm volatile("ld.global.cg.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned short ld_cg_u16(const void* p) {
  unsigned short v;
  asm volatile("ld.global.cg.u16 %0, [%1];" : "=h"(v) : "l"(p) : "memory");
  return v;
}

// ---------------------------------------------------------------- push all-reduce (comm_kernels.cuh) state shared with
// the kernels that fuse its two halves: the row-parallel GEMM pushes its partial straight into the peers' receive buffers,
// the following add+RMSNorm+quantise kernel reduces them (tp.py).  bufs[r]: rank r's receive buffer, f16 [3][world][slot],
// sentinel-filled (0x8000); state (local u32): [0] completed calls, [1] ticket, [2..4] chunks last written per buffer.
struct ArArgs {
  void* const* bufs;
  uint32_t* state;
  long long slot;          // elements per (buffer, rank) slot
  int rank, world;
};
constexpr int AR_STATE_WORDS = 8;
__device__ __forceinline__ uint32_t ar_ld_state(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint4 ar_ld_v4(const void* p) {      // written remotely: never through L1
  uint4 v;
  asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void ar_st_v4(void* p, const uint4 v) {
  asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void ar_st_u16(void* p, unsigned short v) {
  asm volatile("st.volatile.global.u16 [%0], %1;" ::"l"(p), "h"(v) : "memory");
}
// FP16 -0.0 (0x8000) is the "not yet arrived" pattern of the receive buffers
__device__ __forceinline__ bool ar_has_sentinel(uint32_t w) { return (w & 0xFFFFu) == 0x8000u || (w >> 16) == 0x8000u; }
__device__ __forceinline__ bool ar_has_sentinel(const uint4& v) {
  return ar_has_sentinel(v.x) || ar_has_sentinel(v.y) || ar_has_sentinel(v.z) || ar_has_sentinel(v.w);
}
__device__ __forceinline__ uint32_t ar_strip_sentinel(uint32_t w) {
  if ((w & 0xFFFFu) == 0x8000u) w &= 0xFFFF0000u;
  if ((w >> 16) == 0x8000u) w &= 0x0000FFFFu;
  return w;
}
// one 16-byte chunk of the sum: the loads of up to 8 ranks' slots are in flight together (a dependent chain of `world` volatile
// loads per chunk is what an earlier revision spent most of its time in), each is re-polled until its payload is there, and the
// sum is formed in rank order in FP32
__device__ __forceinline__ uint4 ar_reduce_chunk(const uint4* local_cur, long long slot_chunks, long long i, int world, unsigned long long& t0) {
  float acc[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) acc[k] = 0.f;
  for (int r0 = 0; r0 < world; r0 += 8) {
    uint4 v[8];
#pragma unroll
    for (int x = 0; x < 8; ++x)
      if (r0 + x < world) v[x] = ar_ld_v4(local_cur + (long long)(r0 + x) * slot_chunks + i);
#pragma unroll
    for (int x = 0; x < 8; ++x) {
      if (r0 + x < world) {
        // bounded: a peer that never arrives (crashed rank, mismatched call sequence) traps after ~4 s instead of hanging the GPU
        for (uint32_t spins = 0; ar_has_sentinel(v[x]); ++spins) {
          if ((spins & 0x3FFu) == 0x3FFu) {
            unsigned long long now;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
            if (t0 == 0) t0 = now;
            else if (now - t0 > 4000000000ull) asm volatile("trap;");
          }
          v[x] = ar_ld_v4(local_cur + (long long)(r0 + x) * slot_chunks + i);
        }
        const __half2* h = reinterpret_cast<const __half2*>(&v[x]);
#pragma unroll
        for (int k = 0; k < 4; ++k) { const float2 f = __half22float2(h[k]); acc[2 * k] += f.x; acc[2 * k + 1] += f.y; }
      }
    }
  }
  uint4 o;
  __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
  for (int k = 0; k < 4; ++k) oh[k] = __floats2half2_rn(acc[2 * k], acc[2 * k + 1]);
  return o;
}
// this CTA's share of resetting the buffer of the previous call (whatever extent was written into it) to the sentinel
__device__ __forceinline__ void ar_reset_previous(const ArArgs& ar, uint32_t e, int cta, int nctas, int tid, int nthreads) {
  const uint32_t clr = (e + 2) % 3;
  const long long cchunks = (long long)ar_ld_state(ar.state + 2 + clr), slot_chunks = ar.slot / 8;
  const long long cper = (cchunks + nctas - 1) / nctas;
  const long long clo = min((long long)cta * cper, cchunks), chi = min(clo + cper, cchunks);
  const uint4 sv = make_uint4(0x80008000u, 0x80008000u, 0x80008000u, 0x80008000u);
  uint4* base = reinterpret_cast<uint4*>(ar.bufs[ar.rank]) + (long long)clr * ar.world * slot_chunks;
  for (int r = 0; r < ar.world; ++r)
    for (long long i = clo + tid; i < chi; i += nthreads) base[(long long)r * slot_chunks + i] = sv;
}
// end of a consuming kernel: the last CTA to get here publishes the call (all CTAs read state[0] when they started)
__device__ __forceinline__ void ar_complete(const ArArgs& ar, uint32_t e, long long nchunks, int nctas) {
  __threadfence();
  if (atomicAdd(ar.state + 1, 1u) == (uint32_t)nctas - 1) {
    ar.state[2 + e % 3] = (uint32_t)nchunks;
    ar.state[1] = 0;
    __threadfence();
    ar.state[0] = e;
  }
}

}  // namespace atom
