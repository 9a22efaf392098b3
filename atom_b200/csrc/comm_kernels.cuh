// comm_kernels.cuh -- one-shot "push" all-reduce over NVLink peer memory for the tensor-parallel layers.
//
// The row-parallel projections (o_proj, down_proj) of a decode step leave an FP16 [batch, hidden] partial on every rank
// (512 KiB at Llama-65B, batch 32) that must be summed across the ranks: a latency-bound collective (SURVEY.md 8e).
// The reference has no multi-GPU code at all.  This kernel does the exchange itself, with
// no flag round trip and no fence (Lamport-style: the payload is its own arrival signal):
//   1. every CTA pushes its slice of the local partial into slot [e % 3][my rank] of EVERY rank's receive buffer (plain
//      16-byte stores through the NVLink peer mappings: fire and forget).  Receive buffers are pre-filled with a sentinel
//      bit pattern (FP16 -0.0 = 0x8000) that the payload never contains: a -0.0 input is sent as +0.0, which leaves every
//      sum unchanged except that an all-(-0.0) column yields +0.0;
//   2. it resets ITS OWN buffer [(e + 2) % 3] -- the one read in the previous call -- to the sentinel for a later call;
//   3. it polls the `world` slots of its slice in LOCAL memory until no 16-byte chunk holds a sentinel half (a torn write
//      just keeps it polling), sums them in rank order in FP32 (identical on every rank) and writes the FP16 result.
// Three buffers rotate on a device-side call counter (published by the last CTA of the consuming kernel), so the kernel is CUDA-graph capturable and needs no barrier: a peer
// can write buffer e % 3 again only in call e + 3, which it reaches after my push of call e + 2, i.e. after I finished
// call e; and buffer (e + 2) % 3 is not written by anybody before call e + 2, which every peer reaches only after my push
// of call e + 1, i.e. after the reset of call e completed (kernel boundary).
// The two halves also exist fused into their neighbours (tp.py): the row-parallel decode GEMM pushes from its epilogue
// (gemm_i4_sm90.cuh, GemmArgs::ar) and rmsnorm_quant_kernel reduces while it loads its row (quant_kernels.cuh);
// the shared pieces live in ptx_sm90.cuh (ArArgs, ar_*).
#pragma once
#include "ptx_sm90.cuh"

namespace atom {

constexpr int AR_CTAS = 64, AR_THREADS = 256;

// in, out: f16 [numel] local.  numel % 8 == 0, numel <= ar.slot.
__global__ void __launch_bounds__(AR_THREADS)
allreduce_push_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, ArArgs ar, long long nchunks) {
  const int tid = threadIdx.x, bid = blockIdx.x;
  const uint32_t e = ar_ld_state(ar.state) + 1, cur = e % 3;
  const long long slot_chunks = ar.slot / 8;
  const long long per = (nchunks + gridDim.x - 1) / gridDim.x;
  const long long lo = min((long long)bid * per, nchunks), hi = min(lo + per, nchunks);
  // 1. push my slice into slot [cur][rank] of every rank (my own included: the reduction below is then uniform)
  for (long long i = lo + tid; i < hi; i += AR_THREADS) {
    uint4 v = in[i];
    v.x = ar_strip_sentinel(v.x); v.y = ar_strip_sentinel(v.y); v.z = ar_strip_sentinel(v.z); v.w = ar_strip_sentinel(v.w);
    for (int r = 0; r < ar.world; ++r)      // destinations staggered by rank: no two ranks start on the same peer
      ar_st_v4(reinterpret_cast<uint4*>(ar.bufs[(ar.rank + r) % ar.world]) + ((long long)cur * ar.world + ar.rank) * slot_chunks + i, v);
  }
  // 2. reset the buffer of the previous call
  ar_reset_previous(ar, e, bid, gridDim.x, tid, AR_THREADS);
  // 3. poll + reduce in rank order from local memory
  const uint4* local = reinterpret_cast<const uint4*>(ar.bufs[ar.rank]) + (long long)cur * ar.world * slot_chunks;
  unsigned long long t0 = 0;
  for (long long i = lo + tid; i < hi; i += AR_THREADS) out[i] = ar_reduce_chunk(local, slot_chunks, i, ar.world, t0);
  __syncthreads();
  if (tid == 0) ar_complete(ar, e, nchunks, gridDim.x);
}

}  // namespace atom
