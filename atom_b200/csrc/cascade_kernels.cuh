// cascade_kernels.cuh -- shared-prefix decode: the prefix pass of the cascade decode attention.
//
// When several sequences of a decode batch were forked from one parent they begin on the same INT4 pages (kvcache.py), and
// every one of those pages is needed by members x G query rows of each KV head: a small GEMM instead of members separate
// streams.  The cascade splits each group row's attention in two:
//   * prefix pass (this kernel): grid (chunk, KV head, group x row block).  A CTA streams its chunk of the group's shared pages
//     ONCE, dequantises K and V and rotates K at its absolute positions into FP16 tiles with prefill_attn_kernel<true>'s context
//     loader (prefill_ctx_tile: the same arithmetic, the same smem layout), and runs mma.sync m16n8k16 over 64 query rows
//     (member, query head) of that KV head, with an FP32 online softmax.  Each member's q is rotated at its own position
//     len - 1, read from the page table on the device (a graph replay sees new lengths).  It leaves the un-normalised
//     (m, d, acc[128]) of every row and chunk in the FP32 workspace; groups of more than 64 rows take more CTAs, which share the
//     pages through L2.
//   * suffix pass: batch_decode_kernel<..., DecPrefix> (kv_kernels.cuh) over each row's private pages, which folds the row's
//     prefix partials in chunk order into its stripe merge.
// The chunking is fixed by the shared page count and the host-chosen chunk count, and both merges run in a fixed order, so the
// result does not depend on where the pages sit or on the call.
#pragma once
#include "prefill_kernels.cuh"

namespace atom {

// G: query heads per KV head; row_blocks: 64-row blocks per group (grid.z = groups x row_blocks); rope: (cos, sin) table of
// positions up to the longest shared prefix (ops.rope_table)
__global__ void __launch_bounds__(PF_THREADS, 2)
shared_prefix_attn_kernel(const __half* __restrict__ q, KvArgs kv, DecPrefix px, const float2* __restrict__ rope, float log2_theta,
                          int G, int row_blocks, int pdl) {
  __shared__ __align__(16) __half Ks[PF_BK * PF_KPITCH];
  __shared__ __align__(16) __half Vt[128 * PF_VPITCH];
  if (pdl) { griddep_launch_dependents(); griddep_wait(); }       // q comes from the preceding kernels
  const int chunk = blockIdx.x, hkv = blockIdx.y, grp = blockIdx.z / row_blocks, rb = blockIdx.z % row_blocks;
  const int m_begin = px.group_indptr[grp], rows = (px.group_indptr[grp + 1] - m_begin) * G;
  if (rb * PF_BQ >= rows) return;
  const int b0 = px.group_members[m_begin];
  const int prefix = px.shared_pages[b0] * kv.P;
  const int tiles = dec_prefix_tiles(px.shared_pages[b0], kv.P), per = dec_prefix_per(tiles, px.nchunks);
  const int t_begin = chunk * per, t_end = min(tiles, t_begin + per);
  if (t_begin >= t_end) return;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int Hq = kv.H * G;
  const float kFreqStep = log2_theta / 64.f;
  constexpr float kSmScale = 0.08838834764831845f * 1.4426950408889634f;   // 1/sqrt(128) * log2(e), as the decode kernel

  // ---- Q fragments of this warp's 16 rows: row r = (member r / G, query head hkv*G + r % G), rotated in FP32 at len - 1
  const int qrow0 = rb * PF_BQ + warp * 16 + g, qrow1 = qrow0 + 8;
  int brow[2], hrow[2];
  uint32_t qa[8][4];
  {
    float2 lo[2][4][2], hi[2][4][2];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int r = min(rr ? qrow1 : qrow0, rows - 1);
      const int bb = px.group_members[m_begin + r / G];
      brow[rr] = bb; hrow[rr] = hkv * G + r % G;
      const int pos = (kv.indptr[bb + 1] - kv.indptr[bb] - 1) * kv.P + kv.last_page_offset[bb] - 1;
      const __half* qr = q + ((size_t)bb * Hq + hrow[rr]) * 128;
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) {          // columns d = 16 kk + 8 hf + 2 t, d + 1 and their partners d + 64
          const int d = 16 * kk + 8 * hf + 2 * t;
          const float2 x = __half22float2(*reinterpret_cast<const __half2*>(qr + d));
          const float2 y = __half22float2(*reinterpret_cast<const __half2*>(qr + d + 64));
          float s0, c0, s1, c1;
          sincosf((float)pos * exp2f(-(float)d * kFreqStep), &s0, &c0);
          sincosf((float)pos * exp2f(-(float)(d + 1) * kFreqStep), &s1, &c1);
          lo[rr][kk][hf] = make_float2(x.x * c0 - y.x * s0, x.y * c1 - y.y * s1);
          hi[rr][kk][hf] = make_float2(y.x * c0 + x.x * s0, y.y * c1 + x.y * s1);
        }
      }
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int hf = 0; hf < 2; ++hf)
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          qa[kk][2 * hf + rr] = pack_h2(lo[rr][kk][hf].x, lo[rr][kk][hf].y);
          qa[kk + 4][2 * hf + rr] = pack_h2(hi[rr][kk][hf].x, hi[rr][kk][hf].y);
        }
  }

  // the context loader of prefill_attn_kernel<true> with the shared prefix as the "context" of member b0: a prompt of
  // seq_len - prefix tokens sees ctx = prefix, key position k0 + tok is absolute position prefix + k0 + tok
  const int L0 = (kv.indptr[b0 + 1] - kv.indptr[b0] - 1) * kv.P + kv.last_page_offset[b0] - prefix;
  const float2* rope_ctx = rope + (size_t)prefix * 64;

  float o[16][4];
#pragma unroll
  for (int i = 0; i < 16; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

  for (int kt = t_begin; kt < t_end; ++kt) {
    const int a0 = kt * PF_BK;                        // absolute position of the tile's first key
    __syncthreads();                                  // the previous tile has been consumed
    prefill_ctx_tile(kv, b0, L0, hkv, a0 - prefix, rope_ctx, Ks, Vt, tid);
    __syncthreads();

    float s[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        const uint32_t b0f = *reinterpret_cast<const uint32_t*>(&Ks[(8 * j + g) * PF_KPITCH + 16 * kk + 2 * t]);
        const uint32_t b1f = *reinterpret_cast<const uint32_t*>(&Ks[(8 * j + g) * PF_KPITCH + 16 * kk + 8 + 2 * t]);
        mma_16816(s[j], qa[kk], b0f, b1f);
      }
    }
    // scale; keys past the prefix (last tile only) are masked.  Every row sees the same keys: the first tile of the chunk
    // gives every row a finite maximum
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const bool ok = a0 + 8 * j + 2 * t + u < prefix;
        s[j][u] = ok ? s[j][u] * kSmScale : -INFINITY;
        s[j][2 + u] = ok ? s[j][2 + u] * kSmScale : -INFINITY;
        mx0 = fmaxf(mx0, s[j][u]); mx1 = fmaxf(mx1, s[j][2 + u]);
      }
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
    const float a_0 = exp2f(m0 - mn0), a_1 = exp2f(m1 - mn1);
    m0 = mn0; m1 = mn1;
    float sum0 = 0.f, sum1 = 0.f;
    uint32_t pa[4][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float p00 = exp2f(s[j][0] - mn0), p01 = exp2f(s[j][1] - mn0);
      const float p10 = exp2f(s[j][2] - mn1), p11 = exp2f(s[j][3] - mn1);
      sum0 += p00 + p01; sum1 += p10 + p11;
      pa[j >> 1][(j & 1) * 2 + 0] = pack_h2(p00, p01);
      pa[j >> 1][(j & 1) * 2 + 1] = pack_h2(p10, p11);
    }
    l0 = l0 * a_0 + sum0; l1 = l1 * a_1 + sum1;
#pragma unroll
    for (int i = 0; i < 16; ++i) { o[i][0] *= a_0; o[i][1] *= a_0; o[i][2] *= a_1; o[i][3] *= a_1; }
#pragma unroll
    for (int i = 0; i < 16; ++i) {
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint32_t b0f = *reinterpret_cast<const uint32_t*>(&Vt[(8 * i + g) * PF_VPITCH + 16 * kk + 2 * t]);
        const uint32_t b1f = *reinterpret_cast<const uint32_t*>(&Vt[(8 * i + g) * PF_VPITCH + 16 * kk + 8 + 2 * t]);
        mma_16816(o[i], pa[kk], b0f, b1f);
      }
    }
  }

  // ---- un-normalised partial of each live row: (m, d, acc[128]) at [b][h][chunk]
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    if ((rr ? qrow1 : qrow0) >= rows) continue;
    float* dst = px.part + (((size_t)brow[rr] * Hq + hrow[rr]) * px.nchunks + chunk) * DEC_PART;
    if (t == 0) *reinterpret_cast<float2*>(dst) = make_float2(rr ? m1 : m0, rr ? l1 : l0);
#pragma unroll
    for (int i = 0; i < 16; ++i)
      *reinterpret_cast<float2*>(dst + 2 + 8 * i + 2 * t) = make_float2(o[i][2 * rr], o[i][2 * rr + 1]);
  }
}

}  // namespace atom
