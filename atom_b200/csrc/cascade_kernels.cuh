// cascade_kernels.cuh -- shared-prefix decode: the prefix pass of the cascade decode attention.
//
// When several sequences of a decode batch were forked from one parent they begin on the same INT4 pages (kvcache.py), and
// every one of those pages is needed by members x G query rows of each KV head: a small GEMM instead of members separate
// streams.  The cascade splits each group row's attention in two:
//   * prefix pass (this kernel): grid (chunk, KV head, group x row block).  A CTA streams its chunk of the group's shared pages
//     ONCE, dequantises K and V and rotates K at its absolute positions into FP16 tiles with prefill_attn_kernel<true>'s context
//     loader (prefill_ctx_tile: the same arithmetic, the same smem layout), and runs the tile step (attn_tile_step) over 64
//     query rows (member, query head) of that KV head; every row sees every prefix key.  Each member's q is rotated at its own
//     position len - 1, read from the page table on the device (rope_q_frags: a graph replay sees new lengths).  It leaves the
//     un-normalised (m, d, acc[128]) of every row and chunk in the FP32 workspace; groups of more than 64 rows take more CTAs,
//     which share the pages through L2.
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
  const int tid = threadIdx.x, warp = tid >> 5, g = (tid & 31) >> 2;
  const int Hq = kv.H * G;

  // ---- Q fragments of this warp's 16 rows: row r = (member r / G, query head hkv*G + r % G), rotated at len - 1
  const int qrow0 = rb * PF_BQ + warp * 16 + g, qrow1 = qrow0 + 8;
  int brow[2], hrow[2];
  uint32_t qa[8][4];
  {
    const __half* qr[2];
    int pos[2];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int r = min(rr ? qrow1 : qrow0, rows - 1);
      const int bb = px.group_members[m_begin + r / G];
      brow[rr] = bb; hrow[rr] = hkv * G + r % G;
      pos[rr] = (kv.indptr[bb + 1] - kv.indptr[bb] - 1) * kv.P + kv.last_page_offset[bb] - 1;
      qr[rr] = q + ((size_t)bb * Hq + hrow[rr]) * 128;
    }
    rope_q_frags(qa, qr, pos, log2_theta);
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
    // keys past the prefix (last tile only) are masked; every row sees the same keys.  The step's guard for a row without a
    // visible key never fires here: t_begin < t_end, and key 64 t_begin < prefix is visible to every row, so m is finite from
    // the first tile on and the exponentials are taken against m itself
    attn_tile_step(qa, Ks, Vt, a0, [&](int, int kpos) { return kpos < prefix; }, o, m0, m1, l0, l1);
  }

  // ---- un-normalised partial of each live row: (m, d, acc[128]) at [b][h][chunk]
  l0 = quad_sum(l0); l1 = quad_sum(l1);
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    if ((rr ? qrow1 : qrow0) >= rows) continue;
    attn_store_part(px.part + (((size_t)brow[rr] * Hq + hrow[rr]) * px.nchunks + chunk) * DEC_PART, o, rr, rr ? m1 : m0, rr ? l1 : l0);
  }
}

}  // namespace atom
