// verify_kernels.cuh -- speculative verification: multi-token decode attention over the INT4 pages.
//
// Sequence b of the batch ends with S query tokens (1 <= S <= 8) at positions len_b - S .. len_b - 1, whose K/V are already in
// the pages (init_kv_i4 with a stride-S indptr).  Query token i attends to every key at a position <= len_b - S + i: the cached
// tokens before the tail and, causally, the tail itself.
//   * grid (chunk, KV head, sequence).  The S x G query rows of one (sequence, KV head) -- row r = (token r / G, query head
//     hkv*G + r % G) -- fit one 64-row m16n8k16 tile, so a CTA streams its chunk of the sequence's pages ONCE for all of them:
//     64-token tiles dequantised, and K rotated at its absolute positions from the (cos, sin) table, by prefill_attn_kernel<true>'s
//     context loader (prefill_ctx_tile), as the cascade's prefix pass does; the tile step (attn_tile_step) with a per-row causal
//     limit.
//     Warps whose 16 rows are all padding (S x G <= 48) load their share of the tile and skip the MMAs.
//   * q is rotated at its own position, read from the page table on the device, as the cascade rotates it (rope_q_frags): a
//     captured graph replays the launch with new lengths.  K's table covers a bound the caller states.
//   * split-KV: the sequence's ceil(len / 64) tiles are cut into nchunks runs of ceil(tiles / nchunks) consecutive tiles (the last
//     runs may be empty).  With nchunks > 1 each CTA leaves the un-normalised (m, d, acc[128]) of its rows in the FP32 workspace
//     (the DEC_PART layout, [B*S][Hq][nchunks]) and verify_merge_kernel combines them in chunk order.  The tiling depends on the
//     length and the host-chosen chunk count only, and both the tile loop and the merge run in a fixed order: a row's result does
//     not depend on where its pages sit.
#pragma once
#include "prefill_kernels.cuh"

namespace atom {

__host__ __device__ __forceinline__ int verify_tiles(int len) { return (len + PF_BK - 1) / PF_BK; }
__host__ __device__ __forceinline__ int verify_per(int tiles, int nchunks) { return (tiles + nchunks - 1) / nchunks; }
__device__ __forceinline__ int verify_len(const KvArgs& kv, int b) {
  return (kv.indptr[b + 1] - kv.indptr[b] - 1) * kv.P + kv.last_page_offset[b];
}

// o f16 [B*S, Hq, 128], q f16 [B*S, Hq, 128] (pre-RoPE), row b*S + i = token i of sequence b; rope: (cos, sin) table of at least
// max_b len_b positions (ops.rope_table); part: FP32 workspace [B*S][Hq][nchunks][DEC_PART] (unused when nchunks == 1).
// Precondition len_b >= S; a sequence that breaks it (a malformed page table) gets zero rows and no page of it is read.
__global__ void __launch_bounds__(PF_THREADS, 2)
verify_attn_kernel(__half* __restrict__ o, const __half* __restrict__ q, KvArgs kv, const float2* __restrict__ rope, float log2_theta,
                   int S, int G, float* __restrict__ part, int nchunks, int pdl) {
  __shared__ __align__(16) __half Ks[PF_BK * PF_KPITCH];
  __shared__ __align__(16) __half Vt[128 * PF_VPITCH];
  if (pdl) { griddep_launch_dependents(); griddep_wait(); }       // q and the tail's K/V come from the preceding kernels
  const int chunk = blockIdx.x, hkv = blockIdx.y, b = blockIdx.z;
  const int len = verify_len(kv, b);
  const int tid = threadIdx.x, warp = tid >> 5, g = (tid & 31) >> 2;
  const int Hq = kv.H * G, rows = S * G;
  if (len < S) {             // a page table whose sequence is shorter than its query tokens: zeros, no page is read
    if (chunk == 0 && nchunks == 1)
      for (int e = tid; e < rows * 128; e += PF_THREADS)
        o[(((size_t)b * S + e / 128 / G) * Hq + hkv * G + e / 128 % G) * 128 + e % 128] = __float2half_rn(0.f);
    return;
  }
  const int tiles = verify_tiles(len), per = verify_per(tiles, nchunks);
  const int t_begin = chunk * per, t_end = min(tiles, t_begin + per);
  if (t_begin >= t_end) return;
  const bool busy = warp * 16 < rows;                              // warp-uniform: some of this warp's rows are live

  // ---- Q fragments of this warp's 16 rows, rotated at len - S + token; padded rows repeat the last live row and are never stored
  const int qrow0 = warp * 16 + g, qrow1 = qrow0 + 8;
  int lim[2], hrow[2], trow[2];
  uint32_t qa[8][4];
  {
    const __half* qr[2];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int r = min(rr ? qrow1 : qrow0, rows - 1);
      trow[rr] = r / G; hrow[rr] = hkv * G + r % G;
      lim[rr] = len - S + trow[rr];                                // the row's position: keys at positions <= lim are visible
      qr[rr] = q + (((size_t)b * S + trow[rr]) * Hq + hrow[rr]) * 128;
    }
    rope_q_frags(qa, qr, lim, log2_theta);
  }

  // the context loader of prefill_attn_kernel<true> with the whole sequence as the "context" of an empty prompt: key position
  // k0 + tok is absolute position len + k0 + tok, and the table is shifted to match
  const float2* rope_ctx = rope + (size_t)len * 64;

  float acc[16][4];
#pragma unroll
  for (int i = 0; i < 16; ++i) { acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f; }
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

  for (int kt = t_begin; kt < t_end; ++kt) {
    const int a0 = kt * PF_BK;                        // absolute position of the tile's first key
    __syncthreads();                                  // the previous tile has been consumed
    prefill_ctx_tile(kv, b, 0, hkv, a0 - len, rope_ctx, Ks, Vt, tid);
    __syncthreads();
    if (!busy) continue;
    // causal limit (keys past len are past every row's limit); a chunk that starts inside the tail can hold no key for its first rows
    attn_tile_step(qa, Ks, Vt, a0, [&](int rr, int kpos) { return kpos <= lim[rr]; }, acc, m0, m1, l0, l1);
  }
  if (!busy) return;

  l0 = quad_sum(l0); l1 = quad_sum(l1);
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    if ((rr ? qrow1 : qrow0) >= rows) continue;
    const size_t row = ((size_t)b * S + trow[rr]) * Hq + hrow[rr];
    if (nchunks == 1) attn_store_row(o + row * 128, acc, rr, rr ? l1 : l0);                  // the whole sequence
    else attn_store_part(part + (row * nchunks + chunk) * DEC_PART, acc, rr, rr ? m1 : m0, rr ? l1 : l0);   // this chunk's partial
  }
}

// grid (B*S, Hq), 128 threads: element d of row (b*S + i, h) combines the partials of the sequence's non-empty chunks in chunk
// order (chunk 0 always holds key 0, which every row sees: the maximum is finite)
__global__ void __launch_bounds__(128)
verify_merge_kernel(__half* __restrict__ o, const float* __restrict__ part, KvArgs kv, int S, int Hq, int nchunks, int pdl) {
  if (pdl) { griddep_launch_dependents(); griddep_wait(); }
  const int row = blockIdx.x, h = blockIdx.y, d = threadIdx.x;
  const int len = verify_len(kv, row / S);
  if (len < S) { o[((size_t)row * Hq + h) * 128 + d] = __float2half_rn(0.f); return; }   // as verify_attn_kernel: zeros
  const int tiles = verify_tiles(len), per = verify_per(tiles, nchunks);
  const int nck = (tiles + per - 1) / per;
  const float* src = part + ((size_t)row * Hq + h) * nchunks * DEC_PART;
  float mm = -INFINITY;
  for (int k = 0; k < nck; ++k) mm = fmaxf(mm, src[k * DEC_PART]);
  float dd = 0.f, out = 0.f;
  for (int k = 0; k < nck; ++k) {
    const float sx = exp2f(src[k * DEC_PART] - mm);
    dd = fmaf(src[k * DEC_PART + 1], sx, dd);
    out = fmaf(src[k * DEC_PART + 2 + d], sx, out);
  }
  o[((size_t)row * Hq + h) * 128 + d] = __float2half_rn(out / dd);
}

}  // namespace atom
