// beam_kernels.cuh -- beam search on the device: one beam step over the logits rows of every request's live beams
// (atom_beam_select_f16), and the batched page copies of copy-on-write forks (atom_kv_copy_pages_i4); include/atom_b200.h,
// DESIGN section 5.9.
//
// beam_row_kernel runs each row on the sampler's row machinery (sample_kernels.cuh, unchanged): a cluster of
// C = ceil(V / 32768) CTAs holds the row as order-preserving keys, sums the exact Z1 at T = 1 and computes each token's
// log-probability exactly as atom_sample_ex_f16 reports it.  The stop ids' keys are looked up and then masked, and the radix
// select at K = W keeps the row's first W other tokens in its order (key descending, index ascending).  So a row's list -- at
// most W + |stop| entries -- is a function of its logits, W and the stop ids alone.  beam_merge_kernel, one CTA per request,
// orders the lists of the request's rows by fl32(sum + lp), then beam index, then the row's order, and walks them: a stop
// candidate of rank < W is finished, any other one becomes a live beam until there are W.  Every live candidate of the global
// order lies in its row's first W non-stop tokens, and every stop candidate is listed, so the merged order is exact.
#pragma once
#include "sample_kernels.cuh"

namespace atom {

constexpr int BEAM_MAX_WIDTH = 8, BEAM_MAX_STOP = 8;
constexpr int BEAM_LIST = BEAM_MAX_WIDTH + BEAM_MAX_STOP;       // a row's candidate list
constexpr int BEAM_MERGE_THREADS = BEAM_MAX_WIDTH * BEAM_LIST;  // one thread per entry of a request's lists

struct BeamArgs {
  const __half* logits;
  long long ld;
  int V, slice, W, nstop;
  int stop[BEAM_MAX_STOP];
  const int32_t* row_indptr;                       // [B + 1]
  const float* sums;                               // [R]
  unsigned long long* code;                        // [R][BEAM_LIST]: (key << 32) | ~token, 0 = empty
  float* lp;                                       // [R][BEAM_LIST]
  int R;
  int32_t *live, *fin;                             // [B][W][2]: (row, token)
  float *live_key, *fin_key;                       // [B][W]
};

// after the keys of the slice (sample_ex_offset)
struct BeamShared {
  unsigned long long top[BEAM_MAX_WIDTH];          // this CTA's survivors of the select
  uint32_t stopk[BEAM_MAX_STOP];                   // the keys of the stop ids this CTA holds
  uint32_t ntop;
};

// grid (C * R), cluster (C): CTA x is rank x % C of row x / C
__global__ void __launch_bounds__(SAMPLE_THREADS, 1) beam_row_kernel(const BeamArgs a, int pdl) {
  extern __shared__ __align__(16) uint8_t smem_b[];
  SampleShared& s = *reinterpret_cast<SampleShared*>(smem_b);
  BeamShared& e = *reinterpret_cast<BeamShared*>(smem_b + sample_ex_offset(a.slice));
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t rank = cluster_ctarank(), C = cluster_nctarank();
  const long long row = blockIdx.x / C;
  const int lo = (int)rank * a.slice, len = max(0, min(a.V - lo, a.slice));
  if (pdl) { griddep_launch_dependents(); griddep_wait(); }

  // ---- the keys, the row maximum (first index of), finite count, NaN / +inf: sample_row's load pass without penalties
  const unsigned short* src = reinterpret_cast<const unsigned short*>(a.logits + row * a.ld + lo);
  unsigned long long best = 0;
  uint32_t finite = 0, invalid = 0;
#pragma unroll 8
  for (int i = tid; i < len; i += SAMPLE_THREADS) {
    const uint32_t k = sample_key(__ldg(src + i));
    s.keys[i] = (uint16_t)k;
    invalid |= (uint32_t)(k > SAMPLE_KEY_MAX_FINITE || k < SAMPLE_KEY_NEG_INF);
    finite += (uint32_t)(k > SAMPLE_KEY_NEG_INF);
    best = max(best, ((unsigned long long)k << 32) | (0xFFFFFFFFu - (uint32_t)(lo + i)));
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    best = max(best, __shfl_xor_sync(0xFFFFFFFFu, best, o));
    finite += __shfl_xor_sync(0xFFFFFFFFu, finite, o);
    invalid |= __shfl_xor_sync(0xFFFFFFFFu, invalid, o);
  }
  if (lane == 0) { s.red[warp] = best; s.redu[warp] = finite; s.redu[SAMPLE_WARPS + warp] = invalid; }
  for (int i = tid; i < 256; i += SAMPLE_THREADS) { s.h1[i] = 0; s.h2[i] = 0; }
  if (tid == 0) e.ntop = 0;
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < SAMPLE_WARPS; ++w) {
      s.red[0] = max(s.red[0], s.red[w]); s.redu[0] += s.redu[w]; s.redu[SAMPLE_WARPS] |= s.redu[SAMPLE_WARPS + w];
    }
    s.pub[0] = s.red[0]; s.pub[1] = s.redu[0]; s.pub[2] = s.redu[SAMPLE_WARPS];
  }
  sample_cluster_sync();
  if (tid == 0) {
    unsigned long long b = 0, f = 0, inv = 0;
    for (uint32_t r = 0; r < C; ++r) { b = max(b, dsmem_u64(&s.pub[0], r)); f += dsmem_u64(&s.pub[1], r); inv |= dsmem_u64(&s.pub[2], r); }
    s.bc[0] = b; s.bc[1] = f; s.bc[2] = inv;
  }
  __syncthreads();
  best = s.bc[0];
  const bool bad_row = s.bc[2] != 0 || s.bc[1] == 0;
  __syncthreads();
  unsigned long long* code = a.code + row * BEAM_LIST;
  float* lps = a.lp + row * BEAM_LIST;
  if (bad_row) {                                    // no candidates (the sampler returns -1 for such a row)
    if (rank == 0 && tid < BEAM_LIST) code[tid] = 0ull;
    sample_cluster_sync();
    return;
  }

  // ---- Z1 and the log-probability of a key, exactly as sample_logprobs computes them
  const float vmax = sample_value((uint32_t)(best >> 32));
  const unsigned long long z = sample_cluster_sum(s, 3, len, C, [&](int i) { return sample_weight(s.keys[i], vmax, 1.f); });
  const double lnz = log((double)z * 0x1p-40);
  auto lp = [&](uint32_t k) {
    return k <= SAMPLE_KEY_NEG_INF ? -INFINITY : (float)((double)__fsub_rn(sample_value(k), vmax) - lnz);
  };

  // ---- the stop ids: record their keys, then mask them out of the select (key 0 sorts below -inf)
  if (tid < a.nstop) {
    const int t = a.stop[tid];
    if (t >= lo && t < lo + len) e.stopk[tid] = s.keys[t - lo];
  }
  __syncthreads();
  if (tid < a.nstop) {
    const int t = a.stop[tid];
    if (t >= lo && t < lo + len) s.keys[t - lo] = 0;
  }
  __syncthreads();

  // ---- the first W non-stop tokens of the row's order: the top-k cut at K = W, -inf and the masked stop ids excluded
  uint32_t kth = 0;
  int kidx = 0x7FFFFFFF;
  if (a.W < a.V) sample_topk_cut(s, a.W, len, lo, C, rank, 5, kth, kidx);
  for (int i = tid; i < len; i += SAMPLE_THREADS) {
    const uint32_t k = s.keys[i];
    if (k > SAMPLE_KEY_NEG_INF && (k > kth || (k == kth && lo + i <= kidx)))
      e.top[atomicAdd(&e.ntop, 1u)] = ((unsigned long long)k << 32) | (0xFFFFFFFFu - (uint32_t)(lo + i));
  }
  sample_cluster_sync();
  if (rank == 0 && tid == 0) {                      // at most W survivors in the cluster, then the finite stop ids
    int m = 0;
    for (uint32_t r = 0; r < C; ++r) {
      const uint32_t c = dsmem_u32(&e.ntop, r);
      for (uint32_t j = 0; j < c; ++j) {
        const unsigned long long v = dsmem_u64(&e.top[j], r);
        code[m] = v; lps[m] = lp((uint32_t)(v >> 32)); ++m;
      }
    }
    for (int j = 0; j < a.nstop; ++j) {
      const int t = a.stop[j];
      const uint32_t k = dsmem_u32(&e.stopk[j], (uint32_t)(t / a.slice));
      if (k > SAMPLE_KEY_NEG_INF) { code[m] = ((unsigned long long)k << 32) | (0xFFFFFFFFu - (uint32_t)t); lps[m] = lp(k); ++m; }
    }
    for (; m < BEAM_LIST; ++m) code[m] = 0ull;
  }
  sample_cluster_sync();                            // no CTA leaves while rank 0 may still read its shared memory
}

// grid (B), one CTA per request: order its rows' lists and walk them
__global__ void __launch_bounds__(BEAM_MERGE_THREADS) beam_merge_kernel(const BeamArgs a, int pdl) {
  __shared__ float key[BEAM_MERGE_THREADS];
  __shared__ unsigned long long code[BEAM_MERGE_THREADS];
  __shared__ int16_t order[BEAM_MERGE_THREADS];
  __shared__ int s_n;
  const int i = blockIdx.x, tid = threadIdx.x, W = a.W;
  if (pdl) { griddep_launch_dependents(); griddep_wait(); }
  const int r0 = a.row_indptr[i], r1 = a.row_indptr[i + 1], nrows = r1 - r0;
  // a request of more than W rows, or rows outside [0, R), is malformed: it gets no candidates
  const bool ok = nrows > 0 && nrows <= W && r0 >= 0 && r1 <= a.R;
  if (tid == 0) s_n = 0;
  {
    const int j = tid / BEAM_LIST;
    float k = 0.f;
    unsigned long long c = 0;
    if (ok && j < nrows) {
      c = a.code[(long long)(r0 + j) * BEAM_LIST + tid % BEAM_LIST];
      if (c) {
        k = __fadd_rn(a.sums[r0 + j], a.lp[(long long)(r0 + j) * BEAM_LIST + tid % BEAM_LIST]);
        if (isnan(k)) c = 0;
      }
    }
    key[tid] = k; code[tid] = c;
  }
  __syncthreads();
  if (code[tid]) {                                  // position in (key desc, beam asc, row order desc); all entries distinct
    const float k = key[tid];
    const unsigned long long c = code[tid];
    const int j = tid / BEAM_LIST;
    int pos = 0;
    for (int u = 0; u < BEAM_MERGE_THREADS; ++u) {
      if (!code[u]) continue;
      const int ju = u / BEAM_LIST;
      pos += key[u] > k || (key[u] == k && (ju < j || (ju == j && code[u] > c)));
    }
    order[pos] = (int16_t)tid;
    atomicAdd(&s_n, 1);
  }
  __syncthreads();
  if (tid != 0) return;
  int32_t *live = a.live + (long long)i * W * 2, *fin = a.fin + (long long)i * W * 2;
  float *live_key = a.live_key + (long long)i * W, *fin_key = a.fin_key + (long long)i * W;
  int nl = 0, nf = 0;
  for (int rk = 0; rk < s_n && nl < W; ++rk) {
    const int u = order[rk];
    const int t = (int)(0xFFFFFFFFu - (uint32_t)code[u]);
    bool stop = false;
    for (int q = 0; q < a.nstop; ++q) stop |= t == a.stop[q];
    if (stop) {
      if (rk < W) { fin[2 * nf] = r0 + u / BEAM_LIST; fin[2 * nf + 1] = t; fin_key[nf] = key[u]; ++nf; }
    } else {
      live[2 * nl] = r0 + u / BEAM_LIST; live[2 * nl + 1] = t; live_key[nl] = key[u]; ++nl;
    }
  }
  for (; nl < W; ++nl) { live[2 * nl] = -1; live[2 * nl + 1] = -1; live_key[nl] = -1.f; }
  for (; nf < W; ++nf) { fin[2 * nf] = -1; fin[2 * nf + 1] = -1; fin_key[nf] = -1.f; }
}

inline size_t beam_row_smem(int slice) { return sample_ex_offset(slice) + sizeof(BeamShared); }

// ---- atom_kv_copy_pages_i4: pair p copies the first slots[p] token slots of page src[p] to page dst[p], every (layer, K|V,
// head) block of pool.buf (P * 64 bytes, 64 per slot) and pool.param (P * 4 bytes, 4 per slot).  grid (ceil(blocks / 4), n).
constexpr int KV_COPY_THREADS = 256, KV_COPY_BLOCKS_PER_CTA = 4;

__global__ void __launch_bounds__(KV_COPY_THREADS) kv_copy_pages_kernel(uint8_t* buf, uint32_t* param, int pages, int blocks, int P,
                                                                        const int32_t* src, const int32_t* dst, const int32_t* slots,
                                                                        int pdl) {
  if (pdl) { griddep_launch_dependents(); griddep_wait(); }
  const int p = blockIdx.y, s = src[p], d = dst[p], n = slots[p];
  // src < 0 is padding; a pair the kernel cannot honour (src == dst, a page or slot count out of range) is ignored
  if (s < 0 || s == d || s >= pages || d < 0 || d >= pages || n <= 0 || n > P) return;
  const long long page_b = (long long)blocks * P * 64, page_p = (long long)blocks * P;
  const int b0 = blockIdx.x * KV_COPY_BLOCKS_PER_CTA, b1 = min(blocks, b0 + KV_COPY_BLOCKS_PER_CTA);
  const int nv = n * 4;                             // 16-byte vectors of one block's first n slots
  for (int b = b0; b < b1; ++b) {
    const uint4* from = reinterpret_cast<const uint4*>(buf + s * page_b + (long long)b * P * 64);
    uint4* to = reinterpret_cast<uint4*>(buf + d * page_b + (long long)b * P * 64);
    for (int j = threadIdx.x; j < nv; j += KV_COPY_THREADS) to[j] = from[j];
    const uint32_t* pf = param + s * page_p + (long long)b * P;
    uint32_t* pt = param + d * page_p + (long long)b * P;
    for (int j = threadIdx.x; j < n; j += KV_COPY_THREADS) pt[j] = pf[j];
  }
}

}  // namespace atom
