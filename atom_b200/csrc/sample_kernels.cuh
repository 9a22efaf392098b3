// sample_kernels.cuh -- token sampling from FP16 logits: per-row temperature, top-k and top-p, with a counter-based Philox
// stream (atom_sample_f16, include/atom_b200.h; DESIGN section 5.6).
//
// One cluster of C CTAs per row, C = ceil(V / 32768) from V alone (so a row's result never depends on the batch).  CTA r
// holds the contiguous slice [r * slice, r * slice + len) of the row in shared memory as order-preserving 16-bit keys
// (value descending <=> key descending, -0 folded onto +0) and every later pass reads only shared memory.  Each decision
// (row maximum, the top-k key, the top-p key, the tie cut-offs by index, the drawn token) is made identically by every CTA
// of the cluster from partials that the CTAs publish in their shared memory and read over DSMEM in rank order.  All
// cross-thread and cross-CTA sums are integers (counts, and weights in fixed point: round(w * 2^40) with
// w = expf((v - vmax) / T) in FP32), so every sum is exact and the result does not depend on any summation order.
//
// sample_kernel<PEN, EXT> (atom_sample_ex_f16).  PEN: the row's penalty state (a u16 table slot: prompt bit, generated count)
// turns each logit into the penalised l' in the load pass, before it becomes a key; rank 0 records the drawn token in the slot.
// EXT: min-p (a weight threshold folded into the weights), the log-probabilities of the chosen token (one more exact weight
// pass for Z1 at T = 1) and a top-n list (the top-k radix select at K = n, compacted per CTA and ordered by rank 0).
// sample_kernel<false, false> is atom_sample_f16's kernel.
#pragma once
#include "ptx_sm90.cuh"

namespace atom {

constexpr int SAMPLE_THREADS = 1024, SAMPLE_WARPS = SAMPLE_THREADS / 32;
constexpr int SAMPLE_SLICE_MAX = 32768;           // FP16 logits per CTA: 64 KB
constexpr int SAMPLE_MAX_CLUSTER = 8;              // portable cluster size: V <= 262144
constexpr uint32_t SAMPLE_KEY_NEG_INF = 0x03FFu, SAMPLE_KEY_MAX_FINITE = 0xFBFFu;

struct SampleArgs {
  const __half* logits;
  long long ld;                                    // row pitch in elements
  int V, slice;                                    // slice: logits per CTA (the last CTA may hold fewer)
  const float* temperature;
  const int32_t* top_k;
  const float* top_p;
  const unsigned long long* key;                   // [B][2]
  const unsigned long long* counter;               // [B]
  int32_t* out;
};

constexpr int SAMPLE_TOP_N_MAX = 20;

// the options of atom_sample_ex_f16; only the instances that use them read them
struct SampleExArgs {
  const float* min_p;                              // [B] or null (off)
  const float *rep, *freq, *pres;                  // [B] (PEN)
  const int32_t* slots;                            // [B]: the row's table slot, or -1 (PEN)
  uint16_t* table;                                 // [slots][table_ld]: bit 15 in the prompt, bits 0-14 generated count (PEN)
  long long table_ld;
  float* logprob;                                  // [B] or null
  int top_n;                                       // 0 .. SAMPLE_TOP_N_MAX
  int32_t* top_ids;                                // [B][top_n]
  float* top_logprobs;                             // [B][top_n]
};

struct SampleShared {
  unsigned long long pub[16];                      // this CTA's published partials, one slot per exchange (never reused)
  unsigned long long w1[256], w2[256], wfull[256]; // top-p: per-bucket weights (this CTA's), and their cluster sums
  unsigned long long wsum[SAMPLE_WARPS];           // per-warp partials of a search in index order
  unsigned long long red[SAMPLE_WARPS];
  unsigned long long bc[4];                        // block broadcast
  uint32_t h1[256], h2[256], hfull[256];           // top-k: per-bucket counts (this CTA's), and their cluster sums
  uint32_t redu[2 * SAMPLE_WARPS];
  uint16_t keys[SAMPLE_SLICE_MAX];
};
constexpr size_t SAMPLE_SMEM_FIXED = offsetof(SampleShared, keys);

// EXT only, after the keys of the slice
struct SampleExShared {
  unsigned long long top[SAMPLE_TOP_N_MAX];        // this CTA's top-n survivors, (key << 32) | ~index
  unsigned long long all[SAMPLE_TOP_N_MAX];        // rank 0: the cluster's survivors (at most top_n in all)
  double lnz;                                      // ln(Z1 * 2^-40)
  uint32_t ntop, nall;
};
__host__ __device__ inline size_t sample_ex_offset(int slice) { return SAMPLE_SMEM_FIXED + (((size_t)slice * sizeof(uint16_t) + 15) & ~(size_t)15); }

__device__ __forceinline__ uint32_t sample_key(unsigned short h) {
  if (h == 0x8000u) h = 0;                         // -0 == +0, as torch.argmax compares
  return (h & 0x8000u) ? (~h & 0xFFFFu) : (h | 0x8000u);
}
__device__ __forceinline__ float sample_value(uint32_t k) {
  const unsigned short h = (k & 0x8000u) ? (unsigned short)(k & 0x7FFFu) : (unsigned short)(~k & 0xFFFFu);
  return __half2float(__ushort_as_half(h));
}
// the token's weight round(expf(fl(fl(v - vmax) / T)) * 2^40); -inf weighs 0
__device__ __forceinline__ unsigned long long sample_weight(uint32_t k, float vmax, float T) {
  if (k <= SAMPLE_KEY_NEG_INF) return 0ull;
  const float x = __fdiv_rn(__fsub_rn(sample_value(k), vmax), T);
  return __float2ull_rn(expf(x) * 1099511627776.0f);
}

// the penalised logit l' of an FP16 logit h with table entry e (DESIGN section 5.6): -inf stays; repetition r if the token is in
// the prompt or was generated; frequency fl(c * f); presence p if c > 0; one IEEE FP32 rounding each, then FP16 saturated
// (fmaxf drops a NaN from inf - inf, which becomes -65504)
__device__ __forceinline__ unsigned short sample_penalise(unsigned short h, uint32_t e, float r, float f, float p) {
  if (h == 0xFC00u) return h;
  const uint32_t c = e & 0x7FFFu;
  float l = __half2float(__ushort_as_half(h));
  if ((e & 0x8000u) || c) l = l > 0.f ? __fdiv_rn(l, r) : __fmul_rn(l, r);
  l = __fsub_rn(l, __fmul_rn((float)c, f));
  if (c) l = __fsub_rn(l, p);
  return __half_as_ushort(__float2half_rn(fminf(fmaxf(l, -65504.f), 65504.f)));
}

// Philox4x64-10 (Salmon et al., SC'11; the Random123 constants): word 0 of the block at counter (n, 0, 0, 0)
__device__ __forceinline__ unsigned long long philox4x64_w0(unsigned long long k0, unsigned long long k1, unsigned long long n) {
  const unsigned long long M0 = 0xD2E7470EE14C6C93ull, M1 = 0xCA5A826395121157ull;
  unsigned long long c0 = n, c1 = 0, c2 = 0, c3 = 0;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) { k0 += 0x9E3779B97F4A7C15ull; k1 += 0xBB67AE8584CAA73Bull; }
    const unsigned long long hi0 = __umul64hi(M0, c0), lo0 = M0 * c0, hi1 = __umul64hi(M1, c2), lo1 = M1 * c2;
    c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
  }
  return c0;
}
// words 0 and 1 of the same block (the draft rule's acceptance uses word 1)
__device__ __forceinline__ ulonglong2 philox4x64_w01(unsigned long long k0, unsigned long long k1, unsigned long long n) {
  const unsigned long long M0 = 0xD2E7470EE14C6C93ull, M1 = 0xCA5A826395121157ull;
  unsigned long long c0 = n, c1 = 0, c2 = 0, c3 = 0;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) { k0 += 0x9E3779B97F4A7C15ull; k1 += 0xBB67AE8584CAA73Bull; }
    const unsigned long long hi0 = __umul64hi(M0, c0), lo0 = M0 * c0, hi1 = __umul64hi(M1, c2), lo1 = M1 * c2;
    c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
  }
  return make_ulonglong2(c0, c1);
}

__device__ __forceinline__ unsigned long long dsmem_u64(const void* p, uint32_t rank) {
  unsigned long long v;
  asm volatile("ld.shared::cluster.u64 %0, [%1];" : "=l"(v) : "r"(mapa_shared(smem_u32(p), rank)) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t dsmem_u32(const void* p, uint32_t rank) {
  uint32_t v;
  asm volatile("ld.shared::cluster.u32 %0, [%1];" : "=r"(v) : "r"(mapa_shared(smem_u32(p), rank)) : "memory");
  return v;
}
__device__ __forceinline__ void sample_cluster_sync() { cluster_arrive(); cluster_wait(); }

template <typename T>
__device__ __forceinline__ T warp_incl_scan(T v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(0xFFFFFFFFu, v, o);
    if (lane >= o) v += y;
  }
  return v;
}

// cluster sum of a 256-bucket histogram: full[i] = sum over ranks of local[i]
template <typename T>
__device__ __forceinline__ void sample_hist_sum(const T* local, T* full, uint32_t C) {
  sample_cluster_sync();
  for (int i = threadIdx.x; i < 256; i += SAMPLE_THREADS) {
    T acc = 0;
    for (uint32_t r = 0; r < C; ++r) acc += (sizeof(T) == 8) ? (T)dsmem_u64(local + i, r) : (T)dsmem_u32(local + i, r);
    full[i] = acc;
  }
  __syncthreads();
}

// warp 0: the first bucket, from 255 down, whose inclusive cumulative sum reaches target(total); bc[0] = bucket,
// bc[1] = the sum of the buckets above it, bc[2] = the target
template <typename T, typename TF>
__device__ __forceinline__ void sample_select_desc(const T* full, TF target_of, SampleShared& s) {
  const int lane = threadIdx.x & 31;
  T v[8], sum = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) { v[i] = full[255 - 8 * lane - i]; sum += v[i]; }
  const T incl = warp_incl_scan(sum, lane);
  const T total = __shfl_sync(0xFFFFFFFFu, incl, 31);
  const T target = target_of(total);
  const int L = __ffs(__ballot_sync(0xFFFFFFFFu, incl >= target)) - 1;
  if (lane == L) {
    T acc = incl - sum;
    int bin = 255 - 8 * L - 7;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (acc + v[i] >= target) { bin = 255 - 8 * L - i; break; }
      acc += v[i];
    }
    s.bc[0] = (unsigned long long)bin; s.bc[1] = (unsigned long long)acc; s.bc[2] = (unsigned long long)target;
  }
}

// The global index of the first element of the row, in ascending index order, at which the running sum of f reaches past
// t = t_of(sum of f over the row).  Every CTA returns it.  Uses pub[slot] and pub[slot + 1].  Warp w scans the contiguous
// segment [w * seg, (w + 1) * seg) of the slice, lane by lane.
template <typename F, typename TF>
__device__ __forceinline__ int sample_find(SampleShared& s, int slot, int len, int lo, uint32_t C, uint32_t rank, F f, TF t_of) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int seg = ((len + SAMPLE_WARPS - 1) / SAMPLE_WARPS + 31) & ~31;
  {
    const int b = warp * seg, e = min(len, b + seg);
    unsigned long long acc = 0;
    for (int i = b + lane; i < e; i += 32) acc += f(i);
#pragma unroll
    for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xFFFFFFFFu, acc, o);
    if (lane == 0) s.wsum[warp] = acc;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long mine = 0;
    for (int w = 0; w < SAMPLE_WARPS; ++w) mine += s.wsum[w];
    s.pub[slot] = mine;
    s.bc[3] = mine;
  }
  sample_cluster_sync();
  if (threadIdx.x == 0) {
    unsigned long long all = 0, before = 0;
    for (uint32_t r = 0; r < C; ++r) {
      if (r == rank) before = all;
      all += dsmem_u64(&s.pub[slot], r);
    }
    const unsigned long long t = t_of(all);
    s.bc[0] = (t >= before && t - before < s.bc[3]) ? t - before : ~0ull;
  }
  __syncthreads();
  const unsigned long long lt = s.bc[0];
  if (warp == 0) {
    long long found = -1;
    if (lt != ~0ull) {
      const unsigned long long v = s.wsum[lane], incl = warp_incl_scan(v, lane);
      const int L = __ffs(__ballot_sync(0xFFFFFFFFu, incl > lt)) - 1;
      unsigned long long ex = __shfl_sync(0xFFFFFFFFu, incl - v, L);
      const int b = L * seg, e = min(len, b + seg);
      for (int i = b; i < e; i += 32) {
        const unsigned long long x = (i + lane < e) ? f(i + lane) : 0ull;
        const unsigned long long in = warp_incl_scan(x, lane);
        const unsigned hit = __ballot_sync(0xFFFFFFFFu, ex + in > lt);
        if (hit) { found = lo + i + __ffs(hit) - 1; break; }
        ex += __shfl_sync(0xFFFFFFFFu, in, 31);
      }
    }
    if (lane == 0) s.pub[slot + 1] = (unsigned long long)found;
  }
  sample_cluster_sync();
  if (threadIdx.x == 0) {
    long long r = -1;
    for (uint32_t q = 0; q < C; ++q) r = max(r, (long long)dsmem_u64(&s.pub[slot + 1], q));
    s.bc[0] = (unsigned long long)r;
  }
  __syncthreads();
  return (int)(long long)s.bc[0];
}

// The K-th key of the order (kth) and the index of the last token kept at that key (kidx), for 0 < K < V: a two-level radix
// select over the cluster's 256-bucket key histograms (h1 and h2 zero on entry), then the tie cut-off by index.  Uses
// pub[slot] and pub[slot + 1].  The top-n list calls it; sample_kernel's top-k pass is the same code written out in place,
// because calling this instead schedules a few instructions of the plain instance differently from atom_sample_f16's kernel.
__device__ __forceinline__ void sample_topk_cut(SampleShared& s, int K, int len, int lo, uint32_t C, uint32_t rank, int slot,
                                                uint32_t& kth, int& kidx) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int base = 0; base < len; base += SAMPLE_THREADS) {
    const int i = base + tid;
    const uint32_t bin = i < len ? (uint32_t)(s.keys[i] >> 8) : 0x100u;
    const unsigned m = __match_any_sync(0xFFFFFFFFu, bin);
    if (i < len && lane == __ffs(m) - 1) atomicAdd(&s.h1[bin], (uint32_t)__popc(m));
  }
  sample_hist_sum(s.h1, s.hfull, C);
  if (warp == 0) sample_select_desc(s.hfull, [&](uint32_t) { return (uint32_t)K; }, s);
  __syncthreads();
  const uint32_t b1 = (uint32_t)s.bc[0], above1 = (uint32_t)s.bc[1];
  for (int i = tid; i < len; i += SAMPLE_THREADS)
    if ((uint32_t)(s.keys[i] >> 8) == b1) atomicAdd(&s.h2[s.keys[i] & 0xFF], 1u);
  sample_hist_sum(s.h2, s.hfull, C);
  if (warp == 0) sample_select_desc(s.hfull, [&](uint32_t) { return (uint32_t)K - above1; }, s);
  __syncthreads();
  kth = (b1 << 8) | (uint32_t)s.bc[0];
  const unsigned long long need = (unsigned long long)K - above1 - s.bc[1];
  __syncthreads();
  const uint32_t kk = kth;
  kidx = sample_find(s, slot, len, lo, C, rank, [&](int i) { return (unsigned long long)(s.keys[i] == kk); },
                     [&](unsigned long long) { return need - 1; });
}

// the cluster sum of f over the row, returned to every thread; uses pub[slot]
template <typename F>
__device__ __forceinline__ unsigned long long sample_cluster_sum(SampleShared& s, int slot, int len, uint32_t C, F f) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long acc = 0;
  for (int i = threadIdx.x; i < len; i += SAMPLE_THREADS) acc += f(i);
#pragma unroll
  for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(0xFFFFFFFFu, acc, o);
  if (lane == 0) s.wsum[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long mine = 0;
    for (int w = 0; w < SAMPLE_WARPS; ++w) mine += s.wsum[w];
    s.pub[slot] = mine;
  }
  sample_cluster_sync();
  if (threadIdx.x == 0) {
    unsigned long long all = 0;
    for (uint32_t r = 0; r < C; ++r) all += dsmem_u64(&s.pub[slot], r);
    s.bc[0] = all;
  }
  __syncthreads();
  const unsigned long long all = s.bc[0];
  __syncthreads();
  return all;
}

// EXT: the log-probability of the chosen token and the top-n list, both of l' at T = 1 over the whole row.  result is the same
// in every CTA of the cluster, so all take the same branches.  Uses pub[9 .. 11].
__device__ __forceinline__ void sample_logprobs(SampleShared& s, const SampleArgs& a, const SampleExArgs& x, long long row, int len,
                                                int lo, uint32_t C, uint32_t rank, int result, unsigned long long best, float T,
                                                int K, float P, unsigned long long mthr) {
  SampleExShared& e = *reinterpret_cast<SampleExShared*>(reinterpret_cast<uint8_t*>(&s) + sample_ex_offset(a.slice));
  const int tid = threadIdx.x, n = x.top_n;
  const float nan = __int_as_float(0x7FC00000);
  if (result < 0) {                                 // an invalid row
    if (rank == 0) {
      if (tid == 0 && x.logprob) x.logprob[row] = nan;
      if (tid < n) { x.top_ids[row * n + tid] = -1; x.top_logprobs[row * n + tid] = nan; }
    }
    return;
  }
  const float vmax = sample_value((uint32_t)(best >> 32));
  // Z1 = sum of round(expf(l' - max) * 2^40), exact; a draw at T = 1 with nothing truncated has already summed it
  if (!(T == 0.f || K == 1) && T == 1.f && (K == 0 || K >= a.V) && P == 1.f && mthr == 0) {
    if (tid == 0) {
      unsigned long long z = 0;
      for (uint32_t r = 0; r < C; ++r) z += dsmem_u64(&s.pub[7], r);
      e.lnz = log((double)z * 0x1p-40);
    }
  } else {
    const unsigned long long z = sample_cluster_sum(s, 9, len, C, [&](int i) { return sample_weight(s.keys[i], vmax, 1.f); });
    if (tid == 0) e.lnz = log((double)z * 0x1p-40);
  }
  if (tid == 0) e.ntop = 0;
  __syncthreads();
  const double lnz = e.lnz;
  auto lp = [&](uint32_t k) {
    return k <= SAMPLE_KEY_NEG_INF ? -INFINITY : (float)((double)__fsub_rn(sample_value(k), vmax) - lnz);
  };
  if (x.logprob && tid == 0 && result >= lo && result < lo + len) x.logprob[row] = lp(s.keys[result - lo]);
  if (n == 0) return;

  // ---- top-n: the first n tokens of the order on l' (the top-k cut at K = n), -inf excluded; each CTA compacts its own
  uint32_t kth = 0;
  int kidx = 0x7FFFFFFF;
  if (n < a.V) {
    for (int i = tid; i < 256; i += SAMPLE_THREADS) { s.h1[i] = 0; s.h2[i] = 0; }   // nobody reads them since a cluster barrier
    __syncthreads();
    sample_topk_cut(s, n, len, lo, C, rank, 10, kth, kidx);
  }
  for (int i = tid; i < len; i += SAMPLE_THREADS) {
    const uint32_t k = s.keys[i];
    if (k > SAMPLE_KEY_NEG_INF && (k > kth || (k == kth && lo + i <= kidx)))
      e.top[atomicAdd(&e.ntop, 1u)] = ((unsigned long long)k << 32) | (0xFFFFFFFFu - (uint32_t)(lo + i));
  }
  sample_cluster_sync();
  if (rank != 0) return;
  if (tid == 0) {                                   // at most n survivors in the cluster
    uint32_t m = 0;
    for (uint32_t r = 0; r < C; ++r) {
      const uint32_t c = dsmem_u32(&e.ntop, r);
      for (uint32_t j = 0; j < c; ++j) e.all[m++] = dsmem_u64(&e.top[j], r);
    }
    e.nall = m;
  }
  __syncthreads();
  if (tid < n) {                                    // (key desc, index asc) is (key << 32 | ~index) desc; all distinct
    const uint32_t m = e.nall;
    if ((uint32_t)tid < m) {
      const unsigned long long v = e.all[tid];
      uint32_t pos = 0;
      for (uint32_t j = 0; j < m; ++j) pos += e.all[j] > v;
      x.top_ids[row * n + pos] = (int)(0xFFFFFFFFu - (uint32_t)v);
      x.top_logprobs[row * n + pos] = lp((uint32_t)(v >> 32));
    } else {
      x.top_ids[row * n + tid] = -1;
      x.top_logprobs[row * n + tid] = -INFINITY;
    }
  }
}

// One row per cluster; sample_kernel and sample_draft_kernel are its instances.  DRAFT: the row has one candidate token
// drafts[row] (-1: none), accepted or replaced by the rule of atom_sample_draft_f16 (DESIGN section 5.7); never with PEN.
// (the drafts pointer is a pack, empty without DRAFT: an unused parameter changes how the other instances are scheduled)
template <bool PEN, bool EXT, bool DRAFT, typename... Drafts>
__device__ __forceinline__ void sample_row(const SampleArgs a, int pdl, const SampleExArgs x, Drafts... drafts) {
  extern __shared__ __align__(16) uint8_t smem_s[];
  SampleShared& s = *reinterpret_cast<SampleShared*>(smem_s);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t rank = cluster_ctarank(), C = cluster_nctarank();
  const long long row = blockIdx.x / C;
  const int lo = (int)rank * a.slice, len = max(0, min(a.V - lo, a.slice));
  if (pdl) { griddep_launch_dependents(); griddep_wait(); }

  // ---- load the slice as keys (of the penalised logits); the row maximum (first index of), finite count, NaN / +inf (raw)
  const unsigned short* src = reinterpret_cast<const unsigned short*>(a.logits + row * a.ld + lo);
  unsigned long long best = 0;
  uint32_t finite = 0, invalid = 0;
  int slot = -1;
  float rp = 1.f, fp = 0.f, pp = 0.f;
  const uint16_t* tab = nullptr;
  if constexpr (PEN) {
    slot = x.slots[row]; rp = x.rep[row]; fp = x.freq[row]; pp = x.pres[row];
    if (slot >= 0) tab = x.table + slot * x.table_ld + lo;
  }
#pragma unroll 8
  for (int i = tid; i < len; i += SAMPLE_THREADS) {
    const unsigned short h = __ldg(src + i);
    const uint32_t k0 = sample_key(h);
    uint32_t k = k0;
    if constexpr (PEN) { if (tab) k = sample_key(sample_penalise(h, tab[i], rp, fp, pp)); }
    s.keys[i] = (uint16_t)k;
    invalid |= (uint32_t)(k0 > SAMPLE_KEY_MAX_FINITE || k0 < SAMPLE_KEY_NEG_INF);
    finite += (uint32_t)(k0 > SAMPLE_KEY_NEG_INF);
    best = max(best, ((unsigned long long)k << 32) | (0xFFFFFFFFu - (uint32_t)(lo + i)));
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    best = max(best, __shfl_xor_sync(0xFFFFFFFFu, best, o));
    finite += __shfl_xor_sync(0xFFFFFFFFu, finite, o);
    invalid |= __shfl_xor_sync(0xFFFFFFFFu, invalid, o);
  }
  if (lane == 0) { s.red[warp] = best; s.redu[warp] = finite; s.redu[SAMPLE_WARPS + warp] = invalid; }
  for (int i = tid; i < 256; i += SAMPLE_THREADS) { s.h1[i] = 0; s.h2[i] = 0; s.w1[i] = 0; s.w2[i] = 0; }
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

  const float T = a.temperature[row], P = a.top_p[row];
  const int K = a.top_k[row];
  bool bad_param = !(T >= 0.f) || isinf(T) || K < 0 || !(P > 0.f && P <= 1.f);
  if constexpr (PEN) bad_param = bad_param || !(rp > 0.f) || isinf(rp) || !isfinite(fp) || !isfinite(pp);
  int d = -1;
  if constexpr (DRAFT) {
    d = (drafts[row], ...);
    bad_param = bad_param || d < -1 || d >= a.V;
  }
  float M = 0.f;
  if constexpr (EXT) {
    if (x.min_p) M = x.min_p[row];
    bad_param = bad_param || !(M >= 0.f && M <= 1.f);
  }
  // min-p: a token whose weight is below ceil(m * 2^40) weighs 0 (the top token weighs exactly 2^40)
  const unsigned long long mthr = EXT ? (unsigned long long)ceil((double)M * 1099511627776.0) : 0ull;
  auto weight = [&](uint32_t k, float vmax) {
    const unsigned long long w = sample_weight(k, vmax, T);
    if constexpr (EXT) return w >= mthr ? w : 0ull;
    return w;
  };
  int result;
  if (bad_row || bad_param) {
    result = -1;
  } else if (T == 0.f || K == 1) {
    result = (int)(0xFFFFFFFFu - (uint32_t)(best & 0xFFFFFFFFull));
  } else {
    // ---- top-k on the keys: keep key > kth, and key == kth at index <= kidx
    uint32_t kth = 0;
    int kidx = 0x7FFFFFFF;
    if (K > 0 && K < a.V) {
      for (int base = 0; base < len; base += SAMPLE_THREADS) {
        const int i = base + tid;
        const uint32_t bin = i < len ? (uint32_t)(s.keys[i] >> 8) : 0x100u;
        const unsigned m = __match_any_sync(0xFFFFFFFFu, bin);
        if (i < len && lane == __ffs(m) - 1) atomicAdd(&s.h1[bin], (uint32_t)__popc(m));
      }
      sample_hist_sum(s.h1, s.hfull, C);
      if (warp == 0) sample_select_desc(s.hfull, [&](uint32_t) { return (uint32_t)K; }, s);
      __syncthreads();
      const uint32_t b1 = (uint32_t)s.bc[0], above1 = (uint32_t)s.bc[1];
      for (int i = tid; i < len; i += SAMPLE_THREADS)
        if ((uint32_t)(s.keys[i] >> 8) == b1) atomicAdd(&s.h2[s.keys[i] & 0xFF], 1u);
      sample_hist_sum(s.h2, s.hfull, C);
      if (warp == 0) sample_select_desc(s.hfull, [&](uint32_t) { return (uint32_t)K - above1; }, s);
      __syncthreads();
      kth = (b1 << 8) | (uint32_t)s.bc[0];
      const unsigned long long need = (unsigned long long)K - above1 - s.bc[1];
      __syncthreads();
      const uint32_t kk = kth;
      kidx = sample_find(s, 3, len, lo, C, rank, [&](int i) { return (unsigned long long)(s.keys[i] == kk); },
                         [&](unsigned long long) { return need - 1; });
    }
    const float vmax = sample_value((uint32_t)(best >> 32));
    auto topk_keep = [&](int i, uint32_t k) { return k > kth || (k == kth && lo + i <= kidx); };

    // ---- top-p over the top-k survivors: keep the tokens whose exclusive mass, in the total order, is below ceil(p * Z)
    uint32_t pth = 0;
    int pidx = 0x7FFFFFFF;
    if (P < 1.f) {
      for (int i = tid; i < len; i += SAMPLE_THREADS) {
        const uint32_t k = s.keys[i];
        if (!topk_keep(i, k)) continue;
        const unsigned long long w = weight(k, vmax);
        if (w) atomicAdd(&s.w1[k >> 8], w);
      }
      sample_hist_sum(s.w1, s.wfull, C);
      if (warp == 0)
        sample_select_desc(s.wfull, [&](unsigned long long z) { return (unsigned long long)ceil((double)P * (double)z); }, s);
      __syncthreads();
      const uint32_t b1 = (uint32_t)s.bc[0];
      const unsigned long long above1 = s.bc[1], tp = s.bc[2];
      __syncthreads();
      for (int i = tid; i < len; i += SAMPLE_THREADS) {
        const uint32_t k = s.keys[i];
        if ((k >> 8) != b1 || !topk_keep(i, k)) continue;
        const unsigned long long w = weight(k, vmax);
        if (w) atomicAdd(&s.w2[k & 0xFF], w);
      }
      sample_hist_sum(s.w2, s.wfull, C);
      if (warp == 0) sample_select_desc(s.wfull, [&](unsigned long long) { return tp - above1; }, s);
      __syncthreads();
      pth = (b1 << 8) | (uint32_t)s.bc[0];
      const unsigned long long mass_above = above1 + s.bc[1];
      const unsigned long long wt = weight(pth, vmax);                    // > 0: its bucket holds the mass that reaches tp
      const unsigned long long ties = s.wfull[s.bc[0]] / wt;
      const unsigned long long n = min(ties, (tp - mass_above + wt - 1) / wt);
      __syncthreads();
      const uint32_t pk = pth;
      pidx = sample_find(s, 5, len, lo, C, rank,
                         [&](int i) { const uint32_t k = s.keys[i]; return (unsigned long long)(k == pk && topk_keep(i, k)); },
                         [&](unsigned long long) { return n - 1; });
    }

    // ---- the draw: inverse CDF over the kept tokens in ascending index, u = (w0 >> 11) * 2^-53, t = floor(u * Z)
    if constexpr (!DRAFT) {
      const unsigned long long u53 = philox4x64_w0(a.key[2 * row], a.key[2 * row + 1], a.counter[row]) >> 11;
      result = sample_find(
          s, 7, len, lo, C, rank,
          [&](int i) {
            const uint32_t k = s.keys[i];
            const bool keep = topk_keep(i, k) && (k > pth || (k == pth && lo + i <= pidx));
            return keep ? weight(k, vmax) : 0ull;
          },
          [&](unsigned long long z) { return (__umul64hi(u53, z) << 11) | ((u53 * z) >> 53); });
    } else {
      // the candidate d: its kept weight W_d, published by the CTA that holds it (pub[12]); the draw runs over the kept set
      // without d, so the find's total is Z' = Z - W_d.  Accept iff floor(a * Z * 2^-53) < W_d with a = (w1 >> 11); then
      // no token is found.  Otherwise the draw is rule 5's with word 0 over that set (Z' > 0: a rejection needs W_d < Z).
      const ulonglong2 w = philox4x64_w01(a.key[2 * row], a.key[2 * row + 1], a.counter[row]);
      const unsigned long long u53 = w.x >> 11, a53 = w.y >> 11;
      const uint32_t owner = d >= 0 ? (uint32_t)(d / a.slice) : C;
      if (tid == 0) {
        unsigned long long wd = 0;
        if (rank == owner) {
          const int i = d - lo;
          const uint32_t k = s.keys[i];
          if (topk_keep(i, k) && (k > pth || (k == pth && d <= pidx))) wd = weight(k, vmax);
        }
        s.pub[12] = wd;
      }
      result = sample_find(
          s, 7, len, lo, C, rank,
          [&](int i) {
            const uint32_t k = s.keys[i];
            const bool keep = topk_keep(i, k) && (k > pth || (k == pth && lo + i <= pidx)) && lo + i != d;
            return keep ? weight(k, vmax) : 0ull;
          },
          [&](unsigned long long zr) {
            if (owner < C) {
              const unsigned long long wd = dsmem_u64(&s.pub[12], owner), z = zr + wd;
              if (((__umul64hi(a53, z) << 11) | ((a53 * z) >> 53)) < wd) return ~0ull;    // accepted: nothing is found
            }
            return (__umul64hi(u53, zr) << 11) | ((u53 * zr) >> 53);
          });
      if (result < 0 && d >= 0) result = d;         // accepted (a rejection always finds a token)
      if (d >= 0 && (x.logprob || x.top_n)) {       // pub[7] summed Z - W_d: make it Z for the log-probabilities' shortcut
        if (rank == owner && tid == 0) s.pub[7] += s.pub[12];
        sample_cluster_sync();
      }
    }
  }
  if constexpr (EXT) {
    if (x.logprob || x.top_n) sample_logprobs(s, a, x, row, len, lo, C, rank, result, best, T, K, P, mthr);
  }
  sample_cluster_sync();                            // no CTA leaves while another may still read its shared memory
  if (rank == 0 && tid == 0) {
    a.out[row] = result;
    if constexpr (PEN) {                            // record the drawn token: its generated count + 1, saturating
      if (slot >= 0 && result >= 0) {
        uint16_t* e = x.table + slot * x.table_ld + result;
        const uint16_t v = *e;
        if ((v & 0x7FFFu) != 0x7FFFu) *e = (uint16_t)(v + 1);
      }
    }
  }
}

// grid (C * B), cluster (C): CTA x is rank x % C of row x / C
template <bool PEN, bool EXT>
__global__ void __launch_bounds__(SAMPLE_THREADS, 1) sample_kernel(const SampleArgs a, int pdl, const SampleExArgs x) {
  sample_row<PEN, EXT, false>(a, pdl, x);
}

// atom_sample_draft_f16: min-p and log-probabilities as sample_kernel<false, true>, and one candidate per row
__global__ void __launch_bounds__(SAMPLE_THREADS, 1) sample_draft_kernel(const SampleArgs a, int pdl, const SampleExArgs x,
                                                                         const int32_t* drafts) {
  sample_row<false, true, true>(a, pdl, x, drafts);
}

// one table slot set up for a new request (atom_sample_slot_init): CTA j zeroes entries [j * chunk, (j + 1) * chunk) of the
// row, then marks the prompt's tokens among them (bit 15, generated count 0)
constexpr int SAMPLE_INIT_THREADS = 256, SAMPLE_INIT_CHUNK = 4096;
__global__ void __launch_bounds__(SAMPLE_INIT_THREADS) sample_slot_init_kernel(uint16_t* row, long long ld, int V, const int32_t* prompt,
                                                                              int n, int pdl) {
  const long long lo = (long long)blockIdx.x * SAMPLE_INIT_CHUNK, hi = min(ld, lo + SAMPLE_INIT_CHUNK);
  if (pdl) { griddep_launch_dependents(); griddep_wait(); }
  for (long long i = lo + threadIdx.x; i < hi; i += SAMPLE_INIT_THREADS) row[i] = 0;
  __syncthreads();
  for (int j = threadIdx.x; j < n; j += SAMPLE_INIT_THREADS) {
    const int t = prompt[j];
    if (t >= lo && t < hi && t < V) row[t] = 0x8000u;
  }
}

inline int sample_cluster(int V) { return (V + SAMPLE_SLICE_MAX - 1) / SAMPLE_SLICE_MAX; }
inline int sample_slice(int V) { const int c = sample_cluster(V); return ((V + c - 1) / c + 7) & ~7; }

}  // namespace atom
