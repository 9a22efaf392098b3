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

// grid (C * B), cluster (C): CTA x is rank x % C of row x / C
__global__ void __launch_bounds__(SAMPLE_THREADS, 1) sample_kernel(const SampleArgs a, int pdl) {
  extern __shared__ __align__(16) uint8_t smem_s[];
  SampleShared& s = *reinterpret_cast<SampleShared*>(smem_s);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t rank = cluster_ctarank(), C = cluster_nctarank();
  const long long row = blockIdx.x / C;
  const int lo = (int)rank * a.slice, len = max(0, min(a.V - lo, a.slice));
  if (pdl) { griddep_launch_dependents(); griddep_wait(); }

  // ---- load the slice as keys; the row maximum (first index of), finite count, NaN / +inf
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
  const bool bad_param = !(T >= 0.f) || isinf(T) || K < 0 || !(P > 0.f && P <= 1.f);
  int result;
  if (bad_row || bad_param) {
    result = -1;
  } else if (T == 0.f || K == 1) {
    result = (int)(0xFFFFFFFFu - (uint32_t)(best & 0xFFFFFFFFull));
  } else {
    // ---- top-k on the raw keys: keep key > kth, and key == kth at index <= kidx
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
        const unsigned long long w = sample_weight(k, vmax, T);
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
        const unsigned long long w = sample_weight(k, vmax, T);
        if (w) atomicAdd(&s.w2[k & 0xFF], w);
      }
      sample_hist_sum(s.w2, s.wfull, C);
      if (warp == 0) sample_select_desc(s.wfull, [&](unsigned long long) { return tp - above1; }, s);
      __syncthreads();
      pth = (b1 << 8) | (uint32_t)s.bc[0];
      const unsigned long long mass_above = above1 + s.bc[1];
      const unsigned long long wt = sample_weight(pth, vmax, T);          // > 0: its bucket holds the mass that reaches tp
      const unsigned long long ties = s.wfull[s.bc[0]] / wt;
      const unsigned long long n = min(ties, (tp - mass_above + wt - 1) / wt);
      __syncthreads();
      const uint32_t pk = pth;
      pidx = sample_find(s, 5, len, lo, C, rank,
                         [&](int i) { const uint32_t k = s.keys[i]; return (unsigned long long)(k == pk && topk_keep(i, k)); },
                         [&](unsigned long long) { return n - 1; });
    }

    // ---- the draw: inverse CDF over the kept tokens in ascending index, u = (w0 >> 11) * 2^-53, t = floor(u * Z)
    const unsigned long long u53 = philox4x64_w0(a.key[2 * row], a.key[2 * row + 1], a.counter[row]) >> 11;
    result = sample_find(
        s, 7, len, lo, C, rank,
        [&](int i) {
          const uint32_t k = s.keys[i];
          const bool keep = topk_keep(i, k) && (k > pth || (k == pth && lo + i <= pidx));
          return keep ? sample_weight(k, vmax, T) : 0ull;
        },
        [&](unsigned long long z) { return (__umul64hi(u53, z) << 11) | ((u53 * z) >> 53); });
  }
  sample_cluster_sync();                            // no CTA leaves while another may still read its shared memory
  if (rank == 0 && tid == 0) a.out[row] = result;
}

inline int sample_cluster(int V) { return (V + SAMPLE_SLICE_MAX - 1) / SAMPLE_SLICE_MAX; }
inline int sample_slice(int V) { const int c = sample_cluster(V); return ((V + c - 1) / c + 7) & ~7; }

}  // namespace atom
