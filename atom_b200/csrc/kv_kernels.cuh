// kv_kernels.cuh -- paged INT4 KV cache: append (decode / prefill) and batch decode attention with fused RoPE.
//
// Replace AppendPagedKVCacheDecodeKernel / AppendPagedKVCachePrefillKernel
//         (/root/reference/kernels/include/flashinfer/page.cuh:119-216) and
//         BatchDecodeWithPagedKVCacheKernel (/root/reference/kernels/include/flashinfer/decode.cuh:480-689).
// Cache layout is the reference's (utils/kvcache.py:17-24):
//   data  u8  [pages][L][2][H][P][64]   two INT4 per byte, element 2j in the low nibble
//   param f16 [pages][L][2][H][P][2]    (scale, zero);  x = nibble * scale - zero   (quantization.cuh:76)
// K is stored pre-RoPE; RoPE is applied to q at position len-1 and to k at its index, with the base the caller passes.  With
// grouped-query attention H is the number of KV heads.
#pragma once
#include "ptx_sm90.cuh"

namespace atom {

struct KvArgs {
  uint8_t* data;
  __half2* param;
  const int32_t* indptr;
  const int32_t* indices;
  const int32_t* last_page_offset;
  int L, layer, H, P, B;
};

__device__ __forceinline__ size_t kv_row(const KvArgs& kv, int page, int which, int head, int entry) {
  return ((((size_t)page * kv.L + kv.layer) * 2 + which) * kv.H + head) * kv.P + entry;
}

// ---------------------------------------------------------------- K7 / K8: append
// One 16-thread group moves one (token, head): 64 B of K, 64 B of V (4 B per lane each) and the two params.
// append_indptr == nullptr: decode append (one token per sequence, at position seq_len-1).
__global__ void __launch_bounds__(256)
append_kv_kernel(KvArgs kv, const uint8_t* __restrict__ k, const uint8_t* __restrict__ v, const __half2* __restrict__ kp,
                 const __half2* __restrict__ vp, const int32_t* __restrict__ append_indptr, int total_tokens, int pdl) {
  if (pdl) { griddep_launch_dependents(); griddep_wait(); }
  const long long unit = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 4;   // (token, head)
  const int sub = threadIdx.x & 15;
  if (unit >= (long long)total_tokens * kv.H) return;
  const int tok = (int)(unit / kv.H), head = (int)(unit % kv.H);
  int b, pos;
  if (append_indptr == nullptr) {
    b = tok;
    pos = (kv.indptr[b + 1] - kv.indptr[b] - 1) * kv.P + kv.last_page_offset[b] - 1;
  } else {
    int lo = 0, hi = kv.B;                          // largest b with append_indptr[b] <= tok
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (append_indptr[mid] <= tok) lo = mid; else hi = mid; }
    b = lo;
    const int seq_len = (kv.indptr[b + 1] - kv.indptr[b] - 1) * kv.P + kv.last_page_offset[b];
    const int app = append_indptr[b + 1] - append_indptr[b];
    pos = seq_len - app + (tok - append_indptr[b]);
  }
  const int page = kv.indices[kv.indptr[b] + pos / kv.P], entry = pos % kv.P;
  const size_t rk = kv_row(kv, page, 0, head, entry), rv = kv_row(kv, page, 1, head, entry);
  const size_t src = ((size_t)tok * kv.H + head);
  reinterpret_cast<uint32_t*>(kv.data + rk * 64)[sub] = reinterpret_cast<const uint32_t*>(k + src * 64)[sub];
  reinterpret_cast<uint32_t*>(kv.data + rv * 64)[sub] = reinterpret_cast<const uint32_t*>(v + src * 64)[sub];
  if (sub == 0) { kv.param[rk] = kp[src]; kv.param[rv] = vp[src]; }
}

// ---------------------------------------------------------------- K6: batch decode
// G = query heads per KV head (1 = multi-head attention).  grid (B, Hkv): one CTA owns one (sequence, KV head).  The producer
// warp streams every page of that head ONCE (K block, V block and their params are each contiguous) into an 8-stage smem
// ring with cp.async.bulk + mbarrier complete_tx -- enough bytes in flight per SM to cover HBM latency.  The consumer warps
// (4 for G = 1, 8 otherwise) produce the G query heads hkv*G .. hkv*G+G-1: warp w = (query head w % G, page stripe w / G),
// S = consumers / G stripes, stripe s consumes pages s, s+S, ...; a stage is handed back to the producer once the G warps
// that read it have arrived.  KV bytes per step: 136 * len * Hkv -- 1/G of what a head-repeated cache would cost.
// Inside a page a lane = (token slot ts = lane/4, quarter c = lane%4) handles tokens ts, ts+8, ...: for QK it holds the RoPE
// pairs i = 16c..16c+15 (elements i and i+64), for PV the V elements 32c..32c+31.
// RoPE: with z = x_i + j x_{i+64}, rope(x, p) = z e^{j p theta_i} and q.k = Re(zq conj(zk)), so
//   score(t) = Re( [zq e^{j(len-1)theta} e^{-j pagebase theta}] * conj( zk e^{j t_lo theta} ) ):
// the bracket is advanced once per page of the stripe by the constant rotation e^{-j S P theta} (FP32, kept in smem),
// e^{j t_lo theta} comes from a smem table -- no transcendental per token (the reference evaluates __sincosf per element per
// token, decode.cuh:39-71).  The base is an argument (log2 of it); the table, the rotation and the bracket are built from it.
// The per-token arithmetic runs in packed half2: one LOP3 turns two nibbles into the halves (1024+n); HSUB2 makes them
// exact; dequant and rotation are HFMA2 on nibble couples (j, j+4); the q.k products are accumulated in FP32 (FP16
// inputs, exact product, FP32 sum); scores, softmax statistics, the page-level rescale and the output accumulators stay
// FP32 (V is accumulated in half2 only within one page).  An
// all-FP32 version of this kernel executed 75 M warp instructions per layer, 36 % of them nibble extraction/conversion.
// Softmax is blocked per page; V dequant is folded: sum_t p_t (n s_t - z_t) = sum_t (p_t s_t) n - sum_t p_t z_t.
// Split-KV (kSplit): grid (B, Hkv, C) with cluster dims (1, 1, C), C = %cluster_nctarank in {2, 4, 8}.  The page striping extends
// over the cluster: CTA rank r owns the global stripes r*S + s, and global stripe r*S + s takes pages r*S + s + k*S*C, so its
// bracket starts at (len-1 - (r*S + s) P) theta and steps by e^{-j S C P theta}.  The CTA's stripe merge is left un-normalised:
// (m, d, acc[32]) per (head g, quarter c) unit in the (then idle) bracket area; after a cluster barrier every rank combines its
// share of the G*4 units x 8 float4 chunks over ranks 0..C-1 in rank order (FP32, all DSMEM loads in flight together),
// normalises and stores; a second cluster barrier keeps every CTA resident while its shared memory is read.
// Cascade decode (Pre = DecPrefix, see cascade_kernels.cuh): a row of a prefix group starts at its first private page -- the page
// loop and the query bracket skip the row's shared_pages[b] leading pages -- and before the stripe merge each query head folds
// in the un-normalised prefix partials (m, d, acc[128]) the prefix pass left for it, in chunk order.  A row outside any group
// (shared_pages 0) computes exactly what the unsplit kernel computes.
constexpr int DEC_STAGES = 8;
constexpr int DEC_PART = 130;                       // floats per prefix partial: m, d, acc[128]

struct DecPrefix {
  const int32_t* group_indptr;      // [groups + 1]
  const int32_t* group_members;     // rows of each group
  const int32_t* shared_pages;      // [B] leading pages row b shares with its group (0: no group)
  float* part;                      // [B][Hq][nchunks][DEC_PART]
  int nchunks;
};
// the prefix pass's tiling of a shared prefix: `tiles` 64-token tiles, `per` consecutive tiles per chunk (the last chunks may
// be empty); fixed by the shared page count and the host-chosen chunk count alone
__host__ __device__ __forceinline__ int dec_prefix_tiles(int shared_pages, int P) { return (shared_pages * P + 63) / 64; }
__host__ __device__ __forceinline__ int dec_prefix_per(int tiles, int nchunks) { return (tiles + nchunks - 1) / nchunks; }
// leading pages of row b the prefix pass covers: DecPrefix::shared_pages[b], or none (the plain decode kernel).  The kernel adds it
// where a page index starts instead of shifting its page range once: that form changed the PTX register numbering, and so the
// schedule, of the split-KV instantiations, which must stay the code they were.
template <typename... Pre>
__device__ __forceinline__ int dec_shared_pages(int b, const Pre&... pre) {
  if constexpr (sizeof...(Pre) == 1) return (pre.shared_pages[b], ...);
  else return 0;
}

// consumer warps of batch_decode_kernel<G, ...>: four page stripes for G = 1 (4 CTAs per SM), G heads x 8/G stripes otherwise
// (2 CTAs per SM): 16 consumer warps per SM either way
__host__ __device__ constexpr int dec_consumers(int G) { return G == 1 ? 4 : 8; }
__host__ __device__ constexpr int dec_threads(int G) { return 32 * (dec_consumers(G) + 1); }

// dynamic shared memory of batch_decode_kernel<G, ...>, in the order the kernel carves it up
inline size_t batch_decode_smem_bytes(int G, int page_size) {
  const int nc = dec_consumers(G);
  return (size_t)DEC_STAGES * (136 * page_size)      // page ring: K | V | K params | V params
         + (size_t)8 * page_size * 4 * 8             // tabh
         + 64 * 8                                    // stepr
         + nc * 64 * 8                               // brk
         + nc * 4 * 8 * 8                            // brkh
         + nc * 4 * 34 * 4                           // merge
         + 2 * DEC_STAGES * 8 + 128;                 // full / empty barriers, slack
}

__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// Nibbles q and q+4 of `w` as exact halves, one LOP3 + one HSUB2 per couple and one shift per word:
//   q even: ((w >> 4q) & 0x000F000F) | 0x64006400 = (1024 + n_q, 1024 + n_{q+4})           -> minus 1024 = n
//   q odd : ((w >> 4(q-1)) & 0x00F000F0) | 0x64006400 = (1024 + 16 n_q, 1024 + 16 n_{q+4})  -> minus 1024 = 16 n
// (a nibble in mantissa bits 4..7 is worth 16 units of the 1024 binade).  The caller folds the 1/16 of the odd couples into
// the factor it multiplies them with (scale / 16, exact).  w8 = w >> 8 serves q = 2, 3.
__device__ __forceinline__ __half2 nib2x(uint32_t w, uint32_t w8, int q) {
  const uint32_t src = (q & 2) ? w8 : w;
  uint32_t u;      // (src & mask) | magic as ONE LOP3 (the C expression compiles to two: each can carry only one immediate)
  asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(u) : "r"(src), "r"((q & 1) ? 0x00F000F0u : 0x000F000Fu), "r"(0x64006400u));
  return __hsub2(*reinterpret_cast<const __half2*>(&u), __half2half2(__ushort_as_half(0x6400)));
}

// acc += a * b with FP16 inputs, an exact product and FP32 accumulation: Hopper has no mixed-precision scalar FMA, so the
// halves are widened first (the FP32 product of two halves is exact inside the fma, one rounding in all)
__device__ __forceinline__ float fhfma(__half a, __half b, float acc) { return fmaf(__half2float(a), __half2float(b), acc); }

// A lane accumulates the V sums of at most DEC_FP16_RUN of its tokens in half2 before adding them to its FP32 accumulators.
// Each token adds at most 15 * p * (V scale), with p <= 2^6 under the lazy rescale, so a run stays below 4 * 960 * scale: finite
// for V scales below 17 at every page size (P <= 32 has at most four tokens per lane and page; P > 32 flushes after four).
constexpr int DEC_FP16_RUN = 4;

// couple u of word w holds elements (8w + q, 8w + q + 4): move the half2 V sums of a run into the FP32 accumulators
__device__ __forceinline__ void flush_pv(float (&acc)[32], __half2 (&pv)[16]) {
#pragma unroll
  for (int u = 0; u < 16; ++u) {
    const float2 f = __half22float2(pv[u]);
    acc[8 * (u >> 2) + (u & 3)] += f.x;
    acc[8 * (u >> 2) + (u & 3) + 4] += f.y;
    pv[u] = __half2half2(__ushort_as_half(0));
  }
}

// Pre: empty, or one DecPrefix (the cascade's suffix pass; unsplit only).
// kMaxTpl: tokens per lane per page = P / 8 <= kMaxTpl.  kP: page size as a compile-time constant (16 / 32: the sizes the harness
// uses -- all table strides and the token loops become immediates) or 0 = read it from the arguments.  kSplit: the sequence's
// pages are spread over a cluster of C CTAs (see above); false is the one-CTA-per-(sequence, KV head) kernel.
template <int G, int kMaxTpl, int kP, bool kSplit, typename... Pre>
__global__ void __launch_bounds__(dec_threads(G), G == 1 ? 4 : 2)
batch_decode_kernel(__half* __restrict__ o, const __half* __restrict__ q, KvArgs kv, float log2_theta, int pdl, Pre... pre) {
  static_assert(G == 1 || G == 2 || G == 4 || G == 8, "the consumer warps are split into G heads x S page stripes");
  constexpr bool kPre = sizeof...(Pre) == 1;
  static_assert(sizeof...(Pre) <= 1 && !(kPre && kSplit), "the cascade's suffix pass takes one DecPrefix and is unsplit");
  constexpr int kConsumers = dec_consumers(G), kThreads = dec_threads(G), S = kConsumers / G;
  int rank = 0, nranks = 1;                                        // split-KV: this CTA's rank and the cluster size C
  if constexpr (kSplit) { rank = (int)cluster_ctarank(); nranks = (int)cluster_nctarank(); }
  extern __shared__ __align__(128) uint8_t smem_d[];
  if (pdl) { griddep_launch_dependents(); griddep_wait(); }      // q and the newest KV entry come from the preceding kernels
  const int P = kP ? kP : kv.P;
  const int stage_bytes = 2 * 64 * P + 2 * 4 * P;                   // K | V | K params | V params
  uint8_t* ring = smem_d;
  uint2* tabh = reinterpret_cast<uint2*>(smem_d + DEC_STAGES * stage_bytes);    // [8 couples][P][4 quarters] (cos2, sin2) half2
  float2* stepr = reinterpret_cast<float2*>(tabh + 8 * P * 4);     // [64]     e^{-j S P theta_i}
  float2* brk = stepr + 64;                                         // [warps][64] FP32 query bracket per warp
  uint2* brkh = reinterpret_cast<uint2*>(brk + kConsumers * 64);   // [warps][4 quarters][8 couples] (re2, im2) half2 of the page in hand
  float* merge = reinterpret_cast<float*>(brkh + kConsumers * 4 * 8);           // [warps][4 quarters][34]
  uint64_t* full = reinterpret_cast<uint64_t*>(merge + kConsumers * 4 * 34);
  uint64_t* empty = full + DEC_STAGES;

  const int b = blockIdx.x, hkv = blockIdx.y, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ts = lane >> 2, c = lane & 3;
  const int g = warp % G, stripe = warp / G;                       // (the producer warp does not use them)
  const int Hq = kv.H * G;
  const int page_begin = kv.indptr[b], npages = kv.indptr[b + 1] - page_begin;
  const int last_valid = kv.last_page_offset[b];
  const int seq_len = (npages - 1) * P + last_valid;
  const float kFreqStep = log2_theta / 64.f;
  constexpr float kSmScale = 0.08838834764831845f * 1.4426950408889634f;   // 1/sqrt(128) * log2(e)

  if (tid == 0) {
    for (int i = 0; i < DEC_STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], G); }
    fence_barrier_init();
  }
  // table entry (u, tl, c): couple u = (j_a, j_a+4) with j_a = 8(u/4) + u%4, pair index i = 16c + j.  For a fixed u the
  // 32 lanes (tl = ts + 8k, c) of a warp read 32 consecutive 8-B words: conflict free.
  for (int e = tid; e < 8 * P * 4; e += kThreads) {
    const int cc = e & 3, tl = (e >> 2) % P, u = e / (4 * P);
    const int ja = 8 * (u >> 2) + (u & 3);
    float sa, ca, sb, cb;
    sincosf((float)tl * exp2f(-(float)(16 * cc + ja) * kFreqStep), &sa, &ca);
    sincosf((float)tl * exp2f(-(float)(16 * cc + ja + 4) * kFreqStep), &sb, &cb);
    const __half2 c2 = __floats2half2_rn(ca, cb), s2 = __floats2half2_rn(sa, sb);
    tabh[e] = make_uint2(*reinterpret_cast<const uint32_t*>(&c2), *reinterpret_cast<const uint32_t*>(&s2));
  }
  if (tid < 64) {
    const float f = exp2f(-(float)tid * kFreqStep);
    float sn, cs; sincosf((float)(S * nranks * P) * f, &sn, &cs);
    stepr[tid] = make_float2(cs, -sn);
  }
  if (warp < kConsumers) {
    // FP32 query bracket of this warp: zq e^{j (len-1 - (rank*S + stripe)*P) theta} of query head hkv*G + g.  Lane (ts, c) owns couple
    // u = ts of quarter c: the pairs ja = 8(u/4) + u%4 and ja + 4; it keeps the FP32 values in smem and publishes their half2
    // packing.
    const __half* qh = q + ((size_t)b * Hq + hkv * G + g) * 128;
    const int ja = 8 * (ts >> 2) + (ts & 3);
    float2 v2[2];
#pragma unroll
    for (int x = 0; x < 2; ++x) {
      const int i = 16 * c + ja + 4 * x;
      const float f = exp2f(-(float)i * kFreqStep);
      const float xr = __half2float(qh[i]), xi = __half2float(qh[i + 64]);
      float sn, cs;
      if constexpr (kPre) sincosf((float)(seq_len - 1 - (dec_shared_pages(b, pre...) + stripe) * P) * f, &sn, &cs);
      else sincosf((float)(seq_len - 1 - (rank * S + stripe) * P) * f, &sn, &cs);
      v2[x] = make_float2(xr * cs - xi * sn, xi * cs + xr * sn);
      brk[warp * 64 + i] = v2[x];
    }
    const __half2 re2 = __floats2half2_rn(v2[0].x, v2[1].x), im2 = __floats2half2_rn(v2[0].y, v2[1].y);
    brkh[(warp * 4 + c) * 8 + ts] = make_uint2(*reinterpret_cast<const uint32_t*>(&re2), *reinterpret_cast<const uint32_t*>(&im2));
  }
  __syncthreads();

  if (warp == kConsumers) {
    // ------------------------------------------------------------ producer: one elected lane streams the pages
    if (lane == 0) {
      // the CTA's lp-th page (its ring slot order) is global page lp, or split (lp / S) * S * C + rank * S + lp % S
      for (int lp = 0;; ++lp) {
        const int pg = kSplit ? (lp / S) * S * nranks + rank * S + lp % S : lp + dec_shared_pages(b, pre...);
        if (pg >= npages) break;
        const int s = lp % DEC_STAGES;
        mbar_wait(&empty[s], ((lp / DEC_STAGES) & 1) ^ 1);
        const int page = kv.indices[page_begin + pg];
        const size_t rk = kv_row(kv, page, 0, hkv, 0), rv = kv_row(kv, page, 1, hkv, 0);
        uint8_t* st = ring + s * stage_bytes;
        mbar_arrive_expect_tx(&full[s], stage_bytes);
        bulk_g2s(st, kv.data + rk * 64, 64 * P, &full[s]);
        bulk_g2s(st + 64 * P, kv.data + rv * 64, 64 * P, &full[s]);
        bulk_g2s(st + 128 * P, kv.param + rk, 4 * P, &full[s]);
        bulk_g2s(st + 132 * P, kv.param + rv, 4 * P, &full[s]);
      }
    }
    if constexpr (kSplit) {        // the cluster barriers are CTA-wide (.aligned): the producer warp joins both
      __syncwarp();
      cluster_arrive(); cluster_wait();
      cluster_arrive(); cluster_wait();
    }
    return;
  }

  // -------------------------------------------------------------- consumers
  float m = -5e4f, d = 0.f, zsum = 0.f, acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
  const int tpl = P >> 3;                                          // tokens per lane per page
  float2* mybrk = brk + warp * 64 + 16 * c;
  uint2* mybrkh = brkh + (warp * 4 + c) * 8;

  // global page pg of the stripe is the CTA's lp-th (lp = pg unsplit)
  for (int pg = dec_shared_pages(b, pre...) + rank * S + stripe, lp = stripe; pg < npages; pg += S * nranks, lp += S) {
    const int s = lp % DEC_STAGES;
    const int valid = (pg == npages - 1) ? last_valid : P;
    // this page's query bracket as half2 couples (j, j+4); then every lane advances its own couple to the stripe's next
    // page (FP32 in smem, constant rotation e^{-j S P theta}) and publishes the new half2 packing
    __half2 qre2[8], qim2[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const uint2 t = mybrkh[u];
      qre2[u] = *reinterpret_cast<const __half2*>(&t.x);
      qim2[u] = *reinterpret_cast<const __half2*>(&t.y);
    }
    __syncwarp();
    {
      const int ja = 8 * (ts >> 2) + (ts & 3);
      float2 v2[2];
#pragma unroll
      for (int x = 0; x < 2; ++x) {
        const float2 st2 = stepr[16 * c + ja + 4 * x], v = mybrk[ja + 4 * x];
        v2[x] = make_float2(v.x * st2.x - v.y * st2.y, v.y * st2.x + v.x * st2.y);
        mybrk[ja + 4 * x] = v2[x];
      }
      const __half2 re2 = __floats2half2_rn(v2[0].x, v2[1].x), im2 = __floats2half2_rn(v2[0].y, v2[1].y);
      mybrkh[ts] = make_uint2(*reinterpret_cast<const uint32_t*>(&re2), *reinterpret_cast<const uint32_t*>(&im2));
    }
    // (the __syncwarp() at the end of the page orders these writes before the next page's reads)
    mbar_wait(&full[s], (lp / DEC_STAGES) & 1);
    const uint8_t* st = ring + s * stage_bytes;
    const uint8_t* kblk = st;
    const uint8_t* vblk = st + 64 * P;
    const __half2* kpar = reinterpret_cast<const __half2*>(st + 128 * P);
    const __half2* vpar = reinterpret_cast<const __half2*>(st + 132 * P);

    // ---- scores of this lane's tokens
    float x[kMaxTpl];
    float xmax = -5e4f;
#pragma unroll
    for (int i = 0; i < kMaxTpl; ++i) {
      x[i] = 0.f;
      if (i < tpl) {
        const int tl = ts + 8 * i;
        const uint8_t* kr = kblk + tl * 64;
        // the two 8-B halves are read in opposite order by alternate token pairs so that one instruction touches both
        // 32-B halves of the 64-B rows (2-way instead of 4-way bank conflict on the linear page layout)
        const bool swp = (ts & 2) != 0;
        const uint2 k_a = *reinterpret_cast<const uint2*>(kr + (swp ? 32 : 0) + c * 8);
        const uint2 k_b = *reinterpret_cast<const uint2*>(kr + (swp ? 0 : 32) + c * 8);
        const uint2 k_lo = swp ? k_b : k_a;                                    // elements 16c .. 16c+15   (re)
        const uint2 k_hi = swp ? k_a : k_b;                                    // elements 64+16c ..       (im)
        const __half2 kp = kpar[tl];
        const __half2 ks2 = __half2half2(__low2half(kp)), kz2 = __hneg2(__half2half2(__high2half(kp)));
        const __half2 ks2o = __hmul2(ks2, __half2half2(__ushort_as_half(0x2C00)));   // scale / 16 for the odd couples (nib2x)
        const uint32_t kl8[2] = {k_lo.x >> 8, k_lo.y >> 8}, kh8[2] = {k_hi.x >> 8, k_hi.y >> 8};
        const uint2* trow = tabh + tl * 4 + c;
        float xa = 0.f, xb = 0.f;        // q.k is accumulated in FP32 (the reference's compute_qk is all-FP32, decode.cuh:92-124)
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const uint32_t wl = (u < 4) ? k_lo.x : k_lo.y, wh = (u < 4) ? k_hi.x : k_hi.y;
          const __half2 sc2 = (u & 1) ? ks2o : ks2;
          const __half2 kre = __hfma2(nib2x(wl, kl8[u >> 2], u & 3), sc2, kz2), kim = __hfma2(nib2x(wh, kh8[u >> 2], u & 3), sc2, kz2);
          const uint2 t = trow[u * P * 4];
          const __half2 c2 = *reinterpret_cast<const __half2*>(&t.x), s2 = *reinterpret_cast<const __half2*>(&t.y);
          const __half2 rr = __hfma2(kre, c2, __hneg2(__hmul2(kim, s2)));      // Re(zk e^{j t_lo theta})
          const __half2 ri = __hfma2(kim, c2, __hmul2(kre, s2));
          xa = fhfma(__low2half(qre2[u]), __low2half(rr), xa);  xb = fhfma(__high2half(qre2[u]), __high2half(rr), xb);
          xa = fhfma(__low2half(qim2[u]), __low2half(ri), xa);  xb = fhfma(__high2half(qim2[u]), __high2half(ri), xb);
        }
        float xs = xa + xb;
        xs += __shfl_xor_sync(0xffffffffu, xs, 1);
        xs += __shfl_xor_sync(0xffffffffu, xs, 2);
        x[i] = xs * kSmScale;
        if (tl < valid) xmax = fmaxf(xmax, x[i]);
      }
    }
    // ---- one rescale per page, then p * v with the dequant folded; V partial sums of the page in half2, DEC_FP16_RUN tokens at most
    // The running maximum only moves when it is exceeded by more than 2^6: any m gives the same softmax, the weights then reach
    // at most 64 (times 15 x the V scale per token: inside FP16 for a run of four tokens up to V scales of 17), and with 32 lanes
    // per warp "some lane saw a new maximum" would otherwise be true on almost every page -- the 34-FMUL rescale below now runs a
    // few times per sequence.
    const float m_new = (xmax > m + 6.f) ? xmax : m;
    const float sc = exp2f(m - m_new);
    m = m_new;
    if (__any_sync(0xffffffffu, sc != 1.f)) {     // once the running maxima have settled no lane of the warp rescales
      d *= sc; zsum *= sc;
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[i] *= sc;
    }
    __half2 pv[16];
#pragma unroll
    for (int u = 0; u < 16; ++u) pv[u] = __half2half2(__ushort_as_half(0));
#pragma unroll
    for (int i = 0; i < kMaxTpl; ++i) {
      if (i < tpl) {
        const int tl = ts + 8 * i;
        if (tl < valid) {
          const uint4 vw = *reinterpret_cast<const uint4*>(vblk + tl * 64 + c * 16);
          const float2 vp = __half22float2(vpar[tl]);
          const float p = exp2f(x[i] - m_new);
          d += p;
          zsum = fmaf(p, vp.y, zsum);
          const __half2 ps2 = __float2half2_rn(p * vp.x), ps2o = __float2half2_rn(p * vp.x * 0.0625f);
          const uint32_t w4[4] = {vw.x, vw.y, vw.z, vw.w};
          const uint32_t w8[4] = {vw.x >> 8, vw.y >> 8, vw.z >> 8, vw.w >> 8};
#pragma unroll
          for (int u = 0; u < 16; ++u) pv[u] = __hfma2(nib2x(w4[u >> 2], w8[u >> 2], u & 3), (u & 1) ? ps2o : ps2, pv[u]);
        }
      }
      if (kMaxTpl > DEC_FP16_RUN && i % DEC_FP16_RUN == DEC_FP16_RUN - 1 && i + 1 < tpl) flush_pv(acc, pv);   // P > 32
    }
    flush_pv(acc, pv);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);          // the G-th arrival frees the stage
  }
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] -= zsum;      // sum_t p_t z_t is common to all elements of the head

  // merge the 8 token-slot states of the warp (same quarter c: lanes differ in bits 2..4)
#pragma unroll
  for (int off = 4; off < 32; off <<= 1) {
    const float m_o = __shfl_xor_sync(0xffffffffu, m, off), d_o = __shfl_xor_sync(0xffffffffu, d, off);
    const float m_new = fmaxf(m, m_o);
    const float s_a = exp2f(m - m_new), s_b = exp2f(m_o - m_new);
    d = d * s_a + d_o * s_b;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const float a_o = __shfl_xor_sync(0xffffffffu, acc[i], off);
      acc[i] = acc[i] * s_a + a_o * s_b;
    }
    m = m_new;
  }
  if (ts == 0) {
    float* dst = merge + (warp * 4 + c) * 34;
    dst[0] = m; dst[1] = d;
#pragma unroll
    for (int i = 0; i < 32; ++i) dst[2 + i] = acc[i];
  }
  asm volatile("bar.sync 1, %0;" ::"n"(32 * kConsumers) : "memory");     // the consumer warps (the producer warp has left)
  // warp g (< G) combines the S stripes of query head g: they sit in warps g, g + G, ...
  if (warp < G && ts == 0) {
    float mm = -5e4f;
#pragma unroll
    for (int w = 0; w < S; ++w) mm = fmaxf(mm, merge[((w * G + warp) * 4 + c) * 34]);
    float dd = 0.f, out[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) out[i] = 0.f;
    if constexpr (kPre) {      // the prefix partials of query head hkv*G + warp, chunk by chunk, then the stripes
      const DecPrefix& px = (pre, ...);
      const int tiles = dec_prefix_tiles(dec_shared_pages(b, pre...), P), per = dec_prefix_per(tiles, px.nchunks);
      const int nck = tiles ? (tiles + per - 1) / per : 0;
      const float* part = px.part + ((size_t)b * Hq + hkv * G + warp) * px.nchunks * DEC_PART;
      for (int k = 0; k < nck; ++k) mm = fmaxf(mm, part[k * DEC_PART]);
      for (int k = 0; k < nck; ++k) {
        const float* src = part + k * DEC_PART;
        const float sx = exp2f(src[0] - mm);
        dd = fmaf(src[1], sx, dd);
#pragma unroll
        for (int i = 0; i < 32; ++i) out[i] = fmaf(src[2 + 32 * c + i], sx, out[i]);
      }
    }
#pragma unroll
    for (int w = 0; w < S; ++w) {
      const float* src = merge + ((w * G + warp) * 4 + c) * 34;
      const float sx = exp2f(src[0] - mm);
      dd = fmaf(src[1], sx, dd);
#pragma unroll
      for (int i = 0; i < 32; ++i) out[i] = fmaf(src[2 + i], sx, out[i]);
    }
    if constexpr (kSplit) {
      // un-normalised (m, d, acc) of unit (g, c) for the cluster merge, in the bracket area the page loop no longer uses (16-B
      // aligned float4 chunks: acc of unit u at u*32, (m, d) at G*128 + 2u; G*544 bytes <= brk + brkh)
      const int u = warp * 4 + c;
      float* cmb = reinterpret_cast<float*>(brk);
      *reinterpret_cast<float2*>(cmb + G * 128 + 2 * u) = make_float2(mm, dd);
#pragma unroll
      for (int i = 0; i < 32; i += 4) *reinterpret_cast<float4*>(cmb + u * 32 + i) = make_float4(out[i], out[i + 1], out[i + 2], out[i + 3]);
    } else {
      const float inv = 1.f / dd;
      __half* dst = o + ((size_t)b * Hq + hkv * G + warp) * 128 + 32 * c;
#pragma unroll
      for (int i = 0; i < 32; i += 2)
        *reinterpret_cast<__half2*>(dst + i) = __floats2half2_rn(out[i] * inv, out[i + 1] * inv);
    }
  }
  if constexpr (kSplit) {
    __syncwarp();
    cluster_arrive(); cluster_wait();          // every rank's units are staged
    // rank r combines items r*per .. r*per + per-1 of the G*4 units x 8 float4 chunks: over ranks 0..C-1 in rank order, FP32
    const int per = G * 32 / nranks;
    if (tid < per) {
      const int it = rank * per + tid, u = it >> 3, k = it & 7;
      const float* cmb = reinterpret_cast<const float*>(brk);
      const uint32_t a_md = smem_u32(cmb + G * 128 + 2 * u), a_acc = smem_u32(cmb + u * 32 + 4 * k);
      float2 md[8];
      float4 a[8];
#pragma unroll
      for (int r = 0; r < 8; ++r)
        if (r < nranks) { md[r] = ld_dsmem_v2(mapa_shared(a_md, r)); a[r] = ld_dsmem_v4(mapa_shared(a_acc, r)); }
      float mm = -5e4f;
#pragma unroll
      for (int r = 0; r < 8; ++r)
        if (r < nranks) mm = fmaxf(mm, md[r].x);
      float dd = 0.f;
      float4 out = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        if (r < nranks) {
          const float sx = exp2f(md[r].x - mm);
          dd = fmaf(md[r].y, sx, dd);
          out.x = fmaf(a[r].x, sx, out.x); out.y = fmaf(a[r].y, sx, out.y);
          out.z = fmaf(a[r].z, sx, out.z); out.w = fmaf(a[r].w, sx, out.w);
        }
      }
      const float inv = 1.f / dd;
      const __half2 lo = __floats2half2_rn(out.x * inv, out.y * inv), hi = __floats2half2_rn(out.z * inv, out.w * inv);
      __half* dst = o + ((size_t)b * Hq + hkv * G + (u >> 2)) * 128 + 32 * (u & 3) + 4 * k;
      *reinterpret_cast<uint2*>(dst) = make_uint2(*reinterpret_cast<const uint32_t*>(&lo), *reinterpret_cast<const uint32_t*>(&hi));
    }
    __syncwarp();
    cluster_arrive(); cluster_wait();          // no CTA leaves while its units may still be read
  }
}

}  // namespace atom
