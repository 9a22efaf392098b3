// prefill_kernels.cuh -- causal prefill attention over the JUST-QUANTISED INT4 K/V of the prompt tokens.
//
// Replaces the placeholder in the reference's LlamaAttention.forward (punica/models/llama.py:171-190: "HACK" --
// scaled_dot_product_attention on torch.randn K/V) and the eager version round 1 shipped (per-prompt Python loop,
// torch dequantisation, rotary_pos_emb, cuDNN SDPA).  One launch for all prompts and heads:
//   * K and V are the o4 outputs of the k/v projections (packed nibbles + (scale, zero) per token-head, exactly what
//     init_kv_i4 scatters into the page pool, page.cuh:165-216): x = nibble * scale - zero, rounded to FP16 as the
//     decode path sees it;
//   * RoPE (theta = 1e4, pairs (i, i + 64), llama.py:18-32) on q and k from a (cos, sin) table of the positions;
//   * flash-attention recurrence (online softmax in FP32, base 2), FP16 tensor-core MMAs with FP32 accumulation: the tile step
//     attn_tile_step below, which the verify and shared-prefix kernels run too.
// Two launches: kv_dequant_rope_kernel turns the packed K/V into FP16 once (K rotated), because every K/V tile is reused by
// all later query tiles of its prompt; prefill_attn_kernel is the attention proper.
// Tiling: CTA = 64 query rows of one (prompt, head), 4 warps x 16 rows; K/V in 64-token tiles through shared memory
// (K row-major [token][dim], V transposed [dim][token] so both B fragments are contiguous 32-bit loads, padded
// pitches => conflict-free).  The MMA is mma.sync.m16n8k16 (the warp-level tensor path); a wgmma variant is the
// next step for this kernel.
// Prefill over a cached prefix (prefill_attn_kernel<true>): prompt b is the tail of its cached sequence, as init_kv_i4 writes it
// (positions ctx_b .. ctx_b + L_b - 1).  Its queries also attend, without a causal mask, to the ctx_b tokens before it, which the
// kernel reads straight from the INT4 pages (no FP16 scratch grows with the context) -- see the kernel's comment.
#pragma once
#include "ptx_sm90.cuh"
#include "kv_kernels.cuh"

namespace atom {

constexpr int PF_BQ = 64, PF_BK = 64, PF_THREADS = 128;
constexpr int PF_KPITCH = 136;   // halves per K row (128 + 8): rows g, g+1.. land in different banks
constexpr int PF_VPITCH = 72;    // halves per V^T row (64 + 8)

__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}

// k4 u8 [T, H*64], kpar f16 [T, H, 2] = (scale, zero); v4 / vpar likewise (the o4 projections' outputs); pos_of_token i32 [T]
// (position of every token inside its prompt); rope float2 [max_len][64] = (cos, sin)(pos * theta_i).
// kf, vf f16 [T, H*128]: kf = RoPE(dequant(k)), vf = dequant(v); dequantised values are rounded to FP16 BEFORE the rotation:
// that is the K the decode kernel reads back from the cache (x = nibble * scale - zero, quantization.cuh:76).
__global__ void __launch_bounds__(256)
kv_dequant_rope_kernel(const uint8_t* __restrict__ k4, const __half2* __restrict__ kpar, const uint8_t* __restrict__ v4,
                       const __half2* __restrict__ vpar, const int32_t* __restrict__ pos_of_token, const float2* __restrict__ rope,
                       __half* __restrict__ kf, __half* __restrict__ vf, long long token_heads, int H) {
  const long long th = (long long)blockIdx.x * 4 + (threadIdx.x >> 6);
  const int i = threadIdx.x & 63;
  if (th >= token_heads) return;
  const int pos = pos_of_token[th / H];
  const float2 kp = __half22float2(kpar[th]), vp = __half22float2(vpar[th]), cs = rope[(size_t)pos * 64 + i];
  const uint8_t* kb = k4 + th * 64;
  const uint8_t* vb = v4 + th * 64;
  const int sh = 4 * (i & 1);
  const float k1 = __half2float(__float2half_rn((float)((kb[i >> 1] >> sh) & 0xF) * kp.x - kp.y));
  const float k2 = __half2float(__float2half_rn((float)((kb[32 + (i >> 1)] >> sh) & 0xF) * kp.x - kp.y));
  __half* ko = kf + th * 128;
  __half* vo = vf + th * 128;
  ko[i] = __float2half_rn(k1 * cs.x - k2 * cs.y);
  ko[i + 64] = __float2half_rn(k2 * cs.x + k1 * cs.y);
  vo[i] = __float2half_rn((float)((vb[i >> 1] >> sh) & 0xF) * vp.x - vp.y);
  vo[i + 64] = __float2half_rn((float)((vb[32 + (i >> 1)] >> sh) & 0xF) * vp.x - vp.y);
}

// tokens of sequence b cached before its prompt of L tokens (the page table holds seq_len_b = ctx_b + L)
__device__ __forceinline__ int prefill_ctx_len(const KvArgs& kv, int b, int L) {
  return max((kv.indptr[b + 1] - kv.indptr[b] - 1) * kv.P + kv.last_page_offset[b] - L, 0);   // < 0 only on a bad page table
}

// Context tile of prefill_attn_kernel<true>: 64 tokens of sequence b's cached prefix (KV head hk) into Ks / Vt, as
// kv_dequant_rope_kernel would have turned them into kf / vf: x = fp16(n * s - z), K rotated in FP32 at its absolute position
// from the (cos, sin) table and rounded to FP16 (the same fused multiply-adds, pinned with intrinsics).  Token slots outside
// [0, ctx) are zeros (masked by the caller).  Thread = (token tid / 2, pair half tid % 2): the RoPE pairs i = 32 hf .. 32 hf + 31
// of one token, i.e. bytes 16 hf .. 16 hf + 15 and 32 + 16 hf .. 32 + 16 hf + 15 of its K and V rows (one 16-byte load each).
// rope: the table shifted to the prompt's first position (row p = absolute position ctx + p); k0: key position of the tile's first
// slot (-ctx .. -1 are the context tokens)
__device__ __forceinline__ void prefill_ctx_tile(const KvArgs& kv, int b, int L, int hk, int k0, const float2* __restrict__ rope,
                                                 __half* Ks, __half* Vt, int tid) {
  const int ctx = prefill_ctx_len(kv, b, L);
  const int tok = tid >> 1, hf = tid & 1, kpos = k0 + tok, c = ctx + kpos;
  const bool live = c >= 0 && c < ctx;
  size_t rk = 0;
  if (live) rk = kv_row(kv, kv.indices[kv.indptr[b] + c / kv.P], 0, hk, c % kv.P);
  const size_t rv = rk + (size_t)kv.H * kv.P;                  // the V row of the same (page, layer, head, entry)
  {                                                             // K: dequantise, rotate, round, store row-major
    uint4 lo = make_uint4(0, 0, 0, 0), hi = lo;
    float2 p = make_float2(0.f, 0.f);
    if (live) {
      lo = *reinterpret_cast<const uint4*>(kv.data + rk * 64 + 16 * hf);
      hi = *reinterpret_cast<const uint4*>(kv.data + rk * 64 + 32 + 16 * hf);
      p = __half22float2(kv.param[rk]);
    }
    const float2* rp = rope + (ptrdiff_t)kpos * 64 + 32 * hf;
    const uint32_t wl[4] = {lo.x, lo.y, lo.z, lo.w}, wh[4] = {hi.x, hi.y, hi.z, hi.w};
#pragma unroll
    for (int w = 0; w < 4; ++w) {                     // pairs i = 32 hf + 8 w + e, e < 8: nibble e of word w (low and high half)
      uint32_t re[4], im[4];
#pragma unroll
      for (int e = 0; e < 8; e += 2) {
        float4 cs = make_float4(1.f, 0.f, 1.f, 0.f);
        if (live) cs = *reinterpret_cast<const float4*>(rp + 8 * w + e);
        const float a1 = __half2float(__float2half_rn(__fmaf_rn((float)((wl[w] >> (4 * e)) & 0xF), p.x, -p.y)));
        const float a2 = __half2float(__float2half_rn(__fmaf_rn((float)((wh[w] >> (4 * e)) & 0xF), p.x, -p.y)));
        const float b1 = __half2float(__float2half_rn(__fmaf_rn((float)((wl[w] >> (4 * e + 4)) & 0xF), p.x, -p.y)));
        const float b2 = __half2float(__float2half_rn(__fmaf_rn((float)((wh[w] >> (4 * e + 4)) & 0xF), p.x, -p.y)));
        re[e >> 1] = pack_h2(__fmaf_rn(a1, cs.x, -__fmul_rn(a2, cs.y)), __fmaf_rn(b1, cs.z, -__fmul_rn(b2, cs.w)));
        im[e >> 1] = pack_h2(__fmaf_rn(a1, cs.y, __fmul_rn(a2, cs.x)), __fmaf_rn(b1, cs.w, __fmul_rn(b2, cs.z)));
      }
      *reinterpret_cast<uint4*>(&Ks[tok * PF_KPITCH + 32 * hf + 8 * w]) = make_uint4(re[0], re[1], re[2], re[3]);
      *reinterpret_cast<uint4*>(&Ks[tok * PF_KPITCH + 64 + 32 * hf + 8 * w]) = make_uint4(im[0], im[1], im[2], im[3]);
    }
  }
  {                                                             // V: dequantise, round, store transposed
    uint4 lo = make_uint4(0, 0, 0, 0), hi = lo;
    float2 p = make_float2(0.f, 0.f);
    if (live) {
      lo = *reinterpret_cast<const uint4*>(kv.data + rv * 64 + 16 * hf);
      hi = *reinterpret_cast<const uint4*>(kv.data + rv * 64 + 32 + 16 * hf);
      p = __half22float2(kv.param[rv]);
    }
    const uint32_t wl[4] = {lo.x, lo.y, lo.z, lo.w}, wh[4] = {hi.x, hi.y, hi.z, hi.w};
#pragma unroll
    for (int w = 0; w < 4; ++w) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int d = 32 * hf + 8 * w + e;
        Vt[d * PF_VPITCH + tok] = __float2half_rn(__fmaf_rn((float)((wl[w] >> (4 * e)) & 0xF), p.x, -p.y));
        Vt[(d + 64) * PF_VPITCH + tok] = __float2half_rn(__fmaf_rn((float)((wh[w] >> (4 * e)) & 0xF), p.x, -p.y));
      }
    }
  }
}

__device__ __forceinline__ int prefill_ctx_len(int, int) { return 0; }                             // <false>: no cache
__device__ __forceinline__ void prefill_ctx_tile(int, int, int, int, const float2*, __half*, __half*, int) {}

constexpr float ATTN_SCALE_LOG2 = 0.08838834764831845f * 1.4426950408889634f;   // 1/sqrt(128) * log2(e), as the decode kernel

// The consumer of one 64-key tile, shared by the prefill, verify and shared-prefix kernels.  A warp owns 16 query rows of the
// m16n8k16 fragments; a thread holds rows g and g + 8 (row rr = 0, 1; g = lane / 4) and columns 2t, 2t + 1 of each 8-column
// block (t = lane % 4).  S = Q K^T from the rotated Q fragments qa and the tile in Ks (keys k0 .. k0 + 63), scaled to base 2;
// key kpos is kept for row rr where visible(rr, kpos), else -inf.  Then the online softmax in FP32 -- the quad's row maximum,
// the rescale of (o, l), P rounded to FP16 -- and O += P V from the tile in Vt.  A row that has seen no visible key yet keeps
// m = -inf; its exponentials are taken against 0, which keeps exp2(-inf - -inf) out of the recurrence (o and l stay 0).
template <typename Visible>
__device__ __forceinline__ void attn_tile_step(const uint32_t (&qa)[8][4], const __half* Ks, const __half* Vt, int k0, Visible visible,
                                               float (&o)[16][4], float& m0, float& m1, float& l0, float& l1) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  float s[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      const uint32_t b0 = *reinterpret_cast<const uint32_t*>(&Ks[(8 * j + g) * PF_KPITCH + 16 * kk + 2 * t]);
      const uint32_t b1 = *reinterpret_cast<const uint32_t*>(&Ks[(8 * j + g) * PF_KPITCH + 16 * kk + 8 + 2 * t]);
      mma_16816(s[j], qa[kk], b0, b1);
    }
  }
  float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int kpos = k0 + 8 * j + 2 * t + u;
      s[j][u] = visible(0, kpos) ? s[j][u] * ATTN_SCALE_LOG2 : -INFINITY;
      s[j][2 + u] = visible(1, kpos) ? s[j][2 + u] * ATTN_SCALE_LOG2 : -INFINITY;
      mx0 = fmaxf(mx0, s[j][u]); mx1 = fmaxf(mx1, s[j][2 + u]);
    }
  }
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
  const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
  const float base0 = mn0 == -INFINITY ? 0.f : mn0, base1 = mn1 == -INFINITY ? 0.f : mn1;
  const float a0 = exp2f(m0 - base0), a1 = exp2f(m1 - base1);
  m0 = mn0; m1 = mn1;
  float sum0 = 0.f, sum1 = 0.f;
  uint32_t pa[4][4];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float p00 = exp2f(s[j][0] - base0), p01 = exp2f(s[j][1] - base0);
    const float p10 = exp2f(s[j][2] - base1), p11 = exp2f(s[j][3] - base1);
    sum0 += p00 + p01; sum1 += p10 + p11;
    pa[j >> 1][(j & 1) * 2 + 0] = pack_h2(p00, p01);
    pa[j >> 1][(j & 1) * 2 + 1] = pack_h2(p10, p11);
  }
  l0 = l0 * a0 + sum0; l1 = l1 * a1 + sum1;
#pragma unroll
  for (int i = 0; i < 16; ++i) { o[i][0] *= a0; o[i][1] *= a0; o[i][2] *= a1; o[i][3] *= a1; }
#pragma unroll
  for (int i = 0; i < 16; ++i) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const uint32_t b0 = *reinterpret_cast<const uint32_t*>(&Vt[(8 * i + g) * PF_VPITCH + 16 * kk + 2 * t]);
      const uint32_t b1 = *reinterpret_cast<const uint32_t*>(&Vt[(8 * i + g) * PF_VPITCH + 16 * kk + 8 + 2 * t]);
      mma_16816(o[i], pa[kk], b0, b1);
    }
  }
}

// Q fragments of a thread's two rows (row rr: q row qr[rr], position pos[rr]) rotated at positions read on the device, so a
// captured graph replays with new lengths: the angle pos * theta^(-d/64) by FP32 sincosf, the rotation in FP32, rounded to FP16
// once (the decode kernel's arithmetic)
__device__ __forceinline__ void rope_q_frags(uint32_t (&qa)[8][4], const __half* const (&qr)[2], const int (&pos)[2], float log2_theta) {
  const int t = threadIdx.x & 3;
  const float kFreqStep = log2_theta / 64.f;
  float2 lo[2][4][2], hi[2][4][2];
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {            // columns d = 16 kk + 8 hf + 2 t, d + 1 and their partners d + 64
        const int d = 16 * kk + 8 * hf + 2 * t;
        const float2 x = __half22float2(*reinterpret_cast<const __half2*>(qr[rr] + d));
        const float2 y = __half22float2(*reinterpret_cast<const __half2*>(qr[rr] + d + 64));
        float s0, c0, s1, c1;
        sincosf((float)pos[rr] * exp2f(-(float)d * kFreqStep), &s0, &c0);
        sincosf((float)pos[rr] * exp2f(-(float)(d + 1) * kFreqStep), &s1, &c1);
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

// row sum of l over the quad of threads that share a row
__device__ __forceinline__ float quad_sum(float x) {
  x += __shfl_xor_sync(0xffffffffu, x, 1);
  return x + __shfl_xor_sync(0xffffffffu, x, 2);
}

// row rr of this thread's o fragments, normalised by its quad-summed l and rounded to FP16, into the row's 128 halves at dst
__device__ __forceinline__ void attn_store_row(__half* dst, const float (&o)[16][4], int rr, float l) {
  const int t = threadIdx.x & 3;
  const float inv = 1.f / l;
#pragma unroll
  for (int i = 0; i < 16; ++i)
    *reinterpret_cast<uint32_t*>(dst + 8 * i + 2 * t) = pack_h2(o[i][2 * rr] * inv, o[i][2 * rr + 1] * inv);
}

// row rr of this thread's o fragments as an un-normalised partial (m, l, acc[128]) in the DEC_PART layout at dst
__device__ __forceinline__ void attn_store_part(float* dst, const float (&o)[16][4], int rr, float m, float l) {
  const int t = threadIdx.x & 3;
  if (t == 0) *reinterpret_cast<float2*>(dst) = make_float2(m, l);
#pragma unroll
  for (int i = 0; i < 16; ++i)
    *reinterpret_cast<float2*>(dst + 2 + 8 * i + 2 * t) = make_float2(o[i][2 * rr], o[i][2 * rr + 1]);
}

// q f16 [T, H*128] (pre-RoPE, the q projection's output); kf, vf f16 [T, Hkv*128] from kv_dequant_rope_kernel (H % Hkv == 0);
// indptr i32 [B+1]: prompt b owns tokens [indptr[b], indptr[b+1]); out f16 [T, H*128]
// kCtx = false: grid (q tiles, B, H); every prompt is a whole sequence (positions 0 .. L - 1).
// kCtx = true: `cache` is one KvArgs (page table, layer); grid (q tiles * G, Hkv, B), G = H / Hkv -- the q tiles and the G query
// heads of one KV head are adjacent in launch order, so the CTAs that stream the same context pages run together and share them
// through L2.  Prompt b is the tail of the cached sequence b: ctx_b = seq_len_b - L_b, derived as append_kv_kernel derives its
// write position.  The context sits at key positions -ctx_b .. -1, in 64-token tiles that end at -1, before the prompt's own
// causal tiles: every context key precedes every query, so these tiles need no causal mask, only the first (partial) one a length
// mask, and the online-softmax state carries on into the prompt's tiles unchanged.  q is rotated at ctx_b + r.
// Every term of the context path sits behind `if constexpr` or a condition on the constant kCtx, and the cache is a trailing
// parameter pack (empty for <false>): <false> carries none of it.
// <true> asks for two CTAs per SM: at the three CTAs ptxas otherwise aims for (168 registers) its context producer spills.
template <bool kCtx, typename... Cache>
__global__ void __launch_bounds__(PF_THREADS, kCtx ? 2 : 0)
prefill_attn_kernel(const __half* __restrict__ q, const __half* __restrict__ kf, const __half* __restrict__ vf,
                    const int32_t* __restrict__ indptr, const float2* __restrict__ rope, __half* __restrict__ out, int H,
                    int Hkv, Cache... cache) {
  static_assert(sizeof...(Cache) == (kCtx ? 1 : 0), "prefill_attn_kernel<true> takes the cache (one KvArgs), <false> nothing");
  __shared__ __align__(16) __half Ks[PF_BK * PF_KPITCH];
  __shared__ __align__(16) __half Vt[128 * PF_VPITCH];
  int b, h, qt;
  if constexpr (kCtx) {
    const int G = H / Hkv;
    b = blockIdx.z; h = blockIdx.y * G + (int)blockIdx.x % G; qt = (int)blockIdx.x / G;
  } else {
    b = blockIdx.y; h = blockIdx.z; qt = blockIdx.x;
  }
  const int t0 = indptr[b], L = indptr[b + 1] - t0;
  const int q0 = qt * PF_BQ;
  if (q0 >= L) return;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const size_t row_pitch = (size_t)H * 128;
  const size_t kv_pitch = (size_t)Hkv * 128;          // grouped-query attention: query head h reads KV head h / (H / Hkv)
  const int hk = h / (H / Hkv);
  const int ctx = prefill_ctx_len(cache..., b, L);

  if constexpr (kCtx) rope += (size_t)ctx * 64;       // row p of the table = position ctx + p
  // ---- Q fragments of this warp's 16 rows, rotated (FP32 math, rounded to FP16 like `rotary_pos_emb(...).to(q.dtype)`)
  uint32_t qa[8][4];
  {
    const int r0 = q0 + warp * 16 + g, r1 = r0 + 8;
    const __half* q_r0 = q + (size_t)(t0 + min(r0, L - 1)) * row_pitch + h * 128;
    const __half* q_r1 = q + (size_t)(t0 + min(r1, L - 1)) * row_pitch + h * 128;
    const float2* rp0 = rope + (size_t)min(r0, L - 1) * 64;
    const float2* rp1 = rope + (size_t)min(r1, L - 1) * 64;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {            // columns d = 16 kk + 8 hf + 2 t, d + 1 and their partners d + 64
        const int d = 16 * kk + 8 * hf + 2 * t;
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const __half* qr = rr ? q_r1 : q_r0;
          const float2* rp = rr ? rp1 : rp0;
          const float2 lo = __half22float2(*reinterpret_cast<const __half2*>(qr + d));
          const float2 hi = __half22float2(*reinterpret_cast<const __half2*>(qr + d + 64));
          const float2 cs0 = rp[d], cs1 = rp[d + 1];
          qa[kk][2 * hf + rr] = pack_h2(lo.x * cs0.x - hi.x * cs0.y, lo.y * cs1.x - hi.y * cs1.y);
          qa[kk + 4][2 * hf + rr] = pack_h2(hi.x * cs0.x + lo.x * cs0.y, hi.y * cs1.x + lo.y * cs1.y);
        }
      }
    }
  }

  float o[16][4];
#pragma unroll
  for (int i = 0; i < 16; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  const int qrow0 = q0 + warp * 16 + g, qrow1 = qrow0 + 8;

  for (int kt = kCtx ? -((ctx + PF_BK - 1) / PF_BK) : 0; kt <= qt; ++kt) {
    const int k0 = kt * PF_BK;
    __syncthreads();                                  // the previous tile has been consumed
    if (kCtx && kt < 0) {
      // ---- producer, context: 64 cached tokens (key positions k0 .. k0 + 63) dequantised and rotated from the pages
      prefill_ctx_tile(cache..., b, L, hk, k0, rope, Ks, Vt, tid);
    } else {
    // ---- producer: 64 tokens of K (row-major) and V (transposed) into shared memory, 16-byte chunks
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int c = tid + it * PF_THREADS, tok = c >> 4, ch = c & 15, pos = k0 + tok;
      uint4 kv = make_uint4(0, 0, 0, 0), vv = make_uint4(0, 0, 0, 0);        // beyond the prompt: zeros (masked below anyway)
      if (pos < L) {
        const size_t off = (size_t)(t0 + pos) * kv_pitch + hk * 128 + ch * 8;
        kv = *reinterpret_cast<const uint4*>(kf + off);
        vv = *reinterpret_cast<const uint4*>(vf + off);
      }
      *reinterpret_cast<uint4*>(&Ks[tok * PF_KPITCH + ch * 8]) = kv;
      const __half* vh = reinterpret_cast<const __half*>(&vv);
#pragma unroll
      for (int e = 0; e < 8; ++e) Vt[(ch * 8 + e) * PF_VPITCH + tok] = vh[e];
    }
    }
    __syncthreads();
    // causal and prompt-length mask; <true>: the first context tile's slots before the context hold no key.  Rows past the
    // prompt end have every key masked in their first tiles.
    attn_tile_step(qa, Ks, Vt, k0, [&](int rr, int kpos) { return (!kCtx || kpos >= -ctx) && kpos <= (rr ? qrow1 : qrow0) && kpos < L; },
                   o, m0, m1, l0, l1);
  }

  // ---- normalise and store
  l0 = quad_sum(l0); l1 = quad_sum(l1);
  if (qrow0 < L) attn_store_row(out + (size_t)(t0 + qrow0) * row_pitch + h * 128, o, 0, l0);
  if (qrow1 < L) attn_store_row(out + (size_t)(t0 + qrow1) * row_pitch + h * 128, o, 1, l1);
}

}  // namespace atom
