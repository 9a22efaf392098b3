// prefill_kernels.cuh -- causal prefill attention over the JUST-QUANTISED INT4 K/V of the prompt tokens.
//
// Replaces the placeholder in the reference's LlamaAttention.forward (punica/models/llama.py:171-190: "HACK" --
// scaled_dot_product_attention on torch.randn K/V) and the eager version round 1 shipped (per-prompt Python loop,
// torch dequantisation, rotary_pos_emb, cuDNN SDPA).  One launch for all prompts and heads:
//   * K and V are the o4 outputs of the k/v projections (packed nibbles + (scale, zero) per token-head, exactly what
//     init_kv_i4 scatters into the page pool, page.cuh:165-216): x = nibble * scale - zero, rounded to FP16 as the
//     decode path sees it;
//   * RoPE (theta = 1e4, pairs (i, i + 64), llama.py:18-32) on q and k from a (cos, sin) table of the positions;
//   * flash-attention recurrence (online softmax in FP32, base 2), FP16 tensor-core MMAs with FP32 accumulation.
// Two launches: kv_dequant_rope_kernel turns the packed K/V into FP16 once (K rotated), because every K/V tile is reused by
// all later query tiles of its prompt; prefill_attn_kernel is the attention proper.
// Tiling: CTA = 64 query rows of one (prompt, head), 4 warps x 16 rows; K/V in 64-token tiles through shared memory
// (K row-major [token][dim], V transposed [dim][token] so both B fragments are contiguous 32-bit loads, padded
// pitches => conflict-free).  The MMA is mma.sync.m16n8k16 (the warp-level tensor path); a wgmma variant is the
// next step for this kernel.
#pragma once
#include "ptx_sm90.cuh"

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

// q f16 [T, H*128] (pre-RoPE, the q projection's output); kf, vf f16 [T, Hkv*128] from kv_dequant_rope_kernel (H % Hkv == 0);
// indptr i32 [B+1]: prompt b owns tokens [indptr[b], indptr[b+1]); out f16 [T, H*128]
__global__ void __launch_bounds__(PF_THREADS)
prefill_attn_kernel(const __half* __restrict__ q, const __half* __restrict__ kf, const __half* __restrict__ vf,
                    const int32_t* __restrict__ indptr, const float2* __restrict__ rope, __half* __restrict__ out, int H,
                    int Hkv, float scale_log2) {
  __shared__ __align__(16) __half Ks[PF_BK * PF_KPITCH];
  __shared__ __align__(16) __half Vt[128 * PF_VPITCH];
  const int b = blockIdx.y, h = blockIdx.z, qt = blockIdx.x;
  const int t0 = indptr[b], L = indptr[b + 1] - t0;
  const int q0 = qt * PF_BQ;
  if (q0 >= L) return;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const size_t row_pitch = (size_t)H * 128;
  const size_t kv_pitch = (size_t)Hkv * 128;          // grouped-query attention: query head h reads KV head h / (H / Hkv)
  const int hk = h / (H / Hkv);

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

  for (int kt = 0; kt <= qt; ++kt) {
    const int k0 = kt * PF_BK;
    __syncthreads();                                  // the previous tile has been consumed
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
    __syncthreads();

    // ---- S = Q K^T (16 x 64 per warp), FP32
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
    // ---- scale, causal / length mask, online softmax (rows qrow0 and qrow1 of this thread)
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int kpos = k0 + 8 * j + 2 * t + u;
        const bool ok0 = kpos <= qrow0 && kpos < L, ok1 = kpos <= qrow1 && kpos < L;
        s[j][u] = ok0 ? s[j][u] * scale_log2 : -INFINITY;
        s[j][2 + u] = ok1 ? s[j][2 + u] * scale_log2 : -INFINITY;
        mx0 = fmaxf(mx0, s[j][u]); mx1 = fmaxf(mx1, s[j][2 + u]);
      }
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
    // rows past the prompt end have every key masked in their first tiles: keep exp2(-inf - -inf) out of the recurrence
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
    // ---- O += P V
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

  // ---- normalise and store
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.f / l0, i1 = 1.f / l1;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    if (qrow0 < L) *reinterpret_cast<uint32_t*>(out + (size_t)(t0 + qrow0) * row_pitch + h * 128 + 8 * i + 2 * t) = pack_h2(o[i][0] * i0, o[i][1] * i0);
    if (qrow1 < L) *reinterpret_cast<uint32_t*>(out + (size_t)(t0 + qrow1) * row_pitch + h * 128 + 8 * i + 2 * t) = pack_h2(o[i][2] * i1, o[i][3] * i1);
  }
}

}  // namespace atom
