/*
 * atom_oracle.c -- CPU restatement of the efeslab/Atom W4A4 hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under atom_b200/ may import, link or call
 * this file; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs use it, and only as the checker.
 *
 * Every function restates the arithmetic of one reference kernel, op for op
 * (FP32 fused multiply-add where the reference SASS has FFMA, one FP16 RN
 * multiply where it has HMUL2, C roundf() = half-away-from-zero where the
 * reference calls round()).  Citations are relative to /root/reference.
 *
 * Parity status: the reference has no golden vectors for the GEMM or the decode
 * kernel (SURVEY.md section 8c), so this oracle is pinned two other ways:
 *   (1) tests/golden/ *.npz were produced by running the reference's own CPU
 *       golden functions (test_Reorder.cu:41-112 etc.) and its Python
 *       model/quant.py in the build container (tests/golden/make_golden.py);
 *   (2) on the GPU box the reference's own CUDA kernels, compiled unmodified
 *       from /root/reference into oracle/_ref/libatom_ref.so, are run on the
 *       same inputs (tests/test_gpu_vs_reference.py).
 *
 * Build: see oracle/Makefile (plain gcc, no -march=native: the .so travels to
 * the GPU box, whose host CPU may differ).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef uint16_t h16;  /* IEEE binary16 bit pattern */

/* ---- binary16 <-> binary32, bit exact, portable (no F16C dependence) ---- */
static inline float h2f(h16 h) {
  uint32_t s = (uint32_t)(h & 0x8000u) << 16;
  uint32_t e = (h >> 10) & 0x1f, m = h & 0x3ff, u;
  if (e == 0) {
    if (m == 0) u = s;
    else { /* subnormal */
      int sh = 0;
      while (!(m & 0x400)) { m <<= 1; ++sh; }
      m &= 0x3ff;
      u = s | ((uint32_t)(127 - 15 - sh + 1) << 23) | (m << 13);
    }
  } else if (e == 31) u = s | 0x7f800000u | (m << 13);
  else u = s | ((e + 112) << 23) | (m << 13);
  float f; memcpy(&f, &u, 4); return f;
}

/* round-to-nearest-even, matches __float2half_rn */
static inline h16 f2h(float f) {
  uint32_t u; memcpy(&u, &f, 4);
  uint32_t s = (u >> 16) & 0x8000u;
  uint32_t a = u & 0x7fffffffu;
  if (a >= 0x7f800000u) return (h16)(s | 0x7c00u | ((a > 0x7f800000u) ? 0x200u | ((a >> 13) & 0x3ff) : 0));
  if (a >= 0x477ff000u) return (h16)(s | 0x7c00u);           /* >= 65520 -> inf */
  if (a < 0x33000001u) return (h16)s;                          /* < 2^-25 (or ==) -> 0 */
  int e = (int)(a >> 23) - 127;
  uint32_t m = (a & 0x7fffffu) | 0x800000u;
  if (e < -14) {  /* subnormal half */
    int sh = -14 - e + 13;          /* bits to drop */
    uint32_t r = m >> sh, rem = m & ((1u << sh) - 1), half = 1u << (sh - 1);
    if (rem > half || (rem == half && (r & 1))) ++r;
    return (h16)(s | r);
  }
  uint32_t r = ((uint32_t)(e + 15) << 10) | ((m >> 13) & 0x3ff);
  uint32_t rem = m & 0x1fff;
  if (rem > 0x1000 || (rem == 0x1000 && (r & 1))) ++r;  /* carry may bump exponent: correct */
  return (h16)(s | r);
}

/* one FP16 RN multiply (HMUL2 lane): product of two halves is exact in fp32 */
static inline h16 hmul(h16 a, h16 b) { return f2h(h2f(a) * h2f(b)); }

/* ---------------- layout contract (Reorder.cuh:39-50, ops/__init__.py:137) --------------- */
int atom_oracle_scale_index(int row) {
  return (row / 16) * 64 + (row % 8) * 8 + ((row / 8) % 2);
}
int atom_oracle_scale_size(int m) {
  return m / 16 * 64 + 64 - (1 - (m % 16) / 8) * (8 - (m % 8)) * 8;
}

static inline int clampi(int x, int lo, int hi) { return x < lo ? lo : (x > hi ? hi : x); }

/* (int)f with the semantics of PTX cvt.rzi.s32.f32, which the kernels' (int) casts compile to: truncation, saturation
 * to the int range, NaN -> 0.  A plain C cast of NaN or of an out-of-range value is undefined (x86 gives INT_MIN).
 * An all-zero group reaches this with 0 * (1/0) = NaN and must store code 0. */
static inline int cvt_s32(float f) {
  if (f != f) return 0;
  if (f >= 2147483648.f) return 2147483647;
  if (f < -2147483648.f) return (int)(-2147483647 - 1);
  return (int)f;
}

/*
 * Shared quantise tail (Reorder.cuh:107-189, RMSNorm.cuh:160-237, Activate.cuh:108-179).
 * x: hidden FP32 values of one row already in reordered order.
 * groups 0..G-1 -> INT4 (absmax/7), last group -> INT8 (absmax/127).
 */
static void quant_tail_row(const float *x, int hidden, int row, int scale_ldm,
                           int8_t *s8out, uint8_t *s4out, h16 *s8scale, h16 *s4scale) {
  const int ng = hidden / 128;
  const int sidx = atom_oracle_scale_index(row);
  for (int g = 0; g < ng; ++g) {
    const float *xg = x + g * 128;
    float maxv = 0.f;            /* reference starts at -65536 / -1; |x| >= 0 wins */
    for (int i = 0; i < 128; ++i) { float a = fabsf(xg[i]); if (a > maxv) maxv = a; }
    const int last = (g == ng - 1);
    maxv = maxv / (last ? 127.f : 7.f);
    const h16 hs = f2h(maxv);
    h16 *dst = last ? s8scale : (s4scale + (size_t)g * scale_ldm);
    for (int j = 0; j < 4; ++j) dst[sidx + 2 * j] = hs;
    const float r_scale = 1.f / maxv;
    const int lo = last ? -128 : -8, hi = last ? 127 : 7;
    if (last) {
      for (int i = 0; i < 128; ++i)
        s8out[(size_t)row * 128 + i] = (int8_t)clampi(cvt_s32(roundf(xg[i] * r_scale)), lo, hi);
    } else {
      uint8_t *o = s4out + (size_t)row * ((hidden - 128) / 2) + g * 64;
      for (int i = 0; i < 128; i += 2) {
        int q0 = clampi(cvt_s32(roundf(xg[i] * r_scale)), lo, hi);
        int q1 = clampi(cvt_s32(roundf(xg[i + 1] * r_scale)), lo, hi);
        o[i / 2] = (uint8_t)((q0 & 0xf) | ((q1 & 0xf) << 4));   /* PackInt4{low,high}, Reorder.cuh:16-19 */
      }
    }
  }
}

/* K3: reorder_fp16_i4 (kernels/include/Reorder/Reorder.cuh:64-190).
 * The reorder index is read as uint16_t, as the kernels read it: hidden may reach 65536, so an index >= 32768 is a
 * column of the row, not an offset before it. */
void atom_oracle_reorder_fp16_i4(const h16 *in, int seq_len, int hidden, const uint16_t *idx,
                                 int8_t *s8out, uint8_t *s4out, h16 *s8scale, h16 *s4scale) {
  const int ldm = atom_oracle_scale_size(seq_len);
  float *x = (float *)malloc(sizeof(float) * hidden);
  for (int r = 0; r < seq_len; ++r) {
    for (int i = 0; i < hidden; ++i) x[i] = h2f(in[(size_t)r * hidden + idx[i]]);
    quant_tail_row(x, hidden, r, ldm, s8out, s4out, s8scale, s4scale);
  }
  free(x);
}

/* K4: rmsnorm_fp16_i4 (kernels/include/RMSNorm/RMSNorm.cuh:66-238).
 * Sum of squares follows the reference's order: 128 "threads" each fold hidden/128
 * contiguous elements with fmaf, then tree 128->64->32 and shfl_down 16..1.
 * rstd uses 1/sqrtf (the GPU uses rsqrtf, max 2 ulp) => +-1 LSB tolerance in tests.
 * The reorder index is uint16_t, as in K3. */
void atom_oracle_rmsnorm_fp16_i4(const h16 *in, const h16 *w, float eps, int seq_len, int hidden,
                                 const uint16_t *idx, int8_t *s8out, uint8_t *s4out,
                                 h16 *s8scale, h16 *s4scale) {
  const int ldm = atom_oracle_scale_size(seq_len);
  const int ept = hidden / 128;
  float *x = (float *)malloc(sizeof(float) * hidden);
  for (int r = 0; r < seq_len; ++r) {
    const h16 *row = in + (size_t)r * hidden;
    float part[128];
    for (int t = 0; t < 128; ++t) {
      float s = 0.f;
      for (int i = 0; i < ept; ++i) { float v = h2f(row[t * ept + i]); s = fmaf(v, v, s); }
      part[t] = s;
    }
    for (int t = 0; t < 64; ++t) part[t] = part[t] + part[t + 64];
    for (int t = 0; t < 32; ++t) part[t] = part[t] + part[t + 32];
    for (int s = 16; s > 0; s >>= 1)
      for (int t = 0; t < s; ++t) part[t] = part[t] + part[t + s];
    const float rstd = 1.0f / sqrtf(part[0] / (float)hidden + eps);
    for (int i = 0; i < hidden; ++i) {
      int j = idx[i];
      float v = h2f(row[j]) * h2f(w[j]);   /* two FP32 roundings, RMSNorm.cuh:150 */
      v = v * rstd;
      x[i] = h2f(f2h(v));                   /* __float2half then re-widened in the tail */
    }
    quant_tail_row(x, hidden, r, ldm, s8out, s4out, s8scale, s4scale);
  }
  free(x);
}

/* K5: activate_fp16_i4 (kernels/include/Activate/Activate.cuh:67-180): silu(a)*b in FP32 */
void atom_oracle_activate_fp16_i4(const h16 *a, const h16 *b, int seq_len, int hidden,
                                  int8_t *s8out, uint8_t *s4out, h16 *s8scale, h16 *s4scale) {
  const int ldm = atom_oracle_scale_size(seq_len);
  float *x = (float *)malloc(sizeof(float) * hidden);
  for (int r = 0; r < seq_len; ++r) {
    for (int i = 0; i < hidden; ++i) {
      float av = h2f(a[(size_t)r * hidden + i]), bv = h2f(b[(size_t)r * hidden + i]);
      float s = av / (1.0f + expf(-av));
      x[i] = s * bv;
    }
    quant_tail_row(x, hidden, r, ldm, s8out, s4out, s8scale, s4scale);
  }
  free(x);
}

static inline int nib(const uint8_t *p, int k) {  /* signed 4-bit element k of a packed row */
  int v = (p[k >> 1] >> ((k & 1) * 4)) & 0xf;
  return v >= 8 ? v - 16 : v;
}

/*
 * K1 accumulate: FP32 result of the W4A4 GEMM before the output cast.
 * Dense_layer_gemm_i4_o16.cuh:404-434 (dequant), :520-588 (group order 0..G-1),
 * :590-691 (keeper last).  K = total K including the 128 keeper channels.
 * faithful != 0 reproduces the reference's column pairing of B scales
 * (n' = n&~1 for m%16<8, n|1 otherwise); faithful == 0 uses sB[g][n].
 * rows[] selects which A rows to compute (NULL = all M) so that full-size
 * problems can be spot-checked in seconds.
 *
 * ksplit > 1 restates the K split of gemm_i4_sm90.cuh (a cluster of ksplit
 * CTAs along K).  Of the G+1 groups (index G = the keeper), rank r owns
 * [min(r*per, G+1), min(r*per + per, G+1)) with per = ceil((G+1)/ksplit), so
 * a rank may hold no group, or only the keeper.  Each rank runs its own fmaf
 * chain from +0.0f over its groups in order (keeper last on the rank that
 * owns it); the partials are then added in rank order in FP32,
 * ((p0 + p1) + p2) + ..., an empty rank contributing +0.0f; then RN to FP16.
 * The kernel carries a factor 256 on every term (INT4 operands widened to
 * value*16, the keeper's sum shifted by 8) and multiplies by 2^-8 before the
 * cast: a power of two on values that stay normal in FP32, hence exact, so it
 * is not restated.  ksplit = 1 is the single chain above.
 */
static void gemm_acc(const uint8_t *A, const uint8_t *B, const h16 *As, const h16 *Bs,
                     const int8_t *Ak, const int8_t *Bk, const h16 *Aks, const h16 *Bks,
                     int M, int N, int K, int faithful, int ksplit, const int32_t *rows, int nrows,
                     float *acc /* [nrows][N] */) {
  const int G = K / 128 - 1;
  const int Kp = (K - 128) / 2;
  const int ldm = atom_oracle_scale_size(M);
  const int per = (G + 1 + ksplit - 1) / ksplit;
  int8_t *a8 = (int8_t *)malloc((size_t)(K - 128));
  int8_t *b8 = (int8_t *)malloc((size_t)(K - 128));
  for (int ri = 0; ri < nrows; ++ri) {
    const int m = rows ? rows[ri] : ri;
    for (int k = 0; k < K - 128; ++k) a8[k] = (int8_t)nib(A + (size_t)m * Kp, k);
    const int sidx = atom_oracle_scale_index(m);
    const int upper = (m % 16) >= 8;
    for (int n = 0; n < N; ++n) {
      for (int k = 0; k < K - 128; ++k) b8[k] = (int8_t)nib(B + (size_t)n * Kp, k);
      const int np = faithful ? (upper ? (n | 1) : (n & ~1)) : n;
      float sum = 0.f;
      for (int r = 0; r < ksplit; ++r) {
        const int gb = r * per < G + 1 ? r * per : G + 1;
        const int ge = gb + per < G + 1 ? gb + per : G + 1;
        float a = 0.f;
        for (int g = gb; g < ge && g < G; ++g) {
          int32_t c = 0;
          const int8_t *pa = a8 + g * 128, *pb = b8 + g * 128;
          for (int k = 0; k < 128; ++k) c += (int32_t)pa[k] * (int32_t)pb[k];
          h16 rs = hmul(As[(size_t)g * ldm + sidx], Bs[(size_t)g * N + np]);
          a = fmaf((float)c, h2f(rs), a);
        }
        if (ge == G + 1 && ge > gb) {   /* this rank owns the keeper */
          int32_t c = 0;
          const int8_t *pa = Ak + (size_t)m * 128, *pb = Bk + (size_t)n * 128;
          for (int k = 0; k < 128; ++k) c += (int32_t)pa[k] * (int32_t)pb[k];
          h16 rs = hmul(Aks[sidx], Bks[np]);
          a = fmaf((float)c, h2f(rs), a);
        }
        sum = r == 0 ? a : sum + a;
      }
      acc[(size_t)ri * N + n] = sum;
    }
  }
  free(a8); free(b8);
}

/* K1: DenseLayerGEMM_i4_o16 -> FP16 (storeAccumulator, o16.cuh:227-246: __float2half RN).
 * ksplit: the K split of the kernel (1 = the reference's single chain), see gemm_acc. */
void atom_oracle_gemm_i4_o16(const uint8_t *A, const uint8_t *B, const h16 *As, const h16 *Bs,
                             const int8_t *Ak, const int8_t *Bk, const h16 *Aks, const h16 *Bks,
                             h16 *D, int M, int N, int K, int faithful, int ksplit,
                             const int32_t *rows, int nrows) {
  if (!rows) nrows = M;
  float *acc = (float *)malloc(sizeof(float) * (size_t)nrows * N);
  gemm_acc(A, B, As, Bs, Ak, Bk, Aks, Bks, M, N, K, faithful, ksplit, rows, nrows, acc);
  for (size_t i = 0; i < (size_t)nrows * N; ++i) D[i] = f2h(acc[i]);
  free(acc);
}

/* K2: the o4 epilogue: per (row, 128 output columns) asymmetric INT4, x = nibble * scale - zero.
 * signed_minmax != 0 (the default of oracle.py): mn, mx = the min and max of v in the order of f_key (-0 below +0, the
 * kernel's tie rule), scale = (mx - mn) / 15, zero = -mn, q = clamp(roundf((v + zero) * (1/scale)), 0, 15); a constant head
 * has scale +0 and (v + zero) * inf = NaN, which converts to code 0.
 * signed_minmax == 0 restates the reference kernel (e2e/.../GEMM/DenseLayerGEMM_i4_o4.cu:705-787) instead: min/max over |v|
 * and q = (int)roundf(...) & 0xF, which wraps every v below min|v| to a wrong nibble.  Kept only to pin this oracle to the
 * reference's recorded outputs. */
static inline uint32_t f_key(float f) {          /* orders IEEE floats like unsigned integers: -0 < +0 */
  uint32_t b;
  memcpy(&b, &f, 4);
  return b ^ ((b >> 31) ? 0xffffffffu : 0x80000000u);
}

void atom_oracle_gemm_i4_o4(const uint8_t *A, const uint8_t *B, const h16 *As, const h16 *Bs,
                            const int8_t *Ak, const int8_t *Bk, const h16 *Aks, const h16 *Bks,
                            uint8_t *D /*[nrows][N/2]*/, h16 *Dscale /*[nrows][N/128][2]*/,
                            int M, int N, int K, int faithful, int signed_minmax,
                            const int32_t *rows, int nrows) {
  if (!rows) nrows = M;
  float *acc = (float *)malloc(sizeof(float) * (size_t)nrows * N);
  gemm_acc(A, B, As, Bs, Ak, Bk, Aks, Bks, M, N, K, faithful, 1, rows, nrows, acc);
  for (int r = 0; r < nrows; ++r)
    for (int h = 0; h < N / 128; ++h) {
      const float *v = acc + (size_t)r * N + h * 128;
      float mx = -INFINITY, mn = INFINITY;   /* 0xFC00 / 0x7C00 as float, o4.cu:727-728 */
      for (int i = 0; i < 128; ++i) {
        if (!signed_minmax) {
          const float t = fabsf(v[i]);
          if (t > mx) mx = t;
          if (t < mn) mn = t;
        } else {
          if (f_key(v[i]) > f_key(mx)) mx = v[i];
          if (f_key(v[i]) < f_key(mn)) mn = v[i];
        }
      }
      const float scale = (mx - mn) / 15.f, zero = -mn, r_scale = 1.f / scale;
      Dscale[((size_t)r * (N / 128) + h) * 2 + 0] = f2h(scale);
      Dscale[((size_t)r * (N / 128) + h) * 2 + 1] = f2h(zero);
      uint8_t *o = D + (size_t)r * (N / 2) + h * 64;
      for (int i = 0; i < 128; i += 2) {
        int q0 = cvt_s32(roundf((v[i] + zero) * r_scale)), q1 = cvt_s32(roundf((v[i + 1] + zero) * r_scale));
        if (!signed_minmax) {
          q0 &= 0xf; q1 &= 0xf;
        } else {
          q0 = clampi(q0, 0, 15); q1 = clampi(q1, 0, 15);
        }
        o[i / 2] = (uint8_t)(q0 | (q1 << 4));
      }
    }
  free(acc);
}

/* ------------------------- paged INT4 KV cache (page.cuh:18-216) ------------------------- */
/* data  : u8 [pages][L][2][H][P][64]      param : h16 [pages][L][2][H][P][2] = (scale, zero) */
static inline size_t kv_off(int page, int L, int layer, int kv, int H, int head, int P, int entry) {
  return ((((size_t)page * L + layer) * 2 + kv) * H + head) * P + entry;
}

/* K7: AppendPagedKVCacheDecodeKernel (page.cuh:119-163) */
void atom_oracle_append_kv_i4(uint8_t *data, h16 *param, const int32_t *indptr, const int32_t *indices,
                              const int32_t *last_off, const uint8_t *k, const uint8_t *v,
                              const h16 *kp, const h16 *vp, int L, int layer, int H, int P, int B) {
  for (int b = 0; b < B; ++b) {
    int seq_len = (indptr[b + 1] - indptr[b] - 1) * P + last_off[b];
    int page = indices[indptr[b] + (seq_len - 1) / P], entry = (seq_len - 1) % P;
    for (int h = 0; h < H; ++h) {
      size_t ok = kv_off(page, L, layer, 0, H, h, P, entry), ov = kv_off(page, L, layer, 1, H, h, P, entry);
      memcpy(data + ok * 64, k + ((size_t)b * H + h) * 64, 64);
      memcpy(data + ov * 64, v + ((size_t)b * H + h) * 64, 64);
      memcpy(param + ok * 2, kp + ((size_t)b * H + h) * 2, 4);
      memcpy(param + ov * 2, vp + ((size_t)b * H + h) * 2, 4);
    }
  }
}

/* K8: AppendPagedKVCachePrefillKernel (page.cuh:165-216) */
void atom_oracle_init_kv_i4(uint8_t *data, h16 *param, const int32_t *indptr, const int32_t *indices,
                            const int32_t *last_off, const uint8_t *k, const uint8_t *v,
                            const h16 *kp, const h16 *vp, const int32_t *append_indptr,
                            int L, int layer, int H, int P, int B) {
  for (int b = 0; b < B; ++b) {
    int seq_len = (indptr[b + 1] - indptr[b] - 1) * P + last_off[b];
    int app = append_indptr[b + 1] - append_indptr[b], start = seq_len - app;
    for (int j = 0; j < app; ++j) {
      int pos = start + j, page = indices[indptr[b] + pos / P], entry = pos % P;
      size_t tok = (size_t)append_indptr[b] + j;
      for (int h = 0; h < H; ++h) {
        size_t ok = kv_off(page, L, layer, 0, H, h, P, entry), ov = kv_off(page, L, layer, 1, H, h, P, entry);
        memcpy(data + ok * 64, k + (tok * H + h) * 64, 64);
        memcpy(data + ov * 64, v + (tok * H + h) * 64, 64);
        memcpy(param + ok * 2, kp + (tok * H + h) * 2, 4);
        memcpy(param + ov * 2, vp + (tok * H + h) * 2, 4);
      }
    }
  }
}

/*
 * K6: BatchDecodeWithPagedKVCacheKernel (decode.cuh:480-689), head_dim 128, kLlama RoPE.
 * Spec follows decode.cuh:39-71 (RoPE), :92-124 (qk), state.cuh:68-94 (online softmax) and
 * the orphan CPU golden kernels/src/flashinfer/cpu_reference.h:171-234 (dequant
 * nibble*scale - zero).  Exact libm (powf/sinf/cosf/exp2f) replaces the GPU's
 * approximate intrinsics; softmax is evaluated in one pass in double for the
 * normaliser, so tests use rtol/atol 1e-3 (FP16 output).
 */
void atom_oracle_batch_decode_i4(h16 *o, const h16 *q, const uint8_t *data, const h16 *param,
                                 const int32_t *indptr, const int32_t *indices, const int32_t *last_off,
                                 int L, int layer, int H, int P, int B) {
  const int D = 128;
  const float sm_scale = (1.f / sqrtf((float)D)) * 1.44269504088896340736f;
  float freq[128];
  for (int i = 0; i < D; ++i) freq[i] = powf(1e-4f, (float)(2 * (i % (D / 2))) / (float)D);
  for (int b = 0; b < B; ++b) {
    const int npages = indptr[b + 1] - indptr[b];
    const int seq_len = (npages - 1) * P + last_off[b];
    float *s = (float *)malloc(sizeof(float) * (seq_len > 0 ? seq_len : 1));
    for (int h = 0; h < H; ++h) {
      float qv[128], qr[128];
      for (int i = 0; i < D; ++i) qv[i] = h2f(q[((size_t)b * H + h) * D + i]);
      for (int i = 0; i < D; ++i) {
        float e = (float)(seq_len - 1) * freq[i];
        float perm = (i < D / 2) ? -qv[i + D / 2] : qv[i - D / 2];
        qr[i] = qv[i] * cosf(e) + perm * sinf(e);
      }
      float mx = -5e4f;
      for (int t = 0; t < seq_len; ++t) {
        int page = indices[indptr[b] + t / P], entry = t % P;
        size_t off = kv_off(page, L, layer, 0, H, h, P, entry);
        const uint8_t *kp = data + off * 64;
        float sc = h2f(param[off * 2]), ze = h2f(param[off * 2 + 1]);
        float kv[128];
        for (int i = 0; i < D; ++i) kv[i] = (float)((kp[i >> 1] >> ((i & 1) * 4)) & 0xf) * sc - ze;
        float x = 0.f;
        for (int i = 0; i < D; ++i) {
          float e = (float)t * freq[i];
          float perm = (i < D / 2) ? -kv[i + D / 2] : kv[i - D / 2];
          float kr = kv[i] * cosf(e) + perm * sinf(e);
          x += qr[i] * kr * sm_scale;
        }
        s[t] = x;
        if (x > mx) mx = x;
      }
      double den = 0.0, acc[128];
      for (int i = 0; i < D; ++i) acc[i] = 0.0;
      for (int t = 0; t < seq_len; ++t) {
        int page = indices[indptr[b] + t / P], entry = t % P;
        size_t off = kv_off(page, L, layer, 1, H, h, P, entry);
        const uint8_t *vp = data + off * 64;
        float sc = h2f(param[off * 2]), ze = h2f(param[off * 2 + 1]);
        double p = exp2((double)(s[t] - mx));
        den += p;
        for (int i = 0; i < D; ++i)
          acc[i] += p * (double)((float)((vp[i >> 1] >> ((i & 1) * 4)) & 0xf) * sc - ze);
      }
      for (int i = 0; i < D; ++i)
        o[((size_t)b * H + h) * D + i] = f2h((float)(acc[i] / den));
    }
    free(s);
  }
}

/* conversions exposed for the Python side of the tests */
void atom_oracle_h2f(const h16 *in, float *out, size_t n) { for (size_t i = 0; i < n; ++i) out[i] = h2f(in[i]); }
void atom_oracle_f2h(const float *in, h16 *out, size_t n) { for (size_t i = 0; i < n; ++i) out[i] = f2h(in[i]); }
