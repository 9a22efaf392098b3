/*
 * CPU oracle of the grouped-query INT4 paged-KV decode attention -- TEST INFRASTRUCTURE ONLY (tests/gqa_oracle.py builds
 * and loads it; nothing in atom_b200/ does).
 *
 * It restates oracle/atom_oracle.c's atom_oracle_batch_decode_i4 with two more degrees of freedom: Hq = G * Hkv query heads
 * over a cache of Hkv heads (query head h reads KV head h / G), and the RoPE base `theta` as an argument.  The arithmetic
 * per (query head, token) is the same statement for statement, so on a cache whose heads are repeated G times, and with
 * theta = 1e4, the two oracles agree exactly (tests/test_gqa_cpu.py pins that).  The stored goldens pin the multi-head
 * oracle, which is why this one lives in a file of its own.
 *
 * data  : u8 [pages][L][2][Hkv][P][64]      param : f16 [pages][L][2][Hkv][P][2] = (scale, zero);  x = nibble * scale - zero
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef uint16_t h16;

static float h2f(h16 h) {
  uint32_t sign = (uint32_t)(h & 0x8000u) << 16, exp = (h >> 10) & 0x1f, man = h & 0x3ffu, bits;
  if (exp == 0) {
    if (man == 0) bits = sign;
    else {
      int e = -1;
      do { ++e; man <<= 1; } while (!(man & 0x400u));
      bits = sign | ((uint32_t)(127 - 15 - e) << 23) | ((man & 0x3ffu) << 13);
    }
  } else if (exp == 31) bits = sign | 0x7f800000u | (man << 13);
  else bits = sign | ((exp + 112) << 23) | (man << 13);
  float f;
  memcpy(&f, &bits, 4);
  return f;
}

/* round to nearest even, overflow to infinity */
static h16 f2h(float f) {
  uint32_t x;
  memcpy(&x, &f, 4);
  uint32_t sign = (x >> 16) & 0x8000u;
  x &= 0x7fffffffu;
  if (x >= 0x7f800000u) return (h16)(sign | 0x7c00u | (x > 0x7f800000u ? 0x200u : 0));
  if (x >= 0x477ff000u) return (h16)(sign | 0x7c00u);
  if (x < 0x33000001u) return (h16)sign;
  if (x < 0x38800000u) {
    int shift = 126 - (int)(x >> 23);                         /* 14 .. 24 */
    uint32_t man = (x & 0x7fffffu) | 0x800000u;
    uint32_t r = man >> shift, rem = man & ((1u << shift) - 1), half = 1u << (shift - 1);
    if (rem > half || (rem == half && (r & 1))) ++r;
    return (h16)(sign | r);
  }
  uint32_t r = ((x - 0x38000000u) >> 13), rem = x & 0x1fffu;
  if (rem > 0x1000u || (rem == 0x1000u && (r & 1))) ++r;
  return (h16)(sign | r);
}

static size_t kv_off(int page, int L, int layer, int kv, int H, int head, int P, int entry) {
  return ((((size_t)page * L + layer) * 2 + kv) * H + head) * P + entry;
}

void gqa_oracle_batch_decode_i4(h16 *o, const h16 *q, const uint8_t *data, const h16 *param, const int32_t *indptr,
                                const int32_t *indices, const int32_t *last_off, int L, int layer, int Hq, int Hkv, int P, int B,
                                float theta) {
  const int D = 128, G = Hq / Hkv;
  const float sm_scale = (1.f / sqrtf((float)D)) * 1.44269504088896340736f;
  float freq[128];
  for (int i = 0; i < D; ++i) freq[i] = powf(1.f / theta, (float)(2 * (i % (D / 2))) / (float)D);
  for (int b = 0; b < B; ++b) {
    const int npages = indptr[b + 1] - indptr[b];
    const int seq_len = (npages - 1) * P + last_off[b];
    float *s = (float *)malloc(sizeof(float) * (seq_len > 0 ? seq_len : 1));
    for (int h = 0; h < Hq; ++h) {
      const int hk = h / G;
      float qv[128], qr[128];
      for (int i = 0; i < D; ++i) qv[i] = h2f(q[((size_t)b * Hq + h) * D + i]);
      for (int i = 0; i < D; ++i) {
        float e = (float)(seq_len - 1) * freq[i];
        float perm = (i < D / 2) ? -qv[i + D / 2] : qv[i - D / 2];
        qr[i] = qv[i] * cosf(e) + perm * sinf(e);
      }
      float mx = -5e4f;
      for (int t = 0; t < seq_len; ++t) {
        int page = indices[indptr[b] + t / P], entry = t % P;
        size_t off = kv_off(page, L, layer, 0, Hkv, hk, P, entry);
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
        size_t off = kv_off(page, L, layer, 1, Hkv, hk, P, entry);
        const uint8_t *vp = data + off * 64;
        float sc = h2f(param[off * 2]), ze = h2f(param[off * 2 + 1]);
        double p = exp2((double)(s[t] - mx));
        den += p;
        for (int i = 0; i < D; ++i) acc[i] += p * (double)((float)((vp[i >> 1] >> ((i & 1) * 4)) & 0xf) * sc - ze);
      }
      for (int i = 0; i < D; ++i) o[((size_t)b * Hq + h) * D + i] = f2h((float)(acc[i] / den));
    }
    free(s);
  }
}
