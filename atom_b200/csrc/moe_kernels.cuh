// moe_kernels.cuh -- the sparse MoE block of Mixtral around the grouped expert GEMM (gemm_i4_sm90.cuh, EPI_GROUPED).
//
// One block is seven launches, all with sizes known on the host, so the whole block is graph-capturable although the
// routing is data dependent:
//   add_rmsnorm_fp16_i4 (quant_kernels.cuh)  residual sum + the ONE quantised activation tuple all experts read
//   moe_route_kernel                         the FP router on the FP16 normalised row, softmax, top-k, renormalised weights
//   moe_plan_kernel                          rows per expert, segments padded to the token tile, destination rows, tile table
//   moe_gather_kernel                        permute the rows of the activation tuple into the experts' segments
//   gemm_i4_kernel<BN, 1, EPI_GATEUP | EPI_GROUPED>   gate/up + SiLU * up + quantise, per tile of one expert
//   gemm_i4_kernel<BN, 1, EPI_O16 | EPI_GROUPED>      down projection
//   moe_combine_kernel                       out[t] = sum over t's experts, ascending, of fp16(y * w) (FP16 adds from +0)
// Every expert shares expert 0's channel orders (modelutils.reorder_model_mixtral), so nothing is re-quantised per expert.
// Segments start at multiples of the token tile (>= 16): a row's position mod 16 is its position in a per-expert GEMM call,
// which the GEMM's pair-shared weight scales depend on (DESIGN section 4).  Pad rows hold whatever the workspace held; they
// feed only their own accumulator columns and are never stored.
#pragma once
#include "gemm_i4_sm90.cuh"

namespace atom {

constexpr int MOE_MAX_EXPERTS = 64, MOE_MAX_TOPK = 8;
constexpr int ROUTE_THREADS = 512, PLAN_THREADS = 1024, GATHER_THREADS = 128, COMBINE_THREADS = 256;

// ---------------------------------------------------------------- route: one CTA per token
// The normalised row is formed exactly as rmsnorm_quant_kernel forms the values it quantises (same sum-of-squares
// association, same rsqrtf, half(float(x) * float(w) * rstd)), in the reordered channel order the router weight has.
// logit[e] = sum_j y_j * Wr[e, j] in FP32: warp e % 16, lane l folds chunks l, l+32, ... of 8 channels with fmaf (the FP16
// products are exact in FP32), then a 5-level butterfly -- hidden/32 + 5 rounded additions deep.  Softmax in FP32, top-k on
// the logits (an exact tie goes to the lower expert index), weights fp16(p_i / sum of the selected p, in selection order).
__global__ void __launch_bounds__(ROUTE_THREADS)
moe_route_kernel(const __half* __restrict__ x, const __half* __restrict__ w, const int16_t* __restrict__ idx, float eps,
                 const __half* __restrict__ wr, int hidden, int E, int k, int32_t* __restrict__ topk_ids,
                 __half* __restrict__ topk_w, float* __restrict__ logits_out, __half* __restrict__ normed_out, int pdl) {
  extern __shared__ __align__(16) uint8_t smem_r[];
  if (pdl) { griddep_launch_dependents(); griddep_wait(); }
  __half* xs = reinterpret_cast<__half*>(smem_r);
  __half* ws = xs + hidden;
  __half* ys = ws + hidden;
  float* red = reinterpret_cast<float*>(ys + hidden);      // [128] reduction scratch
  float* lg = red + 128;                                    // [E] logits
  const int row = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint4* xr = reinterpret_cast<const uint4*>(x + (size_t)row * hidden);
  for (int i = tid; i < hidden / 8; i += ROUTE_THREADS) {
    reinterpret_cast<uint4*>(xs)[i] = ld_cg_v4(xr + i);
    reinterpret_cast<uint4*>(ws)[i] = ld_cg_v4(reinterpret_cast<const uint4*>(w) + i);
  }
  __syncthreads();
  // sum of squares: thread t < 128 folds hidden/128 contiguous elements, then 128 -> 64 -> 32 -> shfl_down 16..1
  float sumv = 0.f;
  if (tid < 128) {
    const int ept = hidden / 128;
    for (int i = 0; i < ept; ++i) {
      const float f = __half2float(xs[tid * ept + i]);
      sumv = fmaf(f, f, sumv);
    }
    red[tid] = sumv;
  }
  __syncthreads();
  if (tid < 64) red[tid] = sumv = sumv + red[tid + 64];
  __syncthreads();
  if (tid < 32) {
    sumv = sumv + red[tid + 32];
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) sumv += __shfl_down_sync(0xffffffffu, sumv, s);
    if (tid == 0) red[0] = rsqrtf(sumv / (float)hidden + eps);
  }
  __syncthreads();
  const float rstd = red[0];
  for (int j = tid; j < hidden; j += ROUTE_THREADS) {
    const int id = (uint16_t)idx[j];
    ys[j] = __float2half_rn(__half2float(xs[id]) * __half2float(ws[id]) * rstd);
  }
  __syncthreads();
  if (normed_out != nullptr)
    for (int i = tid; i < hidden / 8; i += ROUTE_THREADS)
      reinterpret_cast<uint4*>(normed_out + (size_t)row * hidden)[i] = reinterpret_cast<const uint4*>(ys)[i];
  for (int e = warp; e < E; e += ROUTE_THREADS / 32) {
    const uint4* we = reinterpret_cast<const uint4*>(wr + (size_t)e * hidden);
    float acc = 0.f;
    for (int c = lane; c < hidden / 8; c += 32) {
      const uint4 a = reinterpret_cast<const uint4*>(ys)[c], b = ld_cg_v4(we + c);
      const __half2* ha = reinterpret_cast<const __half2*>(&a);
      const __half2* hb = reinterpret_cast<const __half2*>(&b);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 fa = __half22float2(ha[j]), fb = __half22float2(hb[j]);
        acc = fmaf(fa.x, fb.x, acc);
        acc = fmaf(fa.y, fb.y, acc);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) lg[e] = acc;
  }
  __syncthreads();
  if (tid == 0) {
    float mx = -INFINITY;
    for (int e = 0; e < E; ++e) mx = fmaxf(mx, lg[e]);
    float den = 0.f;
    for (int e = 0; e < E; ++e) den += expf(lg[e] - mx);
    uint64_t taken = 0;
    float p[MOE_MAX_TOPK];
    int sel[MOE_MAX_TOPK];
    float psum = 0.f;
    for (int s = 0; s < k; ++s) {
      int best = -1;
      for (int e = 0; e < E; ++e)
        if (!((taken >> e) & 1) && (best < 0 || lg[e] > lg[best])) best = e;   // strict: the lower index keeps a tie
      taken |= 1ull << best;
      sel[s] = best;
      p[s] = expf(lg[best] - mx) / den;
      psum += p[s];
    }
    for (int s = 0; s < k; ++s) {
      topk_ids[(size_t)row * k + s] = sel[s];
      topk_w[(size_t)row * k + s] = __float2half_rn(p[s] / psum);
    }
  }
  if (logits_out != nullptr && tid < E) logits_out[(size_t)row * E + tid] = lg[tid];
}

// ---------------------------------------------------------------- plan: one CTA
// n = T * k routed slots (row-major [T][k]).  Expert e's segment starts at sum_{e' < e} ceil(count_e' / BN) * BN; inside it
// the slots keep their order (ascending token, as torch.where gives).  tiles[j] = (expert, first row, valid rows, 0) for the
// j-th non-empty BN-row tile in expert order, (0, 0, 0, 0) past the last one.  Ids outside [0, E) are not routed
// (dest_row -1).
__global__ void __launch_bounds__(PLAN_THREADS)
moe_plan_kernel(const int32_t* __restrict__ ids, int n, int E, int BN, int tiles_max, int32_t* __restrict__ dest_row,
                int4* __restrict__ tiles, int pdl) {
  __shared__ int cnt[MOE_MAX_EXPERTS], run[MOE_MAX_EXPERTS], tstart[MOE_MAX_EXPERTS + 1], seg[MOE_MAX_EXPERTS];
  __shared__ int wc[PLAN_THREADS / 32][MOE_MAX_EXPERTS];
  if (pdl) { griddep_launch_dependents(); griddep_wait(); }
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid < MOE_MAX_EXPERTS) cnt[tid] = 0;
  __syncthreads();
  for (int i = tid; i < n; i += PLAN_THREADS) {
    const int e = ids[i];
    if ((unsigned)e < (unsigned)E) atomicAdd(&cnt[e], 1);
  }
  __syncthreads();
  if (tid == 0) {
    int r = 0, t = 0;
    for (int e = 0; e < E; ++e) {
      const int nt = (cnt[e] + BN - 1) / BN;
      seg[e] = run[e] = r; tstart[e] = t;
      r += nt * BN; t += nt;
    }
    tstart[E] = t;
  }
  __syncthreads();
  for (int j = tid; j < tiles_max; j += PLAN_THREADS) {
    int4 tl = make_int4(0, 0, 0, 0);
    if (j < tstart[E]) {
      int e = 0;
      while (tstart[e + 1] <= j) ++e;
      const int i = j - tstart[e];
      tl = make_int4(e, seg[e] + i * BN, min(BN, cnt[e] - i * BN), 0);
    }
    tiles[j] = tl;
  }
  // stable ranks, PLAN_THREADS slots per round: rank in the warp from __match_any_sync, warps in order per expert
  for (int base = 0; base < n; base += PLAN_THREADS) {
    for (int i = tid; i < (PLAN_THREADS / 32) * MOE_MAX_EXPERTS; i += PLAN_THREADS) (&wc[0][0])[i] = 0;
    __syncthreads();
    const int i = base + tid;
    const int e0 = i < n ? ids[i] : -1;
    const bool ok = (unsigned)e0 < (unsigned)E;
    const int e = ok ? e0 : -1;
    const unsigned peers = __match_any_sync(0xffffffffu, e);
    const int rank = __popc(peers & ((1u << lane) - 1u));
    if (ok && rank == 0) wc[warp][e] = __popc(peers);
    __syncthreads();
    if (tid < E) {
      int r = run[tid];
      for (int w = 0; w < PLAN_THREADS / 32; ++w) { const int c = wc[w][tid]; wc[w][tid] = r; r += c; }
      run[tid] = r;
    }
    __syncthreads();
    if (i < n) dest_row[i] = ok ? wc[warp][e] + rank : -1;
    __syncthreads();
  }
}

// ---------------------------------------------------------------- gather: one CTA per routed slot
// Slot i = (token i / k) goes to row dest_row[i] of the permuted tuple: its INT4 row, INT8 keeper row and the scales of
// every group, the latter in the ldmatrix-replicated layout (scale_index(row), 4 replicas) with pitch S(rows_cap).
__global__ void __launch_bounds__(GATHER_THREADS)
moe_gather_kernel(const int8_t* __restrict__ o8, const uint8_t* __restrict__ o4, const __half* __restrict__ s8,
                  const __half* __restrict__ s4, int hidden, int k, int lda_src, const int32_t* __restrict__ dest_row,
                  int8_t* __restrict__ p8, uint8_t* __restrict__ p4, __half* __restrict__ ps8, __half* __restrict__ ps4,
                  int lda_dst, int pdl) {
  if (pdl) { griddep_launch_dependents(); griddep_wait(); }
  const int i = blockIdx.x, tid = threadIdx.x;
  const int r = dest_row[i], t = i / k;
  if (r < 0) return;
  const int chunks = (hidden - 128) / 32;                     // 16-byte chunks of a packed INT4 row
  const uint4* src4 = reinterpret_cast<const uint4*>(o4 + (size_t)t * ((hidden - 128) / 2));
  uint4* dst4 = reinterpret_cast<uint4*>(p4 + (size_t)r * ((hidden - 128) / 2));
  for (int c = tid; c < chunks; c += GATHER_THREADS) dst4[c] = ld_cg_v4(src4 + c);
  if (tid < 8) reinterpret_cast<uint4*>(p8 + (size_t)r * 128)[tid] = ld_cg_v4(reinterpret_cast<const uint4*>(o8 + (size_t)t * 128) + tid);
  const int G = hidden / 128 - 1, si = scale_index(t), di = scale_index(r);
  for (int g = tid; g <= G; g += GATHER_THREADS) {
    const __half v = g < G ? s4[(size_t)g * lda_src + si] : s8[si];
    __half* dst = g < G ? ps4 + (size_t)g * lda_dst : ps8;
#pragma unroll
    for (int j = 0; j < 4; ++j) dst[di + 2 * j] = v;
  }
}

// ---------------------------------------------------------------- combine: one CTA per token
// out[t] = (((+0 + fp16(y[r_1] * w_1)) + fp16(y[r_2] * w_2)) + ...) over t's slots in ascending expert order, one FP16
// rounding per product and per add: bit for bit `out.index_add_(0, tok, (y_e * w).half())` run expert by expert from
// zeros.  The _rn intrinsics keep the compiler from contracting a product and its add into one FMA.
__global__ void __launch_bounds__(COMBINE_THREADS)
moe_combine_kernel(const __half* __restrict__ y, const int32_t* __restrict__ ids, const __half* __restrict__ topw,
                   const int32_t* __restrict__ dest_row, int k, int hidden, __half* __restrict__ out, int pdl) {
  __shared__ int srow[MOE_MAX_TOPK];
  __shared__ __half sw[MOE_MAX_TOPK];
  __shared__ int ns;
  if (pdl) { griddep_launch_dependents(); griddep_wait(); }
  const int t = blockIdx.x, tid = threadIdx.x;
  if (tid == 0) {
    int eid[MOE_MAX_TOPK], m = 0;
    for (int s = 0; s < k; ++s) {
      const int r = dest_row[(size_t)t * k + s];
      if (r < 0) continue;
      const int e = ids[(size_t)t * k + s];
      const __half wv = topw[(size_t)t * k + s];
      int j = m++;
      while (j > 0 && eid[j - 1] > e) { eid[j] = eid[j - 1]; srow[j] = srow[j - 1]; sw[j] = sw[j - 1]; --j; }
      eid[j] = e; srow[j] = r; sw[j] = wv;
    }
    ns = m;
  }
  __syncthreads();
  const int m = ns;
  for (int c = tid; c < hidden / 8; c += COMBINE_THREADS) {
    __half2 acc[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[j] = __float2half2_rn(0.f);
    for (int s = 0; s < m; ++s) {
      const uint4 v = ld_cg_v4(reinterpret_cast<const uint4*>(y + (size_t)srow[s] * hidden) + c);
      const __half2* hv = reinterpret_cast<const __half2*>(&v);
      const __half2 w2 = __half2half2(sw[s]);
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[j] = __hadd2_rn(acc[j], __hmul2_rn(hv[j], w2));
    }
    reinterpret_cast<uint4*>(out + (size_t)t * hidden)[c] = *reinterpret_cast<const uint4*>(acc);
  }
}

}  // namespace atom
