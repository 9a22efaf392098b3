// quant_kernels.cuh -- activation reorder + dynamic per-group quantise kernels (plain, RMSNorm-fused, SiLU-fused).
//
// Replace reorder_fp16_i4_kernel      (/root/reference/kernels/include/Reorder/Reorder.cuh:64-190),
//         rmsnorm_fp16_i4_kernel      (/root/reference/kernels/include/RMSNorm/RMSNorm.cuh:66-238),
//         activate_fp16_i4_kernel     (/root/reference/kernels/include/Activate/Activate.cuh:67-180).
// Outputs are bit-identical to the reference kernels (same IEEE ops in the same association where the order
// matters: the RMSNorm sum of squares), but hidden_dim is a runtime multiple of 128 instead of the constant 4096 /
// 11008, and the work decomposition is one warp per 128-channel quantisation group: a lane owns 4 consecutive
// reordered channels, so INT4 output is one coalesced 64-B warp store and INT8 one 128-B store.
#pragma once
#include "gemm_i4_sm90.cuh"  // scale_index / scale_size

namespace atom {

// One warp quantises one 128-channel group.  v[4]: this lane's channels 4*lane .. 4*lane+3 of the group (FP32).
// Arithmetic of Reorder.cuh:119-170: absmax -> /7 (or /127 for the last group) -> scale stored as half(maxv),
// q = clamp(roundf(x * (1/maxv))).  max() is exact and order-free, so the lane mapping does not matter.
__device__ __forceinline__ void quant_group_store(const float (&v)[4], int lane, int row, int g, int num_groups,
                                                  int scale_ldm, int8_t* __restrict__ s8out, uint8_t* __restrict__ s4out,
                                                  __half* __restrict__ s8scale, __half* __restrict__ s4scale, int hidden) {
  float maxv = fmaxf(fmaxf(fabsf(v[0]), fabsf(v[1])), fmaxf(fabsf(v[2]), fabsf(v[3])));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) maxv = fmaxf(maxv, __shfl_xor_sync(0xffffffffu, maxv, o));
  const bool last = (g == num_groups - 1);
  maxv = maxv / (last ? 127.f : 7.f);                       // IEEE division, as `maxv /= 7`
  const float r_scale = 1.f / maxv;
  if (lane == 0) {
    const __half hs = __float2half_rn(maxv);
    __half* dst = last ? s8scale : s4scale + (size_t)g * scale_ldm;
    const int si = scale_index(row);
#pragma unroll
    for (int j = 0; j < 4; ++j) dst[si + 2 * j] = hs;       // replicated x4 (ldmatrix layout of the reference GEMM)
  }
  int q[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int t = (int)roundf(v[i] * r_scale);              // round half away from zero (CUDA round())
    q[i] = last ? max(-128, min(127, t)) : max(-8, min(7, t));
  }
  if (last) {
    const uint32_t w = (uint32_t)(q[0] & 0xff) | ((uint32_t)(q[1] & 0xff) << 8) | ((uint32_t)(q[2] & 0xff) << 16) |
                       ((uint32_t)(q[3] & 0xff) << 24);
    reinterpret_cast<uint32_t*>(s8out + (size_t)row * 128)[lane] = w;
  } else {
    const uint16_t w = (uint16_t)((q[0] & 0xf) | ((q[1] & 0xf) << 4) | ((q[2] & 0xf) << 8) | ((q[3] & 0xf) << 12));
    reinterpret_cast<uint16_t*>(s4out + (size_t)row * ((hidden - 128) / 2) + g * 64)[lane] = w;
  }
}

// ---------------------------------------------------------------- K3: reorder + quantise
// grid = rows, block = 512 (16 warps); the row is staged in smem once, every warp gathers its groups from there.
constexpr int QUANT_THREADS = 512, QUANT_WARPS = QUANT_THREADS / 32;
__global__ void __launch_bounds__(QUANT_THREADS)
reorder_quant_kernel(const __half* __restrict__ x, const int16_t* __restrict__ idx, int seq_len, int hidden,
                     int8_t* __restrict__ s8out, uint8_t* __restrict__ s4out, __half* __restrict__ s8scale,
                     __half* __restrict__ s4scale, int scale_ldm, int pdl) {
  extern __shared__ __align__(16) uint8_t smem_q[];
  if (pdl) { griddep_launch_dependents(); griddep_wait(); }      // opt-in PDL: the input is the preceding kernel's output
  __half* xs = reinterpret_cast<__half*>(smem_q);
  const int row = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, ng = hidden / 128;
  short4 id_next = (warp < ng) ? *reinterpret_cast<const short4*>(idx + warp * 128 + lane * 4) : make_short4(0, 0, 0, 0);
  const uint4* src = reinterpret_cast<const uint4*>(x + (size_t)row * hidden);
  for (int i = threadIdx.x; i < hidden / 8; i += blockDim.x) reinterpret_cast<uint4*>(xs)[i] = ld_cg_v4(src + i);
  __syncthreads();
  for (int g = warp; g < ng; g += QUANT_WARPS) {
    const short4 id = id_next;
    if (g + QUANT_WARPS < ng) id_next = *reinterpret_cast<const short4*>(idx + (g + QUANT_WARPS) * 128 + lane * 4);
    float v[4] = {__half2float(xs[(uint16_t)id.x]), __half2float(xs[(uint16_t)id.y]), __half2float(xs[(uint16_t)id.z]),
                  __half2float(xs[(uint16_t)id.w])};
    quant_group_store(v, lane, row, g, ng, scale_ldm, s8out, s4out, s8scale, s4scale, hidden);
  }
}

// ---------------------------------------------------------------- K4: RMSNorm + reorder + quantise
// grid = rows, block = 512.  The sum of squares keeps the reference's association so that rstd -- and with it
// every quantised value -- is bit-identical: thread t < 128 folds hidden/128 contiguous elements with fmaf, then
// s[t]+=s[t+64], s[t]+=s[t+32], then shfl_down 16..1 (RMSNorm.cuh:112-141).  The other 12 warps meanwhile stage
// the norm weight; afterwards all 16 warps quantise groups (at decode sizes the kernel is one latency chain per row,
// so the chain is kept short: 2 groups per warp at hidden 4096 instead of 8).
// With `residual` != nullptr the row is x + residual (one FP16 RN add per element, exactly what `residual + hidden_states`
// does in the reference's decoder layer, llama.py:266-292); the sum is also written to `sum_out` (the next residual).
template <bool kReduce>   // kReduce: x is the all-reduced sum, formed on the fly from the push all-reduce's receive buffers
__global__ void __launch_bounds__(QUANT_THREADS)
rmsnorm_quant_kernel(const __half* __restrict__ x, const __half* __restrict__ residual, __half* __restrict__ sum_out,
                     const __half* __restrict__ w, float eps, const int16_t* __restrict__ idx,
                     int seq_len, int hidden, int8_t* __restrict__ s8out, uint8_t* __restrict__ s4out,
                     __half* __restrict__ s8scale, __half* __restrict__ s4scale, int scale_ldm, ArArgs ar, int pdl) {
  extern __shared__ __align__(16) uint8_t smem_q[];
  if (pdl) { griddep_launch_dependents(); griddep_wait(); }
  // kReduce: x is the sum over the ranks of the row-parallel projection's partials, which the GEMM pushed into the
  // receive buffers (reduce half of the push all-reduce, comm_kernels.cuh): each 16-byte chunk is polled until its payload has
  // arrived and summed in rank order in FP32, rounded to FP16 -- the value the stand-alone all-reduce would have delivered
  const uint32_t ar_e = kReduce ? ar_ld_state(ar.state) + 1 : 0;
  const uint4* ar_local = kReduce
      ? reinterpret_cast<const uint4*>(ar.bufs[ar.rank]) + (long long)(ar_e % 3) * ar.world * (ar.slot / 8) : nullptr;
  unsigned long long ar_t0 = 0;
  __half* xs = reinterpret_cast<__half*>(smem_q);
  __half* ws = xs + hidden;                             // norm weight staged too: the gather then never touches global
  float* red = reinterpret_cast<float*>(smem_q + (size_t)hidden * 4);
  const int row = blockIdx.x, tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31, ng = hidden / 128;
  const int ept = hidden / 128;                       // contiguous elements per thread (multiple of 8 when hidden%1024==0)
  const __half* xr = x + (size_t)row * hidden;
  // independent loads first: the first group's reorder indices and the weight row travel while the row is reduced
  short4 id_next = (warp < ng) ? *reinterpret_cast<const short4*>(idx + warp * 128 + lane * 4) : make_short4(0, 0, 0, 0);
  float sumv = 0.f;
  if (kReduce) {      // all 16 warps form the all-reduced row in shared memory first (2 chunks per thread at hidden = 8192)
    for (int ci = tid; ci < hidden / 8; ci += QUANT_THREADS)
      reinterpret_cast<uint4*>(xs)[ci] = ar_reduce_chunk(ar_local, ar.slot / 8, (long long)row * (hidden / 8) + ci, ar.world, ar_t0);
    __syncthreads();
  }
  if (tid >= 128) {
    for (int i = tid - 128; i < hidden / 8; i += QUANT_THREADS - 128)
      reinterpret_cast<uint4*>(ws)[i] = ld_cg_v4(reinterpret_cast<const uint4*>(w) + i);
  } else if ((ept & 7) == 0) {
    for (int i = 0; i < ept; i += 8) {
      uint4 u = kReduce ? *reinterpret_cast<const uint4*>(xs + tid * ept + i) : *reinterpret_cast<const uint4*>(xr + tid * ept + i);
      if (residual != nullptr) {
        const uint4 rr = *reinterpret_cast<const uint4*>(residual + (size_t)row * hidden + tid * ept + i);
        __half2* hu = reinterpret_cast<__half2*>(&u);
        const __half2* hr = reinterpret_cast<const __half2*>(&rr);
#pragma unroll
        for (int j = 0; j < 4; ++j) hu[j] = __hadd2(hu[j], hr[j]);
        *reinterpret_cast<uint4*>(sum_out + (size_t)row * hidden + tid * ept + i) = u;
      }
      *reinterpret_cast<uint4*>(xs + tid * ept + i) = u;
      const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(h[j]);
        sumv = fmaf(f.x, f.x, sumv);
        sumv = fmaf(f.y, f.y, sumv);
      }
    }
  } else {
    for (int i = 0; i < ept; ++i) {
      __half hv = xr[tid * ept + i];
      if (residual != nullptr) {
        hv = __hadd(hv, residual[(size_t)row * hidden + tid * ept + i]);
        sum_out[(size_t)row * hidden + tid * ept + i] = hv;
      }
      xs[tid * ept + i] = hv;
      const float f = __half2float(hv);
      sumv = fmaf(f, f, sumv);
    }
  }
  if (tid < 128) red[tid] = sumv;
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
  for (int g = warp; g < ng; g += QUANT_WARPS) {
    const short4 id = id_next;
    if (g + QUANT_WARPS < ng) id_next = *reinterpret_cast<const short4*>(idx + (g + QUANT_WARPS) * 128 + lane * 4);
    const int ids[4] = {(uint16_t)id.x, (uint16_t)id.y, (uint16_t)id.z, (uint16_t)id.w};
    float v[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      // half(float(x) * float(w) * rstd): two FP32 roundings then RN to half (RMSNorm.cuh:150), widened again for the tail
      const float y = __half2float(xs[ids[i]]) * __half2float(ws[ids[i]]) * rstd;
      v[i] = __half2float(__float2half_rn(y));
    }
    quant_group_store(v, lane, row, g, ng, scale_ldm, s8out, s4out, s8scale, s4scale, hidden);
  }
  if (kReduce) {     // housekeeping of the fused all-reduce, off the critical path
    ar_reset_previous(ar, ar_e, blockIdx.x, gridDim.x, tid, QUANT_THREADS);
    __syncthreads();
    if (tid == 0) ar_complete(ar, ar_e, (long long)seq_len * hidden / 8, gridDim.x);
  }
}

// ---------------------------------------------------------------- K5: SiLU(a) * b + quantise (no reorder)
// one warp per (row, group); 8 warps per block, flattened over rows x groups.

__global__ void __launch_bounds__(256)
activate_quant_kernel(const __half* __restrict__ a, const __half* __restrict__ b, int seq_len, int hidden,
                      int8_t* __restrict__ s8out, uint8_t* __restrict__ s4out, __half* __restrict__ s8scale,
                      __half* __restrict__ s4scale, int scale_ldm, int pdl) {
  if (pdl) { griddep_launch_dependents(); griddep_wait(); }
  const int ng = hidden / 128;
  const long long unit = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (unit >= (long long)seq_len * ng) return;
  const int row = (int)(unit / ng), g = (int)(unit % ng), lane = threadIdx.x & 31;
  const size_t off = (size_t)row * hidden + g * 128 + lane * 4;
  const uint2 ua = *reinterpret_cast<const uint2*>(a + off);
  const uint2 ub = *reinterpret_cast<const uint2*>(b + off);
  const __half2* ha = reinterpret_cast<const __half2*>(&ua);
  const __half2* hb = reinterpret_cast<const __half2*>(&ub);
  float v[4];
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const float2 fa = __half22float2(ha[j]), fb = __half22float2(hb[j]);
    v[2 * j + 0] = silu_ref(fa.x) * fb.x;
    v[2 * j + 1] = silu_ref(fa.y) * fb.y;
  }
  quant_group_store(v, lane, row, g, ng, scale_ldm, s8out, s4out, s8scale, s4scale, hidden);
}

}  // namespace atom
