// gemm_i4_sm90.cuh -- W4A4 group-quantised GEMM with INT8 keeper for H100 (sm_90a).
//
// Replaces the reference's compute_gemm_imma / DenseLayerGEMM_i4[_o4]_kernel (kernels/include/GEMM/Dense_layer_gemm_i4_o16.cuh,
// e2e/punica-atom/punica/ops/csrc/GEMM/DenseLayerGEMM_i4_o4.cu).  Same operands, same layouts, same arithmetic (exact INT32
// group sums, one FP16 multiply of the two scales, FP32 fma accumulation in group order, keeper last, RN cast to half) --
// different machine.  Hopper's warpgroup MMA has no INT4 type, so both operands are widened to INT8 (value * 16: a shift and
// a mask, no sign extension) on their way to the tensor cores:
//
//   TMA: packed INT4 tiles (64 B rows) of the weights (128 channels) and of the tokens (BN rows) -> smem "packed ring"
//   producer warpgroup: one thread issues the TMA loads; all four warps widen the TOKEN tile into the K-major SWIZZLE_128B
//       INT8 operand ("expanded ring") and stage the group's scales next to it
//   two consumer warpgroups, 64 channels each: the WEIGHTS are the wgmma A operand and are widened in REGISTERS (one LDS.128
//       per row and group, no shared-memory round trip); wgmma m64nBNk32 s8 x 4 per 128-wide quantisation group, INT32
//       accumulators in registers; acc = fmaf(float(c), float(hmul(sA, sB)), acc)
//   the INT8 keeper group is TMA'd straight into SWIZZLE_128B tiles (weights read as register fragments, tokens as operand B)
//   epilogue: the FP32 tile is transposed through shared memory ([token][channel]) and leaves as token rows: FP16 (o16),
//       asymmetric INT4 per 128-channel head (o4), both by channel tile (fused q/k/v), SiLU(gate) * up + dynamic quantisation
//       (fused gate/up: the CTA holds the gate and the up rows of the same 128 channels), or FP16 into every rank's
//       all-reduce receive buffer (push).
//   K may be split over a thread-block cluster: every rank stages its partial tile, then sums its share of the token rows
//       from all ranks' shared memory in rank order (deterministic).
//
// Inside a 128-wide group K may be permuted freely as long as both operands agree: k-step j of thread quad q multiplies the
// nibbles of packed word 4q + j, even ones first.  The factor 16 * 16 is carried by the accumulator and removed exactly at
// the output cast.
#pragma once
#include "ptx_sm90.cuh"

namespace atom {

struct GemmArgs {
  const __half* a_scale;         // [G][S(M)]  ldmatrix-replicated layout (Reorder.cuh:39-50)
  const __half* b_scale;         // [G][ldb_scale]
  const __half* a_keeper_scale;  // [S(M)]
  const __half* b_keeper_scale;  // [N]
  __half* d;                     // o16: [M][N]
  uint8_t* d4;                   // o4 : [M][N/2]
  __half2* d_scale;              // o4 : [M][N/128] (scale, zero)
  uint8_t* d4_v;                 // fused q/k/v projection (EPI_QKV): channel tiles [0, seg_tiles) are q -> d (o16), the next
  __half2* d_scale_v;            //   kv_tiles are k -> d4 / d_scale (o4), the last kv_tiles v -> d4_v / d_scale_v (o4)
  int seg_tiles, kv_tiles;       //   (multi-head attention: kv_tiles == seg_tiles; grouped-query: fewer KV heads)
  // fused gate/up projection + SiLU(gate)*up + dynamic quantisation (EPI_GATEUP): the activation 4-tuple that
  // activate_fp16_i4 would have produced (Activate.cuh:67-180); gu_rows = intermediate size I (up rows start at I)
  int8_t* q8_out; uint8_t* q4_out; __half* q8_scale; __half* q4_scale; int gu_rows;
  int ldb_scale;                 // pitch (halves) of the b_scale rows
  int M, N, G;                   // G = number of INT4 groups = K/128 - 1
  int lda_scale;                 // S(M)
  unsigned long long* trace;     // optional device buffer [ctas][128] of clock64 stamps (atom_gemm_set_trace), else null
  ArArgs ar;                     // EPI_PUSH: D goes to slot [call % 3][rank] of every rank's receive buffer (comm_kernels.cuh);
                                 // the consumer is rmsnorm_quant_kernel's reducing variant
  // grouped expert GEMM (EPI_GROUPED): blockIdx.y indexes `tiles`, one (expert, first row, valid rows, 0) per token tile
  // (valid rows 0 = empty); the weights of all experts are stacked, `expert_rows` rows per expert (2I gate/up, H down)
  const int4* tiles;
  int expert_rows;
};

// timeline stamps for pipeline debugging: per CTA  0 start | 1 setup done | 2 main loop done | 3 reduction done | 4 end
__device__ __forceinline__ void trace_stamp(const GemmArgs& a, int slot) {
  if (a.trace != nullptr) {
    const int cta = (blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    a.trace[(size_t)cta * 128 + slot] = (unsigned long long)clock64();
  }
}

__device__ __forceinline__ float silu_ref(float x) { return x / (1.0f + expf(-x)); }   // Activate.cuh:28
__host__ __device__ __forceinline__ int scale_index(int row) { return (row / 16) * 64 + (row % 8) * 8 + ((row / 8) % 2); }
__host__ __device__ __forceinline__ int scale_size(int m) { return m / 16 * 64 + 64 - (1 - (m % 16) / 8) * (8 - (m % 8)) * 8; }

// EPI_QKV: o16 for the q tiles, o4 for the k and v tiles.  EPI_GATEUP: 256 weight rows per CTA (gate tile + up tile).
// EPI_PUSH: EPI_O16 whose result goes to every rank's all-reduce receive buffer.
// EPI_GROUPED: a mode bit or-ed into EPI_O16 / EPI_GATEUP -- the grouped expert GEMM of the MoE block (moe_kernels.cuh).  A
// tile of the token-tile table selects the expert (weight rows and scales) and the rows of the permuted activations; rows
// past the tile's valid count are not stored.  A bit of the epilogue parameter rather than a parameter of its own, so that
// every other instantiation keeps its symbol and its code.
enum { EPI_O16 = 0, EPI_O4 = 1, EPI_QKV = 2, EPI_GATEUP = 3, EPI_PUSH = 4, EPI_GROUPED = 8 };

template <int BN, int kSplit, int kEpi>
struct GemmCfg {
  static constexpr int ROWS = (kEpi & ~EPI_GROUPED) == EPI_GATEUP ? 256 : 128;    // weight rows per CTA
  static constexpr int MT = ROWS / 128;                          // 64-row wgmma tiles per consumer warpgroup
  static constexpr int THREADS = 384;                            // producer warpgroup + two consumer warpgroups
  static constexpr int PACK = BN <= 32 ? 8 : 4;                  // packed ring depth (groups): decode shapes are a weight stream
  static constexpr int EXP = BN <= 64 ? 4 : 3;                   // expanded token tiles / scale slots
  static constexpr int PACK_W = ROWS * 64, PACK_Q = BN * 64;     // bytes per packed group
  static constexpr int EXP_Q = BN * 128 < 1024 ? 1024 : BN * 128;
  static constexpr int SCALE_BYTES = (ROWS + BN) * 2;            // [ROWS] weight-scale halves, [BN] token-scale halves
  static constexpr int OFF_EXP = 0;
  static constexpr int OFF_KEEP_Q = OFF_EXP + EXP * EXP_Q;
  static constexpr int OFF_KEEP_W = OFF_KEEP_Q + EXP_Q;
  static constexpr int OFF_PACK_W = OFF_KEEP_W + ROWS * 128;
  static constexpr int OFF_PACK_Q = OFF_PACK_W + PACK * PACK_W;
  static constexpr int OFF_SCALE = OFF_PACK_Q + PACK * PACK_Q;
  static constexpr int OFF_BAR = OFF_SCALE + (EXP + 1) * SCALE_BYTES;   // slot EXP: the keeper's scales
  static constexpr int NUM_BARS = 2 * PACK + 2 * EXP + 1;
  static constexpr int SMEM_BYTES = OFF_BAR + NUM_BARS * 8 + 1024;   // + slack for the 1024-B alignment fix-up
  static constexpr int TILE_PITCH = ROWS + 4;                    // floats per token row of the staged output tile
  static constexpr int KEEP_TX = ROWS * 128 + BN * 128;
  static_assert(BN == 16 || BN == 32 || BN == 64 || BN == 128, "token tile");
  static_assert(BN * TILE_PITCH * 4 <= OFF_SCALE, "the output tile is staged over the idle operand rings");
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget");
  static_assert(kSplit == 1 || kEpi == EPI_O16 || kEpi == EPI_PUSH, "the quantising epilogues work on un-split FP32 sums");
  static_assert(!(kEpi & EPI_GROUPED) || (kSplit == 1 && BN <= 64), "grouped mode: token tiles of 16 / 32 / 64, no K split");
};

template <int BN, int kSplit, int kEpi>
__global__ void __launch_bounds__(384, 1)
gemm_i4_kernel(const __grid_constant__ CUtensorMap tm_w4,   // packed INT4 weights   (box 64 B x 128 rows)
               const __grid_constant__ CUtensorMap tm_a4,   // packed INT4 tokens    (box 64 B x BN rows)
               const __grid_constant__ CUtensorMap tm_w8,   // INT8 keeper weights   (box 128 B x 128 rows, SW128)
               const __grid_constant__ CUtensorMap tm_a8,   // INT8 keeper tokens    (box 128 B x BN rows, SW128)
               const GemmArgs args) {
  using C = GemmCfg<BN, kSplit, kEpi>;
  constexpr bool kGrouped = (kEpi & EPI_GROUPED) != 0;
  constexpr int kE = kEpi & ~EPI_GROUPED;                    // the epilogue
  constexpr int NR = BN / 2;                                // accumulator registers per 64-row tile
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-B alignment (SWIZZLE_128B atoms) by offsetting the shared array, NOT by integer-casting the pointer:
  // an integer round trip makes the compiler fall back to generic LD/ST for every smem access.
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);

  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::OFF_BAR);
  uint64_t* pack_full = bars;                          // TMA landed the group's packed tiles            (1 + tx)
  uint64_t* pack_empty = pack_full + C::PACK;          // every warp has read them                       (12)
  uint64_t* exp_full = pack_empty + C::PACK;           // token operand + scales of the group in place   (4 producer warps)
  uint64_t* exp_empty = exp_full + C::EXP;             // consumers are done with them                   (8 consumer warps)
  uint64_t* keep_full = exp_empty + C::EXP;            // keeper tiles + scales landed                   (1 + tx, 4 producer warps)

  // the warp index through a shuffle: the compiler then knows the role branches below are warp-uniform
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  // blockIdx.x = output-channel tile: CTAs launched together share the token tile (L2) and stream disjoint weights
  // grouped mode: gtile = the tile's (expert, first row, valid rows, 0).  The table is written by the preceding kernels: nothing of
  // it, of the activations or of the expert's weights is read before griddepcontrol.wait (no weight prefetch ahead of the
  // wait in this mode).  Every grouped-only term below sits in a `kGrouped ?` branch, so the other instantiations compile
  // to the code they had before the mode existed.
  int4 gtile = make_int4(0, 0, 0, 0);
  if constexpr (kGrouped) {
    griddep_wait();
    gtile = args.tiles[blockIdx.y];
    if (gtile.z <= 0) return;                                 // empty tile: the whole CTA leaves before any barrier
  }
  const int n0 = blockIdx.x * 128, m0 = kGrouped ? gtile.y : blockIdx.y * BN;
  const int n_limit = kE == EPI_GATEUP ? args.gu_rows : args.N;   // channels of one weight segment

  // K split over the cluster: groups [g_begin, g_end) of the G+1 groups (index G = INT8 keeper)
  const int total_groups = args.G + 1;
  int g_begin = 0, g_end = total_groups;
  uint32_t krank = 0;
  if constexpr (kSplit > 1) {
    krank = cluster_ctarank();
    const int per = (total_groups + kSplit - 1) / kSplit;
    g_begin = min((int)krank * per, total_groups);
    g_end = min(g_begin + per, total_groups);
  }
  const int n4 = max(0, min(g_end, args.G) - g_begin);        // INT4 groups of this CTA
  const bool has_keeper = g_end == total_groups && g_end > g_begin;
  if (threadIdx.x == 0) trace_stamp(args, 0);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_w4); tma_prefetch_desc(&tm_a4); tma_prefetch_desc(&tm_w8); tma_prefetch_desc(&tm_a8);
    for (int i = 0; i < C::PACK; ++i) { mbar_init(&pack_full[i], 1); mbar_init(&pack_empty[i], 12); }
    for (int i = 0; i < C::EXP; ++i) { mbar_init(&exp_full[i], 4); mbar_init(&exp_empty[i], 8); }
    mbar_init(keep_full, 5);
    fence_barrier_init();
  }
  __syncthreads();
  // split-K: a CTA's shared memory may only be read remotely while that CTA is alive -- every thread arrives here (cheap,
  // non-blocking) and waits before the reduction
  if constexpr (kSplit > 1) cluster_arrive_relaxed();
  if (threadIdx.x == 0) trace_stamp(args, 1);

  if (warp < 4) {
    // ============================================================ producer warpgroup: TMA + token widening + scales
    const int t = threadIdx.x;
    // part 1 = arm the barrier and load the WEIGHT tiles, part 2 = load the TOKEN tile, 0 = both.  The weights do not
    // depend on the preceding kernel and are fetched before griddepcontrol.wait.
    auto issue_stage = [&](int s, int part) {
      const int ps = s % C::PACK, g = g_begin + s;
      if (part != 2) {
        mbar_arrive_expect_tx(&pack_full[ps], C::PACK_W + C::PACK_Q);
        tma_load_2d(smem + C::OFF_PACK_W + ps * C::PACK_W, &tm_w4, &pack_full[ps], g * 64,
                    kGrouped ? gtile.x * args.expert_rows + n0 : n0);
        if constexpr (kE == EPI_GATEUP)
          tma_load_2d(smem + C::OFF_PACK_W + ps * C::PACK_W + 128 * 64, &tm_w4, &pack_full[ps], g * 64,
                      kGrouped ? gtile.x * args.expert_rows + args.gu_rows + n0 : args.gu_rows + n0);
      }
      if (part != 1) tma_load_2d(smem + C::OFF_PACK_Q + ps * C::PACK_Q, &tm_a4, &pack_full[ps], g * 64, m0);
    };
    // a group's scales: weight scales of the tile's channels (16-B chunks), token scales in token order
    auto load_scales = [&](const __half* bs_row, const __half* as_row, uint4& sbv, __half& sav) {
      sbv = make_uint4(0, 0, 0, 0);
      sav = __ushort_as_half(0);
      if (t < C::ROWS / 8) {
        const int seg = t / 16, c = t % 16;                         // gate/up: segment 1 = the up rows
        if (n0 + 8 * c < n_limit) sbv = ld_cg_v4(bs_row + (size_t)seg * args.gu_rows + n0 + 8 * c);
      }
      if (t < BN && m0 + t < (kGrouped ? gtile.y + gtile.z : args.M)) sav = __ushort_as_half(ld_cg_u16(as_row + scale_index(m0 + t)));
    };
    auto store_scales = [&](int slot_idx, const uint4& sbv, __half sav) {
      uint8_t* slot = smem + C::OFF_SCALE + slot_idx * C::SCALE_BYTES;
      if (t < C::ROWS / 8) reinterpret_cast<uint4*>(slot)[t] = sbv;
      if (t < BN) reinterpret_cast<__half*>(slot + C::ROWS * 2)[t] = sav;
    };
    griddep_launch_dependents();
    if (t == 0) {
      const int first = min(C::PACK, n4);
      for (int s = 0; s < first; ++s) issue_stage(s, 1);
      if (has_keeper) {
        mbar_arrive_expect_tx(keep_full, C::KEEP_TX);
        tma_load_2d(smem + C::OFF_KEEP_W, &tm_w8, keep_full, 0, kGrouped ? gtile.x * args.expert_rows + n0 : n0);
        if constexpr (kE == EPI_GATEUP)
          tma_load_2d(smem + C::OFF_KEEP_W + 128 * 128, &tm_w8, keep_full, 0,
                      kGrouped ? gtile.x * args.expert_rows + args.gu_rows + n0 : args.gu_rows + n0);
      }
      griddep_wait();                       // from here on the preceding kernel's output (the activations) may be read
      for (int s = 0; s < first; ++s) issue_stage(s, 2);
      if (has_keeper) tma_load_2d(smem + C::OFF_KEEP_Q, &tm_a8, keep_full, 0, m0);
    } else {
      griddep_wait();
    }
    uint4 sbv;
    __half sav;
    if (has_keeper) {
      load_scales(kGrouped ? args.b_keeper_scale + (size_t)gtile.x * args.expert_rows : args.b_keeper_scale, args.a_keeper_scale, sbv, sav);
      store_scales(C::EXP, sbv, sav);
      __syncwarp();
      if (lane == 0) mbar_arrive(keep_full);
    }
    for (int s = 0; s < n4; ++s) {
      const int ps = s % C::PACK, es = s % C::EXP, g = g_begin + s;
      load_scales((kGrouped ? args.b_scale + (size_t)gtile.x * args.G * args.ldb_scale : args.b_scale) + (size_t)g * args.ldb_scale, args.a_scale + (size_t)g * args.lda_scale, sbv, sav);
      if (t == 0 && s >= 1 && s + C::PACK - 1 < n4) {               // refill the slot the previous group has left
        const int nx = s + C::PACK - 1;
        mbar_wait(&pack_empty[nx % C::PACK], ((nx / C::PACK) - 1) & 1);
        issue_stage(nx, 0);
      }
      mbar_wait(&pack_full[ps], (s / C::PACK) & 1);
      if (s >= C::EXP) mbar_wait(&exp_empty[es], ((s / C::EXP) - 1) & 1);
      const uint8_t* packed = smem + C::OFF_PACK_Q + ps * C::PACK_Q;
      uint8_t* expanded = smem + C::OFF_EXP + es * C::EXP_Q;
#pragma unroll
      for (int c = t; c < BN * 4; c += 128) {
        const int r = c >> 2, qq = c & 3;
        const uint4 w = *reinterpret_cast<const uint4*>(packed + c * 16);
        const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
        uint8_t* row = expanded + (r >> 3) * 1024 + (r & 7) * 128 + 4 * qq;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          *reinterpret_cast<uint32_t*>(row + (((2 * j) ^ (r & 7)) << 4)) = (ww[j] << 4) & 0xF0F0F0F0u;
          *reinterpret_cast<uint32_t*>(row + (((2 * j + 1) ^ (r & 7)) << 4)) = ww[j] & 0xF0F0F0F0u;
        }
      }
      store_scales(es, sbv, sav);
      fence_proxy_async_smem();             // generic-proxy stores -> visible to the wgmma operand fetch
      __syncwarp();
      if (lane == 0) { mbar_arrive(&pack_empty[ps]); mbar_arrive(&exp_full[es]); }
    }
    if constexpr (kSplit > 1) { cluster_wait(); cluster_arrive(); cluster_wait(); cluster_arrive(); cluster_wait(); }
  } else {
    // ============================================================ consumer warpgroups
    const int cw = warp - 4, wg = cw >> 2, wq = cw & 3;          // consumer warp, its warpgroup, warp inside the warpgroup
    const int g8 = lane >> 2, q = lane & 3;
    float acc[C::MT][NR];
#pragma unroll
    for (int t = 0; t < C::MT; ++t)
#pragma unroll
      for (int i = 0; i < NR; ++i) acc[t][i] = 0.f;
    griddep_wait();

    // acc[t] += float(d) * float(hmul(sA[token], sB[channel'])) for the fragment's two channel rows `ch` and `ch + 8`.  As in
    // the reference's fragment layout, a channel pair (2p, 2p+1) shares one weight scale per token: the even channel's for
    // tokens with (token % 16) < 8, the odd channel's for the others (sb = the tile's weight scales, sa = its token scales).
    auto dequant = [&](float (&a)[NR], const uint32_t (&d)[NR], const __half* sa, const __half* sb, int ch, bool keeper) {
      const __half2 lo = *reinterpret_cast<const __half2*>(sb + (ch & ~1)), hi = *reinterpret_cast<const __half2*>(sb + ((ch + 8) & ~1));
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const __half2 sa2 = *reinterpret_cast<const __half2*>(sa + 8 * j + 2 * q);
        const __half2 lo2 = __half2half2((j & 1) ? __high2half(lo) : __low2half(lo)), hi2 = __half2half2((j & 1) ? __high2half(hi) : __low2half(hi));
        const float2 rl = __half22float2(__hmul2(sa2, lo2)), rh = __half22float2(__hmul2(sa2, hi2));
        // INT4 groups carry a factor 256 (both operands are value*16); lift the keeper to the same domain
        const int sh = keeper ? 8 : 0;
        a[4 * j + 0] = fmaf((float)((int32_t)d[4 * j + 0] << sh), rl.x, a[4 * j + 0]);
        a[4 * j + 1] = fmaf((float)((int32_t)d[4 * j + 1] << sh), rl.y, a[4 * j + 1]);
        a[4 * j + 2] = fmaf((float)((int32_t)d[4 * j + 2] << sh), rh.x, a[4 * j + 2]);
        a[4 * j + 3] = fmaf((float)((int32_t)d[4 * j + 3] << sh), rh.y, a[4 * j + 3]);
      }
    };

    for (int s = 0; s < n4; ++s) {
      const int ps = s % C::PACK, es = s % C::EXP;
      mbar_wait(&pack_full[ps], (s / C::PACK) & 1);
      uint4 wa[C::MT], wb[C::MT];
#pragma unroll
      for (int t = 0; t < C::MT; ++t) {
        const uint8_t* p = smem + C::OFF_PACK_W + ps * C::PACK_W + ((wg * C::MT + t) * 64 + wq * 16 + g8) * 64 + q * 16;
        wa[t] = *reinterpret_cast<const uint4*>(p);
        wb[t] = *reinterpret_cast<const uint4*>(p + 8 * 64);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&pack_empty[ps]);
      mbar_wait(&exp_full[es], (s / C::EXP) & 1);
      const uint64_t db = wgmma_desc_k_sw128(smem_u32(smem + C::OFF_EXP + es * C::EXP_Q));
      const __half* sb = reinterpret_cast<const __half*>(smem + C::OFF_SCALE + es * C::SCALE_BYTES);
      const __half* sa = sb + C::ROWS;
#pragma unroll
      for (int t = 0; t < C::MT; ++t) {
        const uint32_t xa[4] = {wa[t].x, wa[t].y, wa[t].z, wa[t].w}, xb[4] = {wb[t].x, wb[t].y, wb[t].z, wb[t].w};
        uint32_t d[NR];
#pragma unroll
        for (int i = 0; i < NR; ++i) d[i] = 0;
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < 4; ++j)     // 4 x K=32 per 128-wide group; +32 B inside the swizzle atom per step
          wgmma_s8_rs(d, (xa[j] << 4) & 0xF0F0F0F0u, (xb[j] << 4) & 0xF0F0F0F0u, xa[j] & 0xF0F0F0F0u, xb[j] & 0xF0F0F0F0u,
                      db + (uint64_t)(2 * j), j > 0);
        wgmma_commit();
        wgmma_wait_all();
        const int ch = (wg * C::MT + t) * 64 + wq * 16 + g8;
        dequant(acc[t], d, sa, sb, ch, false);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&exp_empty[es]);
    }
    if (has_keeper) {
      mbar_wait(keep_full, 0);
      const uint64_t db = wgmma_desc_k_sw128(smem_u32(smem + C::OFF_KEEP_Q));
      const __half* sb = reinterpret_cast<const __half*>(smem + C::OFF_SCALE + C::EXP * C::SCALE_BYTES);
      const __half* sa = sb + C::ROWS;
#pragma unroll
      for (int t = 0; t < C::MT; ++t) {
        const int ch = (wg * C::MT + t) * 64 + wq * 16 + g8;     // row of the CTA's weight tile; rows of 128 B, SW128
        const uint8_t* ra = smem + C::OFF_KEEP_W + (ch >> 3) * 1024 + (ch & 7) * 128 + 4 * q;
        const uint8_t* rb = ra + 1024;                           // row + 8: the next swizzle atom, same row inside it
        uint32_t d[NR];
#pragma unroll
        for (int i = 0; i < NR; ++i) d[i] = 0;
        uint32_t ka[4][4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          ka[j][0] = *reinterpret_cast<const uint32_t*>(ra + (((2 * j) ^ (ch & 7)) << 4));
          ka[j][1] = *reinterpret_cast<const uint32_t*>(rb + (((2 * j) ^ (ch & 7)) << 4));
          ka[j][2] = *reinterpret_cast<const uint32_t*>(ra + (((2 * j + 1) ^ (ch & 7)) << 4));
          ka[j][3] = *reinterpret_cast<const uint32_t*>(rb + (((2 * j + 1) ^ (ch & 7)) << 4));
        }
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < 4; ++j) wgmma_s8_rs(d, ka[j][0], ka[j][1], ka[j][2], ka[j][3], db + (uint64_t)(2 * j), j > 0);
        wgmma_commit();
        wgmma_wait_all();
        dequant(acc[t], d, sa, sb, ch, true);
      }
    }
    if (cw == 0 && lane == 0) trace_stamp(args, 2);

    // ------------------------------------------------------------ stage the FP32 tile as [token][channel]
    asm volatile("bar.sync 1, 256;" ::: "memory");     // both consumer warpgroups have left the operand rings
    float* tile = reinterpret_cast<float*>(smem);
#pragma unroll
    for (int t = 0; t < C::MT; ++t) {
      const int ch = (wg * C::MT + t) * 64 + wq * 16 + g8;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int tk = 8 * j + 2 * q;
        tile[tk * C::TILE_PITCH + ch] = acc[t][4 * j + 0];
        tile[(tk + 1) * C::TILE_PITCH + ch] = acc[t][4 * j + 1];
        tile[tk * C::TILE_PITCH + ch + 8] = acc[t][4 * j + 2];
        tile[(tk + 1) * C::TILE_PITCH + ch + 8] = acc[t][4 * j + 3];
      }
    }
    asm volatile("bar.sync 1, 256;" ::: "memory");
    if constexpr (kSplit > 1) { cluster_wait(); cluster_arrive(); cluster_wait(); }   // every rank's tile is staged
    if (cw == 0 && lane == 0) trace_stamp(args, 3);

    // ------------------------------------------------------------ output: one warp per token row, 4 channels per lane
    constexpr float kInv = 1.0f / 256.0f;   // exact: removes the 16 * 16 operand factor
    // q/k/v: tiles [0, seg_tiles) are q, the next kv_tiles k, the last kv_tiles v (kv_tiles == seg_tiles: three equal parts)
    const int bx = (int)blockIdx.x;
    const int seg = kE == EPI_QKV ? (bx < args.seg_tiles ? 0 : (bx < args.seg_tiles + args.kv_tiles ? 1 : 2)) : 0;
    const int otile = kE == EPI_QKV ? (seg == 0 ? bx : bx - args.seg_tiles - (seg - 1) * args.kv_tiles) : bx;
    const int n_out_dim = kE == EPI_QKV ? (seg == 0 ? args.seg_tiles : args.kv_tiles) * 128 : args.N;   // row length of the output this tile writes
    const int n_out = otile * 128 + lane * 4;
    const bool o16 = kE == EPI_O16 || kE == EPI_PUSH || (kE == EPI_QKV && seg == 0);
    for (int tk = cw; tk < BN; tk += 8) {
      const int m = m0 + tk;
      if (m >= (kGrouped ? gtile.y + gtile.z : args.M)) break;
      if (kSplit > 1 && (tk % kSplit) != (int)krank) continue;  // split-K: rank r reduces + stores the token rows r mod kSplit
      float v[4];
      {
        const float4 f = *reinterpret_cast<const float4*>(tile + tk * C::TILE_PITCH + lane * 4);
        v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
      }
      if constexpr (kSplit > 1) {
        const uint32_t local = smem_u32(tile + tk * C::TILE_PITCH + lane * 4);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float sum = 0.f;
#pragma unroll
          for (int rk = 0; rk < kSplit; ++rk) {
            const float p = rk == (int)krank ? v[e] : ld_dsmem_f32(mapa_shared(local + 4 * e, rk));
            sum = rk == 0 ? p : sum + p;
          }
          v[e] = sum;
        }
      }
      if constexpr (kE == EPI_GATEUP) {
        // SiLU(gate) * up, then the dynamic quantisation of activate_fp16_i4 (Activate.cuh:102-166) for this 128-channel
        // group of the token.  Both projections are rounded to FP16 first, as they are when the reference stores them
        // between the kernels.
        const float4 uf = *reinterpret_cast<const float4*>(tile + tk * C::TILE_PITCH + 128 + lane * 4);
        const float up[4] = {uf.x, uf.y, uf.z, uf.w};
        const bool last = ((int)blockIdx.x == args.gu_rows / 128 - 1);          // the INT8 keeper group of the down projection
        uint32_t ua = 0;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float g = __half2float(__float2half_rn(v[e] * kInv)), u = __half2float(__float2half_rn(up[e] * kInv));
          v[e] = silu_ref(g) * u;
          ua = max(ua, __float_as_uint(fabsf(v[e])));            // |t| >= 0: IEEE bit patterns order like unsigned integers
        }
        ua = __reduce_max_sync(0xffffffffu, ua);
        float maxv = __uint_as_float(ua);
        maxv = maxv / (last ? 127.f : 7.f);                      // IEEE division, as `maxv /= 7`
        const float r_scale = 1.f / maxv;
        int qv[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int tq = (int)roundf(v[e] * r_scale);            // round half away from zero (CUDA round())
          qv[e] = last ? max(-128, min(127, tq)) : max(-8, min(7, tq));
        }
        if (last) {
          *reinterpret_cast<uint32_t*>(args.q8_out + (size_t)m * 128 + lane * 4) =
              (uint32_t)(qv[0] & 0xFF) | ((uint32_t)(qv[1] & 0xFF) << 8) | ((uint32_t)(qv[2] & 0xFF) << 16) | ((uint32_t)(qv[3] & 0xFF) << 24);
        } else {
          const size_t q4_pitch = (size_t)(args.gu_rows - 128) / 2;
          *reinterpret_cast<uint16_t*>(args.q4_out + (size_t)m * q4_pitch + (size_t)blockIdx.x * 64 + lane * 2) =
              (uint16_t)((qv[0] & 0xF) | ((qv[1] & 0xF) << 4) | ((qv[2] & 0xF) << 8) | ((qv[3] & 0xF) << 12));
        }
        if (lane == 0) {
          const __half hs = __float2half_rn(maxv);
          __half* dst = last ? args.q8_scale : args.q4_scale + (size_t)blockIdx.x * args.lda_scale;
          const int si = scale_index(m);
#pragma unroll
          for (int j = 0; j < 4; ++j) dst[si + 2 * j] = hs;     // replicated x4 (ldmatrix layout of the reference GEMM)
        }
      } else if (o16) {
        __half2 h0 = __floats2half2_rn(v[0] * kInv, v[1] * kInv), h1 = __floats2half2_rn(v[2] * kInv, v[3] * kInv);
        if constexpr (kE == EPI_PUSH) {
          // fused all-reduce, push half: the row goes to slot [call % 3][rank] of EVERY rank's receive buffer (-0.0, the
          // buffers' "not yet arrived" pattern, travels as +0.0) as 16-byte stores of 8 consecutive channels: 2-byte stores
          // over NVLink cost an order of magnitude more per byte.  The following add+RMSNorm kernel polls and sums the slots.
          uint32_t w0 = ar_strip_sentinel(*reinterpret_cast<uint32_t*>(&h0)), w1 = ar_strip_sentinel(*reinterpret_cast<uint32_t*>(&h1));
          const uint32_t w2 = __shfl_down_sync(0xffffffffu, w0, 1), w3 = __shfl_down_sync(0xffffffffu, w1, 1);
          if ((lane & 1) == 0 && n0 + lane * 4 < args.N) {
            const uint32_t cur = (ar_ld_state(args.ar.state) + 1) % 3;
            const size_t off = ((size_t)cur * args.ar.world + args.ar.rank) * (size_t)args.ar.slot + (size_t)m * args.N + n_out;
#pragma unroll 1
            for (int r = 0; r < args.ar.world; ++r) {
              int peer = args.ar.rank + r;
              if (peer >= args.ar.world) peer -= args.ar.world;
              ar_st_v4(reinterpret_cast<__half*>(args.ar.bufs[peer]) + off, make_uint4(w0, w1, w2, w3));
            }
          }
        } else if (n0 + lane * 4 < args.N) {   // N is a multiple of 8
          *reinterpret_cast<uint2*>(args.d + (size_t)m * n_out_dim + n_out) =
              make_uint2(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1));
        }
      } else {
        // o4 (DenseLayerGEMM_i4_o4.cu:705-787): per (token, 128-channel head) asymmetric INT4 with the reference's |v| min/max
        uint8_t* d4 = (kE == EPI_QKV && seg == 2) ? args.d4_v : args.d4;
        __half2* d_scale = (kE == EPI_QKV && seg == 2) ? args.d_scale_v : args.d_scale;
        uint32_t umx = 0u, umn = 0x7f800000u;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          v[e] *= kInv;
          const uint32_t ua = __float_as_uint(fabsf(v[e]));      // |v| >= 0: IEEE bit patterns order like unsigned integers
          umx = max(umx, ua); umn = min(umn, ua);
        }
        const float mx = __uint_as_float(__reduce_max_sync(0xffffffffu, umx)), mn = __uint_as_float(__reduce_min_sync(0xffffffffu, umn));
        const float scale = (mx - mn) / 15.f, zero = -mn, r_scale = 1.f / scale;
        uint32_t pk = 0;
#pragma unroll
        for (int e = 0; e < 4; ++e) pk |= ((uint32_t)((int)roundf((v[e] + zero) * r_scale) & 0xF)) << (4 * e);
        *reinterpret_cast<uint16_t*>(d4 + (size_t)m * (n_out_dim / 2) + n_out / 2) = (uint16_t)pk;
        if (lane == 0) d_scale[(size_t)m * (n_out_dim / 128) + otile] = __floats2half2_rn(scale, zero);
      }
    }
    // split-K: no CTA of the cluster leaves while its tile may still be read
    if constexpr (kSplit > 1) { cluster_arrive(); cluster_wait(); }
  }
  if (threadIdx.x == 0) trace_stamp(args, 4);
}

}  // namespace atom
