// gemm_i4_sm90.cuh -- W4A4 group-quantised GEMM with INT8 keeper for H100 (sm_90a).
//
// Replaces the reference's compute_gemm_imma / DenseLayerGEMM_i4[_o4]_kernel (kernels/include/GEMM/Dense_layer_gemm_i4_o16.cuh,
// e2e/punica-atom/punica/ops/csrc/GEMM/DenseLayerGEMM_i4_o4.cu).  Same operands, same layouts, same arithmetic (exact INT32
// group sums, one FP16 multiply of the two scales, FP32 fma accumulation in group order, keeper last, RN cast to half) --
// different machine.  Hopper's warpgroup MMA has no INT4 type, so both operands are widened to INT8 (value * 16: a shift and
// a mask, no sign extension) on their way to the tensor cores:
//
//   TMA: packed INT4 tiles (64 B rows) of the weights (128 channels) and of the tokens (BN rows) -> smem "packed ring"
//   producer warpgroup: one thread issues the TMA loads; three warps widen the TOKEN tile into the K-major SWIZZLE_128B
//       INT8 operand ("expanded ring"), the fourth loads the groups' scales a few groups ahead and stages them next to it
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
  // EPI_RESIDENT: the packed INT4 tokens [M][G * 64] and the INT8 keeper tokens [M][128] (tm_a4 / tm_a8), read with L2 loads
  const uint8_t* a4;
  const uint8_t* a8;
};

// timeline stamps for pipeline debugging (tools/gemm_phase_trace.py), 128 clock64 slots per CTA:
//   0 start | 1 setup done | 2 keeper done (end of the consumers' main loop) | 3 every rank's tile staged | 4 end (thread 0)
//   5 producer past griddepcontrol.wait | 6 split-K reduction + output stores done | 7 consumers leave
// Stamps 2, 3, 6 and 7 come from consumer warp 0, the others from thread 0 (the same SM clock).
// Built with -DATOM_GEMM_TRACE_GROUPS, INT4 group s < TRACE_GROUPS also stamps slot 8 + kind * TRACE_GROUPS + s:
//   producer thread 0:  0 pack_full passed | 3 exp_full (token tile widened)
//   scale warp, lane 0: 1 scale slot free (exp_empty) | 2 scales stored (their loads returned)
//   consumer warp 0:    4 pack_full passed | 5 exp_full passed | 6 group dequantised
// The resident variant (EPI_RESIDENT) stamps 3 once the producers have received everything (group 0's slot), 5 once the
// consumers have (group 0's slot), 4 and 6 per group, and slot 3 of the launch stamps past the cluster barrier before its push.
// A compile-time switch: even untaken, a runtime branch in the per-group loops costs the 16-token split-K launch about
// 0.6 us (H100 80GB HBM3, 700 W).
#ifdef ATOM_GEMM_TRACE_GROUPS
constexpr bool kTraceGroups = true;
#else
constexpr bool kTraceGroups = false;
#endif
constexpr int TRACE_GROUPS = 16;
__device__ __forceinline__ void trace_stamp(const GemmArgs& a, int slot) {
  if (a.trace != nullptr) {
    const int cta = (blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    a.trace[(size_t)cta * 128 + slot] = (unsigned long long)clock64();
  }
}

__device__ __forceinline__ void trace_group(const GemmArgs& a, int kind, int s) {
  if constexpr (kTraceGroups) {
    if (s < TRACE_GROUPS) trace_stamp(a, 8 + kind * TRACE_GROUPS + s);
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
// EPI_RESIDENT: a mode bit or-ed into EPI_O16 / EPI_PUSH for 16-token tiles split over K whose every rank holds at most PACK
// INT4 groups.  The rank's whole K slice then stays in shared memory, one slot per group: the static operands (weights and
// weight scales) are all requested before griddepcontrol.wait, the dynamic ones (token tiles and token scales) in one burst
// after it, the producers widen every token tile and arrive once, and the consumers run the groups with no ring handshakes.
// The split-K partials are pushed to the rank that stores them (st.async) instead of being staged and read remotely.
enum { EPI_O16 = 0, EPI_O4 = 1, EPI_QKV = 2, EPI_GATEUP = 3, EPI_PUSH = 4, EPI_GROUPED = 8, EPI_RESIDENT = 16 };

template <int BN, int kSplit, int kEpi>
struct GemmCfg {
  static constexpr int EPI = kEpi & ~(EPI_GROUPED | EPI_RESIDENT);   // the epilogue
  static constexpr bool RESIDENT = (kEpi & EPI_RESIDENT) != 0;
  static constexpr int ROWS = EPI == EPI_GATEUP ? 256 : 128;    // weight rows per CTA
  static constexpr int MT = ROWS / 128;                          // 64-row wgmma tiles per consumer warpgroup
  static constexpr int THREADS = 384;                            // producer warpgroup + two consumer warpgroups
  static constexpr int PACK = BN <= 32 ? 8 : 4;                  // packed ring depth (groups): decode shapes are a weight stream
  // expanded token tiles / scale slots; resident: one per packed slot
  static constexpr int EXP = RESIDENT ? PACK : (BN <= 64 ? 4 : 3);
  // Decode tiles (BN <= 32) load the scales in a producer warp of their own (SCALE_WARP), SCALE_AHEAD groups ahead, and
  // widen the token tile with the other three; larger tiles need all four warps to widen and load the scales in line.
  // The resident variant loads all its scales up front and widens with all four warps.
  static constexpr bool SCALE_WARP_ON = BN <= 32 && !RESIDENT;
  static constexpr int SCALE_WARP = 3;
  static constexpr int SCALE_AHEAD = 4;                          // groups whose scale loads the scale warp keeps in flight
  static constexpr int SCALE_THREADS = SCALE_WARP_ON ? 32 : 128;  // threads that load and store a group's scales
  static constexpr int WIDEN_THREADS = SCALE_WARP_ON ? 96 : 128;  // threads that widen the token tile
  static constexpr int TOK_PER_THREAD = (BN + SCALE_THREADS - 1) / SCALE_THREADS;
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
  static constexpr int NUM_BARS = 2 * PACK + 2 * EXP + 1 + (RESIDENT ? 1 : 0);   // resident: + the split-K receive barrier
  static constexpr int SMEM_BYTES = OFF_BAR + NUM_BARS * 8 + 1024;   // + slack for the 1024-B alignment fix-up
  static constexpr int TILE_PITCH = ROWS + 4;                    // floats per token row of the staged output tile
  static constexpr int KEEP_TX = ROWS * 128 + BN * 128;
  // resident: rank r receives row tk (tk % kSplit == r) of rank k's FP32 partial tile in slot [k][tk / kSplit] of ROWS floats,
  // over the packed token slots, which this variant does not use (its token tiles are loaded into registers)
  static constexpr int RECV_TX = BN * ROWS * 4;
  static_assert(BN == 16 || BN == 32 || BN == 64 || BN == 128, "token tile");
  static_assert(BN * TILE_PITCH * 4 <= OFF_SCALE, "the output tile is staged over the idle operand rings");
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget");
  static_assert(kSplit == 1 || EPI == EPI_O16 || EPI == EPI_PUSH, "the quantising epilogues work on un-split FP32 sums");
  static_assert(!(kEpi & EPI_GROUPED) || (kSplit == 1 && BN <= 64), "grouped mode: token tiles of 16 / 32 / 64, no K split");
  static_assert(!RESIDENT || (BN == 16 && kSplit > 1 && !(kEpi & EPI_GROUPED)), "resident: split 16-token tiles, not grouped");
  static_assert(!RESIDENT || RECV_TX <= PACK * PACK_Q, "resident: the receive slots fit over the packed token tiles");
  // the next launch's CTA prefetches its weights beside this one: two CTAs per SM (228 KB, 1 KB reserved per CTA)
  static_assert(!RESIDENT || 2 * (SMEM_BYTES + 1024) <= 228 * 1024, "resident: two CTAs per SM");
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
  constexpr int kE = C::EPI;
  constexpr int NR = BN / 2;                                // accumulator registers per 64-row tile
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-B alignment (SWIZZLE_128B atoms) by offsetting the shared array, NOT by integer-casting the pointer:
  // an integer round trip makes the compiler fall back to generic LD/ST for every smem access.
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);

  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::OFF_BAR);
  uint64_t* pack_full = bars;                          // TMA landed the group's packed tiles            (1 + tx)
  uint64_t* pack_empty = pack_full + C::PACK;          // every warp has read them  (the widening + the 8 consumer warps)
  uint64_t* exp_full = pack_empty + C::PACK;           // token operand + scales of the group in place   (4 producer warps)
  uint64_t* exp_empty = exp_full + C::EXP;             // consumers are done with them                   (8 consumer warps)
  uint64_t* keep_full = exp_empty + C::EXP;            // keeper tiles + scales landed     (1 + tx, the scale-loading warps)
  // resident: exp_full[0] = every token tile widened and every scale stored (4 producer warps); keep_full = keeper weights
  // landed (1 + tx); recv_bar = every rank's partials of this rank's token rows landed (1 + RECV_TX, st.async)
  uint64_t* recv_bar = keep_full + 1;

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
    for (int i = 0; i < C::PACK; ++i) { mbar_init(&pack_full[i], 1); mbar_init(&pack_empty[i], C::SCALE_WARP_ON ? 11 : 12); }
    for (int i = 0; i < C::EXP; ++i) { mbar_init(&exp_full[i], 4); mbar_init(&exp_empty[i], 8); }
    mbar_init(keep_full, C::RESIDENT ? 1 : (C::SCALE_WARP_ON ? 2 : 5));
    if constexpr (C::RESIDENT) mbar_init(recv_bar, 1);
    fence_barrier_init();
    if constexpr (C::RESIDENT) mbar_arrive_expect_tx(recv_bar, C::RECV_TX);   // armed before the cluster barrier below
  }
  __syncthreads();
  // split-K: a CTA's shared memory may only be read remotely while that CTA is alive -- every thread arrives here (cheap,
  // non-blocking) and waits before the reduction (resident: before its first remote write)
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
    griddep_launch_dependents();
    if constexpr (C::RESIDENT) {
      // ---------------------------------------------------------- resident slice: slot s = INT4 group g_begin + s, the
      // keeper's scales in slot PACK.  PDL contract: the weight tiles, the keeper weights and the weight scales are static
      // operands of the layer and are read before griddepcontrol.wait; the token tiles and token scales come after it.
      if (t == 0) {
        for (int s = 0; s < n4; ++s) {
          mbar_arrive_expect_tx(&pack_full[s], C::PACK_W);
          tma_load_2d(smem + C::OFF_PACK_W + s * C::PACK_W, &tm_w4, &pack_full[s], (g_begin + s) * 64, n0);
        }
        if (has_keeper) {
          mbar_arrive_expect_tx(keep_full, C::ROWS * 128);
          tma_load_2d(smem + C::OFF_KEEP_W, &tm_w8, keep_full, 0, n0);
        }
      }
      // chunk c of the scales: slot c / 16, weight-scale chunk (8 channels) and token c % 16
      constexpr int CHUNKS = (C::PACK + 1) * 16, PER_T = (CHUNKS + 127) / 128;
      uint4 wsc[PER_T];
      __half asc[PER_T];
#pragma unroll
      for (int i = 0; i < PER_T; ++i) {
        const int c = t + 128 * i, s = c >> 4, col = c & 15;
        wsc[i] = make_uint4(0, 0, 0, 0);
        if (c < CHUNKS && (s < n4 || (s == C::PACK && has_keeper)) && n0 + 8 * col < args.N)
          wsc[i] = ld_cg_v4((s == C::PACK ? args.b_keeper_scale : args.b_scale + (size_t)(g_begin + s) * args.ldb_scale) + n0 + 8 * col);
      }
      griddep_wait();                       // from here on the preceding kernel's output (the activations) may be read
      if (t == 0) trace_stamp(args, 5);
      // Every dynamic input in one burst of L2 loads, all in flight together.  The token tiles do not take the TMA queue:
      // there they wait behind the weight requests of the next launch's CTA on this SM and land one by one.
      // Thread t: 16-B chunk t % 64 (token row r, quarter qq) of the packed tiles of groups s = t / 64 + 2i, and 16-B chunk
      // t of the keeper's INT8 token tile (row t / 8).  Rows past M read as zero, as the TMA box would.
      const int r = (t & 63) >> 2, qq = t & 3, rk = t >> 3, ck = t & 7;
      const size_t pitch4 = (size_t)args.G * 64;
      uint4 tok[C::PACK / 2], ktok = make_uint4(0, 0, 0, 0);
#pragma unroll
      for (int i = 0; i < C::PACK / 2; ++i) {
        const int s = (t >> 6) + 2 * i;
        tok[i] = make_uint4(0, 0, 0, 0);
        if (s < n4 && m0 + r < args.M) tok[i] = ld_cg_v4(args.a4 + (size_t)(m0 + r) * pitch4 + (size_t)(g_begin + s) * 64 + qq * 16);
      }
      if (has_keeper && m0 + rk < args.M) ktok = ld_cg_v4(args.a8 + (size_t)(m0 + rk) * 128 + ck * 16);
#pragma unroll
      for (int i = 0; i < PER_T; ++i) {
        const int c = t + 128 * i, s = c >> 4, tk = c & 15;
        asc[i] = __ushort_as_half(0);
        if (c < CHUNKS && (s < n4 || (s == C::PACK && has_keeper)) && m0 + tk < args.M)
          asc[i] = __ushort_as_half(ld_cg_u16((s == C::PACK ? args.a_keeper_scale : args.a_scale + (size_t)(g_begin + s) * args.lda_scale) +
                                              scale_index(m0 + tk)));
      }
      // widen into the SWIZZLE_128B INT8 operands, as the ring's widening does; the keeper tile as its TMA box would land
#pragma unroll
      for (int i = 0; i < C::PACK / 2; ++i) {
        const int s = (t >> 6) + 2 * i;
        if (s < n4) {
          const uint32_t ww[4] = {tok[i].x, tok[i].y, tok[i].z, tok[i].w};
          uint8_t* row = smem + C::OFF_EXP + s * C::EXP_Q + (r >> 3) * 1024 + (r & 7) * 128 + 4 * qq;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            *reinterpret_cast<uint32_t*>(row + (((2 * j) ^ (r & 7)) << 4)) = (ww[j] << 4) & 0xF0F0F0F0u;
            *reinterpret_cast<uint32_t*>(row + (((2 * j + 1) ^ (r & 7)) << 4)) = ww[j] & 0xF0F0F0F0u;
          }
        }
      }
      if (has_keeper) *reinterpret_cast<uint4*>(smem + C::OFF_KEEP_Q + (rk >> 3) * 1024 + (rk & 7) * 128 + ((ck ^ (rk & 7)) << 4)) = ktok;
#pragma unroll
      for (int i = 0; i < PER_T; ++i) {
        const int c = t + 128 * i, s = c >> 4, col = c & 15;
        if (c < CHUNKS && (s < n4 || (s == C::PACK && has_keeper))) {
          uint8_t* slot = smem + C::OFF_SCALE + s * C::SCALE_BYTES;
          reinterpret_cast<uint4*>(slot)[col] = wsc[i];
          reinterpret_cast<__half*>(slot + C::ROWS * 2)[col] = asc[i];
        }
      }
      // the weight tiles landed long ago; observing them here lets the consumers' single wait below cover them
      for (int s = 0; s < n4; ++s) mbar_wait(&pack_full[s], 0);
      fence_proxy_async_smem();             // generic-proxy stores -> visible to the wgmma operand fetch
      __syncwarp();
      if (lane == 0) mbar_arrive(&exp_full[0]);
      if (t == 0) trace_group(args, 3, 0);
      if constexpr (kSplit > 1) cluster_wait();
      if (t == 0) trace_stamp(args, 4);
      return;
    }
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
      trace_stamp(args, 5);
      for (int s = 0; s < first; ++s) issue_stage(s, 2);
      if (has_keeper) tma_load_2d(smem + C::OFF_KEEP_Q, &tm_a8, keep_full, 0, m0);
    } else {
      griddep_wait();
    }
    // a group's scales: weight scales of the tile's channels (16-B chunks), token scales in token order, loaded by
    // SCALE_THREADS threads (index si)
    struct Scales { uint4 b; __half a[C::TOK_PER_THREAD]; };
    const int si = C::SCALE_WARP_ON ? lane : t;
    const int m_end = kGrouped ? gtile.y + gtile.z : args.M;
    auto load_scales = [&](const __half* bs_row, const __half* as_row, Scales& sc) {
      sc.b = make_uint4(0, 0, 0, 0);
      if (si < C::ROWS / 8) {
        const int seg = si / 16, c = si % 16;                         // gate/up: segment 1 = the up rows
        if (n0 + 8 * c < n_limit) sc.b = ld_cg_v4(bs_row + (size_t)seg * args.gu_rows + n0 + 8 * c);
      }
#pragma unroll
      for (int i = 0; i < C::TOK_PER_THREAD; ++i) {
        const int tk = si + C::SCALE_THREADS * i;
        sc.a[i] = __ushort_as_half(0);
        if (tk < BN && m0 + tk < m_end) sc.a[i] = __ushort_as_half(ld_cg_u16(as_row + scale_index(m0 + tk)));
      }
    };
    auto load_group = [&](int s, Scales& sc) {
      const int g = g_begin + s;
      load_scales((kGrouped ? args.b_scale + (size_t)gtile.x * args.G * args.ldb_scale : args.b_scale) + (size_t)g * args.ldb_scale,
                  args.a_scale + (size_t)g * args.lda_scale, sc);
    };
    auto store_scales = [&](int slot_idx, const Scales& sc) {
      uint8_t* slot = smem + C::OFF_SCALE + slot_idx * C::SCALE_BYTES;
      if (si < C::ROWS / 8) reinterpret_cast<uint4*>(slot)[si] = sc.b;
#pragma unroll
      for (int i = 0; i < C::TOK_PER_THREAD; ++i)
        if (si + C::SCALE_THREADS * i < BN) reinterpret_cast<__half*>(slot + C::ROWS * 2)[si + C::SCALE_THREADS * i] = sc.a[i];
    };
    auto load_keeper = [&](Scales& sc) {
      load_scales(kGrouped ? args.b_keeper_scale + (size_t)gtile.x * args.expert_rows : args.b_keeper_scale, args.a_keeper_scale, sc);
    };
    if (C::SCALE_WARP_ON && warp == C::SCALE_WARP) {
      // ---------------------------------------------------------- scale warp: the per-group weight and token scales
      // Global loads, each an HBM round trip that the next launch's weight prefetch makes long.  Loaded in line by the
      // widening warps, which fence the async proxy once per group, they cost one round trip per group; this warp never
      // fences and keeps SCALE_AHEAD groups of them in flight.
      Scales keep, ahead[C::SCALE_AHEAD];
      if (has_keeper) load_keeper(keep);
#pragma unroll
      for (int u = 0; u < C::SCALE_AHEAD; ++u)
        if (u < n4) load_group(u, ahead[u]);
      if (has_keeper) {
        store_scales(C::EXP, keep);
        __syncwarp();
        if (lane == 0) mbar_arrive(keep_full);
      }
      // unrolled by SCALE_AHEAD so that every register set keeps a fixed place
      for (int s0 = 0; s0 < n4; s0 += C::SCALE_AHEAD) {
#pragma unroll
        for (int u = 0; u < C::SCALE_AHEAD; ++u) {
          const int s = s0 + u, es = s % C::EXP;
          if (s < n4) {
            if (s >= C::EXP) mbar_wait(&exp_empty[es], ((s / C::EXP) - 1) & 1);
            if (lane == 0) trace_group(args, 1, s);
            store_scales(es, ahead[u]);
            if (lane == 0) trace_group(args, 2, s);
            __syncwarp();
            if (lane == 0) mbar_arrive(&exp_full[es]);
            if (s + C::SCALE_AHEAD < n4) load_group(s + C::SCALE_AHEAD, ahead[u]);
          }
        }
      }
    } else {
      // ---------------------------------------------------------- widening warps: the token tile into the INT8 operand
      Scales cur;                            // larger tiles: the group's scales, loaded in line
      if (!C::SCALE_WARP_ON && has_keeper) {
        load_keeper(cur);
        store_scales(C::EXP, cur);
        __syncwarp();
        if (lane == 0) mbar_arrive(keep_full);
      }
      for (int s = 0; s < n4; ++s) {
        const int ps = s % C::PACK, es = s % C::EXP;
        if constexpr (!C::SCALE_WARP_ON) load_group(s, cur);
        if (t == 0 && s >= 1 && s + C::PACK - 1 < n4) {               // refill the slot the previous group has left
          const int nx = s + C::PACK - 1;
          mbar_wait(&pack_empty[nx % C::PACK], ((nx / C::PACK) - 1) & 1);
          issue_stage(nx, 0);
        }
        mbar_wait(&pack_full[ps], (s / C::PACK) & 1);
        if (t == 0) trace_group(args, 0, s);
        if (s >= C::EXP) mbar_wait(&exp_empty[es], ((s / C::EXP) - 1) & 1);
        const uint8_t* packed = smem + C::OFF_PACK_Q + ps * C::PACK_Q;
        uint8_t* expanded = smem + C::OFF_EXP + es * C::EXP_Q;
#pragma unroll
        for (int c = t; c < BN * 4; c += C::WIDEN_THREADS) {
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
        if constexpr (!C::SCALE_WARP_ON) store_scales(es, cur);
        fence_proxy_async_smem();             // generic-proxy stores -> visible to the wgmma operand fetch
        __syncwarp();
        if (lane == 0) { mbar_arrive(&pack_empty[ps]); mbar_arrive(&exp_full[es]); }
        if (t == 0) trace_group(args, 3, s);
      }
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

    if constexpr (C::RESIDENT) {
      // the producers passed every group's pack_full before they arrived: the weight tiles are in place too
      mbar_wait(&exp_full[0], 0);
      if (cw == 0 && lane == 0) trace_group(args, 5, 0);
    }
    for (int s = 0; s < n4; ++s) {
      const int ps = s % C::PACK, es = s % C::EXP;
      if constexpr (!C::RESIDENT) mbar_wait(&pack_full[ps], (s / C::PACK) & 1);
      if (cw == 0 && lane == 0) trace_group(args, 4, s);
      uint4 wa[C::MT], wb[C::MT];
#pragma unroll
      for (int t = 0; t < C::MT; ++t) {
        const uint8_t* p = smem + C::OFF_PACK_W + ps * C::PACK_W + ((wg * C::MT + t) * 64 + wq * 16 + g8) * 64 + q * 16;
        wa[t] = *reinterpret_cast<const uint4*>(p);
        wb[t] = *reinterpret_cast<const uint4*>(p + 8 * 64);
      }
      if constexpr (!C::RESIDENT) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&pack_empty[ps]);
        mbar_wait(&exp_full[es], (s / C::EXP) & 1);
        if (cw == 0 && lane == 0) trace_group(args, 5, s);
      }
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
      if constexpr (!C::RESIDENT) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&exp_empty[es]);
      }
      if (cw == 0 && lane == 0) trace_group(args, 6, s);
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

    float* tile = reinterpret_cast<float*>(smem);
    // resident receive slots: [rank][row tk / kSplit][ROWS floats], channel c at (c & ~15) + 2 (c & 7) + ((c >> 3) & 1), so
    // that a thread's channel pair (ch, ch + 8) is one 8-byte push
    const float* recv = reinterpret_cast<const float*>(smem + C::OFF_PACK_Q);
    if constexpr (C::RESIDENT) {
      // ------------------------------------------------------------ push row tk of the partial tile to rank tk % kSplit
      cluster_wait();                                  // every rank has initialised and armed its recv_bar
      if (cw == 0 && lane == 0) trace_stamp(args, 3);
      const uint32_t rbase = smem_u32(recv), rbar = smem_u32(recv_bar);
#pragma unroll
      for (int t = 0; t < C::MT; ++t) {
        const int ch = (wg * C::MT + t) * 64 + wq * 16 + g8;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int tk = 8 * j + 2 * q + e, dst = tk % kSplit;
            const uint32_t at = rbase + (((int)krank * (BN / kSplit) + tk / kSplit) * C::ROWS + ch + g8) * 4;
            st_async_v2(mapa_shared(at, dst), acc[t][4 * j + e], acc[t][4 * j + 2 + e], mapa_shared(rbar, dst));
          }
      }
      // Every consumer warp waits, so that the CTA stays alive until the last push into it has landed.  The st.async
      // write and its complete-tx on this mbarrier are one operation (PTX ISA, st.async), so once the phase completes no
      // other CTA touches this CTA's shared memory again, and the senders read registers only: no cluster barrier
      // before exit is needed (a CTA's shared memory may be accessed remotely only while that CTA is running).
      mbar_wait<true>(recv_bar, 0);
    } else {
      // ------------------------------------------------------------ stage the FP32 tile as [token][channel]
      asm volatile("bar.sync 1, 256;" ::: "memory");     // both consumer warpgroups have left the operand rings
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
    }

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
      if constexpr (C::RESIDENT) {
        // channels 4 lane .. 4 lane + 3 of every rank's slot, summed in rank order as below
        const float* r0 = recv + (tk / kSplit) * C::ROWS + 16 * (lane >> 2) + 8 * (lane & 1) + ((lane >> 1) & 1);
#pragma unroll
        for (int e = 0; e < 4; ++e) v[e] = r0[2 * e];
#pragma unroll
        for (int rk = 1; rk < kSplit; ++rk)
#pragma unroll
          for (int e = 0; e < 4; ++e) v[e] += r0[rk * (BN / kSplit) * C::ROWS + 2 * e];
      } else {
        const float4 f = *reinterpret_cast<const float4*>(tile + tk * C::TILE_PITCH + lane * 4);
        v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
      }
      if constexpr (kSplit > 1 && !C::RESIDENT) {
        // every remote rank's 4 channels in one 16-B load, all in flight together (one at a time, the remote-load latency
        // stacked up 4 (kSplit - 1) deep per token row), then the rank-order sums
        const uint32_t local = smem_u32(tile + tk * C::TILE_PITCH + lane * 4);
        float4 p[kSplit];
#pragma unroll
        for (int rk = 0; rk < kSplit; ++rk) p[rk] = rk == (int)krank ? make_float4(v[0], v[1], v[2], v[3]) : ld_dsmem_v4(mapa_shared(local, rk));
        v[0] = p[0].x; v[1] = p[0].y; v[2] = p[0].z; v[3] = p[0].w;
#pragma unroll
        for (int rk = 1; rk < kSplit; ++rk) { v[0] += p[rk].x; v[1] += p[rk].y; v[2] += p[rk].z; v[3] += p[rk].w; }
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
        // o4: per (token, 128-channel head) asymmetric INT4, x = nibble * scale - zero, over the SIGNED min and max of the head.
        // (The reference kernel, DenseLayerGEMM_i4_o4.cu:705-787, takes them over |v|, so every v below min|v| -- nearly every
        // negative value -- gets a negative code that its `& 0xF` wraps to a large nibble.)  redux.sync orders integers: the key
        // v >= +0 -> bits | 2^31, v <= -0 -> ~bits orders IEEE floats like unsigned integers, -0 below +0, so the two
        // reductions stay one redux each (fmaxf/fminf shuffles would take five rounds each).  The key order is also the tie
        // rule: a head whose minimum is both -0 and +0 stores zero = +0, one of +0 alone zero = -0, as the oracle does.
        uint8_t* d4 = (kE == EPI_QKV && seg == 2) ? args.d4_v : args.d4;
        __half2* d_scale = (kE == EPI_QKV && seg == 2) ? args.d_scale_v : args.d_scale;
        uint32_t kmx = 0u, kmn = 0xffffffffu;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          v[e] *= kInv;
          const uint32_t b = __float_as_uint(v[e]), key = b ^ ((uint32_t)((int32_t)b >> 31) | 0x80000000u);
          kmx = max(kmx, key); kmn = min(kmn, key);
        }
        kmx = __reduce_max_sync(0xffffffffu, kmx); kmn = __reduce_min_sync(0xffffffffu, kmn);
        const float mx = __uint_as_float(kmx ^ ((uint32_t)((int32_t)~kmx >> 31) | 0x80000000u));
        const float mn = __uint_as_float(kmn ^ ((uint32_t)((int32_t)~kmn >> 31) | 0x80000000u));
        // a constant head: scale +0, 0 * inf = NaN converts to code 0
        const float scale = (mx - mn) / 15.f, zero = -mn, r_scale = 1.f / scale;
        uint32_t pk = 0;
#pragma unroll
        for (int e = 0; e < 4; ++e) pk |= (uint32_t)min(15, max(0, (int)roundf((v[e] + zero) * r_scale))) << (4 * e);
        *reinterpret_cast<uint16_t*>(d4 + (size_t)m * (n_out_dim / 2) + n_out / 2) = (uint16_t)pk;
        if (lane == 0) d_scale[(size_t)m * (n_out_dim / 128) + otile] = __floats2half2_rn(scale, zero);
      }
    }
    if (cw == 0 && lane == 0) trace_stamp(args, 6);
    // split-K: no CTA of the cluster leaves while its tile may still be read (resident: nothing is read remotely)
    if constexpr (kSplit > 1 && !C::RESIDENT) { cluster_arrive(); cluster_wait(); }
    if (cw == 0 && lane == 0) trace_stamp(args, 7);
  }
  if (threadIdx.x == 0) trace_stamp(args, 4);
}

}  // namespace atom
