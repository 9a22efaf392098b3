/*
 * atom_b200.h -- C ABI of libatom_b200.so: the H100 (sm_90a) implementation of the efeslab/Atom W4A4 hot path.
 *
 * One entry point per function that the reference binds into Python through
 * pybind11 (e2e/punica-atom/punica/ops/csrc/punica_ops.cc:270-279 of the reference).  Plain pointers and sizes only;
 * every pointer is a DEVICE pointer owned by the caller, outputs are pre-allocated by the caller (exactly as
 * punica/ops/__init__.py:21-219 does with torch.empty) and the library keeps no reference to them.
 *
 * Conventions
 *   - return value: 0 on success, negative ATOM_E_* otherwise; atom_last_error() returns a thread-local message.
 *     (The reference returns void and never checks cudaGetLastError; its KV ops raise via TORCH_CHECK.)
 *   - `stream` is a cudaStream_t passed as void*.  The reference launches on the legacy default stream; pass the
 *     caller's current stream (NULL = legacy default).  All entry points are asynchronous and graph-capturable
 *     (no allocation, no synchronisation; TMA descriptors are built on the host per call).
 *   - layouts are the reference's, unchanged (see DESIGN.md section 3).
 */
#ifndef ATOM_B200_H_
#define ATOM_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define ATOM_API __attribute__((visibility("default")))
#else
#define ATOM_API
#endif

#define ATOM_OK 0
#define ATOM_E_INVALID (-1) /* bad shape / alignment / null pointer */
#define ATOM_E_CUDA (-2)    /* a CUDA runtime or driver call failed  */
#define ATOM_E_UNSUPPORTED (-3)

/* gemm flags */
#define ATOM_GEMM_AUTO 0u
#define ATOM_GEMM_NO_SPLITK 1u   /* bit-exact accumulation order (groups 0..G-1 then keeper) even for small M */
#define ATOM_GEMM_FORCE_TALL 2u  /* 128-token tiles regardless of M; never splits K */
#define ATOM_GEMM_FORCE_SKINNY 4u /* token tiles of at most 64 regardless of M */
#define ATOM_GEMM_SPLITK2 16u     /* decode shapes: force a 2-way K split (default: chosen from the tile count) */
#define ATOM_GEMM_SPLITK4 32u     /* decode shapes: force a 4-way K split */
#define ATOM_GEMM_SPLITK8 64u     /* force an 8-way K split (cluster of 8) */
/* kernel selectors of earlier versions: accepted for callers that pass them, ignored (there is one GEMM kernel) */
#define ATOM_GEMM_FORCE_WIDE 512u
#define ATOM_GEMM_NO_WIDE 1024u
#define ATOM_GEMM_LEGACY_TALL 256u
#define ATOM_GEMM_LEGACY_SKINNY 128u

ATOM_API int atom_version(void);
ATOM_API const char* atom_last_error(void);

/* Reorder.cuh:39-50 / punica/ops/__init__.py:137 -- the scale layout contract shared by quantise kernels and GEMM */
ATOM_API int atom_scale_index(int row);
ATOM_API int atom_scale_size(int rows);

/* replaces reorder_fp16_i4 (punica_ops.cc:251-260 -> run_reorder_fp16_i4<128,4096>, Reorder.cuh:205-228)
 *   hidden        f16 [seq_len, hidden_dim]      reorder_index i16 [hidden_dim]
 *   o_outliers    i8  [seq_len, 128]             o_norms       u8  [seq_len, (hidden_dim-128)/2]
 *   outlier_scales f16 [scale_size(seq_len)]     norm_scales   f16 [hidden_dim/128-1, scale_size(seq_len)]
 * hidden_dim: any multiple of 128 (the reference is compiled for 4096 only). */
ATOM_API int atom_reorder_fp16_i4(const void* hidden, const void* reorder_index, int seq_len, int hidden_dim, void* o_outliers,
                         void* o_norms, void* outlier_scales, void* norm_scales, void* stream);

/* replaces rmsnorm_fp16_i4 (punica_ops.cc:239-249 -> run_rmsnorm_fp16_i4<128,4096>, RMSNorm.cuh:255-285) */
ATOM_API int atom_rmsnorm_fp16_i4(const void* hidden, const void* weight, float eps, const void* reorder_index, int seq_len,
                         int hidden_dim, void* o_outliers, void* o_norms, void* outlier_scales, void* norm_scales,
                         void* stream);

/* EXTENSION (launch-count reduction, SURVEY.md 8 f4): the residual add of the decoder layer
 * (punica/models/llama.py:266-292, `hidden = residual + hidden`) folded into the following rmsnorm_fp16_i4:
 * sum_out = hidden + residual (FP16 RN, bit-identical to the separate add), then exactly rmsnorm_fp16_i4(sum_out, ...). */
ATOM_API int atom_add_rmsnorm_fp16_i4(const void* hidden, const void* residual, void* sum_out, const void* weight, float eps,
                             const void* reorder_index, int seq_len, int hidden_dim, void* o_outliers, void* o_norms,
                             void* outlier_scales, void* norm_scales, void* stream);

/* replaces activate_fp16_i4 (punica_ops.cc:73-80 -> run_activate_fp16_i4<128,11008>, Activate.cuh:194-218) */
ATOM_API int atom_activate_fp16_i4(const void* a, const void* b, int seq_len, int hidden_dim, void* o_outliers, void* o_norms,
                          void* outlier_scales, void* norm_scales, void* stream);

/* replaces dense_layer_gemm_i4_fp16 (punica_ops.cc:226-237 -> DenseLayerGEMM_i4<nv_half>, DenseLayerGEMM_i4.cu:723-793)
 *   a u8 [M,(K-128)/2]  b u8 [N,(K-128)/2]  a_scale f16 [K/128-1, scale_size(M)]  b_scale f16 [K/128-1, N]
 *   a_keeper i8 [M,128] b_keeper i8 [N,128] a_keeper_scale f16 [scale_size(M)]    b_keeper_scale f16 [N]
 *   d f16 [M,N].   K includes the 128 keeper channels (as in the e2e launcher).  N % 8 == 0, K % 128 == 0, K >= 256.
 * Bit-identity: every path accumulates the groups in the reference's order (0..G-1, keeper last) and is bit-identical to the
 * reference kernel, EXCEPT when K is split over a cluster of s CTAs (flags = ATOM_GEMM_AUTO with M <= 128 when channel tiles
 * alone would not fill the GPU, or ATOM_GEMM_SPLITK2/4/8): rank r then owns groups [min(r*per, G+1), min(r*per+per, G+1)) of the
 * G+1 groups (keeper = group G, per = ceil((G+1)/s)), runs its own FP32 fma chain from +0 over them in order, and the partials
 * are added in rank order, ((p0 + p1) + p2) + ..., before the RN cast -- deterministic, but another association than the
 * reference's, so outputs may differ from it wherever rounding differs (mostly by an ulp; under heavy cancellation by more).
 * ATOM_GEMM_NO_SPLITK restores the reference's order at decode sizes.
 * The weights (b, b_scale, b_keeper, b_keeper_scale) are read before the preceding kernel on `stream` has completed
 * (programmatic dependent launch): they must not be written by the kernel launched immediately before this call. */
ATOM_API int atom_gemm_i4_o16(const void* a, const void* b, const void* a_scale, const void* b_scale, const void* a_keeper,
                     const void* b_keeper, const void* a_keeper_scale, const void* b_keeper_scale, void* d, int64_t M,
                     int64_t N, int64_t K, uint32_t flags, void* stream);

/* replaces dense_layer_gemm_i4_o4 (punica_ops.cc:211-224 -> DenseLayerGEMM_i4_o4, DenseLayerGEMM_i4_o4.cu:808-856)
 *   d u8 [M, N/2] (asymmetric INT4 per 128-column head), d_scale f16 [M, N/128, 2] = (scale, zero).  N % 128 == 0.
 *   x = nibble * scale - zero over the SIGNED min/max of each head (scale = (max - min) / 15, zero = -min, code clamped to
 *   [0, 15]).  The reference kernel takes min/max over |v| and wraps negative values to wrong codes; its output is the same
 *   only on heads whose values are all >= 0. */
ATOM_API int atom_gemm_i4_o4(const void* a, const void* b, const void* a_scale, const void* b_scale, const void* a_keeper,
                    const void* b_keeper, const void* a_keeper_scale, const void* b_keeper_scale, void* d,
                    void* d_scale, int64_t M, int64_t N, int64_t K, uint32_t flags, void* stream);

/* EXTENSION (launch-count reduction, SURVEY.md 8 f4): the q, k and v projections of LlamaAttention
 * (punica/models/llama.py:146-156: dense_layer_gemm_i4_fp16 for q, dense_layer_gemm_i4_o4 for k and v, same input) as ONE
 * launch over row-concatenated weights  b_qkv u8 [3H,(K-128)/2], b_scale_qkv f16 [K/128-1, 3H], b_keeper_qkv i8 [3H,128],
 * b_keeper_scale_qkv f16 [3H]  (rows [0,H) = q, [H,2H) = k, [2H,3H) = v).  Outputs are bit-identical to the three separate
 * calls: q f16 [M,H]; k, v u8 [M,H/2] with k_scale, v_scale f16 [M,H/128,2].  One launch whose channel tile selects the
 * epilogue. */
ATOM_API int atom_gemm_i4_qkv(const void* a, const void* b_qkv, const void* a_scale, const void* b_scale_qkv, const void* a_keeper,
                     const void* b_keeper_qkv, const void* a_keeper_scale, const void* b_keeper_scale_qkv, void* q, void* k,
                     void* k_scale, void* v, void* v_scale, int64_t M, int64_t H, int64_t K, uint32_t flags, void* stream);

/* EXTENSION (grouped-query attention): atom_gemm_i4_qkv with fewer KV heads than query heads.  Rows [0,Hq_dim) of the
 * concatenated weights are q, [Hq_dim, Hq_dim+Hkv_dim) k, the last Hkv_dim v (Hq_dim = query heads * 128, Hkv_dim = KV heads * 128,
 * Hq_dim % Hkv_dim == 0).  q f16 [M,Hq_dim]; k, v u8 [M,Hkv_dim/2] with k_scale, v_scale f16 [M,Hkv_dim/128,2]; bit-identical to
 * the three separate calls.  Hq_dim == Hkv_dim is atom_gemm_i4_qkv. */
ATOM_API int atom_gemm_i4_qkv_gqa(const void* a, const void* b_qkv, const void* a_scale, const void* b_scale_qkv, const void* a_keeper,
                         const void* b_keeper_qkv, const void* a_keeper_scale, const void* b_keeper_scale_qkv, void* q, void* k,
                         void* k_scale, void* v, void* v_scale, int64_t M, int64_t Hq_dim, int64_t Hkv_dim, int64_t K, uint32_t flags,
                         void* stream);

/* EXTENSION (launch-count reduction, SURVEY.md 8 f4): LlamaMLP's gate_proj, up_proj and activate_fp16_i4
 * (punica/models/llama.py:85-87) as ONE launch for decode batches (M <= 64; ATOM_E_UNSUPPORTED above): weights
 * row-concatenated  b_gu u8 [2I,(K-128)/2] (rows [0,I) = gate, [I,2I) = up), b_scale_gu f16 [K/128-1, 2I], b_keeper_gu
 * i8 [2I,128], b_keeper_scale_gu f16 [2I].  Outputs: the activation 4-tuple of activate_fp16_i4(gate, up) -- o_outliers i8
 * [M,128], o_norms u8 [M,(I-128)/2], outlier_scales f16 [scale_size(M)], norm_scales f16 [I/128-1, scale_size(M)] --
 * bit-identical to the three separate calls (both projections are rounded to FP16 before the activation, as there). */
ATOM_API int atom_gemm_i4_gateup_act(const void* a, const void* b_gu, const void* a_scale, const void* b_scale_gu, const void* a_keeper,
                            const void* b_keeper_gu, const void* a_keeper_scale, const void* b_keeper_scale_gu, void* o_outliers,
                            void* o_norms, void* outlier_scales, void* norm_scales, int64_t M, int64_t I, int64_t K, uint32_t flags,
                            void* stream);

/* Debug aid (no reference counterpart): when non-NULL, every GEMM CTA writes 128 clock64() stamps of its pipeline
 * phases to device_buffer[cta*128 ...] (layout in gemm_i4_sm90.cuh).  NULL switches tracing off. */
ATOM_API int atom_gemm_set_trace(void* device_buffer);

/* EXPERIMENTAL (no reference counterpart): programmatic dependent launch.  When enabled (also via
 * ATOM_B200_PDL=1 in the environment) every kernel is launched with programmatic stream serialization: its prologue -- for
 * the GEMM including the first weight tiles -- overlaps the tail of the preceding kernel; everything that reads that
 * kernel's output waits on griddepcontrol.wait.  Results are unchanged.  Off by default. */
ATOM_API int atom_set_pdl(int enable);

/* replaces batch_decode_i4 (punica_ops.cc:82-120 -> FlashInferBatchDecodeKernel_i4<128>, flashinfer_impl.cuh:9-46)
 *   o,q f16 [B,H,128]  kv_data u8 [pages,L,2,H,P,64]  kv_param f16 [pages,L,2,H,P,2]
 *   kv_indptr i32 [B+1]  kv_indices i32 [nnz]  last_page_offset i32 [B] */
ATOM_API int atom_batch_decode_i4(void* o, const void* q, const void* kv_data, const void* kv_param, const void* kv_indptr,
                         const void* kv_indices, const void* last_page_offset, int num_layers, int layer_idx,
                         int num_heads, int page_size, int batch_size, void* stream);

/* EXTENSION (grouped-query attention): batch_decode_i4 for num_q_heads = G * num_kv_heads query heads over a cache of
 * num_kv_heads heads -- the same layout with H = num_kv_heads; query head h attends KV head h / G.
 *   o,q f16 [B,num_q_heads,128]  kv_data u8 [pages,L,2,num_kv_heads,P,64]  kv_param f16 [pages,L,2,num_kv_heads,P,2]
 * One CTA per (sequence, KV head) reads every page of that head once and serves its G query heads.  rope_theta is the RoPE base
 * (1e4 for Llama-1/2, 5e5 for Llama-3, 1e6 for Mixtral).  G in {1, 2, 4, 8}; G = 1 with rope_theta = 1e4 IS
 * atom_batch_decode_i4 (same kernel, same bits); any other ratio returns ATOM_E_UNSUPPORTED. */
ATOM_API int atom_batch_decode_gqa_i4(void* o, const void* q, const void* kv_data, const void* kv_param, const void* kv_indptr,
                             const void* kv_indices, const void* last_page_offset, int num_layers, int layer_idx,
                             int num_q_heads, int num_kv_heads, int page_size, int batch_size, float rope_theta, void* stream);

/* EXTENSION (split-KV decode): atom_batch_decode_gqa_i4 with the KV length of each (sequence, KV head) spread over a cluster of
 * kv_split CTAs whose partial softmax states are merged through distributed shared memory in rank order (no workspace, one
 * launch, deterministic and independent of where the pages sit).  kv_split: 0 = automatic (atom_decode_kv_split on the current
 * device), 1 = never split (the atom_batch_decode_gqa_i4 kernel, bit for bit), 2 / 4 / 8 = that cluster size (a size that cannot
 * be scheduled on the device falls back to the largest smaller one that can); anything else returns ATOM_E_INVALID.
 * atom_batch_decode_i4 and atom_batch_decode_gqa_i4 are this call with kv_split = 0. */
ATOM_API int atom_batch_decode_split_gqa_i4(void* o, const void* q, const void* kv_data, const void* kv_param, const void* kv_indptr,
                                            const void* kv_indices, const void* last_page_offset, int num_layers, int layer_idx,
                                            int num_q_heads, int num_kv_heads, int page_size, int batch_size, float rope_theta,
                                            int kv_split, void* stream);

/* The cluster size kv_split = 0 picks: 1 when batch * num_kv_heads >= sm_count (every SM already has a CTA), otherwise the
 * smallest C in {2, 4, 8} with batch * num_kv_heads * C >= sm_count, and 8 at most.  group (query heads per KV head, 1/2/4/8) is
 * validated.  Returns C, or ATOM_E_INVALID for non-positive sizes or another group. */
ATOM_API int atom_decode_kv_split(int batch, int num_kv_heads, int group, int sm_count);

/* EXTENSION (shared-prefix decode): atom_batch_decode_gqa_i4 for a batch whose rows form prefix groups -- rows forked from one
 * sequence that begin on the same (full) pages.  Two launches on `stream`:
 *   prefix pass: each group's shared pages are streamed once per KV head, dequantised and rotated into FP16 tiles and attended by
 *     all members x G query rows with tensor-core MMAs (FP32 online softmax); the un-normalised (m, d, acc[128]) of every row and
 *     chunk goes to `workspace`;
 *   suffix pass: the decode kernel over each row's private pages, merging the row's prefix partials in chunk order first.
 * Rows outside every group (shared_pages 0) are computed exactly as atom_batch_decode_split_gqa_i4 with kv_split = 1 computes them.
 *   group_indptr i32 [num_groups+1], group_members i32: the rows of group i are group_members[group_indptr[i] .. group_indptr[i+1]]
 *   (at most max_group_size of them, at least two); shared_pages i32 [B]: leading pages row b shares with its group, equal for
 *   every member, 0 outside groups; rope_table f32 [>= longest shared prefix, 64, 2] as for atom_prefill_attention_i4 with base
 *   rope_theta; workspace f32 [B, num_q_heads, nchunks, 130]; nchunks from atom_decode_shared_chunks.
 * Everything else as atom_batch_decode_gqa_i4.  Deterministic: the result depends on nchunks, never on where the pages sit. */
ATOM_API int atom_batch_decode_shared_gqa_i4(void* o, const void* q, const void* kv_data, const void* kv_param, const void* kv_indptr,
                                             const void* kv_indices, const void* last_page_offset, int num_layers, int layer_idx,
                                             int num_q_heads, int num_kv_heads, int page_size, int batch_size, float rope_theta,
                                             const void* group_indptr, const void* group_members, const void* shared_pages,
                                             int num_groups, int max_group_size, const void* rope_table, float* workspace, int nchunks,
                                             void* stream);

/* The prefix-pass chunk count of atom_batch_decode_shared_gqa_i4: the fewest chunks with which num_groups x ceil(batch * group / 64)
 * x num_kv_heads x chunks reaches 2 * sm_count CTAs (group: query heads per KV head; a group's prefix is cut into that many runs
 * of whole 64-token tiles, short prefixes leave some empty).  Returns the count, or ATOM_E_INVALID for non-positive sizes. */
ATOM_API int atom_decode_shared_chunks(int num_groups, int batch, int group, int num_kv_heads, int sm_count);

/* EXTENSION (speculative decoding): multi-token decode attention for a verify step.  Sequence b of the cache ends with
 * tokens_per_seq = S query tokens (1 <= S <= 8) at positions len_b - S .. len_b - 1 whose K/V are already in the pages; token i
 * attends to every key at a position <= len_b - S + i.  q, o f16 [batch_size * S, num_q_heads, 128], row b * S + i = token i of
 * sequence b.  One launch (two when nchunks > 1): each (chunk, KV head, sequence) CTA streams its share of the sequence's pages
 * once for all S x G query rows of that KV head, on tensor cores.  Positions come from the page table on the device.
 *   rope_table f32 [>= max_b len_b, 64, 2] as for atom_prefill_attention_i4 with base rope_theta; workspace f32 [batch_size * S,
 *   num_q_heads, nchunks, 130] (may be NULL when nchunks == 1); nchunks from atom_verify_chunks.
 * Precondition: len_b >= S for every sequence (the device holds the lengths, so it is not checked on the host); the rows of a
 * sequence that breaks it are zeros, and none of its pages is read.
 * Everything else as atom_batch_decode_gqa_i4.  Deterministic: the result depends on nchunks, never on where the pages sit. */
ATOM_API int atom_batch_verify_gqa_i4(void* o, const void* q, const void* kv_data, const void* kv_param, const void* kv_indptr,
                                      const void* kv_indices, const void* last_page_offset, int num_layers, int layer_idx,
                                      int num_q_heads, int num_kv_heads, int page_size, int batch_size, int tokens_per_seq,
                                      float rope_theta, const void* rope_table, float* workspace, int nchunks, void* stream);

/* The chunk count of atom_batch_verify_gqa_i4: 1 when batch * num_kv_heads >= sm_count, otherwise the fewest chunks with which
 * batch x num_kv_heads x chunks reaches 2 * sm_count CTAs, 64 at most (a sequence's 64-token tiles are cut into that many runs;
 * short sequences leave some empty).  Returns the count, or ATOM_E_INVALID for non-positive sizes. */
ATOM_API int atom_verify_chunks(int batch, int num_kv_heads, int sm_count);

/* EXTENSION (SURVEY.md 8 f3): the prefill attention the reference leaves as a placeholder
 * (punica/models/llama.py:171-190, SDPA over torch.randn K/V): causal attention of every prompt over its own just-quantised
 * K/V -- the o4 outputs of the k/v projections, x = nibble * scale - zero (quantization.cuh:76) -- with RoPE(theta 1e4) on q
 * and k at positions 0..len-1, head_dim 128.
 *   q f16 [T, H*128]; k, v u8 [T, H*64]; k_param, v_param f16 [T, H, 2]; seqlen_indptr i32 [B+1]; pos_of_token i32 [T];
 *   rope_table f32 [max_len, 64, 2] = (cos, sin)(pos * 1e4^(-i/64)); k_f16, v_f16 f16 [T, H*128] scratch (caller-owned,
 *   holds RoPE(dequant k) and dequant v afterwards); out f16 [T, H*128].  max_len >= the longest prompt. */
ATOM_API int atom_prefill_attention_i4(const void* q, const void* k, const void* k_param, const void* v, const void* v_param,
                              const void* seqlen_indptr, const void* pos_of_token, const void* rope_table, void* k_f16, void* v_f16,
                              void* out, int total_tokens, int batch_size, int max_len, int num_heads, void* stream);

/* EXTENSION (grouped-query attention): atom_prefill_attention_i4 with num_kv_heads <= num_q_heads (num_q_heads % num_kv_heads == 0).
 *   q, out f16 [T, num_q_heads*128]; k, v u8 [T, num_kv_heads*64]; k_param, v_param f16 [T, num_kv_heads, 2];
 *   k_f16, v_f16 f16 [T, num_kv_heads*128] scratch; rope_table built for the model's RoPE base.  Everything else as above. */
ATOM_API int atom_prefill_attention_gqa_i4(const void* q, const void* k, const void* k_param, const void* v, const void* v_param,
                                  const void* seqlen_indptr, const void* pos_of_token, const void* rope_table, void* k_f16, void* v_f16,
                                  void* out, int total_tokens, int batch_size, int max_len, int num_q_heads, int num_kv_heads,
                                  void* stream);

/* EXTENSION (chunked prefill, prompt continuation): atom_prefill_attention_gqa_i4 over a cached prefix.  Prompt b is the tail of
 * sequence b of the paged INT4 cache (the tokens atom_init_kv_i4 just wrote with the same seqlen_indptr): with seq_len_b from the
 * page table (kv_indptr, last_page_offset) and L_b its prompt length, its ctx_b = seq_len_b - L_b cached tokens come first.  Its
 * queries attend to all of them and, causally, to the prompt's own tokens; q and k are rotated at their absolute positions.
 *   pos_of_token i32 [T]: ctx_b + i for token i of prompt b; rope_table: rows up to max_b(ctx_b + L_b) - 1; k_f16 / v_f16 hold
 *   the prompt's tokens only (no scratch grows with the context); kv_*: the cache as for atom_batch_decode_gqa_i4 (num_kv_heads
 *   heads, layer layer_idx of num_layers, page_size a multiple of 8 up to 64).  num_q_heads / num_kv_heads must be 1, 2, 4 or 8
 *   (ATOM_E_UNSUPPORTED otherwise).  Everything else as atom_prefill_attention_gqa_i4; with every ctx_b = 0 the result equals it. */
ATOM_API int atom_prefill_attention_ctx_gqa_i4(const void* q, const void* k, const void* k_param, const void* v, const void* v_param,
                                      const void* seqlen_indptr, const void* pos_of_token, const void* rope_table, void* k_f16,
                                      void* v_f16, void* out, int total_tokens, int batch_size, int max_len, int num_q_heads,
                                      int num_kv_heads, const void* kv_data, const void* kv_param, const void* kv_indptr,
                                      const void* kv_indices, const void* last_page_offset, int num_layers, int layer_idx,
                                      int page_size, void* stream);

/* EXTENSION (SURVEY.md 8e; the reference has no multi-GPU code): one-shot all-reduce (sum) of an FP16 vector over NVLink peer
 * memory for the tensor-parallel row-parallel projections.  peer_buffers: DEVICE array of `world` pointers to every rank's
 * receive buffer, f16 [3][world][slot_elems], every half initialised to 0x8000 (FP16 -0.0: the "not yet arrived" pattern;
 * a -0.0 input element is transmitted as +0.0), e.g. allocated and exchanged with torch.distributed._symmetric_memory;
 * state: local u32 [atom_allreduce_state_words()], zeroed once.  Every rank must make the same sequence of calls.
 * No flags, fences or barriers: the payload is its own arrival signal (three rotating buffers on a device-side call counter).
 * Graph-capturable; the sum is formed in rank order in FP32 and is bit-identical on all ranks. */
ATOM_API int atom_allreduce_push_f16(const void* in, void* out, const void* peer_buffers, void* state, int64_t numel,
                            int64_t slot_elems, int rank, int world, void* stream);
ATOM_API int atom_allreduce_state_words(void);

/* The same all-reduce with its two halves fused into the kernels around it (decode batches, M <= 64):
 *   atom_gemm_i4_o16_push            the row-parallel projection (o_proj / down_proj shard): atom_gemm_i4_o16 whose epilogue stores D
 *                                    into slot [call % 3][rank] of EVERY rank's receive buffer instead of a local tensor;
 *   atom_reduce_add_rmsnorm_fp16_i4  atom_add_rmsnorm_fp16_i4 whose `hidden` input is the sum over the ranks of those slots: each
 *                                    16-byte chunk is polled until its payload has arrived, summed in rank order in FP32 and rounded
 *                                    to FP16 (bit-identical to what atom_allreduce_push_f16 would have delivered), then added to the
 *                                    residual, normalised and quantised as usual.  hidden_dim % 1024 == 0.
 * The pair must be called in this order with the same (peer_buffers, state) and M x N = seq_len x hidden_dim; pairs and stand-alone
 * atom_allreduce_push_f16 calls on the same buffers may be mixed freely (one call counter). */
ATOM_API int atom_gemm_i4_o16_push(const void* a, const void* b, const void* a_scale, const void* b_scale, const void* a_keeper,
                          const void* b_keeper, const void* a_keeper_scale, const void* b_keeper_scale, const void* peer_buffers,
                          void* state, int64_t slot_elems, int rank, int world, int64_t M, int64_t N, int64_t K, uint32_t flags,
                          void* stream);
ATOM_API int atom_reduce_add_rmsnorm_fp16_i4(const void* peer_buffers, void* state, int64_t slot_elems, int rank, int world,
                                    const void* residual, void* sum_out, const void* weight, float eps, const void* reorder_index,
                                    int seq_len, int hidden_dim, void* o_outliers, void* o_norms, void* outlier_scales,
                                    void* norm_scales, void* stream);

/* EXTENSION (Mixtral sparse MoE block, csrc/moe_kernels.cuh).  E = num_experts <= 64 experts, k = top_k <= min(E, 8) per token.
 * One block: atom_add_rmsnorm_fp16_i4 (the activation tuple every expert reads: all experts share expert 0's channel orders),
 * route, plan, gather, grouped gate/up+act, grouped down, combine -- seven launches whose sizes depend only on (T, E, k), so the
 * block is graph-capturable with data-dependent routing.  BN = token tile = 16 / 32 / 64 for ceil(T*k/E) <= 16 / 32 / more;
 * tiles_max = min(T*k, (T*k + E*(BN-1)) / BN); rows_cap = tiles_max * BN rows of permuted workspace.
 *
 * atom_moe_route_f16: the FP router on the FP16 normalised row.  hidden f16 [T,H] (the residual sum the add+RMSNorm returned),
 *   norm_weight f16 [H], reorder_index i16 [H], router_weight f16 [E,H] in the reordered channel order.  y = half(float(x) *
 *   float(w) * rstd) exactly as atom_rmsnorm_fp16_i4 forms it; logits FP32; softmax FP32; top-k on the logits, an exact tie goes
 *   to the lower expert index.  topk_ids i32 [T,k], topk_weights f16 [T,k] = fp16(p_i / sum of the selected p); optional
 *   (NULL = not written): router_logits f32 [T,E], normed f16 [T,H] (y). */
ATOM_API int atom_moe_route_f16(const void* hidden, const void* norm_weight, float eps, const void* reorder_index, const void* router_weight,
                       int seq_len, int hidden_dim, int num_experts, int top_k, void* topk_ids, void* topk_weights,
                       void* router_logits, void* normed, void* stream);

/* atom_moe_plan: one CTA.  dest_row i32 [T,k]: the permuted row of every (token, slot); expert e's segment starts at
 * sum_{e'<e} ceil(count_e'/BN)*BN, tokens ascending inside it.  tiles i32 [tiles_max,4] = (expert, first row, valid rows, 0), the
 * non-empty tiles in expert order, then (0,0,0,0).  Ids outside [0,E) are not routed (dest_row -1). */
ATOM_API int atom_moe_plan(const void* topk_ids, int seq_len, int num_experts, int top_k, int token_tile, int tiles_max, void* dest_row,
                  void* tiles, void* stream);

/* atom_moe_gather_i4: copy each routed token's rows of the activation tuple (o_outliers i8 [T,128], o_norms u8 [T,(H-128)/2],
 * scales in the layout of S(T)) to row dest_row of the permuted tuple (p_* with rows_cap rows, scales in the layout of
 * S(rows_cap)).  Pad rows are not written. */
ATOM_API int atom_moe_gather_i4(const void* o_outliers, const void* o_norms, const void* outlier_scales, const void* norm_scales, int seq_len,
                       int hidden_dim, int top_k, const void* dest_row, int rows_cap, void* p_outliers, void* p_norms,
                       void* p_outlier_scales, void* p_norm_scales, void* stream);

/* Grouped expert GEMMs over the permuted activations (rows_cap = num_tiles * token_tile rows) and weights stacked over the experts:
 *   gate/up: b_gu u8 [E, 2I, (K-128)/2], b_scale_gu f16 [E, K/128-1, 2I], b_keeper_gu i8 [E, 2I, 128], b_keeper_scale_gu f16 [E, 2I]
 *            (per expert rows [0,I) = gate (w1), [I,2I) = up (w3)); outputs the activation tuple of rows_cap rows for the down
 *            projection, as atom_gemm_i4_gateup_act;
 *   down:    b u8 [E, N, (K-128)/2], b_scale f16 [E, K/128-1, N], b_keeper i8 [E, N, 128], b_keeper_scale f16 [E, N]; d f16 [rows_cap, N].
 * Tile j of the plan's table computes its rows against its expert's weights; rows past its valid count are not stored, empty
 * tiles return at once.  No K split: every stored row is bit-identical to the per-expert atom_gemm_i4_gateup_act / atom_gemm_i4_o16
 * call with ATOM_GEMM_NO_SPLITK on that expert's rows.  Everything (the tile table included) is read after the preceding kernel
 * has completed. */
ATOM_API int atom_gemm_i4_gateup_act_grouped(const void* a, const void* b_gu, const void* a_scale, const void* b_scale_gu, const void* a_keeper,
                                    const void* b_keeper_gu, const void* a_keeper_scale, const void* b_keeper_scale_gu, void* o_outliers,
                                    void* o_norms, void* outlier_scales, void* norm_scales, const void* tiles, int num_tiles,
                                    int token_tile, int64_t rows_cap, int64_t num_experts, int64_t I, int64_t K, void* stream);
ATOM_API int atom_gemm_i4_o16_grouped(const void* a, const void* b, const void* a_scale, const void* b_scale, const void* a_keeper,
                             const void* b_keeper, const void* a_keeper_scale, const void* b_keeper_scale, void* d, const void* tiles,
                             int num_tiles, int token_tile, int64_t rows_cap, int64_t num_experts, int64_t N, int64_t K, void* stream);

/* atom_moe_combine_f16: out f16 [T,H] = sum over t's slots in ascending expert order of fp16(y[dest_row] * w), one FP16 rounding per
 * product and per add, from +0.0 -- bit for bit `out = zeros; out.index_add_(0, tok_e, (y_e * w_e).half())` expert by expert.
 * y f16 [rows_cap,H] (the down projection).  The result is the MoE delta of the residual stream. */
ATOM_API int atom_moe_combine_f16(const void* y, const void* topk_ids, const void* topk_weights, const void* dest_row, int seq_len, int hidden_dim,
                         int top_k, void* out, void* stream);

/* atom_sample_f16: one token id per row of FP16 logits, sampled with per-row temperature, top-k and top-p from a counter-based
 * Philox stream (new: the reference only takes the argmax).
 *   logits f16 [batch, ld] (row b at logits + b*ld, the first vocab entries used; vocab <= 262144)
 *   temperature f32 [batch], top_k i32 [batch] (0 = off), top_p f32 [batch] (1 = off), key u64 [batch][2], counter u64 [batch],
 *   out i32 [batch].  All parameters are read on the device, after the preceding kernel has completed.
 * One total order throughout: value descending, then index ascending (-0 == +0).  Per row:
 *   1. A NaN or +inf logit, all logits -inf, or parameters out of range (T not finite or < 0, top_k < 0, top_p not in (0, 1])
 *      give -1.  A -inf logit is masked: it is never drawn.
 *   2. T == 0 or top_k == 1: the first index of the maximum (torch.argmax).
 *   3. top_k = k > 0: exactly the first k tokens of the order on the raw FP16 logits (ties at the k-th value to lower indices).
 *   4. top_p = p < 1: over the top-k survivors with weights w = round(expf(fl(fl(l - max) / T)) * 2^40) (FP32, then an exact
 *      integer), keep the tokens of the order whose exclusive mass is below ceil(p * Z), Z their total: the shortest prefix
 *      whose mass reaches p.  The top token is always kept.
 *   5. The draw: u = (w0 >> 11) * 2^-53, w0 = word 0 of the Philox4x64-10 block at counter (counter[b], 0, 0, 0) under key
 *      (key[b][0], key[b][1]); the token is the first kept index, ascending, whose running sum of weights exceeds floor(u * Z).
 * The result of a row depends only on that row's logits, parameters, key and counter: not on batch, its position, ld or the
 * launch.  No state: a captured graph replays with new device values. */
ATOM_API int atom_sample_f16(const void* logits, int64_t ld, int batch, int vocab, const void* temperature, const void* top_k,
                             const void* top_p, const void* key, const void* counter, void* out, void* stream);

/* atom_sample_ex_f16: atom_sample_f16 with penalties, min-p and log-probabilities (new: the reference only takes the argmax).
 * The arguments of atom_sample_f16, plus, all read on the device after the preceding kernel has completed:
 *   min_p f32 [batch] or null (off);
 *   rep, freq, pres f32 [batch], slots i32 [batch], table u16 [*][table_ld >= vocab]: all null (no penalties) or all given;
 *   logprob_out f32 [batch] or null; top_n in [0, 20]; top_ids i32 [batch][top_n], top_logprobs f32 [batch][top_n].
 * Penalty state: row b names a slot s = slots[b] of the table, or -1 (none).  An entry holds bit 15 = the token occurs in the
 * request's prompt (a shared system prompt included) and bits 0-14 = how often the request has generated it, saturating at
 * 0x7FFF.  Slots in one call must be distinct.
 * Penalised logit, per token of a row with a slot, from its FP16 value l, each step one IEEE FP32 operation:
 *   1. -inf stays -inf;
 *   2. repetition r, if the token is in the prompt or its count c > 0:  l = l > 0 ? fl(l / r) : fl(l * r);
 *   3. frequency f:  l = fl(l - fl(c * f));
 *   4. presence p, if c > 0:  l = fl(l - p);
 *   5. l' = FP16 round-to-nearest of min(max(l, -65504), 65504) (fmin / fmax: a NaN from inf - inf becomes -65504).
 * Rules 1-5 of atom_sample_f16 then apply to l' instead of the raw logits; the NaN / +inf / all -inf test of rule 1 is still made
 * on the raw row.  Also:
 *   - min-p m in [0, 1], after top-k and before top-p: keep the survivors whose weight W_i >= ceil(m * 2^40) (the top token's
 *     weight is exactly 2^40); top-p then works over what is left.  m = 0 is off.
 *   - Log-probabilities: a log-softmax of l' at temperature 1 over the whole row (independent of T, top-k, top-p and min-p):
 *     lp_i = (fl(l'_i - max l') - ln(Z1 * 2^-40)) in double, rounded to FP32, Z1 = sum over the row of
 *     round(expf(l'_j - max) * 2^40), exact.  logprob_out[b] is the chosen token's lp; top_ids / top_logprobs the first top_n
 *     tokens of the order on l' with theirs, padded with id -1 and lp -inf past the finite tokens.  An invalid row (token -1)
 *     gives lp NaN, ids -1 and top lps NaN.
 *   - Recording: with a slot and a token, the kernel adds one to the token's count in the slot, saturating, in the same launch.
 *   - Parameters out of range give -1, as in rule 1: also r not finite or <= 0, f or p not finite, m not in [0, 1].
 * With no table, no min_p, no logprob_out and top_n = 0 this is atom_sample_f16. */
ATOM_API int atom_sample_ex_f16(const void* logits, int64_t ld, int batch, int vocab, const void* temperature, const void* top_k,
                                const void* top_p, const void* key, const void* counter, const void* min_p, const void* rep,
                                const void* freq, const void* pres, const void* slots, void* table, int64_t table_ld, void* out,
                                void* logprob_out, int top_n, void* top_ids, void* top_logprobs, void* stream);

/* atom_sample_draft_f16: sampling with one candidate token per row, for speculative decoding (new; DESIGN section 5.7).
 * The arguments of atom_sample_ex_f16 without the penalty ones (rep, freq, pres, slots, table, table_ld), plus drafts i32 [batch],
 * read on the device after the preceding kernel has completed.  Rules 1-4, min-p and the log-probabilities are atom_sample_ex_f16's
 * and give the kept weights W (Z = sum of W).  Per row, d = drafts[b]:
 *   - d = -1 (no candidate): rule 5; token, logprob and top-n are bit-identical to atom_sample_ex_f16's for the same row.
 *   - d in [0, vocab): W_d = d's kept weight (0 if d is not kept); a = w1 >> 11, w1 = word 1 of rule 5's Philox block.  The row
 *     accepts d iff floor(a * Z * 2^-53) < W_d (the exact 128-bit product of rule 5); then the token is d.  Otherwise the token
 *     is rule 5's draw with word 0 over the kept set without d, whose total Z - W_d is then > 0.  So P(token = t) = W_t / Z up
 *     to the 2^-53 discretisation of a and u, for every t.  T = 0 or top_k = 1: the first index of the maximum, whatever d.
 *   - d < -1 or d >= vocab: -1, as any parameter out of range.
 * logprob_out is the emitted token's; the top-n list does not depend on d or the draw. */
ATOM_API int atom_sample_draft_f16(const void* logits, int64_t ld, int batch, int vocab, const void* temperature, const void* top_k,
                                   const void* top_p, const void* key, const void* counter, const void* min_p, void* out,
                                   void* logprob_out, int top_n, void* top_ids, void* top_logprobs, const void* drafts, void* stream);

/* atom_spec_commit_propose: one launch per speculative step, one CTA per sequence (new; DESIGN section 5.8).  Token histories:
 * history i32 [num_slots][cap], history_len i32 [num_slots].  Sequence i owns rows row_indptr[i] .. row_indptr[i+1] of tokens
 * (the sampler's output) and cands (the candidates it was given, -1: none), and history slot slots[i].  The kernel
 *   1. commits: m = the first j with cands[j] < 0 or tokens[j] != cands[j] (rows past num_draft + 1 are ignored); tokens 0 .. m
 *      are emitted and appended to the slot, never past cap;
 *   2. proposes by prompt lookup over the slot's history h[0, L): for n = ngram_max down to ngram_min, the latest p with
 *      p + n <= L - 1 and h[p, p + n) == h[L - n, L); the drafts are h[p + n, min(p + n + num_draft, L)), and the first n that
 *      matches wins; no match: no drafts;
 *   3. writes out i32 [batch][2 * num_draft + 3]: emitted (m + 1), draft_len, the emitted tokens [num_draft + 1] and the drafts
 *      [num_draft], both padded with -1.
 * A slot outside [0, num_slots) gives emitted = draft_len = 0 and touches no history.  Needs 1 <= num_draft <= 7 and
 * 1 <= ngram_min <= ngram_max <= 16.  Allocates nothing; all inputs are read after the preceding kernel has completed. */
ATOM_API int atom_spec_commit_propose(const void* tokens, const void* cands, const void* row_indptr, const void* slots, int batch,
                                      void* history, void* history_len, int num_slots, int cap, int num_draft, int ngram_min,
                                      int ngram_max, void* out, void* stream);

/* atom_beam_select_f16: one beam-search step (new; DESIGN section 5.9).  logits f16 [rows][ld], sums f32 [rows] (each row's
 * beam's running sum), row_indptr i32 [batch + 1] (request i owns rows row_indptr[i] .. row_indptr[i+1]; zero rows is allowed),
 * stop_ids: num_stop <= 8 distinct host ids in [0, vocab), width W in [1, 8].  For every row, lp(t) is bit for bit the
 * log-probability atom_sample_ex_f16 reports for token t at T = 1 without penalties; a row holding NaN or +inf, or only -inf,
 * has no candidates, and neither has a token at -inf.  A candidate's key is fl32(sums[row] + lp(t)).  A request's candidates
 * are ordered by key descending, then row ascending, then the row's order (larger logit, then lower id); walking them at rank
 * i = 0, 1, ..: a stop id of rank < W is written to fin, one of rank >= W is skipped, any other token is written to live until
 * there are W.  live and fin i32 [batch][W][2] hold (row, token), live_key and fin_key f32 [batch][W] the keys; unused entries
 * are -1.  A request of more than W rows gets none.  workspace: 16-byte aligned, rows * 192 bytes.  Two launches (the per-row
 * lists, then one CTA per request); every device input is read after the preceding kernel has completed.  With rows = 0 only
 * the second runs (every request gets none), and logits and sums may be null. */
ATOM_API int atom_beam_select_f16(const void* logits, int64_t ld, int rows, int vocab, const void* row_indptr, int batch,
                                  const void* sums, const int* stop_ids, int num_stop, int width, void* workspace, void* live,
                                  void* live_key, void* fin, void* fin_key, void* stream);

/* atom_kv_copy_pages_i4: the page copies of copy-on-write forks in one launch (new; DESIGN section 5.9).  Pair p of src, dst,
 * slots (i32 [n], read on the device after the preceding kernel has completed) copies the first slots[p] token slots of page
 * src[p] to page dst[p] in every (layer, K|V, head) block of kv_data (u8 [num_pages][num_layers][2][num_heads][page_size][64])
 * and kv_param (f16 [...][page_size][2]); the bytes past slots[p] are left untouched.  src < 0 is padding; src == dst, a page
 * outside [0, num_pages) or slots outside [1, page_size] make the pair a no-op. */
ATOM_API int atom_kv_copy_pages_i4(void* kv_data, void* kv_param, int num_pages, int num_layers, int num_heads, int page_size,
                                   const void* src, const void* dst, const void* slots, int n, void* stream);

/* atom_sample_slot_init: set up slot `slot` of a penalty table u16 [*][table_ld] (16-byte aligned, table_ld >= vocab a multiple
 * of 8) for a new request in one launch: zero the row, then set bit 15 of every token in prompt i32 [prompt_len] (ids outside
 * [0, vocab) are ignored). */
ATOM_API int atom_sample_slot_init(void* table, int64_t table_ld, int vocab, int slot, const void* prompt, int prompt_len, void* stream);

/* replaces append_kv_i4 (punica_ops.cc:166-209 -> FlashInferAppendKvKernel_i4<128>, flashinfer_impl.cuh:73-96)
 *   k,v u8 [B,H,64]  k_param,v_param f16 [B,H,2] */
ATOM_API int atom_append_kv_i4(void* kv_data, void* kv_param, const void* kv_indptr, const void* kv_indices,
                      const void* last_page_offset, const void* k, const void* v, const void* k_param,
                      const void* v_param, int num_layers, int layer_idx, int num_heads, int page_size, int batch_size,
                      void* stream);

/* replaces init_kv_i4 (punica_ops.cc:122-164 -> FlashInferInitKvKernel_i4<128>, flashinfer_impl.cuh:48-71)
 *   k,v u8 [sum(len),H,64]  params f16 [sum(len),H,2]  seqlen_indptr i32 [B+1]; total_tokens = seqlen_indptr[B] */
ATOM_API int atom_init_kv_i4(void* kv_data, void* kv_param, const void* kv_indptr, const void* kv_indices,
                    const void* last_page_offset, const void* k, const void* v, const void* k_param,
                    const void* v_param, const void* seqlen_indptr, int total_tokens, int num_layers, int layer_idx,
                    int num_heads, int page_size, int batch_size, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ATOM_B200_H_ */
