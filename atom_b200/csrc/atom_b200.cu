// atom_b200.cu -- C ABI (include/atom_b200.h) and host-side launch logic of libatom_b200.so.
//
// No torch types, no allocation, no synchronisation: every entry point validates its arguments, builds the TMA
// descriptors it needs on the host (cached by (pointer, shape)) and enqueues kernels on the caller's stream.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdlib>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <set>
#include <string>
#include <unordered_map>
#include <utility>

#include "../../include/atom_b200.h"
#include "gemm_i4_sm90.cuh"
#include "kv_kernels.cuh"
#include "prefill_kernels.cuh"
#include "comm_kernels.cuh"
#include "quant_kernels.cuh"
#include "moe_kernels.cuh"

namespace {

thread_local std::string g_err;
unsigned long long* g_trace = nullptr;   // atom_gemm_set_trace

// Programmatic dependent launch (opt-in: ATOM_B200_PDL=1 in the environment, or atom_set_pdl): kernels are launched with
// cudaLaunchAttributeProgrammaticStreamSerialization and told so (`pdl` argument), so that their prologue -- for the GEMM
// including the first weight tiles -- overlaps the tail of the preceding kernel.  Off: plain stream order, and the
// kernels never execute a griddepcontrol instruction.
int g_pdl = -1;
bool pdl_enabled() {
  if (g_pdl < 0) {
    const char* e = getenv("ATOM_B200_PDL");
    g_pdl = (e != nullptr && e[0] == '1') ? 1 : 0;
  }
  return g_pdl == 1;
}

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}

#define ATOM_REQUIRE(cond, ...) \
  do { if (!(cond)) return fail(ATOM_E_INVALID, __VA_ARGS__); } while (0)

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(ATOM_E_CUDA, "%s: %s", what, cudaGetErrorString(e));
  return ATOM_OK;
}

// <<<>>> when PDL is off (the validated path, untouched); cudaLaunchKernelEx with the attribute when it is on
template <typename... KArgs, typename... Args>
int launch_k(const char* what, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args... args) {
  if (!pdl_enabled()) {
    kern<<<grid, block, smem, stream>>>(args..., 0);
  } else {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    cudaError_t e = cudaLaunchKernelEx(&cfg, kern, args..., 1);
    if (e != cudaSuccess) return fail(ATOM_E_CUDA, "%s launch: %s", what, cudaGetErrorString(e));
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(ATOM_E_CUDA, "%s: %s", what, cudaGetErrorString(e));
  return ATOM_OK;
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// cudaFuncAttributeMaxDynamicSharedMemorySize is per (function, device): raise it once for each pair, under a lock
// (the reference calls cudaFuncSetAttribute on every launch, GEMM.cuh:757).
template <typename F>
int ensure_dynamic_smem(F* func, int bytes, const char* what) {
  static std::mutex mu;
  static std::set<std::pair<const void*, int>> done;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return fail(ATOM_E_CUDA, "%s: no current CUDA device", what);
  const std::pair<const void*, int> key(reinterpret_cast<const void*>(func), dev);
  std::lock_guard<std::mutex> lk(mu);
  if (done.count(key)) return ATOM_OK;
  cudaError_t e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return fail(ATOM_E_CUDA, "%s: cudaFuncSetAttribute(smem=%d): %s", what, bytes, cudaGetErrorString(e));
  done.insert(key);
  return ATOM_OK;
}

// ------------------------------------------------------------------------------------------------ TMA descriptors
using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                              const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeFn encode_fn() {
  static EncodeFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<EncodeFn>(p);
  }();
  return fn;
}

struct MapKey {
  const void* ptr; uint64_t inner, rows, pitch; uint32_t box_inner, box_rows, swizzle;
  bool operator==(const MapKey& o) const {
    return ptr == o.ptr && inner == o.inner && rows == o.rows && pitch == o.pitch && box_inner == o.box_inner &&
           box_rows == o.box_rows && swizzle == o.swizzle;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = reinterpret_cast<size_t>(k.ptr);
    auto mix = [&](uint64_t v) { h ^= v + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2); };
    mix(k.inner); mix(k.rows); mix(k.pitch); mix(k.box_inner); mix(k.box_rows); mix(k.swizzle);
    return h;
  }
};
std::mutex g_map_mu;
std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_maps;

// 2-D byte tensor [rows][inner] with row pitch `pitch`; box = box_rows x box_inner bytes; OOB rows read as zero.
// swizzle: 0 = none, 1 = SWIZZLE_128B
int make_map(CUtensorMap* out, const void* ptr, uint64_t inner, uint64_t rows, uint64_t pitch, uint32_t box_inner,
             uint32_t box_rows, int swizzle) {
  MapKey key{ptr, inner, rows, pitch, box_inner, box_rows, (uint32_t)swizzle};
  {
    std::lock_guard<std::mutex> lk(g_map_mu);
    auto it = g_maps.find(key);
    if (it != g_maps.end()) { *out = it->second; return ATOM_OK; }
  }
  EncodeFn fn = encode_fn();
  if (!fn) return fail(ATOM_E_CUDA, "cuTensorMapEncodeTiled is not available from this driver");
  cuuint64_t dims[2] = {inner, rows};
  cuuint64_t strides[1] = {pitch};
  cuuint32_t box[2] = {box_inner, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle == 1 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(ATOM_E_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  std::lock_guard<std::mutex> lk(g_map_mu);
  if (g_maps.size() > 4096) g_maps.clear();
  g_maps.emplace(key, *out);
  return ATOM_OK;
}

// ------------------------------------------------------------------------------------------------ GEMM launch
struct GemmOperands {
  const void *a, *b, *ak, *bk;
  int64_t M, N, K;          // N = weight rows
};

// The GEMM is launched with programmatic stream serialization unless ATOM_B200_GEMM_PDL=0: the kernel fetches only weights
// before griddepcontrol.wait.
int g_gemm_pdl = -1;
bool gemm_pdl_enabled() {
  if (g_gemm_pdl < 0) {
    const char* e = getenv("ATOM_B200_GEMM_PDL");
    g_gemm_pdl = (e != nullptr && e[0] == '0') ? 0 : 1;
  }
  return g_gemm_pdl == 1;
}

// out_channels: channels that get a tile of their own (gate/up: op.N = 2 I weight rows, I output channels)
// token_tiles: grid.y when it is not the tiles of op.M (grouped mode: the length of the token-tile table)
template <int BN, int kSplit, int kEpi>
int launch_gemm(const GemmOperands& op, const atom::GemmArgs& args, cudaStream_t stream, int64_t out_channels = -1,
                int64_t token_tiles = -1) {
  using C = atom::GemmCfg<BN, kSplit, kEpi>;
  auto kern = atom::gemm_i4_kernel<BN, kSplit, kEpi>;
  int rc = ensure_dynamic_smem(kern, C::SMEM_BYTES, "gemm_i4");
  if (rc) return rc;
  const uint64_t kp = (uint64_t)(op.K - 128) / 2;
  CUtensorMap tw4, ta4, tw8, ta8;
  if ((rc = make_map(&tw4, op.b, kp, op.N, kp, 64, 128, 0))) return rc;
  if ((rc = make_map(&ta4, op.a, kp, op.M, kp, 64, BN, 0))) return rc;
  if ((rc = make_map(&tw8, op.bk, 128, op.N, 128, 128, 128, 1))) return rc;
  if ((rc = make_map(&ta8, op.ak, 128, op.M, 128, 128, BN, 1))) return rc;
  const int64_t chan = out_channels > 0 ? out_channels : op.N;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)((chan + 127) / 128), (unsigned)(token_tiles > 0 ? token_tiles : (op.M + BN - 1) / BN), kSplit);
  cfg.blockDim = dim3(C::THREADS);
  cfg.dynamicSmemBytes = C::SMEM_BYTES;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 1; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = kSplit;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (gemm_pdl_enabled()) {
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.numAttrs = 2;
  }
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, tw4, ta4, tw8, ta8, args);
  if (e != cudaSuccess) return fail(ATOM_E_CUDA, "gemm_i4 launch: %s", cudaGetErrorString(e));
  return ATOM_OK;
}

// token tile: the smallest that holds a decode batch, 128 from 65 tokens on
int token_tile(int64_t M, uint32_t flags) {
  if (flags & ATOM_GEMM_FORCE_TALL) return 128;
  const int bn = M <= 16 ? 16 : (M <= 32 ? 32 : (M <= 64 ? 64 : 128));
  return (flags & ATOM_GEMM_FORCE_SKINNY) ? std::min(bn, 64) : bn;
}

template <int kEpi>
int gemm_dispatch(const GemmOperands& op, const atom::GemmArgs& args, uint32_t flags, cudaStream_t stream, int64_t out_channels = -1) {
  const int bn = token_tile(op.M, flags);
  const int64_t tiles = ((out_channels > 0 ? out_channels : op.N) + 127) / 128 * ((op.M + bn - 1) / bn);
  const int groups = args.G + 1;
  // K split over a cluster while the output tiles alone leave SMs of the 132 idle: a decode GEMM is a weight stream, and more
  // CTAs keep more bytes in flight.  The reduction grows with the token tile, so only 16-token tiles split 4-way (two of their
  // CTAs fit an SM: 264 slots), larger tiles 2-way; every rank keeps at least 4 groups; an 8-way split only runs on request.
  // Measured on an H100 (80 GB HBM3, 700 W), device time per launch from a CUDA graph over operand sets larger than L2, split
  // 1 / 2 / 4 / 8: 16 x 4096 x 4096: 23.5 / 15.8 / 12.8 / 16.7 us; 16 x 11008 x 4096: 27.0 / 21.0 / 26.7 / 29.8;
  // 32 x 5120 x 5120: 29.2 / 19.9 / 26.0 / 30.5; 64 x 4096 x 4096: 27.8 / 18.8 / 28.3 / 35.8; 128 x 4096 x 4096: 38.9 / 35.3 / 47.3 / 55.5.
  // The quantising epilogues work on FP32 sums in the reference's order and never split.
  int ksplit = 1;
  if constexpr (kEpi == atom::EPI_O16 || kEpi == atom::EPI_PUSH) {
    if (!(flags & (ATOM_GEMM_NO_SPLITK | ATOM_GEMM_FORCE_TALL))) {
      if (flags & ATOM_GEMM_SPLITK2) ksplit = 2;
      else if (flags & ATOM_GEMM_SPLITK4) ksplit = 4;
      else if (flags & ATOM_GEMM_SPLITK8) ksplit = 8;
      else if (op.M <= 128 && groups >= 8) {
        const int64_t slots = bn == 16 ? 264 : 132;
        ksplit = (bn == 16 && groups >= 16 && tiles * 4 <= slots) ? 4 : (tiles * 2 <= slots ? 2 : 1);
      }
    }
  }
#define ATOM_BN(BN_)                                                                                  \
  do {                                                                                                \
    if constexpr (kEpi == atom::EPI_O16 || kEpi == atom::EPI_PUSH) {                                  \
      if (ksplit == 8) return launch_gemm<BN_, 8, kEpi>(op, args, stream, out_channels);              \
      if (ksplit == 4) return launch_gemm<BN_, 4, kEpi>(op, args, stream, out_channels);              \
      if (ksplit == 2) return launch_gemm<BN_, 2, kEpi>(op, args, stream, out_channels);              \
    }                                                                                                 \
    return launch_gemm<BN_, 1, kEpi>(op, args, stream, out_channels);                                 \
  } while (0)
  if (bn == 16) ATOM_BN(16);
  if (bn == 32) ATOM_BN(32);
  if (bn == 64) ATOM_BN(64);
  if constexpr (kEpi == atom::EPI_GATEUP || kEpi == atom::EPI_PUSH) return fail(ATOM_E_UNSUPPORTED, "gemm_i4: decode batches only (M <= 64)");
  else ATOM_BN(128);
#undef ATOM_BN
}

int gemm_common(const void* a, const void* b, const void* a_scale, const void* b_scale, const void* a_keeper,
                const void* b_keeper, const void* a_keeper_scale, const void* b_keeper_scale, void* d, void* d_scale,
                int64_t M, int64_t N, int64_t K, uint32_t flags, void* stream, bool o4, const atom::ArArgs* ar = nullptr) {
  ATOM_REQUIRE(a && b && a_scale && b_scale && a_keeper && b_keeper && a_keeper_scale && b_keeper_scale && (d || ar),
               "gemm_i4: null pointer argument");
  ATOM_REQUIRE(M > 0 && N > 0, "gemm_i4: M=%lld N=%lld must be positive", (long long)M, (long long)N);
  ATOM_REQUIRE(K >= 256 && K % 128 == 0, "gemm_i4: K=%lld must be a multiple of 128 and >= 256 (INT4 groups + 128 keeper)", (long long)K);
  ATOM_REQUIRE(N % 8 == 0, "gemm_i4: N=%lld must be a multiple of 8", (long long)N);
  ATOM_REQUIRE(!o4 || (N % 128 == 0 && d_scale), "gemm_i4_o4: N=%lld must be a multiple of 128 (one head per scale)", (long long)N);
  ATOM_REQUIRE(aligned16(a) && aligned16(b) && aligned16(a_keeper) && aligned16(b_keeper) && aligned16(d),
               "gemm_i4: operand pointers must be 16-byte aligned");
  if (ar != nullptr) {
    ATOM_REQUIRE(!o4 && M <= 64, "gemm_i4_o16_push: decode batches only (M=%lld <= 64), fp16 output", (long long)M);
    ATOM_REQUIRE(ar->bufs && ar->state && ar->world >= 1 && ar->world <= 32 && ar->rank >= 0 && ar->rank < ar->world && ar->slot % 8 == 0 &&
                 M * N <= ar->slot, "gemm_i4_o16_push: rank=%d world=%d, M x N = %lld must fit a slot of %lld elements", ar->rank, ar->world,
                 (long long)(M * N), (long long)ar->slot);
    flags &= ~ATOM_GEMM_FORCE_TALL;
  }
  ATOM_REQUIRE(aligned16(b_scale) && aligned16(b_keeper_scale), "gemm_i4: weight scale pointers must be 16-byte aligned");
  ATOM_REQUIRE((reinterpret_cast<uintptr_t>(a_scale) & 3) == 0 && (reinterpret_cast<uintptr_t>(a_keeper_scale) & 3) == 0,
               "gemm_i4: activation scale pointers must be 4-byte aligned");
  ATOM_REQUIRE(M < (1ll << 31) && N < (1ll << 31) && K < (1ll << 24), "gemm_i4: dimension too large");
  GemmOperands op{a, b, a_keeper, b_keeper, M, N, K};
  atom::GemmArgs args{};
  args.a_scale = (const __half*)a_scale; args.b_scale = (const __half*)b_scale;
  args.a_keeper_scale = (const __half*)a_keeper_scale; args.b_keeper_scale = (const __half*)b_keeper_scale;
  args.d = o4 ? nullptr : (__half*)d; args.d4 = o4 ? (uint8_t*)d : nullptr; args.d_scale = (__half2*)d_scale;
  args.M = (int)M; args.N = (int)N; args.G = (int)(K / 128 - 1); args.lda_scale = atom::scale_size((int)M); args.trace = g_trace;
  args.ldb_scale = (int)N;
  if (ar != nullptr) { args.ar = *ar; return gemm_dispatch<atom::EPI_PUSH>(op, args, flags, (cudaStream_t)stream); }
  return o4 ? gemm_dispatch<atom::EPI_O4>(op, args, flags, (cudaStream_t)stream) : gemm_dispatch<atom::EPI_O16>(op, args, flags, (cudaStream_t)stream);
}

int quant_check(const char* what, int seq_len, int hidden, const void* o8, const void* o4, const void* s8, const void* s4) {
  ATOM_REQUIRE(seq_len > 0, "%s: seq_len=%d must be positive", what, seq_len);
  ATOM_REQUIRE(hidden >= 256 && hidden % 128 == 0 && hidden <= 65536, "%s: hidden_dim=%d must be a multiple of 128 in [256, 65536]", what, hidden);
  ATOM_REQUIRE(o8 && o4 && s8 && s4, "%s: null output pointer", what);
  return ATOM_OK;
}

}  // namespace

extern "C" {

int atom_version(void) { return 100; }
const char* atom_last_error(void) { return g_err.c_str(); }
int atom_scale_index(int row) { return atom::scale_index(row); }
int atom_scale_size(int rows) { return atom::scale_size(rows); }
int atom_gemm_set_trace(void* device_buffer) { g_trace = (unsigned long long*)device_buffer; return ATOM_OK; }
int atom_set_pdl(int enable) { g_pdl = enable ? 1 : 0; return ATOM_OK; }

int atom_reorder_fp16_i4(const void* hidden, const void* reorder_index, int seq_len, int hidden_dim, void* o_outliers,
                         void* o_norms, void* outlier_scales, void* norm_scales, void* stream) {
  int rc = quant_check("reorder_fp16_i4", seq_len, hidden_dim, o_outliers, o_norms, outlier_scales, norm_scales);
  if (rc) return rc;
  ATOM_REQUIRE(hidden && reorder_index && aligned16(hidden), "reorder_fp16_i4: null or misaligned input");
  if ((rc = ensure_dynamic_smem(atom::reorder_quant_kernel, 65536 * 2, "reorder_fp16_i4"))) return rc;   // one fp16 row, hidden <= 65536
  return launch_k("reorder_fp16_i4", atom::reorder_quant_kernel, dim3(seq_len), dim3(atom::QUANT_THREADS), (size_t)hidden_dim * 2,
                  (cudaStream_t)stream, (const __half*)hidden, (const int16_t*)reorder_index, seq_len, hidden_dim, (int8_t*)o_outliers,
                  (uint8_t*)o_norms, (__half*)outlier_scales, (__half*)norm_scales, atom::scale_size(seq_len));
}

int atom_rmsnorm_fp16_i4(const void* hidden, const void* weight, float eps, const void* reorder_index, int seq_len,
                         int hidden_dim, void* o_outliers, void* o_norms, void* outlier_scales, void* norm_scales,
                         void* stream) {
  int rc = quant_check("rmsnorm_fp16_i4", seq_len, hidden_dim, o_outliers, o_norms, outlier_scales, norm_scales);
  if (rc) return rc;
  ATOM_REQUIRE(hidden && weight && reorder_index && aligned16(hidden) && aligned16(weight), "rmsnorm_fp16_i4: null or misaligned input");
  ATOM_REQUIRE(hidden_dim <= 32768, "rmsnorm_fp16_i4: hidden_dim=%d > 32768 unsupported", hidden_dim);
  if ((rc = ensure_dynamic_smem(atom::rmsnorm_quant_kernel<false>, 32768 * 4 + 512, "rmsnorm_fp16_i4"))) return rc;   // row + weight (fp16) + reduction scratch
  return launch_k("rmsnorm_fp16_i4", atom::rmsnorm_quant_kernel<false>, dim3(seq_len), dim3(atom::QUANT_THREADS), (size_t)hidden_dim * 4 + 512,
                  (cudaStream_t)stream, (const __half*)hidden, (const __half*)nullptr, (__half*)nullptr, (const __half*)weight, eps,
                  (const int16_t*)reorder_index, seq_len, hidden_dim, (int8_t*)o_outliers, (uint8_t*)o_norms, (__half*)outlier_scales,
                  (__half*)norm_scales, atom::scale_size(seq_len), atom::ArArgs{});
}

int atom_add_rmsnorm_fp16_i4(const void* hidden, const void* residual, void* sum_out, const void* weight, float eps,
                             const void* reorder_index, int seq_len, int hidden_dim, void* o_outliers, void* o_norms,
                             void* outlier_scales, void* norm_scales, void* stream) {
  int rc = quant_check("add_rmsnorm_fp16_i4", seq_len, hidden_dim, o_outliers, o_norms, outlier_scales, norm_scales);
  if (rc) return rc;
  ATOM_REQUIRE(hidden && residual && sum_out && weight && reorder_index && aligned16(hidden) && aligned16(residual) && aligned16(sum_out) &&
               aligned16(weight), "add_rmsnorm_fp16_i4: null or misaligned input");
  ATOM_REQUIRE(hidden_dim <= 32768, "add_rmsnorm_fp16_i4: hidden_dim=%d > 32768 unsupported", hidden_dim);
  if ((rc = ensure_dynamic_smem(atom::rmsnorm_quant_kernel<false>, 32768 * 4 + 512, "add_rmsnorm_fp16_i4"))) return rc;
  return launch_k("add_rmsnorm_fp16_i4", atom::rmsnorm_quant_kernel<false>, dim3(seq_len), dim3(atom::QUANT_THREADS), (size_t)hidden_dim * 4 + 512,
                  (cudaStream_t)stream, (const __half*)hidden, (const __half*)residual, (__half*)sum_out, (const __half*)weight, eps,
                  (const int16_t*)reorder_index, seq_len, hidden_dim, (int8_t*)o_outliers, (uint8_t*)o_norms, (__half*)outlier_scales,
                  (__half*)norm_scales, atom::scale_size(seq_len), atom::ArArgs{});
}

// reduce half of the fused all-reduce: `hidden` is the sum over the ranks of what atom_gemm_i4_o16_push stored in the receive buffers
int atom_reduce_add_rmsnorm_fp16_i4(const void* peer_buffers, void* state, int64_t slot_elems, int rank, int world, const void* residual,
                                    void* sum_out, const void* weight, float eps, const void* reorder_index, int seq_len, int hidden_dim,
                                    void* o_outliers, void* o_norms, void* outlier_scales, void* norm_scales, void* stream) {
  int rc = quant_check("reduce_add_rmsnorm_fp16_i4", seq_len, hidden_dim, o_outliers, o_norms, outlier_scales, norm_scales);
  if (rc) return rc;
  ATOM_REQUIRE(peer_buffers && state && residual && sum_out && weight && reorder_index && aligned16(residual) && aligned16(sum_out) &&
               aligned16(weight), "reduce_add_rmsnorm_fp16_i4: null or misaligned input");
  ATOM_REQUIRE(hidden_dim <= 32768 && hidden_dim % 1024 == 0, "reduce_add_rmsnorm_fp16_i4: hidden_dim=%d must be a multiple of 1024, at most 32768", hidden_dim);
  ATOM_REQUIRE(world >= 1 && world <= 32 && rank >= 0 && rank < world && slot_elems % 8 == 0 && (int64_t)seq_len * hidden_dim <= slot_elems,
               "reduce_add_rmsnorm_fp16_i4: rank=%d world=%d, %d x %d must fit a slot of %lld elements", rank, world, seq_len, hidden_dim, (long long)slot_elems);
  if ((rc = ensure_dynamic_smem(atom::rmsnorm_quant_kernel<true>, 32768 * 4 + 512, "reduce_add_rmsnorm_fp16_i4"))) return rc;
  atom::ArArgs ar{(void* const*)peer_buffers, (uint32_t*)state, (long long)slot_elems, rank, world};
  return launch_k("reduce_add_rmsnorm_fp16_i4", atom::rmsnorm_quant_kernel<true>, dim3(seq_len), dim3(atom::QUANT_THREADS), (size_t)hidden_dim * 4 + 512,
                  (cudaStream_t)stream, (const __half*)nullptr, (const __half*)residual, (__half*)sum_out, (const __half*)weight, eps,
                  (const int16_t*)reorder_index, seq_len, hidden_dim, (int8_t*)o_outliers, (uint8_t*)o_norms, (__half*)outlier_scales,
                  (__half*)norm_scales, atom::scale_size(seq_len), ar);
}

int atom_activate_fp16_i4(const void* a, const void* b, int seq_len, int hidden_dim, void* o_outliers, void* o_norms,
                          void* outlier_scales, void* norm_scales, void* stream) {
  int rc = quant_check("activate_fp16_i4", seq_len, hidden_dim, o_outliers, o_norms, outlier_scales, norm_scales);
  if (rc) return rc;
  ATOM_REQUIRE(a && b && aligned16(a) && aligned16(b), "activate_fp16_i4: null or misaligned input");
  const long long units = (long long)seq_len * (hidden_dim / 128);
  return launch_k("activate_fp16_i4", atom::activate_quant_kernel, dim3((unsigned)((units + 7) / 8)), dim3(256), 0, (cudaStream_t)stream,
                  (const __half*)a, (const __half*)b, seq_len, hidden_dim, (int8_t*)o_outliers, (uint8_t*)o_norms,
                  (__half*)outlier_scales, (__half*)norm_scales, atom::scale_size(seq_len));
}

int atom_gemm_i4_o16(const void* a, const void* b, const void* a_scale, const void* b_scale, const void* a_keeper,
                     const void* b_keeper, const void* a_keeper_scale, const void* b_keeper_scale, void* d, int64_t M,
                     int64_t N, int64_t K, uint32_t flags, void* stream) {
  return gemm_common(a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale, d, nullptr, M, N, K,
                     flags, stream, false);
}

// push half of the fused all-reduce (row-parallel projection): D is stored into every rank's receive buffer
int atom_gemm_i4_o16_push(const void* a, const void* b, const void* a_scale, const void* b_scale, const void* a_keeper,
                          const void* b_keeper, const void* a_keeper_scale, const void* b_keeper_scale, const void* peer_buffers,
                          void* state, int64_t slot_elems, int rank, int world, int64_t M, int64_t N, int64_t K, uint32_t flags,
                          void* stream) {
  atom::ArArgs ar{(void* const*)peer_buffers, (uint32_t*)state, (long long)slot_elems, rank, world};
  return gemm_common(a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale, nullptr, nullptr, M, N, K, flags,
                     stream, false, &ar);
}

// q rows [0, Hq), k rows [Hq, Hq + Hkv), v the rest: one launch, (Hq + 2 Hkv) / 128 channel tiles, the tile index selects the
// epilogue (q: FP16, k / v: asymmetric INT4 per head)
static int gemm_qkv(const char* what, const void* a, const void* b_qkv, const void* a_scale, const void* b_scale_qkv, const void* a_keeper,
                    const void* b_keeper_qkv, const void* a_keeper_scale, const void* b_keeper_scale_qkv, void* q, void* k,
                    void* k_scale, void* v, void* v_scale, int64_t M, int64_t Hq, int64_t Hkv, int64_t K, uint32_t flags, void* stream) {
  ATOM_REQUIRE(a && b_qkv && a_scale && b_scale_qkv && a_keeper && b_keeper_qkv && a_keeper_scale && b_keeper_scale_qkv && q && k &&
               k_scale && v && v_scale, "%s: null pointer argument", what);
  ATOM_REQUIRE(K >= 256 && K % 128 == 0, "%s: K=%lld must be a multiple of 128 and >= 256", what, (long long)K);
  ATOM_REQUIRE(aligned16(a) && aligned16(b_qkv) && aligned16(a_keeper) && aligned16(b_keeper_qkv) && aligned16(q) && aligned16(b_scale_qkv) &&
               aligned16(b_keeper_scale_qkv), "%s: operand pointers must be 16-byte aligned", what);
  const int64_t N = Hq + 2 * Hkv;
  ATOM_REQUIRE(M < (1ll << 31) && N < (1ll << 31) && K < (1ll << 24), "%s: dimension too large", what);
  GemmOperands op{a, b_qkv, a_keeper, b_keeper_qkv, M, N, K};
  atom::GemmArgs args{};
  args.a_scale = (const __half*)a_scale; args.a_keeper_scale = (const __half*)a_keeper_scale;
  args.b_scale = (const __half*)b_scale_qkv; args.b_keeper_scale = (const __half*)b_keeper_scale_qkv;
  args.M = (int)M; args.N = (int)N; args.G = (int)(K / 128 - 1); args.lda_scale = atom::scale_size((int)M); args.trace = g_trace;
  args.ldb_scale = (int)N; args.seg_tiles = (int)(Hq / 128); args.kv_tiles = (int)(Hkv / 128);
  args.d = (__half*)q; args.d4 = (uint8_t*)k; args.d_scale = (__half2*)k_scale; args.d4_v = (uint8_t*)v; args.d_scale_v = (__half2*)v_scale;
  return gemm_dispatch<atom::EPI_QKV>(op, args, flags, (cudaStream_t)stream);
}

int atom_gemm_i4_qkv(const void* a, const void* b_qkv, const void* a_scale, const void* b_scale_qkv, const void* a_keeper,
                     const void* b_keeper_qkv, const void* a_keeper_scale, const void* b_keeper_scale_qkv, void* q, void* k,
                     void* k_scale, void* v, void* v_scale, int64_t M, int64_t H, int64_t K, uint32_t flags, void* stream) {
  ATOM_REQUIRE(M > 0 && H > 0 && H % 128 == 0, "gemm_i4_qkv: M=%lld must be positive, H=%lld a positive multiple of 128", (long long)M, (long long)H);
  return gemm_qkv("gemm_i4_qkv", a, b_qkv, a_scale, b_scale_qkv, a_keeper, b_keeper_qkv, a_keeper_scale, b_keeper_scale_qkv, q, k, k_scale,
                  v, v_scale, M, H, H, K, flags, stream);
}

int atom_gemm_i4_qkv_gqa(const void* a, const void* b_qkv, const void* a_scale, const void* b_scale_qkv, const void* a_keeper,
                         const void* b_keeper_qkv, const void* a_keeper_scale, const void* b_keeper_scale_qkv, void* q, void* k,
                         void* k_scale, void* v, void* v_scale, int64_t M, int64_t Hq_dim, int64_t Hkv_dim, int64_t K, uint32_t flags,
                         void* stream) {
  ATOM_REQUIRE(M > 0 && Hq_dim > 0 && Hq_dim % 128 == 0 && Hkv_dim > 0 && Hkv_dim % 128 == 0,
               "gemm_i4_qkv_gqa: M=%lld must be positive, Hq_dim=%lld and Hkv_dim=%lld positive multiples of 128", (long long)M,
               (long long)Hq_dim, (long long)Hkv_dim);
  ATOM_REQUIRE(Hq_dim % Hkv_dim == 0, "gemm_i4_qkv_gqa: Hq_dim=%lld must be a multiple of Hkv_dim=%lld (whole query heads per KV head)",
               (long long)Hq_dim, (long long)Hkv_dim);
  return gemm_qkv("gemm_i4_qkv_gqa", a, b_qkv, a_scale, b_scale_qkv, a_keeper, b_keeper_qkv, a_keeper_scale, b_keeper_scale_qkv, q, k,
                  k_scale, v, v_scale, M, Hq_dim, Hkv_dim, K, flags, stream);
}

int atom_gemm_i4_gateup_act(const void* a, const void* b_gu, const void* a_scale, const void* b_scale_gu, const void* a_keeper,
                            const void* b_keeper_gu, const void* a_keeper_scale, const void* b_keeper_scale_gu, void* o_outliers,
                            void* o_norms, void* outlier_scales, void* norm_scales, int64_t M, int64_t I, int64_t K, uint32_t flags,
                            void* stream) {
  ATOM_REQUIRE(a && b_gu && a_scale && b_scale_gu && a_keeper && b_keeper_gu && a_keeper_scale && b_keeper_scale_gu && o_outliers &&
               o_norms && outlier_scales && norm_scales, "gemm_i4_gateup_act: null pointer argument");
  ATOM_REQUIRE(M > 0 && I >= 256 && I % 128 == 0, "gemm_i4_gateup_act: M=%lld must be positive, I=%lld a multiple of 128 >= 256", (long long)M, (long long)I);
  ATOM_REQUIRE(K >= 256 && K % 128 == 0, "gemm_i4_gateup_act: K=%lld must be a multiple of 128 and >= 256", (long long)K);
  ATOM_REQUIRE(aligned16(a) && aligned16(b_gu) && aligned16(a_keeper) && aligned16(b_keeper_gu) && aligned16(b_scale_gu) &&
               aligned16(b_keeper_scale_gu), "gemm_i4_gateup_act: operand pointers must be 16-byte aligned");
  ATOM_REQUIRE(2 * I < (1ll << 31) && K < (1ll << 24), "gemm_i4_gateup_act: dimension too large");
  if (M > 64) return fail(ATOM_E_UNSUPPORTED, "gemm_i4_gateup_act: fused epilogue exists for decode batches (M <= 64) only; "
                                              "run the two projections and activate_fp16_i4 for M=%lld", (long long)M);
  GemmOperands op{a, b_gu, a_keeper, b_keeper_gu, M, 2 * I, K};
  atom::GemmArgs args{};
  args.a_scale = (const __half*)a_scale; args.a_keeper_scale = (const __half*)a_keeper_scale;
  args.b_scale = (const __half*)b_scale_gu; args.b_keeper_scale = (const __half*)b_keeper_scale_gu;
  args.M = (int)M; args.N = (int)(2 * I); args.G = (int)(K / 128 - 1); args.lda_scale = atom::scale_size((int)M); args.trace = g_trace;
  args.ldb_scale = (int)(2 * I); args.gu_rows = (int)I;
  args.q8_out = (int8_t*)o_outliers; args.q4_out = (uint8_t*)o_norms; args.q8_scale = (__half*)outlier_scales; args.q4_scale = (__half*)norm_scales;
  return gemm_dispatch<atom::EPI_GATEUP>(op, args, flags & ~(uint32_t)ATOM_GEMM_FORCE_TALL, (cudaStream_t)stream, I);
}

int atom_gemm_i4_o4(const void* a, const void* b, const void* a_scale, const void* b_scale, const void* a_keeper,
                    const void* b_keeper, const void* a_keeper_scale, const void* b_keeper_scale, void* d,
                    void* d_scale, int64_t M, int64_t N, int64_t K, uint32_t flags, void* stream) {
  return gemm_common(a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale, d, d_scale, M, N, K,
                     flags, stream, true);
}

static int prefill_attention(const char* what, const void* q, const void* k, const void* k_param, const void* v, const void* v_param,
                             const void* seqlen_indptr, const void* pos_of_token, const void* rope_table, void* k_f16, void* v_f16,
                             void* out, int total_tokens, int batch_size, int max_len, int num_heads, int num_kv_heads, void* stream) {
  ATOM_REQUIRE(q && k && k_param && v && v_param && seqlen_indptr && pos_of_token && rope_table && k_f16 && v_f16 && out,
               "%s: null pointer argument", what);
  ATOM_REQUIRE(batch_size > 0 && num_heads > 0 && max_len > 0, "%s: batch_size=%d num_heads=%d max_len=%d must be positive", what,
               batch_size, num_heads, max_len);
  ATOM_REQUIRE(num_kv_heads > 0 && num_heads % num_kv_heads == 0, "%s: num_q_heads=%d must be a positive multiple of num_kv_heads=%d", what,
               num_heads, num_kv_heads);
  ATOM_REQUIRE(aligned16(q) && aligned16(k) && aligned16(v) && aligned16(k_f16) && aligned16(v_f16) && aligned16(out),
               "%s: pointers must be 16-byte aligned", what);
  if (total_tokens <= 0) return ATOM_OK;
  const long long th = (long long)total_tokens * num_kv_heads;
  atom::kv_dequant_rope_kernel<<<(unsigned)((th + 3) / 4), 256, 0, (cudaStream_t)stream>>>(
      (const uint8_t*)k, (const __half2*)k_param, (const uint8_t*)v, (const __half2*)v_param, (const int32_t*)pos_of_token,
      (const float2*)rope_table, (__half*)k_f16, (__half*)v_f16, th, num_kv_heads);
  int rc = check_launch("prefill_attention_i4 (dequant + RoPE)");
  if (rc) return rc;
  const dim3 grid((unsigned)((max_len + atom::PF_BQ - 1) / atom::PF_BQ), (unsigned)batch_size, (unsigned)num_heads);
  atom::prefill_attn_kernel<<<grid, atom::PF_THREADS, 0, (cudaStream_t)stream>>>(
      (const __half*)q, (const __half*)k_f16, (const __half*)v_f16, (const int32_t*)seqlen_indptr, (const float2*)rope_table,
      (__half*)out, num_heads, num_kv_heads, 0.08838834764831845f * 1.4426950408889634f);
  return check_launch(what);
}

int atom_prefill_attention_i4(const void* q, const void* k, const void* k_param, const void* v, const void* v_param,
                              const void* seqlen_indptr, const void* pos_of_token, const void* rope_table, void* k_f16, void* v_f16,
                              void* out, int total_tokens, int batch_size, int max_len, int num_heads, void* stream) {
  return prefill_attention("prefill_attention_i4", q, k, k_param, v, v_param, seqlen_indptr, pos_of_token, rope_table, k_f16, v_f16, out,
                           total_tokens, batch_size, max_len, num_heads, num_heads, stream);
}

int atom_prefill_attention_gqa_i4(const void* q, const void* k, const void* k_param, const void* v, const void* v_param,
                                  const void* seqlen_indptr, const void* pos_of_token, const void* rope_table, void* k_f16, void* v_f16,
                                  void* out, int total_tokens, int batch_size, int max_len, int num_q_heads, int num_kv_heads,
                                  void* stream) {
  return prefill_attention("prefill_attention_gqa_i4", q, k, k_param, v, v_param, seqlen_indptr, pos_of_token, rope_table, k_f16, v_f16,
                           out, total_tokens, batch_size, max_len, num_q_heads, num_kv_heads, stream);
}

int atom_allreduce_push_f16(const void* in, void* out, const void* peer_buffers, void* state, int64_t numel, int64_t slot_elems,
                            int rank, int world, void* stream) {
  ATOM_REQUIRE(in && out && peer_buffers && state, "allreduce_push_f16: null pointer argument");
  ATOM_REQUIRE(world >= 1 && world <= 32 && rank >= 0 && rank < world, "allreduce_push_f16: rank=%d world=%d", rank, world);
  ATOM_REQUIRE(numel > 0 && numel % 8 == 0 && numel <= slot_elems && slot_elems % 8 == 0,
               "allreduce_push_f16: numel=%lld must be a positive multiple of 8 and fit a slot of %lld elements", (long long)numel, (long long)slot_elems);
  ATOM_REQUIRE(aligned16(in) && aligned16(out), "allreduce_push_f16: in / out must be 16-byte aligned");
  atom::ArArgs ar{(void* const*)peer_buffers, (uint32_t*)state, (long long)slot_elems, rank, world};
  atom::allreduce_push_kernel<<<atom::AR_CTAS, atom::AR_THREADS, 0, (cudaStream_t)stream>>>((const uint4*)in, (uint4*)out, ar, numel / 8);
  return check_launch("allreduce_push_f16");
}

int atom_allreduce_state_words(void) { return atom::AR_STATE_WORDS; }

static int kv_check(const char* what, const void* data, const void* param, const void* indptr, const void* indices,
                    const void* last, int L, int layer, int H, int P, int B) {
  ATOM_REQUIRE(data && param && indptr && indices && last, "%s: null pointer argument", what);
  ATOM_REQUIRE(L > 0 && layer >= 0 && layer < L, "%s: layer_idx=%d out of range [0,%d)", what, layer, L);
  ATOM_REQUIRE(H > 0 && P > 0 && B > 0, "%s: num_heads=%d page_size=%d batch_size=%d must be positive", what, H, P, B);
  return ATOM_OK;
}

int atom_batch_decode_i4(void* o, const void* q, const void* kv_data, const void* kv_param, const void* kv_indptr,
                         const void* kv_indices, const void* last_page_offset, int num_layers, int layer_idx,
                         int num_heads, int page_size, int batch_size, void* stream) {
  int rc = kv_check("batch_decode_i4", kv_data, kv_param, kv_indptr, kv_indices, last_page_offset, num_layers, layer_idx,
                    num_heads, page_size, batch_size);
  if (rc) return rc;
  ATOM_REQUIRE(o && q, "batch_decode_i4: null q/o");
  ATOM_REQUIRE(page_size % 8 == 0 && page_size <= 64, "batch_decode_i4: page_size=%d must be a multiple of 8, at most 64", page_size);
  ATOM_REQUIRE(aligned16(kv_data) && aligned16(kv_param), "batch_decode_i4: KV pool must be 16-byte aligned");
  atom::KvArgs kv{(uint8_t*)kv_data, (__half2*)kv_param, (const int32_t*)kv_indptr, (const int32_t*)kv_indices,
                  (const int32_t*)last_page_offset, num_layers, layer_idx, num_heads, page_size, batch_size};
  const size_t smem = atom::batch_decode_smem_bytes(page_size);
#define ATOM_DECODE(TPL, PG)                                                                                              \
  do {                                                                                                                    \
    if ((rc = ensure_dynamic_smem(atom::batch_decode_kernel<TPL, PG>, 100 * 1024, "batch_decode_i4"))) return rc;         \
    return launch_k("batch_decode_i4", atom::batch_decode_kernel<TPL, PG>, dim3(batch_size, num_heads),                   \
                    dim3(atom::DEC_THREADS), smem, (cudaStream_t)stream, (__half*)o, (const __half*)q, kv);               \
  } while (0)
  if (page_size == 16) ATOM_DECODE(2, 16);      // the two page sizes of the harness / the reference benchmarks: strides as immediates
  if (page_size == 32) ATOM_DECODE(4, 32);
  if (page_size <= 32) ATOM_DECODE(4, 0);
  ATOM_DECODE(8, 0);
#undef ATOM_DECODE
}

int atom_batch_decode_gqa_i4(void* o, const void* q, const void* kv_data, const void* kv_param, const void* kv_indptr,
                             const void* kv_indices, const void* last_page_offset, int num_layers, int layer_idx,
                             int num_q_heads, int num_kv_heads, int page_size, int batch_size, float rope_theta, void* stream) {
  int rc = kv_check("batch_decode_gqa_i4", kv_data, kv_param, kv_indptr, kv_indices, last_page_offset, num_layers, layer_idx,
                    num_kv_heads, page_size, batch_size);
  if (rc) return rc;
  ATOM_REQUIRE(o && q, "batch_decode_gqa_i4: null q/o");
  ATOM_REQUIRE(num_q_heads > 0 && num_q_heads % num_kv_heads == 0,
               "batch_decode_gqa_i4: num_q_heads=%d must be a positive multiple of num_kv_heads=%d", num_q_heads, num_kv_heads);
  ATOM_REQUIRE(rope_theta > 1.f && rope_theta < 1e30f, "batch_decode_gqa_i4: rope_theta=%g must be a finite base above 1", (double)rope_theta);
  const int group = num_q_heads / num_kv_heads;
  // multi-head attention with the reference's RoPE base: the kernel every existing caller runs, untouched
  if (group == 1 && rope_theta == 10000.f)
    return atom_batch_decode_i4(o, q, kv_data, kv_param, kv_indptr, kv_indices, last_page_offset, num_layers, layer_idx, num_kv_heads,
                                page_size, batch_size, stream);
  if (group != 1 && group != 2 && group != 4 && group != 8)
    return fail(ATOM_E_UNSUPPORTED, "batch_decode_gqa_i4: %d query heads per KV head (num_q_heads=%d, num_kv_heads=%d); supported group "
                                    "sizes are 1, 2, 4 and 8", group, num_q_heads, num_kv_heads);
  ATOM_REQUIRE(page_size % 8 == 0 && page_size <= 64, "batch_decode_gqa_i4: page_size=%d must be a multiple of 8, at most 64", page_size);
  ATOM_REQUIRE(aligned16(kv_data) && aligned16(kv_param), "batch_decode_gqa_i4: KV pool must be 16-byte aligned");
  atom::KvArgs kv{(uint8_t*)kv_data, (__half2*)kv_param, (const int32_t*)kv_indptr, (const int32_t*)kv_indices,
                  (const int32_t*)last_page_offset, num_layers, layer_idx, num_kv_heads, page_size, batch_size};
  const size_t smem = atom::batch_decode_gqa_smem_bytes(page_size);
  const float log2_theta = log2f(rope_theta);
#define ATOM_DECODE_GQA(G_, TPL, PG)                                                                                         \
  do {                                                                                                                       \
    if ((rc = ensure_dynamic_smem(atom::batch_decode_gqa_kernel<G_, TPL, PG>, 100 * 1024, "batch_decode_gqa_i4"))) return rc; \
    return launch_k("batch_decode_gqa_i4", atom::batch_decode_gqa_kernel<G_, TPL, PG>, dim3(batch_size, num_kv_heads),       \
                    dim3(atom::GQA_THREADS), smem, (cudaStream_t)stream, (__half*)o, (const __half*)q, kv, log2_theta);      \
  } while (0)
#define ATOM_DECODE_GQA_P(G_)                    \
  do {                                           \
    if (page_size == 16) ATOM_DECODE_GQA(G_, 2, 16); \
    if (page_size == 32) ATOM_DECODE_GQA(G_, 4, 32); \
    ATOM_DECODE_GQA(G_, 8, 0);                   \
  } while (0)
  if (group == 1) ATOM_DECODE_GQA(1, 8, 0);       // multi-head attention with another RoPE base: eight page stripes, any page size
  if (group == 2) ATOM_DECODE_GQA_P(2);
  if (group == 4) ATOM_DECODE_GQA_P(4);
  ATOM_DECODE_GQA_P(8);
#undef ATOM_DECODE_GQA_P
#undef ATOM_DECODE_GQA
}

int atom_append_kv_i4(void* kv_data, void* kv_param, const void* kv_indptr, const void* kv_indices,
                      const void* last_page_offset, const void* k, const void* v, const void* k_param,
                      const void* v_param, int num_layers, int layer_idx, int num_heads, int page_size, int batch_size,
                      void* stream) {
  int rc = kv_check("append_kv_i4", kv_data, kv_param, kv_indptr, kv_indices, last_page_offset, num_layers, layer_idx,
                    num_heads, page_size, batch_size);
  if (rc) return rc;
  ATOM_REQUIRE(k && v && k_param && v_param, "append_kv_i4: null k/v");
  atom::KvArgs kv{(uint8_t*)kv_data, (__half2*)kv_param, (const int32_t*)kv_indptr, (const int32_t*)kv_indices,
                  (const int32_t*)last_page_offset, num_layers, layer_idx, num_heads, page_size, batch_size};
  const long long threads = (long long)batch_size * num_heads * 16;
  return launch_k("append_kv_i4", atom::append_kv_kernel, dim3((unsigned)((threads + 255) / 256)), dim3(256), 0, (cudaStream_t)stream, kv,
                  (const uint8_t*)k, (const uint8_t*)v, (const __half2*)k_param, (const __half2*)v_param,
                  (const int32_t*)nullptr, batch_size);
}

int atom_init_kv_i4(void* kv_data, void* kv_param, const void* kv_indptr, const void* kv_indices,
                    const void* last_page_offset, const void* k, const void* v, const void* k_param,
                    const void* v_param, const void* seqlen_indptr, int total_tokens, int num_layers, int layer_idx,
                    int num_heads, int page_size, int batch_size, void* stream) {
  int rc = kv_check("init_kv_i4", kv_data, kv_param, kv_indptr, kv_indices, last_page_offset, num_layers, layer_idx,
                    num_heads, page_size, batch_size);
  if (rc) return rc;
  ATOM_REQUIRE(k && v && k_param && v_param && seqlen_indptr, "init_kv_i4: null k/v/seqlen_indptr");
  if (total_tokens <= 0) return ATOM_OK;
  atom::KvArgs kv{(uint8_t*)kv_data, (__half2*)kv_param, (const int32_t*)kv_indptr, (const int32_t*)kv_indices,
                  (const int32_t*)last_page_offset, num_layers, layer_idx, num_heads, page_size, batch_size};
  const long long threads = (long long)total_tokens * num_heads * 16;
  return launch_k("init_kv_i4", atom::append_kv_kernel, dim3((unsigned)((threads + 255) / 256)), dim3(256), 0, (cudaStream_t)stream, kv,
                  (const uint8_t*)k, (const uint8_t*)v, (const __half2*)k_param, (const __half2*)v_param,
                  (const int32_t*)seqlen_indptr, total_tokens);
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ sparse MoE block
namespace {

int64_t moe_tiles_max(int64_t slots, int64_t E, int bn) { return std::min(slots, (slots + E * (bn - 1)) / bn); }


// both grouped GEMMs: weights stacked over the experts, expert_rows rows each; a = the permuted activations of rows_cap rows
int gemm_grouped_check(const char* what, const void* a, const void* b, const void* a_scale, const void* b_scale,
                              const void* a_keeper, const void* b_keeper, const void* a_keeper_scale, const void* b_keeper_scale,
                              const void* tiles, int num_tiles, int token_tile, int64_t rows_cap, int64_t num_experts,
                              int64_t expert_rows, int64_t K) {
  ATOM_REQUIRE(a && b && a_scale && b_scale && a_keeper && b_keeper && a_keeper_scale && b_keeper_scale && tiles,
               "%s: null pointer argument", what);
  ATOM_REQUIRE(token_tile == 16 || token_tile == 32 || token_tile == 64, "%s: token_tile=%d must be 16, 32 or 64", what, token_tile);
  ATOM_REQUIRE(num_tiles > 0 && rows_cap == (int64_t)num_tiles * token_tile,
               "%s: rows_cap=%lld must be num_tiles=%d x token_tile=%d", what, (long long)rows_cap, num_tiles, token_tile);
  ATOM_REQUIRE(num_experts >= 1 && num_experts <= atom::MOE_MAX_EXPERTS, "%s: num_experts=%lld must be in [1, 64]", what,
               (long long)num_experts);
  ATOM_REQUIRE(K >= 256 && K % 128 == 0, "%s: K=%lld must be a multiple of 128 and >= 256", what, (long long)K);
  ATOM_REQUIRE(aligned16(a) && aligned16(b) && aligned16(a_keeper) && aligned16(b_keeper) && aligned16(b_scale) && aligned16(b_keeper_scale) &&
               aligned16(tiles), "%s: operand pointers must be 16-byte aligned", what);
  ATOM_REQUIRE((reinterpret_cast<uintptr_t>(a_scale) & 3) == 0 && (reinterpret_cast<uintptr_t>(a_keeper_scale) & 3) == 0,
               "%s: activation scale pointers must be 4-byte aligned", what);
  ATOM_REQUIRE(num_experts * expert_rows < (1ll << 31) && rows_cap < (1ll << 31) && K < (1ll << 24), "%s: dimension too large", what);
  return ATOM_OK;
}

template <int kEpi>
int gemm_grouped_dispatch(const GemmOperands& op, const atom::GemmArgs& args, int token_tile, int num_tiles, int64_t out_channels,
                                 cudaStream_t stream) {
  if (token_tile == 16) return launch_gemm<16, 1, kEpi | atom::EPI_GROUPED>(op, args, stream, out_channels, num_tiles);
  if (token_tile == 32) return launch_gemm<32, 1, kEpi | atom::EPI_GROUPED>(op, args, stream, out_channels, num_tiles);
  return launch_gemm<64, 1, kEpi | atom::EPI_GROUPED>(op, args, stream, out_channels, num_tiles);
}

}  // namespace

extern "C" {

int atom_moe_route_f16(const void* hidden, const void* norm_weight, float eps, const void* reorder_index, const void* router_weight,
                       int seq_len, int hidden_dim, int num_experts, int top_k, void* topk_ids, void* topk_weights,
                       void* router_logits, void* normed, void* stream) {
  ATOM_REQUIRE(hidden && norm_weight && reorder_index && router_weight && topk_ids && topk_weights, "moe_route_f16: null pointer argument");
  ATOM_REQUIRE(seq_len > 0, "moe_route_f16: seq_len=%d must be positive", seq_len);
  ATOM_REQUIRE(hidden_dim >= 256 && hidden_dim % 128 == 0 && hidden_dim <= 32768,
               "moe_route_f16: hidden_dim=%d must be a multiple of 128 in [256, 32768]", hidden_dim);
  ATOM_REQUIRE(num_experts >= 1 && num_experts <= atom::MOE_MAX_EXPERTS && top_k >= 1 && top_k <= std::min(num_experts, atom::MOE_MAX_TOPK),
               "moe_route_f16: num_experts=%d must be in [1, 64], top_k=%d in [1, min(num_experts, 8)]", num_experts, top_k);
  ATOM_REQUIRE(aligned16(hidden) && aligned16(norm_weight) && aligned16(router_weight) && (!normed || aligned16(normed)),
               "moe_route_f16: hidden, norm_weight, router_weight and normed must be 16-byte aligned");
  const size_t smem = (size_t)hidden_dim * 6 + (128 + atom::MOE_MAX_EXPERTS) * 4;
  int rc = ensure_dynamic_smem(atom::moe_route_kernel, 32768 * 6 + (128 + atom::MOE_MAX_EXPERTS) * 4, "moe_route_f16");
  if (rc) return rc;
  return launch_k("moe_route_f16", atom::moe_route_kernel, dim3(seq_len), dim3(atom::ROUTE_THREADS), smem, (cudaStream_t)stream,
                  (const __half*)hidden, (const __half*)norm_weight, (const int16_t*)reorder_index, eps, (const __half*)router_weight,
                  hidden_dim, num_experts, top_k, (int32_t*)topk_ids, (__half*)topk_weights, (float*)router_logits, (__half*)normed);
}

int atom_moe_plan(const void* topk_ids, int seq_len, int num_experts, int top_k, int token_tile, int tiles_max, void* dest_row,
                  void* tiles, void* stream) {
  ATOM_REQUIRE(topk_ids && dest_row && tiles, "moe_plan: null pointer argument");
  ATOM_REQUIRE(seq_len > 0 && num_experts >= 1 && num_experts <= atom::MOE_MAX_EXPERTS && top_k >= 1 &&
               top_k <= std::min(num_experts, atom::MOE_MAX_TOPK),
               "moe_plan: seq_len=%d must be positive, num_experts=%d in [1, 64], top_k=%d in [1, min(num_experts, 8)]", seq_len,
               num_experts, top_k);
  ATOM_REQUIRE(token_tile == 16 || token_tile == 32 || token_tile == 64, "moe_plan: token_tile=%d must be 16, 32 or 64", token_tile);
  const int64_t slots = (int64_t)seq_len * top_k;
  ATOM_REQUIRE(slots < (1ll << 30) && tiles_max >= moe_tiles_max(slots, num_experts, token_tile),
               "moe_plan: tiles_max=%d is below min(T*k, (T*k + E*(BN-1)) / BN) = %lld", tiles_max,
               (long long)moe_tiles_max(slots, num_experts, token_tile));
  ATOM_REQUIRE(aligned16(tiles), "moe_plan: tiles must be 16-byte aligned");
  return launch_k("moe_plan", atom::moe_plan_kernel, dim3(1), dim3(atom::PLAN_THREADS), 0, (cudaStream_t)stream,
                  (const int32_t*)topk_ids, (int)slots, num_experts, token_tile, tiles_max, (int32_t*)dest_row, (int4*)tiles);
}

int atom_moe_gather_i4(const void* o_outliers, const void* o_norms, const void* outlier_scales, const void* norm_scales, int seq_len,
                       int hidden_dim, int top_k, const void* dest_row, int rows_cap, void* p_outliers, void* p_norms,
                       void* p_outlier_scales, void* p_norm_scales, void* stream) {
  int rc = quant_check("moe_gather_i4", seq_len, hidden_dim, p_outliers, p_norms, p_outlier_scales, p_norm_scales);
  if (rc) return rc;
  ATOM_REQUIRE(o_outliers && o_norms && outlier_scales && norm_scales && dest_row, "moe_gather_i4: null input pointer");
  ATOM_REQUIRE(top_k >= 1 && top_k <= atom::MOE_MAX_TOPK && rows_cap > 0, "moe_gather_i4: top_k=%d must be in [1, 8], rows_cap=%d positive",
               top_k, rows_cap);
  ATOM_REQUIRE(aligned16(o_outliers) && aligned16(o_norms) && aligned16(p_outliers) && aligned16(p_norms),
               "moe_gather_i4: INT4 / INT8 rows must be 16-byte aligned");
  return launch_k("moe_gather_i4", atom::moe_gather_kernel, dim3((unsigned)(seq_len * top_k)), dim3(atom::GATHER_THREADS), 0,
                  (cudaStream_t)stream, (const int8_t*)o_outliers, (const uint8_t*)o_norms, (const __half*)outlier_scales,
                  (const __half*)norm_scales, hidden_dim, top_k, atom::scale_size(seq_len), (const int32_t*)dest_row, (int8_t*)p_outliers,
                  (uint8_t*)p_norms, (__half*)p_outlier_scales, (__half*)p_norm_scales, atom::scale_size(rows_cap));
}

int atom_gemm_i4_gateup_act_grouped(const void* a, const void* b_gu, const void* a_scale, const void* b_scale_gu, const void* a_keeper,
                                    const void* b_keeper_gu, const void* a_keeper_scale, const void* b_keeper_scale_gu, void* o_outliers,
                                    void* o_norms, void* outlier_scales, void* norm_scales, const void* tiles, int num_tiles,
                                    int token_tile, int64_t rows_cap, int64_t num_experts, int64_t I, int64_t K, void* stream) {
  int rc = gemm_grouped_check("gemm_i4_gateup_act_grouped", a, b_gu, a_scale, b_scale_gu, a_keeper, b_keeper_gu, a_keeper_scale,
                              b_keeper_scale_gu, tiles, num_tiles, token_tile, rows_cap, num_experts, 2 * I, K);
  if (rc) return rc;
  ATOM_REQUIRE(o_outliers && o_norms && outlier_scales && norm_scales, "gemm_i4_gateup_act_grouped: null output pointer");
  ATOM_REQUIRE(I >= 256 && I % 128 == 0, "gemm_i4_gateup_act_grouped: I=%lld must be a multiple of 128 >= 256", (long long)I);
  GemmOperands op{a, b_gu, a_keeper, b_keeper_gu, rows_cap, num_experts * 2 * I, K};
  atom::GemmArgs args{};
  args.a_scale = (const __half*)a_scale; args.a_keeper_scale = (const __half*)a_keeper_scale;
  args.b_scale = (const __half*)b_scale_gu; args.b_keeper_scale = (const __half*)b_keeper_scale_gu;
  args.M = (int)rows_cap; args.N = (int)(2 * I); args.G = (int)(K / 128 - 1); args.lda_scale = atom::scale_size((int)rows_cap);
  args.trace = g_trace; args.ldb_scale = (int)(2 * I); args.gu_rows = (int)I;
  args.q8_out = (int8_t*)o_outliers; args.q4_out = (uint8_t*)o_norms; args.q8_scale = (__half*)outlier_scales; args.q4_scale = (__half*)norm_scales;
  args.tiles = (const int4*)tiles; args.expert_rows = (int)(2 * I);
  return gemm_grouped_dispatch<atom::EPI_GATEUP>(op, args, token_tile, num_tiles, I, (cudaStream_t)stream);
}

int atom_gemm_i4_o16_grouped(const void* a, const void* b, const void* a_scale, const void* b_scale, const void* a_keeper,
                             const void* b_keeper, const void* a_keeper_scale, const void* b_keeper_scale, void* d, const void* tiles,
                             int num_tiles, int token_tile, int64_t rows_cap, int64_t num_experts, int64_t N, int64_t K, void* stream) {
  int rc = gemm_grouped_check("gemm_i4_o16_grouped", a, b, a_scale, b_scale, a_keeper, b_keeper, a_keeper_scale, b_keeper_scale, tiles,
                              num_tiles, token_tile, rows_cap, num_experts, N, K);
  if (rc) return rc;
  ATOM_REQUIRE(d && aligned16(d), "gemm_i4_o16_grouped: d must be a 16-byte aligned pointer");
  ATOM_REQUIRE(N > 0 && N % 8 == 0, "gemm_i4_o16_grouped: N=%lld must be a positive multiple of 8", (long long)N);
  GemmOperands op{a, b, a_keeper, b_keeper, rows_cap, num_experts * N, K};
  atom::GemmArgs args{};
  args.a_scale = (const __half*)a_scale; args.b_scale = (const __half*)b_scale;
  args.a_keeper_scale = (const __half*)a_keeper_scale; args.b_keeper_scale = (const __half*)b_keeper_scale;
  args.d = (__half*)d; args.M = (int)rows_cap; args.N = (int)N; args.G = (int)(K / 128 - 1);
  args.lda_scale = atom::scale_size((int)rows_cap); args.trace = g_trace; args.ldb_scale = (int)N;
  args.tiles = (const int4*)tiles; args.expert_rows = (int)N;
  return gemm_grouped_dispatch<atom::EPI_O16>(op, args, token_tile, num_tiles, N, (cudaStream_t)stream);
}

int atom_moe_combine_f16(const void* y, const void* topk_ids, const void* topk_weights, const void* dest_row, int seq_len, int hidden_dim,
                         int top_k, void* out, void* stream) {
  ATOM_REQUIRE(y && topk_ids && topk_weights && dest_row && out, "moe_combine_f16: null pointer argument");
  ATOM_REQUIRE(seq_len > 0 && hidden_dim > 0 && hidden_dim % 8 == 0 && top_k >= 1 && top_k <= atom::MOE_MAX_TOPK,
               "moe_combine_f16: seq_len=%d must be positive, hidden_dim=%d a multiple of 8, top_k=%d in [1, 8]", seq_len, hidden_dim, top_k);
  ATOM_REQUIRE(aligned16(y) && aligned16(out), "moe_combine_f16: y and out must be 16-byte aligned");
  return launch_k("moe_combine_f16", atom::moe_combine_kernel, dim3(seq_len), dim3(atom::COMBINE_THREADS), 0, (cudaStream_t)stream,
                  (const __half*)y, (const int32_t*)topk_ids, (const __half*)topk_weights, (const int32_t*)dest_row, top_k, hidden_dim,
                  (__half*)out);
}

}  // extern "C"
