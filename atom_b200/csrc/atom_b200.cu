// atom_b200.cu -- C ABI (include/atom_b200.h) and host-side launch logic of libatom_b200.so.
//
// No torch types, no allocation, no synchronisation: every entry point validates its arguments, builds the TMA
// descriptors it needs on the host (cached by (pointer, shape)) and enqueues kernels on the caller's stream.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
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
template <int BN, int kSplit, int kEpi>
int launch_gemm(const GemmOperands& op, const atom::GemmArgs& args, cudaStream_t stream, int64_t out_channels = -1) {
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
  cfg.gridDim = dim3((unsigned)((chan + 127) / 128), (unsigned)((op.M + BN - 1) / BN), kSplit);
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

int atom_gemm_i4_qkv(const void* a, const void* b_qkv, const void* a_scale, const void* b_scale_qkv, const void* a_keeper,
                     const void* b_keeper_qkv, const void* a_keeper_scale, const void* b_keeper_scale_qkv, void* q, void* k,
                     void* k_scale, void* v, void* v_scale, int64_t M, int64_t H, int64_t K, uint32_t flags, void* stream) {
  ATOM_REQUIRE(a && b_qkv && a_scale && b_scale_qkv && a_keeper && b_keeper_qkv && a_keeper_scale && b_keeper_scale_qkv && q && k &&
               k_scale && v && v_scale, "gemm_i4_qkv: null pointer argument");
  ATOM_REQUIRE(M > 0 && H > 0 && H % 128 == 0, "gemm_i4_qkv: M=%lld must be positive, H=%lld a positive multiple of 128", (long long)M, (long long)H);
  ATOM_REQUIRE(K >= 256 && K % 128 == 0, "gemm_i4_qkv: K=%lld must be a multiple of 128 and >= 256", (long long)K);
  ATOM_REQUIRE(aligned16(a) && aligned16(b_qkv) && aligned16(a_keeper) && aligned16(b_keeper_qkv) && aligned16(q) && aligned16(b_scale_qkv) &&
               aligned16(b_keeper_scale_qkv), "gemm_i4_qkv: operand pointers must be 16-byte aligned");
  ATOM_REQUIRE(M < (1ll << 31) && 3 * H < (1ll << 31) && K < (1ll << 24), "gemm_i4_qkv: dimension too large");
  const int64_t N = 3 * H;
  // one launch: 3H/128 channel tiles, the tile index selects the epilogue (q: FP16, k / v: asymmetric INT4 per head)
  GemmOperands op{a, b_qkv, a_keeper, b_keeper_qkv, M, N, K};
  atom::GemmArgs args{};
  args.a_scale = (const __half*)a_scale; args.a_keeper_scale = (const __half*)a_keeper_scale;
  args.b_scale = (const __half*)b_scale_qkv; args.b_keeper_scale = (const __half*)b_keeper_scale_qkv;
  args.M = (int)M; args.N = (int)N; args.G = (int)(K / 128 - 1); args.lda_scale = atom::scale_size((int)M); args.trace = g_trace;
  args.ldb_scale = (int)N; args.seg_tiles = (int)(H / 128);
  args.d = (__half*)q; args.d4 = (uint8_t*)k; args.d_scale = (__half2*)k_scale; args.d4_v = (uint8_t*)v; args.d_scale_v = (__half2*)v_scale;
  return gemm_dispatch<atom::EPI_QKV>(op, args, flags, (cudaStream_t)stream);
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

int atom_prefill_attention_i4(const void* q, const void* k, const void* k_param, const void* v, const void* v_param,
                              const void* seqlen_indptr, const void* pos_of_token, const void* rope_table, void* k_f16, void* v_f16,
                              void* out, int total_tokens, int batch_size, int max_len, int num_heads, void* stream) {
  ATOM_REQUIRE(q && k && k_param && v && v_param && seqlen_indptr && pos_of_token && rope_table && k_f16 && v_f16 && out,
               "prefill_attention_i4: null pointer argument");
  ATOM_REQUIRE(batch_size > 0 && num_heads > 0 && max_len > 0, "prefill_attention_i4: batch_size=%d num_heads=%d max_len=%d must be positive",
               batch_size, num_heads, max_len);
  ATOM_REQUIRE(aligned16(q) && aligned16(k) && aligned16(v) && aligned16(k_f16) && aligned16(v_f16) && aligned16(out),
               "prefill_attention_i4: pointers must be 16-byte aligned");
  if (total_tokens <= 0) return ATOM_OK;
  const long long th = (long long)total_tokens * num_heads;
  atom::kv_dequant_rope_kernel<<<(unsigned)((th + 3) / 4), 256, 0, (cudaStream_t)stream>>>(
      (const uint8_t*)k, (const __half2*)k_param, (const uint8_t*)v, (const __half2*)v_param, (const int32_t*)pos_of_token,
      (const float2*)rope_table, (__half*)k_f16, (__half*)v_f16, th, num_heads);
  int rc = check_launch("prefill_attention_i4 (dequant + RoPE)");
  if (rc) return rc;
  const dim3 grid((unsigned)((max_len + atom::PF_BQ - 1) / atom::PF_BQ), (unsigned)batch_size, (unsigned)num_heads);
  atom::prefill_attn_kernel<<<grid, atom::PF_THREADS, 0, (cudaStream_t)stream>>>(
      (const __half*)q, (const __half*)k_f16, (const __half*)v_f16, (const int32_t*)seqlen_indptr, (const float2*)rope_table,
      (__half*)out, num_heads, 0.08838834764831845f * 1.4426950408889634f);
  return check_launch("prefill_attention_i4");
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
