// weight_stream_probe.cu -- how fast can the decode GEMM's INT4 weight tiles reach shared memory, by fetch geometry?
//
// Built at run time by tools/weight_stream_probe.py (not part of libatom_b200.so).  The kernel reproduces the launch
// conditions of gemm_i4_kernel<16, 4, EPI_O16> at N = K = 4096: the same grid (32 channel tiles x 4-rank K cluster), 384
// threads and dynamic shared memory (two CTAs per SM), programmatic dependent launch with every weight request issued before
// griddepcontrol.wait, and oracle.split_ranges' group partition (ranks 0-2: 8 groups, rank 3: 7).  It moves nothing but rank
// r's K range of its 128 weight rows into shared memory, waits for its mbarriers and exits.
#include "../atom_b200/csrc/gemm_i4_sm90.cuh"

#include <vector>

namespace {

using atom::mbar_arrive_expect_tx;
using atom::mbar_init;
using atom::mbar_wait;
using atom::smem_u32;

constexpr int kRows = 4096;                      // N: weight rows
constexpr int kK = 4096;
constexpr int kPitch = (kK - 128) / 2;            // 1984 B: packed INT4 bytes per row (31 groups of 64 B)
constexpr int kGroups = kK / 128;                 // 31 INT4 groups + the keeper
constexpr int kSplit = 4;
constexpr int kSmem = atom::GemmCfg<16, kSplit, atom::EPI_O16>::SMEM_BYTES;
constexpr int kRing = 64 * 1024;                  // the weight ring: 8 groups x 128 rows x 64 B

enum Variant { V_A = 0, V_B, V_C, V_D256, V_D512, V_D256U8, V_E, V_F, V_G, V_COUNT };

__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void bulk_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_prefetch_l2(const void* src, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(reinterpret_cast<uint64_t>(src)), "r"(bytes) : "memory");
}

// one launch: every CTA requests its weight bytes (before griddepcontrol.wait), then waits for them to land
__global__ void __launch_bounds__(384, 1)
probe_kernel(const __grid_constant__ CUtensorMap tm, const uint8_t* w, int variant) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kRing);
  const uint32_t rank = atom::cluster_ctarank();
  const int per = (kGroups + kSplit - 1) / kSplit;
  const int g_begin = min((int)rank * per, kGroups), g_end = min(g_begin + per, kGroups);
  const int n4 = max(0, min(g_end, kGroups - 1) - g_begin);
  const int n0 = blockIdx.x * 128;
  // stages (one mbarrier each) and bytes per stage
  int stages = n4, stage_bytes = 128 * 64;
  if (variant == V_C) { stages = (n4 + 1) / 2; stage_bytes = 128 * 128; }
  if (variant == V_D256 || variant == V_D256U8) { stages = (n4 + 3) / 4; stage_bytes = 128 * 256; }
  if (variant == V_D512 || variant == V_E) { stages = 1; stage_bytes = 128 * 512; }
  if (variant == V_F) { stages = 1; stage_bytes = 128 * 64 * n4; }
  if (threadIdx.x == 0) {
    atom::tma_prefetch_desc(&tm);
    for (int i = 0; i < stages; ++i) mbar_init(&bars[i], 1);
    atom::fence_barrier_init();
  }
  __syncthreads();
  atom::griddep_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (variant == V_G && warp == 1) {
    // the cluster's 128 rows are one contiguous block of 128 x pitch bytes; each rank prefetches a quarter of it into L2
    const size_t block = (size_t)128 * kPitch, quarter = block / kSplit;
    const size_t lo = (size_t)n0 * kPitch + rank * quarter;
    const size_t hi = min(lo + quarter, (size_t)kRows * kPitch);
    constexpr size_t kChunk = 4096;
    for (size_t o = lo + lane * kChunk; o < hi; o += 32 * kChunk) bulk_prefetch_l2(w + o, (uint32_t)min(kChunk, hi - o));
  }
  if (variant == V_F) {
    // one 1-D bulk copy per row: 128 row spans of n4 x 64 B, issued by warp 0, all on one mbarrier
    if (warp == 0) {
      if (lane == 0) mbar_arrive_expect_tx(&bars[0], stage_bytes);
      __syncwarp();
      for (int r = lane; r < 128; r += 32)
        bulk_load_1d(smem + r * 64 * n4, w + (size_t)(n0 + r) * kPitch + g_begin * 64, 64 * n4, &bars[0]);
    }
  } else if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) {
      mbar_arrive_expect_tx(&bars[s], stage_bytes);
      uint8_t* dst = smem + s * stage_bytes;
      switch (variant) {
        case V_A: case V_B: case V_G: atom::tma_load_2d(dst, &tm, &bars[s], (g_begin + s) * 64, n0); break;
        case V_C: atom::tma_load_2d(dst, &tm, &bars[s], (g_begin + 2 * s) * 64, n0); break;
        case V_D256: atom::tma_load_2d(dst, &tm, &bars[s], (g_begin + 4 * s) * 8, n0); break;      // 8-byte elements
        case V_D512: atom::tma_load_2d(dst, &tm, &bars[s], g_begin * 8, n0); break;
        case V_D256U8: atom::tma_load_2d(dst, &tm, &bars[s], (g_begin + 4 * s) * 64, n0); break;
        case V_E: tma_load_3d(dst, &tm, &bars[s], 0, n0, g_begin); break;
      }
    }
  }
  atom::griddep_wait();
  if (threadIdx.x == 0)
    for (int s = 0; s < stages; ++s) mbar_wait(&bars[s], 0);
  __syncthreads();
}

// reference point: a plain coalesced read of the same bytes, 16-byte vectors, every byte once
__global__ void __launch_bounds__(256)
stream_read_kernel(const uint4* w, size_t n16, unsigned* sink) {
  uint32_t x = 0;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + 3 * stride < n16; i += 4 * stride) {
    uint4 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u] = atom::ld_cg_v4(w + i + u * stride);
#pragma unroll
    for (int u = 0; u < 4; ++u) x ^= v[u].x ^ v[u].y ^ v[u].z ^ v[u].w;
  }
  for (; i < n16; i += stride) { const uint4 v = atom::ld_cg_v4(w + i); x ^= v.x ^ v.y ^ v.z ^ v.w; }
  if (x == 0x9e3779b9u) sink[0] = x;              // keeps the loads; practically never stores
}

using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                              const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

char g_err[512];

int encode(CUtensorMap* m, int variant, void* ptr) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
    snprintf(g_err, sizeof g_err, "cuTensorMapEncodeTiled unavailable");
    return -1;
  }
  EncodeFn fn = reinterpret_cast<EncodeFn>(p);
  CUtensorMapDataType ty = CU_TENSOR_MAP_DATA_TYPE_UINT8;
  CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_NONE;
  CUtensorMapL2promotion l2 = CU_TENSOR_MAP_L2_PROMOTION_L2_128B;
  cuuint32_t rank = 2, estr[3] = {1, 1, 1};
  cuuint64_t dims[3] = {kPitch, kRows, 1}, strides[2] = {kPitch, 0};
  cuuint32_t box[3] = {64, 128, 1};
  switch (variant) {
    case V_B: l2 = CU_TENSOR_MAP_L2_PROMOTION_L2_256B; break;
    case V_C: box[0] = 128; sw = CU_TENSOR_MAP_SWIZZLE_128B; break;
    case V_D256: ty = CU_TENSOR_MAP_DATA_TYPE_UINT64; dims[0] = kPitch / 8; box[0] = 32; break;
    case V_D512: ty = CU_TENSOR_MAP_DATA_TYPE_UINT64; dims[0] = kPitch / 8; box[0] = 64; break;
    case V_D256U8: box[0] = 256; break;
    case V_E:
      // (64 B, row, group): strides {pitch, 64}, box {64, 128, 8} -- the per-group [row][64 B] layout in one request
      rank = 3; dims[0] = 64; dims[1] = kRows; dims[2] = kGroups - 1; strides[0] = kPitch; strides[1] = 64;
      box[0] = 64; box[1] = 128; box[2] = 8;
      break;
    default: break;
  }
  CUresult r = fn(m, ty, rank, ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    snprintf(g_err, sizeof g_err, "cuTensorMapEncodeTiled rejected the map: CUresult %d", (int)r);
    return (int)r;
  }
  return 0;
}

#define CK(x)                                                                                    \
  do {                                                                                           \
    cudaError_t e_ = (x);                                                                        \
    if (e_ != cudaSuccess) {                                                                     \
      snprintf(g_err, sizeof g_err, "%s: %s (line %d)", #x, cudaGetErrorString(e_), __LINE__);  \
      return -2;                                                                                 \
    }                                                                                            \
  } while (0)

}  // namespace

extern "C" {

const char* probe_last_error() { return g_err; }
int probe_variants() { return V_COUNT; }     // variant ids 0..V_COUNT-1; V_COUNT = the plain coalesced read
int probe_tensor_bytes() { return kRows * kPitch; }

// µs per launch of `variant` over `nsets` weight tensors (one CUDA graph of `rounds` x `nsets` back-to-back launches,
// replayed `reps` times after `warm` replays).  Returns 0, or a CUresult (> 0) if the tensor map is rejected, or < 0.
int probe_run(int variant, void* const* sets, int nsets, int rounds, int warm, int reps, float* us_per_launch) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { snprintf(g_err, sizeof g_err, "no CUDA device"); return -1; }
  std::vector<CUtensorMap> maps(nsets);
  if (variant < V_COUNT)
    for (int i = 0; i < nsets; ++i) {
      const int rc = encode(&maps[i], variant, sets[i]);
      if (rc) return rc;
    }
  unsigned* sink = nullptr;
  CK(cudaMalloc(&sink, 16));
  CK(cudaFuncSetAttribute(probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
  cudaStream_t st;
  CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  auto launch = [&](int i) -> cudaError_t {
    if (variant == V_COUNT) {
      stream_read_kernel<<<sms * 8, 256, 0, st>>>(reinterpret_cast<const uint4*>(sets[i]), (size_t)kRows * kPitch / 16, sink);
      return cudaGetLastError();
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(kRows / 128, 1, kSplit);
    cfg.blockDim = dim3(384);
    cfg.dynamicSmemBytes = kSmem;
    cfg.stream = st;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 1; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = kSplit;
    attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 2;
    return cudaLaunchKernelEx(&cfg, probe_kernel, maps[i], static_cast<const uint8_t*>(sets[i]), variant);
  };
  // eager once (module load, errors surface here), then the graph
  for (int i = 0; i < nsets; ++i) CK(launch(i));
  CK(cudaStreamSynchronize(st));
  cudaGraph_t g;
  cudaGraphExec_t ge;
  CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
  for (int r = 0; r < rounds; ++r)
    for (int i = 0; i < nsets; ++i) {
      const cudaError_t e = launch(i);
      if (e != cudaSuccess) { cudaStreamEndCapture(st, &g); CK(e); }
    }
  CK(cudaStreamEndCapture(st, &g));
  CK(cudaGraphInstantiate(&ge, g, 0));
  for (int i = 0; i < warm; ++i) CK(cudaGraphLaunch(ge, st));
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  CK(cudaEventRecord(e0, st));
  for (int i = 0; i < reps; ++i) CK(cudaGraphLaunch(ge, st));
  CK(cudaEventRecord(e1, st));
  CK(cudaEventSynchronize(e1));
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, e0, e1));
  *us_per_launch = ms * 1000.f / ((float)reps * rounds * nsets);
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  cudaGraphExecDestroy(ge); cudaGraphDestroy(g);
  cudaStreamDestroy(st);
  cudaFree(sink);
  return 0;
}

}  // extern "C"
