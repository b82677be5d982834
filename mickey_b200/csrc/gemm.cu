// Host side of the GEMM family: TMA descriptor encoding, launch dispatch, and the SIMT debug kernel.
#include "gemm.h"
#include "gemm_tc.cuh"

#include <algorithm>
#include <cstdarg>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <unordered_map>

namespace mk {

// ---- cuTensorMapEncodeTiled through the runtime's driver entry point (no -lcuda needed) ---------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

// Descriptors are pure functions of (pointer, shape, box); the engine reuses the same workspace and
// weight buffers every call, so they are cached.
struct MapKey {
  const void* ptr; long long rows, cols, ld; int box;
  long long groups;          // 0: 2-D operand map; > 0: 3-D output map over [groups, rows, cols]
  bool operator==(const MapKey& o) const {
    return ptr == o.ptr && rows == o.rows && cols == o.cols && ld == o.ld && box == o.box && groups == o.groups;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = reinterpret_cast<size_t>(k.ptr);
    h = h * 1000003u ^ (size_t)k.rows; h = h * 1000003u ^ (size_t)k.cols; h = h * 1000003u ^ (size_t)k.ld;
    h = h * 1000003u ^ (size_t)k.groups;
    return h * 1000003u ^ (size_t)k.box;
  }
};
static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_map_cache;
static std::mutex g_map_mutex;

static int encode_tensor_map_out_f16(CUtensorMap* map, const void* ptr, long long groups, long long rows, long long cols,
                                     int box_rows);

static int cached_map(const MapKey& key, CUtensorMap* map) {
  std::lock_guard<std::mutex> lock(g_map_mutex);
  auto it = g_map_cache.find(key);
  if (it != g_map_cache.end()) { *map = it->second; return MK_OK; }
  int rc = key.groups ? encode_tensor_map_out_f16(map, key.ptr, key.groups, key.rows, key.cols, key.box)
                      : encode_tensor_map_2d(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, key.ptr, key.rows, key.cols, key.ld, key.box);
  if (rc == MK_OK) {
    if (g_map_cache.size() > 4096) g_map_cache.clear();
    g_map_cache.emplace(key, *map);
  }
  return rc;
}

int make_tensor_map_f16(CUtensorMap* map, const void* ptr, long long rows, long long cols, long long ld_elems,
                        int box_rows) {
  return cached_map(MapKey{ptr, rows, cols, ld_elems, box_rows, 0}, map);
}

int make_tensor_map_out_f16(CUtensorMap* map, void* ptr, long long groups, long long rows, long long cols, int box_rows) {
  return cached_map(MapKey{ptr, rows, cols, cols, box_rows, groups}, map);
}

static_assert(BLOCK_K * 2 == 128, "an fp16 operand box is one 128-byte swizzle row wide");

int encode_tensor_map_2d(CUtensorMap* map, CUtensorMapDataType dtype, const void* ptr, long long rows, long long cols,
                         long long ld_elems, int box_rows) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) { set_last_error("cuTensorMapEncodeTiled entry point not available"); return MK_ERR_CUDA; }
  const int esize = dtype == CU_TENSOR_MAP_DATA_TYPE_FLOAT32 ? 4 : 2;
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (ld_elems * esize) % 16) {
    set_last_error("tensor map operand must be 16-byte aligned with ld %% %d == 0 (ptr=%p ld=%lld)", 16 / esize, ptr, ld_elems);
    return MK_ERR_INVALID;
  }
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld_elems * esize};
  cuuint32_t box[2] = {(cuuint32_t)(128 / esize), (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, dtype, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_last_error("cuTensorMapEncodeTiled failed with CUresult %d", (int)r); return MK_ERR_CUDA; }
  return MK_OK;
}

// Contiguous fp16 [groups][rows][cols] output: box = 64 columns (128 bytes) x box_rows rows x 1, 128-byte swizzle on the
// shared-memory side, rows beyond `rows` clipped by the hardware in every group.
static int encode_tensor_map_out_f16(CUtensorMap* map, const void* ptr, long long groups, long long rows, long long cols,
                                     int box_rows) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) { set_last_error("cuTensorMapEncodeTiled entry point not available"); return MK_ERR_CUDA; }
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (cols % 8)) {
    set_last_error("TMA output must be 16-byte aligned with cols %% 8 == 0 (ptr=%p cols=%lld)", ptr, cols);
    return MK_ERR_INVALID;
  }
  cuuint64_t dims[3] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)groups};
  cuuint64_t strides[2] = {(cuuint64_t)cols * 2, (cuuint64_t)cols * 2 * (cuuint64_t)rows};
  cuuint32_t box[3] = {64, (cuuint32_t)box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_last_error("cuTensorMapEncodeTiled (fp16 output) failed with CUresult %d", (int)r); return MK_ERR_CUDA; }
  return MK_OK;
}

// fp32 [groups][n][n] tensor with row pitch `pitch` floats: box = 32 columns (128 bytes) x 32 rows x 1, 128-byte swizzle
// on the shared-memory side (the layout dual_store_chunk_tma writes), out-of-range rows / columns clipped by the hardware.
static int encode_tensor_map_out_f32(CUtensorMap* map, const void* ptr, long long n, long long pitch, long long groups) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) { set_last_error("cuTensorMapEncodeTiled entry point not available"); return MK_ERR_CUDA; }
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (pitch % 4) || pitch < n) {
    set_last_error("TMA output needs a 16-byte aligned base and a row pitch that is a multiple of 4 floats (ptr=%p pitch=%lld)", ptr, pitch);
    return MK_ERR_INVALID;
  }
  cuuint64_t dims[3] = {(cuuint64_t)n, (cuuint64_t)n, (cuuint64_t)groups};
  cuuint64_t strides[2] = {(cuuint64_t)pitch * 4, (cuuint64_t)pitch * 4 * (cuuint64_t)n};
  cuuint32_t box[3] = {32, 32, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_last_error("cuTensorMapEncodeTiled (fp32 output) failed with CUresult %d", (int)r); return MK_ERR_CUDA; }
  return MK_OK;
}

static const OutMaps& no_out_maps() { static OutMaps z = {}; return z; }

// ---- SIMT debug kernel --------------------------------------------------------------------------------
// Same operand addressing and the same epilogues as the wgmma kernel, computed with plain FFMA.  It is
// NOT a product path: it exists so that a GPU test can tell a wgmma/TMA descriptor bug from an epilogue
// bug (tests/test_gpu_ops.py runs both and compares); tests reach it through impl = 2 (GEMM_IMPL_SIMT).
template <int BN, int EPI>
__global__ void __launch_bounds__(128)
gemm_simt_kernel(const __half* __restrict__ A, long long a_rows, long long lda, const __half* __restrict__ B,
                 long long b_rows, long long ldb, const GemmParams p) {
  __shared__ __align__(16) __half As[BLOCK_M][BLOCK_K + 8];
  __shared__ __half Bs[BN][BLOCK_K + 8];
  pdl_trigger();
  pdl_wait();
  const GemmTile tile = gemm_tile<BN>(p, blockIdx.x);
  const int g = tile.g, m0 = tile.m0, n0 = tile.n0;
  const int t = threadIdx.x;
  float acc[BN];
#pragma unroll
  for (int j = 0; j < BN; ++j) acc[j] = 0.f;
  const int a_col0 = p.a_col_base + g * p.a_col_group_off;
  const long long a_row0 = (long long)m0 + (long long)g * p.a_row_group_off;
  const long long b_row0 = (long long)n0 + (long long)g * p.b_row_group_off;
  for (int kc = 0; kc < p.k_chunks; ++kc) {
    const int tap = kc / p.chunks_per_tap, kin = kc - tap * p.chunks_per_tap;
    for (int idx = t; idx < BLOCK_M * BLOCK_K; idx += 128) {
      const int r = idx / BLOCK_K, c = idx % BLOCK_K;
      const long long row = a_row0 + r + p.tap_shift[tap];
      const long long col = a_col0 + kin * BLOCK_K + c;
      As[r][c] = (row >= 0 && row < a_rows && col < lda) ? A[row * lda + col] : __float2half(0.f);
    }
    for (int idx = t; idx < BN * BLOCK_K; idx += 128) {
      const int r = idx / BLOCK_K, c = idx % BLOCK_K;
      const long long row = b_row0 + r;
      Bs[r][c] = (row < b_rows) ? B[row * ldb + (long long)kc * BLOCK_K + c] : __float2half(0.f);
    }
    __syncthreads();
    for (int k = 0; k < BLOCK_K; ++k) {
      const float a = __half2float(As[t][k]);
#pragma unroll
      for (int j = 0; j < BN; ++j) acc[j] = fmaf(a, __half2float(Bs[j][k]), acc[j]);
    }
    __syncthreads();
  }
  const int m = m0 + t;
  float v[32];
  if constexpr (EPI == EPI_LN) {
    float sum = 0.f;
    for (int j = 0; j < BN; ++j) sum += acc[j];
    const float mean = sum / BN;
    float sq = 0.f;
    for (int j = 0; j < BN; ++j) { const float d = acc[j] - mean; sq += d * d; }
    const float rstd = rsqrtf(sq / BN + p.eps);
    for (int c = 0; c < BN / 32; ++c) {
      for (int j = 0; j < 32; ++j) v[j] = acc[c * 32 + j];
      ln_store_chunk(p, g, m, n0 + c * 32, v, mean, rstd);
    }
  } else if constexpr (EPI == EPI_LSE || EPI == EPI_DUAL) {
    // the matcher epilogues exist on the wgmma kernel only (launch_gemm rejects them for this kernel)
  } else {
    for (int c = 0; c < BN / 32; ++c) {
      if (n0 + c * 32 < p.N) {
        for (int j = 0; j < 32; ++j) v[j] = acc[c * 32 + j];
        epilogue_chunk<EPI>(p, g, m, n0 + c * 32, v);
      }
    }
  }
}

bool pdl_enabled() {
  static int v = -1;
  // on by default (MICKEY_PDL=0 disables): the next kernel's prologue overlaps this kernel's tail
  if (v < 0) { const char* e = getenv("MICKEY_PDL"); v = (e && strcmp(e, "0") == 0) ? 0 : 1; }
  return v == 1;
}

// ---- dispatch -----------------------------------------------------------------------------------------
int sm_count() {
  static int n[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  int& c = n[dev & 63];
  if (!c) { cudaDeviceGetAttribute(&c, cudaDevAttrMultiProcessorCount, dev); if (c <= 0) c = 132; }
  return c;
}

// Persistent instantiations get one CTA per SM (fewer if there are fewer tiles); the one-tile-per-CTA ones one CTA per
// tile.  PAIR: two-CTA clusters, as many as can be resident at once (fewer if there are fewer tile pairs).  That count
// comes from the occupancy API, not from SMs / 2: a cluster's CTAs share a GPC, and a GPC with an odd number of free
// SMs leaves one idle; a grid beyond the resident clusters would run a second wave.
template <int BN, int EPI, int STAGES, bool PERSISTENT, bool PAIR = false>
static int launch_tc(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, cudaStream_t stream,
                     const OutMaps& om = no_out_maps()) {
  static unsigned long long attr_mask = 0;
  static int max_clusters[64] = {0};
  constexpr int smem = gemm_smem_bytes<BN, EPI, STAGES, PERSISTENT>();
  auto kernel = gemm_tc_kernel<BN, EPI, STAGES, PERSISTENT, PAIR>;
  cudaLaunchConfig_t cfg = {};
  cfg.blockDim = dim3(gemm_threads<PERSISTENT>()); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int n_attr = 0;
  if constexpr (PAIR) {
    attr[n_attr].id = cudaLaunchAttributeClusterDimension;
    attr[n_attr].val.clusterDim.x = 2; attr[n_attr].val.clusterDim.y = 1; attr[n_attr++].val.clusterDim.z = 1;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n_attr;
  int dev = 0;
  if constexpr (PAIR) cudaGetDevice(&dev);
  if (first_use_on_device(attr_mask)) {
    MK_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    if constexpr (PAIR) {
      cfg.gridDim = dim3(2 * sm_count());
      MK_CUDA_CHECK(cudaOccupancyMaxActiveClusters(&max_clusters[dev & 63], kernel, &cfg));
    }
  }
  const int tiles = gemm_tile_count<BN>(p);
  if constexpr (PAIR) {
    const int n_clusters = max_clusters[dev & 63];
    if (n_clusters <= 0) { set_last_error("GEMM: no two-CTA cluster of %d bytes of shared memory fits on this device", smem); return MK_ERR_UNSUPPORTED; }
    cfg.gridDim = dim3(2 * std::min(gemm_tile_count<BN, 2>(p), n_clusters));
  } else {
    cfg.gridDim = dim3(PERSISTENT ? std::min(tiles, sm_count()) : tiles);
  }
  if (pdl_enabled()) {
    attr[n_attr].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n_attr++].val.programmaticStreamSerializationAllowed = 1;
  }
  cfg.numAttrs = n_attr;
  MK_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kernel, tmA, tmB, p, om));
  return MK_OK;
}

// Grids of at most ~1.25 tiles per SM run one tile per CTA on a deep ring (more bytes in flight per tile).  Grids of more
// than 8 tiles per SM run the persistent kernel on CTA pairs that share each B tile: every ViT-B GEMM and head GEMM of
// the 32-pair batch (>= 1060 M-tiles).
// The ones in between run one tile per CTA with two CTAs per SM: every GEMM of a single ViT-S pair (at most 544 tiles),
// where the persistent kernel measured slower.
static bool deep_ring(int tiles, const GemmParams& p) {
  return (long long)tiles <= (long long)sm_count() * 5 / 4 && p.k_chunks > 3;
}
static bool persistent_grid(int tiles) { return tiles > 8 * sm_count(); }

template <int BN, int EPI>
static int launch_one(const GemmOperand& A, const GemmOperand& B, const GemmParams& p, cudaStream_t stream, int impl) {
  const int tiles = gemm_tile_count<BN>(p);
  if (impl == GEMM_IMPL_SIMT) {
    MK_CUDA_CHECK(launch_k(gemm_simt_kernel<BN, EPI>, dim3(tiles), dim3(128), 0, stream, reinterpret_cast<const __half*>(A.ptr),
                           (long long)A.rows, (long long)A.ld, reinterpret_cast<const __half*>(B.ptr), (long long)B.rows,
                           (long long)B.ld, p));
  } else {
    CUtensorMap tmA, tmB;
    int rc = make_tensor_map_f16(&tmA, A.ptr, A.rows, A.cols, A.ld, BLOCK_M);
    if (rc) return rc;
    if constexpr (persistent_epilogue<EPI>()) {
      // the persistent kernel: CTA pairs that share B (each loads half of the B box), unless the test / benchmark
      // selection asks for the unpaired kernel
      const bool forced = impl == GEMM_IMPL_TC_PAIRED || impl == GEMM_IMPL_TC_UNPAIRED;
      if (forced || persistent_grid(tiles)) {
        const bool pair = impl != GEMM_IMPL_TC_UNPAIRED;
        rc = make_tensor_map_f16(&tmB, B.ptr, B.rows, B.cols, B.ld, pair ? BN / 2 : BN);
        if (rc) return rc;
        if (pair) return launch_tc<BN, EPI, ring_stages<BN>(), true, true>(tmA, tmB, p, stream);
        return launch_tc<BN, EPI, ring_stages<BN>(), true>(tmA, tmB, p, stream);
      }
    }
    rc = make_tensor_map_f16(&tmB, B.ptr, B.rows, B.cols, B.ld, BN);
    if (rc) return rc;
    if constexpr (EPI == EPI_DUAL) {
      if (p.out_tma) {
        // the three N x N outputs leave through TMA tensor stores
        OutMaps om = {};
        float* outs[3] = {p.scores, p.kp_scores, p.final_scores};
        for (int i = 0; i < 3; ++i)
          if (outs[i]) { rc = encode_tensor_map_out_f32(&om.m[i], outs[i], p.n_valid, p.out_pitch, p.groups); if (rc) return rc; }
        return launch_tc<BN, EPI, shallow_stages<BN>(), false>(tmA, tmB, p, stream, om);
      }
    }
    if (deep_ring(tiles, p)) return launch_tc<BN, EPI, deep_stages<BN>(), false>(tmA, tmB, p, stream);
    return launch_tc<BN, EPI, shallow_stages<BN>(), false>(tmA, tmB, p, stream);
  }
  MK_CUDA_CHECK(cudaGetLastError());
  return MK_OK;
}

template <int EPI>
static int launch_bn(int bn, const GemmOperand& A, const GemmOperand& B, const GemmParams& p, cudaStream_t s, int impl) {
  if (bn == 128) return launch_one<128, EPI>(A, B, p, s, impl);
  if (bn == 64) return launch_one<64, EPI>(A, B, p, s, impl);
  set_last_error("unsupported BLOCK_N %d", bn);
  return MK_ERR_INVALID;
}

int launch_gemm(int epi, const GemmOperand& A, const GemmOperand& B, const GemmParams& p, cudaStream_t stream, int impl) {
  if (p.k_chunks <= 0 || p.M <= 0 || p.N <= 0 || p.groups <= 0) { set_last_error("bad GEMM shape"); return MK_ERR_INVALID; }
  const bool matcher = (epi == EPI_LSE || epi == EPI_DUAL);
  if (matcher && impl == GEMM_IMPL_SIMT) { set_last_error("the matcher epilogues run on the wgmma kernel only"); return MK_ERR_UNSUPPORTED; }
  if (matcher && (p.part_ld % 128 || p.part_ld < p.n_valid)) { set_last_error("matcher: part_ld must be n_valid rounded up to 128"); return MK_ERR_INVALID; }
  if (epi == EPI_DUAL && p.out_pitch < p.n_valid) { set_last_error("matcher: out_pitch %lld < n_valid %d", p.out_pitch, p.n_valid); return MK_ERR_INVALID; }
  if (!matcher && (p.N % 32)) { set_last_error("GEMM N=%d must be a multiple of 32", p.N); return MK_ERR_INVALID; }
  int bn = (matcher || p.N % 128 == 0) ? 128 : 64;
  if (!matcher && p.N % bn) { set_last_error("GEMM N=%d not tileable", p.N); return MK_ERR_INVALID; }
  if (epi == EPI_LN && p.N != 128) { set_last_error("EPI_LN needs N == 128"); return MK_ERR_INVALID; }
  switch (epi) {
    case EPI_STORE_H: return launch_bn<EPI_STORE_H>(bn, A, B, p, stream, impl);
    case EPI_RESID_F: return launch_bn<EPI_RESID_F>(bn, A, B, p, stream, impl);
    case EPI_PATCH:   return launch_bn<EPI_PATCH>(bn, A, B, p, stream, impl);
    case EPI_CONV:    return launch_bn<EPI_CONV>(bn, A, B, p, stream, impl);
    case EPI_STORE_F: return launch_bn<EPI_STORE_F>(bn, A, B, p, stream, impl);
    case EPI_LN:      return launch_one<128, EPI_LN>(A, B, p, stream, impl);
    case EPI_LSE:     return launch_one<128, EPI_LSE>(A, B, p, stream, impl);
    case EPI_DUAL:    return launch_one<128, EPI_DUAL>(A, B, p, stream, impl);
  }
  set_last_error("unknown epilogue %d", epi);
  return MK_ERR_INVALID;
}

// ---- error string -------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* last_error() { return g_err; }

}  // namespace mk
