// Common definitions for the mickey_b200 CUDA kernels (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>

#define MK_OK 0
#define MK_ERR_INVALID -1
#define MK_ERR_CUDA -2
#define MK_ERR_MISSING_TENSOR -3
#define MK_ERR_UNSUPPORTED -4

namespace mk {

// ---- GEMM ("D = A * B^T" with A [M,K] K-major fp16, B [N,K] K-major fp16, fp32 accumulate) ----------
// One kernel family serves: ViT linears, patch embedding, 3x3 convolutions of the heads (as 9 row-shifted
// K-slabs over a zero-padded NHWC image), the linear-attention projections, and the descriptor
// correlation of the matcher.  The epilogue is selected at compile time.
enum Epi : int {
  EPI_STORE_H = 0,   // out_h = act(acc + bias)            fp16           (qkv, fc1+GELU, mlp.0+ReLU)
  EPI_RESID_F = 1,   // out_f += gamma * (acc + bias)      fp32 in place  (attn.proj, mlp.fc2 + LayerScale + residual)
  EPI_PATCH   = 2,   // out_f[row_map(m)] = acc + aux[m % tok][n]         (patch embed + bias + pos-embed)
  EPI_CONV    = 3,   // out_h = mask(act(acc + bias + res_h) + aux)       (3x3 / 1x1 conv, BN folded, shortcut, PE)
  EPI_STORE_F = 4,   // out_f = acc                        fp32           (linear-attention q,k,v)
  EPI_LN      = 5,   // out = LN_128(acc) [+ out_f]        fp16 (+fp32)   (merge+norm1, mlp.2+norm2+residual)
  EPI_LSE     = 6,   // per-tile (max, sum exp) partials of every row AND every column of S/T   (matcher pass 1)
  EPI_DUAL    = 7,   // scores = exp(2 S/T - lse_row - lse_col), kp_scores, final_scores          (matcher pass 2)
};

enum Act : int { ACT_NONE = 0, ACT_GELU = 1, ACT_RELU = 2 };

struct GemmParams {
  int M, N;                 // logical output rows / cols per group
  int k_chunks;             // number of 64-element K chunks in total (all taps)
  int chunks_per_tap;       // K chunks per tap (= k_chunks when num_taps == 1)
  int num_taps;
  int tap_shift[9];         // A row shift per tap (3x3 conv over the flattened padded image)
  int groups;               // independent GEMMs of one launch (gemm_tile orders their tiles)
  int a_row_group_off, a_col_group_off, a_col_base;   // A coordinates added per group
  int b_row_group_off;      // B rows added per group (usually N)
  int act;
  // epilogue operands (meaning depends on Epi)
  const float* bias;  int bias_group_off;
  const float* gamma; const float* beta; int ln_group_off;
  float* out_f; long long out_f_ld; long long out_f_group_off;
  __half* out_h; long long out_h_ld; long long out_h_group_off;
  const __half* res_h; long long res_h_ld; long long res_h_group_off;
  const float* aux; int aux_group_mask;   // pos table (EPI_PATCH: [tok, N]) / PE table (EPI_CONV: [rows_per_img, N])
  int pad_h2, pad_w2;       // padded token grid (rows per image = pad_h2 * pad_w2); 0 = no pad masking
  int tok_per_img;          // EPI_PATCH: patch tokens per image
  float eps;
  // matcher
  int n_valid;              // valid rows == valid cols per pair
  float inv_temp;
  const float* dustbin;     // device scalar or nullptr
  // EPI_LSE out: online-softmax partials in the log2 domain, float2 (max, sum 2^(x - max)) per slot:
  //   part_row[(g * 2*tiles + 2*n_tile + half) * part_ld + row]   (a warp's 64 columns of one row)
  //   part_col[(g * 4*tiles + 4*m_tile + q)    * part_ld + col]   (a warp's 32 rows of one column)
  // with tiles = part_ld / 128.  Slot-major, so that both the warps' stores and the reduce kernel's loads coalesce.
  float2* part_row; float2* part_col;
  int part_ld;              // n_valid rounded up to a multiple of 128
  float lse_bound;          // > 0: every |S| <= lse_bound (L2-normalised descriptors: 1): the partials use the fixed shift
                            // lse_bound / T instead of true maxima (one exponential per cell, no max reductions)
  // EPI_DUAL in: log2-domain log-sum-exp of every row / column of the dustbin-augmented S/T, [groups, part_ld]
  const float* lse_r; const float* lse_c;
  const float* scr0; const float* scr1; // [groups, n_valid]
  float* scores; float* kp_scores; float* final_scores;   // [groups, n_valid, out_pitch]; scores / kp_scores may be NULL (lean)
  long long out_pitch;      // row pitch of the three N x N outputs in floats (n_valid = contiguous, the reference's layout)
  int out_tma;              // 1: rows are 16-byte aligned (pitch % 4 == 0) -> the outputs leave through TMA tensor stores
};

// Tensor maps of the matcher's three outputs (scores, kp_scores, final_scores: fp32 [groups][n_valid][n_valid] with row
// pitch out_pitch, box 32 x 32, 128-byte swizzle on the shared-memory side).  Every GEMM kernel carries the parameter;
// only EPI_DUAL with out_tma reads it.
struct OutMaps { CUtensorMap m[3]; };

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// Function attributes (cudaFuncSetAttribute) and the SM count belong to a DEVICE: one-time setup is keyed on the
// current device, not on the process (a second handle on cuda:1 must run its own).
static inline bool first_use_on_device(unsigned long long& mask) {
  int d = 0;
  cudaGetDevice(&d);
  const unsigned long long bit = 1ull << (d & 63);
  if (mask & bit) return false;
  mask |= bit;
  return true;
}

// ---- programmatic dependent launch (PDL) ---------------------------------------------------------------
// Every kernel of the pipeline is launched with cudaLaunchAttributeProgrammaticStreamSerialization: it lets the
// NEXT kernel's CTAs be scheduled as soon as this grid has issued pdl_trigger() and SM resources free up, so the
// next kernel's prologue (mbarrier init, tensor-map prefetch, index math) overlaps this kernel's
// tail.  pdl_wait() blocks until all prerequisite grids have completed and their memory is visible; every kernel
// executes it before its first access to global memory.  Both are no-ops when launched without the attribute.
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
#endif

bool pdl_enabled();   // default on; MICKEY_PDL=0 disables

template <typename... KArgs, typename... Args>
static inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace mk

#define MK_CUDA_CHECK(x)                                                                      \
  do {                                                                                        \
    cudaError_t e_ = (x);                                                                     \
    if (e_ != cudaSuccess) {                                                                  \
      mk::set_last_error("%s failed at %s:%d: %s", #x, __FILE__, __LINE__, cudaGetErrorString(e_)); \
      return MK_ERR_CUDA;                                                                     \
    }                                                                                         \
  } while (0)

#define MK_TRY(x) do { int rc_ = (x); if (rc_ != MK_OK) return rc_; } while (0)

namespace mk {
void set_last_error(const char* fmt, ...);

// Row pitch (floats) of an fp32 [B, N, N] argument: <= 0 means contiguous (N).  A pitch below N would make rows overlap
// and is rejected; `what` names the entry point and the argument in the message ("mk_match: nn_pitch").
static inline int resolve_pitch(long long& pitch, int N, const char* what) {
  if (pitch <= 0) pitch = N;
  if (pitch < N) { set_last_error("%s %lld < N %d", what, pitch, N); return MK_ERR_INVALID; }
  return MK_OK;
}
}
