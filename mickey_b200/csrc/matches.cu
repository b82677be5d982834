// Mutual-nearest-neighbour correspondences of score matrices: featureMatcher.get_matches_list
// (lib/models/MicKey/modules/utils/feature_matcher.py:19-46), batched.
//
// scores fp32 [B][N][N] with row pitch `pitch` floats.  As in the reference, the last row and column are dropped, so the
// candidates are rows i and columns j in [0, W), W = N - 1.  (i, j) is a match when j is the first argmax of row i, i is
// the first argmax of column j (a NaN counts as maximal, as in torch.max) and exp(scores[i][j]) > min_conf, with exp
// evaluated in double and rounded to fp32.  The matches are sorted by score, descending, equal scores by ascending i.
//
// Two kernels, one read of the matrix:
//   strips:   block (strip, pair) reads STRIP_ROWS rows across the full width.  Each warp owns ROWS_PER_WARP consecutive rows
//             and walks the columns in 128-wide chunks (16-byte loads when the rows are 16-byte aligned); a lane keeps the
//             running (max, argmax) of each of its rows and folds its rows into per-column partials, which the block folds
//             across warps and stores to slot (pair, strip, column).  Row results go to (pair, row).
//   select:   one block per pair folds the column partials, applies the mutual and threshold tests, sorts the survivors
//             in shared memory by a 64-bit key (score descending, i ascending; non-survivors carry the all-ones key) and
//             writes matches / scores / count.
// No atomics: the "better" relation below is a total order on (value, index), so every fold gives the same winner in
// any order and the output is bit-for-bit deterministic.
#include "common.cuh"

namespace mk {
namespace {

constexpr int MM_WARPS = 8;
constexpr int ROWS_PER_WARP = 8;
constexpr int STRIP_ROWS = MM_WARPS * ROWS_PER_WARP;   // 64 rows per strip block
constexpr int CHUNK = 128;                             // columns per step: 32 lanes x 4
constexpr int MAX_SORT = 4096;                         // candidates per pair (N - 1 <= 4096)
constexpr int SELECT_THREADS = 1024;

struct Best { float v; int i; };

// (v, i) ranks above (bv, bi): NaN above every number, then larger value, then smaller index (torch.max's first index)
__device__ __forceinline__ bool better(float v, int i, float bv, int bi) {
  if (isnan(v)) return !isnan(bv) || i < bi;
  if (isnan(bv)) return false;
  return v > bv || (v == bv && i < bi);
}

__device__ __forceinline__ void fold(Best& b, float v, int i) {
  if (better(v, i, b.v, b.i)) { b.v = v; b.i = i; }
}

__device__ __forceinline__ Best warp_fold(Best b) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float v = __shfl_xor_sync(0xffffffffu, b.v, o);
    const int i = __shfl_xor_sync(0xffffffffu, b.i, o);
    fold(b, v, i);
  }
  return b;
}

template <bool VEC>
__global__ void __launch_bounds__(MM_WARPS * 32)
mutual_strips_kernel(const float* __restrict__ scores, long long pitch, int N, int n_strips, Best* __restrict__ row_best,
                     Best* __restrict__ col_part) {
  __shared__ Best cols[MM_WARPS][CHUNK];
  pdl_wait();
  const int W = N - 1;
  const int pair = blockIdx.y, strip = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r0 = strip * STRIP_ROWS + warp * ROWS_PER_WARP;
  const float* base = scores + (size_t)pair * N * pitch;
  Best rb[ROWS_PER_WARP];
#pragma unroll
  for (int r = 0; r < ROWS_PER_WARP; ++r) rb[r] = Best{-INFINITY, INT_MAX};
  for (int c0 = 0; c0 < W; c0 += CHUNK) {
    Best cb[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) cb[q] = Best{-INFINITY, INT_MAX};
    // VEC: lane owns columns c0 + 4 lane + q (one 16-byte load); otherwise c0 + lane + 32 q (four coalesced loads)
    float x[ROWS_PER_WARP][4];
#pragma unroll
    for (int r = 0; r < ROWS_PER_WARP; ++r) {
      const int row = r0 + r;
      const float* p = base + (size_t)row * pitch + c0;
      if (VEC) {
        // the 16 bytes at a valid column c < W end before pitch (pitch % 4 == 0, pitch >= N), and row <= N - 2 is followed
        // by row N - 1, so the load stays inside the matrix even where it covers columns >= W
        float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
        if (row < W && c0 + 4 * lane < W) t = __ldcs(reinterpret_cast<const float4*>(p) + lane);
        x[r][0] = t.x; x[r][1] = t.y; x[r][2] = t.z; x[r][3] = t.w;
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) x[r][q] = (row < W && c0 + lane + 32 * q < W) ? __ldcs(p + lane + 32 * q) : 0.f;
      }
    }
#pragma unroll
    for (int r = 0; r < ROWS_PER_WARP; ++r) {
      const int row = r0 + r;
      if (row >= W) break;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int col = c0 + (VEC ? 4 * lane + q : lane + 32 * q);
        if (col < W) {
          fold(rb[r], x[r][q], col);
          fold(cb[q], x[r][q], row);
        }
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) cols[warp][VEC ? 4 * lane + q : lane + 32 * q] = cb[q];
    __syncthreads();
    if (threadIdx.x < CHUNK && c0 + threadIdx.x < W) {
      Best b = cols[0][threadIdx.x];
#pragma unroll
      for (int w = 1; w < MM_WARPS; ++w) fold(b, cols[w][threadIdx.x].v, cols[w][threadIdx.x].i);
      col_part[((size_t)pair * n_strips + strip) * W + c0 + threadIdx.x] = b;
    }
    __syncthreads();
  }
  pdl_trigger();
#pragma unroll
  for (int r = 0; r < ROWS_PER_WARP; ++r) {
    const Best b = warp_fold(rb[r]);
    if (lane == 0 && r0 + r < W) row_best[(size_t)pair * W + r0 + r] = b;
  }
}

// ascending order of the key = descending score, then ascending row; -0 and +0 compare equal as in torch.sort
__device__ __forceinline__ unsigned long long sort_key(float v, int i) {
  unsigned u = __float_as_uint(v + 0.0f);                      // -0 + 0 = +0
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);              // monotone map of the float order onto unsigned
  return ((unsigned long long)(~u) << 32) | (unsigned)i;
}

__global__ void __launch_bounds__(SELECT_THREADS)
mutual_select_kernel(const Best* __restrict__ row_best, const Best* __restrict__ col_part, int N, int n_strips, int n_sort,
                     float min_conf, int* __restrict__ matches, float* __restrict__ match_scores, int* __restrict__ count) {
  extern __shared__ unsigned long long keys[];                 // [n_sort] then int col_arg[W]
  int* col_arg = reinterpret_cast<int*>(keys + n_sort);
  pdl_wait();
  const int W = N - 1, pair = blockIdx.x;
  const Best* rows = row_best + (size_t)pair * W;
  for (int j = threadIdx.x; j < W; j += blockDim.x) {
    Best b = col_part[(size_t)pair * n_strips * W + j];
    for (int s = 1; s < n_strips; ++s) {
      const Best c = col_part[((size_t)pair * n_strips + s) * W + j];
      fold(b, c.v, c.i);
    }
    col_arg[j] = b.i;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n_sort; i += blockDim.x) {
    unsigned long long k = ~0ull;
    if (i < W) {
      const Best r = rows[i];
      // exp in double, rounded to fp32; a NaN maximum fails the comparison
      if (col_arg[r.i] == i && __double2float_rn(exp((double)r.v)) > min_conf) k = sort_key(r.v, i);
    }
    keys[i] = k;
  }
  __syncthreads();
  // bitonic sort of n_sort (a power of two) keys
  for (int size = 2; size <= n_sort; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int t = threadIdx.x; t < n_sort / 2; t += blockDim.x) {
        const int lo = 2 * t - (t & (stride - 1));
        const int hi = lo + stride;
        const bool up = (lo & size) == 0;
        const unsigned long long a = keys[lo], b = keys[hi];
        if ((a > b) == up) { keys[lo] = b; keys[hi] = a; }
      }
      __syncthreads();
    }
  }
  pdl_trigger();
  __shared__ int n_kept;
  if (threadIdx.x == 0) {
    // the survivors are the keys below the all-ones sentinel, now a prefix: find its end by bisection
    int lo = 0, hi = n_sort;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (keys[mid] != ~0ull) lo = mid + 1; else hi = mid; }
    n_kept = lo;
    count[pair] = lo;
  }
  __syncthreads();
  int* m = matches + (size_t)pair * W * 2;
  float* ms = match_scores + (size_t)pair * W;
  for (int k = threadIdx.x; k < W; k += blockDim.x) {
    int i = -1, j = -1;
    float v = 0.f;
    if (k < n_kept) {
      i = (int)(unsigned)keys[k];
      const Best r = rows[i];
      j = r.i; v = r.v;
    }
    m[2 * k] = i; m[2 * k + 1] = j; ms[k] = v;
  }
}

}  // namespace

long long mutual_matches_ws_bytes(int B, int N) {
  if (B <= 0 || N < 2) return 0;
  const long long W = N - 1, strips = (W + STRIP_ROWS - 1) / STRIP_ROWS;
  return (long long)B * W * (1 + strips) * (long long)sizeof(Best);
}

int mutual_matches(const float* scores, long long pitch, int B, int N, float min_conf, int* matches, float* match_scores,
                   int* count, void* ws, long long ws_bytes, cudaStream_t s) {
  MK_TRY(resolve_pitch(pitch, N, "mk_mutual_matches: nn_pitch"));
  if (!scores || !matches || !match_scores || !count || !ws || B <= 0 || N < 2 || N - 1 > MAX_SORT || isnan(min_conf) ||
      isinf(min_conf)) {
    set_last_error("mk_mutual_matches: need non-NULL scores / matches / match_scores / count / workspace, B > 0, "
                   "2 <= N <= %d, pitch >= N and a finite min_conf (got B %d, N %d, pitch %lld, min_conf %g)",
                   MAX_SORT + 1, B, N, pitch, (double)min_conf);
    return MK_ERR_INVALID;
  }
  if (ws_bytes < mutual_matches_ws_bytes(B, N)) {
    set_last_error("mk_mutual_matches: workspace of %lld bytes, %lld needed", ws_bytes, mutual_matches_ws_bytes(B, N));
    return MK_ERR_INVALID;
  }
  const int W = N - 1, strips = ceil_div(W, STRIP_ROWS);
  Best* row_best = reinterpret_cast<Best*>(ws);
  Best* col_part = row_best + (size_t)B * W;
  const bool vec = pitch % 4 == 0 && reinterpret_cast<uintptr_t>(scores) % 16 == 0;
  const dim3 grid(strips, B);
  if (vec)
    MK_CUDA_CHECK(launch_k(mutual_strips_kernel<true>, grid, dim3(MM_WARPS * 32), 0, s, scores, pitch, N, strips, row_best, col_part));
  else
    MK_CUDA_CHECK(launch_k(mutual_strips_kernel<false>, grid, dim3(MM_WARPS * 32), 0, s, scores, pitch, N, strips, row_best, col_part));
  int n_sort = 2;
  while (n_sort < W) n_sort <<= 1;
  const size_t smem = (size_t)n_sort * sizeof(unsigned long long) + (size_t)W * sizeof(int);
  static unsigned long long configured = 0;
  if (first_use_on_device(configured))
    MK_CUDA_CHECK(cudaFuncSetAttribute(mutual_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)(MAX_SORT * sizeof(unsigned long long) + MAX_SORT * sizeof(int))));
  MK_CUDA_CHECK(launch_k(mutual_select_kernel, dim3(B), dim3(SELECT_THREADS), smem, s, row_best, col_part, N, strips, n_sort,
                         min_conf, matches, match_scores, count));
  return MK_OK;
}

}  // namespace mk
