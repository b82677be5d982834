// MicKey's training loss, the parts that are expensive and not differentiated (reference
// lib/models/MicKey/modules/loss/loss_class.py, MetricPoseLoss.RANSAC_vectorized):
//
//  1. outer draw  : IT_MATCHES x "NUM_SAMPLES_MATCHES of N*N cells ~ final_scores" (:136-138), the solver's sampler
//                   (ransac.cu sample_outer), plus the loss's own pre-check of the matrix (:126-131) as status bit 4.
//  2. hypotheses  : per (pair, outer iteration) one block gathers and back-projects its S cells (:140-152); each warp
//                   takes hypotheses: C of S without replacement ~ the cells' scores (:159), then the refinement of
//                   :163-196 (masked Kabsch, hard inliers at INLIER_REF_TH, the do_ref / inliers_pre / inliers_final
//                   bookkeeping).  Output: inliers_final as a bitmask and the drawn indices; the pose on that mask is
//                   recomputed with autograd by mickey_b200/loss.py.
//  3. gradient    : probs_grad = mask_b (sum_i [cell in S_i] loss_i - count baseline_b) / IM (:251-261, :299-316),
//                   dense [B, N, N], summed in iteration order without atomics.
#include "../../include/mickey_b200.h"
#include "ops.h"
#include "ransac_dev.cuh"

namespace mk {

namespace {

constexpr int LOSS_THREADS = 256;
constexpr int LOSS_WARPS = LOSS_THREADS / 32;
constexpr uint32_t LOSS_INNER_TAG = 0xA54FF53Au;     // 4th Philox counter of the inner draw (the solver's is 0x3c6ef372)

// hypotheses of one block: (pair b, outer iteration s_in) = blockIdx.x
__global__ void __launch_bounds__(LOSS_THREADS)
loss_hyp_kernel(const int* __restrict__ idx, const float* __restrict__ fs, long long pitch, const float* __restrict__ kps0,
                const float* __restrict__ d0, const float* __restrict__ kps1, const float* __restrict__ d1,
                const float* __restrict__ K0, const float* __restrict__ K1, int N, int IM, int IR, int S, int C, int n_ref,
                float th_ref, const int* __restrict__ inner_idx, const unsigned long long* __restrict__ seed_ptr,
                int* __restrict__ inner_out, uint32_t* __restrict__ inl_out, int* __restrict__ status) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ float sm[];
  float* X = sm;                 // [3][S]
  float* Y = sm + 3 * S;         // [3][S]
  float* cdf = sm + 6 * S;       // [S] inclusive prefix sums of the cells' scores
  __shared__ float warp_tot[LOSS_WARPS];
  __shared__ float Ki0[9], Ki1[9];
  __shared__ int drawn[LOSS_WARPS][LOSS_MAX_C], srt[LOSS_WARPS][LOSS_MAX_C];
  const int s = blockIdx.x, b = s / IM, s_in = s - b * IM;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int words = S / 32;
  // the pre-check failed (a NaN, inf or negative cell in the batch): the reference skips the search (:131)
  if (*(volatile int*)status & MK_LOSS_STATUS_PRECHECK) {
    for (int i = tid; i < IR * words; i += LOSS_THREADS) inl_out[(long long)s * IR * words + i] = 0u;
    for (int i = tid; i < IR * C; i += LOSS_THREADS) inner_out[(long long)s * IR * C + i] = -1;
    return;
  }
  if (tid == 0) { inv3x3(K0 + b * 9, Ki0); inv3x3(K1 + b * 9, Ki1); }
  __syncthreads();
  // gather_set's layout: thread t owns entries t * per + j < S, so at S < 256 (or S not a multiple of 256) the
  // trailing threads own none and add 0 to the scan
  const int per = (S + LOSS_THREADS - 1) / LOSS_THREADS;
  const int own = min(per, max(S - tid * per, 0));
  float run;
  gather_set(idx, fs, kps0, d0, kps1, d1, Ki0, Ki1, N, pitch, b, s, S, LOSS_THREADS, X, Y, cdf, run);
  float inc = run;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float v = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += v;
  }
  if (lane == 31) warp_tot[warp] = inc;
  __syncthreads();
  float base = inc - run;
  for (int w = 0; w < warp; ++w) base += warp_tot[w];
  for (int j = 0; j < own; ++j) cdf[tid * per + j] += base;
  __syncthreads();
  const float W = cdf[S - 1];
  // torch.multinomial raises on a row that sums to zero (:159; the reference's try/except then zeroes the batch)
  if (tid == 0 && !(W > 0.f)) atomicOr(status, MK_LOSS_STATUS_INNER);
  const Philox rng(*seed_ptr ^ 0x9E3779B97F4A7C15ull);
  auto weight = [&](int i) { return cdf[i] - ((i > 0) ? cdf[i - 1] : 0.f); };

  for (int h = warp; h < IR; h += LOSS_WARPS) {
    const long long gh = (long long)s * IR + h;
    // ---- C of S without replacement: successive sampling on the cdf (the solver's inner draw, from 3 to C entries)
    if (lane == 0) {
      if (inner_idx) {
        for (int k = 0; k < C; ++k) drawn[warp][k] = inner_idx[gh * C + k];
      } else {
        float removed = 0.f;
        uint4 r = make_uint4(0, 0, 0, 0);
        for (int k = 0; k < C; ++k) {
          if ((k & 3) == 0) r = rng((uint32_t)h, (uint32_t)s_in, (uint32_t)b, LOSS_INNER_TAG + (uint32_t)(k >> 2));
          const uint32_t bits = ((k & 3) == 0) ? r.x : ((k & 3) == 1) ? r.y : ((k & 3) == 2) ? r.z : r.w;
          float target = u01_from_bits(bits) * (W - removed);
          // skip the mass of already drawn entries, in ascending index order
          for (int j = 0; j < k; ++j) {
            const int a = srt[warp][j];
            const float ex = weight(a);
            if (target >= cdf[a] - ex) target += ex;
          }
          int pick = cdf_search(cdf, S, fminf(target, W * 0.99999994f));
          // rounding (or a set with fewer than C positive scores) may land on a drawn entry: advance to the next free one
          for (int guard = 0; guard < C; ++guard) {
            bool taken = false;
            for (int j = 0; j < k; ++j) taken |= (drawn[warp][j] == pick);
            if (!taken) break;
            pick = (pick + 1) % S;
          }
          drawn[warp][k] = pick;
          int j = k;                                   // insertion into the ascending copy
          while (j > 0 && srt[warp][j - 1] > pick) { srt[warp][j] = srt[warp][j - 1]; --j; }
          srt[warp][j] = pick;
          removed += weight(pick);
        }
      }
    }
    __syncwarp();
    // ---- the refinement (:163-196) on masks held as bits: lane owns entries lane + 32 k, k < S / 32
    unsigned long long cur = 0ull;
    for (int k = 0; k < C; ++k) {
      const int e = drawn[warp][k];
      if (e >= 0 && e < S && (e & 31) == lane) cur |= 1ull << (e >> 5);
    }
    unsigned long long fin = cur;
    int pre = C;                                       // inliers_pre starts at NUM_CORR_3d3d (:166)
    for (int it = 0; it < n_ref; ++it) {
      // weighted_procrustes(use_mask, w = cur) (solvers.py:13-29), moments in fp64
      double m[7] = {0, 0, 0, 0, 0, 0, 0};
      for (int k = 0; k < words; ++k)
        if ((cur >> k) & 1ull) {
          const int i = lane + 32 * k;
          m[0] += 1.0;
          m[1] += X[i]; m[2] += X[S + i]; m[3] += X[2 * S + i];
          m[4] += Y[i]; m[5] += Y[S + i]; m[6] += Y[2 * S + i];
        }
#pragma unroll
      for (int q = 0; q < 7; ++q)
#pragma unroll
        for (int o = 16; o; o >>= 1) m[q] += __shfl_xor_sync(0xffffffffu, m[q], o);
      const double wn = 1.0 / (m[0] + 1e-16);
      const double xm[3] = {m[1] * wn, m[2] * wn, m[3] * wn}, ym[3] = {m[4] * wn, m[5] * wn, m[6] * wn};
      double H[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
      for (int k = 0; k < words; ++k)
        if ((cur >> k) & 1ull) {
          const int i = lane + 32 * k;
          const double a[3] = {X[i] - xm[0], X[S + i] - xm[1], X[2 * S + i] - xm[2]};
          const double c[3] = {Y[i] - ym[0], Y[S + i] - ym[1], Y[2 * S + i] - ym[2]};
#pragma unroll
          for (int p = 0; p < 3; ++p)
#pragma unroll
            for (int q = 0; q < 3; ++q) H[p * 3 + q] += a[p] * c[q];
        }
#pragma unroll
      for (int q = 0; q < 9; ++q)
#pragma unroll
        for (int o = 16; o; o >>= 1) H[q] += __shfl_xor_sync(0xffffffffu, H[q], o);
      double Rd[9];
      kabsch_rotation(H, Rd);                          // replicated on every lane (same inputs, same result)
      float R[9], t[3];
#pragma unroll
      for (int i = 0; i < 9; ++i) R[i] = (float)Rd[i];
#pragma unroll
      for (int i = 0; i < 3; ++i) t[i] = (float)(ym[i] - (Rd[i * 3] * xm[0] + Rd[i * 3 + 1] * xm[1] + Rd[i * 3 + 2] * xm[2]));
      // hard inliers at INLIER_REF_TH (training_utils.py:71-75)
      unsigned long long ref = 0ull;
      for (int k = 0; k < words; ++k) {
        const int i = lane + 32 * k;
        const float x0 = X[i], x1 = X[S + i], x2 = X[2 * S + i];
        const float r0 = R[0] * x0 + R[1] * x1 + R[2] * x2 + t[0] - Y[i];
        const float r1 = R[3] * x0 + R[4] * x1 + R[5] * x2 + t[1] - Y[S + i];
        const float r2 = R[6] * x0 + R[7] * x1 + R[8] * x2 + t[2] - Y[2 * S + i];
        if (th_ref - sqrtf(r0 * r0 + r1 * r1 + r2 * r2 + 1e-6f) >= 0.f) ref |= 1ull << k;
      }
      int cnt = __popcll(ref);
#pragma unroll
      for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
      // do_ref = count > inliers_pre: inliers_final takes the mask that produced this pose, the next pose uses its
      // inliers (:189-192); a hypothesis that stops improving is never refined again
      if (cnt <= pre) break;
      pre = cnt; fin = cur; cur = ref;
    }
    uint32_t* dst = inl_out + gh * words;
    for (int w = 0; w < words; ++w) {
      const uint32_t word = __ballot_sync(0xffffffffu, (fin >> w) & 1ull);
      if (lane == (w & 31)) dst[w] = word;
    }
    if (lane < C) inner_out[gh * C + lane] = drawn[warp][lane];
    __syncwarp();                                      // drawn[warp] is rewritten by the next hypothesis
  }
}

// one block per stream: its S cells sorted ascending (bitonic in shared memory, padded to a power of two)
constexpr int SORT_THREADS = 512;
__global__ void __launch_bounds__(SORT_THREADS)
loss_sort_kernel(const int* __restrict__ idx, int S, int S2, int* __restrict__ sorted) {
  pdl_wait();
  pdl_trigger();
  __shared__ int v[LOSS_MAX_S];
  const int s = blockIdx.x;
  for (int i = threadIdx.x; i < S2; i += SORT_THREADS) v[i] = (i < S) ? idx[(long long)s * S + i] : 0x7fffffff;
  __syncthreads();
  for (int k = 2; k <= S2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < S2; i += SORT_THREADS) {
        const int p = i ^ j;
        if (p > i) {
          const int a = v[i], c = v[p];
          const bool asc = (i & k) == 0;
          if ((a > c) == asc) { v[i] = c; v[p] = a; }
        }
      }
      __syncthreads();
    }
  for (int i = threadIdx.x; i < S; i += SORT_THREADS) sorted[(long long)s * S + i] = v[i];
}

__device__ __forceinline__ bool sorted_contains(const int* a, int n, int c) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < c) lo = mid + 1; else hi = mid;
  }
  return lo < n && a[lo] == c;
}

// one thread per drawn (stream, entry): the first outer iteration that drew the cell writes it, summing the losses of
// every iteration that drew it in iteration order (the reference's `gradients += gradients_tmp`, :251-261), then
// - count * baseline, / IM, * mask_topk (:299-316), each rounded as the reference's separate tensor ops round it.
// Cells never drawn keep the zeros the caller's memset wrote.
__global__ void __launch_bounds__(256)
loss_grad_kernel(const int* __restrict__ sorted, const float* __restrict__ loss_value, const float* __restrict__ baseline,
                 const float* __restrict__ mask, int B, int IM, int S, long long cells, float* __restrict__ grad) {
  pdl_wait();
  pdl_trigger();
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)B * IM * S) return;
  const int s = (int)(g / S), b = s / IM, i = s - b * IM;
  const int c = sorted[g];
  if (c < 0 || (long long)c >= cells) return;
  if (g % S > 0 && sorted[g - 1] == c) return;          // a repeated cell within one set counts once (index_put)
  float acc = 0.f, cnt = 0.f;
  for (int i2 = 0; i2 < IM; ++i2) {
    if (i2 != i && !sorted_contains(sorted + ((long long)b * IM + i2) * S, S, c)) continue;
    if (i2 < i) return;                                 // an earlier iteration drew it: that thread writes
    acc = __fadd_rn(acc, loss_value[b * IM + i2]);
    cnt += 1.f;
  }
  const float v = __fsub_rn(acc, __fmul_rn(cnt, baseline[b]));
  grad[(long long)b * cells + c] = __fmul_rn(__fdiv_rn(v, (float)IM), mask[b]);
}

}  // namespace

long long loss_search_ws_bytes(int B, int IM) { return (long long)sampler_workspace_bytes(B, IM) + 512; }

int loss_search(const float* fs, long long pitch, const float* kps0, const float* d0, const float* kps1, const float* d1,
                const float* K0, const float* K1, int B, int N, int IM, int IR, int S, int C, int n_ref, float th_ref,
                unsigned long long seed, const int* outer_idx, const int* inner_idx, int* sampled_out, int* inner_out,
                uint32_t* inl_out, int* status, void* ws, long long ws_bytes, cudaStream_t st) {
  MK_TRY(resolve_pitch(pitch, N, "mk_loss_search: pitch"));
  if (!fs || !kps0 || !d0 || !kps1 || !d1 || !K0 || !K1 || !sampled_out || !inner_out || !inl_out || !status || !ws || B <= 0 ||
      N <= 0 || IM <= 0 || IR <= 0 || n_ref < 0 || S <= 0 || S % 32 || S > LOSS_MAX_S || C < 1 ||
      C > LOSS_MAX_C || C > S || (long long)N * N < S || (long long)N * N > 0x7fffffffLL || !(th_ref == th_ref)) {
    // S % 32: the inlier masks are whole 32-bit words, one bit per set entry
    set_last_error("mk_loss_search: need non-NULL inputs, outputs, status and workspace, B, N, IM, IR > 0, pitch >= N, "
                   "n_ref >= 0, S a multiple of 32 up to %d and <= N*N, 1 <= C <= min(%d, S), N*N < 2^31 and th_ref not NaN "
                   "(got B %d N %d pitch %lld IM %d IR %d S %d C %d n_ref %d)", LOSS_MAX_S, LOSS_MAX_C, B, N, pitch, IM, IR,
                   S, C, n_ref);
    return MK_ERR_INVALID;
  }
  if (ws_bytes < loss_search_ws_bytes(B, IM)) {
    set_last_error("mk_loss_search: workspace of %lld bytes, %lld needed", ws_bytes, loss_search_ws_bytes(B, IM));
    return MK_ERR_INVALID;
  }
  MK_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int), st));
  const size_t off = ((size_t)sampler_workspace_bytes(B, IM) + 255) & ~(size_t)255;      // seed word after the sampler's
  unsigned long long* sd = reinterpret_cast<unsigned long long*>(reinterpret_cast<uint8_t*>(ws) + off);
  if (const int rc = seed_set(sd, seed, st)) return rc;
  // the sampler always runs: its histogram pass decides status bits 0 and 4 for injected draws too
  if (const int rc = sample_outer(fs, B, N, pitch, IM, S, sd, ws, sampled_out, status, st, 1 | MK_LOSS_STATUS_PRECHECK)) return rc;
  if (outer_idx)
    MK_CUDA_CHECK(cudaMemcpyAsync(sampled_out, outer_idx, (size_t)B * IM * S * sizeof(int), cudaMemcpyDeviceToDevice, st));
  const size_t smem = (size_t)7 * S * sizeof(float);
  static unsigned long long configured = 0;
  if (first_use_on_device(configured))
    MK_CUDA_CHECK(cudaFuncSetAttribute(loss_hyp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 7 * LOSS_MAX_S * 4));
  MK_CUDA_CHECK(launch_k(loss_hyp_kernel, dim3(B * IM), dim3(LOSS_THREADS), smem, st, (const int*)sampled_out, fs, pitch, kps0,
                         d0, kps1, d1, K0, K1, N, IM, IR, S, C, n_ref, th_ref, inner_idx, (const unsigned long long*)sd, inner_out,
                         inl_out, status));
  return MK_OK;
}

long long loss_gradient_ws_bytes(int B, int IM, int S) {
  return (B <= 0 || IM <= 0 || S <= 0) ? 0 : (long long)B * IM * S * (long long)sizeof(int);
}

int loss_gradient(const int* sampled, const float* loss_value, const float* baseline, const float* mask, int B, int N, int IM,
                  int S, float* grad, void* ws, long long ws_bytes, cudaStream_t st) {
  if (!sampled || !loss_value || !baseline || !mask || !grad || !ws || B <= 0 || N <= 0 || IM <= 0 || S <= 0 ||
      S > LOSS_MAX_S || (long long)N * N > 0x7fffffffLL) {
    set_last_error("mk_loss_gradient: need non-NULL inputs, output and workspace, B, N, IM > 0, 0 < S <= %d and N*N < 2^31 "
                   "(got B %d N %d IM %d S %d)", LOSS_MAX_S, B, N, IM, S);
    return MK_ERR_INVALID;
  }
  if (ws_bytes < loss_gradient_ws_bytes(B, IM, S)) {
    set_last_error("mk_loss_gradient: workspace of %lld bytes, %lld needed", ws_bytes, loss_gradient_ws_bytes(B, IM, S));
    return MK_ERR_INVALID;
  }
  const long long cells = (long long)N * N;
  int* sorted = reinterpret_cast<int*>(ws);
  int S2 = 1;
  while (S2 < S) S2 <<= 1;
  MK_CUDA_CHECK(cudaMemsetAsync(grad, 0, (size_t)B * cells * sizeof(float), st));
  MK_CUDA_CHECK(launch_k(loss_sort_kernel, dim3(B * IM), dim3(SORT_THREADS), 0, st, sampled, S, S2, sorted));
  const long long n = (long long)B * IM * S;
  MK_CUDA_CHECK(launch_k(loss_grad_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, (const int*)sorted, loss_value,
                         baseline, mask, B, IM, S, cells, grad));
  return MK_OK;
}

}  // namespace mk
