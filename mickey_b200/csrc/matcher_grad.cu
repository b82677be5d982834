// The dual-softmax matcher on the caller's descriptors, and its backward (include/mickey_b200.h mk_dual_softmax*).
// Reference: dualSoftmax.forward (lib/models/MicKey/modules/utils/feature_matcher.py:64-83), kp_matrix_scores
// (compute_correspondences.py:46-50) and final_scores = scores * kp_scores (model.py:201).
//
// Forward: the descriptors are split into the hi / lo fp16 operands of desc_out_kernel, then the three launches of mk_match
// run unchanged (EPI_LSE -> matcher_lse_reduce -> EPI_DUAL), so the outputs are bit-identical to mk_match.
//
// Backward (DESIGN.md §6e).  Per pair, s_ij = <d0_i, d1_j> / T, augmented by the dustbin alpha; r_i / c_j the row / column
// log-sum-exps (the forward's lse_r / lse_c, log2 domain); P = exp(s - r), Q = exp(s - c), scores = P Q, kp = sig0_i sig1_j.
//   w_ij = (Gs + Gf kp) scores,  h_ij = Gk + Gf scores,  W_i = sum_j w_ij,  W'_j = sum_i w_ij
//   dS_ij = 2 w_ij - P_ij W_i - Q_ij W'_j
//   dd0_i = (1/T) sum_j dS_ij d1_j,  dd1_j = (1/T) sum_i dS_ij d0_i,  dsig0_i = sum_j h_ij sig1_j,  dsig1_j = sum_i h_ij sig0_i
//   dalpha = -sum_pairs [ sum_i e^(alpha - r_i) W_i + sum_j e^(alpha - c_j) W'_j ]
// Three passes, all in fp32 FMA (dS needs the fp32 exponent range: P W sits far below fp16's normals), none of which writes
// an N x N intermediate:
//   1. stats    : one CTA per 64 x 64 tile of (i, j) recomputes S, reads the tile of each given gradient and writes the
//                 tile's row partials (W, dsig0) and column partials (W', dsig1) to fixed slots;
//   2. fold     : sums the slots in index order; forms the alpha terms; one block sums those in pair order;
//   3. contract : one CTA per 64-keypoint block of one axis walks every tile of the other axis, recomputes S, forms dS in
//                 shared memory and accumulates dS (x) the other image's descriptors into a 64 x 128 fp32 block.
// No atomics: every sum has a fixed order, so the outputs are bit-identical run to run, and a pair's dd / dsig do not
// depend on the other pairs of the batch.
#include "../../include/mickey_b200.h"
#include "gemm.h"
#include "ops.h"

#include <cstring>

namespace mk {

namespace {

constexpr int DSM_MAX_N = 8192;
constexpr int DC = 128;                // descriptor channels
constexpr int TG = 64;                 // tile edge in keypoints
constexpr int LDT = TG + 1;            // shared-memory row stride (conflict-free column reads)
constexpr int GT = 256;                // threads per CTA: (ty, tx) = (tid / 16, tid % 16), 4 x 4 cells each
constexpr float LOG2E = 1.4426950408889634f;
constexpr size_t TILE_FLOATS = (size_t)DC * LDT;
constexpr size_t STATS_SMEM = 2 * TILE_FLOATS * sizeof(float);
constexpr size_t CONTRACT_SMEM = (2 * TILE_FLOATS + (size_t)TG * LDT) * sizeof(float);

int npad128(int N) { return ceil_div(N, 128) * 128; }
int ntiles(int N) { return ceil_div(N, TG); }

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// ---- forward operands ---------------------------------------------------------------------------------------------
// Block (x, b, r): tokens [32x, 32x + 32) of pair b, role r.  dsc fp32 [B, 128, N] -> dsc_x fp16 [(r*B + b)*N + tok, 384]
// split exactly as desc_out_kernel / bank_gather_kernel do (role 0 [hi | lo | hi], role 1 [hi | hi | lo]);
// scr [B, N] (or 1 when NULL) -> scr_out [(r*B + b)*N + tok].
__global__ void __launch_bounds__(256)
dsm_operands_kernel(const float* __restrict__ d0, const float* __restrict__ d1, const float* __restrict__ s0,
                    const float* __restrict__ s1, int B, int N, __half* __restrict__ dsc_x, float* __restrict__ scr_out) {
  __shared__ float tile[128][33];
  pdl_wait();
  pdl_trigger();
  const int r = blockIdx.z, b = blockIdx.y, n0 = blockIdx.x * 32, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const long long orow = (long long)r * B + b;
  const float* src = (r ? d1 : d0) + (size_t)b * 128 * N;
  const float* scr = r ? s1 : s0;
  if (t < 32 && n0 + lane < N) scr_out[orow * N + n0 + lane] = scr ? __ldg(scr + (size_t)b * N + n0 + lane) : 1.0f;
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    const int c = warp + 8 * k, n = n0 + lane;
    tile[c][lane] = n < N ? __ldg(src + (size_t)c * N + n) : 0.f;
  }
  __syncthreads();
  for (int j = warp; j < 32 && n0 + j < N; j += 8) {
    __half* dst = dsc_x + (orow * N + n0 + j) * 384;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int c = 64 * half + 2 * lane;
      const float v0 = tile[c][j], v1 = tile[c + 1][j];
      const __half h0 = __float2half_rn(v0), h1 = __float2half_rn(v1);
      const __half2 hi = __halves2half2(h0, h1);
      const __half2 lo = __halves2half2(__float2half_rn(v0 - __half2float(h0)), __float2half_rn(v1 - __half2float(h1)));
      *reinterpret_cast<__half2*>(dst + c) = hi;
      *reinterpret_cast<__half2*>(dst + 128 + c) = r ? hi : lo;
      *reinterpret_cast<__half2*>(dst + 256 + c) = r ? lo : hi;
    }
  }
}

struct FwdLayout { size_t dsc_x, scr, part_row, part_col, total; };
FwdLayout fwd_layout(int B, int N) {
  const size_t np = (size_t)npad128(N);
  FwdLayout L;
  L.dsc_x = 0;
  L.scr = align256(L.dsc_x + (size_t)2 * B * N * 384 * sizeof(__half));
  L.part_row = align256(L.scr + (size_t)2 * B * N * sizeof(float));
  L.part_col = align256(L.part_row + (size_t)B * (np / 64) * np * sizeof(float2));
  L.total = align256(L.part_col + (size_t)B * (np / 32) * np * sizeof(float2));
  return L;
}

// ---- backward ---------------------------------------------------------------------------------------------------------
struct GradArgs {
  const float* d0; const float* d1;          // [B, 128, N]
  const float* s0; const float* s1;          // [B, N] or NULL (kp = 1)
  const float* lse_r; const float* lse_c;    // [B, lse_ld], log2 domain
  const float* gs; const float* gk; const float* gf;   // [B, N, ld] or NULL
  long long gs_ld, gk_ld, gf_ld;
  int N, lse_ld, nt, np;                     // nt tiles of TG; np = nt * TG (slot row length)
  float k2, inv_t;                           // log2(e) / T, 1 / T
  float2* rowpart; float2* colpart;          // [B][nt][np]: (W, dsig0) per (column tile, row), (W', dsig1) per (row tile, column)
  const float* Wr; const float* Wc;          // [B][np]
};

struct BwdLayout { size_t rowpart, colpart, Wr, Wc, aterm, total; };
BwdLayout bwd_layout(int B, int N) {
  const size_t nt = (size_t)ntiles(N), np = nt * TG;
  BwdLayout L;
  L.rowpart = 0;
  L.colpart = align256(L.rowpart + (size_t)B * nt * np * sizeof(float2));
  L.Wr = align256(L.colpart + (size_t)B * nt * np * sizeof(float2));
  L.Wc = align256(L.Wr + (size_t)B * np * sizeof(float));
  L.aterm = align256(L.Wc + (size_t)B * np * sizeof(float));
  L.total = align256(L.aterm + (size_t)B * 2 * np * sizeof(float));
  return L;
}

// dst[c * LDT + t] = d[c][n0 + t] for t < TG (0 beyond N); d is one image's [128][N] block
__device__ __forceinline__ void load_tile(const float* __restrict__ d, int N, int n0, float* __restrict__ dst) {
  for (int k = threadIdx.x; k < DC * TG; k += GT) {
    const int c = k / TG, t = k % TG, n = n0 + t;
    dst[c * LDT + t] = n < N ? __ldg(d + (size_t)c * N + n) : 0.f;
  }
}

// s[a][b] = sum_c A[c][ty + 16 a] * Bm[c][tx + 16 b], c in ascending order
__device__ __forceinline__ void s_tile(const float* __restrict__ A, const float* __restrict__ Bm, int ty, int tx, float (&s)[4][4]) {
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) s[a][b] = 0.f;
#pragma unroll 8
  for (int c = 0; c < DC; ++c) {
    float av[4], bv[4];
#pragma unroll
    for (int a = 0; a < 4; ++a) av[a] = A[c * LDT + ty + 16 * a];
#pragma unroll
    for (int b = 0; b < 4; ++b) bv[b] = Bm[c * LDT + tx + 16 * b];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) s[a][b] = fmaf(av[a], bv[b], s[a][b]);
  }
}

__device__ __forceinline__ float grad_at(const float* g, long long ld, int N, int pb, int i, int j) {
  return __ldg(g + ((size_t)pb * N + i) * (size_t)ld + j);
}

// Pass 1.  grid (column tile jt, row tile it, pair), dynamic smem STATS_SMEM.
__global__ void __launch_bounds__(GT)
dsm_grad_stats_kernel(GradArgs a) {
  extern __shared__ float sm[];
  __shared__ float2 colred[GT / 32][TG];
  pdl_wait();
  pdl_trigger();
  float* A = sm;
  float* Bm = sm + TILE_FLOATS;
  const int jt = blockIdx.x, it = blockIdx.y, pb = blockIdx.z, N = a.N;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int i0 = it * TG, j0 = jt * TG;
  load_tile(a.d0 + (size_t)pb * DC * N, N, i0, A);
  load_tile(a.d1 + (size_t)pb * DC * N, N, j0, Bm);
  __syncthreads();
  float s[4][4];
  s_tile(A, Bm, ty, tx, s);
  float lr[4], lc[4], s0v[4], s1v[4];
  bool iok[4], jok[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int i = i0 + ty + 16 * q, j = j0 + tx + 16 * q;
    iok[q] = i < N; jok[q] = j < N;
    lr[q] = iok[q] ? __ldg(a.lse_r + (size_t)pb * a.lse_ld + i) : 0.f;
    lc[q] = jok[q] ? __ldg(a.lse_c + (size_t)pb * a.lse_ld + j) : 0.f;
    s0v[q] = (a.s0 && iok[q]) ? __ldg(a.s0 + (size_t)pb * N + i) : 1.f;
    s1v[q] = (a.s1 && jok[q]) ? __ldg(a.s1 + (size_t)pb * N + j) : 1.f;
  }
  float wr[4], hr[4], wc[4], hc[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) { wr[q] = 0.f; hr[q] = 0.f; wc[q] = 0.f; hc[q] = 0.f; }
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (!(iok[p] && jok[q])) continue;
      const int i = i0 + ty + 16 * p, j = j0 + tx + 16 * q;
      const float x = s[p][q] * a.k2;
      const float P = exp2f(x - lr[p]), Q = exp2f(x - lc[q]), sc = P * Q;
      const float kp = s0v[p] * s1v[q];
      const float gs = a.gs ? grad_at(a.gs, a.gs_ld, N, pb, i, j) : 0.f;
      const float gk = a.gk ? grad_at(a.gk, a.gk_ld, N, pb, i, j) : 0.f;
      const float gf = a.gf ? grad_at(a.gf, a.gf_ld, N, pb, i, j) : 0.f;
      const float w = (gs + gf * kp) * sc, h = gk + gf * sc;
      wr[p] += w; hr[p] += h * s1v[q];
      wc[q] += w; hc[q] += h * s0v[p];
    }
  // rows: the 16 threads of a row (lane bits 0-3) hold its 64 columns
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int o = 8; o >= 1; o >>= 1) {
      wr[p] += __shfl_xor_sync(0xffffffffu, wr[p], o);
      hr[p] += __shfl_xor_sync(0xffffffffu, hr[p], o);
    }
  if (tx == 0) {
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int i = i0 + ty + 16 * p;
      if (i < N) a.rowpart[((size_t)pb * a.nt + jt) * a.np + i] = make_float2(wr[p], hr[p]);
    }
  }
  // columns: the two ty of a warp (lane bit 4), then the 8 warps in order
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    wc[q] += __shfl_xor_sync(0xffffffffu, wc[q], 16);
    hc[q] += __shfl_xor_sync(0xffffffffu, hc[q], 16);
  }
  if ((tid & 16) == 0) {
#pragma unroll
    for (int q = 0; q < 4; ++q) colred[tid >> 5][tx + 16 * q] = make_float2(wc[q], hc[q]);
  }
  __syncthreads();
  if (tid < TG && j0 + tid < N) {
    float2 v = colred[0][tid];
#pragma unroll
    for (int w = 1; w < GT / 32; ++w) { v.x += colred[w][tid].x; v.y += colred[w][tid].y; }
    a.colpart[((size_t)pb * a.nt + it) * a.np + j0 + tid] = v;
  }
}

// Pass 2.  grid (ceil(N / 256), B, 2): z = 0 rows, z = 1 columns; the slots are summed in index order.
__global__ void __launch_bounds__(256)
dsm_grad_fold_kernel(const float2* __restrict__ rowpart, const float2* __restrict__ colpart, const float* __restrict__ lse_r,
                     const float* __restrict__ lse_c, const float* __restrict__ dustbin, int N, int nt, int np, int lse_ld,
                     float* __restrict__ Wr, float* __restrict__ Wc, float* __restrict__ dscr0, float* __restrict__ dscr1,
                     float* __restrict__ aterm) {
  pdl_wait();
  pdl_trigger();
  const int i = blockIdx.x * 256 + threadIdx.x, pb = blockIdx.y, z = blockIdx.z;
  if (i >= N) return;
  const float2* src = (z ? colpart : rowpart) + (size_t)pb * nt * np + i;
  float W = 0.f, D = 0.f;
  for (int t = 0; t < nt; ++t) {
    const float2 v = __ldg(src + (size_t)t * np);
    W += v.x; D += v.y;
  }
  (z ? Wc : Wr)[(size_t)pb * np + i] = W;
  float* ds = z ? dscr1 : dscr0;
  if (ds) ds[(size_t)pb * N + i] = D;
  if (dustbin) {
    const float l = __ldg((z ? lse_c : lse_r) + (size_t)pb * lse_ld + i);
    aterm[((size_t)pb * 2 + z) * np + i] = exp2f(__ldg(dustbin) * LOG2E - l) * W;
  }
}

// dalpha = -(sum over pairs, in pair order, of each pair's row and column terms).  One block.
__global__ void __launch_bounds__(256)
dsm_grad_alpha_kernel(const float* __restrict__ aterm, int B, int N, int np, float* __restrict__ ddustbin) {
  __shared__ float red[256];
  pdl_wait();
  pdl_trigger();
  const int tid = threadIdx.x;
  float total = 0.f;
  for (int pb = 0; pb < B; ++pb) {
    float acc = 0.f;
    for (int z = 0; z < 2; ++z)
      for (int i = tid; i < N; i += 256) acc += __ldg(aterm + ((size_t)pb * 2 + z) * np + i);
    red[tid] = acc;
    __syncthreads();
    for (int o = 128; o >= 1; o >>= 1) {
      if (tid < o) red[tid] += red[tid + o];
      __syncthreads();
    }
    if (tid == 0) total += red[0];
    __syncthreads();
  }
  if (tid == 0) *ddustbin = -total;
}

// Pass 3.  ROLE 0: a CTA owns 64 rows i and gives dd0; ROLE 1: 64 columns j and gives dd1.  grid (ntiles, B), dynamic smem
// CONTRACT_SMEM: own descriptors [128][LDT], the other image's tile [128][LDT], dS [64 i][LDT].
template <int ROLE>
__global__ void __launch_bounds__(GT, 2)
dsm_grad_contract_kernel(GradArgs a, float* __restrict__ out) {
  extern __shared__ float sm[];
  pdl_wait();
  pdl_trigger();
  float* own = sm;
  float* oth = sm + TILE_FLOATS;
  float* dS = sm + 2 * TILE_FLOATS;
  const int o0 = blockIdx.x * TG, pb = blockIdx.y, N = a.N;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const float* d_own = (ROLE ? a.d1 : a.d0) + (size_t)pb * DC * N;
  const float* d_oth = (ROLE ? a.d0 : a.d1) + (size_t)pb * DC * N;
  load_tile(d_own, N, o0, own);
  float acc[4][8];
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int q = 0; q < 8; ++q) acc[p][q] = 0.f;
  for (int t = 0; t < a.nt; ++t) {
    const int x0 = t * TG;
    const int i0 = ROLE ? x0 : o0, j0 = ROLE ? o0 : x0;
    __syncthreads();                                     // the previous tile's contraction is done with oth / dS
    load_tile(d_oth, N, x0, oth);
    __syncthreads();
    float s[4][4];
    s_tile(ROLE ? oth : own, ROLE ? own : oth, ty, tx, s);
    float lr[4], lc[4], wi[4], wj[4], s0v[4], s1v[4];
    bool iok[4], jok[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int i = i0 + ty + 16 * q, j = j0 + tx + 16 * q;
      iok[q] = i < N; jok[q] = j < N;
      lr[q] = iok[q] ? __ldg(a.lse_r + (size_t)pb * a.lse_ld + i) : 0.f;
      lc[q] = jok[q] ? __ldg(a.lse_c + (size_t)pb * a.lse_ld + j) : 0.f;
      wi[q] = iok[q] ? __ldg(a.Wr + (size_t)pb * a.np + i) : 0.f;
      wj[q] = jok[q] ? __ldg(a.Wc + (size_t)pb * a.np + j) : 0.f;
      s0v[q] = (a.s0 && iok[q]) ? __ldg(a.s0 + (size_t)pb * N + i) : 1.f;
      s1v[q] = (a.s1 && jok[q]) ? __ldg(a.s1 + (size_t)pb * N + j) : 1.f;
    }
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float d = 0.f;
        if (iok[p] && jok[q]) {
          const int i = i0 + ty + 16 * p, j = j0 + tx + 16 * q;
          const float x = s[p][q] * a.k2;
          const float P = exp2f(x - lr[p]), Q = exp2f(x - lc[q]), sc = P * Q;
          const float gs = a.gs ? grad_at(a.gs, a.gs_ld, N, pb, i, j) : 0.f;
          const float gf = a.gf ? grad_at(a.gf, a.gf_ld, N, pb, i, j) : 0.f;
          const float w = (gs + gf * (s0v[p] * s1v[q])) * sc;
          d = 2.f * w - P * wi[p] - Q * wj[q];
        }
        dS[(ty + 16 * p) * LDT + tx + 16 * q] = d;
      }
    __syncthreads();
    // acc[own ty + 16 p][channel tx + 16 q] += sum_k dS(own, k) * oth[channel][k], k in ascending order
#pragma unroll 4
    for (int k = 0; k < TG; ++k) {
      float dv[4], ov[8];
#pragma unroll
      for (int p = 0; p < 4; ++p) dv[p] = ROLE ? dS[k * LDT + ty + 16 * p] : dS[(ty + 16 * p) * LDT + k];
#pragma unroll
      for (int q = 0; q < 8; ++q) ov[q] = oth[(tx + 16 * q) * LDT + k];
#pragma unroll
      for (int p = 0; p < 4; ++p)
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[p][q] = fmaf(dv[p], ov[q], acc[p][q]);
    }
  }
  __syncthreads();
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int q = 0; q < 8; ++q) oth[(tx + 16 * q) * LDT + ty + 16 * p] = acc[p][q] * a.inv_t;
  __syncthreads();
  for (int k = tid; k < DC * TG; k += GT) {
    const int c = k / TG, t = k % TG, n = o0 + t;
    if (n < N) out[((size_t)pb * DC + c) * N + n] = oth[c * LDT + t];
  }
}

bool bad_temperature(float T) { return !(T > 0.f) || !(1.0f / T < 3.0e38f); }

int set_smem_attributes() {
  static unsigned long long done = 0;
  if (!first_use_on_device(done)) return MK_OK;
  MK_CUDA_CHECK(cudaFuncSetAttribute(dsm_grad_stats_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)STATS_SMEM));
  MK_CUDA_CHECK(cudaFuncSetAttribute(dsm_grad_contract_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CONTRACT_SMEM));
  MK_CUDA_CHECK(cudaFuncSetAttribute(dsm_grad_contract_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CONTRACT_SMEM));
  return MK_OK;
}

}  // namespace

}  // namespace mk

using namespace mk;

long long mk_dual_softmax_ws_bytes(int B, int N) {
  if (B < 1 || N < 2 || N > DSM_MAX_N) return 0;
  return (long long)fwd_layout(B, N).total;
}

long long mk_dual_softmax_backward_ws_bytes(int B, int N) {
  if (B < 1 || N < 2 || N > DSM_MAX_N) return 0;
  return (long long)bwd_layout(B, N).total;
}

int mk_dual_softmax(const float* dsc0, const float* dsc1, const float* scr0, const float* scr1, const float* dustbin,
                    float temperature, int B, int N, int unit_norm, float* scores, float* kp_scores, float* final_scores,
                    long long nn_pitch, float* lse_r, float* lse_c, void* ws, long long ws_bytes, void* stream) {
  if (!dsc0 || !dsc1 || !lse_r || !lse_c || !ws || B < 1 || N < 2 || N > DSM_MAX_N || bad_temperature(temperature) ||
      (scr0 == nullptr) != (scr1 == nullptr)) {
    set_last_error("mk_dual_softmax: need dsc0, dsc1, lse_r, lse_c and a workspace, B >= 1, 2 <= N <= %d, a positive finite "
                   "temperature, and scr0 / scr1 both given or both NULL (got B %d N %d T %g)", DSM_MAX_N, B, N, (double)temperature);
    return MK_ERR_INVALID;
  }
  // outputs: all three (scr required), final_scores alone, or scores alone
  const bool full = scores && kp_scores && final_scores, only_final = !scores && !kp_scores && final_scores,
             only_scores = scores && !kp_scores && !final_scores;
  if (!(full || only_final || only_scores) || (full && !scr0)) {
    set_last_error("mk_dual_softmax: write scores, kp_scores and final_scores together (with scr0 / scr1), final_scores "
                   "alone, or scores alone");
    return MK_ERR_INVALID;
  }
  if (nn_pitch <= 0) nn_pitch = N;
  if (nn_pitch < N) { set_last_error("mk_dual_softmax: nn_pitch %lld < N %d", nn_pitch, N); return MK_ERR_INVALID; }
  const FwdLayout L = fwd_layout(B, N);
  if (ws_bytes < (long long)L.total) {
    set_last_error("mk_dual_softmax: workspace of %lld bytes, %lld needed", ws_bytes, (long long)L.total);
    return MK_ERR_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* w = reinterpret_cast<uint8_t*>(ws);
  __half* dsc_x = reinterpret_cast<__half*>(w + L.dsc_x);
  float* scr = reinterpret_cast<float*>(w + L.scr);
  // scores alone leave through the lean path with kp = 1 * 1, so final_scores = scores exactly
  const bool use_scr = scr0 && !only_scores;
  MK_CUDA_CHECK(launch_k(dsm_operands_kernel, dim3(ceil_div(N, 32), B, 2), dim3(256), 0, st, dsc0, dsc1, use_scr ? scr0 : nullptr,
                         use_scr ? scr1 : nullptr, B, N, dsc_x, scr));
  float* out_final = only_scores ? scores : final_scores;
  float* out_scores = full ? scores : nullptr;
  float* out_kp = full ? kp_scores : nullptr;
  const int npad = npad128(N);
  const float inv_t = 1.0f / temperature;
  const long long rows = (long long)B * N;
  GemmOperand A0{dsc_x, rows, 384, 384}, A1{dsc_x + (size_t)rows * 384, rows, 384, 384};
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.M = N; p.N = N; p.k_chunks = 384 / 64; p.chunks_per_tap = p.k_chunks; p.num_taps = 1;
  p.groups = B; p.a_row_group_off = N; p.b_row_group_off = N; p.n_valid = N; p.inv_temp = inv_t; p.part_ld = npad;
  GemmParams p1 = p;
  p1.part_row = reinterpret_cast<float2*>(w + L.part_row);
  p1.part_col = reinterpret_cast<float2*>(w + L.part_col);
  p1.lse_bound = (unit_norm && inv_t <= 25.0f) ? 1.001f : 0.0f;     // mk_match's rule for DSC_HEAD.NORM_DSC
  int rc = launch_gemm(EPI_LSE, A0, A1, p1, st, GEMM_IMPL_TC);
  if (rc != MK_OK) return rc;
  rc = matcher_lse_reduce(p1.part_row, p1.part_col, dustbin, B, N, npad, lse_r, lse_c, st);
  if (rc != MK_OK) return rc;
  GemmParams p2 = p;
  p2.lse_r = lse_r; p2.lse_c = lse_c; p2.scr0 = scr; p2.scr1 = scr + (size_t)B * N;
  p2.scores = out_scores; p2.kp_scores = out_kp; p2.final_scores = out_final; p2.out_pitch = nn_pitch;
  p2.out_tma = (nn_pitch % 4 == 0 && reinterpret_cast<uintptr_t>(out_final) % 16 == 0 &&
                (!out_scores || (reinterpret_cast<uintptr_t>(out_scores) % 16 == 0 && reinterpret_cast<uintptr_t>(out_kp) % 16 == 0))) ? 1 : 0;
  return launch_gemm(EPI_DUAL, A0, A1, p2, st, GEMM_IMPL_TC);
}

int mk_dual_softmax_backward(const float* dsc0, const float* dsc1, const float* scr0, const float* scr1, const float* dustbin,
                             float temperature, int B, int N, const float* lse_r, const float* lse_c, const float* grad_scores,
                             long long gs_pitch, const float* grad_kp, long long gk_pitch, const float* grad_final,
                             long long gf_pitch, float* ddsc0, float* ddsc1, float* dscr0, float* dscr1, float* ddustbin,
                             void* ws, long long ws_bytes, void* stream) {
  if (!dsc0 || !dsc1 || !lse_r || !lse_c || !ddsc0 || !ddsc1 || !ws || B < 1 || N < 2 || N > DSM_MAX_N ||
      bad_temperature(temperature) || (scr0 == nullptr) != (scr1 == nullptr)) {
    set_last_error("mk_dual_softmax_backward: need dsc0, dsc1, lse_r, lse_c, ddsc0, ddsc1 and a workspace, B >= 1, "
                   "2 <= N <= %d, a positive finite temperature, and scr0 / scr1 both given or both NULL (got B %d N %d T %g)",
                   DSM_MAX_N, B, N, (double)temperature);
    return MK_ERR_INVALID;
  }
  if (!grad_scores && !grad_kp && !grad_final) {
    set_last_error("mk_dual_softmax_backward: at least one of grad_scores, grad_kp, grad_final is needed");
    return MK_ERR_INVALID;
  }
  if (scr0 ? (!dscr0 || !dscr1) : (grad_kp != nullptr)) {
    set_last_error("mk_dual_softmax_backward: with scr0 / scr1, dscr0 and dscr1 are required; without them there is no "
                   "kp_scores, so grad_kp must be NULL");
    return MK_ERR_INVALID;
  }
  if (dustbin && !ddustbin) { set_last_error("mk_dual_softmax_backward: the dustbin needs ddustbin"); return MK_ERR_INVALID; }
  long long* pitch[3] = {&gs_pitch, &gk_pitch, &gf_pitch};
  for (long long* pp : pitch) {
    if (*pp <= 0) *pp = N;
    if (*pp < N) { set_last_error("mk_dual_softmax_backward: gradient pitch %lld < N %d", *pp, N); return MK_ERR_INVALID; }
  }
  const BwdLayout L = bwd_layout(B, N);
  if (ws_bytes < (long long)L.total) {
    set_last_error("mk_dual_softmax_backward: workspace of %lld bytes, %lld needed", ws_bytes, (long long)L.total);
    return MK_ERR_INVALID;
  }
  {
    const int rc = set_smem_attributes();
    if (rc != MK_OK) return rc;
  }
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* w = reinterpret_cast<uint8_t*>(ws);
  GradArgs a;
  a.d0 = dsc0; a.d1 = dsc1; a.s0 = scr0; a.s1 = scr1; a.lse_r = lse_r; a.lse_c = lse_c;
  a.gs = grad_scores; a.gk = grad_kp; a.gf = grad_final; a.gs_ld = gs_pitch; a.gk_ld = gk_pitch; a.gf_ld = gf_pitch;
  a.N = N; a.lse_ld = npad128(N); a.nt = ntiles(N); a.np = a.nt * TG;
  a.inv_t = 1.0f / temperature; a.k2 = a.inv_t * LOG2E;
  a.rowpart = reinterpret_cast<float2*>(w + L.rowpart); a.colpart = reinterpret_cast<float2*>(w + L.colpart);
  float* Wr = reinterpret_cast<float*>(w + L.Wr);
  float* Wc = reinterpret_cast<float*>(w + L.Wc);
  float* aterm = reinterpret_cast<float*>(w + L.aterm);
  a.Wr = Wr; a.Wc = Wc;
  MK_CUDA_CHECK(launch_k(dsm_grad_stats_kernel, dim3(a.nt, a.nt, B), dim3(GT), STATS_SMEM, st, a));
  MK_CUDA_CHECK(launch_k(dsm_grad_fold_kernel, dim3(ceil_div(N, 256), B, 2), dim3(256), 0, st, (const float2*)a.rowpart,
                         (const float2*)a.colpart, lse_r, lse_c, dustbin, N, a.nt, a.np, a.lse_ld, Wr, Wc, scr0 ? dscr0 : nullptr,
                         scr0 ? dscr1 : nullptr, aterm));
  if (dustbin) MK_CUDA_CHECK(launch_k(dsm_grad_alpha_kernel, dim3(1), dim3(256), 0, st, (const float*)aterm, B, N, a.np, ddustbin));
  MK_CUDA_CHECK(launch_k(dsm_grad_contract_kernel<0>, dim3(a.nt, B), dim3(GT), CONTRACT_SMEM, st, a, ddsc0));
  MK_CUDA_CHECK(launch_k(dsm_grad_contract_kernel<1>, dim3(a.nt, B), dim3(GT), CONTRACT_SMEM, st, a, ddsc1));
  return MK_OK;
}
