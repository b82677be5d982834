// The heads' linear-attention transformer (Transformer_self_att, att_layers/transformer.py:75-103) for training: forward
// and backward in fp32 on the CUDA cores (include/mickey_b200.h mk_head_transformer*, DESIGN.md §6g).
//
// Activations are token-major fp32 [T = B*N, C].  Per layer (x = the layer input, C = 128, 8 heads of 16 channels):
//   qkv = x Wqkv^T, phi = elu + 1 on q and k                      htr_gemm<HE_PHI>
//   S = sum_s phi(k_s) (x) v_s, Ksum = sum_s phi(k_s) per image   htr_kv_partial -> htr_fold (fixed slots of 32 tokens)
//   msg_l = Z_l phi(q_l) S, Z_l = 1 / (phi(q_l) . Ksum + 1e-6)     htr_attn_fwd   (= the reference's N Z phi(q) KV, KV = S / N)
//   m1 = LN1(msg Wm^T)                                             htr_gemm<HE_LN>     (a 64 x 128 tile holds whole rows)
//   h = relu([x | m1] W0^T)                                        htr_gemm<HE_RELU>   ([x | m1] is one [T, 256] buffer)
//   out = x + LN2(h W2^T)                                          htr_gemm<HE_LN_RES> (written into the next layer's x)
// Backward with w_l = phi(q_l) S and g_l = dmsg_l (the closed form of DESIGN.md §6g, in terms of S rather than KV):
//   dphi(q_l) = Z_l g_l S^T - Z_l^2 (g_l . w_l) Ksum,  dS = sum_l Z_l phi(q_l) (x) g_l,  dKsum = -sum_l Z_l^2 (g_l . w_l) phi(q_l)
//   dphi(k_s) = dS v_s + dKsum,  dv_s = dS^T phi(k_s),  elu'(t) = min(phi(t), 1)
// dX = dY W and dW = dY^T X run through the same tile GEMM: it reads either operand in either layout through shared memory,
// so no transposed copy of an activation or a weight is made.  dW and the LayerNorm parameters' gradients sum fixed token
// slots, then fold the slots in index order; no atomics anywhere, so every output is bit-identical run to run, and an
// image's output and input gradient do not depend on the other images of the batch (every per-image reduction runs over
// slots aligned to that image's tokens).
#include "../../include/mickey_b200.h"
#include "ops.h"

#include <cstring>

namespace mk {

namespace {

constexpr int D = 128, D2 = 256, D3 = 384, NH = 8, DH = 16;
constexpr int SKV = NH * DH * DH + NH * DH;   // S and Ksum of one image: 2176 floats
constexpr int AT = 32;                         // tokens per attention slot
constexpr int LNT = 64;                        // tokens per LayerNorm-gradient slot
constexpr int WSLOT = 512;                     // tokens per weight-gradient slot
constexpr int BM = 64, BN = 128, BK = 16, GT = 256;
constexpr float LN_EPS = 1e-5f, ATT_EPS = 1e-6f;

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// ---- tile GEMM: out[m, n] = epi(sum_k A(m, k) B(k, n)) ---------------------------------------------------------------
// A(m, k) = A[m*lda + k] (AL = 0, rows contiguous in k) or A[k*lda + m] (AL = 1); B(k, n) = B[n*ldb + k] (BL = 0) or
// B[k*ldb + n] (BL = 1).  64 x 128 output tile, 256 threads with 4 x 8 cells each, k in steps of 16 through two shared-
// memory stages.  K is cut into slots of kslot along blockIdx.z (dW: one partial product per token slot).
enum HEpi : int {
  HE_STORE = 0,   // out = acc                                    (dmsg, dW slot partials)
  HE_PHI = 1,     // out = n < 256 ? phi(acc) : acc               (q | k | v)
  HE_RELU = 2,    // out = max(acc, 0)                            (mlp.0)
  HE_MASK = 3,    // out = R > 0 ? acc : 0                        (dh through the ReLU, R = h)
  HE_ADD = 4,     // out = acc + R                                (dX plus the residual / concat paths; R may alias out)
  HE_LN = 5,      // out = LN(acc) gamma + beta; xhat, rstd saved (merge + norm1)
  HE_LN_RES = 6,  // out = R + LN(acc) gamma + beta; xhat, rstd   (mlp.2 + norm2 + residual; R may alias out)
};

struct HGemm {
  const float* A; long long lda;
  const float* B; long long ldb;
  int M, N, K, kslot;
  float* out; long long ldo, out_slot;
  const float* R; long long ldr;
  const float* gamma; const float* beta;
  float* xhat; float* rstd;
};

__device__ __forceinline__ float phi(float t) { return t > 0.f ? t + 1.f : expf(t); }

template <int AL, int BL, int EPI>
__global__ void __launch_bounds__(GT) htr_gemm_kernel(HGemm p) {
  __shared__ __align__(16) float As[2][BK][BM + 4];
  __shared__ __align__(16) float Bs[2][BK][BN + 4];
  pdl_wait();
  pdl_trigger();
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int kb = blockIdx.z * p.kslot, ke = min(p.K, kb + p.kslot);
  float acc[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  float4 ra, rb[2];
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);

  auto load = [&](int k0) {
    if (AL == 0) {
      const int m = m0 + (tid >> 2), k = k0 + (tid & 3) * 4;
      ra = m < p.M ? *reinterpret_cast<const float4*>(p.A + (long long)m * p.lda + k) : z4;
    } else {
      const int k = k0 + (tid >> 4), m = m0 + (tid & 15) * 4;
      ra = k < ke ? *reinterpret_cast<const float4*>(p.A + (long long)k * p.lda + m) : z4;
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int idx = tid + GT * i;
      if (BL == 0) {
        const int n = n0 + (idx >> 2), k = k0 + (idx & 3) * 4;
        rb[i] = *reinterpret_cast<const float4*>(p.B + (long long)n * p.ldb + k);
      } else {
        const int k = k0 + (idx >> 5), n = n0 + (idx & 31) * 4;
        rb[i] = k < ke ? *reinterpret_cast<const float4*>(p.B + (long long)k * p.ldb + n) : z4;
      }
    }
  };
  auto store = [&](int s) {
    if (AL == 0) {
      const int r = tid >> 2, kq = (tid & 3) * 4;
      As[s][kq + 0][r] = ra.x; As[s][kq + 1][r] = ra.y; As[s][kq + 2][r] = ra.z; As[s][kq + 3][r] = ra.w;
    } else {
      *reinterpret_cast<float4*>(&As[s][tid >> 4][(tid & 15) * 4]) = ra;
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int idx = tid + GT * i;
      if (BL == 0) {
        const int n = idx >> 2, kq = (idx & 3) * 4;
        Bs[s][kq + 0][n] = rb[i].x; Bs[s][kq + 1][n] = rb[i].y; Bs[s][kq + 2][n] = rb[i].z; Bs[s][kq + 3][n] = rb[i].w;
      } else {
        *reinterpret_cast<float4*>(&Bs[s][idx >> 5][(idx & 31) * 4]) = rb[i];
      }
    }
  };

  const int nk = (ke - kb + BK - 1) / BK;
  load(kb);
  store(0);
  __syncthreads();
  for (int it = 0; it < nk; ++it) {
    const int s = it & 1;
    if (it + 1 < nk) load(kb + (it + 1) * BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      const float4 a = *reinterpret_cast<const float4*>(&As[s][kk][ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[s][kk][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[s][kk][64 + tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w};
      const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (it + 1 < nk) store(s ^ 1);
    __syncthreads();
  }

  // ---- epilogue: cells (m0 + ty*4 + i, n0 + tx*4 + j) for j < 4 and (.., n0 + 64 + tx*4 + j - 4) for j >= 4
  float* out = p.out + (long long)blockIdx.z * p.out_slot;
  if constexpr (EPI == HE_LN || EPI == HE_LN_RES) {
    // the tile holds whole 128-channel rows (N = 128); a row's 16 threads are 16 consecutive lanes of one warp
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float s = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) s += acc[i][j];
#pragma unroll
      for (int o = 1; o < 16; o <<= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      const float mean = s * (1.0f / D);
      float q = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        acc[i][j] -= mean;
        q = fmaf(acc[i][j], acc[i][j], q);
      }
#pragma unroll
      for (int o = 1; o < 16; o <<= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
      const float rs = 1.0f / sqrtf(q * (1.0f / D) + LN_EPS);
      const int m = m0 + ty * 4 + i;
      if (m >= p.M) continue;
      if (tx == 0) p.rstd[m] = rs;
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const int c = hf * 64 + tx * 4;
        float xh[4], y[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          xh[j] = acc[i][hf * 4 + j] * rs;
          y[j] = fmaf(xh[j], __ldg(p.gamma + c + j), __ldg(p.beta + c + j));
        }
        *reinterpret_cast<float4*>(p.xhat + (long long)m * D + c) = make_float4(xh[0], xh[1], xh[2], xh[3]);
        if (EPI == HE_LN_RES) {
          const float4 r = *reinterpret_cast<const float4*>(p.R + (long long)m * p.ldr + c);
          y[0] += r.x; y[1] += r.y; y[2] += r.z; y[3] += r.w;
        }
        *reinterpret_cast<float4*>(out + (long long)m * p.ldo + c) = make_float4(y[0], y[1], y[2], y[3]);
      }
    }
  } else {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= p.M) continue;
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
      const int n = n0 + hf * 64 + tx * 4;
      float v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = acc[i][hf * 4 + j];
      if (EPI == HE_PHI && n < 2 * D) {
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = phi(v[j]);
      }
      if (EPI == HE_RELU) {
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = fmaxf(v[j], 0.f);
      }
      if (EPI == HE_MASK || EPI == HE_ADD) {
        const float4 r4 = *reinterpret_cast<const float4*>(p.R + (long long)m * p.ldr + n);
        const float r[4] = {r4.x, r4.y, r4.z, r4.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = EPI == HE_MASK ? (r[j] > 0.f ? v[j] : 0.f) : v[j] + r[j];
      }
      *reinterpret_cast<float4*>(out + (long long)m * p.ldo + n) = make_float4(v[0], v[1], v[2], v[3]);
    }
  }
  }
}

// ---- fixed-order fold of slot partials: out[b*ob + i] = sum_c part[b*pb + c*ps + i], c = 0 .. nslots-1 ----------------
__global__ void __launch_bounds__(256) htr_fold_kernel(const float* __restrict__ part, int nslots, long long ps, long long pb,
                                                       int n, float* __restrict__ out, long long ob) {
  pdl_wait();
  pdl_trigger();
  const int i = blockIdx.x * 256 + threadIdx.x, b = blockIdx.y;
  if (i >= n) return;
  const float* q = part + (long long)b * pb + i;
  float s = 0.f;
  for (int c = 0; c < nslots; ++c) s += q[(long long)c * ps];
  out[(long long)b * ob + i] = s;
}

// ---- layout changes: channel-major [B, 128, HW] <-> token-major [B*HW, ld] ---------------------------------------------
// Block (x, b): tokens [32x, 32x + 32) of image b.  cm_to_tm adds pe[c, y, x] (row stride 256) when pe is given.
__global__ void __launch_bounds__(256) htr_cm_to_tm_kernel(const float* __restrict__ src, const float* __restrict__ pe, int HW,
                                                           int w, float* __restrict__ dst, int ldd) {
  __shared__ float tile[D][33];
  pdl_wait();
  pdl_trigger();
  const int b = blockIdx.y, n0 = blockIdx.x * 32, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = n0 + lane;
  const int py = n / w, px = n - py * w;
#pragma unroll 4
  for (int k = 0; k < 16; ++k) {
    const int c = warp + 8 * k;
    float v = 0.f;
    if (n < HW) {
      v = __ldg(src + ((long long)b * D + c) * HW + n);
      if (pe) v += __ldg(pe + (long long)c * 65536 + py * 256 + px);
    }
    tile[c][lane] = v;
  }
  __syncthreads();
  for (int j = warp; j < 32 && n0 + j < HW; j += 8)
    *reinterpret_cast<float4*>(dst + ((long long)b * HW + n0 + j) * ldd + lane * 4) =
        make_float4(tile[lane * 4][j], tile[lane * 4 + 1][j], tile[lane * 4 + 2][j], tile[lane * 4 + 3][j]);
}

__global__ void __launch_bounds__(256) htr_tm_to_cm_kernel(const float* __restrict__ src, int lds, int HW, float* __restrict__ dst) {
  __shared__ float tile[D][33];
  pdl_wait();
  pdl_trigger();
  const int b = blockIdx.y, n0 = blockIdx.x * 32, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int j = warp; j < 32 && n0 + j < HW; j += 8) {
    const float4 v = *reinterpret_cast<const float4*>(src + ((long long)b * HW + n0 + j) * lds + lane * 4);
    tile[lane * 4][j] = v.x; tile[lane * 4 + 1][j] = v.y; tile[lane * 4 + 2][j] = v.z; tile[lane * 4 + 3][j] = v.w;
  }
  __syncthreads();
  if (n0 + lane >= HW) return;
#pragma unroll 4
  for (int k = 0; k < 16; ++k) {
    const int c = warp + 8 * k;
    dst[((long long)b * D + c) * HW + n0 + lane] = tile[c][lane];
  }
}

// q_proj | k_proj | v_proj -> one [384, 128] weight
__global__ void __launch_bounds__(256) htr_pack_qkv_kernel(const float* __restrict__ q, const float* __restrict__ k,
                                                           const float* __restrict__ v, float* __restrict__ dst) {
  pdl_wait();
  pdl_trigger();
  const int i = blockIdx.x * 256 + threadIdx.x;          // float4 index, 3 * 4096 of them
  const int which = i >> 12, j = i & 4095;
  const float* s = which == 0 ? q : which == 1 ? k : v;
  reinterpret_cast<float4*>(dst)[i] = __ldg(reinterpret_cast<const float4*>(s) + j);
}

// ---- linear attention ---------------------------------------------------------------------------------------------------
// Block (c, b): tokens [32c, 32c + 32) of image b.  part[(b*nch + c)*SKV]: S [8][16][16] then Ksum [8][16] of the slot.
__global__ void __launch_bounds__(256) htr_kv_partial_kernel(const float* __restrict__ qkv, int N, int nch, float* __restrict__ part) {
  __shared__ __align__(16) float sk[AT][D];
  __shared__ __align__(16) float sv[AT][D];
  pdl_wait();
  pdl_trigger();
  const int b = blockIdx.y, c = blockIdx.x, t0 = c * AT, tid = threadIdx.x;
  const int nt = min(AT, N - t0);
  for (int idx = tid; idx < AT * 32; idx += 256) {
    const int r = idx >> 5, ch = (idx & 31) * 4;
    float4 kk = make_float4(0.f, 0.f, 0.f, 0.f), vv = kk;
    if (r < nt) {
      const float* row = qkv + ((long long)b * N + t0 + r) * D3;
      kk = *reinterpret_cast<const float4*>(row + D + ch);
      vv = *reinterpret_cast<const float4*>(row + 2 * D + ch);
    }
    *reinterpret_cast<float4*>(&sk[r][ch]) = kk;
    *reinterpret_cast<float4*>(&sv[r][ch]) = vv;
  }
  __syncthreads();
  const int h = tid >> 5, d = (tid >> 1) & 15, v0 = (tid & 1) * 8;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, ks = 0.f;
  for (int r = 0; r < nt; ++r) {
    const float kd = sk[r][h * DH + d];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = fmaf(kd, sv[r][h * DH + v0 + j], acc[j]);
    ks += kd;
  }
  float* o = part + ((long long)b * nch + c) * SKV;
#pragma unroll
  for (int j = 0; j < 8; ++j) o[h * 256 + d * DH + v0 + j] = acc[j];
  if (v0 == 0) o[NH * 256 + h * DH + d] = ks;
}

// S of image b into shared memory, heads 260 floats apart (conflict-free float4 reads across the 8 heads of a warp)
constexpr int SLD = 260;
__device__ __forceinline__ void load_s(const float* __restrict__ S, float (*Ss)[SLD], float (*Ks)[DH]) {
  for (int i = threadIdx.x; i < NH * 256; i += 256) Ss[i >> 8][i & 255] = S[i];
  if (threadIdx.x < NH * DH) Ks[threadIdx.x >> 4][threadIdx.x & 15] = S[NH * 256 + threadIdx.x];
}

__device__ __forceinline__ void load16(const float* p, float* v) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float4 t = *reinterpret_cast<const float4*>(p + 4 * j);
    v[4 * j] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w;
  }
}

// Z and w = phi(q) S of one (token, head); the forward and the backward share it, so both see the same bits
__device__ __forceinline__ float attn_zw(const float* q, const float* Ssh, const float* Ksh, float* w) {
  float den = 0.f;
#pragma unroll
  for (int d = 0; d < DH; ++d) den = fmaf(q[d], Ksh[d], den);
#pragma unroll
  for (int v = 0; v < DH; ++v) w[v] = 0.f;
#pragma unroll
  for (int d = 0; d < DH; ++d)
#pragma unroll
    for (int v4 = 0; v4 < 4; ++v4) {
      const float4 s = *reinterpret_cast<const float4*>(Ssh + d * DH + v4 * 4);
      w[v4 * 4] = fmaf(q[d], s.x, w[v4 * 4]); w[v4 * 4 + 1] = fmaf(q[d], s.y, w[v4 * 4 + 1]);
      w[v4 * 4 + 2] = fmaf(q[d], s.z, w[v4 * 4 + 2]); w[v4 * 4 + 3] = fmaf(q[d], s.w, w[v4 * 4 + 3]);
    }
  return 1.0f / (den + ATT_EPS);
}

// Block (c, b), thread (token r = tid / 8, head h = tid % 8): msg = Z phi(q) S.
__global__ void __launch_bounds__(256) htr_attn_fwd_kernel(const float* __restrict__ qkv, const float* __restrict__ S, int N,
                                                           float* __restrict__ msg) {
  __shared__ __align__(16) float Ss[NH][SLD];
  __shared__ float Ks[NH][DH];
  pdl_wait();
  pdl_trigger();
  const int b = blockIdx.y, h = threadIdx.x & 7, t = blockIdx.x * AT + (threadIdx.x >> 3);
  load_s(S + (long long)b * SKV, Ss, Ks);
  __syncthreads();
  if (t >= N) return;
  const long long tok = (long long)b * N + t;
  float q[DH], w[DH];
  load16(qkv + tok * D3 + h * DH, q);
  const float Z = attn_zw(q, Ss[h], Ks[h], w);
  float* o = msg + tok * D + h * DH;
#pragma unroll
  for (int v4 = 0; v4 < 4; ++v4)
    *reinterpret_cast<float4*>(o + 4 * v4) = make_float4(Z * w[4 * v4], Z * w[4 * v4 + 1], Z * w[4 * v4 + 2], Z * w[4 * v4 + 3]);
}

// Backward, part 1.  Block (c, b), thread (token r, head h): dq into dqkv[:, 0:128]; the slot's partial dS (sum over its
// tokens of Z phi(q) (x) g) and dKsum (sum of -Z^2 (g . w) phi(q)) into part[(b*nch + c)*SKV].
__global__ void __launch_bounds__(256) htr_attn_bwd_q_kernel(const float* __restrict__ qkv, const float* __restrict__ S,
                                                             const float* __restrict__ dmsg, int N, int nch,
                                                             float* __restrict__ dqkv, float* __restrict__ part) {
  __shared__ __align__(16) float Ss[NH][SLD];
  __shared__ float Ks[NH][DH];
  __shared__ __align__(16) float qs[AT][D];
  __shared__ __align__(16) float gs[AT][D];
  __shared__ float zs[AT][NH], cs[AT][NH];
  pdl_wait();
  pdl_trigger();
  const int b = blockIdx.y, c = blockIdx.x, tid = threadIdx.x, h = tid & 7, r = tid >> 3, t = c * AT + r;
  load_s(S + (long long)b * SKV, Ss, Ks);
  __syncthreads();
  float q[DH], g[DH], w[DH];
  float Z = 0.f, cc = 0.f;
  const long long tok = (long long)b * N + t;
  if (t < N) {
    load16(qkv + tok * D3 + h * DH, q);
    load16(dmsg + tok * D + h * DH, g);
    Z = attn_zw(q, Ss[h], Ks[h], w);
    float gw = 0.f;
#pragma unroll
    for (int v = 0; v < DH; ++v) gw = fmaf(g[v], w[v], gw);
    cc = -(Z * Z) * gw;
  } else {
#pragma unroll
    for (int d = 0; d < DH; ++d) q[d] = g[d] = 0.f;
  }
#pragma unroll
  for (int d = 0; d < DH; ++d) { qs[r][h * DH + d] = q[d]; gs[r][h * DH + d] = g[d]; }
  zs[r][h] = Z;
  cs[r][h] = cc;
  if (t < N) {
    float* o = dqkv + tok * D3 + h * DH;
#pragma unroll 2
    for (int d = 0; d < DH; ++d) {
      float sg = 0.f;
#pragma unroll
      for (int v = 0; v < DH; ++v) sg = fmaf(g[v], Ss[h][d * DH + v], sg);
      o[d] = fmaf(Z, sg, cc * Ks[h][d]) * fminf(qs[r][h * DH + d], 1.f);
    }
  }
  __syncthreads();
  const int h2 = tid >> 5, d = (tid >> 1) & 15, v0 = (tid & 1) * 8;
  const int nt = min(AT, N - c * AT);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, ks = 0.f;
  for (int rr = 0; rr < nt; ++rr) {
    const float qd = qs[rr][h2 * DH + d];
    const float a = zs[rr][h2] * qd;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = fmaf(a, gs[rr][h2 * DH + v0 + j], acc[j]);
    ks = fmaf(cs[rr][h2], qd, ks);
  }
  float* o = part + ((long long)b * nch + c) * SKV;
#pragma unroll
  for (int j = 0; j < 8; ++j) o[h2 * 256 + d * DH + v0 + j] = acc[j];
  if (v0 == 0) o[NH * 256 + h2 * DH + d] = ks;
}

// Backward, part 2.  dS, dKsum of image b (folded): dk = (dS v + dKsum) elu'(k), dv = dS^T phi(k) into dqkv[:, 128:384].
__global__ void __launch_bounds__(256) htr_attn_bwd_kv_kernel(const float* __restrict__ qkv, const float* __restrict__ dS, int N,
                                                              float* __restrict__ dqkv) {
  __shared__ __align__(16) float Ss[NH][SLD];
  __shared__ float Ks[NH][DH];
  pdl_wait();
  pdl_trigger();
  const int b = blockIdx.y, h = threadIdx.x & 7, t = blockIdx.x * AT + (threadIdx.x >> 3);
  load_s(dS + (long long)b * SKV, Ss, Ks);
  __syncthreads();
  if (t >= N) return;
  const long long tok = (long long)b * N + t;
  float k[DH], v[DH], dk[DH], dv[DH];
  load16(qkv + tok * D3 + D + h * DH, k);
  load16(qkv + tok * D3 + 2 * D + h * DH, v);
#pragma unroll
  for (int j = 0; j < DH; ++j) dv[j] = 0.f;
#pragma unroll
  for (int d = 0; d < DH; ++d) {
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < DH; ++j) {
      const float x = Ss[h][d * DH + j];
      s = fmaf(x, v[j], s);
      dv[j] = fmaf(x, k[d], dv[j]);
    }
    dk[d] = (s + Ks[h][d]) * fminf(k[d], 1.f);
  }
  float* o = dqkv + tok * D3 + D + h * DH;
#pragma unroll
  for (int v4 = 0; v4 < 4; ++v4) {
    *reinterpret_cast<float4*>(o + 4 * v4) = make_float4(dk[4 * v4], dk[4 * v4 + 1], dk[4 * v4 + 2], dk[4 * v4 + 3]);
    *reinterpret_cast<float4*>(o + D + 4 * v4) = make_float4(dv[4 * v4], dv[4 * v4 + 1], dv[4 * v4 + 2], dv[4 * v4 + 3]);
  }
}

// ---- LayerNorm backward: dz = rstd (g gamma - mean(g gamma) - xhat mean(g gamma xhat)) -----------------------------------
// Block c: tokens [64c, 64c + 64), a warp per token, 4 channels per lane.  part[c*256 + ch] = sum g xhat (dgamma), part[c*256 +
// 128 + ch] = sum g (dbeta) over the block's tokens, in token order per warp, then the 8 warps in order.
__global__ void __launch_bounds__(256) htr_ln_bwd_kernel(const float* __restrict__ g, const float* __restrict__ xhat,
                                                         const float* __restrict__ rstd, const float* __restrict__ gamma, int T,
                                                         float* __restrict__ dz, float* __restrict__ part) {
  __shared__ float red[8][2 * D];
  pdl_wait();
  pdl_trigger();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, ch = lane * 4;
  const float4 gm4 = __ldg(reinterpret_cast<const float4*>(gamma) + lane);
  const float gm[4] = {gm4.x, gm4.y, gm4.z, gm4.w};
  float dg[4] = {0.f, 0.f, 0.f, 0.f}, db[4] = {0.f, 0.f, 0.f, 0.f};
  for (int i = 0; i < LNT / 8; ++i) {
    const int t = blockIdx.x * LNT + warp * (LNT / 8) + i;
    if (t >= T) break;
    const float4 g4 = *reinterpret_cast<const float4*>(g + (long long)t * D + ch);
    const float4 x4 = *reinterpret_cast<const float4*>(xhat + (long long)t * D + ch);
    const float gv[4] = {g4.x, g4.y, g4.z, g4.w}, xv[4] = {x4.x, x4.y, x4.z, x4.w};
    float gg[4], s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      gg[j] = gv[j] * gm[j];
      s1 += gg[j];
      s2 = fmaf(gg[j], xv[j], s2);
      dg[j] = fmaf(gv[j], xv[j], dg[j]);
      db[j] += gv[j];
    }
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    const float m1 = s1 * (1.0f / D), m2 = s2 * (1.0f / D), r = rstd[t];
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = r * (gg[j] - m1 - xv[j] * m2);
    *reinterpret_cast<float4*>(dz + (long long)t * D + ch) = make_float4(o[0], o[1], o[2], o[3]);
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) { red[warp][ch + j] = dg[j]; red[warp][D + ch + j] = db[j]; }
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) s += red[w][threadIdx.x];
  part[(long long)blockIdx.x * 2 * D + threadIdx.x] = s;
}

// ---- host side -----------------------------------------------------------------------------------------------------------
struct FwdL {      // one layer's activations (offsets in bytes); with save = 0 every layer shares one set
  size_t cat, qkv, msg, xh1, xh2, h, rs1, rs2, S, bytes;
};
struct FwdLayout { FwdL layer; size_t layer_stride, xout, kvpart, wqkv, total; };

FwdL fwd_layer(long long T, int B) {
  FwdL L;
  size_t o = 0;
  auto take = [&](size_t n) { const size_t r = o; o = align256(o + n * sizeof(float)); return r; };
  L.cat = take((size_t)T * D2); L.qkv = take((size_t)T * D3); L.msg = take((size_t)T * D);
  L.xh1 = take((size_t)T * D); L.xh2 = take((size_t)T * D); L.h = take((size_t)T * D2);
  L.rs1 = take((size_t)T); L.rs2 = take((size_t)T); L.S = take((size_t)B * SKV);
  L.bytes = o;
  return L;
}

FwdLayout fwd_layout(int B, int N, int layers, int save) {
  const long long T = (long long)B * N;
  FwdLayout F;
  F.layer = fwd_layer(T, B);
  F.layer_stride = save ? F.layer.bytes : 0;
  size_t o = F.layer.bytes + (size_t)(save ? layers - 1 : 0) * F.layer.bytes;
  F.xout = o; o = align256(o + (size_t)T * D * sizeof(float));
  F.kvpart = o; o = align256(o + (size_t)B * ceil_div(N, AT) * SKV * sizeof(float));
  F.wqkv = o; o = align256(o + (size_t)D3 * D * sizeof(float));
  F.total = o;
  return F;
}

struct BwdLayout { size_t gA, gB, dy, dh, dm, dqkv, lnpart, apart, dS, wpart, wqkv, total; };
BwdLayout bwd_layout(int B, int N) {
  const long long T = (long long)B * N;
  BwdLayout L;
  size_t o = 0;
  auto take = [&](size_t n) { const size_t r = o; o = align256(o + n * sizeof(float)); return r; };
  L.gA = take((size_t)T * D); L.gB = take((size_t)T * D); L.dy = take((size_t)T * D); L.dh = take((size_t)T * D2);
  L.dm = take((size_t)T * D); L.dqkv = take((size_t)T * D3);
  L.lnpart = take((size_t)ceil_div((int)T, LNT) * 2 * D);
  L.apart = take((size_t)B * ceil_div(N, AT) * SKV);
  L.dS = take((size_t)B * SKV);
  L.wpart = take((size_t)ceil_div((int)T, WSLOT) * D2 * D2);
  L.wqkv = take((size_t)D3 * D);
  L.total = o;
  return L;
}

// The GEMMs put 64-token tiles in gridDim.y and the per-image kernels put B there, both capped at 65535.  The layer cap only
// keeps the saved-activation workspace size far from size_t overflow.
constexpr long long MAX_TOKENS = 65535LL * BM;
constexpr int MAX_B = 65535, MAX_LAYERS = 1024;

bool geometry_ok(int B, int h, int w, int layers) {
  return B >= 1 && h >= 1 && w >= 1 && B <= MAX_B && layers >= 1 && layers <= MAX_LAYERS &&
         (long long)B * h * w <= MAX_TOKENS;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

bool layer_ok(const mk_htr_layer& l) {
  const float* ps[10] = {l.q_proj, l.k_proj, l.v_proj, l.merge, l.mlp0, l.mlp2, l.norm1_w, l.norm1_b, l.norm2_w, l.norm2_b};
  for (const float* p : ps)
    if (!p || !aligned16(p)) return false;
  return true;
}

template <int AL, int BL, int EPI>
cudaError_t gemm(const HGemm& p, int slots, cudaStream_t st) {
  return launch_k(htr_gemm_kernel<AL, BL, EPI>, dim3(p.N / BN, ceil_div(p.M, BM), slots), dim3(GT), 0, st, p);
}

HGemm gp(const float* A, long long lda, const float* Bm, long long ldb, int M, int N, int K, float* out, long long ldo) {
  HGemm p;
  memset(&p, 0, sizeof(p));
  p.A = A; p.lda = lda; p.B = Bm; p.ldb = ldb; p.M = M; p.N = N; p.K = K; p.kslot = K; p.out = out; p.ldo = ldo;
  return p;
}

// dW [M, Nw] = sum over the T tokens of A(t, m) B(t, n): slot partials, then the fold into out
cudaError_t weight_grad(const float* A, long long lda, const float* Bm, long long ldb, int M, int Nw, int T, float* wpart,
                        float* out, cudaStream_t st) {
  HGemm p = gp(A, lda, Bm, ldb, M, Nw, T, wpart, Nw);
  p.kslot = WSLOT;
  p.out_slot = (long long)M * Nw;
  const int slots = ceil_div(T, WSLOT);
  cudaError_t e = gemm<1, 1, HE_STORE>(p, slots, st);
  if (e != cudaSuccess) return e;
  return launch_k(htr_fold_kernel, dim3(ceil_div(M * Nw, 256), 1), dim3(256), 0, st, (const float*)wpart, slots, p.out_slot,
                  0LL, M * Nw, out, 0LL);
}

}  // namespace

}  // namespace mk

using namespace mk;

long long mk_head_transformer_ws_bytes(int B, int h, int w, int num_layers, int save) {
  if (!geometry_ok(B, h, w, num_layers)) return -1;
  return (long long)fwd_layout(B, h * w, num_layers, save ? 1 : 0).total;
}

long long mk_head_transformer_backward_ws_bytes(int B, int h, int w, int num_layers) {
  if (!geometry_ok(B, h, w, num_layers)) return -1;
  return (long long)bwd_layout(B, h * w).total;
}

int mk_head_transformer(const float* x, const float* pe, int B, int h, int w, const mk_htr_layer* layers, int num_layers,
                        float* out, int save, void* ws, long long ws_bytes, void* stream) {
  if (!x || !out || !ws || !layers || !geometry_ok(B, h, w, num_layers) || (pe && (h > 256 || w > 256)) || !aligned16(x) ||
      !aligned16(out) || !aligned16(ws) || (pe && !aligned16(pe))) {
    set_last_error("mk_head_transformer: need x, out, layers and a 16-byte aligned workspace, B, h, w >= 1, 1 <= num_layers "
                   "<= 1024, B <= 65535, B*h*w <= 4194240, and h, w <= 256 with the positional encoding (got B %d h %d w %d layers %d)",
                   B, h, w, num_layers);
    return MK_ERR_INVALID;
  }
  for (int l = 0; l < num_layers; ++l)
    if (!layer_ok(layers[l])) {
      set_last_error("mk_head_transformer: layer %d has a NULL or misaligned parameter", l);
      return MK_ERR_INVALID;
    }
  const int N = h * w, T = B * N, nch = ceil_div(N, AT);
  const FwdLayout F = fwd_layout(B, N, num_layers, save ? 1 : 0);
  if (ws_bytes < (long long)F.total) {
    set_last_error("mk_head_transformer: workspace of %lld bytes, %lld needed", ws_bytes, (long long)F.total);
    return MK_ERR_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* base = reinterpret_cast<uint8_t*>(ws);
  auto at = [&](int l, size_t off) { return reinterpret_cast<float*>(base + (size_t)l * F.layer_stride + off); };
  float* xout = reinterpret_cast<float*>(base + F.xout);
  float* kvpart = reinterpret_cast<float*>(base + F.kvpart);
  float* wqkv = reinterpret_cast<float*>(base + F.wqkv);
  MK_CUDA_CHECK(launch_k(htr_cm_to_tm_kernel, dim3(nch, B), dim3(256), 0, st, x, pe, N, w, at(0, F.layer.cat), D2));
  for (int l = 0; l < num_layers; ++l) {
    const mk_htr_layer& P = layers[l];
    float* cat = at(l, F.layer.cat);
    float* qkv = at(l, F.layer.qkv);
    float* S = at(l, F.layer.S);
    float* msg = at(l, F.layer.msg);
    float* hb = at(l, F.layer.h);
    MK_CUDA_CHECK(launch_k(htr_pack_qkv_kernel, dim3(48), dim3(256), 0, st, P.q_proj, P.k_proj, P.v_proj, wqkv));
    MK_CUDA_CHECK((gemm<0, 0, HE_PHI>(gp(cat, D2, wqkv, D, T, D3, D, qkv, D3), 1, st)));
    MK_CUDA_CHECK(launch_k(htr_kv_partial_kernel, dim3(nch, B), dim3(256), 0, st, (const float*)qkv, N, nch, kvpart));
    MK_CUDA_CHECK(launch_k(htr_fold_kernel, dim3(ceil_div(SKV, 256), B), dim3(256), 0, st, (const float*)kvpart, nch, (long long)SKV,
                       (long long)nch * SKV, SKV, S, (long long)SKV));
    MK_CUDA_CHECK(launch_k(htr_attn_fwd_kernel, dim3(nch, B), dim3(256), 0, st, (const float*)qkv, (const float*)S, N, msg));
    HGemm pm = gp(msg, D, P.merge, D, T, D, D, cat + D, D2);
    pm.gamma = P.norm1_w; pm.beta = P.norm1_b; pm.xhat = at(l, F.layer.xh1); pm.rstd = at(l, F.layer.rs1);
    MK_CUDA_CHECK((gemm<0, 0, HE_LN>(pm, 1, st)));
    MK_CUDA_CHECK((gemm<0, 0, HE_RELU>(gp(cat, D2, P.mlp0, D2, T, D2, D2, hb, D2), 1, st)));
    const bool last = l + 1 == num_layers;
    HGemm p2 = gp(hb, D2, P.mlp2, D2, T, D, D2, last ? xout : at(l + 1, F.layer.cat), last ? D : D2);
    p2.R = cat; p2.ldr = D2; p2.gamma = P.norm2_w; p2.beta = P.norm2_b; p2.xhat = at(l, F.layer.xh2); p2.rstd = at(l, F.layer.rs2);
    MK_CUDA_CHECK((gemm<0, 0, HE_LN_RES>(p2, 1, st)));
  }
  MK_CUDA_CHECK(launch_k(htr_tm_to_cm_kernel, dim3(nch, B), dim3(256), 0, st, (const float*)xout, D, N, out));
  return MK_OK;
}

int mk_head_transformer_backward(const void* saved, const float* grad_out, int B, int h, int w, const mk_htr_layer* layers,
                                 int num_layers, float* grad_x, mk_htr_layer_grads* grads, void* ws, long long ws_bytes,
                                 void* stream) {
  if (!saved || !grad_out || !layers || !grads || !ws || !geometry_ok(B, h, w, num_layers) || !aligned16(saved) ||
      !aligned16(grad_out) || !aligned16(ws) || (grad_x && !aligned16(grad_x))) {
    set_last_error("mk_head_transformer_backward: need the forward's saved workspace, grad_out, layers, grads and a 16-byte "
                   "aligned workspace, B, h, w >= 1, 1 <= num_layers <= 1024, B <= 65535 and B*h*w <= 4194240 (got B %d h %d w %d "
                   "layers %d)",
                   B, h, w, num_layers);
    return MK_ERR_INVALID;
  }
  for (int l = 0; l < num_layers; ++l)
    if (!layer_ok(layers[l])) {
      set_last_error("mk_head_transformer_backward: layer %d has a NULL or misaligned parameter", l);
      return MK_ERR_INVALID;
    }
  const int N = h * w, T = B * N, nch = ceil_div(N, AT), nln = ceil_div(T, LNT);
  const FwdLayout F = fwd_layout(B, N, num_layers, 1);
  const BwdLayout L = bwd_layout(B, N);
  if (ws_bytes < (long long)L.total) {
    set_last_error("mk_head_transformer_backward: workspace of %lld bytes, %lld needed", ws_bytes, (long long)L.total);
    return MK_ERR_INVALID;
  }
  // need_below(l): some gradient flows through layer l's input (the input's own, or a parameter's of a layer below l)
  int first_grad = num_layers;
  for (int l = num_layers - 1; l >= 0; --l) {
    const mk_htr_layer_grads& G = grads[l];
    if (G.q_proj || G.k_proj || G.v_proj || G.merge || G.mlp0 || G.mlp2 || G.norm1_w || G.norm1_b || G.norm2_w || G.norm2_b)
      first_grad = l;
  }
  auto need_below = [&](int l) { return grad_x != nullptr || l > first_grad; };
  const bool any_below = grad_x != nullptr || first_grad < num_layers;
  if (!any_below) return MK_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const uint8_t* sv = reinterpret_cast<const uint8_t*>(saved);
  auto at = [&](int l, size_t off) { return reinterpret_cast<const float*>(sv + (size_t)l * F.layer_stride + off); };
  uint8_t* wb = reinterpret_cast<uint8_t*>(ws);
  auto wf = [&](size_t off) { return reinterpret_cast<float*>(wb + off); };
  float *g = wf(L.gA), *gn = wf(L.gB), *dy = wf(L.dy), *dh = wf(L.dh), *dm = wf(L.dm), *dqkv = wf(L.dqkv);
  float *lnpart = wf(L.lnpart), *apart = wf(L.apart), *dS = wf(L.dS), *wpart = wf(L.wpart), *wqkv = wf(L.wqkv);
  auto ln_fold = [&](float* dgamma, float* dbeta) -> cudaError_t {
    cudaError_t e = cudaSuccess;
    if (dgamma) e = launch_k(htr_fold_kernel, dim3(1, 1), dim3(256), 0, st, (const float*)lnpart, nln, (long long)2 * D, 0LL, D, dgamma, 0LL);
    if (e == cudaSuccess && dbeta)
      e = launch_k(htr_fold_kernel, dim3(1, 1), dim3(256), 0, st, (const float*)(lnpart + D), nln, (long long)2 * D, 0LL, D, dbeta, 0LL);
    return e;
  };
  MK_CUDA_CHECK(launch_k(htr_cm_to_tm_kernel, dim3(nch, B), dim3(256), 0, st, grad_out, (const float*)nullptr, N, w, g, D));
  for (int l = num_layers - 1; l >= 0; --l) {
    const mk_htr_layer& P = layers[l];
    const mk_htr_layer_grads& G = grads[l];
    const float *cat = at(l, F.layer.cat), *qkv = at(l, F.layer.qkv), *msg = at(l, F.layer.msg), *hb = at(l, F.layer.h);
    // norm2, mlp.2
    MK_CUDA_CHECK(launch_k(htr_ln_bwd_kernel, dim3(nln), dim3(256), 0, st, (const float*)g, at(l, F.layer.xh2), at(l, F.layer.rs2),
                       P.norm2_w, T, dy, lnpart));
    MK_CUDA_CHECK(ln_fold(G.norm2_w, G.norm2_b));
    if (G.mlp2) MK_CUDA_CHECK(weight_grad(dy, D, hb, D2, D, D2, T, wpart, G.mlp2, st));
    const bool rest = need_below(l) || G.mlp0 || G.merge || G.norm1_w || G.norm1_b || G.q_proj || G.k_proj || G.v_proj;
    if (!rest) break;
    // ReLU, mlp.0: dcat = dh W0; its x half joins the residual path, its m1 half goes to norm1
    {
      HGemm p = gp(dy, D, P.mlp2, D2, T, D2, D, dh, D2);
      p.R = hb; p.ldr = D2;
      MK_CUDA_CHECK((gemm<0, 1, HE_MASK>(p, 1, st)));
    }
    if (G.mlp0) MK_CUDA_CHECK(weight_grad(dh, D2, cat, D2, D2, D2, T, wpart, G.mlp0, st));
    if (need_below(l)) {
      HGemm p = gp(dh, D2, P.mlp0, D2, T, D, D2, gn, D);
      p.R = g; p.ldr = D;
      MK_CUDA_CHECK((gemm<0, 1, HE_ADD>(p, 1, st)));
    }
    MK_CUDA_CHECK((gemm<0, 1, HE_STORE>(gp(dh, D2, P.mlp0 + D, D2, T, D, D2, dm, D), 1, st)));
    // norm1, merge
    MK_CUDA_CHECK(launch_k(htr_ln_bwd_kernel, dim3(nln), dim3(256), 0, st, (const float*)dm, at(l, F.layer.xh1), at(l, F.layer.rs1),
                       P.norm1_w, T, dy, lnpart));
    MK_CUDA_CHECK(ln_fold(G.norm1_w, G.norm1_b));
    if (G.merge) MK_CUDA_CHECK(weight_grad(dy, D, msg, D, D, D, T, wpart, G.merge, st));
    MK_CUDA_CHECK((gemm<0, 1, HE_STORE>(gp(dy, D, P.merge, D, T, D, D, dm, D), 1, st)));
    // linear attention
    MK_CUDA_CHECK(launch_k(htr_attn_bwd_q_kernel, dim3(nch, B), dim3(256), 0, st, qkv, at(l, F.layer.S), (const float*)dm, N, nch,
                       dqkv, apart));
    MK_CUDA_CHECK(launch_k(htr_fold_kernel, dim3(ceil_div(SKV, 256), B), dim3(256), 0, st, (const float*)apart, nch, (long long)SKV,
                       (long long)nch * SKV, SKV, dS, (long long)SKV));
    MK_CUDA_CHECK(launch_k(htr_attn_bwd_kv_kernel, dim3(nch, B), dim3(256), 0, st, qkv, (const float*)dS, N, dqkv));
    float* wg[3] = {G.q_proj, G.k_proj, G.v_proj};
    for (int i = 0; i < 3; ++i)
      if (wg[i]) MK_CUDA_CHECK(weight_grad(dqkv + i * D, D3, cat, D2, D, D, T, wpart, wg[i], st));
    if (!need_below(l)) break;
    MK_CUDA_CHECK(launch_k(htr_pack_qkv_kernel, dim3(48), dim3(256), 0, st, P.q_proj, P.k_proj, P.v_proj, wqkv));
    {
      HGemm p = gp(dqkv, D3, wqkv, D, T, D, D3, gn, D);
      p.R = gn; p.ldr = D;
      MK_CUDA_CHECK((gemm<0, 1, HE_ADD>(p, 1, st)));
    }
    float* t = g; g = gn; gn = t;
  }
  if (grad_x) MK_CUDA_CHECK(launch_k(htr_tm_to_cm_kernel, dim3(nch, B), dim3(256), 0, st, (const float*)g, D, N, grad_x));
  return MK_OK;
}
