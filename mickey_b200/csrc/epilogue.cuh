// GEMM epilogues shared by the wgmma kernel and the SIMT debug kernel.
// Contract: the calling thread owns output row `m` (local to its group `g`) and receives the fp32
// accumulators of 32 consecutive columns n0..n0+31 in v[32] (one row per thread; the wgmma kernel reads
// them from the accumulator tile it parked in shared memory).
#pragma once
#include "common.cuh"

namespace mk {

// exact-erf GELU (reference layers/mlp.py:23 nn.GELU()): erf by Abramowitz-Stegun 7.1.26 (|abs err| < 1.5e-7 in
// exact arithmetic).  rcp/ex2 are the single-instruction MUFU approximations (1-2 ulp): the IEEE __frcp_rn / __expf
// forms expand to Newton iterations and range fix-ups that made this epilogue ~30 instructions per element (ncu).
__device__ __forceinline__ float rcp_approx(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float ex2_approx_f(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float gelu_erf(float x) {
  const float z = fabsf(x) * 0.70710678118654752f;
  const float t = rcp_approx(fmaf(0.3275911f, z, 1.0f));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  const float erf_abs = fmaf(-poly * t, ex2_approx_f(-1.4426950408889634f * z * z), 1.0f);
  const float hx = 0.5f * x;
  return fmaf(hx, copysignf(erf_abs, x), hx);
}

// The same function on two values, written pairwise: the same operations in the same order as gelu_erf, hence the same
// bits; the polynomial is carried negated (RN is symmetric) so that no separate negation is needed.
__device__ __forceinline__ void fma2_f32(float& d0, float& d1, float a0, float a1, float b0, float b1, float c0, float c1) {
  d0 = __fmaf_rn(a0, b0, c0);
  d1 = __fmaf_rn(a1, b1, c1);
}
__device__ __forceinline__ void mul2_f32(float& d0, float& d1, float a0, float a1, float b0, float b1) {
  d0 = __fmul_rn(a0, b0);
  d1 = __fmul_rn(a1, b1);
}
__device__ __forceinline__ void gelu_erf2(float x0, float x1, float& y0, float& y1) {
  float z0, z1, d0, d1, n0, n1, q0, q1, w0, w1, e0, e1, h0, h1;
  mul2_f32(z0, z1, fabsf(x0), fabsf(x1), 0.70710678118654752f, 0.70710678118654752f);
  fma2_f32(d0, d1, z0, z1, 0.3275911f, 0.3275911f, 1.0f, 1.0f);
  const float t0 = rcp_approx(d0), t1 = rcp_approx(d1);
  fma2_f32(n0, n1, t0, t1, -1.061405429f, -1.061405429f, 1.453152027f, 1.453152027f);       // -poly
  fma2_f32(n0, n1, n0, n1, t0, t1, -1.421413741f, -1.421413741f);
  fma2_f32(n0, n1, n0, n1, t0, t1, 0.284496736f, 0.284496736f);
  fma2_f32(n0, n1, n0, n1, t0, t1, -0.254829592f, -0.254829592f);
  mul2_f32(q0, q1, n0, n1, t0, t1);                                                          // (-poly) * t
  mul2_f32(w0, w1, z0, z1, -1.4426950408889634f, -1.4426950408889634f);
  mul2_f32(w0, w1, w0, w1, z0, z1);
  const float x20 = ex2_approx_f(w0), x21 = ex2_approx_f(w1);
  fma2_f32(e0, e1, q0, q1, x20, x21, 1.0f, 1.0f);                                            // erf(|x| / sqrt 2)
  mul2_f32(h0, h1, x0, x1, 0.5f, 0.5f);
  fma2_f32(y0, y1, h0, h1, copysignf(e0, x0), copysignf(e1, x1), h0, h1);
}

__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == ACT_GELU) return gelu_erf(x);
  if (act == ACT_RELU) return fmaxf(x, 0.0f);
  return x;
}

__device__ __forceinline__ void store_h32(__half* dst, const float* v) {
  // dst is 16-byte aligned by construction (ld and column offsets are multiples of 8)
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    __half2 h0 = __floats2half2_rn(v[q * 8 + 0], v[q * 8 + 1]);
    __half2 h1 = __floats2half2_rn(v[q * 8 + 2], v[q * 8 + 3]);
    __half2 h2 = __floats2half2_rn(v[q * 8 + 4], v[q * 8 + 5]);
    __half2 h3 = __floats2half2_rn(v[q * 8 + 6], v[q * 8 + 7]);
    uint4 u;
    u.x = *reinterpret_cast<uint32_t*>(&h0);
    u.y = *reinterpret_cast<uint32_t*>(&h1);
    u.z = *reinterpret_cast<uint32_t*>(&h2);
    u.w = *reinterpret_cast<uint32_t*>(&h3);
    reinterpret_cast<uint4*>(dst)[q] = u;
  }
}

__device__ __forceinline__ void add_vec32(float (&v)[32], const float* __restrict__ b) {
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const float4 t = __ldg(reinterpret_cast<const float4*>(b) + q);
    v[q * 4 + 0] += t.x; v[q * 4 + 1] += t.y; v[q * 4 + 2] += t.z; v[q * 4 + 3] += t.w;
  }
}

__device__ __forceinline__ bool pad_valid(const GemmParams& p, int m, int& pos) {
  const int per_img = p.pad_h2 * p.pad_w2;
  pos = m % per_img;
  const int y = pos / p.pad_w2, x = pos % p.pad_w2;
  return y >= 1 && y <= p.pad_h2 - 2 && x >= 1 && x <= p.pad_w2 - 2;
}

// ---- per-chunk epilogues ---------------------------------------------------------------------------
template <int EPI>
__device__ __forceinline__ void epilogue_chunk(const GemmParams& p, int g, int m, int n0, float (&v)[32]) {
  if constexpr (EPI == EPI_STORE_H) {
    if (m >= p.M) return;
    if (p.bias) add_vec32(v, p.bias + (size_t)g * p.bias_group_off + n0);
    if (p.act == ACT_GELU) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = gelu_erf(v[j]);
    } else if (p.act == ACT_RELU) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.0f);
    }
    store_h32(p.out_h + (size_t)g * p.out_h_group_off + (size_t)m * p.out_h_ld + n0, v);
  } else if constexpr (EPI == EPI_RESID_F) {
    if (m >= p.M) return;
    float* o = p.out_f + (size_t)m * p.out_f_ld + n0;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      float4 x = reinterpret_cast<float4*>(o)[q];
      const float4 gm = __ldg(reinterpret_cast<const float4*>(p.gamma + n0) + q);
      const float4 bs = __ldg(reinterpret_cast<const float4*>(p.bias + n0) + q);
      x.x += gm.x * (v[q * 4 + 0] + bs.x);
      x.y += gm.y * (v[q * 4 + 1] + bs.y);
      x.z += gm.z * (v[q * 4 + 2] + bs.z);
      x.w += gm.w * (v[q * 4 + 3] + bs.w);
      reinterpret_cast<float4*>(o)[q] = x;
    }
  } else if constexpr (EPI == EPI_PATCH) {
    if (m >= p.M) return;
    const int img = m / p.tok_per_img, tk = m % p.tok_per_img;
    float* o = p.out_f + ((size_t)img * (p.tok_per_img + 1) + 1 + tk) * p.out_f_ld + n0;
    const float* a = p.aux + (size_t)tk * p.N + n0;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(a) + q);
      float4 x;
      x.x = v[q * 4 + 0] + t.x; x.y = v[q * 4 + 1] + t.y; x.z = v[q * 4 + 2] + t.z; x.w = v[q * 4 + 3] + t.w;
      reinterpret_cast<float4*>(o)[q] = x;
    }
  } else if constexpr (EPI == EPI_CONV) {
    if (m >= p.M) return;
    int pos = 0;
    const bool valid = p.pad_h2 ? pad_valid(p, m, pos) : true;
    if (p.bias) add_vec32(v, p.bias + (size_t)g * p.bias_group_off + n0);
    if (p.res_h) {
      const uint4* r = reinterpret_cast<const uint4*>(p.res_h + (size_t)g * p.res_h_group_off + (size_t)m * p.res_h_ld + n0);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        uint4 u = r[q];
        const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float2 f = __half22float2(h[e]);
          v[q * 8 + e * 2] += f.x;
          v[q * 8 + e * 2 + 1] += f.y;
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = apply_act(v[j], p.act);
    if (p.aux && ((p.aux_group_mask >> g) & 1)) add_vec32(v, p.aux + (size_t)pos * p.N + n0);
    if (!valid) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = 0.0f;
    }
    if (p.out_f) {
      float* o = p.out_f + (size_t)g * p.out_f_group_off + (size_t)m * p.out_f_ld + n0;
#pragma unroll
      for (int q = 0; q < 8; ++q)
        reinterpret_cast<float4*>(o)[q] = make_float4(v[q * 4], v[q * 4 + 1], v[q * 4 + 2], v[q * 4 + 3]);
    }
    if (p.out_h) store_h32(p.out_h + (size_t)g * p.out_h_group_off + (size_t)m * p.out_h_ld + n0, v);
  } else if constexpr (EPI == EPI_STORE_F) {
    if (m >= p.M) return;
    float* o = p.out_f + (size_t)g * p.out_f_group_off + (size_t)m * p.out_f_ld + n0;
#pragma unroll
    for (int q = 0; q < 8; ++q)
      reinterpret_cast<float4*>(o)[q] = make_float4(v[q * 4], v[q * 4 + 1], v[q * 4 + 2], v[q * 4 + 3]);
  }
}

// ---- staged (coalesced) epilogue -----------------------------------------------------------------------
// The wgmma kernel first parks a warp's 32 x W block of fp32 accumulators in shared memory (rows of W floats, the
// 16-byte chunks of a row XOR-swizzled by acc_idx) and then calls epilogue_rows: lane l owns columns col_base + l*CPL .. (CPL = W/32) of
// every row, so each global load/store instruction of the warp covers ONE contiguous row segment (128-256 B)
// instead of 32 different rows — 4-8x fewer L1 wavefronts than the thread-per-row form above.
// Float offset of element (r, c) of a staged 32 x W block (W = 32 or 64).  Chunk k = c / 4 of row r is stored at chunk
// k ^ h with h = 2 (r % 4) + ((r ^ r / 4 ^ k / 8) & 1) < 8, a permutation of the row's chunks that keeps 16-byte
// accesses whole.  Every access pattern of the block is free of bank conflicts: the park's float2 stores (rows r..r+3,
// chunks 2m, 2m + 1 per half-warp), acc_chunk's float4 reads (one chunk of rows 0..7 per quarter-warp), epilogue_rows'
// float4 reads (chunks 0, 2, .., 14 of one row, or 0, 2, 4, 6 of rows 2t, 2t + 1).
// A row stride of W + 4 left the park's stores 2-way conflicted while the tensor cores wait for it.
template <int W> __device__ __forceinline__ int acc_idx(int r, int c) {
  const int k = c >> 2;
  const int h = 2 * (r & 3) + ((r ^ (r >> 2) ^ (k >> 3)) & 1);
  return r * W + ((k ^ h) << 2) + (c & 3);
}

// Lane layout of the staged epilogue: a lane owns EIGHT consecutive columns (one 16-byte fp16 store, two 16-byte fp32
// accesses) of one row per step; W/8 lanes cover a row, so a warp instruction covers 32/(W/8) whole rows.  The first
// version gave a lane 1-2 columns of every row: 4-byte stores, per-row predicates, 64-bit index math and run-time
// activation branches made it ~37 SASS instructions per output element; this form is ~3 per element.
__device__ __forceinline__ void ld8(const float* p, float (&v)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void ldg8(const float* p, float (&v)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p)), b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void st8(float* p, const float (&v)[8]) {
  reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
}
__device__ __forceinline__ void st8h(__half* p, const float (&v)[8]) {
  __half2 h0 = __floats2half2_rn(v[0], v[1]), h1 = __floats2half2_rn(v[2], v[3]);
  __half2 h2 = __floats2half2_rn(v[4], v[5]), h3 = __floats2half2_rn(v[6], v[7]);
  uint4 u;
  u.x = *reinterpret_cast<uint32_t*>(&h0); u.y = *reinterpret_cast<uint32_t*>(&h1);
  u.z = *reinterpret_cast<uint32_t*>(&h2); u.w = *reinterpret_cast<uint32_t*>(&h3);
  *reinterpret_cast<uint4*>(p) = u;
}
__device__ __forceinline__ void ld8h(const __half* p, float (&v)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int e = 0; e < 4; ++e) { const float2 f = __half22float2(h[e]); v[2 * e] = f.x; v[2 * e + 1] = f.y; }
}

template <int EPI, int W, int ACT>
__device__ __forceinline__ void epilogue_rows_impl(const GemmParams& p, int g, int row0, int lane, int col_base,
                                                   const float* __restrict__ stage, float mean_l, float rstd_l) {
  constexpr int LPR = W / 8;             // lanes per row
  constexpr int RPS = 32 / LPR;          // rows per step
  constexpr int STEPS = 32 / RPS;
  constexpr bool GLOBAL_IN = (EPI == EPI_RESID_F || EPI == EPI_PATCH || EPI == EPI_CONV || EPI == EPI_LN);
  constexpr int U = GLOBAL_IN ? 2 : 4;   // steps whose loads are all issued before the first store
  static_assert(W % 8 == 0 && 32 % LPR == 0 && STEPS % U == 0, "staged epilogue: W in {32, 64}");
  const int seg = lane % LPR, rsub = lane / LPR;
  const int col = col_base + seg * 8;
  float bias[8], gam[8], bet[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { bias[i] = 0.f; gam[i] = 1.f; bet[i] = 0.f; }
  if constexpr (EPI == EPI_STORE_H || EPI == EPI_CONV) { if (p.bias) ldg8(p.bias + (size_t)g * p.bias_group_off + col, bias); }
  if constexpr (EPI == EPI_RESID_F) { ldg8(p.bias + col, bias); ldg8(p.gamma + col, gam); }
  if constexpr (EPI == EPI_LN) { ldg8(p.gamma + (size_t)g * p.ln_group_off + col, gam); ldg8(p.beta + (size_t)g * p.ln_group_off + col, bet); }
  const bool use_aux = (EPI == EPI_CONV) && p.aux && ((p.aux_group_mask >> g) & 1);
  const bool use_res = (EPI == EPI_CONV) && p.res_h;
  const bool ln_res = (EPI == EPI_LN) && p.out_f;
  const int rows = min(32, p.M - row0);
  // per-row index math is done once by lane r (for row r) and fetched with a shuffle
  int my_pos = 0, my_valid = 1, my_orow = 0;
  {
    const int mr = row0 + lane;
    if constexpr (EPI == EPI_CONV || EPI == EPI_LN) {
      if (p.pad_h2) { int pos; my_valid = pad_valid(p, mr, pos) ? 1 : 0; my_pos = pos; }
    }
    if constexpr (EPI == EPI_PATCH) {
      const int img = mr / p.tok_per_img;
      my_pos = mr - img * p.tok_per_img;                 // token index inside the image
      my_orow = img * (p.tok_per_img + 1) + 1 + my_pos;  // row of the token matrix (cls rows skipped)
    }
  }
  float* out_f = p.out_f ? p.out_f + (size_t)g * p.out_f_group_off + col : nullptr;
  __half* out_h = p.out_h ? p.out_h + (size_t)g * p.out_h_group_off + col : nullptr;
#pragma unroll 1
  for (int s0 = 0; s0 < STEPS; s0 += U) {
    float v[U][8], x[U][8], a[U][8];
    int pos[U], orow[U];
    bool valid[U], live[U];
    float mean[U], rstd[U];
    // ---- phase 1: staged accumulators + every global operand of the U steps (independent loads in flight)
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int r = (s0 + u) * RPS + rsub;
      const size_t m = (size_t)(row0 + r);
      live[u] = r < rows;
      {
        const float4 a = *reinterpret_cast<const float4*>(stage + acc_idx<W>(r, seg * 8));
        const float4 b = *reinterpret_cast<const float4*>(stage + acc_idx<W>(r, seg * 8 + 4));
        v[u][0] = a.x; v[u][1] = a.y; v[u][2] = a.z; v[u][3] = a.w; v[u][4] = b.x; v[u][5] = b.y; v[u][6] = b.z; v[u][7] = b.w;
      }
      pos[u] = __shfl_sync(0xffffffffu, my_pos, r);
      orow[u] = __shfl_sync(0xffffffffu, my_orow, r);
      valid[u] = __shfl_sync(0xffffffffu, my_valid, r) != 0;
      mean[u] = 0.f; rstd[u] = 0.f;
      if constexpr (EPI == EPI_LN) { mean[u] = __shfl_sync(0xffffffffu, mean_l, r); rstd[u] = __shfl_sync(0xffffffffu, rstd_l, r); }
#pragma unroll
      for (int k = 0; k < 8; ++k) { x[u][k] = 0.f; a[u][k] = 0.f; }
      if (live[u]) {
        if constexpr (EPI == EPI_RESID_F) ld8(out_f + m * p.out_f_ld, x[u]);
        if constexpr (EPI == EPI_PATCH) ldg8(p.aux + (size_t)pos[u] * p.N + col, a[u]);
        if constexpr (EPI == EPI_CONV) {
          if (use_res) ld8h(p.res_h + (size_t)g * p.res_h_group_off + m * p.res_h_ld + col, x[u]);
          if (use_aux) ldg8(p.aux + (size_t)pos[u] * p.N + col, a[u]);
        }
        if constexpr (EPI == EPI_LN) { if (ln_res) ld8(out_f + m * p.out_f_ld, x[u]); }
      }
    }
    // ---- phase 2: arithmetic + stores
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (!live[u]) continue;
      const int r = (s0 + u) * RPS + rsub;
      const size_t m = (size_t)(row0 + r);
      if constexpr (EPI == EPI_STORE_H) {
        if constexpr (ACT == ACT_GELU) {
#pragma unroll
          for (int k = 0; k < 8; k += 2) gelu_erf2(v[u][k] + bias[k], v[u][k + 1] + bias[k + 1], v[u][k], v[u][k + 1]);
        } else {
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const float t = v[u][k] + bias[k];
            v[u][k] = (ACT == ACT_RELU) ? fmaxf(t, 0.f) : t;
          }
        }
        st8h(out_h + m * p.out_h_ld, v[u]);
      } else if constexpr (EPI == EPI_RESID_F) {
#pragma unroll
        for (int k = 0; k < 8; ++k) x[u][k] = fmaf(gam[k], v[u][k] + bias[k], x[u][k]);
        st8(out_f + m * p.out_f_ld, x[u]);
      } else if constexpr (EPI == EPI_PATCH) {
#pragma unroll
        for (int k = 0; k < 8; ++k) v[u][k] += a[u][k];
        st8(out_f + (size_t)orow[u] * p.out_f_ld, v[u]);
      } else if constexpr (EPI == EPI_CONV) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          float t = v[u][k] + bias[k] + x[u][k];
          t = ((ACT == ACT_RELU) ? fmaxf(t, 0.f) : ((ACT == ACT_GELU) ? gelu_erf(t) : t)) + a[u][k];
          v[u][k] = valid[u] ? t : 0.f;
        }
        if (out_f) st8(out_f + m * p.out_f_ld, v[u]);
        if (out_h) st8h(out_h + m * p.out_h_ld, v[u]);
      } else if constexpr (EPI == EPI_STORE_F) {
        st8(out_f + m * p.out_f_ld, v[u]);
      } else if constexpr (EPI == EPI_LN) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float t = (v[u][k] - mean[u]) * rstd[u] * gam[k] + bet[k] + x[u][k];
          v[u][k] = valid[u] ? t : 0.f;
        }
        if (ln_res) st8(out_f + m * p.out_f_ld, v[u]);
        st8h(out_h + m * p.out_h_ld, v[u]);
      }
    }
  }
}

template <int EPI, int W>
__device__ __forceinline__ void epilogue_rows(const GemmParams& p, int g, int row0, int lane, int col_base,
                                              const float* __restrict__ stage, float mean_l, float rstd_l) {
  // the activation is a compile-time parameter of the body (one uniform branch per call instead of one per element)
  if constexpr (EPI == EPI_STORE_H || EPI == EPI_CONV) {
    if (p.act == ACT_GELU) epilogue_rows_impl<EPI, W, ACT_GELU>(p, g, row0, lane, col_base, stage, mean_l, rstd_l);
    else if (p.act == ACT_RELU) epilogue_rows_impl<EPI, W, ACT_RELU>(p, g, row0, lane, col_base, stage, mean_l, rstd_l);
    else epilogue_rows_impl<EPI, W, ACT_NONE>(p, g, row0, lane, col_base, stage, mean_l, rstd_l);
  } else {
    epilogue_rows_impl<EPI, W, ACT_NONE>(p, g, row0, lane, col_base, stage, mean_l, rstd_l);
  }
}

// ---- TMA tensor stores (cp.async.bulk.tensor.3d.global.shared::cta) ---------------------------------------------
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, uint32_t src_smem, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(map), "r"(src_smem), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- matcher epilogues (reference modules/utils/feature_matcher.py:64-83) -----------------------------------
// softmax(dim=1) * softmax(dim=2) of the dustbin-augmented S/T equals exp(2 s - lse_row - lse_col) with the two
// log-sum-exps taken over the valid cells plus the dustbin.  Pass 1 (EPI_LSE) emits, from ONE evaluation of the S tile,
// online-softmax partials (max, sum) of every row over the warp's 64 columns and of every column over the warp's 32
// rows; a tiny kernel (matcher_lse_reduce_kernel) folds the partials and the dustbin into the two vectors; pass 2
// (EPI_DUAL) re-evaluates S and writes the outputs.  Everything is kept relative to true row / column maxima, so no
// logit range (un-normalised descriptors, small temperatures) can underflow a whole row.  All in the log2 domain.
//
// Transposing reductions over a warp: lane l holds part[j] = its row's value for column j; after the recursive-halving
// exchange (31 shuffles) lane j holds the reduction over the 32 rows of column j.  Fixed order, bit-reproducible.
__device__ __forceinline__ float warp_colmax32(float (&part)[32], int lane) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    const bool upper = (lane & o) != 0;
#pragma unroll
    for (int i = 0; i < o; ++i) {
      const float send = upper ? part[i] : part[i + o];
      const float keep = upper ? part[i + o] : part[i];
      part[i] = fmaxf(keep, __shfl_xor_sync(0xffffffffu, send, o));
    }
  }
  return part[0];
}

__device__ __forceinline__ float warp_rowsum32(float (&part)[32], int lane) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    const bool upper = (lane & o) != 0;
#pragma unroll
    for (int i = 0; i < o; ++i) {
      const float send = upper ? part[i] : part[i + o];
      const float keep = upper ? part[i + o] : part[i];
      part[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
    }
  }
  return part[0];
}

#define MK_NEG_INF (__int_as_float(0xff800000))          /* -inf */

// One 32 x 32 chunk of pass 1.  x[j] = S[row][col0 + j] * inv_temp * log2(e), or -inf outside the valid rows / columns.
// Updates the row's running (rmax, rsum) and stores the column partial of the warp's 32 rows.
__device__ __forceinline__ void lse_chunk(const GemmParams& p, int g, int col0, int lane, int col_slot, bool row_ok,
                                          const float (&v)[32], float& rmax, float& rsum) {
  const float k2 = p.inv_temp * 1.4426950408889634f;
  float x[32], t[32];
  float cm = MK_NEG_INF;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    x[j] = (row_ok && col0 + j < p.n_valid) ? v[j] * k2 : MK_NEG_INF;
    cm = fmaxf(cm, x[j]);
    t[j] = x[j];
  }
  // rows: online update over the chunks of this warp (a row with no valid cell keeps (-inf, 0))
  const float nm = fmaxf(rmax, cm);
  const float base = (nm == MK_NEG_INF) ? 0.f : nm;
  float acc = 0.f;
#pragma unroll
  for (int j = 0; j < 32; ++j) acc += ex2_approx_f(x[j] - base);
  rsum = rsum * ex2_approx_f(rmax - base) + acc;
  rmax = nm;
  // columns: max over the 32 rows, then the sum relative to it
  const float cmax_l = warp_colmax32(t, lane);
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const float cj = __shfl_sync(0xffffffffu, cmax_l, j);
    t[j] = ex2_approx_f(x[j] - ((cj == MK_NEG_INF) ? 0.f : cj));
  }
  const float csum_l = warp_rowsum32(t, lane);
  const int col = col0 + lane;
  if (col < p.n_valid) p.part_col[((size_t)g * (p.part_ld / 32) + col_slot) * p.part_ld + col] = make_float2(cmax_l, csum_l);
}

// The same chunk when every |S| is known to be <= p.lse_bound (L2-normalised descriptors, DSC_HEAD.NORM_DSC: True, and a
// temperature for which 2 * bound / T stays inside the fp32 exponent range): one fixed shift serves rows and columns,
// so a cell costs ONE exponential and the column partial one transposing sum (no max passes).  Slots hold (shift, sum).
__device__ __forceinline__ void lse_chunk_bounded(const GemmParams& p, int g, int col0, int lane, int col_slot, bool row_ok,
                                                  const float (&v)[32], float& rsum) {
  const float k2 = p.inv_temp * 1.4426950408889634f, sh = p.lse_bound * k2;
  float t[32];
  float acc0 = 0.f, acc1 = 0.f;
#pragma unroll
  for (int j = 0; j < 32; j += 2) {
    const float e0 = (row_ok && col0 + j < p.n_valid) ? ex2_approx_f(fmaf(v[j], k2, -sh)) : 0.f;
    const float e1 = (row_ok && col0 + j + 1 < p.n_valid) ? ex2_approx_f(fmaf(v[j + 1], k2, -sh)) : 0.f;
    t[j] = e0; t[j + 1] = e1;
    acc0 += e0; acc1 += e1;
  }
  rsum += acc0 + acc1;
  const float csum_l = warp_rowsum32(t, lane);
  const int col = col0 + lane;
  if (col < p.n_valid) p.part_col[((size_t)g * (p.part_ld / 32) + col_slot) * p.part_ld + col] = make_float2(sh, csum_l);
}

// Pass 2, one 32 x 32 chunk, coalesced: the warp owns rows row0..row0+31 (lane == row on entry).  Each lane evaluates
// its row's scores with the column terms read from the warp's staging block (broadcast loads), the block is transposed
// through `stage` ([32][33] floats + 64 floats of column operands, warp-private), then lane == column writes one
// contiguous 128-byte row segment per store instruction.  scores / kp_scores may be NULL ("lean" mode).
__device__ __forceinline__ void dual_store_chunk(const GemmParams& p, int g, int row0, int lane, int n0,
                                                 const float (&v)[32], float* stage, float lr, float s0) {
  const float k2x2 = 2.0f * p.inv_temp * 1.4426950408889634f;
  const size_t gv = (size_t)g * p.n_valid;
  const size_t go = (size_t)g * p.n_valid * (size_t)p.out_pitch;
  const int col = n0 + lane;
  const bool col_ok = col < p.n_valid;
  float* lcs = stage + 32 * 33;
  const float lc_l = col_ok ? __ldg(p.lse_c + (size_t)g * p.part_ld + col) : -MK_NEG_INF;     // +inf -> score 0
  const float s1 = col_ok ? __ldg(p.scr1 + gv + col) : 0.0f;
  lcs[lane] = lc_l;
  __syncwarp();
#pragma unroll
  for (int j = 0; j < 32; ++j) stage[lane * 33 + j] = ex2_approx_f(fmaf(v[j], k2x2, -lr) - lcs[j]);
  __syncwarp();
  const int rows = min(32, p.n_valid - row0);
  const bool full = p.scores != nullptr;
#pragma unroll 4
  for (int r = 0; r < rows; ++r) {
    const float sc = stage[r * 33 + lane];
    const float kp = __shfl_sync(0xffffffffu, s0, r) * s1;
    if (col_ok) {
      const size_t o = go + (size_t)(row0 + r) * (size_t)p.out_pitch + col;
      if (full) { p.scores[o] = sc; p.kp_scores[o] = kp; }
      p.final_scores[o] = sc * kp;
    }
  }
  __syncwarp();
}

// Pass 2 through TMA: the outputs' rows are 16-byte aligned (row pitch padded to a multiple of 4 floats; the unpadded
// N = 1938 rows of the reference's contiguous layout are only 8-byte aligned, which no tensor map can describe).
// thread == row: a lane computes its row's 32 scores, kp_scores and final_scores and writes them as eight 16-byte
// chunks per output into the warp's three 32 x 32 fp32 staging boxes in the 128-byte-swizzle pattern (chunk k of row r
// at chunk k ^ (r & 7): conflict-free), then one lane issues three tensor stores (hardware clips rows / columns beyond
// n_valid).  No transposition pass, full 128-byte lines on the way to L2.
// `stage`: 3 x 4 KB, 1024-byte aligned, warp-private; `aux`: 64 floats (column operands), warp-private.
__device__ __forceinline__ void dual_store_chunk_tma(const GemmParams& p, const OutMaps& om, int g, int row0, int lane, int n0,
                                                     const float (&v)[32], float* stage, float* aux, float lr, float s0,
                                                     float lc_l, float s1_l) {
  // lc_l / s1_l: column operands of column n0 + lane (lse of the column, +inf beyond n_valid; keypoint score), loaded by
  // the caller for all of the warp's chunks at once so that their latency is paid once per tile
  const float k2x2 = 2.0f * p.inv_temp * 1.4426950408889634f;
  const bool full = p.scores != nullptr;
  // the previous chunk's stores must have finished READING the staging boxes
  if (lane == 0) tma_store_wait_read();
  __syncwarp();
  aux[lane] = lc_l;
  aux[32 + lane] = s1_l;
  __syncwarp();
  float4* b_sc = reinterpret_cast<float4*>(stage) + lane * 8;
  float4* b_kp = b_sc + 256;
  float4* b_fs = b_sc + 512;
  const int sw = lane & 7;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float4 lc = *reinterpret_cast<const float4*>(aux + 4 * k), s1 = *reinterpret_cast<const float4*>(aux + 32 + 4 * k);
    float4 sc, kp, fs;
    sc.x = ex2_approx_f(fmaf(v[4 * k + 0], k2x2, -lr) - lc.x); sc.y = ex2_approx_f(fmaf(v[4 * k + 1], k2x2, -lr) - lc.y);
    sc.z = ex2_approx_f(fmaf(v[4 * k + 2], k2x2, -lr) - lc.z); sc.w = ex2_approx_f(fmaf(v[4 * k + 3], k2x2, -lr) - lc.w);
    kp.x = s0 * s1.x; kp.y = s0 * s1.y; kp.z = s0 * s1.z; kp.w = s0 * s1.w;
    fs.x = sc.x * kp.x; fs.y = sc.y * kp.y; fs.z = sc.z * kp.z; fs.w = sc.w * kp.w;
    const int kk = k ^ sw;
    if (full) { b_sc[kk] = sc; b_kp[kk] = kp; }
    b_fs[kk] = fs;
  }
  fence_async_smem();
  __syncwarp();
  if (lane == 0) {
    const uint32_t sa = (uint32_t)__cvta_generic_to_shared(stage);
    if (full) { tma_store_3d(&om.m[0], sa, n0, row0, g); tma_store_3d(&om.m[1], sa + 4096, n0, row0, g); }
    tma_store_3d(&om.m[2], sa + 8192, n0, row0, g);
    tma_store_commit();
  }
}

// EPI_LN: normalise the 128-wide row (N == 128 == tile width), then optional residual add.
//   out_f (if set): x32[m] = x32[m] + LN(acc)  (in place), fp16 copy of the sum -> out_h
//   else          : out_h = LN(acc)
__device__ __forceinline__ void ln_store_chunk(const GemmParams& p, int g, int m, int n0, float (&v)[32],
                                               float mean, float rstd) {
  if (m >= p.M) return;
  const float* gm = p.gamma + (size_t)g * p.ln_group_off + n0;
  const float* bt = p.beta + (size_t)g * p.ln_group_off + n0;
#pragma unroll
  for (int j = 0; j < 32; ++j) v[j] = (v[j] - mean) * rstd * __ldg(gm + j) + __ldg(bt + j);
  if (p.out_f) {
    float* o = p.out_f + (size_t)g * p.out_f_group_off + (size_t)m * p.out_f_ld + n0;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      float4 x = reinterpret_cast<float4*>(o)[q];
      v[q * 4 + 0] += x.x; v[q * 4 + 1] += x.y; v[q * 4 + 2] += x.z; v[q * 4 + 3] += x.w;
    }
  }
  if (p.pad_h2) {
    int pos;
    if (!pad_valid(p, m, pos)) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = 0.0f;
    }
  }
  if (p.out_f) {
    float* o = p.out_f + (size_t)g * p.out_f_group_off + (size_t)m * p.out_f_ld + n0;
#pragma unroll
    for (int q = 0; q < 8; ++q)
      reinterpret_cast<float4*>(o)[q] = make_float4(v[q * 4], v[q * 4 + 1], v[q * 4 + 2], v[q * 4 + 3]);
  }
  store_h32(p.out_h + (size_t)g * p.out_h_group_off + (size_t)m * p.out_h_ld + n0, v);
}

}  // namespace mk
