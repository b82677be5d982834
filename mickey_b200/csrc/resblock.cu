// The heads' residual block (BasicBlock, extractor_utils.py:12-35) for training: forward and backward with TF32 wgmma
// convolutions and training-mode batch norm (include/mickey_b200.h mk_resblock*, DESIGN.md §6h).
//
// Activations live in the engine's padded NHWC layout (DESIGN.md §3): row r = b (h+2)(w+2) + (y+1)(w+2) + (x+1) of an
// [R, C] fp32 buffer, R = B (h+2)(w+2), with a zero ring around every image.  The weight gradients also need each
// operand channel-major, [C, Rp] with Rp = R rounded up to 4 (a 16-byte pitch); the kernels that write an operand write
// both copies.  Every MMA operand is rounded to TF32 (cvt.rna) by the kernel that writes it.
//
// One TF32 wgmma GEMM (rb_gemm_kernel) serves the three convolution forms.  TF32 wgmma reads both operands K-major:
//   forward   Z[r, co]      = sum_t sum_ci X[r + off(t), ci] W[co, t, ci]      A = X [R, cin], B = W as [cout, 9 cin]
//   dgrad     dX[r, ci]     = sum_t sum_co dZ[r + off(t), co] W[co, 8 - t, ci] A = dZ [R, cout], B = W as [cin, 9 cout]
//   wgrad     dW[co, t, ci] = sum_p dZ[p, co] X[p + off(t), ci]                A = dZ^T [cout, Rp], B = X^T [cin, Rp]
// with off(t) = (ky - 1)(w+2) + (kx - 1).  The forward and dgrad K loops walk taps x 32-channel chunks, a tap being a
// row offset of the A tile that TMA zero-fills beyond the buffer.  The wgrad runs one GEMM per tap: its shift off(t)
// falls on the contiguous (pixel) dimension of X^T, where a TMA box must start 16-byte aligned, so a small kernel first
// writes X^T shifted by off(t) into an aligned buffer.  The pixel range is cut into a fixed number of slots whose partial
// products are folded in slot order.
//
// Batch-norm statistics are exact fp64 sums over fixed row slots, folded in slot order (mean first, then the centred
// second moment), and running statistics are updated as F.batch_norm does.  No atomics anywhere: every output, gradient
// and running statistic is bit-identical run to run.
#include "../../include/mickey_b200.h"
#include "gemm.h"
#include "gemm_tc.cuh"

#include <algorithm>
#include <cstring>

namespace mk {

namespace {

constexpr int RB_BM = 128;                // GEMM tile rows (two consumer warpgroups of 64)
constexpr int RB_BK = 32;                 // fp32 per 128-byte swizzle row: one K chunk
constexpr int RB_THREADS = 288;           // 8 MMA warps + 1 producer warp
constexpr int RB_TILE = 32;               // element-wise kernels: 32 rows x 32 channels per block
constexpr long long RB_MAX_ROWS = 1LL << 24;
constexpr int RB_MAX_C = 4096;
constexpr int RB_WG_TARGET = 264;         // wgrad CTAs aimed at (two per SM's worth of 132 SMs)
constexpr int RB_WG_MAX_SLOTS = 32;

template <int BN> constexpr int rb_stages() { return BN == 128 ? 5 : 6; }
template <int BN> constexpr int rb_smem_bytes() { return rb_stages<BN>() * (RB_BM * 128 + BN * 128) + 1024 + 256; }

__device__ __forceinline__ float tf32r(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

__device__ __forceinline__ void wgmma_tf32_m64n64k8(float (&d)[32], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.eq.u32 p, 1, 1;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b));
}

__device__ __forceinline__ void wgmma_tf32_m64n128k8(float (&d)[64], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.eq.u32 p, 1, 1;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b));
}

// ---- the TF32 convolution GEMM ------------------------------------------------------------------------------------
struct RbGemm {
  int M, N;                 // output rows / columns (wgrad: N = taps * cin)
  int k_chunks;             // forward / dgrad: taps * cpt; wgrad: pixel chunks of 32
  int cpt;                  // forward / dgrad: K chunks per tap
  int taps;
  int shift[9];             // forward / dgrad: A row offset per tap
  int cin;                  // wgrad: input channels (the output columns of this tap)
  int chunks_per_slot;      // wgrad
  float* out; long long ldo; long long slot_stride;
};

// Forward / dgrad: blockIdx.x = m_tile * n_tiles + n_tile.  Wgrad (one tap per launch, p.out at the tap's columns):
// blockIdx = (ci block, m tile, slot).  Warps 0-7 are two MMA warpgroups (tile rows 0-63 / 64-127), warp 8 the TMA producer.
template <int BN, bool WGRAD>
__global__ void __launch_bounds__(RB_THREADS, 1)
rb_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const RbGemm p) {
  constexpr int STAGES = rb_stages<BN>();
  constexpr int A_BYTES = RB_BM * 128, STAGE_BYTES = A_BYTES + BN * 128;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const uint32_t full0 = base + STAGES * STAGE_BYTES, empty0 = full0 + 8 * STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  int m0, n0, kc0 = 0, kc1 = p.k_chunks;
  float* out = p.out;
  if constexpr (WGRAD) {
    n0 = blockIdx.x * BN;
    m0 = blockIdx.y * RB_BM;
    kc0 = blockIdx.z * p.chunks_per_slot;
    kc1 = min(p.k_chunks, kc0 + p.chunks_per_slot);
    out += (long long)blockIdx.z * p.slot_stride;
  } else {
    const int nt = (p.N + BN - 1) / BN;
    n0 = (blockIdx.x % nt) * BN;
    m0 = (blockIdx.x / nt) * RB_BM;
  }
  const int n_lim = WGRAD ? p.cin : p.N;

  if (warp == 8 && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, 8);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();

  if (warp == 8) {
    if (elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kc = kc0; kc < kc1; ++kc) {
        mbar_wait(empty0 + 8 * stage, phase ^ 1);
        const uint32_t sa = base + stage * STAGE_BYTES, fb = full0 + 8 * stage;
        mbar_expect_tx(fb, STAGE_BYTES);
        if constexpr (WGRAD) {
          tma_load_2d(sa, &tmA, fb, kc * RB_BK, m0);
          tma_load_2d(sa + A_BYTES, &tmB, fb, kc * RB_BK, n0);
        } else {
          const int t = kc / p.cpt, kin = kc - t * p.cpt;
          tma_load_2d(sa, &tmA, fb, kin * RB_BK, m0 + p.shift[t]);
          tma_load_2d(sa + A_BYTES, &tmB, fb, kc * RB_BK, n0);
        }
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  const int wg = warp >> 2;
  float d[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
  int stage = 0;
  uint32_t phase = 0;
  for (int kc = kc0; kc < kc1; ++kc) {
    mbar_wait(full0 + 8 * stage, phase);
    const uint32_t sa = base + stage * STAGE_BYTES;
    const uint64_t da = gmma_desc_sw128(sa + wg * (64 * 128));
    const uint64_t db = gmma_desc_sw128(sa + A_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < RB_BK / 8; ++k) {
      // 8 fp32 = 32 bytes along K inside the 128-byte swizzle row: +2 in the (addr >> 4) field
      if constexpr (BN == 128) wgmma_tf32_m64n128k8(d, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2));
      else wgmma_tf32_m64n64k8(d, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2));
    }
    wgmma_commit();
    wgmma_wait<1>();
    reg_fence(d);
    if (kc > kc0 && lane == 0) mbar_arrive(empty0 + 8 * (stage == 0 ? STAGES - 1 : stage - 1));
    if (++stage == STAGES) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  reg_fence(d);
  pdl_trigger();
  // fragment layout of wgmma m64nNk8: d[4j + 2h + e] = (row 16 (warp & 3) + lane / 4 + 8 h, column 8 j + 2 (lane & 3) + e)
  const int r_base = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int c = n0 + 8 * j + 2 * (lane & 3);
    if (c >= n_lim) continue;                          // n_lim is a multiple of 32: c < n_lim implies c + 1 < n_lim
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = r_base + 8 * h;
      if (r < p.M) *reinterpret_cast<float2*>(out + (long long)r * p.ldo + c) = make_float2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
    }
  }
}

// ---- element-wise kernels -----------------------------------------------------------------------------------------
struct Geo { int B, h, w, H2, W2, P, R, Rp; };

__device__ __forceinline__ bool interior(const Geo& g, int r, int& b, int& y, int& x) {
  b = r / g.P;
  const int rem = r - b * g.P;
  const int yy = rem / g.W2;
  y = yy - 1;
  x = rem - yy * g.W2 - 1;
  return r < g.R && y >= 0 && y < g.h && x >= 0 && x < g.w;
}

struct Nchw { const float* p; long long sb, sc, sy, sx; };
__device__ __forceinline__ float ld_nchw(const Nchw& t, int b, int c, int y, int x) {
  return t.p[b * t.sb + c * t.sc + y * t.sy + x * t.sx];
}

enum PackMode : int {
  PK_NCHW = 0,     // v = src(b, c, y, x) [* (mask(b, c, y, x) > 0)]                         (input, grad_out through ReLU)
  PK_BN_FWD = 1,   // v = relu(bn(Z[r, c]))                                                  (BN1-apply + ReLU)
  PK_BN_BWD = 2,   // g = G[r, c] [* (Mk[r, c] > 0)]; v = k (g - a - xhat bb)                 (BN backward)
};

struct Pack {
  int C;
  Nchw src, mask;                 // PK_NCHW
  const float* Z; const float* G; const float* Mk;   // [R, C]
  const float* mean; const float* rstd; const float* gamma; const float* beta;   // PK_BN_FWD (bn)
  const float* coef;              // PK_BN_BWD: k [C], a [C], bb [C]
  int bn;
  float* o_f32; float* o_tf; float* o_cm;   // [R, C] fp32, [R, C] TF32, [C, Rp] TF32 (each optional)
};

// One 32-row x 32-channel tile per block (32 x 8 threads): computed in the reading layout, written through shared memory
// in both the row-major and the channel-major layouts.  Ring rows (and rows R..Rp of the channel-major copy) are zero.
template <int MODE>
__global__ void __launch_bounds__(256) rb_pack_kernel(Geo g, Pack k) {
  __shared__ float t[RB_TILE][RB_TILE + 1];
  pdl_wait();
  const int r0 = blockIdx.x * RB_TILE, c0 = blockIdx.y * RB_TILE, tx = threadIdx.x, ty = threadIdx.y;
  if (MODE == PK_NCHW) {
    const int r = r0 + tx;
    int b, y, x;
    const bool in = interior(g, r, b, y, x);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = c0 + ty + 8 * i;
      float v = 0.f;
      if (in) {
        v = ld_nchw(k.src, b, c, y, x);
        if (k.mask.p && !(ld_nchw(k.mask, b, c, y, x) > 0.f)) v = 0.f;
      }
      t[tx][ty + 8 * i] = v;
    }
  } else {
    const int c = c0 + tx;
    float m = 0.f, rs = 1.f, ga = 1.f, be = 0.f, kk = 1.f, aa = 0.f, bb = 0.f;
    if (k.bn) {
      m = k.mean[c]; rs = k.rstd[c];
      if (MODE == PK_BN_FWD) { ga = k.gamma[c]; be = k.beta[c]; }
      else { kk = k.coef[c]; aa = k.coef[k.C + c]; bb = k.coef[2 * k.C + c]; }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = r0 + ty + 8 * i;
      int b, y, x;
      float v = 0.f;
      if (interior(g, r, b, y, x)) {
        const long long e = (long long)r * k.C + c;
        if (MODE == PK_BN_FWD) {
          v = k.Z[e];
          if (k.bn) v = (v - m) * rs * ga + be;
          v = fmaxf(v, 0.f);
        } else {
          float gv = k.G[e];
          if (k.Mk && !(k.Mk[e] > 0.f)) gv = 0.f;
          v = k.bn ? kk * (gv - aa - (k.Z[e] - m) * rs * bb) : gv;
        }
      }
      t[ty + 8 * i][tx] = v;
    }
  }
  __syncthreads();
  pdl_trigger();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = r0 + ty + 8 * i, c = c0 + tx;
    if (r < g.R) {
      const float v = t[ty + 8 * i][tx];
      const long long e = (long long)r * k.C + c;
      if (k.o_f32) k.o_f32[e] = v;
      if (k.o_tf) k.o_tf[e] = tf32r(v);
    }
  }
  if (k.o_cm) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = c0 + ty + 8 * i, r = r0 + tx;
      if (r < g.Rp) k.o_cm[(long long)c * g.Rp + r] = tf32r(t[tx][ty + 8 * i]);
    }
  }
}

// Per-slot, per-channel fp64 sums over the interior rows of slot s: s1 = sum u, s2 = sum u v with
// u = G[r, c] [* (Mk > 0)] [- shift[c]] and v = Zx ? (Zx[r, c] - mean[c]) rstd[c] : u.
// grid (C / 32, slots), 32 x 8 threads; part = double [2][slots][C].
struct Stats {
  int C, rows_per_slot;
  const float* G; const float* Mk; const float* shift; const float* Zx; const float* mean; const float* rstd;
  double* part;
};
__global__ void __launch_bounds__(256) rb_stats_kernel(Geo g, Stats s) {
  __shared__ double red[2][8][32];
  pdl_wait();
  const int c = blockIdx.x * 32 + threadIdx.x, ty = threadIdx.y;
  const int rb = blockIdx.y * s.rows_per_slot, re = min(g.R, rb + s.rows_per_slot);
  const float sh = s.shift ? s.shift[c] : 0.f;
  const float m = s.Zx ? s.mean[c] : 0.f, rs = s.Zx ? s.rstd[c] : 0.f;
  double s1 = 0.0, s2 = 0.0;
  for (int r = rb + ty; r < re; r += 8) {
    int b, y, x;
    if (!interior(g, r, b, y, x)) continue;
    const long long e = (long long)r * s.C + c;
    float u = s.G[e];
    if (s.Mk && !(s.Mk[e] > 0.f)) u = 0.f;
    const double ud = (double)u - (double)sh;
    const double vd = s.Zx ? ((double)s.Zx[e] - (double)m) * (double)rs : ud;
    s1 += ud;
    s2 += ud * vd;
  }
  red[0][ty][threadIdx.x] = s1;
  red[1][ty][threadIdx.x] = s2;
  __syncthreads();
  pdl_trigger();
  if (ty == 0) {
    double a = 0.0, q = 0.0;
    for (int i = 0; i < 8; ++i) { a += red[0][i][threadIdx.x]; q += red[1][i][threadIdx.x]; }
    const int slots = gridDim.y;
    s.part[(long long)blockIdx.y * s.C + c] = a;
    s.part[((long long)slots + blockIdx.y) * s.C + c] = q;
  }
}

enum FoldMode : int { FD_MEAN = 0, FD_VAR = 1, FD_EVAL = 2, FD_BWD = 3 };
struct Fold {
  int C, slots, train;
  double count;                       // B h w
  const double* part;
  float eps, momentum;                // momentum: the exponential-average factor of this call
  float* mean; float* rstd;           // [C] in the workspace
  float* run_mean; float* run_var;    // the module's buffers
  const float* gamma;
  float* dgamma; float* dbeta;        // FD_BWD outputs (optional)
  float* coef;                        // FD_BWD: k, a, bb [3][C]
};
__global__ void __launch_bounds__(128) rb_fold_kernel(int mode, Fold f) {
  pdl_wait();
  const int c = blockIdx.x * 128 + threadIdx.x;
  if (c >= f.C) return;
  double s1 = 0.0, s2 = 0.0;
  if (mode != FD_EVAL)
    for (int s = 0; s < f.slots; ++s) {
      s1 += f.part[(long long)s * f.C + c];
      s2 += f.part[((long long)f.slots + s) * f.C + c];
    }
  if (mode == FD_MEAN) {
    f.mean[c] = (float)(s1 / f.count);
  } else if (mode == FD_VAR) {
    const double var = s2 / f.count;
    f.rstd[c] = (float)(1.0 / sqrt(var + (double)f.eps));
    const float mom = f.momentum;
    f.run_mean[c] = mom * f.mean[c] + (1.f - mom) * f.run_mean[c];
    f.run_var[c] = mom * (float)(var * f.count / (f.count - 1.0)) + (1.f - mom) * f.run_var[c];
  } else if (mode == FD_EVAL) {
    f.mean[c] = f.run_mean[c];
    f.rstd[c] = 1.f / sqrtf(f.run_var[c] + f.eps);
  } else {
    if (f.dbeta) f.dbeta[c] = (float)s1;
    if (f.dgamma) f.dgamma[c] = (float)s2;
    f.coef[c] = f.gamma[c] * f.rstd[c];
    f.coef[f.C + c] = f.train ? (float)(s1 / f.count) : 0.f;
    f.coef[2 * f.C + c] = f.train ? (float)(s2 / f.count) : 0.f;
  }
  pdl_trigger();
}

// out (NCHW, contiguous) = act(bn2(Z2[r, c]) + S) with S = Ssc[r, c] (1x1 shortcut) or x(b, c, y, x) (identity)
struct Final {
  int C, bn, relu;
  const float* Z; const float* mean; const float* rstd; const float* gamma; const float* beta;
  const float* Ssc; Nchw x;
  float* out;
};
__global__ void __launch_bounds__(256) rb_final_kernel(Geo g, Final k) {
  __shared__ float t[RB_TILE][RB_TILE + 1];
  pdl_wait();
  const int r0 = blockIdx.x * RB_TILE, c0 = blockIdx.y * RB_TILE, tx = threadIdx.x, ty = threadIdx.y;
  {
    const int c = c0 + tx;
    float m = 0.f, rs = 1.f, ga = 1.f, be = 0.f;
    if (k.bn) { m = k.mean[c]; rs = k.rstd[c]; ga = k.gamma[c]; be = k.beta[c]; }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = r0 + ty + 8 * i;
      float v = 0.f;
      if (r < g.R) {
        const long long e = (long long)r * k.C + c;
        v = k.Z[e];
        if (k.bn) v = (v - m) * rs * ga + be;
        if (k.Ssc) v += k.Ssc[e];
      }
      t[ty + 8 * i][tx] = v;
    }
  }
  __syncthreads();
  pdl_trigger();
  const int r = r0 + tx;
  int b, y, x;
  if (!interior(g, r, b, y, x)) return;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = c0 + ty + 8 * i;
    float v = t[tx][ty + 8 * i];
    if (!k.Ssc) v += ld_nchw(k.x, b, c, y, x);
    if (k.relu) v = fmaxf(v, 0.f);
    k.out[(((long long)b * k.C + c) * g.h + y) * g.w + x] = v;
  }
}

// dX (NCHW, contiguous) = D1[r, c] + D2[r, c] (either optional), summed in that order
__global__ void __launch_bounds__(256) rb_dx_kernel(Geo g, int C, const float* D1, const float* D2, float* dx) {
  __shared__ float t[RB_TILE][RB_TILE + 1];
  pdl_wait();
  const int r0 = blockIdx.x * RB_TILE, c0 = blockIdx.y * RB_TILE, tx = threadIdx.x, ty = threadIdx.y;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = r0 + ty + 8 * i;
    float v = 0.f;
    if (r < g.R) {
      const long long e = (long long)r * C + c0 + tx;
      if (D1) v = D1[e];
      if (D2) v = D1 ? v + D2[e] : D2[e];
    }
    t[ty + 8 * i][tx] = v;
  }
  __syncthreads();
  pdl_trigger();
  const int r = r0 + tx;
  int b, y, x;
  if (!interior(g, r, b, y, x)) return;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int c = c0 + ty + 8 * i;
    dx[(((long long)b * C + c) * g.h + y) * g.w + x] = t[tx][ty + 8 * i];
  }
}

// Weight re-layout and TF32 rounding of W [cout, cin, taps] (the torch layout):
//   dgrad = 0: out[co][t][ci] = W[co][ci][t]            (forward B, [cout, taps cin])
//   dgrad = 1: out[ci][t][co] = W[co][ci][taps - 1 - t]  (dgrad B, [cin, taps cout])
__global__ void __launch_bounds__(256) rb_weight_kernel(const float* W, int cout, int cin, int taps, int dgrad, float* out) {
  pdl_wait();
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x, n = (long long)cout * cin * taps;
  if (i >= n) return;
  int co, ci, t;
  if (!dgrad) { ci = (int)(i % cin); t = (int)((i / cin) % taps); co = (int)(i / ((long long)cin * taps)); }
  else { co = (int)(i % cout); t = taps - 1 - (int)((i / cout) % taps); ci = (int)(i / ((long long)cout * taps)); }
  out[i] = tf32r(W[((long long)co * cin + ci) * taps + t]);
  pdl_trigger();
}

// dst[c][p] = src[c][p + off] (zero outside [0, Rp)): a wgrad tap's operand, aligned for TMA
__global__ void __launch_bounds__(256) rb_shift_kernel(const float* src, float* dst, int C, int Rp, int off) {
  pdl_wait();
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= (long long)C * Rp) return;
  const int p = (int)(i % Rp) + off;
  dst[i] = p >= 0 && p < Rp ? src[i + off] : 0.f;
  pdl_trigger();
}

// dW[co][ci][t] = sum over the slots s, in order, of part[s][co][t cin + ci]
__global__ void __launch_bounds__(256) rb_wfold_kernel(const float* part, int slots, long long slot_stride, int cout, int cin,
                                                       int taps, float* dw) {
  pdl_wait();
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x, n = (long long)cout * cin * taps;
  if (i >= n) return;
  const int t = (int)(i % taps), ci = (int)((i / taps) % cin), co = (int)(i / ((long long)taps * cin));
  const float* p = part + (long long)co * taps * cin + (long long)t * cin + ci;
  float acc = 0.f;
  for (int s = 0; s < slots; ++s) acc += p[(long long)s * slot_stride];
  dw[i] = acc;
  pdl_trigger();
}

// ---- host side ----------------------------------------------------------------------------------------------------
static_assert(RB_BK * 4 == 128, "encode_tensor_map_2d's fp32 box is one 128-byte swizzle row: RB_BK columns");

size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }

Geo geo(int B, int h, int w) {
  Geo g;
  g.B = B; g.h = h; g.w = w; g.H2 = h + 2; g.W2 = w + 2; g.P = g.H2 * g.W2; g.R = B * g.P; g.Rp = (g.R + 3) & ~3;
  return g;
}

void conv_shifts(const Geo& g, int taps, int* shift) {
  for (int t = 0; t < 9; ++t) shift[t] = 0;
  if (taps == 9)
    for (int t = 0; t < 9; ++t) shift[t] = (t / 3 - 1) * g.W2 + (t % 3 - 1);
}

int stat_slots(const Geo& g) { return std::max(1, std::min(128, ceil_div(g.R, 256))); }

int bn_of(int n) { return n >= 128 ? 128 : 64; }

// wgrad pixel slots: enough CTAs per tap's launch to fill the GPU, never an empty slot
void wgrad_plan(const Geo& g, int cout, int cin, int taps, int& slots, int& cps) {
  const int bn = bn_of(cin);
  const int tiles = ceil_div(cout, RB_BM) * ceil_div(cin, bn);      // one launch per tap
  const int kch = ceil_div(g.R, RB_BK);
  int s = std::max(1, std::min(RB_WG_MAX_SLOTS, ceil_div(RB_WG_TARGET, tiles)));
  s = std::min(s, kch);
  cps = ceil_div(kch, s);
  slots = ceil_div(kch, cps);
}

template <int BN, bool WGRAD>
cudaError_t launch_gemm(const CUtensorMap& a, const CUtensorMap& b, const RbGemm& p, dim3 grid, cudaStream_t st) {
  constexpr int smem = rb_smem_bytes<BN>();
  cudaError_t e = cudaFuncSetAttribute(rb_gemm_kernel<BN, WGRAD>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return e;
  return launch_k(rb_gemm_kernel<BN, WGRAD>, grid, dim3(RB_THREADS), smem, st, a, b, p);
}

// forward / dgrad: out [R, N] = sum_t A[r + shift(t)] . Bw[n, t, :]; A [R, K1] (K1 = channels), Bw [N, taps K1]
int conv_fwd(const Geo& g, const float* A, int K1, const float* Bw, int N, int taps, float* out, cudaStream_t st) {
  CUtensorMap ta, tb;
  MK_TRY(encode_tensor_map_2d(&ta, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, A, g.R, K1, K1, RB_BM));
  const int bn = bn_of(N);
  MK_TRY(encode_tensor_map_2d(&tb, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, Bw, N, (long long)taps * K1, (long long)taps * K1, bn));
  RbGemm p;
  memset(&p, 0, sizeof(p));
  p.M = g.R; p.N = N; p.cpt = K1 / RB_BK; p.k_chunks = taps * p.cpt; p.taps = taps;
  conv_shifts(g, taps, p.shift);
  p.out = out; p.ldo = N;
  const dim3 grid(ceil_div(g.R, RB_BM) * ceil_div(N, bn));
  MK_CUDA_CHECK((bn == 128 ? launch_gemm<128, false>(ta, tb, p, grid, st) : launch_gemm<64, false>(ta, tb, p, grid, st)));
  return MK_OK;
}

// wgrad: dW [cout, cin, taps] from dZT [cout, Rp] and XT [cin, Rp]; per-tap shifted operand in xs [cin, Rp] (taps = 9),
// partials in part
int conv_wgrad(const Geo& g, const float* dZT, const float* XT, int cout, int cin, int taps, float* xs, float* part, float* dw,
               cudaStream_t st) {
  int slots, cps;
  wgrad_plan(g, cout, cin, taps, slots, cps);
  const int bn = bn_of(cin);
  int shift[9];
  conv_shifts(g, taps, shift);
  CUtensorMap ta, tb;
  MK_TRY(encode_tensor_map_2d(&ta, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, dZT, cout, g.Rp, g.Rp, RB_BM));
  RbGemm p;
  memset(&p, 0, sizeof(p));
  p.M = cout; p.N = cin; p.k_chunks = ceil_div(g.R, RB_BK); p.taps = 1; p.cin = cin; p.chunks_per_slot = cps;
  p.ldo = (long long)taps * cin; p.slot_stride = (long long)cout * taps * cin;
  const dim3 grid(ceil_div(cin, bn), ceil_div(cout, RB_BM), slots);
  const long long n_op = (long long)cin * g.Rp;
  for (int t = 0; t < taps; ++t) {
    const float* B = XT;
    if (shift[t] != 0) {
      MK_CUDA_CHECK(launch_k(rb_shift_kernel, dim3((unsigned)((n_op + 255) / 256)), dim3(256), 0, st, XT, xs, cin, g.Rp, shift[t]));
      B = xs;
    }
    MK_TRY(encode_tensor_map_2d(&tb, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, B, cin, g.Rp, g.Rp, bn));
    p.out = part + (long long)t * cin;
    MK_CUDA_CHECK((bn == 128 ? launch_gemm<128, true>(ta, tb, p, grid, st) : launch_gemm<64, true>(ta, tb, p, grid, st)));
  }
  const long long n = (long long)cout * cin * taps;
  MK_CUDA_CHECK(launch_k(rb_wfold_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, (const float*)part, slots,
                         p.slot_stride, cout, cin, taps, dw));
  return MK_OK;
}

int relayout(const float* W, int cout, int cin, int taps, int dgrad, float* out, cudaStream_t st) {
  const long long n = (long long)cout * cin * taps;
  MK_CUDA_CHECK(launch_k(rb_weight_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, W, cout, cin, taps, dgrad, out));
  return MK_OK;
}

template <int MODE>
int pack(const Geo& g, const Pack& k, cudaStream_t st) {
  MK_CUDA_CHECK(launch_k(rb_pack_kernel<MODE>, dim3(ceil_div(g.Rp, RB_TILE), k.C / RB_TILE), dim3(32, 8), 0, st, g, k));
  return MK_OK;
}

int stats(const Geo& g, const Stats& s, cudaStream_t st) {
  MK_CUDA_CHECK(launch_k(rb_stats_kernel, dim3(s.C / 32, stat_slots(g)), dim3(32, 8), 0, st, g, s));
  return MK_OK;
}

int fold(int mode, const Fold& f, cudaStream_t st) {
  MK_CUDA_CHECK(launch_k(rb_fold_kernel, dim3(ceil_div(f.C, 128)), dim3(128), 0, st, mode, f));
  return MK_OK;
}

// ---- workspace layouts ----
struct FwdWs {
  // the saved region (what the backward reads), offsets from its base
  size_t z1, z2, a1, a1T, xT, st;   // st: mean1, rstd1, mean2, rstd2 [4][cout]
  size_t saved;
  // the scratch workspace, offsets from its base
  size_t xp, sc, wk1, wk2, wksc, spart;
  size_t total;
};
FwdWs fwd_ws(const Geo& g, int cin, int cout) {
  FwdWs L;
  size_t o = 0;
  const size_t R = g.R, Rp = g.Rp;
  auto put = [&](size_t bytes) { const size_t at = o; o += al256(bytes); return at; };
  L.z1 = put(R * cout * 4); L.z2 = put(R * cout * 4); L.a1 = put(R * cout * 4); L.a1T = put(Rp * cout * 4);
  L.xT = put(Rp * cin * 4); L.st = put(4 * (size_t)cout * 4);
  L.saved = o;
  o = 0;
  L.xp = put(R * cin * 4); L.sc = put(cin != cout ? R * cout * 4 : 0);
  L.wk1 = put((size_t)cout * 9 * cin * 4); L.wk2 = put((size_t)cout * 9 * cout * 4);
  L.wksc = put(cin != cout ? (size_t)cout * cin * 4 : 0);
  L.spart = put(2 * (size_t)stat_slots(g) * cout * 8);
  L.total = o;
  return L;
}

struct BwdWs { size_t gf, gr, grT, dz, dzT, da1, dxc, dxs, wd, wdsc, xs, wpart, spart, coef, total; };
BwdWs bwd_ws(const Geo& g, int cin, int cout) {
  BwdWs L;
  size_t o = 0;
  const size_t R = g.R, Rp = g.Rp;
  const bool sc = cin != cout;
  auto put = [&](size_t bytes) { const size_t at = o; o += al256(bytes); return at; };
  L.gf = put(R * cout * 4);
  L.gr = put(sc ? R * cout * 4 : 0); L.grT = put(sc ? Rp * cout * 4 : 0);
  L.dz = put(R * cout * 4); L.dzT = put(Rp * cout * 4); L.da1 = put(R * cout * 4);
  L.dxc = put(R * cin * 4); L.dxs = put(sc ? R * cin * 4 : 0);
  L.wd = put((size_t)9 * cout * std::max(cin, cout) * 4); L.wdsc = put(sc ? (size_t)cin * cout * 4 : 0);
  L.xs = put(Rp * std::max(cin, cout) * 4);
  size_t wp = 0;
  const int shapes[3][3] = {{cout, cin, 9}, {cout, cout, 9}, {cout, cin, 1}};
  for (int i = 0; i < (sc ? 3 : 2); ++i) {
    int slots, cps;
    wgrad_plan(g, shapes[i][0], shapes[i][1], shapes[i][2], slots, cps);
    wp = std::max(wp, (size_t)slots * shapes[i][0] * shapes[i][1] * shapes[i][2] * 4);
  }
  L.wpart = put(wp);
  L.spart = put(2 * (size_t)stat_slots(g) * cout * 8);
  L.coef = put(3 * (size_t)cout * 4);
  L.total = o;
  return L;
}

bool geometry_ok(int B, int h, int w, int cin, int cout) {
  if (B < 1 || h < 1 || w < 1 || cin < 32 || cout < 32 || cin > RB_MAX_C || cout > RB_MAX_C || cin % 32 || cout % 32) return false;
  return (long long)B * (h + 2) * (w + 2) <= RB_MAX_ROWS;
}

bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

}  // namespace mk

using namespace mk;

static const char* RB_GEOM_MSG = "B, h, w >= 1, B (h+2)(w+2) <= 16777216, channel counts multiples of 32 in [32, 4096]";

long long mk_resblock_ws_bytes(int B, int h, int w, int cin, int cout) {
  if (!geometry_ok(B, h, w, cin, cout)) return -1;
  return (long long)fwd_ws(geo(B, h, w), cin, cout).total;
}

long long mk_resblock_saved_bytes(int B, int h, int w, int cin, int cout) {
  if (!geometry_ok(B, h, w, cin, cout)) return -1;
  return (long long)fwd_ws(geo(B, h, w), cin, cout).saved;
}

long long mk_resblock_backward_ws_bytes(int B, int h, int w, int cin, int cout) {
  if (!geometry_ok(B, h, w, cin, cout)) return -1;
  return (long long)bwd_ws(geo(B, h, w), cin, cout).total;
}

int mk_resblock_layout(int B, int h, int w, int cin, int cout, long long* saved_off, long long* bwd_off) {
  if (!saved_off || !bwd_off || !geometry_ok(B, h, w, cin, cout)) {
    set_last_error("mk_resblock_layout: need two arrays of 6 offsets, %s", RB_GEOM_MSG);
    return MK_ERR_INVALID;
  }
  const Geo g = geo(B, h, w);
  const FwdWs S = fwd_ws(g, cin, cout);
  const BwdWs L = bwd_ws(g, cin, cout);
  const size_t so[6] = {S.z1, S.z2, S.a1, S.a1T, S.xT, S.st}, bo[6] = {L.gf, L.dz, L.dzT, L.da1, L.dxc, L.dxs};
  for (int i = 0; i < 6; ++i) { saved_off[i] = (long long)so[i]; bwd_off[i] = (long long)bo[i]; }
  return MK_OK;
}

int mk_resblock_forward(const float* x, const long long* x_strides, int B, int h, int w, int cin, int cout,
                        const mk_resblock_params* P, int flags, float* out, void* saved, long long saved_bytes, void* ws,
                        long long ws_bytes, void* stream) {
  const bool train = flags & MK_RB_TRAIN, relu = flags & MK_RB_RELU, save = flags & MK_RB_SAVE, bn = flags & MK_RB_BN;
  if (!x || !x_strides || !P || !out || !saved || !ws || !al16(saved) || !al16(ws) || !al16(out) ||
      !geometry_ok(B, h, w, cin, cout)) {
    set_last_error("mk_resblock_forward: need x, its strides, the parameters, out, a 16-byte aligned saved region and workspace, %s "
                   "(got B %d h %d w %d cin %d cout %d)", RB_GEOM_MSG, B, h, w, cin, cout);
    return MK_ERR_INVALID;
  }
  if (flags & ~(MK_RB_TRAIN | MK_RB_RELU | MK_RB_SAVE | MK_RB_BN)) {
    set_last_error("mk_resblock_forward: unknown flag bits 0x%x", flags);
    return MK_ERR_INVALID;
  }
  if (!P->w1 || !P->w2 || (cin != cout) != (P->wsc != nullptr)) {
    set_last_error("mk_resblock_forward: need w1, w2, and wsc exactly when cin != cout");
    return MK_ERR_INVALID;
  }
  if (bn && (!P->bn1_w || !P->bn1_b || !P->bn1_mean || !P->bn1_var || !P->bn2_w || !P->bn2_b || !P->bn2_mean || !P->bn2_var ||
             !(P->eps1 > 0.f) || !(P->eps2 > 0.f))) {
    set_last_error("mk_resblock_forward: batch norm needs weight, bias, running mean and variance of both layers and eps > 0");
    return MK_ERR_INVALID;
  }
  if (bn && train && (long long)B * h * w < 2) {
    set_last_error("mk_resblock_forward: training-mode batch norm needs more than one value per channel (B h w = 1)");
    return MK_ERR_INVALID;
  }
  const Geo g = geo(B, h, w);
  const FwdWs L = fwd_ws(g, cin, cout);
  if (ws_bytes < (long long)L.total || saved_bytes < (long long)L.saved) {
    set_last_error("mk_resblock_forward: saved region of %lld bytes (%lld needed) and workspace of %lld bytes (%lld needed)",
                   saved_bytes, (long long)L.saved, ws_bytes, (long long)L.total);
    return MK_ERR_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* wb = reinterpret_cast<uint8_t*>(ws);
  uint8_t* sb = reinterpret_cast<uint8_t*>(saved);
  auto F = [&](size_t off) { return reinterpret_cast<float*>(wb + off); };
  auto SV = [&](size_t off) { return reinterpret_cast<float*>(sb + off); };
  float *z1 = SV(L.z1), *z2 = SV(L.z2), *a1 = SV(L.a1), *a1T = SV(L.a1T), *xT = SV(L.xT), *xp = F(L.xp), *sc = F(L.sc);
  float *mean1 = SV(L.st), *rstd1 = mean1 + cout, *mean2 = mean1 + 2 * cout, *rstd2 = mean1 + 3 * cout;
  double* spart = reinterpret_cast<double*>(wb + L.spart);
  const Nchw xin{x, x_strides[0], x_strides[1], x_strides[2], x_strides[3]};
  const double count = (double)B * h * w;

  // input: TF32 padded NHWC (+ channel-major for the weight gradients)
  {
    Pack k;
    memset(&k, 0, sizeof(k));
    k.C = cin; k.src = xin; k.o_tf = xp; k.o_cm = save ? xT : nullptr;
    MK_TRY(pack<PK_NCHW>(g, k, st));
  }
  MK_TRY(relayout(P->w1, cout, cin, 9, 0, F(L.wk1), st));
  MK_TRY(relayout(P->w2, cout, cout, 9, 0, F(L.wk2), st));
  if (P->wsc) MK_TRY(relayout(P->wsc, cout, cin, 1, 0, F(L.wksc), st));

  auto bn_stats = [&](const float* Z, const float* gamma, float* mean, float* rstd, float* rm, float* rv, float eps,
                      float mom) -> int {
    Fold f;
    memset(&f, 0, sizeof(f));
    f.C = cout; f.slots = stat_slots(g); f.train = train; f.count = count; f.part = spart; f.eps = eps; f.momentum = mom;
    f.mean = mean; f.rstd = rstd; f.run_mean = rm; f.run_var = rv; f.gamma = gamma;
    if (!train) return fold(FD_EVAL, f, st);
    Stats s;
    memset(&s, 0, sizeof(s));
    s.C = cout; s.rows_per_slot = ceil_div(g.R, f.slots); s.G = Z; s.part = spart;
    MK_TRY(stats(g, s, st));
    MK_TRY(fold(FD_MEAN, f, st));
    s.shift = mean;
    MK_TRY(stats(g, s, st));
    return fold(FD_VAR, f, st);
  };

  // conv1 -> BN1 -> ReLU
  MK_TRY(conv_fwd(g, xp, cin, F(L.wk1), cout, 9, z1, st));
  if (bn) MK_TRY(bn_stats(z1, P->bn1_w, mean1, rstd1, P->bn1_mean, P->bn1_var, P->eps1, P->momentum1));
  {
    Pack k;
    memset(&k, 0, sizeof(k));
    k.C = cout; k.Z = z1; k.bn = bn; k.mean = mean1; k.rstd = rstd1; k.gamma = P->bn1_w; k.beta = P->bn1_b;
    k.o_tf = a1; k.o_cm = save ? a1T : nullptr;
    MK_TRY(pack<PK_BN_FWD>(g, k, st));
  }
  // conv2 -> BN2, shortcut, add, ReLU
  MK_TRY(conv_fwd(g, a1, cout, F(L.wk2), cout, 9, z2, st));
  if (bn) MK_TRY(bn_stats(z2, P->bn2_w, mean2, rstd2, P->bn2_mean, P->bn2_var, P->eps2, P->momentum2));
  if (P->wsc) MK_TRY(conv_fwd(g, xp, cin, F(L.wksc), cout, 1, sc, st));
  Final k;
  memset(&k, 0, sizeof(k));
  k.C = cout; k.bn = bn; k.relu = relu; k.Z = z2; k.mean = mean2; k.rstd = rstd2; k.gamma = P->bn2_w; k.beta = P->bn2_b;
  k.Ssc = P->wsc ? sc : nullptr; k.x = xin; k.out = out;
  MK_CUDA_CHECK(launch_k(rb_final_kernel, dim3(ceil_div(g.R, RB_TILE), cout / RB_TILE), dim3(32, 8), 0, st, g, k));
  return MK_OK;
}

int mk_resblock_backward(const void* saved, const float* grad_out, const long long* g_strides, const float* out, int B, int h,
                         int w, int cin, int cout, const mk_resblock_params* P, int flags, int want,
                         const mk_resblock_grads* G, void* ws, long long ws_bytes, void* stream) {
  const bool train = flags & MK_RB_TRAIN, relu = flags & MK_RB_RELU, bn = flags & MK_RB_BN;
  if (!saved || !grad_out || !g_strides || !P || !G || !ws || !al16(saved) || !al16(ws) || (relu && !out) ||
      !geometry_ok(B, h, w, cin, cout)) {
    set_last_error("mk_resblock_backward: need the forward's saved workspace, grad_out and its strides, out (with ReLU), the "
                   "parameters, the gradient table and a 16-byte aligned workspace, %s (got B %d h %d w %d cin %d cout %d)",
                   RB_GEOM_MSG, B, h, w, cin, cout);
    return MK_ERR_INVALID;
  }
  if ((flags & ~(MK_RB_TRAIN | MK_RB_RELU | MK_RB_SAVE | MK_RB_BN)) || (want & ~0xFF)) {
    set_last_error("mk_resblock_backward: unknown flag bits 0x%x or gradient bits 0x%x", flags, want);
    return MK_ERR_INVALID;
  }
  const bool sc = cin != cout;
  if (!P->w1 || !P->w2 || sc != (P->wsc != nullptr) || (bn && (!P->bn1_w || !P->bn2_w))) {
    set_last_error("mk_resblock_backward: need w1, w2, wsc exactly when cin != cout, and the BN weights with batch norm");
    return MK_ERR_INVALID;
  }
  float* const outs[8] = {G->dx, G->w1, G->w2, G->wsc, G->bn1_w, G->bn1_b, G->bn2_w, G->bn2_b};
  const char* names[8] = {"dx", "w1", "w2", "wsc", "bn1_w", "bn1_b", "bn2_w", "bn2_b"};
  for (int i = 0; i < 8; ++i)
    if ((want >> i & 1) && (!outs[i] || (i == 3 && !sc) || (i >= 4 && !bn))) {
      set_last_error("mk_resblock_backward: gradient %s requested but %s", names[i], !outs[i] ? "its pointer is NULL" : "the block has no such parameter");
      return MK_ERR_INVALID;
    }
  const Geo g = geo(B, h, w);
  const FwdWs S = fwd_ws(g, cin, cout);
  const BwdWs L = bwd_ws(g, cin, cout);
  if (ws_bytes < (long long)L.total) {
    set_last_error("mk_resblock_backward: workspace of %lld bytes, %lld needed", ws_bytes, (long long)L.total);
    return MK_ERR_INVALID;
  }
  if (!want) return MK_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const uint8_t* sv = reinterpret_cast<const uint8_t*>(saved);
  auto SV = [&](size_t off) { return reinterpret_cast<const float*>(sv + off); };
  uint8_t* wb = reinterpret_cast<uint8_t*>(ws);
  auto F = [&](size_t off) { return reinterpret_cast<float*>(wb + off); };
  const float *z1 = SV(S.z1), *z2 = SV(S.z2), *a1 = SV(S.a1), *a1T = SV(S.a1T), *xT = SV(S.xT);
  const float *mean1 = SV(S.st), *rstd1 = mean1 + cout, *mean2 = mean1 + 2 * cout, *rstd2 = mean1 + 3 * cout;
  float *gf = F(L.gf), *gr = F(L.gr), *grT = F(L.grT), *dz = F(L.dz), *dzT = F(L.dzT), *da1 = F(L.da1), *dxc = F(L.dxc),
        *dxs = F(L.dxs), *wd = F(L.wd), *xs = F(L.xs), *wpart = F(L.wpart), *coef = F(L.coef);
  double* spart = reinterpret_cast<double*>(wb + L.spart);
  const bool want_dx = want & MK_RB_GRAD_X;
  const bool below2 = want & (MK_RB_GRAD_X | MK_RB_GRAD_W1 | MK_RB_GRAD_BN1_W | MK_RB_GRAD_BN1_B);
  const bool below_bn2 = below2 || (want & MK_RB_GRAD_W2);
  const double count = (double)B * h * w;

  // 1. g = grad_out * (out > 0): fp32 for BN2 and the identity path, TF32 copies for the shortcut's contractions
  {
    Pack k;
    memset(&k, 0, sizeof(k));
    k.C = cout; k.src = Nchw{grad_out, g_strides[0], g_strides[1], g_strides[2], g_strides[3]};
    if (relu) k.mask = Nchw{out, (long long)cout * h * w, (long long)h * w, (long long)w, 1LL};
    k.o_f32 = gf;
    if (sc && want_dx) k.o_tf = gr;
    if (sc && (want & MK_RB_GRAD_WSC)) k.o_cm = grT;
    MK_TRY(pack<PK_NCHW>(g, k, st));
  }
  // 2. the shortcut's wgrad and dgrad
  if (sc && (want & MK_RB_GRAD_WSC)) MK_TRY(conv_wgrad(g, grT, xT, cout, cin, 1, xs, wpart, G->wsc, st));
  if (sc && want_dx) {
    MK_TRY(relayout(P->wsc, cout, cin, 1, 1, F(L.wdsc), st));
    MK_TRY(conv_fwd(g, gr, cout, F(L.wdsc), cin, 1, dxs, st));
  }
  // BN backward: sums of g and g xhat, then dz = gamma rstd / M (M g - sum g - xhat sum g xhat), TF32 in both layouts
  auto bn_bwd = [&](const float* Gin, const float* Mk, const float* Z, const float* mean, const float* rstd, const float* gamma,
                    float* dgamma, float* dbeta, bool need_nhwc, bool need_cm) -> int {
    Pack k;
    memset(&k, 0, sizeof(k));
    k.C = cout; k.G = Gin; k.Mk = Mk; k.Z = Z; k.bn = bn; k.mean = mean; k.rstd = rstd; k.coef = coef;
    k.o_tf = need_nhwc ? dz : nullptr; k.o_cm = need_cm ? dzT : nullptr;
    if (bn) {
      Stats s;
      memset(&s, 0, sizeof(s));
      s.C = cout; s.rows_per_slot = ceil_div(g.R, stat_slots(g)); s.G = Gin; s.Mk = Mk; s.Zx = Z; s.mean = mean; s.rstd = rstd;
      s.part = spart;
      MK_TRY(stats(g, s, st));
      Fold f;
      memset(&f, 0, sizeof(f));
      f.C = cout; f.slots = stat_slots(g); f.train = train; f.count = count; f.part = spart; f.rstd = const_cast<float*>(rstd);
      f.gamma = gamma; f.dgamma = dgamma; f.dbeta = dbeta; f.coef = coef;
      MK_TRY(fold(FD_BWD, f, st));
    }
    if (!need_nhwc && !need_cm) return MK_OK;
    return pack<PK_BN_BWD>(g, k, st);
  };
  // 3. BN2 backward
  if (below_bn2 || (want & (MK_RB_GRAD_BN2_W | MK_RB_GRAD_BN2_B)))
    MK_TRY(bn_bwd(gf, nullptr, z2, mean2, rstd2, P->bn2_w, (want & MK_RB_GRAD_BN2_W) ? G->bn2_w : nullptr,
                  (want & MK_RB_GRAD_BN2_B) ? G->bn2_b : nullptr, below2, want & MK_RB_GRAD_W2));
  // 4. conv2's wgrad and dgrad
  if (want & MK_RB_GRAD_W2) MK_TRY(conv_wgrad(g, dzT, a1T, cout, cout, 9, xs, wpart, G->w2, st));
  if (below2) {
    MK_TRY(relayout(P->w2, cout, cout, 9, 1, wd, st));
    MK_TRY(conv_fwd(g, dz, cout, wd, cout, 9, da1, st));
    // 5-6. the ReLU1 mask and BN1 backward
    MK_TRY(bn_bwd(da1, a1, z1, mean1, rstd1, P->bn1_w, (want & MK_RB_GRAD_BN1_W) ? G->bn1_w : nullptr,
                  (want & MK_RB_GRAD_BN1_B) ? G->bn1_b : nullptr, want_dx, want & MK_RB_GRAD_W1));
    // 7. conv1's wgrad, and its dgrad only for dX
    if (want & MK_RB_GRAD_W1) MK_TRY(conv_wgrad(g, dzT, xT, cout, cin, 9, xs, wpart, G->w1, st));
    if (want_dx) {
      MK_TRY(relayout(P->w1, cout, cin, 9, 1, wd, st));
      MK_TRY(conv_fwd(g, dz, cout, wd, cin, 9, dxc, st));
    }
  }
  // 8. dX = conv1's data gradient + the shortcut's
  if (want_dx)
    MK_CUDA_CHECK(launch_k(rb_dx_kernel, dim3(ceil_div(g.R, RB_TILE), cin / RB_TILE), dim3(32, 8), 0, st, g, cin,
                           (const float*)dxc, (const float*)(sc ? dxs : gf), G->dx));
  return MK_OK;
}

long long mk_op_conv_tf32_ws_bytes(int mode, int B, int h, int w, int cin, int cout, int taps) {
  if (mode < 0 || mode > 2 || (taps != 1 && taps != 9) || !geometry_ok(B, h, w, cin, cout)) return -1;
  const Geo g = geo(B, h, w);
  if (mode < 2) return (long long)al256((size_t)9 * cin * cout * 4);
  int slots, cps;
  wgrad_plan(g, cout, cin, taps, slots, cps);
  return (long long)(al256((size_t)slots * cout * cin * taps * 4) + al256((size_t)g.Rp * cin * 4));
}

int mk_op_conv_tf32(int mode, const float* a, const float* b, float* out, int B, int h, int w, int cin, int cout, int taps,
                    void* ws, long long ws_bytes, void* stream) {
  const long long need = mk_op_conv_tf32_ws_bytes(mode, B, h, w, cin, cout, taps);
  if (!a || !b || !out || !ws || need < 0 || ws_bytes < need || !al16(a) || !al16(b) || !al16(ws)) {
    set_last_error("mk_op_conv_tf32: need mode 0-2, taps 1 or 9, 16-byte aligned a, b and a workspace of "
                   "mk_op_conv_tf32_ws_bytes bytes, %s (got mode %d B %d h %d w %d cin %d cout %d taps %d ws %lld)",
                   RB_GEOM_MSG, mode, B, h, w, cin, cout, taps, ws_bytes);
    return MK_ERR_INVALID;
  }
  const Geo g = geo(B, h, w);
  cudaStream_t st = (cudaStream_t)stream;
  float* wk = reinterpret_cast<float*>(ws);
  if (mode == 0) {             // out [R, cout] = conv(a [R, cin] padded NHWC, b = W [cout, cin, taps])
    MK_TRY(relayout(b, cout, cin, taps, 0, wk, st));
    return conv_fwd(g, a, cin, wk, cout, taps, out, st);
  }
  if (mode == 1) {             // out [R, cin] = dgrad(a = dZ [R, cout] padded NHWC, b = W [cout, cin, taps])
    MK_TRY(relayout(b, cout, cin, taps, 1, wk, st));
    return conv_fwd(g, a, cout, wk, cin, taps, out, st);
  }
  // out = dW [cout, cin, taps] from a = dZ^T [cout, Rp], b = X^T [cin, Rp]
  int slots, cps;
  wgrad_plan(g, cout, cin, taps, slots, cps);
  float* xs = wk + al256((size_t)slots * cout * cin * taps * 4) / 4;
  return conv_wgrad(g, a, b, cout, cin, taps, xs, wk, out, st);
}
