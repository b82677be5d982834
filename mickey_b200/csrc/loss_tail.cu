// The differentiable tail of MicKey's training loss (reference lib/models/MicKey/modules/loss/loss_class.py:140-152,
// 199-248), forward and backward, for mickey_b200/loss.py's opt-in CUDA tail.  Inputs are mk_loss_search's outputs as
// they are: the drawn cells int32 [B*IM, S] and the inliers_final bit words [B*IM*IR, S/32].
//
// Forward, one block per (pair b, outer iteration) set, one warp per hypothesis h (IR of them):
//   X_i, Y_i   = depth * K^-1 (u, v, 1) of the set's S cells (inv3x3 of ransac_dev.cuh, products in fp64)
//   a, b       = sum w_i X_i / (W1 + 1e-16), sum w_i Y_i / (W1 + 1e-16), W1 = sum |w_i|, w the inlier bits
//   H          = sum (X_i - a) (w_i (Y_i - b))^T;  R = kabsch_rotation(H) (= V Z U^T);  t = b - R a
//   score_h    = sum_i sigmoid(5/th (th - sqrt(|R X_i + t - Y_i|^2 + 1e-6))) over all S entries
//   lv, lr, lt = VCRE (both directions, image axes clipped to [0, 720], tanh(./80) when soft) or POSE_ERR
//                (acos(clip(c, +-0.99999)) + L1 translation, tanh(./0.9) when soft), plus lr, lt in both cases
// then per set the softmax of score / T over the IR hypotheses (with the null hypothesis for loss_value when enabled).
// Every sum runs in fp64 over lane-strided entries and a butterfly, so every lane holds the same bits.
//
// Backward.  Per hypothesis the softmax, tanh, acos / clip (torch's subgradients: clamp passes where min <= x <= max,
// abs / sign give 0 at 0) and the score give G_R = dL/dR, g_t = dL/dt; the rotation needs no SVD: R H is symmetric at
// the optimum, so with P = sym(R H), M = tr(P) I - P, B = G_R R^T and g = (B32 - B23, B13 - B31, B21 - B12),
//     G_H = -R^T [y]x,  y = M^-1 g,
// (M's eigenvalues are l_j + l_k for the singular values l, the last signed by Z).  Then per entry i, summed over the
// set's hypotheses in order h = 0 .. IR-1:
//     dX_i = w_i G_H (Y_i - b) + w_i g_a / (W1 + eps) + c_i R^T r_i,   dY_i = w_i G_H^T (X_i - a) + w_i g_b / (W1 + eps) - c_i r_i
// with r_i = R X_i + t - Y_i, c_i = dL/dscore * dsigmoid/dd / d_i, g_a = -R^T g_t - G_H (eps b), g_b = g_t - G_H^T (eps a)
// (eps = 1e-16: sum w_i (Y_i - b) = eps b exactly), and through the back-projection to (u, v, depth).
// Finally each keypoint sums the contributions of the (outer iteration, entry) pairs that drew it in ascending order,
// one thread per keypoint: no float atomics, so the gradients are the same bits on every run.
#include <cfloat>

#include "../../include/mickey_b200.h"
#include "ops.h"
#include "ransac_dev.cuh"

namespace mk {

namespace {

constexpr int TAIL_THREADS = 256;
constexpr int TAIL_WARPS = TAIL_THREADS / 32;
constexpr int SCATTER_THREADS = 256, SCATTER_TILE = 2048;
constexpr double TAIL_EPS = 1e-16;
constexpr double VCRE_H = 720.0;        // vcre_loss(H=720): both image axes are clipped to [0, 720]

// the forward's saved state per hypothesis (doubles)
enum : int { HR = 0, HT = 9, HA = 12, HB = 15, HH = 18, HW1 = 27, HSC = 28, HLV = 29, HLR = 30, HLT = 31, HQ = 32, HSM = 33,
             HYP_STRIDE = 34 };
// per set: loss_value, loss_rot, loss_trans
constexpr int SET_STRIDE = 4;
// the backward's per-hypothesis coefficients: G_H, g_a / (W1 + eps), g_b / (W1 + eps), -5/th dL/dscore
enum : int { CGH = 0, CGA = 9, CGB = 12, CGS = 15, COEF_STRIDE = 16 };

struct TailArgs {
  const int* sampled; const uint32_t* bits;
  const float *kps0, *d0, *kps1, *d1, *K0, *K1, *Kori0, *Kori1, *T, *grid;
  int B, N, IM, IR, S;
  int loss_type, soft, null_hyp;
  double th, temperature, null_score, null_loss;
};

struct TailWs { double* hyp; double* set; double* coef; double* contrib; };

inline size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }

TailWs carve_tail(void* ws, int B, int IM, int IR, int S) {
  const size_t sets = (size_t)B * IM, hyps = sets * IR;
  uint8_t* p = reinterpret_cast<uint8_t*>(ws);
  TailWs w;
  w.hyp = reinterpret_cast<double*>(p);                   p += align256(hyps * HYP_STRIDE * sizeof(double));
  w.set = reinterpret_cast<double*>(p);                   p += align256(sets * SET_STRIDE * sizeof(double));
  w.coef = reinterpret_cast<double*>(p);                  p += align256(hyps * COEF_STRIDE * sizeof(double));
  w.contrib = reinterpret_cast<double*>(p);
  return w;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ double sigmoid(double x) { return 1.0 / (1.0 + exp(-x)); }

__device__ __forceinline__ bool inlier(const uint32_t* wb, int i) { return (wb[i >> 5] >> (i & 31)) & 1u; }

// The set's X / Y [3][S] in shared memory, and the fp32 K^-1 of both images (as the search's gather_set computes them).
__device__ void load_set(const TailArgs& A, int s, int b, double* X, double* Y, float* Ki0, float* Ki1) {
  if (threadIdx.x == 0) { inv3x3(A.K0 + b * 9, Ki0); inv3x3(A.K1 + b * 9, Ki1); }
  __syncthreads();
  const int N = A.N;
  for (int i = threadIdx.x; i < A.S; i += blockDim.x) {
    const int cell = A.sampled[(long long)s * A.S + i];
    const int i0 = cell / N, i1 = cell - i0 * N;
    const double u0 = A.kps0[((long long)b * 2 + 0) * N + i0], v0 = A.kps0[((long long)b * 2 + 1) * N + i0];
    const double u1 = A.kps1[((long long)b * 2 + 0) * N + i1], v1 = A.kps1[((long long)b * 2 + 1) * N + i1];
    const double z0 = A.d0[(long long)b * N + i0], z1 = A.d1[(long long)b * N + i1];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      X[r * A.S + i] = z0 * ((double)Ki0[r * 3] * u0 + (double)Ki0[r * 3 + 1] * v0 + (double)Ki0[r * 3 + 2]);
      Y[r * A.S + i] = z1 * ((double)Ki1[r * 3] * u1 + (double)Ki1[r * 3 + 1] * v1 + (double)Ki1[r * 3 + 2]);
    }
  }
  __syncthreads();
}

__device__ __forceinline__ void ground_truth(const TailArgs& A, int b, double Rgt[9], double tgt[3]) {
  const float* T = A.T + (long long)b * 16;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int j = 0; j < 3; ++j) Rgt[i * 3 + j] = T[i * 4 + j];
    tgt[i] = T[i * 4 + 3];
  }
}

__device__ __forceinline__ void load_k(const float* K, double k[9]) {
#pragma unroll
  for (int i = 0; i < 9; ++i) k[i] = K[i];
}

__device__ __forceinline__ void matvec(const double M[9], const double x[3], double y[3]) {
#pragma unroll
  for (int i = 0; i < 3; ++i) y[i] = M[i * 3] * x[0] + M[i * 3 + 1] * x[1] + M[i * 3 + 2] * x[2];
}

__device__ __forceinline__ void matTvec(const double M[9], const double x[3], double y[3]) {
#pragma unroll
  for (int i = 0; i < 3; ++i) y[i] = M[i] * x[0] + M[3 + i] * x[1] + M[6 + i] * x[2];
}

__device__ __forceinline__ double clip(double x, double lo, double hi) { return fmin(fmax(x, lo), hi); }

// One virtual point's projection distance |clip(uv_gt) - clip(uv_pred)| with pred = proj(K res), and (when grad) the
// gradient of g * distance with respect to res.
__device__ __forceinline__ double vcre_point(const double K[9], const double e[3], const double res[3], double g, double gres[3]) {
  double xg[3], x[3];
  matvec(K, e, xg);
  matvec(K, res, x);
  const double zg = xg[2] + 1e-16, z = x[2] + 1e-16;
  const double ug[2] = {xg[0] / zg, xg[1] / zg}, up[2] = {x[0] / z, x[1] / z};
  const double df[2] = {clip(ug[0], 0.0, VCRE_H) - clip(up[0], 0.0, VCRE_H), clip(ug[1], 0.0, VCRE_H) - clip(up[1], 0.0, VCRE_H)};
  const double v = sqrt(df[0] * df[0] + df[1] * df[1] + 1e-6);
  if (gres) {
    double gu[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) gu[j] = (up[j] >= 0.0 && up[j] <= VCRE_H) ? -g * df[j] / v : 0.0;
    const double gx[3] = {gu[0] / z, gu[1] / z, -(gu[0] * x[0] + gu[1] * x[1]) / (z * z)};
    matTvec(K, gx, gres);
  }
  return v;
}

// Per hypothesis: the VCRE sum over this lane's virtual points of both directions (forward), or their contribution to
// G_R / g_t with weight g per point distance (backward, gR / gt non-NULL).
__device__ double vcre_lane(const TailArgs& A, const double R[9], const double t[3], const double Rgt[9], const double tgt[3],
                            const double Ko0[9], const double Ko1[9], int lane, double g, double* gR, double* gt) {
  double acc = 0.0;
  for (int k = lane; k < MK_VCRE_POINTS; k += 32) {
    const double e[3] = {A.grid[k * 3], A.grid[k * 3 + 1], A.grid[k * 3 + 2]};
    // image 0: res = Rgt^T (R e + t - tgt)
    double p[3], res[3], gres[3];
    matvec(R, e, p);
#pragma unroll
    for (int i = 0; i < 3; ++i) p[i] += t[i] - tgt[i];
    matTvec(Rgt, p, res);
    acc += vcre_point(Ko0, e, res, g, gR ? gres : nullptr);
    if (gR) {
      double gp[3];
      matvec(Rgt, gres, gp);
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        gt[i] += gp[i];
#pragma unroll
        for (int j = 0; j < 3; ++j) gR[i * 3 + j] += gp[i] * e[j];
      }
    }
    // image 1, the inverse poses: res = Rgt R^T (e - t) + Rgt Rgt^T tgt (T_0to1 is fp32, so Rgt is orthogonal to ~1e-7
    // only, and the reference's inverse keeps the product)
    const double q[3] = {e[0] - t[0], e[1] - t[1], e[2] - t[2]};
    double pp[3], rt[3], rrt[3];
    matTvec(R, q, pp);
    matvec(Rgt, pp, res);
    matTvec(Rgt, tgt, rt);
    matvec(Rgt, rt, rrt);
#pragma unroll
    for (int i = 0; i < 3; ++i) res[i] += rrt[i];
    acc += vcre_point(Ko1, e, res, g, gR ? gres : nullptr);
    if (gR) {
      double gpp[3], gq[3];
      matTvec(Rgt, gres, gpp);
      matvec(R, gpp, gq);
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        gt[i] -= gq[i];
#pragma unroll
        for (int j = 0; j < 3; ++j) gR[i * 3 + j] += q[i] * gpp[j];
      }
    }
  }
  return acc;
}

__device__ __forceinline__ double rot_cos(const double R[9], const double Rgt[9]) {
  double tr = 0.0;
#pragma unroll
  for (int i = 0; i < 9; ++i) tr += R[i] * Rgt[i];
  return (tr - 1.0) / 2.0;
}

constexpr double ACOS_CLIP = 0.99999;

__global__ void __launch_bounds__(TAIL_THREADS)
loss_tail_fwd_kernel(TailArgs A, TailWs W, float* __restrict__ loss_value, float* __restrict__ loss_rot,
                     float* __restrict__ loss_trans, int* __restrict__ status) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ double shm[];
  double* X = shm;
  double* Y = shm + 3 * A.S;
  __shared__ float Ki0[9], Ki1[9];
  const int s = blockIdx.x, b = s / A.IM, S = A.S, words = S / 32;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  load_set(A, s, b, X, Y, Ki0, Ki1);
  double Rgt[9], tgt[3], Ko0[9], Ko1[9];
  ground_truth(A, b, Rgt, tgt);
  load_k(A.Kori0 + b * 9, Ko0);
  load_k(A.Kori1 + b * 9, Ko1);
  const double k5 = 5.0 / A.th;

  for (int h = warp; h < A.IR; h += TAIL_WARPS) {
    const long long gh = (long long)s * A.IR + h;
    const uint32_t* wb = A.bits + gh * words;
    // weighted means: w * X as a product, so a NaN or inf anywhere in the set reaches R and t as it does in torch
    double m[7] = {0, 0, 0, 0, 0, 0, 0};
    for (int i = lane; i < S; i += 32) {
      const double w = inlier(wb, i) ? 1.0 : 0.0;
      m[0] += w;
#pragma unroll
      for (int r = 0; r < 3; ++r) { m[1 + r] += w * X[r * S + i]; m[4 + r] += w * Y[r * S + i]; }
    }
#pragma unroll
    for (int q = 0; q < 7; ++q) m[q] = warp_sum(m[q]);
    const double W1 = m[0], wn = 1.0 / (W1 + TAIL_EPS);
    const double a[3] = {m[1] * wn, m[2] * wn, m[3] * wn}, bm[3] = {m[4] * wn, m[5] * wn, m[6] * wn};
    double H[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = lane; i < S; i += 32) {
      const double w = inlier(wb, i) ? 1.0 : 0.0;
      const double xa[3] = {X[i] - a[0], X[S + i] - a[1], X[2 * S + i] - a[2]};
      const double yb[3] = {w * (Y[i] - bm[0]), w * (Y[S + i] - bm[1]), w * (Y[2 * S + i] - bm[2])};
#pragma unroll
      for (int p = 0; p < 3; ++p)
#pragma unroll
        for (int q = 0; q < 3; ++q) H[p * 3 + q] += xa[p] * yb[q];
    }
#pragma unroll
    for (int q = 0; q < 9; ++q) H[q] = warp_sum(H[q]);
    double R[9], t[3];
    kabsch_rotation(H, R);
    double Ra[3];
    matvec(R, a, Ra);
    bool finite = true;
#pragma unroll
    for (int i = 0; i < 3; ++i) { t[i] = bm[i] - Ra[i]; finite = finite && fabs(t[i]) <= DBL_MAX; }
#pragma unroll
    for (int i = 0; i < 9; ++i) finite = finite && fabs(R[i]) <= DBL_MAX;
    if (!finite && lane == 0) atomicOr(status, MK_LOSS_TAIL_STATUS_NONFINITE);
    // soft inlier count over all S entries (training_utils.py:55-61)
    double sc = 0.0;
    for (int i = lane; i < S; i += 32) {
      const double x[3] = {X[i], X[S + i], X[2 * S + i]};
      double r[3];
      matvec(R, x, r);
      r[0] += t[0] - Y[i]; r[1] += t[1] - Y[S + i]; r[2] += t[2] - Y[2 * S + i];
      const double d = sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + 1e-6);
      sc += sigmoid(k5 * (A.th - d));
    }
    sc = warp_sum(sc);
    // rotation and translation errors (loss_utils.py:85-110), and the loss
    const double lr = fabs(acos(clip(rot_cos(R, Rgt), -ACOS_CLIP, ACOS_CLIP)));
    const double lt = fabs(t[0] - tgt[0]) + fabs(t[1] - tgt[1]) + fabs(t[2] - tgt[2]);
    double lv;
    if (A.loss_type == 0) {
      const double raw = warp_sum(vcre_lane(A, R, t, Rgt, tgt, Ko0, Ko1, lane, 0.0, nullptr, nullptr)) / (2.0 * MK_VCRE_POINTS);
      lv = A.soft ? tanh(raw / 80.0) : raw;
    } else {
      lv = A.soft ? tanh(lr / 0.9) + tanh(lt / 0.9) : lr + lt;
    }
    if (lane == 0) {
      double* o = W.hyp + gh * HYP_STRIDE;
      for (int i = 0; i < 9; ++i) { o[HR + i] = R[i]; o[HH + i] = H[i]; }
      for (int i = 0; i < 3; ++i) { o[HT + i] = t[i]; o[HA + i] = a[i]; o[HB + i] = bm[i]; }
      o[HW1] = W1; o[HSC] = sc; o[HLV] = lv; o[HLR] = lr; o[HLT] = lt;
    }
  }
  __syncthreads();
  // the set's softmaxes (:238-248): warp 0, hypotheses in lane-strided order, butterflies
  if (warp == 0) {
    double* hyp = W.hyp + (long long)s * A.IR * HYP_STRIDE;
    const double iT = 1.0 / A.temperature;
    double mx = -INFINITY;
    for (int h = lane; h < A.IR; h += 32) mx = fmax(mx, hyp[h * HYP_STRIDE + HSC] * iT);
    mx = warp_max(mx);
    const double mxn = A.null_hyp ? fmax(mx, A.null_score * iT) : mx;
    double z = 0.0, zn = 0.0;
    for (int h = lane; h < A.IR; h += 32) {
      z += exp(hyp[h * HYP_STRIDE + HSC] * iT - mx);
      zn += exp(hyp[h * HYP_STRIDE + HSC] * iT - mxn);
    }
    z = warp_sum(z);
    zn = warp_sum(zn);
    const double en = A.null_hyp ? exp(A.null_score * iT - mxn) : 0.0;
    zn += en;
    double lv = 0.0, lr = 0.0, lt = 0.0;
    for (int h = lane; h < A.IR; h += 32) {
      double* o = hyp + h * HYP_STRIDE;
      const double sm = exp(o[HSC] * iT - mx) / z, q = exp(o[HSC] * iT - mxn) / zn;
      o[HSM] = sm; o[HQ] = q;
      lv += q * o[HLV]; lr += sm * o[HLR]; lt += sm * o[HLT];
    }
    lv = warp_sum(lv) + (en / zn) * A.null_loss;
    lr = warp_sum(lr);
    lt = warp_sum(lt);
    if (lane == 0) {
      double* o = W.set + (long long)s * SET_STRIDE;
      o[0] = lv; o[1] = lr; o[2] = lt;
      loss_value[s] = (float)lv; loss_rot[s] = (float)lr; loss_trans[s] = (float)lt;
    }
  }
}

// G_H = -R^T [M^-1 g]x  (the header comment of this file)
__device__ void rotation_backward(const double R[9], const double H[9], const double GR[9], double GH[9]) {
  double RH[9];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) RH[i * 3 + j] = R[i * 3] * H[j] + R[i * 3 + 1] * H[3 + j] + R[i * 3 + 2] * H[6 + j];
  double P[9];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) P[i * 3 + j] = 0.5 * (RH[i * 3 + j] + RH[j * 3 + i]);
  const double tr = P[0] + P[4] + P[8];
  double M[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) M[i] = ((i % 4 == 0) ? tr : 0.0) - P[i];
  double Bm[9];     // G_R R^T
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) Bm[i * 3 + j] = GR[i * 3] * R[j * 3] + GR[i * 3 + 1] * R[j * 3 + 1] + GR[i * 3 + 2] * R[j * 3 + 2];
  const double g[3] = {Bm[7] - Bm[5], Bm[2] - Bm[6], Bm[3] - Bm[1]};
  // M symmetric: y = adj(M) g / det(M)
  const double c00 = M[4] * M[8] - M[5] * M[7], c01 = M[5] * M[6] - M[3] * M[8], c02 = M[3] * M[7] - M[4] * M[6];
  const double c11 = M[0] * M[8] - M[2] * M[6], c12 = M[2] * M[3] - M[0] * M[5], c22 = M[0] * M[4] - M[1] * M[3];
  const double det = M[0] * c00 + M[1] * c01 + M[2] * c02;
  const double y[3] = {(c00 * g[0] + c01 * g[1] + c02 * g[2]) / det, (c01 * g[0] + c11 * g[1] + c12 * g[2]) / det,
                       (c02 * g[0] + c12 * g[1] + c22 * g[2]) / det};
  const double Y[9] = {0, -y[2], y[1], y[2], 0, -y[0], -y[1], y[0], 0};
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) GH[i * 3 + j] = -(R[i] * Y[j] + R[3 + i] * Y[3 + j] + R[6 + i] * Y[6 + j]);
}

__global__ void __launch_bounds__(TAIL_THREADS)
loss_tail_bwd_kernel(TailArgs A, TailWs W, const float* __restrict__ g_lv, const float* __restrict__ g_lr,
                     const float* __restrict__ g_lt) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ double shm[];
  double* X = shm;
  double* Y = shm + 3 * A.S;
  __shared__ float Ki0[9], Ki1[9];
  const int s = blockIdx.x, b = s / A.IM, S = A.S, words = S / 32;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  load_set(A, s, b, X, Y, Ki0, Ki1);
  double Rgt[9], tgt[3], Ko0[9], Ko1[9];
  ground_truth(A, b, Rgt, tgt);
  load_k(A.Kori0 + b * 9, Ko0);
  load_k(A.Kori1 + b * 9, Ko1);
  const double k5 = 5.0 / A.th, iT = 1.0 / A.temperature;
  const double* set = W.set + (long long)s * SET_STRIDE;
  const double gv = g_lv[s], gr = g_lr[s], gtr = g_lt[s];

  // ---- per hypothesis: dL/dscore, G_R, g_t, then G_H, g_a, g_b
  for (int h = warp; h < A.IR; h += TAIL_WARPS) {
    const long long gh = (long long)s * A.IR + h;
    const double* o = W.hyp + gh * HYP_STRIDE;
    double R[9], t[3], H[9], a[3], bm[3];
#pragma unroll
    for (int i = 0; i < 9; ++i) { R[i] = o[HR + i]; H[i] = o[HH + i]; }
#pragma unroll
    for (int i = 0; i < 3; ++i) { t[i] = o[HT + i]; a[i] = o[HA + i]; bm[i] = o[HB + i]; }
    const double q = o[HQ], sm = o[HSM], lv = o[HLV], lr = o[HLR], lt = o[HLT];
    // softmaxes: loss_value over IR (+ null), loss_rot / loss_trans over IR
    const double gs = (gv * q * (lv - set[0]) + gr * sm * (lr - set[1]) + gtr * sm * (lt - set[2])) * iT;
    double dlv = gv * q, dlr = gr * sm, dlt = gtr * sm;
    double GR[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, gt[3] = {0, 0, 0};
    if (A.loss_type == 0) {
      const double graw = dlv * (A.soft ? (1.0 - lv * lv) / 80.0 : 1.0);
      vcre_lane(A, R, t, Rgt, tgt, Ko0, Ko1, lane, graw / (2.0 * MK_VCRE_POINTS), GR, gt);
    } else if (A.soft) {
      const double tr_ = tanh(lr / 0.9), tt_ = tanh(lt / 0.9);
      dlr += dlv * (1.0 - tr_ * tr_) / 0.9;
      dlt += dlv * (1.0 - tt_ * tt_) / 0.9;
    } else {
      dlr += dlv;
      dlt += dlv;
    }
    // the score's path through R and t (its direct path through X, Y is taken per entry below)
    const double cs = -k5 * gs;
    for (int i = lane; i < S; i += 32) {
      const double x[3] = {X[i], X[S + i], X[2 * S + i]};
      double r[3];
      matvec(R, x, r);
      r[0] += t[0] - Y[i]; r[1] += t[1] - Y[S + i]; r[2] += t[2] - Y[2 * S + i];
      const double d = sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + 1e-6);
      const double sg = sigmoid(k5 * (A.th - d));
      const double c = cs * sg * (1.0 - sg) / d;
#pragma unroll
      for (int p = 0; p < 3; ++p) {
        gt[p] += c * r[p];
#pragma unroll
        for (int j = 0; j < 3; ++j) GR[p * 3 + j] += c * r[p] * x[j];
      }
    }
#pragma unroll
    for (int i = 0; i < 9; ++i) GR[i] = warp_sum(GR[i]);
#pragma unroll
    for (int i = 0; i < 3; ++i) gt[i] = warp_sum(gt[i]);
    // rotation and translation errors: clamp passes the gradient on [-0.99999, 0.99999] only, acos' = -1/sqrt(1-c^2),
    // abs' = sign (acos of a clipped cosine is > 0); the L1 term's sign is 0 at 0
    const double c = rot_cos(R, Rgt);
    if (c >= -ACOS_CLIP && c <= ACOS_CLIP) {
      const double f = dlr * (-1.0 / sqrt(1.0 - c * c)) * 0.5;
#pragma unroll
      for (int i = 0; i < 9; ++i) GR[i] += f * Rgt[i];
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const double dt = t[i] - tgt[i];
      gt[i] += dlt * (dt > 0.0 ? 1.0 : dt < 0.0 ? -1.0 : 0.0);
    }
    // t = b - R a also moves with R
#pragma unroll
    for (int p = 0; p < 3; ++p)
#pragma unroll
      for (int j = 0; j < 3; ++j) GR[p * 3 + j] -= gt[p] * a[j];
    double GH[9];
    rotation_backward(R, H, GR, GH);
    // t = b - R a;  H's own dependence on the means: sum w_i (Y_i - b) = eps b, sum w_i (X_i - a) = eps a
    double RtG[3], GHb[3], GHta[3];
    matTvec(R, gt, RtG);
    const double eb[3] = {TAIL_EPS * bm[0], TAIL_EPS * bm[1], TAIL_EPS * bm[2]};
    const double ea[3] = {TAIL_EPS * a[0], TAIL_EPS * a[1], TAIL_EPS * a[2]};
    matvec(GH, eb, GHb);
    matTvec(GH, ea, GHta);
    if (lane == 0) {
      const double wn = 1.0 / (o[HW1] + TAIL_EPS);
      double* cf = W.coef + gh * COEF_STRIDE;
      for (int i = 0; i < 9; ++i) cf[CGH + i] = GH[i];
      for (int i = 0; i < 3; ++i) { cf[CGA + i] = (-RtG[i] - GHb[i]) * wn; cf[CGB + i] = (gt[i] - GHta[i]) * wn; }
      cf[CGS] = cs;
    }
  }
  __syncthreads();

  // ---- per entry: the sum over the set's hypotheses in order, then the back-projection
  for (int i = threadIdx.x; i < S; i += TAIL_THREADS) {
    const double x[3] = {X[i], X[S + i], X[2 * S + i]}, y[3] = {Y[i], Y[S + i], Y[2 * S + i]};
    double dX[3] = {0, 0, 0}, dY[3] = {0, 0, 0};
    for (int h = 0; h < A.IR; ++h) {
      const long long gh = (long long)s * A.IR + h;
      const double* o = W.hyp + gh * HYP_STRIDE;
      const double* cf = W.coef + gh * COEF_STRIDE;
      const double* R = o + HR;
      double r[3];
      matvec(R, x, r);
#pragma unroll
      for (int p = 0; p < 3; ++p) r[p] += o[HT + p] - y[p];
      const double d = sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + 1e-6);
      const double sg = sigmoid(k5 * (A.th - d));
      const double c = cf[CGS] * sg * (1.0 - sg) / d;
      double Rtr[3];
      matTvec(R, r, Rtr);
#pragma unroll
      for (int p = 0; p < 3; ++p) { dX[p] += c * Rtr[p]; dY[p] -= c * r[p]; }
      if (inlier(A.bits + gh * words, i)) {
        const double yb[3] = {y[0] - o[HB], y[1] - o[HB + 1], y[2] - o[HB + 2]};
        const double xa[3] = {x[0] - o[HA], x[1] - o[HA + 1], x[2] - o[HA + 2]};
        double u[3], v[3];
        matvec(cf + CGH, yb, u);
        matTvec(cf + CGH, xa, v);
#pragma unroll
        for (int p = 0; p < 3; ++p) { dX[p] += u[p] + cf[CGA + p]; dY[p] += v[p] + cf[CGB + p]; }
      }
    }
    // X = z K^-1 (u, v, 1): du = z dX . Ki[:,0], dv = z dX . Ki[:,1], dz = dX . Ki (u, v, 1)
    const int cell = A.sampled[(long long)s * S + i];
    const int i0 = cell / A.N, i1 = cell - i0 * A.N;
    double* out = W.contrib + ((long long)s * S + i) * 6;
#pragma unroll
    for (int img = 0; img < 2; ++img) {
      const float* Ki = img ? Ki1 : Ki0;
      const double* g = img ? dY : dX;
      const int n = img ? i1 : i0;
      const float* kps = img ? A.kps1 : A.kps0;
      const double z = (img ? A.d1 : A.d0)[(long long)b * A.N + n];
      const double u = kps[((long long)b * 2 + 0) * A.N + n], v = kps[((long long)b * 2 + 1) * A.N + n];
      double gu = 0.0, gvv = 0.0, gz = 0.0;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        gu += g[r] * (double)Ki[r * 3];
        gvv += g[r] * (double)Ki[r * 3 + 1];
        gz += g[r] * ((double)Ki[r * 3] * u + (double)Ki[r * 3 + 1] * v + (double)Ki[r * 3 + 2]);
      }
      out[img * 3 + 0] = z * gu; out[img * 3 + 1] = z * gvv; out[img * 3 + 2] = gz;
    }
  }
}

// One thread per keypoint n of pair b = blockIdx.y: the sum of the contributions of every (outer iteration, entry) of the
// pair that drew n, in ascending order, written for every keypoint (0 where none drew it).
__global__ void __launch_bounds__(SCATTER_THREADS)
loss_tail_scatter_kernel(const int* __restrict__ sampled, const double* __restrict__ contrib, int N, int IM, int S,
                         float* __restrict__ dkps0, float* __restrict__ dkps1, float* __restrict__ dd0,
                         float* __restrict__ dd1) {
  pdl_wait();
  pdl_trigger();
  __shared__ int k0[SCATTER_TILE], k1[SCATTER_TILE];
  const int b = blockIdx.y, n = blockIdx.x * SCATTER_THREADS + threadIdx.x;
  const long long base = (long long)b * IM * S, total = (long long)IM * S;
  double acc[6] = {0, 0, 0, 0, 0, 0};
  for (long long j0 = 0; j0 < total; j0 += SCATTER_TILE) {
    const int len = (int)min((long long)SCATTER_TILE, total - j0);
    __syncthreads();
    for (int j = threadIdx.x; j < len; j += SCATTER_THREADS) {
      const int cell = sampled[base + j0 + j];
      k0[j] = cell / N;
      k1[j] = cell - (cell / N) * N;
    }
    __syncthreads();
    if (n < N)
      for (int j = 0; j < len; ++j) {
        const bool h0 = k0[j] == n, h1 = k1[j] == n;
        if (h0 | h1) {
          const double* c = contrib + (base + j0 + j) * 6;
          if (h0) { acc[0] += c[0]; acc[1] += c[1]; acc[2] += c[2]; }
          if (h1) { acc[3] += c[3]; acc[4] += c[4]; acc[5] += c[5]; }
        }
      }
  }
  if (n >= N) return;
  dkps0[((long long)b * 2 + 0) * N + n] = (float)acc[0];
  dkps0[((long long)b * 2 + 1) * N + n] = (float)acc[1];
  dd0[(long long)b * N + n] = (float)acc[2];
  dkps1[((long long)b * 2 + 0) * N + n] = (float)acc[3];
  dkps1[((long long)b * 2 + 1) * N + n] = (float)acc[4];
  dd1[(long long)b * N + n] = (float)acc[5];
}

constexpr int TAIL_MAX_GRID_Y = 65535;

// every size and parameter of both calls; the message names the entry point
int tail_check(const char* what, int B, int N, int IM, int IR, int S, int loss_type, float th, float temperature) {
  const long long sets = (long long)B * IM;
  if (B < 1 || B > TAIL_MAX_GRID_Y || N < 1 || (long long)N * N > 0x7fffffffLL || IM < 1 || IR < 1 || S < 32 ||
      S > LOSS_MAX_S || S % 32 || sets > 0x7fffffffLL || sets * IR > 0x7fffffffLL || (loss_type != 0 && loss_type != 1) ||
      !(th > 0.f && th <= FLT_MAX) || !(fabsf(temperature) > 0.f && fabsf(temperature) <= FLT_MAX)) {
    set_last_error("%s: need 1 <= B <= %d, N >= 1 with N*N < 2^31, IM >= 1, IR >= 1, B*IM*IR < 2^31, S a multiple of 32 "
                   "up to %d, loss_type 0 (VCRE) or 1 (POSE_ERR), a finite positive inlier threshold and a finite non-zero "
                   "temperature (got B %d N %d IM %d IR %d S %d loss_type %d th %g temperature %g)", what, TAIL_MAX_GRID_Y,
                   LOSS_MAX_S, B, N, IM, IR, S, loss_type, (double)th, (double)temperature);
    return MK_ERR_INVALID;
  }
  return MK_OK;
}

int tail_configure() {
  static unsigned long long configured = 0;
  if (first_use_on_device(configured)) {
    MK_CUDA_CHECK(cudaFuncSetAttribute(loss_tail_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       6 * LOSS_MAX_S * (int)sizeof(double)));
    MK_CUDA_CHECK(cudaFuncSetAttribute(loss_tail_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       6 * LOSS_MAX_S * (int)sizeof(double)));
  }
  return MK_OK;
}

}  // namespace

long long loss_tail_ws_bytes(int B, int N, int IM, int IR, int S) {
  if (tail_check("mk_loss_tail_ws_bytes", B, N, IM, IR, S, 0, 1.f, 1.f) != MK_OK) return -1;
  const size_t sets = (size_t)B * IM, hyps = sets * IR;
  return (long long)(align256(hyps * HYP_STRIDE * sizeof(double)) + align256(sets * SET_STRIDE * sizeof(double)) +
                     align256(hyps * COEF_STRIDE * sizeof(double)) + sets * S * 6 * sizeof(double));
}

}  // namespace mk

using namespace mk;

namespace {

// the pointers both calls read, NULL-checked together
bool tail_inputs_ok(const int* sampled, const unsigned int* bits, const float* kps0, const float* d0, const float* kps1,
                    const float* d1, const float* K0, const float* K1, const float* Kori0, const float* Kori1, const float* T,
                    const float* grid, const void* ws) {
  return sampled && bits && kps0 && d0 && kps1 && d1 && K0 && K1 && Kori0 && Kori1 && T && grid && ws;
}

TailArgs tail_args(const int* sampled, const unsigned int* bits, const float* kps0, const float* d0, const float* kps1,
                   const float* d1, const float* K0, const float* K1, const float* Kori0, const float* Kori1, const float* T,
                   const float* grid, int B, int N, int IM, int IR, int S, int loss_type, int soft, int null_hyp, float th,
                   float temperature, float null_score, float null_loss) {
  return TailArgs{sampled, reinterpret_cast<const uint32_t*>(bits), kps0, d0, kps1, d1, K0, K1, Kori0, Kori1, T, grid,
                  B, N, IM, IR, S, loss_type, soft ? 1 : 0, null_hyp ? 1 : 0, (double)th, (double)temperature,
                  (double)null_score, (double)null_loss};
}

}  // namespace

extern "C" long long mk_loss_tail_ws_bytes(int B, int N, int it_matches, int it_ransac, int n_sample) {
  return loss_tail_ws_bytes(B, N, it_matches, it_ransac, n_sample);
}

extern "C" int mk_loss_tail_forward(const int* sampled_idx_dev, const unsigned int* inliers_dev, const float* kps0_dev,
                                    const float* depth0_dev, const float* kps1_dev, const float* depth1_dev,
                                    const float* K0_dev, const float* K1_dev, const float* Kori0_dev, const float* Kori1_dev,
                                    const float* T_0to1_dev, const float* grid_dev, int B, int N, int it_matches,
                                    int it_ransac, int n_sample, int loss_type, int soft_clipping, int null_hypothesis,
                                    float inlier_3d_th, float score_temperature, float null_score, float null_loss,
                                    float* loss_value_dev, float* loss_rot_dev, float* loss_trans_dev, int* status_dev,
                                    void* ws_dev, long long ws_bytes, void* stream) {
  if (!tail_inputs_ok(sampled_idx_dev, inliers_dev, kps0_dev, depth0_dev, kps1_dev, depth1_dev, K0_dev, K1_dev, Kori0_dev,
                      Kori1_dev, T_0to1_dev, grid_dev, ws_dev) || !loss_value_dev || !loss_rot_dev || !loss_trans_dev ||
      !status_dev) {
    set_last_error("mk_loss_tail_forward: every input, output, the status word and the workspace must be non-NULL");
    return MK_ERR_INVALID;
  }
  MK_TRY(tail_check("mk_loss_tail_forward", B, N, it_matches, it_ransac, n_sample, loss_type, inlier_3d_th, score_temperature));
  if (null_hypothesis && !(fabsf(null_score) <= FLT_MAX && fabsf(null_loss) <= FLT_MAX)) {
    set_last_error("mk_loss_tail_forward: the null hypothesis needs a finite score and loss (got %g, %g)", (double)null_score,
                   (double)null_loss);
    return MK_ERR_INVALID;
  }
  const long long need = loss_tail_ws_bytes(B, N, it_matches, it_ransac, n_sample);
  if (ws_bytes < need) {
    set_last_error("mk_loss_tail_forward: workspace of %lld bytes, %lld needed", ws_bytes, need);
    return MK_ERR_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  MK_TRY(tail_configure());
  const TailArgs A = tail_args(sampled_idx_dev, inliers_dev, kps0_dev, depth0_dev, kps1_dev, depth1_dev, K0_dev, K1_dev,
                               Kori0_dev, Kori1_dev, T_0to1_dev, grid_dev, B, N, it_matches, it_ransac, n_sample, loss_type,
                               soft_clipping, null_hypothesis, inlier_3d_th, score_temperature, null_score, null_loss);
  MK_CUDA_CHECK(cudaMemsetAsync(status_dev, 0, sizeof(int), st));
  MK_CUDA_CHECK(launch_k(loss_tail_fwd_kernel, dim3(B * it_matches), dim3(TAIL_THREADS), (size_t)6 * n_sample * sizeof(double),
                         st, A, carve_tail(ws_dev, B, it_matches, it_ransac, n_sample), loss_value_dev, loss_rot_dev,
                         loss_trans_dev, status_dev));
  return MK_OK;
}

extern "C" int mk_loss_tail_backward(const int* sampled_idx_dev, const unsigned int* inliers_dev, const float* kps0_dev,
                                     const float* depth0_dev, const float* kps1_dev, const float* depth1_dev,
                                     const float* K0_dev, const float* K1_dev, const float* Kori0_dev,
                                     const float* Kori1_dev, const float* T_0to1_dev, const float* grid_dev, int B, int N,
                                     int it_matches, int it_ransac, int n_sample, int loss_type, int soft_clipping,
                                     int null_hypothesis, float inlier_3d_th, float score_temperature,
                                     const float* grad_loss_value_dev, const float* grad_loss_rot_dev,
                                     const float* grad_loss_trans_dev, float* dkps0_dev, float* dkps1_dev,
                                     float* ddepth0_dev, float* ddepth1_dev, void* ws_dev, long long ws_bytes,
                                     void* stream) {
  if (!tail_inputs_ok(sampled_idx_dev, inliers_dev, kps0_dev, depth0_dev, kps1_dev, depth1_dev, K0_dev, K1_dev, Kori0_dev,
                      Kori1_dev, T_0to1_dev, grid_dev, ws_dev) || !grad_loss_value_dev || !grad_loss_rot_dev ||
      !grad_loss_trans_dev || !dkps0_dev || !dkps1_dev || !ddepth0_dev || !ddepth1_dev) {
    set_last_error("mk_loss_tail_backward: every input, upstream gradient, output and the workspace must be non-NULL");
    return MK_ERR_INVALID;
  }
  MK_TRY(tail_check("mk_loss_tail_backward", B, N, it_matches, it_ransac, n_sample, loss_type, inlier_3d_th,
                    score_temperature));
  const long long need = loss_tail_ws_bytes(B, N, it_matches, it_ransac, n_sample);
  if (ws_bytes < need) {
    set_last_error("mk_loss_tail_backward: workspace of %lld bytes, %lld needed", ws_bytes, need);
    return MK_ERR_INVALID;
  }
  cudaStream_t st = (cudaStream_t)stream;
  MK_TRY(tail_configure());
  const TailArgs A = tail_args(sampled_idx_dev, inliers_dev, kps0_dev, depth0_dev, kps1_dev, depth1_dev, K0_dev, K1_dev,
                               Kori0_dev, Kori1_dev, T_0to1_dev, grid_dev, B, N, it_matches, it_ransac, n_sample, loss_type,
                               soft_clipping, null_hypothesis, inlier_3d_th, score_temperature, 0.f, 0.f);
  const TailWs W = carve_tail(ws_dev, B, it_matches, it_ransac, n_sample);
  MK_CUDA_CHECK(launch_k(loss_tail_bwd_kernel, dim3(B * it_matches), dim3(TAIL_THREADS), (size_t)6 * n_sample * sizeof(double),
                         st, A, W, grad_loss_value_dev, grad_loss_rot_dev, grad_loss_trans_dev));
  MK_CUDA_CHECK(launch_k(loss_tail_scatter_kernel, dim3((unsigned)ceil_div(N, SCATTER_THREADS), (unsigned)B),
                         dim3(SCATTER_THREADS), 0, st, sampled_idx_dev, (const double*)W.contrib, N, it_matches, n_sample,
                         dkps0_dev, dkps1_dev, ddepth0_dev, ddepth1_dev));
  return MK_OK;
}
