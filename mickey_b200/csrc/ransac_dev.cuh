// Device helpers shared by the solver (ransac.cu) and the training loss (loss.cu): the counter-based generator,
// the gather + back-projection of a sampled set, the fp64 Kabsch rotation and the cdf search of the inner draws.
#pragma once
#include "common.cuh"

namespace mk {

// ---- Philox4x32-7 (7 rounds pass BigCrush: Salmon et al., SC'11) ----------------------------------------
struct Philox {
  uint32_t k0, k1;
  __device__ __forceinline__ Philox(unsigned long long seed) : k0((uint32_t)seed), k1((uint32_t)(seed >> 32)) {}
  __device__ __forceinline__ uint4 operator()(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3) const {
    uint32_t a = k0, b = k1;
#pragma unroll
    for (int r = 0; r < 7; ++r) {
      const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
      const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
      c0 = hi1 ^ c1 ^ a; c1 = lo1; c2 = hi0 ^ c3 ^ b; c3 = lo0;
      a += 0x9E3779B9u; b += 0xBB67AE85u;
    }
    return make_uint4(c0, c1, c2, c3);
  }
};

__device__ __forceinline__ float u01_from_bits(uint32_t x) { return ((float)(x >> 8) + 0.5f) * 5.9604644775390625e-8f; }

// ---- gather + back-projection ----------------------------------------------------------------------------------
__device__ __forceinline__ void inv3x3(const float* K, float* Ki) {
  const double a = K[0], b = K[1], c = K[2], d = K[3], e = K[4], f = K[5], g = K[6], h = K[7], i = K[8];
  const double A = e * i - f * h, Bc = -(d * i - f * g), C = d * h - e * g;
  const double det = a * A + b * Bc + c * C;
  const double id = 1.0 / det;
  Ki[0] = (float)(A * id);  Ki[1] = (float)(-(b * i - c * h) * id); Ki[2] = (float)((b * f - c * e) * id);
  Ki[3] = (float)(Bc * id); Ki[4] = (float)((a * i - c * g) * id);  Ki[5] = (float)(-(a * f - c * d) * id);
  Ki[6] = (float)(C * id);  Ki[7] = (float)(-(a * h - b * g) * id); Ki[8] = (float)((a * e - b * d) * id);
}

// Back-projected 3D points of one set of sampled matches, straight into the block's shared memory (X[3][n_s], Y[3][n_s])
// together with the per-thread inclusive running sums of the match weights (cdf, when wanted): with
// per = ceil(n_s / n_threads), thread t owns the samples t * per + j (j < per) that are < n_s (the order the weights'
// prefix sums are defined in); threads past the end own none and keep run = 0.  When n_threads divides n_s this is
// the plain split t * per .. t * per + per - 1.
__device__ __forceinline__ void gather_set(const int* __restrict__ idx, const float* __restrict__ fs,
                                           const float* __restrict__ kps0, const float* __restrict__ d0,
                                           const float* __restrict__ kps1, const float* __restrict__ d1,
                                           const float* Ki0, const float* Ki1, int N, long long pitch, int b, long long s, int n_s,
                                           int n_threads, float* X, float* Y, float* cdf, float& run) {
  const int per = (n_s + n_threads - 1) / n_threads;
  const int own = min(per, max(n_s - (int)threadIdx.x * per, 0));          // samples this thread owns
  run = 0.f;
  // groups of 8 samples: the index -> keypoint / depth / score loads of a group are independent and issued together (the
  // score is a random access into the N x N matrix: one DRAM round trip per GROUP, not per sample); the running sum follows
  for (int j0 = 0; j0 < own; j0 += 8) {
    float wv[8];
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      wv[jj] = 0.f;
      if (j0 + jj < own) {
        const int i = threadIdx.x * per + j0 + jj;
        const int cell = idx[s * n_s + i];
        const int i0 = cell / N, i1 = cell - i0 * N;
        const float u0 = kps0[((long long)b * 2 + 0) * N + i0], v0 = kps0[((long long)b * 2 + 1) * N + i0];
        const float u1 = kps1[((long long)b * 2 + 0) * N + i1], v1 = kps1[((long long)b * 2 + 1) * N + i1];
        const float z0 = d0[(long long)b * N + i0], z1 = d1[(long long)b * N + i1];
        if (cdf) wv[jj] = fs[(long long)b * N * pitch + (long long)i0 * pitch + i1];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          X[r * n_s + i] = z0 * (Ki0[r * 3] * u0 + Ki0[r * 3 + 1] * v0 + Ki0[r * 3 + 2]);
          Y[r * n_s + i] = z1 * (Ki1[r * 3] * u1 + Ki1[r * 3 + 1] * v1 + Ki1[r * 3 + 2]);
        }
      }
    }
    if (cdf) {
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        if (j0 + jj < own) { run += wv[jj]; cdf[threadIdx.x * per + j0 + jj] = run; }
    }
  }
}

// ---- 3x3 SVD (one-sided Jacobi, fp64) and Kabsch ------------------------------------------------------------------
// H = U S V^T.  Returns R = V diag(1,1,det(U V^T)) U^T (solvers.py:45-50).  With u3 := u1 x u2 and v3 := v1 x v2 both
// factors are proper rotations, so R = V U^T already has det +1 and equals the reference's sign-fixed product for
// every rank >= 2 matrix (3-point hypotheses are always rank <= 2: the third singular direction is a cross product,
// not a division by ~0).
// H is first scaled by the power of two that puts max|H_ij| in [1, 2): R does not depend on the scale, every step of
// the sweep is homogeneous in it and a power-of-two scale is exact, so R is bit-identical to the unscaled sweep wherever
// both stay in the normal range, and the absolute guards below (1e-300) mean the same thing at every scale.  A NaN or
// +-inf anywhere in H gives R = NaN in all nine entries; H == 0 gives the identity.
// __host__ __device__ so that host tests can build the same function (tests/test_kabsch_host.py).
__host__ __device__ inline void kabsch_rotation(const double* Hin, double* R) {
  double A[3][3], V[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
  double hmax = 0.0;
  bool finite = true;
#pragma unroll
  for (int i = 0; i < 9; ++i) {
    const double a = fabs(Hin[i]);
    finite = finite && a <= 1.7976931348623157e308;            // false for NaN and +-inf
    hmax = fmax(hmax, a);
  }
  if (!finite) {
#pragma unroll
    for (int i = 0; i < 9; ++i) R[i] = nan("");
    return;
  }
  if (hmax == 0.0) {     // H == 0: identity
#pragma unroll
    for (int i = 0; i < 9; ++i) R[i] = (i % 4 == 0) ? 1.0 : 0.0;
    return;
  }
  int ex;
  frexp(hmax, &ex);                                             // hmax = m 2^ex, m in [0.5, 1)
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) A[i][j] = ldexp(Hin[i * 3 + j], 1 - ex);
  for (int sweep = 0; sweep < 12; ++sweep) {
    double off = 0.0;
#pragma unroll
    for (int pq = 0; pq < 3; ++pq) {
      const int p = (pq == 2) ? 1 : 0, q = (pq == 0) ? 1 : 2;
      double al = 0, be = 0, ga = 0;
#pragma unroll
      for (int i = 0; i < 3; ++i) { al += A[i][p] * A[i][p]; be += A[i][q] * A[i][q]; ga += A[i][p] * A[i][q]; }
      const double lim = 1e-15 * sqrt(al * be);
      if (fabs(ga) > lim && fabs(ga) > 1e-300) {
        off = fmax(off, fabs(ga) / fmax(sqrt(al * be), 1e-300));
        const double zeta = (be - al) / (2.0 * ga);
        const double t = copysign(1.0, zeta) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          const double ap = A[i][p], aq = A[i][q];
          A[i][p] = c * ap - s * aq; A[i][q] = s * ap + c * aq;
          const double vp = V[i][p], vq = V[i][q];
          V[i][p] = c * vp - s * vq; V[i][q] = s * vp + c * vq;
        }
      }
    }
    if (off < 1e-14) break;
  }
  double sg[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) sg[j] = sqrt(A[0][j] * A[0][j] + A[1][j] * A[1][j] + A[2][j] * A[2][j]);
  int i1 = 0;
  if (sg[1] > sg[i1]) i1 = 1;
  if (sg[2] > sg[i1]) i1 = 2;
  int i2 = (i1 + 1) % 3, i3 = (i1 + 2) % 3;
  if (sg[i3] > sg[i2]) { const int tmp = i2; i2 = i3; i3 = tmp; }
  double u1[3], u2[3], v1[3], v2[3];
  // s1 > 0.5: the scaled H has an entry >= 1, and the rotations keep the Frobenius norm, so max_j sg[j]^2 >= 1/3
  const double s1 = sg[i1], s2 = sg[i2];
#pragma unroll
  for (int i = 0; i < 3; ++i) { u1[i] = A[i][i1] / s1; v1[i] = V[i][i1]; v2[i] = V[i][i2]; }
  if (s2 > 1e-14 * s1) {
#pragma unroll
    for (int i = 0; i < 3; ++i) u2[i] = A[i][i2] / s2;
    // re-orthogonalise u2 against u1 (guards the nearly rank-1 case)
    const double d = u1[0] * u2[0] + u1[1] * u2[1] + u1[2] * u2[2];
    double nn = 0;
#pragma unroll
    for (int i = 0; i < 3; ++i) { u2[i] -= d * u1[i]; nn += u2[i] * u2[i]; }
    nn = 1.0 / sqrt(nn);
#pragma unroll
    for (int i = 0; i < 3; ++i) u2[i] *= nn;
  } else {
    // rank 1 (collinear sample): the optimum is not unique; pick the completion that maps v2 -> any unit vector
    // orthogonal to u1 (the reference's LAPACK choice is equally arbitrary)
    int k = 0;
    if (fabs(u1[1]) < fabs(u1[k])) k = 1;
    if (fabs(u1[2]) < fabs(u1[k])) k = 2;
    double e[3] = {0, 0, 0};
    e[k] = 1.0;
    const double d = u1[k];
    double nn = 0;
#pragma unroll
    for (int i = 0; i < 3; ++i) { u2[i] = e[i] - d * u1[i]; nn += u2[i] * u2[i]; }
    nn = 1.0 / sqrt(nn);
#pragma unroll
    for (int i = 0; i < 3; ++i) u2[i] *= nn;
  }
  const double u3[3] = {u1[1] * u2[2] - u1[2] * u2[1], u1[2] * u2[0] - u1[0] * u2[2], u1[0] * u2[1] - u1[1] * u2[0]};
  const double v3[3] = {v1[1] * v2[2] - v1[2] * v2[1], v1[2] * v2[0] - v1[0] * v2[2], v1[0] * v2[1] - v1[1] * v2[0]};
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) R[i * 3 + j] = v1[i] * u1[j] + v2[i] * u2[j] + v3[i] * u3[j];
}

__device__ __forceinline__ int cdf_search(const float* cdf, int n, float target) {
  // first i with cdf[i] > target
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (cdf[mid] > target) hi = mid; else lo = mid + 1;
  }
  return lo;
}

}  // namespace mk
