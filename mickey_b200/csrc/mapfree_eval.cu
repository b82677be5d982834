// Map-free benchmark grading: the per-frame errors of the benchmark's MetricManager (benchmark/metrics.py), trans_err,
// rot_err and reproj_err, in fp64, for every graded frame of a split in one launch.
//
// A frame arrives as the submission line and poses.txt store it: world-to-camera q = (w, x, y, z) with any non-zero norm,
// and t.  Both poses are first turned camera-to-world as benchmark/utils.py::convert_world2cam_to_cam2world does:
//     qi = conj(q) / |q|^2,    c = -vec(qi (x) (0, t) (x) conj(qi))
// (rotate_vector with is_normalized=True uses the conjugate, so for |q| != 1 the centre c is scaled by 1/|q|^4).
//   trans_err  = |c_est - c_gt|.
//   rot_err    = asin(|vec(q1 (x) q2^-1)|) * 114.59155902616465 with q1 = qi_gt / |qi_gt|, q2 = qi_est / |qi_est|
//                (quat_angle_error, sin variant, called with label = est and pred = gt: the operand order is kept).
//   reproj_err = mean over the 196 virtual points X of |clip(proj(K X)) - clip(proj(K (M X)))|,
//                M = [R_est c_est]^-1 [R_gt c_gt], R = quat2mat(qi) (which normalises, so R does not depend on |q|),
//                proj(h) = (h0 / h2, h1 / h2) with no test on the depth h2 (a point behind the camera divides by a negative
//                or zero depth, as numpy does) and clip to [0, W] x [0, H] with a NaN passed through, as np.clip does.
//                [R c]^-1 is taken as [R^T, -R^T c]; R is orthonormal to rounding, so this agrees with the reference's
//                np.linalg.inv to rounding.
//
// Layout: one warp per frame, MF_WARPS frames per block; the grid's 196 points are staged in shared memory once per
// block, after pdl_wait() (launch_k launches carry the PDL attribute).  Every lane computes the frame's transforms (a few
// dozen flops), lane l projects points l, l + 32, ... and sums its distances in ascending point order; a butterfly over
// the 32 lanes then adds the partial sums.  The order depends on nothing but the point index, so a frame's three values
// are the same bits alone, inside any batch and on every run.
#include "common.cuh"
#include "../../include/mickey_b200.h"

#include <cfloat>

namespace mk {
namespace {

constexpr int MF_WARPS = 8;
constexpr int MF_THREADS = MF_WARPS * 32;
constexpr int MF_POINTS = MK_VCRE_POINTS;

struct Quat { double w, x, y, z; };

__device__ __forceinline__ Quat qmult(const Quat a, const Quat b) {
  return {a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
          a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z, a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x};
}

__device__ __forceinline__ double qdot(const Quat q) { return q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z; }

__device__ __forceinline__ Quat qinverse(const Quat q) {
  const double n = qdot(q);
  return {q.w / n, -q.x / n, -q.y / n, -q.z / n};
}

// world-to-camera (q, t) -> camera-to-world rotation quaternion qi and camera centre c
__device__ __forceinline__ void to_cam2world(const double* q, const double* t, Quat& qi, double c[3]) {
  qi = qinverse(Quat{q[0], q[1], q[2], q[3]});
  const Quat r = qmult(qi, qmult(Quat{0.0, t[0], t[1], t[2]}, Quat{qi.w, -qi.x, -qi.y, -qi.z}));
  c[0] = -r.x; c[1] = -r.y; c[2] = -r.z;
}

// transforms3d's quat2mat: the identity below machine epsilon, else the rotation of q / |q|
__device__ __forceinline__ void quat2mat(const Quat q, double R[9]) {
  const double n = qdot(q);
  if (n < DBL_EPSILON) {
    for (int i = 0; i < 9; ++i) R[i] = (i % 4 == 0) ? 1.0 : 0.0;
    return;
  }
  const double s = 2.0 / n;
  const double X = q.x * s, Y = q.y * s, Z = q.z * s;
  const double wX = q.w * X, wY = q.w * Y, wZ = q.w * Z, xX = q.x * X, xY = q.x * Y, xZ = q.x * Z;
  const double yY = q.y * Y, yZ = q.y * Z, zZ = q.z * Z;
  R[0] = 1.0 - (yY + zZ); R[1] = xY - wZ;         R[2] = xZ + wY;
  R[3] = xY + wZ;         R[4] = 1.0 - (xX + zZ); R[5] = yZ - wX;
  R[6] = xZ - wY;         R[7] = yZ + wX;         R[8] = 1.0 - (xX + yY);
}

// np.clip(v, 0, hi): NaN stays NaN, +-inf go to the borders
__device__ __forceinline__ double clip(const double v, const double hi) {
  return v != v ? v : (v < 0.0 ? 0.0 : (v > hi ? hi : v));
}

__global__ void __launch_bounds__(MF_THREADS) mapfree_frame_metrics_kernel(
    const double* __restrict__ q_est, const double* __restrict__ t_est, const double* __restrict__ q_gt,
    const double* __restrict__ t_gt, const double* __restrict__ Kall, const double* __restrict__ grid, int P, double W,
    double H, double* __restrict__ err) {
  __shared__ double pts[MF_POINTS * 3];
  pdl_wait();
  for (int i = threadIdx.x; i < MF_POINTS * 3; i += MF_THREADS) pts[i] = grid[i];
  __syncthreads();
  const int f = blockIdx.x * MF_WARPS + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (f >= P) return;

  Quat qe, qg;
  double ce[3], cg[3];
  to_cam2world(q_est + 4 * f, t_est + 3 * f, qe, ce);
  to_cam2world(q_gt + 4 * f, t_gt + 3 * f, qg, cg);

  // rotation: qmult(pred, qinverse(label)) on the normalised quaternions, pred = gt, label = est
  const double ng = sqrt(qdot(qg)), ne = sqrt(qdot(qe));
  const Quat q1{qg.w / ng, qg.x / ng, qg.y / ng, qg.z / ng}, q2{qe.w / ne, qe.x / ne, qe.y / ne, qe.z / ne};
  const Quat s = qmult(q1, qinverse(q2));
  const double rot_err = asin(sqrt(s.x * s.x + s.y * s.y + s.z * s.z)) * 114.59155902616465;
  const double dc0 = ce[0] - cg[0], dc1 = ce[1] - cg[1], dc2 = ce[2] - cg[2];
  const double trans_err = sqrt(dc0 * dc0 + dc1 * dc1 + dc2 * dc2);

  // residual M = [Re ce]^-1 [Rg cg] = [Re^T Rg, Re^T (cg - ce)]
  double Re[9], Rg[9], M[12];
  quat2mat(qe, Re);
  quat2mat(qg, Rg);
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) M[4 * i + j] = Re[i] * Rg[j] + Re[3 + i] * Rg[3 + j] + Re[6 + i] * Rg[6 + j];
    M[4 * i + 3] = Re[i] * (cg[0] - ce[0]) + Re[3 + i] * (cg[1] - ce[1]) + Re[6 + i] * (cg[2] - ce[2]);
  }
  double K[9];
  for (int i = 0; i < 9; ++i) K[i] = Kall[9 * f + i];

  double acc = 0.0;
  for (int n = lane; n < MF_POINTS; n += 32) {
    const double x = pts[3 * n], y = pts[3 * n + 1], z = pts[3 * n + 2];
    double h0 = K[0] * x + K[1] * y + K[2] * z, h1 = K[3] * x + K[4] * y + K[5] * z, h2 = K[6] * x + K[7] * y + K[8] * z;
    const double ug = clip(h0 / h2, W), vg = clip(h1 / h2, H);
    const double px = M[0] * x + M[1] * y + M[2] * z + M[3], py = M[4] * x + M[5] * y + M[6] * z + M[7],
                 pz = M[8] * x + M[9] * y + M[10] * z + M[11];
    h0 = K[0] * px + K[1] * py + K[2] * pz; h1 = K[3] * px + K[4] * py + K[5] * pz; h2 = K[6] * px + K[7] * py + K[8] * pz;
    const double du = ug - clip(h0 / h2, W), dv = vg - clip(h1 / h2, H);
    acc += sqrt(du * du + dv * dv);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) {
    err[3 * f] = trans_err;
    err[3 * f + 1] = rot_err;
    err[3 * f + 2] = acc / (double)MF_POINTS;
  }
}

}  // namespace

static int mapfree_frame_metrics(const double* q_est, const double* t_est, const double* q_gt, const double* t_gt,
                                 const double* K, const double* grid, int P, int W, int H, double* err, cudaStream_t st) {
  // every argument is checked before anything is launched
  if (!q_est || !t_est || !q_gt || !t_gt || !K || !grid || !err) {
    set_last_error("mk_mapfree_frame_metrics: q_est, t_est, q_gt, t_gt, K, grid and err must be non-NULL");
    return MK_ERR_INVALID;
  }
  if (P < 1 || P > MK_MAPFREE_MAX_FRAMES || W < 1 || H < 1) {
    set_last_error("mk_mapfree_frame_metrics: need 1 <= P <= %d and a positive image size (got P %d, W %d, H %d)",
                   MK_MAPFREE_MAX_FRAMES, P, W, H);
    return MK_ERR_INVALID;
  }
  MK_CUDA_CHECK(launch_k(mapfree_frame_metrics_kernel, dim3(ceil_div(P, MF_WARPS)), dim3(MF_THREADS), 0, st, q_est, t_est,
                         q_gt, t_gt, K, grid, P, (double)W, (double)H, err));
  return MK_OK;
}

}  // namespace mk

extern "C" int mk_mapfree_frame_metrics(const double* q_est_dev, const double* t_est_dev, const double* q_gt_dev,
                                        const double* t_gt_dev, const double* K_dev, const double* grid_dev, int P,
                                        int W, int H, double* err_dev, void* stream) {
  return mk::mapfree_frame_metrics(q_est_dev, t_est_dev, q_gt_dev, t_gt_dev, K_dev, grid_dev, P, W, H, err_dev,
                                   (cudaStream_t)stream);
}
