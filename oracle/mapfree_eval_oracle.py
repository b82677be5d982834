"""fp64 numpy restatement of the Map-free benchmark's per-frame errors: MetricManager's trans_err, rot_err (sin variant)
and reproj_err (benchmark/metrics.py, benchmark/reprojection.py, benchmark/utils.py), one frame at a time.

It takes what mk_mapfree_frame_metrics takes (world-to-camera poses as a submission line and poses.txt hold them, K, the
image size) and performs the benchmark's numpy operations on arrays of the benchmark's shapes: the transforms3d
quaternion formulas, np.linalg.inv of the estimate's 4x4 camera-to-world matrix, (K @ X.T).T and np.clip of both
projections.  tests/golden/reference_mapfree_eval.json pins it to the live benchmark; the GPU tests hold the kernel to it,
and the CPU tests grade whole submissions with it in the kernel's place.
"""
import numpy as np

from mickey_b200.loss import vcre_grid

_EYE = np.concatenate([vcre_grid().numpy(), np.ones((196, 1))], -1)          # [196, 4], eye_coords_glob


def qmult(a, b):
    w1, x1, y1, z1 = a
    w2, x2, y2, z2 = b
    return np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 + y1 * w2 + z1 * x2 - x1 * z2, w1 * z2 + z1 * w2 + x1 * y2 - y1 * x2])


def qconjugate(q):
    return q * np.array([1.0, -1.0, -1.0, -1.0])


def qinverse(q):
    return qconjugate(q) / np.dot(q, q)


def quat2mat(q):
    """The rotation of q / |q|; the identity where |q|^2 is below machine epsilon."""
    w, x, y, z = q
    n = w * w + x * x + y * y + z * z
    if n < np.finfo(np.float64).eps:
        return np.eye(3)
    s = 2.0 / n
    X, Y, Z = x * s, y * s, z * s
    wX, wY, wZ, xX, xY, xZ, yY, yZ, zZ = w * X, w * Y, w * Z, x * X, x * Y, x * Z, y * Y, y * Z, z * Z
    return np.array([[1.0 - (yY + zZ), xY - wZ, xZ + wY],
                     [xY + wZ, 1.0 - (xX + zZ), yZ - wX],
                     [xZ - wY, yZ + wX, 1.0 - (xX + yY)]])


def world2cam_to_cam2world(q, t):
    """convert_world2cam_to_cam2world: (qinverse(q), -rotate_vector(t, qinverse(q))), rotate_vector with its default
    is_normalized=True (the conjugate), so a non-unit q scales the centre by 1/|q|^4."""
    qi = qinverse(np.asarray(q, dtype=np.float64))
    v = np.zeros(4)
    v[1:] = t
    return qi, -qmult(qi, qmult(v, qconjugate(qi)))[1:]


def project(pts, K, W, H):
    """[n, 3/4] camera points -> [n, 2] pixels clipped to [0, W] x [0, H]; no depth test (numpy divides by any depth)."""
    uv_h = (K @ pts[:, :3].T).T
    uv = uv_h[:, :2] / uv_h[:, -1:]
    uv[:, 0] = np.clip(uv[:, 0], 0, W)
    uv[:, 1] = np.clip(uv[:, 1], 0, H)
    return uv


def frame_errors(q_est, t_est, q_gt, t_gt, K, W, H):
    """One frame, world-to-camera poses -> (trans_err, rot_err, reproj_err)."""
    qe, ce = world2cam_to_cam2world(q_est, t_est)
    qg, cg = world2cam_to_cam2world(q_gt, t_gt)
    trans_err = np.linalg.norm(ce - cg)
    # quat_angle_error(label=q_est, pred=q_gt): qmult(pred, qinverse(label)) on the normalised quaternions
    # (normalised along axis 1 of a [1, 4] array, as the benchmark does: a different summation than the 1-D norm's)
    q1 = (qg[None] / np.linalg.norm(qg[None], axis=1, keepdims=True))[0]
    q2 = (qe[None] / np.linalg.norm(qe[None], axis=1, keepdims=True))[0]
    s = qmult(q1, qinverse(q2))
    rot_err = np.arcsin(np.linalg.norm(s[1:])) * 114.59155902616465
    cam2w_est, cam2w_gt = np.eye(4), np.eye(4)
    cam2w_est[:3, :3], cam2w_est[:3, -1] = quat2mat(qe), ce
    cam2w_gt[:3, :3], cam2w_gt[:3, -1] = quat2mat(qg), cg
    uv_gt = project(_EYE, K, W, H)
    uv_pred = project((np.linalg.inv(cam2w_est) @ cam2w_gt @ _EYE.T).T, K, W, H)
    reproj_err = float(np.linalg.norm(uv_gt - uv_pred, ord=2, axis=1).mean())
    return trans_err, rot_err, reproj_err


def frame_metrics(q_est, t_est, q_gt, t_gt, K, W, H):
    """The frames' errors as mk_mapfree_frame_metrics returns them: q [P, 4], t [P, 3], K [P, 3, 3], W and H scalars or
    [P] -> fp64 [P, 3] = trans_err, rot_err, reproj_err."""
    q_est, t_est, q_gt, t_gt, K = (np.asarray(a, dtype=np.float64) for a in (q_est, t_est, q_gt, t_gt, K))
    P = q_est.shape[0]
    W = np.broadcast_to(np.asarray(W, dtype=np.float64), (P,))
    H = np.broadcast_to(np.asarray(H, dtype=np.float64), (P,))
    out = np.empty((P, 3))
    with np.errstate(divide="ignore", invalid="ignore"):
        for i in range(P):
            out[i] = frame_errors(q_est[i], t_est[i], q_gt[i], t_gt[i], K[i], W[i], H[i])
    return out
