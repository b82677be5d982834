"""The fp64 Kabsch rotation (`kabsch_rotation`, csrc/ransac_dev.cuh): a table of 3x3 cases, a 50-digit reference,
bounds that hold for every finite H, and a vectorised numpy restatement of the one-sided Jacobi sweep that exists only
so that mutations can be planted and shown to be rejected.

Notation: H = U diag(sigma) V^T with sigma_1 >= sigma_2 >= sigma_3 >= 0, d = det(U) det(V) (= sign det H when H is
regular), R_ref = V diag(1, 1, d) U^T, the rotation that maximises tr(R H).  u = 2^-53.

Bounds, for every finite H (they hold where the optimum is not unique, too):
  - orthogonality    max |R^T R - I|                                          <= C_ORTH u
  - determinant      |det R - 1|                                              <= C_DET u
  - optimality       sigma_1 + sigma_2 + d sigma_3 - tr(R H)                  <= C_OPT u sigma_1
and, element by element, the polar-factor perturbation bound with the sign fix:
  - |R - R_ref| <= C_ELEM u kappa,   kappa = sigma_1 / min_{i<j} (s_i + s_j),  s = (sigma_1, sigma_2, d sigma_3),
so kappa = sigma_1 / (sigma_2 + d sigma_3): a det < 0 matrix with sigma_2 ~ sigma_3 is ill-posed, as is rank 1
(kappa = inf: no element bound).  A rank-1 completion (the kernel's branch sigma_2 <= 1e-14 sigma_1) is checked for
optimality and for R u_1 = v_1 (|R u_1 - v_1| <= C_ELEM u).  H = 0 gives the identity; a NaN or +-inf anywhere in H
gives nine NaNs.

R_ref, sigma and d come from mpmath at 50 digits on the exact fp64 H: an fp64 SVD's own error is also u kappa.
When H is formed from fp32 points in fp64 (the solver's hypotheses and refinements), `formation_bound` adds the
rounding of the centroid and of the sum of outer products, 2 |dH|_F / (sigma_2 + d sigma_3) (the same perturbation
bound), and the caller adds 2^-24 |R| for the fp32 store.
"""
from __future__ import annotations

import math

import mpmath
import numpy as np

U64 = 2.0 ** -53
U32 = 2.0 ** -24
C_ORTH, C_DET, C_OPT, C_ELEM = 32.0, 32.0, 16.0, 64.0
RANK1_TOL = 1e-14                  # the kernel's rank-2 threshold on sigma_2 / sigma_1


# ---------------------------------------------------------------------------------------------------------------
# the case table
# ---------------------------------------------------------------------------------------------------------------
def rand_rot(rng, n):
    """n Haar-random proper rotations [n, 3, 3]."""
    Q, Rq = np.linalg.qr(rng.standard_normal((n, 3, 3)))
    Q = Q * np.sign(np.diagonal(Rq, axis1=1, axis2=2))[:, None, :]
    return Q * np.sign(np.linalg.det(Q))[:, None, None]


def axis_angle(axis, ang):
    """Rotations [n, 3, 3] about unit axes [n, 3] by angles [n] (fp64 Rodrigues)."""
    axis = np.asarray(axis, dtype=np.float64)
    axis = axis / np.linalg.norm(axis, axis=-1, keepdims=True)
    ang = np.asarray(ang, dtype=np.float64)
    x, y, z = axis[..., 0], axis[..., 1], axis[..., 2]
    Kx = np.zeros(axis.shape[:-1] + (3, 3))
    Kx[..., 0, 1], Kx[..., 0, 2], Kx[..., 1, 0] = -z, y, z
    Kx[..., 1, 2], Kx[..., 2, 0], Kx[..., 2, 1] = -x, -y, x
    s, c = np.sin(ang)[..., None, None], np.cos(ang)[..., None, None]
    return np.eye(3) + s * Kx + (1 - c) * (Kx @ Kx)


def with_sv(rng, s, det_sign=1.0):
    """H = Q diag(s) P for seeded rotations Q, P; det_sign = -1 flips the sign of the third singular value."""
    s = np.atleast_2d(np.asarray(s, dtype=np.float64)).copy()
    s[:, 2] *= det_sign
    n = s.shape[0]
    return rand_rot(rng, n) @ (s[:, :, None] * rand_rot(rng, n))


def kernel_H(X, Y):
    """H of point sets X, Y [n, k, 3] (fp32 values) formed in fp64 as the solver's hypotheses do: the centroid is the
    fp64 sum / k, then H += (x - xm)(y - ym)^T over the points in order."""
    X, Y = np.asarray(X, dtype=np.float64), np.asarray(Y, dtype=np.float64)
    k = X.shape[1]
    xm, ym = np.zeros(X.shape[:1] + (3,)), np.zeros(X.shape[:1] + (3,))
    for j in range(k):
        xm, ym = xm + X[:, j], ym + Y[:, j]
    xm, ym = xm / k, ym / k
    H = np.zeros(X.shape[:1] + (3, 3))
    for j in range(k):
        H = H + (X[:, j] - xm)[:, :, None] * (Y[:, j] - ym)[:, None, :]
    return H


def point_sets(rng, n, k, kind, rel=0.0):
    """Seeded fp32 point sets (X, Y) [n, k, 3] of one kind: 'noisy' (Y = R X + t + noise), 'collinear',
    'coincident', 'near_collinear' (off the line by rel of the spread), 'coplanar', 'mirrored' (Y = X reflected)."""
    R, t = rand_rot(rng, n), rng.standard_normal((n, 1, 3))
    base = rng.uniform(-1.0, 1.0, (n, 1, 3)) + np.array([0.0, 0.0, 4.0])
    if kind == "collinear" or kind == "near_collinear":
        d = rng.standard_normal((n, 1, 3))
        X = base + rng.uniform(-1, 1, (n, k, 1)) * d
        if kind == "near_collinear":
            X = X + rel * rng.standard_normal((n, k, 3)) * np.linalg.norm(d, axis=-1, keepdims=True)
    elif kind == "coincident":
        X = np.repeat(base, k, axis=1)
    elif kind == "coplanar":
        e1, e2 = rng.standard_normal((n, 1, 3)), rng.standard_normal((n, 1, 3))
        X = base + rng.uniform(-1, 1, (n, k, 1)) * e1 + rng.uniform(-1, 1, (n, k, 1)) * e2
    else:
        X = base + rng.uniform(-1, 1, (n, k, 3))
    X = X.astype(np.float32).astype(np.float64)
    if kind == "mirrored":
        Y = X * np.array([-1.0, 1.0, 1.0]) + t
    else:
        Y = X @ np.swapaxes(R, 1, 2) + t
        if kind == "noisy":
            Y = Y + 0.01 * rng.standard_normal(Y.shape)
    return X.astype(np.float32), Y.astype(np.float32)


def case_table(seed=0, per=12):
    """{class: H [n, 3, 3] fp64}: every class of DESIGN §2's Kabsch table."""
    rng = np.random.default_rng(seed)
    T = {}
    T["random"] = rng.standard_normal((4 * per, 3, 3))
    for gap in (1e-1, 1e-4, 1e-7, 1e-10):
        for sgn, nm in ((1.0, "pos"), (-1.0, "neg")):
            T[f"gap12_{gap:.0e}_{nm}"] = with_sv(rng, [[1.0, 1.0 - gap, 0.3]] * per, sgn)
            T[f"gap23_{gap:.0e}_{nm}"] = with_sv(rng, [[1.0, 0.5, 0.5 - gap]] * per, sgn)
    T["s2_eq_s3_neg"] = with_sv(rng, [[1.0, 0.4, 0.4]] * per, -1.0)
    for r in (1e-1, 1e-3, 1e-6, 1e-9, 1e-12, 1e-15):
        T[f"rank2_{r:.0e}"] = with_sv(rng, [[1.0, r, 0.0]] * per)
    ia, ib = rng.integers(-8, 9, (2, per, 2, 3)).astype(np.float64)       # integer vectors: exact fp64 products
    T["rank2_exact"] = ia[:, 0, :, None] * ib[:, 0, None, :] + ia[:, 1, :, None] * ib[:, 1, None, :]
    T["rank1_exact"] = ia[:, 0, :, None] * ib[:, 0, None, :]
    T["rank1_near"] = with_sv(rng, [[1.0, 1e-15, 1e-16]] * per)
    T["s1_eq_s2_eq_s3"] = with_sv(rng, [[2.0, 2.0, 2.0]] * per)
    T["s1_eq_s2_s3_zero"] = with_sv(rng, [[1.0, 1.0, 0.0]] * per)
    # 180 degree rotations: H = R180^T diag(s) so that R_ref = R180 and tr(H) < 0 (identity is far from optimal)
    ax = rng.standard_normal((per, 3))
    T["rot180"] = np.swapaxes(axis_angle(ax, np.full(per, math.pi)), 1, 2) @ np.diag([1.0, 0.8, 0.6])
    diag = [np.diag([3.0, 2.0, 1.0]), np.diag([-3.0, 2.0, 1.0]), np.diag([3.0, -2.0, -1.0]), np.diag([-1.0, -2.0, -3.0]),
            np.diag([1.0, 2.0, 3.0]), np.diag([2.0, 2.0, -2.0])]
    perm = [np.eye(3)[[1, 0, 2]] * 2.0, np.eye(3)[[2, 0, 1]] * np.array([1.0, -2.0, 3.0]), -np.eye(3)[[2, 1, 0]]]
    T["diagonal"] = np.stack(diag + perm)
    T["zero"] = np.zeros((1, 3, 3))
    base = rng.standard_normal((per, 3, 3))
    for e in (-1074 + 60, -1000, -500, -200, 200, 500, 1000):
        T[f"scale_2^{e}"] = np.ldexp(base, e)
    sub = rng.standard_normal((per, 3, 3)) * 2.0 ** -1070                 # subnormal entries, rounded
    T["subnormal"] = np.where(sub == 0, 2.0 ** -1074, sub)
    nf = []
    for v in (np.nan, np.inf, -np.inf):
        for pos in range(9):
            h = rng.standard_normal(9)
            h[pos] = v
            nf.append(h.reshape(3, 3))
    T["nonfinite"] = np.stack(nf)
    T["pts_noisy3"] = kernel_H(*point_sets(rng, 4 * per, 3, "noisy"))
    T["pts_collinear3"] = kernel_H(*point_sets(rng, per, 3, "collinear"))
    T["pts_coincident3"] = kernel_H(*point_sets(rng, per, 3, "coincident"))
    for rel in (1e-3, 1e-5, 1e-7):
        T[f"pts_near_collinear3_{rel:.0e}"] = kernel_H(*point_sets(rng, per, 3, "near_collinear", rel))
    T["pts_coplanar64"] = kernel_H(*point_sets(rng, per, 64, "coplanar"))
    T["pts_mirrored64"] = kernel_H(*point_sets(rng, per, 64, "mirrored"))
    T["pts_mirrored3"] = kernel_H(*point_sets(rng, per, 3, "mirrored"))
    return T


# ---------------------------------------------------------------------------------------------------------------
# the 50-digit reference
# ---------------------------------------------------------------------------------------------------------------
class Ref:
    """Per-matrix reference quantities (fp64 arrays over the batch)."""

    def __init__(self, H):
        H = np.asarray(H, dtype=np.float64).reshape(-1, 3, 3)
        n = H.shape[0]
        self.H = H
        self.finite = np.isfinite(H).reshape(n, 9).all(1)
        # every quantity below belongs to Hs = 2^shift H with max|Hs_ij| in [1, 2): R does not depend on the scale, and
        # the singular values of a subnormal or huge H are then representable in fp64
        hmax = np.where(self.finite, np.abs(np.where(np.isfinite(H), H, 0.0)).reshape(n, 9).max(1), 0.0)
        self.shift = np.where(hmax > 0, 1 - np.frexp(hmax)[1], 0)
        self.Hs = np.where(self.finite[:, None, None], np.ldexp(np.where(np.isfinite(H), H, 0.0), self.shift[:, None, None]), 0.0)
        self.R = np.full((n, 3, 3), np.nan)
        self.sig = np.zeros((n, 3))
        self.d = np.ones(n)
        self.u1, self.v1 = np.zeros((n, 3)), np.zeros((n, 3))
        with mpmath.workdps(50):
            for i in range(n):
                if not self.finite[i] or not H[i].any():
                    continue
                A = mpmath.matrix(self.Hs[i].tolist())
                U, S, Vt = mpmath.svd_r(A)
                d = mpmath.sign(mpmath.det(U) * mpmath.det(Vt))
                D = mpmath.diag([1, 1, d])
                Rm = Vt.T * D * U.T
                self.R[i] = np.array(Rm.tolist(), dtype=np.float64)
                self.sig[i] = [float(S[0]), float(S[1]), float(S[2])]
                self.d[i] = float(d)
                self.u1[i] = [float(U[j, 0]) for j in range(3)]
                self.v1[i] = [float(Vt[0, j]) for j in range(3)]
        s1, s2, s3 = self.sig[:, 0], self.sig[:, 1], self.sig[:, 2]
        den = s2 + self.d * s3
        with np.errstate(divide="ignore", invalid="ignore"):
            self.kappa = np.where(den > 0, s1 / np.where(den > 0, den, 1.0), np.inf)
        self.kappa[s1 == 0] = 1.0
        # the kernel takes its rank-1 branch where its own sigma_2 estimate is <= 1e-14 sigma_1: within a factor 2 of
        # the threshold either branch is correct; past it the completion is arbitrary and only optimality is checked
        self.rank1 = (s2 <= 2 * RANK1_TOL * s1) & (s1 > 0)
        self.kappa[self.rank1] = np.inf


def _mp_metrics(H, R):
    """(max|R^T R - I|, |det R - 1|, tr(R H)) at 50 digits; tr is returned scaled by nothing (fp64 of the exact)."""
    with mpmath.workdps(50):
        Rm = mpmath.matrix(R.tolist())
        E = Rm.T * Rm - mpmath.eye(3)
        orth = max(abs(E[i, j]) for i in range(3) for j in range(3))
        det = abs(mpmath.det(Rm) - 1)
        tr = mpmath.fsum(Rm[i, j] * mpmath.mpf(float(H[j, i])) for i in range(3) for j in range(3))
        return float(orth), float(det), tr


def check(H, R, ref: Ref | None = None, extra_elem=None):
    """Ratios err / bound for R = kabsch(H) ([n, 3, 3] fp64); every ratio must be <= 1.  Returns a dict of arrays:
    'orth', 'det', 'opt', 'elem' (nan where kappa = inf), 'rank1' (R u_1 = v_1, nan where not rank 1), 'nonfinite'
    (1 where H is not finite and R is not all-NaN, else 0), 'zero' (H = 0 and R != I).  `extra_elem` [n] is added to the
    element bound (formation of H, fp32 store)."""
    H = np.asarray(H, dtype=np.float64).reshape(-1, 3, 3)
    R = np.asarray(R, dtype=np.float64).reshape(-1, 3, 3)
    ref = ref if ref is not None else Ref(H)
    n = H.shape[0]
    out = {k: np.full(n, np.nan) for k in ("orth", "det", "opt", "elem", "rank1")}
    out["nonfinite"] = np.zeros(n)
    out["zero"] = np.zeros(n)
    for i in range(n):
        if not ref.finite[i]:
            out["nonfinite"][i] = 0.0 if np.isnan(R[i]).all() else np.inf
            continue
        if not H[i].any():
            out["zero"][i] = 0.0 if np.array_equal(R[i], np.eye(3)) else np.inf
            continue
        if not np.isfinite(R[i]).all():
            for k in ("orth", "det", "opt"):
                out[k][i] = np.inf
            continue
        orth, det, tr = _mp_metrics(ref.Hs[i], R[i])
        s1, s2, s3 = ref.sig[i]
        with mpmath.workdps(50):
            gap = float((mpmath.mpf(s1) + s2 + ref.d[i] * s3 - tr) / s1)
        out["orth"][i] = orth / (C_ORTH * U64)
        out["det"][i] = det / (C_DET * U64)
        # a rank-1 completion may turn the sigma_2 direction anywhere: it loses up to 2 sigma_2
        out["opt"][i] = max(gap, 0.0) / (C_OPT * U64 + (2 * s2 / s1 if ref.rank1[i] else 0.0))
        if np.isfinite(ref.kappa[i]):
            bound = C_ELEM * U64 * ref.kappa[i] + (0.0 if extra_elem is None else extra_elem[i])
            out["elem"][i] = np.abs(R[i] - ref.R[i]).max() / bound
        if ref.rank1[i]:
            out["rank1"][i] = np.abs(R[i] @ ref.u1[i] - ref.v1[i]).max() / (C_ELEM * U64)
    return out


def worst(ratios, mask=None):
    """max over every ratio (nan ignored) of the rows in `mask`."""
    m = 0.0
    for v in ratios.values():
        v = v if mask is None else v[mask]
        if v.size and not np.isnan(v).all():
            m = max(m, float(np.nanmax(v)))
    return m


def formation_bound(X, Y, ref: Ref):
    """Element bound on R from forming H in fp64 from fp32 points [n, k, 3] (centroid and sum of outer products):
    |dH_ij| <= (3k + 6) u sum_p (|a_pi| + M_x)(|c_pj| + M_y) with a, c the centred points and M the largest |coordinate|,
    and |dR| <= 2 |dH|_F / (sigma_2 + d sigma_3)."""
    X, Y = np.asarray(X, dtype=np.float64), np.asarray(Y, dtype=np.float64)
    k = X.shape[1]
    a, c = X - X.mean(1, keepdims=True), Y - Y.mean(1, keepdims=True)
    Mx, My = np.abs(X).max((1, 2))[:, None, None], np.abs(Y).max((1, 2))[:, None, None]
    dH = (3 * k + 6) * U64 * np.einsum("npi,npj->nij", np.abs(a) + Mx, np.abs(c) + My)
    dH = np.ldexp(dH, ref.shift[:, None, None])                # in the units of ref.sig
    den = ref.sig[:, 1] + ref.d * ref.sig[:, 2]
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(den > 0, 2.0 * np.linalg.norm(dH, axis=(1, 2)) / den, np.inf)


# ---------------------------------------------------------------------------------------------------------------
# the restatement (for planting mutations)
# ---------------------------------------------------------------------------------------------------------------
MUTATIONS = ("sweeps3", "h_fp32", "no_sign_fix", "no_reorth", "rank_tol_1e-6")


def kabsch_np(H, mutation=None):
    """kabsch_rotation restated over a batch [n, 3, 3] in numpy fp64, operation for operation; `mutation` plants one
    of MUTATIONS: the sweep cap at 3, H rounded to fp32 (as if accumulated in fp32), R = V U^T from LAPACK's factors
    without the sign fix, u_2 not re-orthogonalised against u_1, the rank-2 threshold moved from 1e-14 to 1e-6."""
    H = np.asarray(H, dtype=np.float64).reshape(-1, 3, 3)
    if mutation == "h_fp32":
        with np.errstate(over="ignore"):                     # the 2^500 and 2^1000 classes overflow fp32: inf
            H = H.astype(np.float32).astype(np.float64)
    if mutation == "no_sign_fix":
        U, _, Vt = np.linalg.svd(np.where(np.isfinite(H), H, 0.0))
        return np.swapaxes(Vt, 1, 2) @ np.swapaxes(U, 1, 2)
    n = H.shape[0]
    R = np.full((n, 3, 3), np.nan)
    finite = np.isfinite(H).reshape(n, 9).all(1)
    hmax = np.where(finite, np.abs(np.where(np.isfinite(H), H, 0.0)).reshape(n, 9).max(1), 0.0)
    R[finite & (hmax == 0)] = np.eye(3)
    ok = finite & (hmax > 0)
    _, ex = np.frexp(hmax[ok])
    A = np.ldexp(H[ok], (1 - ex)[:, None, None])
    m = A.shape[0]
    V = np.repeat(np.eye(3)[None], m, 0)
    done = np.zeros(m, dtype=bool)
    sweeps = 3 if mutation == "sweeps3" else 12
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for _ in range(sweeps):
            off = np.zeros(m)
            for p, q in ((0, 1), (0, 2), (1, 2)):
                al, be, ga = np.zeros(m), np.zeros(m), np.zeros(m)
                for i in range(3):
                    al = al + A[:, i, p] * A[:, i, p]
                    be = be + A[:, i, q] * A[:, i, q]
                    ga = ga + A[:, i, p] * A[:, i, q]
                sq = np.sqrt(al * be)
                rot = (np.abs(ga) > 1e-15 * sq) & (np.abs(ga) > 1e-300) & ~done
                off = np.where(rot, np.fmax(off, np.abs(ga) / np.fmax(sq, 1e-300)), off)
                zeta = (be - al) / (2.0 * ga)
                t = np.copysign(1.0, zeta) / (np.abs(zeta) + np.sqrt(1.0 + zeta * zeta))
                c = 1.0 / np.sqrt(1.0 + t * t)
                s = c * t
                c, s = c[:, None], s[:, None]
                ap, aq, vp, vq = A[:, :, p].copy(), A[:, :, q].copy(), V[:, :, p].copy(), V[:, :, q].copy()
                r = rot[:, None]
                A[:, :, p] = np.where(r, c * ap - s * aq, ap)
                A[:, :, q] = np.where(r, s * ap + c * aq, aq)
                V[:, :, p] = np.where(r, c * vp - s * vq, vp)
                V[:, :, q] = np.where(r, s * vp + c * vq, vq)
            done |= off < 1e-14
        sg = np.sqrt(A[:, 0] * A[:, 0] + A[:, 1] * A[:, 1] + A[:, 2] * A[:, 2])       # [m, 3] column norms
        ar = np.arange(m)
        i1 = np.zeros(m, dtype=int)
        i1 = np.where(sg[:, 1] > sg[ar, i1], 1, i1)
        i1 = np.where(sg[:, 2] > sg[ar, i1], 2, i1)
        i2, i3 = (i1 + 1) % 3, (i1 + 2) % 3
        sw = sg[ar, i3] > sg[ar, i2]
        i2, i3 = np.where(sw, i3, i2), np.where(sw, i2, i3)
        s1, s2 = sg[ar, i1], sg[ar, i2]
        u1 = A[ar, :, i1] / s1[:, None]
        v1, v2 = V[ar, :, i1], V[ar, :, i2]
        tol = 1e-6 if mutation == "rank_tol_1e-6" else RANK1_TOL
        full = s2 > tol * s1
        # rank >= 2: u2 = A[:, i2] / s2 re-orthogonalised against u1
        u2f = A[ar, :, i2] / s2[:, None]
        if mutation != "no_reorth":
            d = u1[:, 0] * u2f[:, 0] + u1[:, 1] * u2f[:, 1] + u1[:, 2] * u2f[:, 2]
            u2f = u2f - d[:, None] * u1
        nn = u2f[:, 0] * u2f[:, 0] + u2f[:, 1] * u2f[:, 1] + u2f[:, 2] * u2f[:, 2]
        u2f = u2f * (1.0 / np.sqrt(nn))[:, None]
        # rank 1: u2 = e_k - u1[k] u1 normalised, k the smallest |u1[k]| (first on ties)
        k = np.zeros(m, dtype=int)
        k = np.where(np.abs(u1[:, 1]) < np.abs(u1[ar, k]), 1, k)
        k = np.where(np.abs(u1[:, 2]) < np.abs(u1[ar, k]), 2, k)
        e = np.zeros((m, 3))
        e[ar, k] = 1.0
        u2r = e - u1[ar, k][:, None] * u1
        nn = u2r[:, 0] * u2r[:, 0] + u2r[:, 1] * u2r[:, 1] + u2r[:, 2] * u2r[:, 2]
        u2r = u2r * (1.0 / np.sqrt(nn))[:, None]
        u2 = np.where(full[:, None], u2f, u2r)

        def cross(a, b):
            return np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                             a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)

        u3, v3 = cross(u1, u2), cross(v1, v2)
        R[ok] = v1[:, :, None] * u1[:, None, :] + v2[:, :, None] * u2[:, None, :] + v3[:, :, None] * u3[:, None, :]
    return R


def per_class(table, kabsch_fn, refs=None):
    """{class: (worst ratio, ratios)} of kabsch_fn over the table; refs caches Ref per class."""
    out = {}
    for name, H in table.items():
        ref = refs[name] if refs is not None else Ref(H)
        r = check(H, kabsch_fn(H), ref)
        out[name] = (worst(r), r)
    return out
