"""The fp64 Kabsch rotation on the device, with the bounds of tests/kabsch_check.py:

- mk_op_kabsch (one kabsch_rotation per thread) on the whole case table, scale and non-finite classes included;
- the solver's hypotheses (hyp_Rt) on planted point sets whose fp32 back-projection the test knows bit for bit
  (K = diag(f, f, 1), f a power of two, cx = cy = 0: the kernel's point is fl32(z (u / f)), one rounding), with the
  triples injected, ill-conditioned ones included; the restated 3-sweep Jacobi must be rejected there too;
- the quaternion writer (mk_pose_to_submission through submission.pack_poses) on ~10^5 fp32 rotations near 0 and pi.
max(err / bound) per class is printed (pytest -s) and quoted in DESIGN §2.
"""

import mpmath
import numpy as np
import pytest
import torch

from mickey_b200 import _lib
from mickey_b200 import submission as mksub
from mickey_b200.config import mickey_cfg
from mickey_b200.model import MickeyRelativePose
from mickey_b200.weights import synthetic_state_dict
from tests import kabsch_check as kc
from tests.gpu_util import stream


pytestmark = pytest.mark.gpu
DEV = "cuda"
U, U32 = kc.U64, kc.U32


def op_kabsch(H):
    lib = _lib.load()
    Hd = torch.from_numpy(np.ascontiguousarray(np.asarray(H, dtype=np.float64).reshape(-1, 9))).to(DEV)
    Rd = torch.full_like(Hd, 7.0)
    _lib.check(lib.mk_op_kabsch(_lib.ptr(Hd), _lib.ptr(Rd), Hd.shape[0], stream()), "mk_op_kabsch")
    torch.cuda.synchronize()
    return Rd.cpu().numpy().reshape(-1, 3, 3)


def test_mk_op_kabsch_on_the_case_table():
    T = kc.case_table()
    res = {}
    for name, H in T.items():
        w, _ = kc.per_class({name: H}, op_kabsch)[name]
        res[name] = w
    print("\n[mk_op_kabsch] max(err / bound) per class: " + ", ".join(f"{k} {w:.2g}" for k, w in res.items()))
    bad = {k: w for k, w in res.items() if not w <= 1.0}
    assert not bad, bad


def test_mk_op_kabsch_rejects_bad_arguments():
    lib = _lib.load()
    H = torch.zeros(4, 9, dtype=torch.float64, device=DEV)
    for args in ((_lib.ptr(H), _lib.ptr(H), -1), (None, _lib.ptr(H), 4), (_lib.ptr(H), None, 4)):
        assert lib.mk_op_kabsch(*args, stream()) != 0
        assert b"kabsch" in lib.mk_last_error()
    assert lib.mk_op_kabsch(_lib.ptr(H), _lib.ptr(H), 0, stream()) == 0


# ---------------------------------------------------------------------------------------------------------------
# the solver's hypotheses on planted point sets
# ---------------------------------------------------------------------------------------------------------------
F = 512.0                                  # focal length, a power of two: K^-1 is exact
N_S = 2048
REUSED = 4096


def to_image(P):
    """fp32 (u, v, z) of 3D points P [n, 3] and the exact fp32 point the kernel back-projects: fl32(z (u / f))."""
    P = np.asarray(P, dtype=np.float64)
    z = P[:, 2].astype(np.float32)
    u = (P[:, 0] * F / P[:, 2]).astype(np.float32)
    v = (P[:, 1] * F / P[:, 2]).astype(np.float32)
    X = np.stack([z * (u / np.float32(F)), z * (v / np.float32(F)), z], 1)        # float32 ops: one rounding each
    return u, v, z, X.astype(np.float32)


def hypothesis_classes(seed=0, per=48):
    """{class: (X, Y) [n, 3, 3] 3D triples}; the triples the existing checks drop (sigma_2 < 1e-3 sigma_1) included.
    'rot_3rad' is an exact rotation by 3 rad: the class where a truncated sweep is most often wrong."""
    rng = np.random.default_rng(seed)
    out = {"noisy": kc.point_sets(rng, 2 * per, 3, "noisy"), "collinear": kc.point_sets(rng, per, 3, "collinear"),
           "coincident": kc.point_sets(rng, per, 3, "coincident"), "mirrored": kc.point_sets(rng, 2 * per, 3, "mirrored")}
    for rel in (1e-3, 1e-5, 1e-7):
        out[f"near_collinear_{rel:.0e}"] = kc.point_sets(rng, per, 3, "near_collinear", rel)
    X = rng.uniform(-1, 1, (2 * per, 3, 3)) + [0, 0, 4]
    R = kc.axis_angle(rng.standard_normal((2 * per, 3)), np.full(2 * per, 3.0))
    out["rot_3rad"] = (X.astype(np.float32), (X @ np.swapaxes(R, 1, 2) + [0.3, -0.2, 0.1]).astype(np.float32))
    return out


def exact_H(X, Y):
    """H of fp32 point sets [n, k, 3], formed in extended precision and rounded once to fp64."""
    X, Y = np.asarray(X, dtype=np.longdouble), np.asarray(Y, dtype=np.longdouble)
    a, c = X - X.mean(1, keepdims=True), Y - Y.mean(1, keepdims=True)
    return np.einsum("npi,npj->nij", a, c).astype(np.float64)


@pytest.fixture(scope="module")
def solved():
    classes = hypothesis_classes()
    names = list(classes)
    Xs = np.concatenate([classes[k][0] for k in names]).reshape(-1, 3)
    Ys = np.concatenate([classes[k][1] for k in names]).reshape(-1, 3)
    n_tri = Xs.shape[0] // 3
    assert Xs.shape[0] <= N_S
    rng = np.random.default_rng(1)
    fill = N_S - Xs.shape[0]
    Xs = np.concatenate([Xs, rng.uniform(-1, 1, (fill, 3)) + [0, 0, 4]])
    Ys = np.concatenate([Ys, rng.uniform(-1, 1, (fill, 3)) + [0, 0, 4]])
    u0, v0, z0, X32 = to_image(Xs)
    u1, v1, z1, Y32 = to_image(Ys)
    # 4096 more hypotheses from random triples of the rot_3rad block's points (a triple's points are distinct)
    off = 3 * sum(classes[k][0].shape[0] for k in names[:names.index("rot_3rad")])
    n_rot = 3 * classes["rot_3rad"][0].shape[0]
    extra = np.stack([rng.choice(n_rot, 3, replace=False) for _ in range(REUSED)]) + off
    tri = np.concatenate([np.arange(3 * n_tri).reshape(n_tri, 3), extra])
    IR = tri.shape[0]
    cfg = mickey_cfg("vits", 1, IR)
    model = MickeyRelativePose(cfg)
    model.load_state_dict(synthetic_state_dict(cfg, seed=3), strict=True)
    model = model.cuda().eval()
    N = N_S
    model._engine()._ws_for(1, 14 * 64, 14 * 32)                               # a 64 x 32 grid: N = 2048 keypoints
    K = torch.tensor([[[F, 0, 0], [0, F, 0], [0, 0, 1.0]]])
    batch = {"final_scores": torch.ones(1, N, N), "kps0": torch.from_numpy(np.stack([u0, v0]))[None],
             "kps1": torch.from_numpy(np.stack([u1, v1]))[None], "depth_kp0": torch.from_numpy(z0)[None, None],
             "depth_kp1": torch.from_numpy(z1)[None, None], "K_color0": K, "K_color1": K}
    batch = {k: v.to(DEV) for k, v in batch.items()}
    outer = (torch.arange(N_S) * (N + 1)).int()[None].to(DEV)                   # set position i = keypoint pair (i, i)
    inner = torch.from_numpy(tri).int().to(DEV)
    with torch.no_grad():
        model.e2e_Procrustes.estimate_pose_vectorized(batch, outer_idx=outer, inner_idx=inner, seed=5)
    torch.cuda.synchronize()
    Rt = model._engine().ws_view("hyp_Rt", torch.float32, (IR, 12)).double().cpu().numpy()
    cls = np.concatenate([[k] * classes[k][0].shape[0] for k in names] + [["rot_3rad_reused"] * REUSED])
    out = dict(Rt=Rt, X=X32[tri], Y=Y32[tri], cls=cls, names=names + ["rot_3rad_reused"])
    del model
    torch.cuda.empty_cache()
    return out


def hyp_ratios(R32, t32, X, Y):
    """err / bound of fp32 rotations and translations [n] for the fp32 triples X, Y [n, 3, 3]."""
    H = exact_H(X, Y)
    ref = kc.Ref(H)
    form = kc.formation_bound(X, Y, ref)
    n = len(H)
    r = np.zeros(n)
    Xl, Yl = np.asarray(X, dtype=np.longdouble), np.asarray(Y, dtype=np.longdouble)
    xm, ym = Xl.mean(1), Yl.mean(1)
    for i in range(n):
        R = R32[i]
        if not np.isfinite(R).all():
            r[i] = np.inf
            continue
        if not H[i].any():
            r[i] = 0.0 if np.array_equal(R, np.eye(3)) else np.inf
            continue
        # condition-free, with the fp32 store (9 entries each rounded by <= 2^-24 relative): within 12 * 2^-24
        s1, s2, s3 = ref.sig[i]
        orth = np.abs(R.T @ R - np.eye(3)).max() / (12 * U32)
        det = abs(np.linalg.det(R) - 1) / (12 * U32)
        gap = (s1 + s2 + ref.d[i] * s3 - float(np.sum(R.T * ref.Hs[i]))) / s1
        opt = max(gap, 0.0) / (12 * U32 + kc.C_OPT * U + (2 * s2 / s1 if ref.rank1[i] else 0.0))
        r[i] = max(orth, det, opt)
        if np.isfinite(ref.kappa[i]):
            eb = kc.C_ELEM * U * ref.kappa[i] + form[i]                       # the fp64 rotation's error
            r[i] = max(r[i], float((np.abs(R - ref.R[i]) / (U32 * np.abs(ref.R[i]) + eb)).max()))
            t_ref = ym[i] - ref.R[i].astype(np.longdouble) @ xm[i]
            tb = (U32 * np.abs(t_ref) + eb * np.abs(xm[i]).sum() + 8 * U * (np.abs(ym[i]) + np.abs(xm[i]).sum()))
            r[i] = max(r[i], float((np.abs(t32[i] - t_ref) / tb).max()))
        else:
            # ill-posed: t must still be the kernel's own R applied to the centroids
            t_own = ym[i] - R.astype(np.longdouble) @ xm[i]
            tb = U32 * (np.abs(t_own) + 2 * np.abs(xm[i]).sum()) + 8 * U * (np.abs(ym[i]) + np.abs(xm[i]).sum())
            r[i] = max(r[i], float((np.abs(t32[i] - t_own) / tb).max()))
    return r


def test_solver_hypotheses_on_planted_triples(solved):
    Rt, X, Y, cls = solved["Rt"], solved["X"], solved["Y"], solved["cls"]
    r = hyp_ratios(Rt[:, :9].reshape(-1, 3, 3), Rt[:, 9:], X, Y)
    per = {k: float(r[cls == k].max()) for k in solved["names"]}
    print("\n[solver hypotheses] max(err / bound) per class: " + ", ".join(f"{k} {w:.2g}" for k, w in per.items()))
    assert not {k: w for k, w in per.items() if not w <= 1.0}, per


def test_solver_hypothesis_bound_rejects_a_truncated_jacobi(solved):
    """The restated sweep capped at 3, with the kernel's own fp64 formation of H, rounded to fp32 like hyp_Rt."""
    X, Y, cls = solved["X"], solved["Y"], solved["cls"]
    H = kc.kernel_H(X, Y)
    Rm = kc.kabsch_np(H, "sweeps3")
    xm, ym = X.astype(np.float64).mean(1), Y.astype(np.float64).mean(1)
    tm = ym - np.einsum("nij,nj->ni", Rm, xm)
    r = hyp_ratios(Rm.astype(np.float32).astype(np.float64), tm.astype(np.float32).astype(np.float64), X, Y)
    rejected = {k: int((r[cls == k] > 1).sum()) for k in solved["names"]}
    print(f"\n[solver hypotheses, 3-sweep Jacobi] triples rejected per class: {rejected}")
    # a 3x3 sweep on a rank-2 triple converges fast: 3 sweeps leave ~1 % of the 3-rad rotations wrong
    assert rejected["rot_3rad"] + rejected["rot_3rad_reused"] >= 20, rejected


# ---------------------------------------------------------------------------------------------------------------
# the refinements: the solver's finalize_pair and the loss's search, on planted sets
# ---------------------------------------------------------------------------------------------------------------
def to_image_exact(P):
    """Like to_image, on a grid where z (u / f) is exact in fp32 (z = k / 16 with k < 2^7, u = m / 64 with |m| < 2^17),
    so that the fp64 oracle's back-projection equals the kernel's fp32 point bit for bit."""
    P = np.asarray(P, dtype=np.float64)
    z = np.clip(np.round(P[:, 2] * 16), 32, 127) / 16
    u = np.clip(np.round(P[:, 0] * F / z * 64), -(2 ** 17 - 1), 2 ** 17 - 1) / 64
    v = np.clip(np.round(P[:, 1] * F / z * 64), -(2 ** 17 - 1), 2 ** 17 - 1) / 64
    X = np.stack([z * (u / F), z * (v / F), z], 1)
    assert np.array_equal(X.astype(np.float32).astype(np.float64), X)
    return u.astype(np.float32), v.astype(np.float32), z.astype(np.float32), X


def planted_set(kind, n, rng):
    """3D correspondences (X, Y) [n, 3] of one refinement class; 40 % outliers are displaced by 0.5 .. 1 m.
    'coplanar': the inliers on a plane (rank-2 H over the full set); 'mirrored': Y = X reflected in a thin slab, so
    H has det < 0 and the sign fix decides R; 's2_eq_s3_neg': a rod whose two thin axes are equal and reflected,
    sigma_2 = sigma_3 with det < 0 (the optimum is not unique); 'growing': inliers with 0.06 m of noise, so the
    inlier set of a 3-point hypothesis grows over the refinements."""
    R = kc.axis_angle([[0.3, 1.0, 0.2]], [0.4])[0]
    t = np.array([0.3, -0.2, 0.25])
    if kind == "coplanar":
        a, b = rng.uniform(-1.5, 1.5, (2, n))
        X = np.stack([a, b, 4 + 0.3 * a - 0.2 * b], 1)
        Y = X @ R.T + t
    elif kind == "mirrored":
        X = np.stack([rng.uniform(-0.05, 0.05, n), rng.uniform(-1.5, 1.5, n), 4 + rng.uniform(-1, 1, n)], 1)
        Y = X * [-1.0, 1.0, 1.0] + t
    elif kind == "s2_eq_s3_neg":
        X = np.stack([rng.uniform(-1.5, 1.5, n), rng.uniform(-0.02, 0.02, n), 4 + rng.uniform(-0.02, 0.02, n)], 1)
        Y = X * [1.0, -1.0, 1.0] + t
    else:
        X = np.stack([rng.uniform(-1.5, 1.5, n), rng.uniform(-1.5, 1.5, n), 4 + rng.uniform(-1, 1, n)], 1)
        Y = X @ R.T + t + 0.06 * rng.standard_normal((n, 3))
    out = rng.random(n) < 0.4
    d = rng.standard_normal((n, 3))
    Y[out] += d[out] / np.linalg.norm(d[out], axis=1, keepdims=True) * rng.uniform(0.5, 1.0, (int(out.sum()), 1))
    return X, Y, ~out


REF_KINDS = ("coplanar", "mirrored", "s2_eq_s3_neg", "growing")


def _resid(X, Y, R, t):
    return np.sqrt(((X @ R.T + t - Y) ** 2).sum(1) + 1e-6)


def band(X, Y, t):
    """epsilon of the hard-inlier test: the kernel's fp32 residual of |R x + t - y| is within 16 * 2^-24 of
    (3 max|x| + |t| + max|y|) of the fp64 one (a handful of fp32 roundings of terms of that size)."""
    return 16 * U32 * (3 * np.abs(X).max() + np.abs(t).sum() + np.abs(Y).max())


def refine_fp64(X, Y, tri, th, n_ref):
    """finalize_pair in fp64 on exact points: the hypothesis of the triple, then up to n_ref refinements on the hard
    inliers.  Returns (R, t, mask, the final inlier set's H and its point indices, steps, smallest |th - dist| over every
    inlier test that decided the result)."""
    def fit(idx):
        H = exact_H(X[None, idx], Y[None, idx])
        R = kc.Ref(H).R[0]
        return R, Y[idx].mean(0) - R @ X[idx].mean(0), H[0]
    R, t, H = fit(tri)
    idx, prev, margin, steps = tri, 3.0, np.inf, 0
    for _ in range(n_ref):
        d = _resid(X, Y, R, t)
        margin = min(margin, np.abs(th - d).min())
        inl = np.flatnonzero(th - d >= 0)
        if not (len(inl) >= 3 and len(inl) > prev):
            break
        prev, idx, steps = len(inl), inl, steps + 1
        R, t, H = fit(inl)
    d = _resid(X, Y, R, t)
    return R, t, th - d >= 0, H, idx, steps, min(margin, np.abs(th - d).min())


@pytest.fixture(scope="module")
def refined():
    """One pair per class, one hypothesis per pair (the triple injected: three inliers), the outer set injected."""
    from oracle import mickey_oracle as mo
    rng = np.random.default_rng(11)
    B, N = len(REF_KINDS), N_S
    sets = [planted_set(k, N, rng) for k in REF_KINDS]
    img = [(to_image_exact(X), to_image_exact(Y)) for X, Y, _ in sets]
    tris = [np.flatnonzero(inl)[[0, 1, 2]] for _, _, inl in sets]
    cfg = mickey_cfg("vits", 1, 1)
    model = MickeyRelativePose(cfg)
    model.load_state_dict(synthetic_state_dict(cfg, seed=3), strict=True)
    model = model.cuda().eval()
    model._engine()._ws_for(B, 14 * 64, 14 * 32)
    kps0 = torch.from_numpy(np.stack([np.stack([a[0], a[1]]) for a, _ in img]))
    kps1 = torch.from_numpy(np.stack([np.stack([b[0], b[1]]) for _, b in img]))
    d0 = torch.from_numpy(np.stack([a[2] for a, _ in img]))[:, None]
    d1 = torch.from_numpy(np.stack([b[2] for _, b in img]))[:, None]
    K = torch.tensor([[[F, 0, 0], [0, F, 0], [0, 0, 1.0]]]).repeat(B, 1, 1)
    fs = torch.ones(B, N, N)
    outer = (torch.arange(N_S) * (N + 1)).repeat(B, 1)
    inner = torch.from_numpy(np.stack(tris)).long()
    batch = {k: v.to(DEV) for k, v in dict(final_scores=fs, kps0=kps0, kps1=kps1, depth_kp0=d0, depth_kp1=d1,
                                            K_color0=K, K_color1=K).items()}
    with torch.no_grad():
        R, t, _ = model.e2e_Procrustes.estimate_pose_vectorized(batch, outer_idx=outer.int().to(DEV),
                                                                 inner_idx=inner.int().to(DEV), seed=5)
    torch.cuda.synchronize()
    res = batch["_solver"]
    assert int(res["status"].item()) == 0
    mask = res["inlier_mask"].cpu().numpy() > 0.5
    Ro, to, _ = mo.solve_pose(fs.double(), kps0.double(), d0.double(), kps1.double(), d1.double(), K.double(),
                              K.double(), cfg, outer_idx=outer, inner_idx=inner)
    out = dict(R=R.double().cpu().numpy(), t=t.double().cpu().numpy().reshape(B, 3), mask=mask,
               Ro=Ro.double().numpy(), to=to.double().numpy().reshape(B, 3), X=[a[3] for a, _ in img],
               Y=[b[3] for _, b in img], tris=tris, cfg=cfg)
    del model
    torch.cuda.empty_cache()
    return out


def test_solver_refinement_on_planted_sets(refined):
    """finalize_pair's final R, t and hard-inlier mask against the fp64 oracle (solve_pose, both draws injected) and
    an fp64 restatement with a 50-digit rotation: |R - R_ref| <= 2^-24 |R_ref| + 2 (64 u kappa + formation), where the
    oracle's own fp64 rotation error takes the second share; t likewise through the centroid.  Where the optimum is
    not unique (kappa = inf) R is held to orthogonality and optimality on the final H.  The mask must be equal except
    for points within epsilon (band) of TH_INLIER; a hypothesis any of whose inlier tests was that close is reported."""
    p = refined["cfg"].PROCRUSTES
    th, n_ref = float(p.TH_INLIER), int(p.NUM_REFINEMENTS)
    report = {}
    for b, kind in enumerate(REF_KINDS):
        X, Y = refined["X"][b], refined["Y"][b]
        R_ref, t_ref, m_ref, H, idx, steps, margin = refine_fp64(X, Y, refined["tris"][b], th, n_ref)
        eps = band(X, Y, t_ref)
        R, t, mask = refined["R"][b], refined["t"][b], refined["mask"][b]
        Ro, to = refined["Ro"][b], refined["to"][b]
        # the hard mask: equal to the oracle's at its own final pose except inside the band
        d_o = _resid(X, Y, Ro, to)
        assert not ((mask != (th - d_o >= 0)) & (np.abs(th - d_o) > eps)).any(), (kind, eps)
        if margin <= eps:
            report[kind] = f"decided inside the band ({margin:.2g} <= {eps:.2g}): mask only"
            continue
        ref = kc.Ref(H[None])
        form = kc.formation_bound(X[None, idx], Y[None, idx], ref)[0]
        xm = np.abs(X[idx].mean(0)).sum()
        if np.isfinite(ref.kappa[0]):
            eb = 2 * (kc.C_ELEM * U * ref.kappa[0] + form)
            rR = float((np.abs(R - R_ref) / (U32 * np.abs(R_ref) + eb)).max())
            rO = float((np.abs(Ro - R_ref) / (eb / 2)).max())
            tb = U32 * np.abs(t_ref) + eb * xm + 16 * U * (np.abs(Y).max() + xm)
            rt = float((np.abs(t - t_ref) / tb).max())
            rtO = float((np.abs(to - t_ref) / tb).max())
            report[kind] = f"{steps} refinements, kappa {ref.kappa[0]:.3g}: R {rR:.2g} t {rt:.2g} (oracle R {rO:.2g} t {rtO:.2g})"
            assert max(rR, rt, rO, rtO) <= 1.0, (kind, report[kind])
        else:
            s1, s2, s3 = ref.sig[0]
            orth = np.abs(R.T @ R - np.eye(3)).max() / (12 * U32)
            gap = max(s1 + s2 + ref.d[0] * s3 - float(np.sum(R.T * ref.Hs[0])), 0.0) / s1 / (12 * U32 + kc.C_OPT * U)
            report[kind] = f"{steps} refinements, ill-posed: orthogonality {orth:.2g}, optimality {gap:.2g}"
            assert max(orth, gap) <= 1.0, (kind, report[kind])
        assert np.array_equal(mask, m_ref), kind
    print("\n[solver refinement] " + "; ".join(f"{k}: {v}" for k, v in report.items()))
    assert "growing" in report and not report["growing"].startswith(("0 ", "1 "))


@pytest.mark.parametrize("C", [3, 4, 8, 16])
def test_loss_refinement_on_planted_sets(C):
    """mk_loss_search with both draws injected, S = 256, one outer set per class: inliers_final must equal
    oracle/loss_oracle.refine in fp64 on the same exact points, except for hypotheses whose deciding inlier tests came
    within epsilon (band) of INLIER_REF_TH (the oracle's margin)."""
    from mickey_b200.loss import LossParams, loss_search
    from oracle import loss_oracle
    from tests import loss_cases
    S, IR = 256, 64
    p = LossParams(loss_cases.loss_cfg(it_matches=len(REF_KINDS), it_ransac=IR))
    p.n_sample, p.num_corr = S, C
    IM = len(REF_KINDS)
    N = IM * S
    rng = np.random.default_rng(20 + C)
    Xs, Ys, inner, eps = [], [], [], []
    for s, kind in enumerate(REF_KINDS):
        X, Y, inl = planted_set(kind, S, rng)
        (u0, v0, z0, X), (u1, v1, z1, Y) = to_image_exact(X), to_image_exact(Y)
        Xs.append((u0, v0, z0, X)); Ys.append((u1, v1, z1, Y))
        good = np.flatnonzero(inl)
        inner.append(np.stack([rng.choice(good, C, replace=False) for _ in range(IR)]))
        eps.append(band(X, Y, np.array([0.3, 0.2, 0.25])))
    cat = lambda L, i: np.concatenate([a[i] for a in L])
    kps0 = torch.from_numpy(np.stack([cat(Xs, 0), cat(Xs, 1)]))[None]
    kps1 = torch.from_numpy(np.stack([cat(Ys, 0), cat(Ys, 1)]))[None]
    d0, d1 = torch.from_numpy(cat(Xs, 2))[None, None], torch.from_numpy(cat(Ys, 2))[None, None]
    K = torch.tensor([[[F, 0, 0], [0, F, 0], [0, 0, 1.0]]])
    outer = torch.stack([(torch.arange(S) + s * S) * (N + 1) for s in range(IM)])
    inner_t = torch.from_numpy(np.concatenate(inner)).long()
    fs = torch.ones(1, N, N)
    _, _, inl_k, status = loss_search(fs.to(DEV), kps0.to(DEV), d0.to(DEV), kps1.to(DEV), d1.to(DEV), K.to(DEV),
                                      K.to(DEV), p, 7, outer.to(DEV), inner_t.to(DEV))
    assert status == 0, status
    inl_k = inl_k.cpu().numpy()
    report = {}
    for s, kind in enumerate(REF_KINDS):
        X = torch.from_numpy(Xs[s][3])[None].expand(IR, S, 3)
        Y = torch.from_numpy(Ys[s][3])[None].expand(IR, S, 3)
        ref, margin = loss_oracle.refine(X, Y, torch.from_numpy(inner[s]).long(), p)
        got = inl_k[s * IR:(s + 1) * IR]
        differ = (got != ref.numpy()).any(1)
        excused = margin.numpy() <= eps[s]
        assert not (differ & ~excused).any(), (kind, C, np.flatnonzero(differ & ~excused)[:5])
        report[kind] = f"{int(differ.sum())} differ / {int(excused.sum())} in band / mean |final| {ref.sum(1).mean():.0f}"
    print(f"\n[loss refinement C={C}] " + "; ".join(f"{k}: {v}" for k, v in report.items()))


# ---------------------------------------------------------------------------------------------------------------
# the quaternion writer
# ---------------------------------------------------------------------------------------------------------------
def quat_classes(seed=0, per=8192):
    rng = np.random.default_rng(seed)
    ax = rng.standard_normal((per, 3))
    coord = np.eye(3)[rng.integers(0, 3, per)] * rng.choice([-1.0, 1.0], (per, 1))
    out = {}
    for nm, ang in (("angle_0", 0.0), ("angle_1e-8", 1e-8), ("angle_1e-4", 1e-4)):
        out[nm] = kc.axis_angle(ax, np.full(per, ang))
    out["random"] = kc.rand_rot(rng, 4 * per)
    for dlt in (1e-8, 1e-6, 1e-4, 1e-2):
        out[f"pi-{dlt:.0e}"] = kc.axis_angle(ax, np.full(per, np.pi - dlt))
        out[f"pi-{dlt:.0e}_coord"] = kc.axis_angle(coord, np.full(per, np.pi - dlt))
    return out


def refined_quaternion(R):
    """Principal eigenvector (x, y, z, w -> returned as w, x, y, z) of transforms3d's K(R), from fp64 eigh refined by
    one first-order correction in numpy's long double, sign fixed so that w >= 0.  long double is 80-bit on x86-64 and
    128-bit on aarch64; either way the correction leaves an error far below u, which `mp_quaternion` checks at 50
    digits on a sample of every class."""
    R = np.asarray(R, dtype=np.float64)
    Qxx, Qyx, Qzx, Qxy, Qyy, Qzy, Qxz, Qyz, Qzz = [R.reshape(-1, 9)[:, k] for k in range(9)]
    K = np.zeros((R.shape[0], 4, 4), dtype=np.longdouble)
    L = lambda v: np.asarray(v, dtype=np.longdouble)
    K[:, 0, 0] = (L(Qxx) - L(Qyy) - L(Qzz)) / 3
    K[:, 1, 1] = (L(Qyy) - L(Qxx) - L(Qzz)) / 3
    K[:, 2, 2] = (L(Qzz) - L(Qxx) - L(Qyy)) / 3
    K[:, 3, 3] = (L(Qxx) + L(Qyy) + L(Qzz)) / 3
    K[:, 0, 1] = K[:, 1, 0] = (L(Qyx) + L(Qxy)) / 3
    K[:, 0, 2] = K[:, 2, 0] = (L(Qzx) + L(Qxz)) / 3
    K[:, 1, 2] = K[:, 2, 1] = (L(Qzy) + L(Qyz)) / 3
    K[:, 0, 3] = K[:, 3, 0] = (L(Qyz) - L(Qzy)) / 3
    K[:, 1, 3] = K[:, 3, 1] = (L(Qzx) - L(Qxz)) / 3
    K[:, 2, 3] = K[:, 3, 2] = (L(Qxy) - L(Qyx)) / 3
    lam, Q = np.linalg.eigh(K.astype(np.float64))
    lam, Q = lam.astype(np.longdouble), Q.astype(np.longdouble)
    q = Q[:, :, 3]
    res = np.einsum("nij,nj->ni", K, q) - lam[:, 3, None] * q
    for j in range(3):
        qj = Q[:, :, j]
        q = q - (np.einsum("ni,ni->n", qj, res) / (lam[:, j] - lam[:, 3]))[:, None] * qj
    q = q / np.sqrt((q * q).sum(1, keepdims=True))
    q = np.concatenate([q[:, 3:], q[:, :3]], 1)
    q = np.where(q[:, :1] < 0, -q, q)
    return q.astype(np.float64), (lam[:, 3] - lam[:, 2]).astype(np.float64)


def mp_quaternion(R):
    """The same eigenvector at 50 digits (mpmath.eigsy), w >= 0."""
    Rm = [[mpmath.mpf(float(x)) for x in row] for row in np.asarray(R, dtype=np.float64)]
    (Qxx, Qyx, Qzx), (Qxy, Qyy, Qzy), (Qxz, Qyz, Qzz) = Rm                # transforms3d names M.flat so
    K = mpmath.matrix([[Qxx - Qyy - Qzz, Qyx + Qxy, Qzx + Qxz, Qyz - Qzy],
                       [Qyx + Qxy, Qyy - Qxx - Qzz, Qzy + Qyz, Qzx - Qxz],
                       [Qzx + Qxz, Qzy + Qyz, Qzz - Qxx - Qyy, Qxy - Qyx],
                       [Qyz - Qzy, Qzx - Qxz, Qxy - Qyx, Qxx + Qyy + Qzz]]) / 3
    E, Q = mpmath.eigsy(K)
    k = max(range(4), key=lambda i: E[i])
    q = [Q[3, k], Q[0, k], Q[1, k], Q[2, k]]
    sgn = -1 if q[0] < 0 else 1
    return np.array([float(sgn * c) for c in q])


def test_quaternion_writer_against_extended_precision():
    C_Q = 64.0
    classes = quat_classes()
    names = list(classes)
    R = np.concatenate([classes[k] for k in names]).astype(np.float32)
    cls = np.concatenate([[k] * len(classes[k]) for k in names])
    n = len(R)
    special = np.zeros((4, 3, 3), dtype=np.float32)                      # zero pose, NaN in R, inf and NaN in t
    special[1:] = np.eye(3, dtype=np.float32)
    special[1, 1, 2] = np.nan
    R_all = np.concatenate([R, special])
    t = np.random.default_rng(2).standard_normal((n + 4, 1, 3)).astype(np.float32)
    t[n] = 0
    t[n + 2, 0, 1] = np.inf
    t[n + 3, 0, 0] = np.nan
    inl = np.random.default_rng(3).uniform(0, 500, (n + 4, 1)).astype(np.float32)
    rec = mksub.poses_to_records(mksub.pack_poses(torch.from_numpy(R_all).to(DEV), torch.from_numpy(t).to(DEV),
                                                  torch.from_numpy(inl).to(DEV)))
    assert rec[n, 8] == 1.0 and rec[n + 1, 8] == 0.0 and rec[n + 2, 8] == 0.0 and rec[n + 3, 8] == 0.0
    assert (rec[:n, 8] == 1.0).all()
    q_ref, gap = refined_quaternion(R.astype(np.float64))
    with mpmath.workdps(50):                                              # the reference itself, on 16 rows per class
        for k in names:
            rows = np.flatnonzero(cls == k)[:: max(1, int((cls == k).sum()) // 16)]
            for i in rows:
                qm = mp_quaternion(R[i])
                if abs(qm[0]) > 1e-12:                                    # w ~ 0: the sign of q is free
                    assert np.abs(q_ref[i] - qm).max() <= 2 * U, (k, i, q_ref[i], qm)
    assert gap.min() > 1.0                                                # K(R)'s eigen-gap is ~4/3
    q = rec[:n, :4]
    bound = C_Q * U
    err = np.abs(q - q_ref).max(1)
    near0 = np.abs(q_ref[:, 0]) <= bound                                  # w ~ 0: the whole quaternion's sign is free
    err = np.where(near0, np.minimum(err, np.abs(q + q_ref).max(1)), err)
    per = {k: float(err[cls == k].max() / bound) for k in names}
    print("\n[quaternion writer] max(err / bound) per class: " + ", ".join(f"{k} {w:.2g}" for k, w in per.items()))
    assert not {k: w for k, w in per.items() if not w <= 1.0}, per
    # the text: the Python writer's formatting of the reference quaternion, except within the bound of a 6-decimal
    # rounding boundary
    names_img = [f"s/frame_{i:06}.jpg" for i in range(n + 4)]
    ours = [str(p) for p in mksub.records_to_poses(rec, names_img)]
    valid = [i for i in range(n + 4) if rec[i, 8] != 0.0]
    assert len(ours) == len(valid) == n + 1
    ref_rec = rec.copy()
    ref_rec[:n, :4] = q_ref
    theirs = [str(p) for p in mksub.records_to_poses(ref_rec, names_img)]
    frac = np.abs(q_ref * 1e6 - np.floor(q_ref * 1e6) - 0.5) * 1e-6
    # a component within the bound of 0 may print as 0.000000 or -0.000000: zero is a boundary of the sign
    boundary = (frac <= 2 * bound).any(1) | (np.abs(q_ref) <= bound).any(1)
    diff = [i for i in range(n) if ours[i] != theirs[i]]
    assert all(boundary[i] or near0[i] for i in diff), [(ours[i], theirs[i], rec[i, :4].tolist(), q_ref[i].tolist())
                                                        for i in diff if not (boundary[i] or near0[i])][:3]
    print(f"[quaternion writer] {n} rotations, {len(diff)} lines differ from the extended-precision writer "
          f"(all within the bound of a rounding boundary or at w ~ 0)")
