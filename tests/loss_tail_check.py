"""The CUDA loss tail (csrc/loss_tail.cu, LossTail) element by element against the fp64 closed form
(oracle/loss_tail_oracle.py tail_closed_form) on the kernel's own fp32 inputs and fp32 K^-1, with a derived bound, and
a planted harness that builds the tail's inputs directly (drawn cells and inlier bit words), bypassing the search.

Notation: u = 2^-53; for a set of S entries the summation depth n_d = S/32 + 5 (the kernel: lane-strided partial sums,
then a butterfly) + log2(S) + 8 (torch's pairwise reductions, plus the few products that form each term); C_E = 16.
Per hypothesis h with H = U diag(sigma) V^T, d = sign det, kappa_h = sigma_1 / (sigma_2 + d sigma_3) (M's smallest
|eigenvalue| is sigma_2 + d sigma_3: M = tr(P) I - P has eigenvalues l_j + l_k of the signed singular values l).

The oracle sees exactly the kernel's inputs: the fp32 leaves, K^-1 rounded to fp32 (asserted round-safe), the fp32 VCRE
grid, the fp32 upstream gradients and the fp32 loss parameters (kernel_params).  Then, for every fp32 output element y with oracle value y*:   |y - y*| <= 2^-24 |y*| + E(y)

- The pose.  H and the means are sums of S terms formed from the same fp32 inputs by both sides, each with error
  <= n_d u times the sum of the terms' magnitudes; the Kabsch rotation turns a relative perturbation e of H into
  kappa e of R (tests/kabsch_check.py), and t = b - R a follows.  So R and t carry a relative error
      pi_h = C_E u n_d (1 + kappa_h).
- The hypothesis's losses and backward coefficients.  G_H = -R^T [M^-1 g]x takes one more factor kappa (M^-1 on a
  perturbed M); acos(c) and its derivative -1/sqrt(1 - c^2) turn an error in c into 1 / (1 - c^2) times it (inside
  the clip; 1 outside); a VCRE projection x / z turns a relative error of res into (1 + (|res_x| + |res_y|) / |res_z|)^2
  times it (value and derivative; this is the 1 / z^2 of the behind-the-camera and grazing points):
      rho_h = pi_h (1 + kappa_h) (1 + a_h) v_h,   a_h = 1 / (1 - c_h^2) inside the clip, 0 outside, v_h that factor.
- The softmaxes.  A score's error is u n_d S plus its sensitivity to the pose, pi_h k5 sum_i sg_i (1 - sg_i)
  (|X_i| + |Y_i| + |t|) (the oracle's `score_sens`); divided by |T| it is an error tau_s of the logits, and every softmax
  weight of the set carries a relative error omega_s = expm1(2 C_E tau_s).
- Values (per set): loss_value charges sum_h q_h (rho_h L_h + omega_s (|lv_h| + |loss_value|)) + omega_s q_null
  (|null loss| + |loss_value|) + C_E u n_d sum |terms|, with L_h the magnitude lv is formed from (|lv_h| plus 1440 px
  for VCRE, pi + |t| + |tgt| for POSE_ERR, times the tanh slope when soft); loss_rot and loss_trans likewise with sm
  and pi + |lr_h|, |lt_h| + |t| + |tgt|.
- Gradients (per keypoint element): each (hypothesis, entry) term of dX / dY -- w G_H (Y - b), w g_a / W1, c R^T r and
  their dY counterparts -- is charged (rho_h + omega_s + C_E u n_d) times its magnitude, formed with absolute values
  throughout (|G_H| <= |R|^T |[y]x| with |y| <= |g|_2 / (sigma_2 + d sigma_3), |g| from |G_R| |R|^T and |G_R| from every
  term's |.|, and the score's dL/dscore as q (|lv_h| + |loss_value|) / |T|), so cancellation across hypotheses, entries
  and outer iterations is paid for; then through |K^-1| and |z| and summed over the keypoint's draws, as the values are.
  The score's direct term c R^T r adds 2 pi_h |c| (2 + k5 d) (|X| + |Y| + |t|) (the oracle's `cres`): the residual r is
  a difference of O(|X|) terms and carries pi_h (|X| + |Y| + |t|) absolutely however small it is, and c = k5 dL/dscore
  sg (1 - sg) / d moves by (k5 + 1/d) per unit of d; the means enter G_H (Y - b) as |Y - b| + |b|.

A hypothesis with kappa > 1e12 is ill-posed: its set is left out of the value comparison (tests on the degenerate
contract cover it).  The random-perturbation probe `probe_ratio` (inputs moved by 2^-46 relative, the oracle's change
divided by 128 E) is a cross-check of E's shape; it is expected well below 1.
"""
from __future__ import annotations

import copy
import math

import numpy as np
import torch

from mickey_b200.loss import LossParams
from oracle import loss_tail_oracle as lto
from tests import loss_cases

U64 = 2.0 ** -53
U32 = 2.0 ** -24
C_E = 16.0
KAPPA_ILL = 1e12
QUANTITIES = ("loss_value", "loss_rot", "loss_trans", "dkps0", "ddepth0", "dkps1", "ddepth1")


def kernel_params(p: LossParams) -> LossParams:
    """p with the parameters the C ABI takes as fp32 rounded to fp32: INLIER_3D_TH, SCORE_TEMPERATURE, the null
    hypothesis's loss and score (TH_OUTLIERS * S).  A far outlier's sigmoid exp(-5/th (d - th)) turns th's fp32 rounding
    into ~1e-6 of its value, so the oracle must see the kernel's parameters, not the config's."""
    f32 = lambda x: float(np.float32(x))
    q = copy.copy(p)
    q.inlier_3d_th, q.score_temperature, q.max_loss_null = f32(p.inlier_3d_th), f32(p.score_temperature), f32(p.max_loss_null)
    q.th_outliers = f32(p.th_outliers * p.n_sample) / p.n_sample
    return q


def depth_n(S):
    return S / 32 + 5 + math.log2(S) + 8


def kinv_is_safe(K):
    """True when no element of the exact inverse of the fp32 K lies within 2^-40 relative of an fp32 rounding midpoint:
    then the kernel's fp64 inverse (inv3x3) rounds to the same fp32 bits as the oracle's."""
    Ki = torch.linalg.inv(K.double()).reshape(-1)
    f = Ki.float().double()
    ulp = torch.nextafter(f.float(), torch.full_like(f.float(), float("inf"))).double() - f
    frac = ((Ki - f) / ulp).abs()                       # 0.5 at a midpoint
    return bool(((frac - 0.5).abs() * ulp > 2.0 ** -40 * Ki.abs()).all())


def kappas(out):
    """Per hypothesis kappa = sigma_1 / |lambda_min(M)| (inf for H = 0 or rank 1)."""
    s1 = torch.linalg.svdvals(out["H"])[:, 0]
    lam = out["mag"]["lam"]
    k = torch.where(lam > 0, s1 / lam.clamp_min(1e-300), torch.full_like(s1, float("inf")))
    return torch.where(s1 > 0, k, torch.full_like(s1, float("inf")))


def bounds(out, p: LossParams, tgt):
    """{quantity: E} (without the 2^-24 |y*| store term) and the per-hypothesis kappa, from an oracle result."""
    m = out["mag"]
    S, IR = p.n_sample, p.it_ransac
    nd = depth_n(S)
    kap = kappas(out)
    kf = torch.where(torch.isfinite(kap), kap, torch.zeros_like(kap))
    pi = C_E * U64 * nd * (1 + kf)
    a = torch.where(m["inside"], 1 / (1 - m["cos"] ** 2), torch.zeros_like(m["cos"]))
    rho = pi * (1 + kf) * (1 + a) * m["vamp"]
    sets = rho.numel() // IR
    tau = ((U64 * nd * S + pi * m["score_sens"]).reshape(sets, IR).amax(1) / abs(p.score_temperature))
    omega = torch.expm1(2 * C_E * tau)                                            # [sets]
    rho2 = rho.reshape(sets, IR)
    B = tgt.shape[0]
    tmag = (m["t"].abs().sum(-1) + tgt.reshape(B, 3).abs().sum(-1).repeat_interleave(sets // B * IR)).reshape(sets, IR)
    slope_v = (1 / 80 if p.loss_type == "VCRE" else 1 / 0.9) if p.soft_clipping else 1.0
    L = m["lv"].abs() + slope_v * (1440.0 if p.loss_type == "VCRE" else math.pi + tmag)
    E = {}
    q, sm = m["q"], m["sm"]
    lv_s = out["loss_value"].abs()[:, None]
    E["loss_value"] = ((q * (rho2 * L + omega[:, None] * (m["lv"].abs() + lv_s))).sum(1)
                       + C_E * U64 * nd * (q * m["lv"].abs()).sum(1))
    if m["qn"] is not None:
        E["loss_value"] = E["loss_value"] + (omega + C_E * U64 * nd) * m["qn"] * (abs(p.max_loss_null) + lv_s[:, 0])
    for k, mag in (("loss_rot", math.pi + m["lr"].abs()), ("loss_trans", m["lt"].abs() + tmag)):
        o = out[k].abs()[:, None]
        E[k] = (sm * (rho2 * mag + omega[:, None] * (mag + o))).sum(1) + C_E * U64 * nd * (sm * mag).sum(1)
    # gradients: every term weighted by its hypothesis's relative error, then the magnitudes' back-projection and scatter
    wgt = (rho2 + omega[:, None] + C_E * U64 * nd).reshape(-1)[:, None, None]
    N = out["dkps0"].shape[2]
    res = (2 * pi[:, None] * m["cres"]).unsqueeze(-1)
    for img, T in (("0", m["TX"]), ("1", m["TY"])):
        dk, dd = lto.scatter_entries(T * wgt + res, m["sets"][int(img)], m["bidx"], B, N, IR, absolute=True)
        E["dkps" + img], E["ddepth" + img] = dk, dd
    return E, kap


def compare(got, out, p: LossParams, tgt, label="", mutations_ok=False):
    """max(err / bound) per quantity of the kernel's fp32 outputs `got` ({quantity: tensor}) against the oracle `out`.
    Sets with an ill-posed hypothesis (kappa > 1e12) are left out.  Asserts every ratio <= 1 unless mutations_ok, with a
    message naming the pair, the outer iteration, the keypoint and the worst kappa of the set."""
    E, kap = bounds(out, p, tgt)
    IM, IR = p.it_matches, p.it_ransac
    kset = kap.reshape(-1, IR).amax(1)
    ok_set = kset <= KAPPA_ILL
    B = out["dkps0"].shape[0]
    ratios, fails = {}, []
    for k in QUANTITIES:
        want = out[k].double()
        g = got[k].detach().double().cpu().reshape(want.shape)
        bound = U32 * want.abs() + E[k]
        err = (g - want).abs()
        r = torch.where(err == 0, torch.zeros_like(err), err / bound.clamp_min(1e-300))
        r = torch.where(torch.isfinite(g), r, torch.full_like(r, float("inf")))
        if k.startswith("loss"):
            r = torch.where(ok_set, r, torch.zeros_like(r))
        else:
            ill_pairs = (~ok_set).reshape(B, IM).any(1)
            r = torch.where(ill_pairs.reshape(B, *([1] * (r.dim() - 1))), torch.zeros_like(r), r)
        raw = r
        ratios[k] = float(r.max()) if r.numel() else 0.0
        if not ratios[k] <= 1:
            idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(int(r.reshape(-1).argmax())), r.shape))
            if k.startswith("loss"):
                s = idx[0]
                where = f"pair {s // IM}, outer iteration {s % IM}, kappa {float(kset[s]):.3g}"
            else:
                b, n = idx[0], idx[-1]
                where = f"pair {b}, keypoint {n}, component {idx[1]}, worst kappa in the pair {float(kset.reshape(B, IM)[b].max()):.3g}"
            fails.append(f"{label} {k}: {int((r > 1).sum())} elements out; worst {float(raw.reshape(-1)[int(r.reshape(-1).argmax())]):.3g} "
                         f"at {where}: got {float(g[idx]):.9g}, want {float(want[idx]):.9g}, bound {float(bound[idx]):.3g}")
    if not mutations_ok:
        assert not fails, "\n".join(fails)
    return ratios, fails


def probe_ratio(args, p, ups, Kinv, seed=0, rel=2.0 ** -46):
    """max over the gradient elements of |oracle(inputs (1 + rel xi)) - oracle(inputs)| / (128 E): the change of the
    oracle under a perturbation 2^7 times u, against the bound's rounding term E (the 2^-24 store term left out)."""
    kps0, d0, kps1, d1 = args[:4]
    p = kernel_params(p)
    base = lto.tail_closed_form(*args, p, *ups, Kinv=Kinv, grid=KERNEL_GRID)
    E, kap = bounds(base, p, args[9])
    g = torch.Generator().manual_seed(seed)
    pert = [x * (1 + rel * (2 * torch.rand(x.shape, generator=g, dtype=x.dtype) - 1)) for x in (kps0, d0, kps1, d1)]
    moved = lto.tail_closed_form(*pert, *args[4:], p, *ups, Kinv=Kinv, grid=KERNEL_GRID)
    worst = 0.0
    for k in ("dkps0", "ddepth0", "dkps1", "ddepth1"):
        r = (moved[k] - base[k]).abs() / (E[k] * (rel / U64)).clamp_min(1e-300)
        worst = max(worst, float(r[E[k] > 0].max()) if bool((E[k] > 0).any()) else 0.0)
    return worst


# ---------------------------------------------------------------------------------------------------------------
# planted problems
# ---------------------------------------------------------------------------------------------------------------
KERNEL_GRID = lto.vcre_grid().float().double()          # the kernel reads MetricPoseLoss's fp32 grid
K_PIN = torch.tensor([[600.0, 0.0, 360.0], [0.0, 600.0, 270.0], [0.0, 0.0, 1.0]], dtype=torch.float32)


def rot(axis, ang):
    axis = np.asarray(axis, dtype=np.float64)
    axis = axis / np.linalg.norm(axis)
    Kx = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + math.sin(ang) * Kx + (1 - math.cos(ang)) * (Kx @ Kx)


def gt_pose():
    return rot([0.2, 1.0, 0.1], math.radians(12.0)), np.array([0.25, -0.1, 0.22])


def whitened(rng, k):
    """k points [k, 3] with zero mean and identity covariance (exactly, to fp64 rounding)."""
    z = rng.standard_normal((k, 3))
    z = z - z.mean(0)
    L = np.linalg.cholesky(z.T @ z / k)
    return z @ np.linalg.inv(L).T


def group_points(rng, k, kind, rel=0.0, gap=0.0):
    """k 3-D points in camera 0 of one kind: 'well' (a box 1.5-4 m in front), 'coplanar', 'near_collinear' (off a line
    by rel of its length), 'gap' (covariance eigenvalues 1, 0.5, 0.5 (1 - gap): sigma_2 ~ sigma_3 for a mirror)."""
    c = np.array([0.0, 0.0, 2.6])
    if kind == "near_collinear":
        d = rng.standard_normal(3)
        d /= np.linalg.norm(d)
        return c + rng.uniform(-0.8, 0.8, (k, 1)) * d + rel * 0.8 * rng.standard_normal((k, 3))
    if kind == "coplanar":
        e1, e2 = rng.standard_normal(3), rng.standard_normal(3)
        return c + rng.uniform(-0.5, 0.5, (k, 1)) * e1 + rng.uniform(-0.5, 0.5, (k, 1)) * e2
    if kind == "gap":
        Q = rot(rng.standard_normal(3), rng.uniform(0, math.pi))
        s = np.sqrt(np.array([1.0, 0.5, 0.5 * (1 - gap)])) * 0.3
        return c + (whitened(rng, k) * s) @ Q.T
    return c + rng.uniform(-1, 1, (k, 3)) * np.array([0.8, 0.6, 0.8])


class Planted:
    """A tail problem built directly: B pairs, N keypoints, IM sets of S entries, IR hypotheses per set.  Entry (set s,
    entry j) of pair b uses its own keypoint perm_b[s S + j] in both images (cell k N + k), so every set's geometry is
    free; keypoints past IM S are drawn by none.  `fill(b, s)` returns (X [S, 3] in camera 0, Y [S, 3] in camera 1,
    inlier bits [IR, S] bool)."""

    def __init__(self, B, N, IM, IR, S, fill, seed=0, loss="VCRE", soft=True, null=True, T=None, gt=None):
        assert IM * S <= N
        self.rng = np.random.default_rng(seed)
        cfg = loss_cases.loss_cfg(loss, soft, null, it_matches=IM, it_ransac=IR)
        cfg.LOSS_CLASS.SAMPLER.NUM_SAMPLES_MATCHES = S
        if T is not None:
            cfg.LOSS_CLASS.GENERATE_HYPOTHESES.SCORE_TEMPERATURE = T
        self.p = p = LossParams(cfg)
        Rgt, tgt = gt or gt_pose()
        self.Rgt, self.tgt = Rgt, tgt
        K = K_PIN.numpy().astype(np.float64)
        kps0, kps1 = np.zeros((B, 2, N)), np.zeros((B, 2, N))
        d0, d1 = np.ones((B, 1, N)), np.ones((B, 1, N))
        for arr in (kps0, kps1):
            arr[:] = self.rng.uniform(0, 700, arr.shape)
        sampled = np.zeros((B * IM, S), dtype=np.int64)
        bits = np.zeros((B * IM * IR, S), dtype=bool)
        for b in range(B):
            perm = self.rng.permutation(N)
            for s in range(IM):
                X, Y, w = fill(self, b, s)
                ks = perm[s * S:(s + 1) * S]
                for P, kp, dp in ((X, kps0, d0), (Y, kps1, d1)):
                    x = P @ K.T
                    kp[b, 0, ks], kp[b, 1, ks] = x[:, 0] / x[:, 2], x[:, 1] / x[:, 2]
                    dp[b, 0, ks] = P[:, 2]
                sampled[b * IM + s] = ks * N + ks
                bits[(b * IM + s) * IR:(b * IM + s + 1) * IR] = w
        f = lambda a: torch.from_numpy(np.ascontiguousarray(a)).float()
        self.kps0, self.d0, self.kps1, self.d1 = f(kps0), f(d0), f(kps1), f(d1)
        self.K = K_PIN.expand(B, 3, 3).contiguous()
        T4 = np.tile(np.eye(4), (B, 1, 1))
        T4[:, :3, :3], T4[:, :3, 3] = Rgt, tgt
        self.T = f(T4)
        self.sampled = torch.from_numpy(sampled).int()
        self.inl = torch.from_numpy(bits.astype(np.float64))
        self.B, self.N = B, N

    @staticmethod
    def pack(inl, S):
        """{0,1} [H, S] -> int32 bit words [H, S/32] (mk_loss_search's layout)."""
        w = inl.to(torch.int64).reshape(inl.shape[0], S // 32, 32) << torch.arange(32)
        w = w.sum(-1)
        return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)

    def oracle(self, ups, mutation=None):
        """The fp64 closed form on the fp32 inputs and the kernel's K^-1."""
        Kd = self.K.double()
        T = self.T.double()
        Kinv = (lto.kernel_kinv(self.K), lto.kernel_kinv(self.K))
        return lto.tail_closed_form(self.kps0.double(), self.d0.double(), self.kps1.double(), self.d1.double(), Kd, Kd,
                                    Kd, Kd, T[:, :3, :3], T[:, :3, 3:].transpose(1, 2), self.sampled, self.inl,
                                    kernel_params(self.p), *ups, mutation=mutation, Kinv=Kinv, grid=KERNEL_GRID)

    def tgt_t(self):
        return self.T.double()[:, :3, 3:].transpose(1, 2)

    def upstream(self, seed=1):
        """Upstream gradients of the three outputs, fp32 values (what LossTail.backward hands the kernel)."""
        g = torch.Generator().manual_seed(seed)
        return [torch.randn(self.B * self.p.it_matches, generator=g).double() for _ in range(3)]


def pose_fill(kind="well", rel=0.0, gap=0.0, noise=2e-3, inliers="most", n_out=0, R_off=None, t_off=None, mirror=False):
    """A fill for Planted: one group of S points of `kind` moved by the pair's pose (Rgt R_off, tgt + t_off), or
    mirrored; every hypothesis takes a random subset of the group ('most': 70-100 %, 'all', or an int count) plus
    n_out outlier entries whose Y is random."""
    def fill(pl, b, s):
        rng, S, IR = pl.rng, pl.p.n_sample, pl.p.it_ransac
        X = group_points(rng, S, kind, rel, gap)
        R = pl.Rgt @ (np.eye(3) if R_off is None else R_off)
        t = pl.tgt + (0 if t_off is None else np.asarray(t_off))
        if mirror:
            Y = (X - X.mean(0)) * np.array([-1.0, 1.0, 1.0]) + X.mean(0) + t
        else:
            Y = X @ R.T + t + noise * rng.standard_normal(X.shape)
        n_in = S - n_out
        if n_out:
            Y[n_in:] = group_points(rng, n_out, "well")
        w = np.zeros((IR, S), dtype=bool)
        for h in range(IR):
            if inliers == "all":
                w[h, :n_in] = True
            else:
                k = int(inliers) if not isinstance(inliers, str) else int(rng.integers(max(3, (7 * n_in) // 10), n_in + 1))
                w[h, rng.choice(n_in, k, replace=False)] = True
            if n_out:
                w[h, n_in + rng.integers(0, n_out)] = rng.random() < 0.5
        return X, Y, w
    return fill


THETA_C = math.acos(0.99999)


def planted_table():
    """{class: (Planted kwargs, fill)} of the planted table (DESIGN §6m)."""
    T = {}
    small = dict(B=2, N=200, IM=2, IR=8, S=64)
    T["well_all"] = (small, pose_fill(inliers="all"))
    T["exactly_3"] = (small, pose_fill(inliers=3, noise=0.0))
    T["coplanar"] = (small, pose_fill("coplanar", inliers="all", noise=0.0))
    for rel in (1e-3, 1e-5):
        T[f"near_collinear_{rel:.0e}"] = (small, pose_fill("near_collinear", rel=rel, inliers="all", noise=0.0))
    for gap in (1e-2, 1e-4):
        T[f"mirrored_gap_{gap:.0e}"] = (small, pose_fill("gap", gap=gap, inliers="all", mirror=True))
    for name, ang in (("rot_0", 0.0), ("rot_thc_minus", THETA_C * (1 - 1e-3)), ("rot_thc_plus", THETA_C * (1 + 1e-3)),
                      ("rot_1deg", math.radians(1.0)), ("rot_90deg", math.pi / 2),
                      ("rot_180_minus_thc_minus", math.pi - THETA_C * (1 - 1e-3)),
                      ("rot_180_minus_thc_plus", math.pi - THETA_C * (1 + 1e-3))):
        for loss in ("POSE_ERR", "VCRE"):
            T[f"{name}_{loss}"] = (dict(small, loss=loss),
                                   pose_fill(inliers="all", noise=0.0, R_off=rot([0.3, -0.5, 1.0], ang)))
    for name, off in (("vcre_out_x", [3.0, 0, 0]), ("vcre_out_y", [0, -2.5, 0]), ("vcre_behind", [0, 0, -5.0]),
                      ("vcre_grazing", [0, 0, -2.0])):
        T[name] = (dict(small, loss="VCRE"), pose_fill(inliers="all", t_off=off))
    # an exact pose (VCRE distances ~0, so 1 / v ~ 1e3 px^-1) and a 20 m ground-truth translation: Rgt Rgt^T tgt - tgt
    # (Rgt from fp32 is orthogonal to ~1e-7) moves the inverse direction's projections by ~1e-3 px
    T["vcre_far_tgt"] = (dict(small, loss="VCRE", gt=(gt_pose()[0], np.array([0.5, -0.3, 20.0]))),
                         pose_fill(inliers="all", noise=0.0))
    for loss in ("VCRE", "POSE_ERR"):
        for soft in (True, False):
            for null in (True, False):
                T[f"branch_{loss}_soft{int(soft)}_null{int(null)}"] = (dict(small, loss=loss, soft=soft, null=null),
                                                                        pose_fill(n_out=8))
    for temp in (1e-3, 1e2):
        T[f"temperature_{temp:g}"] = (dict(small, T=temp), pose_fill(n_out=8))
    return T


SHAPES = [dict(B=1, N=256, IM=2, IR=ir, S=32) for ir in (1, 7, 8, 9, 32, 33, 40)]
SHAPES += [dict(B=1, N=4176, IM=1, IR=8, S=2048), dict(B=3, N=4176, IM=64, IR=2, S=32), dict(B=1, N=4176, IM=65, IR=2, S=32),
           dict(B=1, N=4176, IM=129, IR=2, S=32), dict(B=3, N=255, IM=2, IR=8, S=64), dict(B=1, N=257, IM=4, IR=4, S=64)]


def shape_id(kw):
    return "B{B}_N{N}_IM{IM}_IR{IR}_S{S}".format(**kw)


def build(name_or_kw, seed=0):
    """A Planted problem of a table class name or of a shape (kwargs) on well-conditioned data."""
    if isinstance(name_or_kw, str):
        kw, fill = planted_table()[name_or_kw]
        return Planted(fill=fill, seed=seed, **kw)
    return Planted(fill=pose_fill(n_out=4 if name_or_kw["S"] >= 64 else 0), seed=seed, **name_or_kw)


def shared_keypoints(pl: Planted):
    """Rewrite pl's draws so that one keypoint of pair 0 is drawn by entry 0 of every outer iteration (the keypoint of
    set 0's entry 0, so its geometry stays consistent only in set 0: the other sets see an extra point).  Returns the
    keypoint's index."""
    IM, N = pl.p.it_matches, pl.N
    k = int(pl.sampled[0, 0]) // N
    for s in range(1, IM):
        pl.sampled[s, 0] = k * N + k
    return k
