"""tests/loss_tail_check.py's element bound and planted table without a GPU.

- The bound accepts the fp64 oracle against itself re-evaluated in another valid order (entries and hypotheses of every
  set permuted), stored to fp32.
- It rejects every planted mutation of oracle/loss_tail_oracle.py on the loss fixtures and the planted table; the
  mutations test_gpu_loss.py::compare's normwise bound accepts (computed here with the fp32 autograd tail) are printed.
- Each planted class has its intended property in fp64: kappa range, the acos clip straddle, VCRE points outside the
  image and behind the camera, exact-zero H where intended.
- The random-perturbation probe stays below the bound's rounding term.
"""
import copy

import numpy as np
import pytest
import torch

from oracle import loss_oracle as lo
from oracle import loss_tail_oracle as lto
from tests import loss_cases
from tests import loss_tail_check as ltc

FIX = np.load(loss_cases.FIXTURE)
NEW_MUTATIONS = lto.TAIL_MUTATIONS[5:]


class Fixture(ltc.Planted):
    """A loss fixture case with its recorded draws and fp64 inliers_final, on its fp32-rounded inputs."""

    def __init__(self, name):
        cfg = loss_cases.case_cfg(name)
        from mickey_b200.loss import LossParams
        self.p = p = LossParams(cfg)
        batch = {k: v.float() for k, v in loss_cases.case_batch(name).items()}
        ref = lo.metric_pose_loss({k: v.double() for k, v in batch.items()}, p,
                                  outer_idx=torch.from_numpy(FIX[f"{name}/outer_idx"]).long(),
                                  inner_idx=torch.from_numpy(FIX[f"{name}/inner_idx"]).long())
        self.kps0, self.d0, self.kps1, self.d1 = batch["kps0"], batch["depth_kp0"], batch["kps1"], batch["depth_kp1"]
        self.K, self.T, self.Kori = batch["K_color0"], batch["T_0to1"], batch["Kori_color0"]
        assert torch.equal(batch["K_color0"], batch["K_color1"]) and torch.equal(batch["Kori_color0"], batch["Kori_color1"])
        self.sampled, self.inl = ref["sampled"].int(), ref["inliers_final"].double()
        self.B, self.N = self.kps0.shape[0], self.kps0.shape[2]

    def oracle(self, ups, mutation=None, dtype=torch.float64):
        Kd, Ko, T = self.K.double(), self.Kori.double(), self.T.double()
        Kinv = (lto.kernel_kinv(self.K), lto.kernel_kinv(self.K))
        return lto.tail_closed_form(self.kps0.double(), self.d0.double(), self.kps1.double(), self.d1.double(), Kd, Kd,
                                    Ko, Ko, T[:, :3, :3], T[:, :3, 3:].transpose(1, 2), self.sampled, self.inl,
                                    ltc.kernel_params(self.p), *ups, mutation=mutation, Kinv=Kinv, grid=ltc.KERNEL_GRID)


def _permuted(pl, seed):
    """pl with every set's entries and hypotheses permuted (the same problem in another summation order)."""
    g = torch.Generator().manual_seed(seed)
    IM, IR, S = pl.p.it_matches, pl.p.it_ransac, pl.p.n_sample
    sets = pl.sampled.shape[0]
    q = copy.copy(pl)
    inl = pl.inl.reshape(sets, IR, S)
    samp, new_inl = pl.sampled.clone(), inl.clone()
    for s in range(sets):
        pe, ph = torch.randperm(S, generator=g), torch.randperm(IR, generator=g)
        samp[s] = pl.sampled[s, pe]
        new_inl[s] = inl[s][ph][:, pe]
    q.sampled, q.inl = samp, new_inl.reshape(sets * IR, S)
    return q


def _got(out):
    return {k: out[k].float() for k in ltc.QUANTITIES}


FIXTURES = list(loss_cases.CASES)
PLANTED = ["well_all", "exactly_3", "near_collinear_1e-03", "mirrored_gap_1e-02", "rot_thc_plus_POSE_ERR",
           "rot_180_minus_thc_minus_VCRE", "vcre_behind", "vcre_out_x", "branch_POSE_ERR_soft0_null0", "temperature_0.001"]


def _problem(name):
    return Fixture(name) if name in loss_cases.CASES else ltc.build(name)


def test_kernel_kinv_is_round_safe():
    for K in [ltc.K_PIN] + [loss_cases.case_batch(n)["K_color0"].float() for n in ("vits_vcre", "vitb_vcre")]:
        assert ltc.kinv_is_safe(K)


@pytest.mark.parametrize("name", FIXTURES + PLANTED)
def test_bound_accepts_the_oracle_in_another_order(name):
    pl = _problem(name)
    ups = pl.upstream(3)
    want = pl.oracle(ups)
    other = _permuted(pl, 7).oracle(ups)
    r, _ = ltc.compare(_got(other), want, pl.p, pl.tgt_t(), name)
    print(name, {k: f"{v:.3g}" for k, v in r.items()})


def _old_bound_accepts(pl, ups, want, mutated):
    """test_gpu_loss.py::compare's allowance, with the fp32 autograd tail as its 'fp32 oracle': values within 5e-4 of
    their largest magnitude, gradients within 2 max|fp32 - fp64| + 5e-3 max|fp64|."""
    leaves = [x.float().clone().requires_grad_() for x in (pl.kps0, pl.d0, pl.kps1, pl.d1)]
    T = pl.T.float()
    K = pl.K.float()
    Ko = getattr(pl, "Kori", K).float()
    vals = lto.tail_autograd(*leaves, K, K, Ko, Ko, T[:, :3, :3], T[:, :3, 3:].transpose(1, 2), pl.sampled,
                             pl.inl.float(), pl.p)
    grads = torch.autograd.grad(sum((v * u.float()).sum() for v, u in zip(vals, ups)), leaves)
    for k, v in zip(("loss_value", "loss_rot", "loss_trans"), vals):
        if float((mutated[k] - want[k]).abs().max()) > 5e-4 * float(want[k].abs().max()):
            return False
    for k, g32 in zip(("dkps0", "ddepth0", "dkps1", "ddepth1"), grads):
        allowed = 2 * float((g32.double() - want[k]).abs().max()) + 5e-3 * float(want[k].abs().max())
        if float((mutated[k] - want[k]).abs().max()) > allowed:
            return False
    return True


def test_bound_rejects_every_mutation():
    """Every mutation is rejected by the element bound on at least one fixture (and planted class for those that need a
    geometry the fixtures do not have: a VCRE point behind the camera, a VCRE distance near 0 with a far ground truth)."""
    rejected = {m: [] for m in NEW_MUTATIONS}
    old_accepts = {m: True for m in NEW_MUTATIONS}
    for name in FIXTURES + ["well_all", "vcre_behind", "vcre_far_tgt", "branch_VCRE_soft1_null1"]:
        pl = _problem(name)
        ups = pl.upstream(5)
        want = pl.oracle(ups)
        for m in NEW_MUTATIONS:
            mo = pl.oracle(ups, m)
            _, fails = ltc.compare(_got(want) | {k: mo[k] for k in ltc.QUANTITIES}, want, pl.p, pl.tgt_t(), name,
                                   mutations_ok=True)
            if fails:
                rejected[m].append(name)
            if name in loss_cases.CASES and old_accepts[m]:
                old_accepts[m] = _old_bound_accepts(pl, ups, want, mo)
    print("rejected by the element bound on:", rejected)
    print("accepted by test_gpu_loss.py::compare's bound on every fixture:", [m for m, a in old_accepts.items() if a])
    assert all(rejected.values()), rejected
    assert all(any(n in loss_cases.CASES for n in rejected[m]) for m in ("ki_fp64", "scatter_drop_last", "last_hyp_dropped"))


def test_planted_classes_have_their_properties():
    for name, (lo_k, hi_k) in (("well_all", (0.1, 10)), ("coplanar", (0.1, 1e3)), ("near_collinear_1e-03", (1e4, 1e8)),
                               ("near_collinear_1e-05", (1e8, 1e11)), ("mirrored_gap_1e-02", (50, 1e3)),
                               ("mirrored_gap_1e-04", (5e3, 1e5))):
        pl = ltc.build(name)
        out = pl.oracle(pl.upstream())
        k = ltc.kappas(out)
        assert float(k.min()) >= lo_k and float(k.max()) <= hi_k, (name, float(k.min()), float(k.max()))
        if name.startswith("mirrored"):
            assert bool((torch.linalg.det(out["H"]) < 0).all())
        if name == "coplanar":
            s = torch.linalg.svdvals(out["H"])
            assert float((s[:, 2] / s[:, 0]).max()) < 1e-5
    pl = ltc.build("exactly_3")
    assert bool((pl.inl.sum(1) == 3).all())
    # the acos clip: inside below theta_c, outside above (and at 180 deg - theta_c the other way)
    for name, inside in (("rot_thc_minus_POSE_ERR", False), ("rot_thc_plus_POSE_ERR", True),
                         ("rot_180_minus_thc_minus_POSE_ERR", False), ("rot_180_minus_thc_plus_POSE_ERR", True),
                         ("rot_0_POSE_ERR", False), ("rot_90deg_POSE_ERR", True)):
        pl = ltc.build(name)
        m = pl.oracle(pl.upstream())["mag"]
        assert bool((m["inside"] == inside).all()), (name, m["cos"].min(), m["cos"].max())
    # VCRE: predicted projections outside [0, 720] on either axis, and behind the camera
    for name, axis in (("vcre_out_x", 0), ("vcre_out_y", 1), ("vcre_behind", 2)):
        pl = ltc.build(name)
        out = pl.oracle(pl.upstream())
        R, t = out["R"], out["t"]
        Rgt, tgt = pl.T.double()[:1, :3, :3], pl.T.double()[:1, :3, 3]
        e = lto.vcre_grid().unsqueeze(0)
        res = (e @ R.transpose(1, 2) + (t - tgt).unsqueeze(1)) @ Rgt
        x = res @ ltc.K_PIN.double().T
        if axis == 2:
            assert bool((x[..., 2] < 0).any())
        else:
            uv = x[..., axis] / x[..., 2]
            assert bool(((uv < 0) | (uv > 720)).any())
    # H exactly zero for W1 = 0 and W1 = 1; at rounding level when three inlier entries share one image-0 keypoint (the
    # mean of three equal values times 1 / 3 need not return the value); rank 1 for two distinct points
    for kind in ("w0", "w1", "shared", "rank1"):
        H = kernel_H(degenerate(kind))[0]
        s = torch.linalg.svdvals(H)
        if kind in ("w0", "w1"):
            assert bool((H == 0).all()), kind
        elif kind == "shared":
            assert float(H.abs().max()) < 1e-12, kind
        else:
            assert float(s[1]) <= 1e-12 * float(s[0]) and float(s[0]) > 1e-3, kind


def kernel_H(pl):
    """H of every hypothesis as the kernel forms it: fp64 means with w / (W1 + 1e-16), then the sum of outer products."""
    sets, _ = lto._set_points(pl.kps0.double(), pl.d0.double(), pl.kps1.double(), pl.d1.double(), pl.K.double(),
                              pl.K.double(), pl.sampled, pl.p.it_matches, (lto.kernel_kinv(pl.K), lto.kernel_kinv(pl.K)))
    X, Y = sets[0][0].repeat_interleave(pl.p.it_ransac, 0), sets[1][0].repeat_interleave(pl.p.it_ransac, 0)
    w = pl.inl
    wn = 1.0 / (w.sum(1, keepdim=True) + 1e-16)
    a, b = (w.unsqueeze(-1) * X).sum(1) * wn, (w.unsqueeze(-1) * Y).sum(1) * wn
    return (X - a.unsqueeze(1)).transpose(1, 2) @ (w.unsqueeze(-1) * (Y - b.unsqueeze(1)))


def degenerate(kind):
    """A B = 1, IM = 2, IR = 8, S = 64 problem whose hypothesis 0 of set 0 is degenerate: 'w0' no inlier, 'w1' one,
    'shared' three inlier entries that draw one image-0 keypoint, 'rank1' two distinct inlier points."""
    pl = ltc.Planted(B=1, N=200, IM=2, IR=8, S=64, fill=ltc.pose_fill(inliers="all"), seed=3)
    S, N = pl.p.n_sample, pl.N
    row = torch.zeros(S, dtype=torch.float64)
    if kind == "w1":
        row[5] = 1
    elif kind in ("shared", "rank1"):
        row[[5, 9, 13] if kind == "shared" else [5, 9]] = 1
    if kind == "shared":
        k0 = int(pl.sampled[0, 5]) // N
        for j in (9, 13):
            pl.sampled[0, j] = k0 * N + int(pl.sampled[0, j]) % N
    pl.inl[0] = row
    return pl


@pytest.mark.parametrize("name", ["well_all", "vcre_out_x", "branch_POSE_ERR_soft1_null1"])
def test_perturbation_probe_stays_inside_the_bound(name):
    pl = ltc.build(name)
    Kd, T = pl.K.double(), pl.T.double()
    args = [pl.kps0.double(), pl.d0.double(), pl.kps1.double(), pl.d1.double(), Kd, Kd, Kd, Kd, T[:, :3, :3],
            T[:, :3, 3:].transpose(1, 2), pl.sampled, pl.inl]
    r = ltc.probe_ratio(args, pl.p, pl.upstream(), (lto.kernel_kinv(pl.K), lto.kernel_kinv(pl.K)))
    print(name, "probe change / (128 E):", f"{r:.3g}")
    assert r <= 1.0
