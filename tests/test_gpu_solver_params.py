"""The pose solver across its PROCRUSTES parameters, against fp64.

Every other solver test runs the released values (NUM_SAMPLED_MATCHES 2048, 4 refinements, thresholds 0.15 / 0.3).
CASES is a covering table, not a product: every value of

    NUM_SAMPLED_MATCHES {256, 512, 1024, 1792, 2048}   ransac_solve_kernel's gather_set and cdf scan at n_s / 256 != 8
    NUM_REFINEMENTS     {0, 1, 7}                      finalize_pair without refinement and past the default 4
    (TH_INLIER, TH_SOFT_INLIER) {(0.05, 0.1), (0.5, 1.0), (0.15, 0.15)}
    IT_RANSAC           {1, 7, 9, 100}                 partial blocks of 8 hypotheses
    IT_MATCHES          {1, 3, 20}

appears in at least one row.  Each row runs at N = 1938 on a pitch-1952 view (the engine's layout; the pad columns hold
NaN, so a read of them shows) and at N = 850 contiguous, on planted problems (tests/planted.py) whose inliers carry
Gaussian noise, so that the inlier set grows over the refinements.  The drop-in solvers accept NUM_SAMPLED_MATCHES =
2048 only (the reference's limit); the C ABI takes the whole range, so every call here goes through it: the handle-free
mk_procrustes_solve and mk_solve_pose on an Engine built from the row's config, which must agree bit for bit.

- Both draws injected (the oracle's, torch.multinomial): hypothesis scores, every hyp_Rt, the winner, the pose and the
  inlier mask against oracle.solve_pose.  No refinement: the pose is the winning hyp_Rt bit for bit.  7 refinements:
  the oracle refined some pair more than 4 times.
- The kernel's own draws: every outer stream is the fp64 race at the row's n_s up to the key band, every unambiguous
  inner triple the bit-exact restatement on that n_s's cdf, and the pose the oracle's with both draws re-injected.
- Planted mutations of the restatement, each rejected where the row makes it differ: the outer draw taken at n_s =
  2048, the refinements capped at 4, TH_SOFT_INLIER in the final inlier count.
"""
import ctypes as C

import pytest
import torch

from mickey_b200 import _lib
from mickey_b200.config import mickey_cfg
from mickey_b200.engine import Engine, nn_pitch
from mickey_b200.weights import synthetic_state_dict
from oracle import mickey_oracle as mo
from tests import draws, planted, stages
from tests.common import rotation_angle_deg

pytestmark = pytest.mark.gpu
DEV = "cuda"
SEED = stages.SEED
B = 4
NOISE = 0.1                                  # metres, on planted points 2-6 m deep

# id -> (NUM_SAMPLED_MATCHES, NUM_REFINEMENTS, TH_INLIER, TH_SOFT_INLIER, IT_RANSAC, IT_MATCHES)
CASES = {
    "s256_ref7": (256, 7, 0.15, 0.15, 9, 3),
    "s512_ref0": (512, 0, 0.05, 0.1, 7, 20),
    "s1024_ref1": (1024, 1, 0.5, 1.0, 1, 1),
    "s1792_ref0": (1792, 0, 0.15, 0.15, 100, 3),
    "s2048_ref1": (2048, 1, 0.05, 0.1, 100, 20),
}
# id -> (gh, gw, final_scores at the engine's padded pitch)
SHAPES = {"n1938_pitch1952": (51, 38, True), "n850_contiguous": (34, 25, False)}


def case_cfg(case):
    S, n_ref, th, th_soft, IR, IM = CASES[case]
    cfg = mickey_cfg("vits", IM, IR)
    p = cfg.PROCRUSTES
    p.NUM_SAMPLED_MATCHES, p.NUM_REFINEMENTS, p.TH_INLIER, p.TH_SOFT_INLIER = S, n_ref, th, th_soft
    return cfg


@pytest.fixture(scope="module")
def base_engine():
    cfg = mickey_cfg("vits", 1, 1)
    eng = Engine(cfg, torch.device("cuda", torch.cuda.current_device()))
    eng.load_state_dict(synthetic_state_dict(cfg, seed=0))
    yield eng
    del eng
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", params=list(SHAPES))
def problem(request):
    gh, gw, pitched = SHAPES[request.param]
    N = gh * gw
    p = planted.planted_problem((gh, gw), batch=B, seed=0, noise=NOISE)
    fs = p["final_scores"].to(DEV)
    if pitched:
        buf = torch.full((B, N, nn_pitch(N)), float("nan"), device=DEV)
        buf[:, :, :N] = fs
        fs = buf[:, :, :N]
        assert fs.stride(1) == 1952
    K = p["K"].to(DEV)
    batch = {"final_scores": fs, "kps0": p["kps0"].to(DEV), "kps1": p["kps1"].to(DEV), "depth_kp0": p["depth0"].to(DEV),
             "depth_kp1": p["depth1"].to(DEV), "K_color0": K, "K_color1": K}
    yield request.param, gh, gw, batch
    torch.cuda.empty_cache()


class Solvers:
    """Both C entries of the solver for one row of CASES: mk_procrustes_solve and mk_solve_pose on an Engine built from
    the row's config (weights shared with base_engine; its geometry gives the handle N)."""

    def __init__(self, case, base, gh, gw):
        self.cfg = case_cfg(case)
        p = self.cfg.PROCRUSTES
        self.S, self.n_ref, self.th, self.th_soft = p.NUM_SAMPLED_MATCHES, p.NUM_REFINEMENTS, p.TH_INLIER, p.TH_SOFT_INLIER
        self.IR, self.IM = p.IT_RANSAC, p.IT_MATCHES
        self.eng = Engine(self.cfg, base.device)
        self.eng.load_state_dict(None, share_with=base)
        self.eng._ws_for(B, 14 * gh, 14 * gw)

    def procrustes(self, batch, seed, outer=None, inner=None):
        fs, pitch = _lib.pitched(batch["final_scores"])
        N = fs.shape[1]
        kps = torch.cat([batch["kps0"], batch["kps1"]]).contiguous()
        depth = torch.cat([batch["depth_kp0"], batch["depth_kp1"]]).contiguous()
        lib = _lib.load()
        res = {"pose": torch.empty(B, 13, device=DEV), "best_set": torch.empty(B, dtype=torch.int32, device=DEV),
               "inlier_mask": torch.empty(B, self.S, device=DEV),
               "sampled_idx": torch.empty(B * self.IM, self.S, dtype=torch.int32, device=DEV),
               "hyp_scores": torch.empty(B, self.IM * self.IR, device=DEV),
               "status": torch.zeros(1, dtype=torch.int32, device=DEV)}
        ws = _lib.workspace(lib.mk_procrustes_ws_bytes(B, N, self.IM, self.IR, self.S), DEV, "mk_procrustes_ws_bytes")
        p = _lib.ptr
        oi, ii = (None if i is None else i.to(DEV, torch.int32).contiguous() for i in (outer, inner))
        _lib.check(lib.mk_procrustes_solve(
            p(fs), pitch, p(kps), p(depth), p(batch["K_color0"]), p(batch["K_color1"]), B, N, self.IM, self.IR, self.S, 3,
            self.n_ref, self.th, self.th_soft, C.c_ulonglong(seed), p(oi), p(ii), p(res["pose"]), p(res["best_set"]),
            p(res["inlier_mask"]), p(res["sampled_idx"]), p(res["hyp_scores"]), p(res["status"]), p(ws), ws.numel(),
            _lib.stream()), "mk_procrustes_solve")
        torch.cuda.synchronize()
        return res

    def engine(self, batch, seed, outer=None, inner=None):
        kps = torch.cat([batch["kps0"], batch["kps1"]]).contiguous()
        depth = torch.cat([batch["depth_kp0"], batch["depth_kp1"]]).contiguous()
        res = self.eng.solve(batch["final_scores"], kps, depth, batch["K_color0"], batch["K_color1"], seed,
                             outer_idx=outer, inner_idx=inner)
        torch.cuda.synchronize()
        res["hyp_Rt"] = self.eng.ws_view("hyp_Rt", torch.float32, (B * self.IM * self.IR, 12)).clone()
        return res

    def both(self, batch, seed, outer=None, inner=None):
        """Both entries on the same inputs: every output bit for bit; returns the engine's (with hyp_Rt)."""
        a, b = self.procrustes(batch, seed, outer, inner), self.engine(batch, seed, outer, inner)
        for k in ("pose", "best_set", "inlier_mask", "sampled_idx", "hyp_scores", "status"):
            assert torch.equal(a[k], b[k]), k
        assert int(b["status"].item()) == 0
        return b


def oracle(batch, cfg, **kw):
    tr = {}
    d = {k: v.double() for k, v in batch.items()}
    R, t, inl = mo.solve_pose(d["final_scores"], d["kps0"], d["depth_kp0"], d["kps1"], d["depth_kp1"], d["K_color0"],
                              d["K_color1"], cfg, trace=tr, **kw)
    return R.reshape(B, 3, 3), t.reshape(B, 3), inl.reshape(B), tr


def pose_misses(R, t, Ro, to):
    """Per pair: the pose outside the bounds of tests/test_gpu_procrustes.py (1e-2 degrees, 1e-3 m)."""
    return (rotation_angle_deg(R, Ro).to(DEV) >= 1e-2) | ((t.double() - to).abs().amax(1) >= 1e-3)


def check_against_oracle(s, res, ref, label):
    """hyp_scores, hyp_Rt, the winner, the pose, the soft inlier count and the hard inlier mask against the oracle run
    on the same draws.  Returns (pose, whether the winner is the oracle's) per pair."""
    Ro, to, inlo, tr = ref
    hyp, refh = res["hyp_scores"].double(), tr["hyp_scores"].double()
    assert bool(((hyp - refh).abs() <= 1e-3 * refh.abs() + 1e-3).all()), label
    # every hypothesis's [R | t] against an fp64 Kabsch of its triple (well-conditioned triples, kabsch_check's bounds)
    X, Y = tr["X"], tr["Y"]
    s_of = torch.arange(B * s.IM, device=DEV).repeat_interleave(s.IR)
    inner = tr["inner_idx"]
    Xk, Yk = X[s_of[:, None], inner], Y[s_of[:, None], inner]
    Rr, trr = mo.kabsch(Xk, Yk)
    sv = torch.linalg.svdvals((Xk - Xk.mean(1, keepdim=True)).transpose(1, 2) @ (Yk - Yk.mean(1, keepdim=True)))
    well = sv[:, 1] > 1e-3 * sv[:, 0]
    assert float(well.float().mean()) > 0.5, label
    got = res["hyp_Rt"].double()
    trr = trr.reshape(-1, 3)
    miss = ((got[:, :9] - Rr.reshape(-1, 9)).abs().amax(1) > 1e-3) | ((got[:, 9:] - trr).abs() > 1e-3 * (1 + trr.abs())).any(1)
    assert int((miss & well).sum()) == 0, (label, int((miss & well).sum()))
    # the winner (tie-tolerant), then the pose, the count and the mask where it is the oracle's
    win = hyp.argmax(1)
    assert bool((refh.gather(1, win[:, None])[:, 0] >= refh.max(1).values * (1 - 1e-3)).all()), label
    same = win == tr["best"]
    R, t, inl = res["pose"][:, :9].reshape(B, 3, 3), res["pose"][:, 9:12], res["pose"][:, 12]
    assert not bool(pose_misses(R, t, Ro, to)[same].any()), label
    assert bool(((inl.double() - inlo).abs() <= 1e-3 * inlo.abs() + 1e-3)[same].all()), label
    bs = tr["best_set"]
    Xb, Yb = X[bs], Y[bs]
    resid = mo.residual_norm(Xb, Yb, Ro, to[:, None])
    border = (resid - s.th).abs() <= 1e-4                       # fp32 residuals within 1e-4 m of the threshold
    mask_ref = (resid <= s.th).double()
    ok = (res["inlier_mask"].double() == mask_ref) | border
    assert bool(ok[same].all()), label
    assert torch.equal(res["best_set"].long()[same], bs[same])
    return (R, t, inl), same


@pytest.mark.parametrize("case", list(CASES))
def test_injected_draws_against_the_oracle(problem, base_engine, case):
    shape, gh, gw, batch = problem
    s = Solvers(case, base_engine, gh, gw)
    label = f"{case} {shape}"
    g = torch.Generator(device=DEV).manual_seed(1)
    ref = oracle(batch, s.cfg, generator=g)
    tr = ref[3]
    res = s.both(batch, SEED, tr["outer_idx"], tr["inner_idx"])
    (R, t, inl), same = check_against_oracle(s, res, ref, label)
    assert bool(same.any()), label
    rejected = 0
    if s.n_ref == 0:                      # the pose is the winning hypothesis's [R | t], bit for bit
        Rt = res["hyp_Rt"].reshape(B, s.IM * s.IR, 12)
        hyp = res["hyp_scores"]
        for b in range(B):
            top = (hyp[b] == hyp[b].max()).nonzero()[:, 0]
            assert any(torch.equal(Rt[b, h], res["pose"][b, :12]) for h in top.tolist()), (label, b)
    if s.n_ref > 4:
        assert tr["n_refinements"] > 4, (label, tr["n_refinements"])
        cfg4 = s.cfg.clone()
        cfg4.PROCRUSTES.NUM_REFINEMENTS = 4
        R4, t4, _, _ = oracle(batch, cfg4, outer_idx=tr["outer_idx"], inner_idx=tr["inner_idx"])
        assert bool(pose_misses(R, t, R4, t4)[same].any()), f"{label}: refinements capped at 4 not rejected"
        rejected += 1
    if s.th_soft != s.th:                 # TH_SOFT_INLIER in the final count
        bs = tr["best_set"]
        soft = mo.soft_inliers(tr["X"][bs], tr["Y"][bs], ref[0], ref[1][:, None], s.th_soft).reshape(B)
        assert bool(((inl.double() - soft).abs() > 1e-3 * soft.abs() + 1e-3)[same].any()), \
            f"{label}: TH_SOFT_INLIER in the final count not rejected"
        rejected += 1
    assert rejected or s.n_ref == 0
    print(f"\n[{label}] oracle draws: same winner in {int(same.sum())}/{B} pairs, oracle refinements "
          f"{tr['n_refinements']}, {rejected} planted mutations rejected")


@pytest.mark.parametrize("case", list(CASES))
def test_own_draws(problem, base_engine, case):
    shape, gh, gw, batch = problem
    s = Solvers(case, base_engine, gh, gw)
    label = f"{case} {shape}"
    fs = batch["final_scores"]
    own = s.both(batch, SEED)
    outer = own["sampled_idx"].long()
    got = outer.reshape(B, s.IM, s.S)
    diff = band = 0
    for b in range(B):
        d, n = stages.band_all(fs[b].contiguous(), got[b], b, s.IM, SEED, label, n_s=s.S)
        diff, band = max(diff, d), max(band, n)
    rejected = 0
    if s.S != 2048:                       # the outer draw taken at n_s = 2048, cut to the first n_s cells
        _, key = next(draws.outer_keys(fs[0].contiguous().reshape(-1).double(), SEED, 0, [0]))
        assert not draws.band_check(draws.reference_draw(key, 2048)[:s.S], key, s.S)["ok"], label
        rejected += 1
    b_of = torch.arange(B, device=DEV).repeat_interleave(s.IM)
    s_in = torch.arange(s.IM, device=DEV).repeat(B)
    w = fs.contiguous().reshape(B, -1)[b_of[:, None], outer]
    idx, amb = draws.inner_draw(draws.inner_cdf(w.float()), SEED, b_of, s_in, s.IR)
    inner = idx.reshape(-1, 3)
    again = s.both(batch, SEED, outer, inner)
    clear = ~amb.reshape(B * s.IM * s.IR)
    assert float(clear.float().mean()) > 0.99, label
    assert torch.equal(again["hyp_scores"].reshape(-1)[clear], own["hyp_scores"].reshape(-1)[clear]), label
    assert torch.equal(again["hyp_Rt"][clear], own["hyp_Rt"][clear]), label
    if bool(clear.all()):
        assert all(torch.equal(again[k], own[k]) for k in ("pose", "best_set", "inlier_mask")), label
    ref = oracle(batch, s.cfg, outer_idx=outer, inner_idx=inner)
    _, same = check_against_oracle(s, again, ref, label)
    assert rejected or s.S == 2048
    print(f"\n[{label}] kernel draws: max cells differing from fp64 {diff}, in band {band}; {int((~clear).sum())} "
          f"ambiguous triples; same winner in {int(same.sum())}/{B} pairs; {rejected} planted mutations rejected")
