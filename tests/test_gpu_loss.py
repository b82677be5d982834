"""The training loss on the GPU (mickey_b200/loss.py: CUDA search and gradient, autograd tail) against the fp64 oracle
(oracle/loss_oracle.py), with the oracle's torch.multinomial draws injected, on the fixture batches and once at
production size (B = 8, 720x540 so N = 1938, IT_MATCHES = IT_RANSAC = 20, 512 samples, 8-point hypotheses, from the
engine's own final_scores); then the contract cases and the kernel's own draws.

Bounds.
- inliers_final: equal for every hypothesis, except where some inlier test of its refinement had a residual within
  EPS_M = 1e-5 m of INLIER_REF_TH.  The kernel tests fp32 residuals of an fp64 Kabsch rounded to fp32; with points a few
  metres away the residual's rounding error is a few 1e-7 m, so 1e-5 m leaves a wide margin.  The count is printed.
- loss_value, baseline, avg_loss: 5e-4 of their largest magnitude.  The tail runs in fp32: the pose of a near-degenerate
  8-point hypothesis moves by its SVD's condition number times the fp32 rounding, and POSE_ERR without clipping passes
  that straight into the loss.  The fp32 oracle against the fp64 one on the fixtures (CPU) differs by up to 1.1e-4.
- probs_grad: identical support and |got - want| <= 5e-4 max|loss_value|.  A cell drawn by every outer iteration of its
  pair has the value (sum - IM * (sum / IM)) / IM, zero up to rounding: whether it rounds to exactly 0 is an accident of
  the summation, so for those cells only the bound applies (cells never drawn must be exactly 0).  A value is (sum of the drawing iterations'
  losses - count * baseline) / IM, a difference of nearly equal terms of size up to max|loss_value|, so its error is set
  by the losses' error, not by its own size (fp32 oracle against fp64 on the fixtures: up to 1.3e-4 of max|probs_grad|).
- kps / depth grads, avg_loss_rot / avg_loss_trans: |got - want| <= 2 |fp32 oracle - want| + 5e-3 max|want| (5e-4 for
  the two scalars).  The reference's own arithmetic is ill-conditioned here, so the bound is what that arithmetic loses
  in fp32 on the same data and draws, twice over: the gradients pass through torch's SVD backward, whose terms carry
  1 / (s_i^2 - s_j^2), and the rotation loss is acos((trace - 1) / 2), whose derivative 1 / sqrt(1 - c^2) turns the fp32
  rounding of c near 1 (small rotation errors) into relative errors of several percent (POSE_ERR fixture: 9 %).
"""
import math

import numpy as np
import pytest
import torch

from mickey_b200.loss import LossParams, MetricPoseLoss, STATUS_INNER, STATUS_PRECHECK, loss_search
from oracle import loss_oracle as lo
from tests import draws, loss_cases

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS_M = 1e-5
FIX = np.load(loss_cases.FIXTURE)


def _cuda(batch):
    return {k: v.to(DEV) for k, v in batch.items()}


def _rel(got, want):
    got, want = got.detach().double(), want.detach().double()
    return float((got - want).abs().max() / want.abs().max().clamp_min(1e-30))


def check_gradient(grad, want, sampled, loss_value, IM):
    """probs_grad against a reference: the support rule and the bound of the module docstring."""
    B, N = want.shape[0], want.shape[1]
    count = torch.zeros(B, N * N, device=grad.device)
    for s in range(B * IM):
        count[s // IM, sampled[s].long()] += 1
    count = count.reshape(B, N, N)
    assert bool((grad[count == 0] == 0).all())
    partial = (count > 0) & (count < IM)
    assert torch.equal((grad != 0)[partial], (want != 0)[partial])
    err = float((grad.double() - want.double()).abs().max())
    assert err <= 5e-4 * float(loss_value.abs().max()), err


def compare(batch, cfg, generator=None, outer=None, inner=None, label=""):
    """Run the oracle (fp64, draws from `generator` unless given) and MetricPoseLoss with the same draws; check every
    bound of the module docstring.  Returns (oracle result, loss outputs)."""
    p = LossParams(cfg)
    ref = lo.metric_pose_loss(batch, p, outer_idx=outer, inner_idx=inner, generator=generator)
    assert ref["num_valid_h"] == 1
    loss = MetricPoseLoss(cfg)
    avg, out, (grad,), nv = loss(batch, seed=7, outer_idx=ref["sampled"], inner_idx=ref["inner"])
    assert nv == 1
    _, _, inl, status = loss_search(batch["final_scores"], batch["kps0"], batch["depth_kp0"], batch["kps1"],
                                    batch["depth_kp1"], batch["K_color0"], batch["K_color1"], p, 7, ref["sampled"],
                                    ref["inner"])
    assert status == 0
    diff = (inl.double() != ref["inliers_final"]).any(1)
    near = ref["margin"] <= EPS_M
    print(f"{label}: {int(diff.sum())} of {diff.numel()} hypotheses differ in inliers_final, all near the threshold; "
          f"{int(near.sum())} have a residual within {EPS_M} m of it")
    assert not bool((diff & ~near).any())
    if bool(diff.any()):
        return ref, None          # a near-threshold flip changes that hypothesis's pose; values are not comparable
    assert _rel(loss.last_loss_value, ref["loss_value"]) < 5e-4
    assert _rel(loss.last_baseline, ref["baseline"]) < 5e-4
    assert _rel(avg, ref["avg_loss"]) < 5e-4
    check_gradient(grad, ref["probs_grad"], ref["sampled"], ref["loss_value"].detach(), p.it_matches)
    ref32 = lo.metric_pose_loss(batch, p, outer_idx=ref["sampled"], inner_idx=ref["inner"], dtype=torch.float32)
    avg.backward()
    ref["avg_loss"].backward()
    ref32["avg_loss"].backward()

    def within(got, want, fp32, rel):
        got, want, fp32 = got.detach().double(), want.detach().double(), fp32.detach().double()
        err, allowed = float((got - want).abs().max()), 2 * float((fp32 - want).abs().max()) + rel * float(want.abs().max())
        return err <= allowed, (err, allowed)

    for k in ("kps0", "kps1", "depth0", "depth1"):
        ok, info = within(out[k].grad, ref[k].grad, ref32[k].grad, 5e-3)
        assert ok, (k, info)
    for k in ("avg_loss_rot", "avg_loss_trans"):
        ok, info = within(out[k], ref[k], ref32[k], 5e-4)
        assert ok, (k, info)
    assert torch.equal(out["mask_topk"].double(), ref["mask_topk"])
    return ref, (avg, out, grad)


@pytest.mark.parametrize("name", list(loss_cases.CASES))
def test_fixture_cases_match_oracle_with_reference_draws(name):
    p = f"{name}/"
    compare(_cuda(loss_cases.case_batch(name)), loss_cases.case_cfg(name),
            outer=torch.from_numpy(FIX[p + "outer_idx"]).long().to(DEV),
            inner=torch.from_numpy(FIX[p + "inner_idx"]).long().to(DEV), label=name)


def test_loss_values_match_reference_fixture():
    """The GPU loss against the live reference's own numbers (fp32 both sides, bounds of the module docstring)."""
    for name in loss_cases.CASES:
        p = f"{name}/"
        batch = _cuda(loss_cases.case_batch(name))
        loss = MetricPoseLoss(loss_cases.case_cfg(name))
        avg, out, (grad,), nv = loss(batch, outer_idx=torch.from_numpy(FIX[p + "outer_idx"]).to(DEV),
                                     inner_idx=torch.from_numpy(FIX[p + "inner_idx"]).to(DEV))
        assert nv == 1
        assert abs(float(avg) - float(FIX[p + "avg_loss"])) <= 5e-4 * abs(float(FIX[p + "avg_loss"])), name
        want = torch.zeros(grad.numel(), device=DEV)
        want[torch.from_numpy(FIX[p + "grad_idx"]).to(DEV)] = torch.from_numpy(FIX[p + "grad_val"]).to(DEV)
        check_gradient(grad, want.reshape(grad.shape), torch.from_numpy(FIX[p + "outer_idx"]).to(DEV),
                       torch.from_numpy(FIX[p + "loss_value"]), loss.p.it_matches)


@pytest.fixture(scope="module")
def production():
    """The engine's final_scores of 8 synthetic 720x540 ViT-S pairs, with kps / depth, a planted pose and K."""
    from mickey_b200.config import mickey_cfg
    from mickey_b200.model import MickeyRelativePose
    from mickey_b200.weights import synthetic_state_dict
    from tests.common import synthetic_pair
    cfg = mickey_cfg("vits", 20, 20)
    model = MickeyRelativePose(cfg)
    model.load_state_dict(synthetic_state_dict(cfg, seed=3), strict=True)
    model = model.cuda().eval()
    data = {k: v.to(DEV) for k, v in synthetic_pair(8, 720, 540, seed=17).items()}
    with torch.no_grad():
        model.compute_matches(data)
    fs = data["_final_scores_fused"]
    B, N = fs.shape[0], fs.shape[1]
    assert (B, N) == (8, 1938)
    K = data["K_color0"].float()
    T = loss_cases.planted_pose().float().to(DEV).unsqueeze(0).repeat(B, 1, 1)
    return {"final_scores": fs.contiguous(), "kps0": data["kps0"].float(), "kps1": data["kps1"].float(),
            "depth_kp0": data["depth_kp0"].float(), "depth_kp1": data["depth_kp1"].float(), "K_color0": K,
            "K_color1": data["K_color1"].float(), "Kori_color0": K, "Kori_color1": data["K_color1"].float(), "T_0to1": T}


def test_production_size_matches_oracle(production):
    cfg = loss_cases.loss_cfg(it_matches=20, it_ransac=20, topk=True)
    compare(production, cfg, generator=torch.Generator(DEV).manual_seed(11), label="production B=8 N=1938 20x20")


def test_own_outer_draws_pass_band_check(production):
    """Every outer stream of the production batch is the fp64 exponential race's top 512 up to the 1e-4 key band."""
    p = LossParams(loss_cases.loss_cfg(it_matches=20, it_ransac=20))
    b_ = production
    seed = 0x1234ABCD5678
    sampled, _, _, status = loss_search(b_["final_scores"], b_["kps0"], b_["depth_kp0"], b_["kps1"], b_["depth_kp1"],
                                        b_["K_color0"], b_["K_color1"], p, seed)
    assert status == 0
    B, N = b_["final_scores"].shape[:2]
    IM = p.it_matches
    n_diff = 0
    for b in range(B):
        pr = b_["final_scores"][b].reshape(-1).double()
        for s, key in draws.outer_keys(pr, seed, b, range(IM)):
            r = draws.band_check(sampled[b * IM + s], key, p.n_sample)
            assert r["ok"], (b, s, r)
            n_diff += r["n_diff"]
    print(f"outer draws: {B * IM} streams pass the band check, {n_diff} cells differ inside the band")


def test_same_seed_gives_identical_gradient(production):
    cfg = loss_cases.loss_cfg(it_matches=20, it_ransac=20, topk=True)
    g = [MetricPoseLoss(cfg)(production, seed=99)[2][0] for _ in range(2)]
    assert torch.equal(g[0], g[1])
    assert bool((g[0] != 0).any())


# ---- the inner law ------------------------------------------------------------------------------------------------
def successive_law(w, k):
    """P(the first k draws of successive sampling ~ w are the set A), for every k-subset A of the positive entries, by a
    DP over subsets: f(A) = sum_{a in A} f(A - a) w_a / (W - w(A - a))."""
    pos = [i for i, x in enumerate(w) if x > 0]
    W = math.fsum(w[i] for i in pos)
    f = {frozenset(): 1.0}
    for size in range(1, k + 1):
        nf = {}
        for A, pa in f.items():
            rest = W - math.fsum(w[i] for i in A)
            for a in pos:
                if a not in A:
                    B = A | {a}
                    nf[B] = nf.get(B, 0.0) + pa * w[a] / rest
        f = nf
    return {tuple(sorted(A)): v for A, v in f.items()}


def test_inner_law_chi2():
    """65,536 hypotheses, each drawing 8 of a set whose 10 positive scores span three decades (the other 502 are 0):
    the drawn 8-sets follow successive sampling's law by chi^2, the first three draws follow draws.law3, and the
    uniform law and the with-replacement triple law are rejected by the same statistics."""
    wts = [1.0, 0.5, 0.3, 0.2, 0.1, 0.05, 0.03, 0.02, 0.01, 0.005]
    N, S, IM, IR = 64, 512, 64, 1024
    fs = torch.zeros(1, N, N, device=DEV)
    cells = torch.randperm(N * N, generator=torch.Generator().manual_seed(3))[:S].to(DEV)
    pos_at = [5, 70, 129, 200, 255, 256, 300, 400, 480, 511]          # set positions of the positive cells
    fs.view(-1)[cells[pos_at]] = torch.tensor(wts, device=DEV)
    outer = cells.unsqueeze(0).repeat(IM, 1)
    z = torch.zeros(1, 2, N, device=DEV)
    d = torch.ones(1, 1, N, device=DEV)
    K = torch.eye(3, device=DEV).unsqueeze(0)
    p = LossParams(loss_cases.loss_cfg(it_matches=IM, it_ransac=IR))
    _, inner, _, status = loss_search(fs, z, d, z, d, K, K, p, 2024, outer)
    assert status == 0
    inner = inner.cpu()
    idx_of = {q: i for i, q in enumerate(pos_at)}
    assert set(inner.unique().tolist()) == set(pos_at)
    sets = inner.sort(1).values
    cnt = {}
    for row in sets.tolist():
        key = tuple(idx_of[q] for q in row)
        cnt[key] = cnt.get(key, 0) + 1
    law8 = successive_law(wts, 8)
    assert abs(sum(law8.values()) - 1) < 1e-12
    p8 = draws.chi2_pvalue(cnt, law8)
    uniform = {k: 1 / len(law8) for k in law8}
    assert p8 > 1e-6 and draws.chi2_pvalue(cnt, uniform) < 1e-6
    first3 = {}
    for row in inner[:, :3].tolist():
        key = tuple(sorted(idx_of[q] for q in row))
        first3[key] = first3.get(key, 0) + 1
    p3 = draws.chi2_pvalue(first3, draws.law3(wts))
    assert p3 > 1e-6 and draws.chi2_pvalue(first3, draws.law3_with_replacement(wts)) < 1e-6
    print(f"inner law: p = {p8:.3g} (8-sets), {p3:.3g} (first three draws)")


# ---- contract cases -----------------------------------------------------------------------------------------------
def _run(batch, cfg, **kw):
    return MetricPoseLoss(cfg)(batch, seed=5, **kw)


def _is_zero_result(res, B):
    avg, out, (grad,), nv = res
    return nv == 0 and float(grad.abs().max()) == 0 and float(out["avg_loss_rot"]) == 0


def test_contract_nan_cell_skips_the_search():
    batch = _cuda(loss_cases.case_batch("vits_vcre"))
    batch["final_scores"][1, 3, 4] = float("nan")
    cfg = loss_cases.case_cfg("vits_vcre")
    p = LossParams(cfg)
    *_, status = loss_search(batch["final_scores"], batch["kps0"], batch["depth_kp0"], batch["kps1"], batch["depth_kp1"],
                             batch["K_color0"], batch["K_color1"], p, 5)
    assert status & STATUS_PRECHECK and status & 1
    res = _run(batch, cfg)
    assert _is_zero_result(res, 2) and float(res[0]) == 0
    assert lo.metric_pose_loss(batch, p)["num_valid_h"] == 0


def test_contract_all_zero_pair_and_topk_nan():
    """An all-zero pair makes the outer torch.multinomial raise: zero result; with top-K at B = 4, avg_loss = 0/0."""
    batch = _cuda(loss_cases.case_batch("vits_topk_b4"))
    batch["final_scores"][2].zero_()
    res = _run(batch, loss_cases.case_cfg("vits_topk_b4"))
    assert _is_zero_result(res, 4) and math.isnan(float(res[0]))
    assert lo.metric_pose_loss(batch, LossParams(loss_cases.case_cfg("vits_topk_b4")))["num_valid_h"] == 0


def test_contract_few_positive_cells_and_sets():
    """Pair 1 with 300 positive cells (< 512): no failure, every positive cell in every set.  Pair 0 with 5: the inner
    draws take the 5 positive entries first, then fill; still no failure, as torch.multinomial does not raise."""
    batch = _cuda(loss_cases.case_batch("vits_vcre"))
    cfg = loss_cases.case_cfg("vits_vcre")
    p = LossParams(cfg)
    g = torch.Generator().manual_seed(8)
    for b, k in ((1, 300), (0, 5)):
        keep = torch.randperm(210 * 210, generator=g)[:k].to(DEV)
        row = batch["final_scores"][b].view(-1)
        new = torch.zeros_like(row)
        new[keep] = row[keep] + 1e-3
        row.copy_(new)
    sampled, inner, _, status = loss_search(batch["final_scores"], batch["kps0"], batch["depth_kp0"], batch["kps1"],
                                            batch["depth_kp1"], batch["K_color0"], batch["K_color1"], p, 5)
    assert status == 0
    IM = p.it_matches
    for b in (0, 1):
        posc = set(torch.nonzero(batch["final_scores"][b].view(-1)).view(-1).tolist())
        for s in range(IM):
            assert posc <= set(sampled[b * IM + s].tolist())
    pos0 = set(torch.nonzero(batch["final_scores"][0].view(-1)).view(-1).tolist())
    for h in range(IM * p.it_ransac):
        s = h // p.it_ransac
        first = {int(sampled[s, int(q)]) for q in inner[h, :5]}
        assert first == pos0
        assert len(set(inner[h].tolist())) == p.num_corr
    assert _run(batch, cfg)[3] == 1


def test_contract_zero_sum_set_sets_inner_bit():
    """An injected set of zero cells: the inner torch.multinomial would raise, so the zero result."""
    batch = _cuda(loss_cases.case_batch("vits_vcre"))
    cfg = loss_cases.case_cfg("vits_vcre")
    p = LossParams(cfg)
    zero_cells = torch.nonzero(batch["final_scores"][0].view(-1) == 0).view(-1)
    assert zero_cells.numel() >= p.n_sample
    outer = torch.from_numpy(FIX["vits_vcre/outer_idx"]).to(DEV).long()
    outer[1] = zero_cells[:p.n_sample]
    *_, status = loss_search(batch["final_scores"], batch["kps0"], batch["depth_kp0"], batch["kps1"], batch["depth_kp1"],
                             batch["K_color0"], batch["K_color1"], p, 5, outer)
    assert status == STATUS_INNER
    assert _is_zero_result(_run(batch, cfg, outer_idx=outer), 2)


def test_contract_topk_masks_gradient_rows():
    batch = _cuda(loss_cases.case_batch("vits_topk_b4"))
    avg, out, (grad,), nv = _run(batch, loss_cases.case_cfg("vits_topk_b4"))
    m = out["mask_topk"]
    assert nv == 1 and int(m.sum()) == 1                 # int(4 * 30 / 100) = 1 pair below the 2nd smallest baseline
    for b in range(4):
        assert (float(grad[b].abs().max()) > 0) == bool(m[b] > 0)
