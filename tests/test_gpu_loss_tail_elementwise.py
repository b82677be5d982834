"""The CUDA loss tail (LossTail, csrc/loss_tail.cu) element by element against the fp64 closed form on its own fp32
inputs and fp32 K^-1, under tests/loss_tail_check.py's derived bound (|y - y*| <= 2^-24 |y*| + E).  The autograd tail
is fp32 and is not held to this bound.

- Every place of test_gpu_loss_tail.py (7 fixtures, B = 8 720x540 VCRE / POSE_ERR, both warm-up configs at B = 24, the
  12-row S / C / NUM_REF_STEPS sweep) with the oracle's draws injected.  The tail runs on the search's own inlier bits
  and the oracle on the same bits, so a near-threshold flip cannot make values incomparable.  Each place also reports the
  new element bound against test_gpu_loss.py::compare's normwise allowance.
- The planted table and the launch-shape edges (IR 1..40, S 32 / 2048, IM S at the scatter's 2048-entry tile edge, N at
  the scatter's block edges, B 1 / 3), through LossTail directly.
- Each planted mutation is rejected against the kernel's outputs on at least one case.
- A pair's outputs are the same bits alone and inside a batch of 8.
- The degenerate-hypothesis contract: a hypothesis whose G_H is not finite makes every keypoint its set drew non-finite,
  and nothing else.  W1 = 0 and W1 = 1 give H = 0 exactly and must show it; three inlier entries sharing one image-0
  keypoint and two distinct points give H = 0 / rank 1 only to rounding, where G_H may stay finite.  The autograd
  tail's pattern is printed beside each.
"""
import json
import time

import numpy as np
import pytest
import torch

from mickey_b200.loss import LossParams, LossTail, MetricPoseLoss, _loss_search_bits
from oracle import loss_oracle as lo
from oracle import loss_tail_oracle as lto
from tests import elementwise, loss_cases
from tests import loss_tail_check as ltc
from tests.test_gpu_loss import production  # noqa: F401  (a fixture)
from tests.test_gpu_loss_configs import SWEEP, SWEEP_IDS, WARMUP, _padded, warmup  # noqa: F401  (warmup: a fixture)
from tests.test_loss_tail_check_host import degenerate

pytestmark = pytest.mark.gpu
DEV = "cuda"
FIX = np.load(loss_cases.FIXTURE)
T0 = time.time()


def run_tail(pl_inputs, p, ups):
    """LossTail forward and backward on the GPU: ({quantity: fp32 tensor on the CPU}, status)."""
    kps0, d0, kps1, d1, K0, K1, Ko0, Ko1, T, sampled, bits = (x.to(DEV).contiguous() for x in pl_inputs)
    leaves = [x.clone().requires_grad_() for x in (kps0, d0, kps1, d1)]
    grid = MetricPoseLoss.__new__(MetricPoseLoss)
    grid._grid = {}
    g = grid._vcre_grid(torch.device(DEV))
    lv, lr, lt, status = LossTail.apply(*leaves, sampled, bits, K0, K1, Ko0, Ko1, T, g, p, True)
    grads = torch.autograd.grad([lv, lr, lt], leaves, [u.float().to(DEV) for u in ups])
    out = {"loss_value": lv, "loss_rot": lr, "loss_trans": lt}
    out.update(dict(zip(("dkps0", "ddepth0", "dkps1", "ddepth1"), grads)))
    return {k: v.detach().cpu() for k, v in out.items()}, int(status.item())


def planted_inputs(pl):
    return (pl.kps0, pl.d0, pl.kps1, pl.d1, pl.K, pl.K, pl.K, pl.K, pl.T, pl.sampled, ltc.Planted.pack(pl.inl, pl.p.n_sample))


def _record(label, ratios):
    for k, v in ratios.items():
        elementwise.record(f"loss_tail {k}", label, v)
    print(f"{label}: max(err / bound) " + json.dumps({k: float(f"{v:.3g}") for k, v in ratios.items()}))


def check_planted(pl, label, ups=None):
    ups = ups or pl.upstream()
    got, status = run_tail(planted_inputs(pl), pl.p, ups)
    assert status == 0, label
    want = pl.oracle(ups)
    ratios, _ = ltc.compare(got, want, pl.p, pl.tgt_t(), label)
    _record(label, ratios)
    return got, want, ups


# ---- the existing places --------------------------------------------------------------------------------------------
def check_place(batch, cfg, label, generator=None, outer=None, inner=None):
    p = LossParams(cfg)
    ref = lo.metric_pose_loss(batch, p, outer_idx=outer, inner_idx=inner, generator=generator)
    sampled, _, bits, status = _loss_search_bits(batch["final_scores"], batch["kps0"], batch["depth_kp0"], batch["kps1"],
                                                 batch["depth_kp1"], batch["K_color0"], batch["K_color1"], p, 7,
                                                 ref["sampled"], ref["inner"])
    assert status == 0
    f32 = lambda k: batch[k].float().contiguous()
    inputs = (f32("kps0"), f32("depth_kp0"), f32("kps1"), f32("depth_kp1"), f32("K_color0"), f32("K_color1"),
              f32("Kori_color0"), f32("Kori_color1"), f32("T_0to1"), sampled, bits)
    B = batch["kps0"].shape[0]
    g = torch.Generator().manual_seed(3)
    ups = [torch.randn(B * p.it_matches, generator=g).double() for _ in range(3)]        # fp32 values, as the kernel gets
    got, st = run_tail(inputs, p, ups)
    assert st == 0
    c = [x.cpu() for x in inputs]
    inl = torch.from_numpy(((bits.cpu().numpy().view(np.uint32)[..., None] >> np.arange(32, dtype=np.uint32)) & 1)
                           .reshape(bits.shape[0], -1).astype(np.float64))
    T = c[8].double()
    Kinv = (lto.kernel_kinv(c[4]), lto.kernel_kinv(c[5]))
    for K in c[4:6]:
        assert ltc.kinv_is_safe(K)
    args = [x.double() for x in c[:8]] + [T[:, :3, :3], T[:, :3, 3:].transpose(1, 2), c[9].cpu(), inl]
    want = lto.tail_closed_form(*args, ltc.kernel_params(p), *ups, Kinv=Kinv, grid=ltc.KERNEL_GRID)
    ratios, _ = ltc.compare(got, want, p, T[:, :3, 3:].transpose(1, 2), label)
    _record(label, ratios)
    # the new element bound against test_gpu_loss.py::compare's allowance (fp32 autograd tail as its 'fp32 oracle')
    E, _ = ltc.bounds(want, p, T[:, :3, 3:].transpose(1, 2))
    leaves = [x.float().clone().requires_grad_() for x in c[:4]]
    vals = lto.tail_autograd(*leaves, *[x.float() for x in c[4:8]], T[:, :3, :3].float(),
                             T[:, :3, 3:].transpose(1, 2).float(), c[9], inl.float(), p)
    grads = torch.autograd.grad(sum((v * u.float()).sum() for v, u in zip(vals, ups)), leaves)
    old = {}
    for k, v in zip(("loss_value", "loss_rot", "loss_trans"), vals):
        old[k] = 5e-4 * float(want[k].abs().max())
    for k, g32 in zip(("dkps0", "ddepth0", "dkps1", "ddepth1"), grads):
        old[k] = 2 * float((g32.double() - want[k]).abs().max()) + 5e-3 * float(want[k].abs().max())
    rel = {k: float((ltc.U32 * want[k].abs() + E[k]).max()) / old[k] for k in ltc.QUANTITIES}
    print(f"{label}: max(new element bound) / old normwise allowance " + json.dumps({k: float(f"{v:.3g}") for k, v in rel.items()}))
    for k, v in rel.items():
        elementwise.record(f"loss_tail new/old {k}", label, v)


def _cuda(batch):
    return {k: v.to(DEV) for k, v in batch.items()}


@pytest.mark.parametrize("name", list(loss_cases.CASES))
def test_fixture_cases_elementwise(name):
    check_place(_cuda(loss_cases.case_batch(name)), loss_cases.case_cfg(name), name,
                outer=torch.from_numpy(FIX[f"{name}/outer_idx"]).long().to(DEV),
                inner=torch.from_numpy(FIX[f"{name}/inner_idx"]).long().to(DEV))


@pytest.mark.parametrize("loss", ["VCRE", "POSE_ERR"])
def test_production_size_elementwise(production, loss):
    cfg = loss_cases.loss_cfg(loss=loss, it_matches=20, it_ransac=20, topk=True)
    check_place(production, cfg, f"production B=8 N=1938 {loss}", generator=torch.Generator(DEV).manual_seed(11))


@pytest.mark.parametrize("name", WARMUP)
def test_warmup_configs_elementwise(warmup, name):
    check_place(warmup, loss_cases.reference_cfg(name), f"{name} B=24 N=850 S=64",
                generator=torch.Generator(DEV).manual_seed(29))


@pytest.mark.parametrize("S,C,n_ref,IR,padded,loss,null", SWEEP, ids=SWEEP_IDS)
def test_sweep_elementwise(S, C, n_ref, IR, padded, loss, null):
    batch = _cuda(loss_cases.case_batch("vits_vcre"))
    if padded:
        batch["final_scores"] = _padded(batch["final_scores"], 224)
    cfg = loss_cases.loss_cfg(loss=loss, null=null, it_matches=4, it_ransac=IR)
    g = cfg.LOSS_CLASS.GENERATE_HYPOTHESES
    cfg.LOSS_CLASS.SAMPLER.NUM_SAMPLES_MATCHES, g.NUM_CORR_3d3d, g.NUM_REF_STEPS = S, C, n_ref
    check_place(batch, cfg, f"S {S} C {C} n_ref {n_ref} IR {IR}", generator=torch.Generator(DEV).manual_seed(S + C + IR))


# ---- the planted table and the shape edges ---------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(ltc.planted_table()))
def test_planted_table_elementwise(name):
    check_planted(ltc.build(name), name)


@pytest.mark.parametrize("kw", ltc.SHAPES, ids=[ltc.shape_id(k) for k in ltc.SHAPES])
def test_shape_edges_elementwise(kw):
    pl = ltc.build(kw)
    got, _, _ = check_planted(pl, ltc.shape_id(kw))
    # keypoints no entry drew get exactly 0
    drawn = torch.zeros(pl.B, pl.N, dtype=torch.bool)
    cell = pl.sampled.long()
    bidx = torch.arange(pl.B).repeat_interleave(pl.p.it_matches)[:, None].expand_as(cell)
    drawn[bidx.reshape(-1), (cell // pl.N).reshape(-1)] = True
    for k in ("dkps0", "ddepth0"):
        assert bool((got[k].transpose(1, 2)[~drawn] == 0).all()), k


def test_shared_keypoints_elementwise():
    """One keypoint drawn by entry 0 of every outer iteration of pair 0 (IM = 64, so its sum crosses no tile but takes
    64 contributions), checked element by element."""
    pl = ltc.build(dict(B=2, N=4176, IM=64, IR=4, S=64))
    k = ltc.shared_keypoints(pl)
    got, want, _ = check_planted(pl, "one keypoint drawn by every outer iteration")
    assert float(want["dkps0"][0, :, k].abs().max()) > 0


def test_mutations_are_rejected_against_the_kernel():
    """Every new mutation of the oracle, taken as the reference, is rejected against the kernel's outputs somewhere."""
    rejected = {m: [] for m in lto.TAIL_MUTATIONS[5:]}
    for name in ("well_all", "vcre_behind", "vcre_far_tgt", "branch_VCRE_soft1_null1", "mirrored_gap_1e-02"):
        pl = ltc.build(name)
        ups = pl.upstream()
        got, _ = run_tail(planted_inputs(pl), pl.p, ups)
        for m in rejected:
            _, fails = ltc.compare(got, pl.oracle(ups, m), pl.p, pl.tgt_t(), name, mutations_ok=True)
            if fails:
                rejected[m].append(name)
    print("rejected against the kernel on:", rejected)
    assert all(rejected.values()), rejected


def test_pair_alone_equals_pair_in_a_batch():
    pl = ltc.build(dict(B=8, N=300, IM=2, IR=8, S=64))
    ups = pl.upstream()
    got8, _ = run_tail(planted_inputs(pl), pl.p, ups)
    b, IM, IR = 5, pl.p.it_matches, pl.p.it_ransac
    one = [pl.kps0[b:b + 1], pl.d0[b:b + 1], pl.kps1[b:b + 1], pl.d1[b:b + 1]] + [pl.K[b:b + 1]] * 4
    bits = ltc.Planted.pack(pl.inl, pl.p.n_sample)[b * IM * IR:(b + 1) * IM * IR]
    one += [pl.T[b:b + 1], pl.sampled[b * IM:(b + 1) * IM], bits]
    got1, _ = run_tail(one, pl.p, [u[b * IM:(b + 1) * IM] for u in ups])
    for k in ltc.QUANTITIES:
        a = got8[k][b * IM:(b + 1) * IM] if k.startswith("loss") else got8[k][b:b + 1]
        assert torch.equal(a, got1[k]), k


# ---- the degenerate-hypothesis contract -----------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["w0", "w1", "shared", "rank1"])
def test_degenerate_hypothesis_makes_its_set_non_finite(kind):
    pl = degenerate(kind)
    ups = pl.upstream()
    got, status = run_tail(planted_inputs(pl), pl.p, ups)
    assert status == 0
    assert all(bool(torch.isfinite(got[k]).all()) for k in ("loss_value", "loss_rot", "loss_trans"))
    N, S = pl.N, pl.p.n_sample
    set0 = pl.sampled[0].long()
    drawn0, drawn1 = torch.zeros(N, dtype=torch.bool), torch.zeros(N, dtype=torch.bool)
    drawn0[set0 // N], drawn1[set0 % N] = True, True
    bad0 = ~torch.isfinite(got["dkps0"][0]).all(0) | ~torch.isfinite(got["ddepth0"][0, 0])
    bad1 = ~torch.isfinite(got["dkps1"][0]).all(0) | ~torch.isfinite(got["ddepth1"][0, 0])
    # the autograd tail (fp32, torch.svd's backward) on the same inputs
    leaves = [x.to(DEV).clone().requires_grad_() for x in (pl.kps0, pl.d0, pl.kps1, pl.d1)]
    K, T = pl.K.to(DEV), pl.T.to(DEV)
    vals = lto.tail_autograd(*leaves, K, K, K, K, T[:, :3, :3], T[:, :3, 3:].transpose(1, 2), pl.sampled.to(DEV),
                             pl.inl.float().to(DEV), pl.p)
    ag = torch.autograd.grad(sum((v * u.float().to(DEV)).sum() for v, u in zip(vals, ups)), leaves)
    ag_bad0 = (~torch.isfinite(ag[0][0]).all(0) | ~torch.isfinite(ag[1][0, 0])).cpu()
    print(f"{kind}: CUDA tail non-finite keypoints {int(bad0.sum())} / {int(bad1.sum())} (set 0 draws "
          f"{int(drawn0.sum())} / {int(drawn1.sum())}); autograd tail {int(ag_bad0.sum())} in image 0, "
          f"max |grad| {float(torch.nan_to_num(ag[0], nan=0.0, posinf=0.0, neginf=0.0).abs().max()):.3g}")
    if kind in ("w0", "w1"):
        # H is exactly zero (a = X for W1 = 1), so M = 0 and G_H is NaN: every keypoint the set drew, and only those
        assert torch.equal(bad0, drawn0) and torch.equal(bad1, drawn1), kind
    else:
        # H is zero or rank 1 only to rounding: G_H may come out finite (and huge); where it does not, the rule holds
        assert (not bool(bad0.any()) or torch.equal(bad0, drawn0)) and (not bool(bad1.any()) or torch.equal(bad1, drawn1))


def test_wall_time_report():
    print(f"test_gpu_loss_tail_elementwise.py: {time.time() - T0:.1f} s to here")
