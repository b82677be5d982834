"""The training loss with its differentiable tail in CUDA (MetricPoseLoss(cfg, cuda_tail=True), csrc/loss_tail.cu) against
the fp64 oracle (oracle/loss_oracle.py) with the oracle's draws injected, under tests/test_gpu_loss.py's bounds:
inliers_final equal apart from near-threshold flips; loss_value, baseline and avg_loss within 5e-4; probs_grad by
check_gradient; kps / depth gradients and avg_loss_rot / avg_loss_trans within 2 |fp32 oracle - fp64| + 5e-3 max|fp64|
(5e-4 for the two scalars).  Each comparison also runs the autograd tail on the same data and prints max(err / bound) of
both, per quantity.  The places: every loss fixture case, B = 8 at 720x540 under VCRE and POSE_ERR, both warm-up
configurations at B = 24, 480x360 (S = 64, pitch 864), and test_gpu_loss_configs.py's S / C / NUM_REF_STEPS sweep.

Then: bit-identical gradients over two calls; the zero result exactly where the autograd tail gives it; inference_mode
values equal to grad-mode values with nothing kept; a converted training model's step with an Adam update.
"""
import json
import os

import numpy as np
import pytest
import torch

from mickey_b200 import _lib
from mickey_b200.loss import LossParams, LossTail, MetricPoseLoss, _loss_search_bits, loss_search
from oracle import loss_oracle as lo
from tests import loss_cases
from tests.test_gpu_loss import EPS_M, check_gradient, production  # noqa: F401  (production: a fixture)
from tests.test_gpu_loss_configs import SWEEP, SWEEP_IDS, WARMUP, _padded, warmup  # noqa: F401  (warmup: a fixture)

pytestmark = pytest.mark.gpu
DEV = "cuda"
FIX = np.load(loss_cases.FIXTURE)
RATIOS = {}


def _cuda(batch):
    return {k: v.to(DEV) for k, v in batch.items()}


def _rel(got, want):
    got, want = got.detach().double(), want.detach().double()
    return float((got - want).abs().max() / want.abs().max().clamp_min(1e-30))


def _record(label, ratios):
    RATIOS[label] = ratios
    out_dir = os.environ.get("MICKEY_TEST_RESULTS")
    if out_dir:
        with open(os.path.join(out_dir, "loss_tail_ratios.json"), "w") as f:
            json.dump(RATIOS, f, indent=1)


def compare_tail(batch, cfg, generator=None, outer=None, inner=None, label=""):
    """Both tails against the fp64 oracle with the oracle's draws.  Asserts every bound for the CUDA tail; returns
    {"cuda": {quantity: err / bound}, "autograd": {...}} (None when a near-threshold flip makes values incomparable)."""
    p = LossParams(cfg)
    ref = lo.metric_pose_loss(batch, p, outer_idx=outer, inner_idx=inner, generator=generator)
    assert ref["num_valid_h"] == 1
    _, _, inl, status = loss_search(batch["final_scores"], batch["kps0"], batch["depth_kp0"], batch["kps1"],
                                    batch["depth_kp1"], batch["K_color0"], batch["K_color1"], p, 7, ref["sampled"],
                                    ref["inner"])
    assert status == 0
    diff = (inl.double() != ref["inliers_final"]).any(1)
    assert not bool((diff & ~(ref["margin"] <= EPS_M)).any())
    if bool(diff.any()):
        print(f"{label}: {int(diff.sum())} near-threshold flips in inliers_final; values not comparable")
        return None
    ref32 = lo.metric_pose_loss(batch, p, outer_idx=ref["sampled"], inner_idx=ref["inner"], dtype=torch.float32)
    ref["avg_loss"].backward()
    ref32["avg_loss"].backward()
    lv_max = float(ref["loss_value"].detach().abs().max())
    ratios = {}
    for variant in ("cuda", "autograd"):
        loss = MetricPoseLoss(cfg, cuda_tail=variant == "cuda")
        avg, out, (grad,), nv = loss(batch, seed=7, outer_idx=ref["sampled"], inner_idx=ref["inner"])
        assert nv == 1
        avg.backward()
        r = {"loss_value": _rel(loss.last_loss_value, ref["loss_value"]) / 5e-4,
             "baseline": _rel(loss.last_baseline, ref["baseline"]) / 5e-4,
             "avg_loss": _rel(avg, ref["avg_loss"]) / 5e-4,
             "probs_grad": float((grad.double() - ref["probs_grad"].double()).abs().max()) / (5e-4 * lv_max)}
        for k, rel in (("kps0", 5e-3), ("kps1", 5e-3), ("depth0", 5e-3), ("depth1", 5e-3), ("avg_loss_rot", 5e-4),
                       ("avg_loss_trans", 5e-4)):
            got = out[k].grad if k.startswith(("kps", "depth")) else out[k]
            want = ref[k].grad if k.startswith(("kps", "depth")) else ref[k]
            fp32 = ref32[k].grad if k.startswith(("kps", "depth")) else ref32[k]
            got, want, fp32 = got.detach().double(), want.detach().double(), fp32.detach().double()
            allowed = 2 * float((fp32 - want).abs().max()) + rel * float(want.abs().max())
            r[k] = float((got - want).abs().max()) / allowed
        if variant == "cuda":
            check_gradient(grad, ref["probs_grad"], ref["sampled"], ref["loss_value"].detach(), p.it_matches)
            assert torch.equal(out["mask_topk"].double(), ref["mask_topk"])
        ratios[variant] = r
    print(f"{label}: max(err / bound) " + json.dumps({v: {k: round(x, 4) for k, x in r.items()} for v, r in ratios.items()}))
    _record(label, ratios)
    bad = {k: x for k, x in ratios["cuda"].items() if not x <= 1}
    assert not bad, (label, bad)
    return ratios


@pytest.mark.parametrize("name", list(loss_cases.CASES))
def test_fixture_cases_match_oracle(name):
    compare_tail(_cuda(loss_cases.case_batch(name)), loss_cases.case_cfg(name),
                 outer=torch.from_numpy(FIX[f"{name}/outer_idx"]).long().to(DEV),
                 inner=torch.from_numpy(FIX[f"{name}/inner_idx"]).long().to(DEV), label=name)


@pytest.mark.parametrize("loss", ["VCRE", "POSE_ERR"])
def test_production_size_matches_oracle(production, loss):
    cfg = loss_cases.loss_cfg(loss=loss, it_matches=20, it_ransac=20, topk=True)
    compare_tail(production, cfg, generator=torch.Generator(DEV).manual_seed(11), label=f"production B=8 N=1938 {loss}")


@pytest.mark.parametrize("name", WARMUP)
def test_warmup_configs_match_oracle(warmup, name):
    cfg = loss_cases.reference_cfg(name)
    assert LossParams(cfg).n_sample == 64
    compare_tail(warmup, cfg, generator=torch.Generator(DEV).manual_seed(29), label=f"{name} B=24 N=850 S=64")


@pytest.mark.parametrize("S,C,n_ref,IR,padded,loss,null", SWEEP, ids=SWEEP_IDS)
def test_sweep_matches_oracle(S, C, n_ref, IR, padded, loss, null):
    batch = _cuda(loss_cases.case_batch("vits_vcre"))
    if padded:
        batch["final_scores"] = _padded(batch["final_scores"], 224)
    cfg = loss_cases.loss_cfg(loss=loss, null=null, it_matches=4, it_ransac=IR)
    g = cfg.LOSS_CLASS.GENERATE_HYPOTHESES
    cfg.LOSS_CLASS.SAMPLER.NUM_SAMPLES_MATCHES, g.NUM_CORR_3d3d, g.NUM_REF_STEPS = S, C, n_ref
    compare_tail(batch, cfg, generator=torch.Generator(DEV).manual_seed(S + C + IR), label=f"S {S} C {C} n_ref {n_ref} IR {IR}")


# ---- determinism, the zero result, inference mode ---------------------------------------------------------------------
def _grads(loss, batch, **kw):
    avg, out, (grad,), nv = loss(batch, **kw)
    assert nv == 1
    avg.backward()
    return [out[k].grad for k in ("kps0", "kps1", "depth0", "depth1")] + [grad, avg.detach()]


def test_two_calls_give_bit_identical_gradients(production):
    loss = MetricPoseLoss(loss_cases.loss_cfg(it_matches=20, it_ransac=20, topk=True), cuda_tail=True)
    a, b = _grads(loss, production, seed=99), _grads(loss, production, seed=99)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert all(bool((x != 0).any()) for x in a[:4])


def _zero_both(batch, cfg, **kw):
    """Both tails on the same batch: (num_valid_h, the result is the zero result) of each."""
    res = {}
    for cuda in (False, True):
        avg, out, (grad,), nv = MetricPoseLoss(cfg, cuda_tail=cuda)(batch, seed=5, **kw)
        res[cuda] = (nv, nv == 0 and float(grad.abs().max()) == 0 and float(out["avg_loss_rot"]) == 0)
    return res


def test_zero_result_where_the_autograd_tail_gives_it():
    name = "vits_vcre"
    cfg = loss_cases.case_cfg(name)
    outer = torch.from_numpy(FIX[f"{name}/outer_idx"]).long().to(DEV)
    inner = torch.from_numpy(FIX[f"{name}/inner_idx"]).long().to(DEV)
    N = 210
    cell = int(outer[1, 5])                      # a keypoint pair 0's second outer iteration drew
    cases = {}
    b = _cuda(loss_cases.case_batch(name))
    b["depth_kp0"][0, 0, cell // N] = float("nan")
    cases["nan depth at a drawn keypoint"] = (b, dict(outer_idx=outer, inner_idx=inner))
    b = _cuda(loss_cases.case_batch(name))
    b["kps1"][0, 1, cell % N] = float("inf")
    cases["inf kps at a drawn keypoint"] = (b, dict(outer_idx=outer, inner_idx=inner))
    b = _cuda(loss_cases.case_batch(name))
    b["final_scores"][1, 3, 4] = float("nan")
    cases["nan cell (pre-check bit)"] = (b, {})
    b = _cuda(loss_cases.case_batch(name))
    b["final_scores"][1].zero_()
    cases["all-zero pair (outer multinomial bit)"] = (b, {})
    b = _cuda(loss_cases.case_batch(name))
    zero_cells = torch.nonzero(b["final_scores"][0].view(-1) == 0).view(-1)
    o = outer.clone()
    o[1] = zero_cells[:512]
    cases["zero-sum set (inner multinomial bit)"] = (b, dict(outer_idx=o))
    b = _cuda(loss_cases.case_batch(name))
    cases["valid batch"] = (b, dict(outer_idx=outer, inner_idx=inner))
    for label, (batch, kw) in cases.items():
        r = _zero_both(batch, cfg, **kw)
        print(f"{label}: autograd tail {r[False]}, CUDA tail {r[True]}")
        assert r[True] == r[False], label
        assert r[True] == ((1, False) if label == "valid batch" else (0, True)), label


def test_inference_mode_values_equal_grad_mode_and_keep_nothing():
    name = "vits_topk_b4"
    cfg = loss_cases.case_cfg(name)
    batch = _cuda(loss_cases.case_batch(name))
    kw = dict(seed=3, outer_idx=torch.from_numpy(FIX[f"{name}/outer_idx"]).to(DEV),
              inner_idx=torch.from_numpy(FIX[f"{name}/inner_idx"]).to(DEV))
    loss = MetricPoseLoss(cfg, cuda_tail=True)
    avg, out, (grad,), nv = loss(batch, **kw)
    lv = loss.last_loss_value
    with torch.inference_mode():
        avg_i, out_i, (grad_i,), nv_i = loss(batch, **kw)
    assert nv_i == nv == 1 and torch.equal(loss.last_loss_value, lv) and torch.equal(avg_i, avg.detach())
    assert torch.equal(grad_i, grad)
    for k in ("avg_loss_rot", "avg_loss_trans"):
        assert torch.equal(out_i[k], out[k].detach())
    # LossTail itself: the workspace is kept only when a backward can follow
    p = loss.p
    sampled, _, bits, status = _loss_search_bits(batch["final_scores"], batch["kps0"], batch["depth_kp0"], batch["kps1"],
                                                 batch["depth_kp1"], batch["K_color0"], batch["K_color1"], p, 3,
                                                 kw["outer_idx"], kw["inner_idx"])
    assert status == 0
    B, N = batch["kps0"].shape[0], batch["kps0"].shape[2]
    ws_bytes = _lib.load().mk_loss_tail_ws_bytes(B, N, p.it_matches, p.it_ransac, p.n_sample)
    consts = [batch[k].float().contiguous() for k in ("K_color0", "K_color1", "Kori_color0", "Kori_color1", "T_0to1")]
    leaves = [batch[k].detach().clone().requires_grad_() for k in ("kps0", "depth_kp0", "kps1", "depth_kp1")]
    grid = loss._vcre_grid(torch.device(DEV))
    kept = {}
    for mode in ("inference", "grad"):
        torch.cuda.synchronize()
        m0 = torch.cuda.memory_allocated()
        if mode == "inference":
            with torch.inference_mode():
                res = LossTail.apply(*leaves, sampled, bits, *consts, grid, p, False)
        else:
            res = LossTail.apply(*leaves, sampled, bits, *consts, grid, p, True)
        kept[mode] = torch.cuda.memory_allocated() - m0
        outs = [r.detach().clone() for r in res[:3]]
        if mode == "grad":
            assert all(torch.equal(a, b) for a, b in zip(outs, prev))
        prev = outs
        del res
    print(f"memory held after the call: {kept}, workspace {ws_bytes} bytes")
    assert kept["inference"] < ws_bytes <= kept["grad"]


# ---- a converted training model ----------------------------------------------------------------------------------------
def test_converted_model_trains_with_the_cuda_tail():
    """use_cuda_modules(model, cuda_tail=True), then a B = 8, 720x540 training step through backward_step (restated in
    test_gpu_training_lifecycle.train_step) and one Adam step: finite gradients and parameters, and the step moves them."""
    from mickey_b200.training import use_cuda_modules
    from tests.test_gpu_heads_training import converted_model, step_batch
    from tests.test_gpu_training_lifecycle import train_step
    model = converted_model("curriculum_learning")
    loss = model.loss_fn
    assert use_cuda_modules(model, cuda_tail=True) is model and model.loss_fn is loss and loss.cuda_tail
    ims, data = step_batch(8, 540, 720, seed=31)
    _, upstream, total, grads = train_step(model, ims, data)
    assert all(bool(torch.isfinite(g).all()) for g in grads.values()) and np.isfinite(total)
    assert any(bool((u != 0).any()) for u in upstream[1:])
    opt = torch.optim.Adam(model.parameters(), lr=model.cfg.TRAINING.LR, eps=1e-6)
    with_grad = {n: p.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
    opt.step()
    params = dict(model.named_parameters())
    assert all(bool(torch.isfinite(params[n]).all()) for n in with_grad)
    moved = sum(not torch.equal(params[n].detach(), v) for n, v in with_grad.items())
    print(f"Adam step: {moved} of {len(with_grad)} parameters with a gradient moved, total norm {total:.4g}")
    assert moved > 0
