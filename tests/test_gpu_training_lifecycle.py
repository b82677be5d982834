"""A converted MicKey training model (mickey_b200.training.use_cuda_modules) beyond one train-mode backward: the heads in
eval mode, running statistics over successive optimiser steps, the validation step, a validation as the model's first
call, and the checkpoint the inference engine loads.

Every comparison with fp64 uses test_gpu_heads_training.py's gate: ||ours - fp64|| / ||fp64|| at most 1.5x the error of
the same chain in eager fp32 torch on the GPU under torch's default TF32 flags, with an absolute floor of 1e-6 (the
training step's gradients also per tensor at 3x, as there).  The fp64 and eager chains start from the model's current
state and the same backbone features and, in training, take the same upstream gradients, so a stale weight or statistic
shows as an error of its own rather than being hidden in accumulated drift.  With MICKEY_TEST_RESULTS set to a directory,
the measured errors and ratios are written to training_lifecycle_ratios.json there.

The parts of the reference's MicKeyTrainingModel (lib/models/MicKey/model.py) that these runs go through are restated
here with line references, since the converted model is model_from_tree's stand-in: is_eval_model, validation_step up to
the loss (its pose metrics stay the reference's torch code), backward_step and on_save_checkpoint.
"""
import copy
import json
import os

import pytest
import torch

from oracle import heads_oracle as ho
from oracle import mickey_oracle as mo
from tests.common import synthetic_pair
from tests.golden.make_training_tree import training_cfg
from tests.test_gpu_heads_training import (DEV, FLOOR, HEADS, RATIO, SHAPES, STEP_CASES, STEP_TENSOR_RATIO,
                                           converted_model, correspondences, extract, match, rel, seeded_head,
                                           step_batch)

pytestmark = pytest.mark.gpu
ORDER = ("det_offset", "depth_head", "det_head", "dsc_head")       # MicKey_Extractor.forward's call order
RESULTS = {}
STEPS = 3
TRAINED = {}                                                        # case -> the model after the lockstep test's steps


def record(key, errs):
    dump(key, {k: {"ours": a, "eager_fp32_tf32": b, "ratio": a / b if b else None} for k, (a, b) in errs.items()})


def dump(key, value):
    RESULTS[key] = value
    out_dir = os.environ.get("MICKEY_TEST_RESULTS")
    if out_dir:
        with open(os.path.join(out_dir, "training_lifecycle_ratios.json"), "w") as f:
            json.dump(RESULTS, f, indent=1)


def over(errs, ratio=RATIO):
    return {k: e for k, e in errs.items() if e[0] > ratio * e[1] + FLOOR}


# ---- the reference's MicKeyTrainingModel, restated ---------------------------------------------------------------------
def is_eval_model(model, is_eval):
    """MicKeyTrainingModel.is_eval_model (model.py:308-318)."""
    ex = model.compute_matches.extractor
    for name in ("depth_head", "det_offset", "dsc_head", "det_head"):
        if is_eval:
            getattr(ex, name).eval()
        else:
            getattr(ex, name).train()


def on_save_checkpoint(checkpoint):
    """MicKeyTrainingModel.on_save_checkpoint (model.py:291-298): the frozen DINOv2 tensors stay out of the checkpoint."""
    for key in [k for k in checkpoint["state_dict"] if "dinov2" in k]:
        del checkpoint["state_dict"][key]


def forward_pair(model, ims):
    """self(batch): ComputeCorrespondences.forward (compute_correspondences.py:52-92), two extractor calls with separate
    batch statistics, the matcher and kp_scores; prepare_batch_for_loss's final_scores (model.py:198-203)."""
    ex = model.compute_matches.extractor
    feats, cs = [], []
    for im in ims:
        f, outs = extract(ex, im)
        feats.append(f)
        cs.append(correspondences(*outs))
    return feats, cs, match(model.compute_matches.matcher.matching_mat, cs[0], cs[1])


def loss_batch(data, cs, final):
    return dict(data, final_scores=final, kps0=cs[0][0], kps1=cs[1][0], depth_kp0=cs[0][1], depth_kp1=cs[1][1])


def head_grads(model):
    ex = model.compute_matches.extractor
    grads = {f"{n}.{k}": p.grad for n in HEADS for k, p in getattr(ex, n).named_parameters() if p.requires_grad}
    grads["matching_mat.dustbin_score"] = model.compute_matches.matcher.matching_mat.dustbin_score.grad
    return grads


def train_step(model, ims, data):
    """training_step (model.py:51-59) and backward_step (:91-147) up to opt.step(): zero_grad, avg_loss.backward(), the
    backward through the heads and the matcher, clip_grad_norm_.  Returns (backbone features, upstream gradients, the
    clipped total norm, {name: gradient after clipping})."""
    feats, cs, final = forward_pair(model, ims)
    batch = loss_batch(data, cs, final)
    avg_loss, outputs, probs_grad, num_its = model.loss_fn(batch)
    assert num_its == 1
    for p in model.parameters():
        p.grad = None
    avg_loss.backward()
    upstream = (probs_grad[0], outputs["kps0"].grad, outputs["kps1"].grad, outputs["depth0"].grad, outputs["depth1"].grad)
    assert all(u is not None and bool(torch.isfinite(u).all()) for u in upstream)
    torch.autograd.backward((torch.log(batch["final_scores"] + 1e-16), batch["kps0"], batch["kps1"], batch["depth_kp0"],
                             batch["depth_kp1"]), upstream)
    grads = head_grads(model)
    assert all(g is not None for g in grads.values())
    total = float(torch.nn.utils.clip_grad_norm_(model.parameters(), max_norm=5))
    return feats, upstream, total, grads


def loss_draws(loss_fn, final, seed):
    """Draws to inject into the loss: the outer sets by score without replacement as the reference's multinomial draws
    them, the inner C-of-S sets uniformly without replacement."""
    p = loss_fn.p
    B, N = final.shape[0], final.shape[1]
    g = torch.Generator(device=final.device).manual_seed(seed)
    w = final.detach().reshape(B, 1, N * N).expand(B, p.it_matches, N * N).reshape(B * p.it_matches, N * N)
    outer = torch.multinomial(w, p.n_sample, replacement=False, generator=g)
    inner = torch.rand(B * p.it_matches * p.it_ransac, p.n_sample, generator=g, device=final.device).argsort(1)
    return outer.int(), inner[:, :p.num_corr].int()


def validation_step(model, ims, data, seed):
    """MicKeyTrainingModel.validation_step (model.py:66-89) up to the loss, with the loss's draws injected.  Its pose
    metrics (e2e_Procrustes, pose_error_torch, vcre_torch) stay the reference's torch code and are not run here."""
    is_eval_model(model, True)
    feats, cs, final = forward_pair(model, ims)
    batch = loss_batch(data, cs, final)
    draws = loss_draws(model.loss_fn, final, seed)
    avg_loss, outputs, probs_grad, num_its = model.loss_fn(batch, seed=seed, outer_idx=draws[0], inner_idx=draws[1])
    outputs["loss"] = avg_loss
    return feats, cs, batch, outputs, draws


# ---- the fp64 and eager fp32 chains --------------------------------------------------------------------------------------
def head_state(model):
    ex = model.compute_matches.extractor
    return {n: {k: (t.detach().clone(), t.requires_grad) for k, t in getattr(ex, n).state_dict(keep_vars=True).items()}
            for n in HEADS}


def cast_state(sd0, dtype, leaves=None, prefix=""):
    sd = {}
    for n, (t, rg) in sd0.items():
        v = t.detach().to(dtype if t.is_floating_point() else t.dtype).clone()
        sd[n] = v.requires_grad_() if rg and leaves is not None else v
        if rg and leaves is not None:
            leaves[prefix + n] = sd[n]
    return sd


def step_chain(model, sd0, feats, upstream, dtype):
    """The training step from the same backbone features in `dtype`: every head through oracle/heads_oracle.py in train
    mode, twice (once per image set, the second call's running-statistics update starting from the first one's result),
    the matcher and the outer product, driven by the same upstream gradients.  Returns ({name: gradient}, the total norm,
    {name: running statistic after both calls})."""
    from oracle.mickey_oracle import dual_softmax as ds_oracle
    config = model.cfg["MICKEY"]
    leaves = {}
    sds = {n: cast_state(sd0[n], dtype, leaves, n + ".") for n in HEADS}
    mat = model.compute_matches.matcher.matching_mat
    dustbin = mat.dustbin_score.detach().to(dtype).clone().requires_grad_()
    leaves["matching_mat.dustbin_score"] = dustbin
    running, cs = {}, []
    for f in feats:
        outs = []
        for n in ORDER:
            out, run = ho.head_chain(sds[n], n, config, f.to(dtype))
            for k, v in run.items():
                sds[n][k] = v
                running[f"{n}.{k}"] = v
            outs.append(out)
        cs.append(correspondences(*outs))
    final = match(lambda d0, d1: ds_oracle(d0, d1, mat.temperature, dustbin), cs[0], cs[1])
    torch.autograd.backward((torch.log(final + 1e-16), cs[0][0], cs[1][0], cs[0][1], cs[1][1]),
                            tuple(u.to(dtype) for u in upstream))
    grads = {n: t.grad for n, t in leaves.items()}
    return grads, float(torch.stack([g.double().norm() for g in grads.values()]).norm()), running


def eval_chain(model, sd0, feats, dtype):
    """The eval-mode forward of both image sets from the same backbone features in `dtype`: scr, kps, depth, dsc and
    final_scores."""
    config = model.cfg["MICKEY"]
    sds = {n: cast_state(sd0[n], dtype) for n in HEADS}
    mat = model.compute_matches.matcher.matching_mat
    with torch.no_grad():
        cs = [correspondences(*[ho.head_chain(sds[n], n, config, f.to(dtype), train=False)[0] for n in ORDER])
              for f in feats]
        final = match(lambda d0, d1: mo.dual_softmax(d0, d1, mat.temperature, mat.dustbin_score.detach().to(dtype)),
                      cs[0], cs[1])
    return pair_outputs(cs, final)


def pair_outputs(cs, final):
    cat = lambda i: torch.cat([cs[0][i], cs[1][i]])
    return {"kps": cat(0), "depth": cat(1), "scr": cat(2), "dsc": cat(3), "final_scores": final}


# ---- a. each head in eval mode ---------------------------------------------------------------------------------------
EVAL_SHAPES = SHAPES + [(1, 1, 1), (2, 7, 7), (2, 5, 9)]
# cuDNN runs the eager chain's convolutions at these small edge shapes in full fp32 even under allow_tf32, so there the
# eager chain is no TF32 yardstick (its output error is 1e-5 or less, ours that of TF32): at the edges an error is also
# accepted up to 2^-10 on the output and dx, and up to 5e-2 on a parameter gradient, about the largest gradient error
# both chains show at the training shapes
EDGE_FLOOR = {"out": 2 ** -10, "dx": 2 ** -10, "grad": 5e-2}


def eval_head_chain(sd0, name, config, x, go, dtype):
    sd = cast_state(sd0, dtype, leaves={})
    xx = x.to(dtype).clone().requires_grad_()
    out, running = ho.head_chain(sd, name, config, xx, train=False)
    assert running == {}
    names = [n for n, (t, rg) in sd0.items() if rg]
    grads = torch.autograd.grad(out, [xx] + [sd[n] for n in names], go.to(dtype))
    return {"out": out.detach(), "dx": grads[0], **dict(zip(names, grads[1:]))}


@pytest.mark.parametrize("shape", EVAL_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("name", list(HEADS))
def test_head_eval_mode_against_fp64(name, shape):
    """Each head in eval mode with seeded running statistics: no_grad, inference_mode and the grad-enabled (saving) path
    give the same bits and change no parameter, statistic or counter; output, input gradient and every parameter
    gradient against the fp64 eval chain, gated as the training step's gradients are: the output and dx at 1.5x the
    eager chain, all parameter gradients as one vector at 1.5x, each alone at 3x.  B = 1 at 1 x 1 is legal in eval mode only; at 7 x 7 the score head has one
    interior cell, at 5 x 9 and 1 x 1 none, and its output is exactly zero."""
    B, h, w = shape
    config = training_cfg()["MICKEY"]
    head = seeded_head(HEADS[name], config, seed=20 + len(name)).eval()
    before = {n: t.detach().clone() for n, t in head.state_dict().items()}
    sd0 = {n: (t.detach().clone(), t.requires_grad) for n, t in head.state_dict(keep_vars=True).items()}
    g = torch.Generator(device=DEV).manual_seed(B * h * w + 1)
    x = torch.randn(B, 1024, h, w, generator=g, device=DEV)
    with torch.no_grad():
        out_no_grad = head(x)
    with torch.inference_mode():
        out_inference = head(x)
    xr = x.clone().requires_grad_()
    out = head(xr)
    assert out.requires_grad
    assert torch.equal(out_no_grad, out_inference) and torch.equal(out_no_grad, out.detach())
    go = torch.randn(out.shape, generator=g, device=DEV)
    out.backward(go)
    after = head.state_dict()
    assert list(after) == list(before)
    changed = [n for n in before if not torch.equal(after[n], before[n])]
    assert not changed, f"eval mode changed {changed}"
    if name == "det_head" and min(h, w) <= 2 * ho.BORDER:
        assert torch.equal(out, torch.zeros_like(out))
    ours = {"out": out.detach(), "dx": xr.grad, **{n: p.grad for n, p in head.named_parameters() if p.requires_grad}}
    ref = eval_head_chain(sd0, name, config, x, go, torch.float64)
    eager = eval_head_chain(sd0, name, config, x, go, torch.float32)
    assert set(ours) == set(ref)
    errs = {k: (rel(ours[k], ref[k]), rel(eager[k], ref[k])) for k in ref}
    params = [k for k in ref if k not in ("out", "dx")]
    cat = lambda g: torch.cat([g[k].double().flatten() for k in params])
    groups = {"all parameters": (rel(cat(ours), cat(ref)), rel(cat(eager), cat(ref)))}
    record(f"eval {name} {B}x{h}x{w}", {**groups, **errs})
    edge = shape not in SHAPES
    floor = lambda k: (EDGE_FLOOR["grad" if k in params or k in groups else k] if edge else 0.0)
    bad = {k: e for k, e in {**groups, **errs}.items()
           if e[0] > max((STEP_TENSOR_RATIO if k in params else RATIO) * e[1], floor(k)) + FLOOR}
    assert not bad, f"{name} {shape} eval mode (ours, eager fp32) relative errors: {bad}"


# ---- b. running statistics and successive steps, in lockstep with fp64 -----------------------------------------------
def bn_counters(model):
    ex = model.compute_matches.extractor
    return {f"{n}.{k}": int(b) for n in HEADS for k, b in getattr(ex, n).named_buffers() if k.endswith("num_batches_tracked")}


@pytest.mark.parametrize("case", list(STEP_CASES))
def test_successive_steps_in_lockstep_with_fp64(case):
    """Three steps as the reference takes them, Adam(lr=TRAINING.LR, eps=1e-6) as configure_optimizers (model.py:282-289)
    builds it.  At each step the chains start from the model's current state: every gradient gated as in the single-step
    test, every running statistic against two successive fp64 updates, num_batches_tracked up by exactly 2.  Two
    differences from the single-step test: the clipped total norm is held to what the gradients' error allows rather than
    to the eager chain's (one scalar, whose error a lucky cancellation makes arbitrarily small in either chain), and a
    single tensor is also accepted up to 5e-2, as at the eval-mode edges: at the warm-up's 16 x 15 maps cuDNN can run the
    eager chain's narrow last-block convolutions in full fp32 (every head's gradients as one vector stay at 1.5x)."""
    assert torch.backends.cudnn.allow_tf32
    config, B, H, W = STEP_CASES[case]
    torch.manual_seed(0)
    model = converted_model(config)
    ex = model.compute_matches.extractor
    opt = torch.optim.Adam(model.parameters(), lr=model.cfg.TRAINING.LR, eps=1e-6)
    for step in range(STEPS):
        sd0 = head_state(model)
        counters = bn_counters(model)
        ims, data = step_batch(B, H, W, seed=100 * (step + 1) + B)
        opt.zero_grad()
        feats, upstream, total, ours = train_step(model, ims, data)
        g64, t64, r64 = step_chain(model, sd0, feats, upstream, torch.float64)
        g32, t32, r32 = step_chain(model, sd0, feats, upstream, torch.float32)
        scale = min(1.0, 5.0 / (total + 1e-6))
        ours = {k: g / scale for k, g in ours.items()}
        errs = {k: (rel(ours[k], g64[k]), rel(g32[k], g64[k])) for k in g64}
        cat = lambda g, n: torch.cat([g[k].double().flatten() for k in g64 if k.startswith(n + ".")])
        groups = {f"{n} (all parameters)": (rel(cat(ours, n), cat(g64, n)), rel(cat(g32, n), cat(g64, n))) for n in HEADS}
        everything = lambda g: torch.cat([g[k].double().flatten() for k in g64])
        groups["all parameters"] = (rel(everything(ours), everything(g64)), rel(everything(g32), everything(g64)))
        # the clipped total is one scalar, whose error a lucky cancellation can make arbitrarily small in either chain:
        # it is held to what the gradients allow, | ||ours|| - ||fp64|| | <= ||ours - fp64||
        assert abs(total - t64) <= float((everything(ours) - everything(g64)).norm()) + 1e-6 * t64
        running = {f"{n}.{k}": b for n in HEADS for k, b in getattr(ex, n).named_buffers() if "running" in k}
        assert set(running) == set(r64)
        stats = {k: (rel(running[k], r64[k]), rel(r32[k], r64[k])) for k in r64}
        record(f"step {step + 1} {case}", {**groups, **stats, **errs})
        bad = over(groups)
        assert not bad, f"{case} step {step + 1} (ours, eager fp32) relative errors: {bad}"
        bad = {k: e for k, e in errs.items() if e[0] > max(STEP_TENSOR_RATIO * e[1], EDGE_FLOOR["grad"]) + FLOOR}
        assert not bad, f"{case} step {step + 1} (ours, eager fp32) relative errors: {bad}"
        bad = over(stats)
        assert not bad, f"{case} step {step + 1} running statistics (ours, eager fp32) relative errors: {bad}"
        assert bn_counters(model) == {k: v + 2 for k, v in counters.items()}
        opt.step()
    TRAINED[case] = model


# ---- c. the validation step ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(STEP_CASES))
def test_validation_step_against_fp64(case):
    """validation_step under torch.inference_mode (Lightning 2's default for validation): scr, kps, depth, dsc and
    final_scores against the fp64 eval chain from the same backbone features; avg_loss bit for bit the grad-enabled call
    with the same draws, every loss output finite.  Back in train mode, the next step's gradients are those of a copy
    of the model that never validated, bit for bit."""
    config, B, H, W = STEP_CASES[case]
    torch.manual_seed(0)
    model = converted_model(config)
    twin = copy.deepcopy(model)
    sd0 = head_state(model)
    before = {k: v.clone() for k, v in model.state_dict().items() if "dinov2" not in k}
    ims, data = step_batch(B, H, W, seed=B + 1)
    with torch.inference_mode():
        feats, cs, batch, outputs, draws = validation_step(model, ims, data, seed=B + 2)
    assert not any(getattr(model.compute_matches.extractor, n).training for n in HEADS)
    ours = pair_outputs(cs, batch["final_scores"])
    ref = eval_chain(model, sd0, feats, torch.float64)
    eager = eval_chain(model, sd0, feats, torch.float32)
    errs = {k: (rel(ours[k], ref[k]), rel(eager[k], ref[k])) for k in ref}
    record(f"validation {case}", errs)
    bad = over(errs)
    assert not bad, f"{case} validation (ours, eager fp32) relative errors: {bad}"
    avg_loss = outputs["loss"]
    assert bool(torch.isfinite(avg_loss))
    finite = lambda v: bool(torch.isfinite(v.detach()).all())
    assert all(finite(v) for v in outputs.values() if torch.is_tensor(v)), \
        [k for k, v in outputs.items() if torch.is_tensor(v) and not finite(v)]
    again = model.loss_fn({k: v.clone() if torch.is_tensor(v) else v for k, v in batch.items()}, seed=B + 2,
                          outer_idx=draws[0], inner_idx=draws[1])[0]
    assert torch.equal(again, avg_loss)
    after = {k: v for k, v in model.state_dict().items() if "dinov2" not in k}
    assert all(torch.equal(after[k], v) for k, v in before.items())
    is_eval_model(model, False)
    ims, data = step_batch(B, H, W, seed=B + 3)
    results = []
    for m in (model, twin):
        torch.manual_seed(5)
        results.append(train_step(m, ims, data))
    (_, _, total, grads), (_, _, total_twin, grads_twin) = results
    assert total == total_twin
    assert all(torch.equal(grads[k], grads_twin[k]) for k in grads)
    assert all(torch.equal(a, b) for a, b in zip(model.state_dict().values(), twin.state_dict().values()))


# ---- d. a validation as the model's first call -------------------------------------------------------------------------
def test_first_call_under_inference_mode_then_a_training_step():
    """trainer.validate on a resumed checkpoint, or Lightning's sanity check, calls the model first under inference_mode:
    the packed backbone, its workspace and anything a module caches are then made there.  The training step after it
    runs and gives the gradients of a model whose first call was the training step, bit for bit."""
    config, B, H, W = STEP_CASES["vitl_224x210_b2_overlap_warm_up"]
    ims, data = step_batch(B, H, W, seed=11)
    results = {}
    for validate_first in (False, True):
        torch.manual_seed(0)
        model = converted_model(config)
        assert model.compute_matches.extractor.dinov2_vitl14._packed is None
        if validate_first:
            with torch.inference_mode():
                validation_step(model, ims, data, seed=12)
            is_eval_model(model, False)
        torch.manual_seed(13)
        results[validate_first] = train_step(model, ims, data)
        del model
    (_, _, total, grads), (_, _, total_v, grads_v) = results[False], results[True]
    assert total == total_v
    assert all(torch.equal(grads[k], grads_v[k]) for k in grads)


# ---- e. the handoff to the inference engine ----------------------------------------------------------------------------
HANDOFF_CASE = "vitl_720x540_b8_curriculum"


def test_checkpoint_handoff_to_the_inference_engine(monkeypatch):
    """The converted model after the lockstep test's three steps, saved as on_save_checkpoint leaves it, loaded the way
    build_model (mickey_b200/model.py:489-499) loads a checkpoint but with the training model's own backbone: the engine's
    compute_matches on a 720 x 540 pair against the fp64 oracle on that checkpoint, at test_gpu_parity.py's
    thresholds (the descriptors, like the scores, also at the reference's own fp16 deviation); the training model's own eval-mode outputs agree with the engine's within the sum of their fp64 errors."""
    from mickey_b200.model import MickeyRelativePose
    monkeypatch.setenv("MICKEY_SYNTHETIC_BACKBONE", "0")          # the backbone must be the training model's
    model = TRAINED.get(HANDOFF_CASE)
    if model is None:                                            # run alone: take the same three steps unchecked
        config, B, H, W = STEP_CASES[HANDOFF_CASE]
        torch.manual_seed(0)
        model = converted_model(config)
        opt = torch.optim.Adam(model.parameters(), lr=model.cfg.TRAINING.LR, eps=1e-6)
        for step in range(STEPS):
            opt.zero_grad()
            train_step(model, *step_batch(B, H, W, seed=100 * (step + 1) + B))
            opt.step()
    state = model.state_dict()
    ckpt = {"state_dict": dict(state)}
    on_save_checkpoint(ckpt)
    assert ckpt["state_dict"] and not any("dinov2" in k for k in ckpt["state_dict"])
    pre = mo.BACKBONE
    backbone = {k[len(pre):]: v for k, v in state.items() if k.startswith(pre)}
    inf = MickeyRelativePose(model.cfg, dinov2_weights=backbone)
    inf.on_load_checkpoint(ckpt)
    inf.load_state_dict(ckpt["state_dict"], strict=True)
    inf = inf.cuda().eval()
    loaded = inf.state_dict()
    assert set(loaded) == set(state)
    assert all(torch.equal(loaded[k].cpu(), state[k].cpu().to(loaded[k].dtype)) for k in state)

    data = {k: v.to(DEV) for k, v in synthetic_pair(1, 720, 540, seed=21).items()}
    inf.compute_matches(data)
    torch.cuda.synchronize()
    sd64 = {k: v.to(DEV, torch.float64) if v.is_floating_point() else v.to(DEV) for k, v in loaded.items()}
    with torch.no_grad():
        ref = mo.compute_correspondences(sd64, {k: v.double() if torch.is_tensor(v) else v for k, v in data.items()},
                                         model.cfg)
    names = {"kps": ("kps0", "kps1"), "depth": ("depth_kp0", "depth_kp1"), "scr": ("scr0", "scr1"),
             "dsc": ("dsc0", "dsc1")}
    pair = lambda d, k: torch.cat([d[names[k][0]], d[names[k][1]]]).double() if k in names else d[k].double()
    kps_px = lambda a, b: float((a - b).abs().max())
    dist = {k: (kps_px if k == "kps" else rel) for k in ("kps", "depth", "scr", "dsc", "scores", "kp_scores")}
    engine = {k: dist[k](pair(data, k), pair(ref, k)) for k in dist}
    yard = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "fp16_yardstick.json")))["vitl_720x540"]
    dump("handoff engine vs fp64", engine)

    # the training model's own eval-mode outputs on the same pair
    is_eval_model(model, True)
    with torch.inference_mode():
        _, cs, _ = forward_pair(model, [data["image0"], data["image1"]])
        scores = model.compute_matches.matcher.matching_mat(cs[0][3], cs[1][3])
        kp_scores = torch.matmul(cs[0][2].transpose(2, 1), cs[1][2])
    is_eval_model(model, False)
    train = {"kps0": cs[0][0], "kps1": cs[1][0], "depth_kp0": cs[0][1], "depth_kp1": cs[1][1], "scr0": cs[0][2],
             "scr1": cs[1][2], "dsc0": cs[0][3], "dsc1": cs[1][3], "scores": scores, "kp_scores": kp_scores}
    training = {k: dist[k](pair(train, k), pair(ref, k)) for k in dist}
    # the training model against the engine, relative to the fp64 norm as both fp64 errors are
    between = {k: (kps_px(pair(train, k), pair(data, k)) if k == "kps" else
                   float((pair(train, k) - pair(data, k)).norm() / pair(ref, k).norm())) for k in dist}
    dump("handoff training model vs fp64", training)
    dump("handoff training model vs engine", between)
    # test_gpu_parity.py's thresholds.  The descriptors, like the scores there, are also held to the deviation of the
    # reference's own fp16 configuration from its fp32 path at ViT-L 720 x 540 (1.2e-3): the fp16 backbone alone
    # brings the engine's descriptors near 1e-3 (the heads from the same backbone features add 5e-4 in both the CUDA
    # and the eager fp32 chain, test_validation_step_against_fp64)
    assert engine["dsc"] < max(1e-3, yard["dsc"]), engine
    assert engine["scores"] < max(1e-3, yard["scores"]), engine
    assert engine["scr"] < 1e-4 and engine["kp_scores"] < 1e-4, engine
    assert engine["kps"] < 3e-2, engine
    assert engine["depth"] < 5e-3, engine
    bad = {k: (between[k], training[k], engine[k]) for k in dist if between[k] > training[k] + engine[k] + 1e-12}
    assert not bad, f"training model vs engine, (between, training vs fp64, engine vs fp64): {bad}"
