"""The four drop-in heads (mickey_b200.heads) in train mode at both training shapes, against the fp64 chain of
oracle/heads_oracle.py: rb1 -> rb2 -> rb3 -> transformer -> rb4 -> output layer, with the dims the reference configs use
(1024 -> 512 -> 256 -> 128 -> 64, or 128 for the descriptor head).

Every output, every parameter gradient and every updated running statistic is compared as ||ours - fp64|| / ||fp64||.
The training step's backward (test_training_step_backward_against_fp64, on a model converted by use_cuda_modules) is
gated at 1.5x per head, over all its parameters' gradients as one vector, and on clip_grad_norm_'s total norm; each
gradient tensor alone, the dustbin's included, at 3x.
The gate: at most 1.5x as far from fp64 as the same chain run in eager fp32 torch on the GPU under torch's default TF32
flags (F.conv2d, the oracle's batch norm, transformer and output layers), with an absolute floor of 1e-6 where both are
tiny.  Element-wise bounds do not fit a chain of four batch-normed blocks: fp32 rounding flips ReLU masks.  With
MICKEY_TEST_RESULTS set to a directory, the measured errors and ratios are written to heads_training_ratios.json there.
"""
import json
import os

import pytest
import torch

from mickey_b200.heads import DeepResBlock_depth, DeepResBlock_desc, DeepResBlock_det, DeepResBlock_offset
from oracle import heads_oracle as ho
from tests.golden.make_training_tree import training_cfg

pytestmark = pytest.mark.gpu
DEV = "cuda"
HEADS = {"det_head": DeepResBlock_det, "det_offset": DeepResBlock_offset, "depth_head": DeepResBlock_depth,
         "dsc_head": DeepResBlock_desc}
SHAPES = [(8, 51, 38), (24, 34, 25)]
RATIO, FLOOR = 1.5, 1e-6
RESULTS = {}


def seeded_head(cls, config, seed):
    torch.manual_seed(seed)
    head = cls(config).to(DEV).train()
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, b in head.named_buffers():
            if n.endswith("running_mean"):
                b.copy_(0.1 * torch.randn(b.shape, generator=g))
            elif n.endswith("running_var"):
                b.copy_(1 + 0.5 * torch.rand(b.shape, generator=g))
        for n, p in head.named_parameters():
            if "bn" in n and n.endswith("weight"):
                p.copy_(1 + 0.2 * torch.randn(p.shape, generator=g))
            elif "bn" in n and n.endswith("bias"):
                p.copy_(0.1 * torch.randn(p.shape, generator=g))
    return head


def chain(sd0, name, config, x, go, dtype):
    sd = {n: (t.detach().to(dtype).clone().requires_grad_() if t.is_floating_point() and rg else
              t.detach().to(dtype if t.is_floating_point() else t.dtype).clone()) for n, (t, rg) in sd0.items()}
    out, running = ho.head_chain(sd, name, config, x.to(dtype))
    names = [n for n, (t, rg) in sd0.items() if rg]
    grads = torch.autograd.grad(out, [sd[n] for n in names], go.to(dtype))
    return out.detach(), dict(zip(names, grads)), running


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-300))


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("name", list(HEADS))
def test_head_train_mode_against_fp64(name, shape):
    assert torch.backends.cudnn.allow_tf32            # the comparator runs under torch's default flags
    B, h, w = shape
    config = training_cfg()["MICKEY"]
    head = seeded_head(HEADS[name], config, seed=10 + len(name))
    sd0 = {n: (t, t.requires_grad) for n, t in head.state_dict(keep_vars=True).items()}
    sd0 = {n: (t.detach().clone(), rg) for n, (t, rg) in sd0.items()}
    g = torch.Generator(device=DEV).manual_seed(B * h)
    x = torch.randn(B, 1024, h, w, generator=g, device=DEV)
    out = head(x)
    go = torch.randn(out.shape, generator=g, device=DEV)
    out.backward(go)
    ours = {"out": out.detach(), **{n: p.grad for n, p in head.named_parameters() if p.requires_grad},
            **{n: b for n, b in head.named_buffers() if "running" in n}}
    o64, g64, r64 = chain(sd0, name, config, x, go, torch.float64)
    o32, g32, r32 = chain(sd0, name, config, x, go, torch.float32)
    ref = {"out": o64, **g64, **r64}
    eager = {"out": o32, **g32, **r32}
    assert set(ours) == set(ref)
    errs = {k: (rel(ours[k], ref[k]), rel(eager[k], ref[k])) for k in ref}
    RESULTS[f"{name} {B}x{h}x{w}"] = {k: {"ours": a, "eager_fp32_tf32": b, "ratio": a / b if b else None}
                                      for k, (a, b) in errs.items()}
    out_dir = os.environ.get("MICKEY_TEST_RESULTS")
    if out_dir:
        with open(os.path.join(out_dir, "heads_training_ratios.json"), "w") as f:
            json.dump(RESULTS, f, indent=1)
    bad = {k: e for k, e in errs.items() if e[0] > RATIO * e[1] + FLOOR}
    assert not bad, f"{name} {shape} (ours, eager fp32) relative errors: {bad}"


# ---- the training step's backward on a model converted by use_cuda_modules ----------------------------------------------
def converted_model(config, seed=0):
    """The recorded reference MicKeyTrainingModel tree (ViT-L, fp16 backbone) moved onto the CUDA modules by
    use_cuda_modules, then loaded with seeded synthetic weights."""
    from mickey_b200.config import mickey_cfg
    from mickey_b200.training import use_cuda_modules
    from mickey_b200.weights import synthetic_state_dict
    from tests.test_heads_host import model_from_tree
    model = use_cuda_modules(model_from_tree(config))
    model.load_state_dict(synthetic_state_dict(mickey_cfg("vitl"), seed), strict=True)
    return model.to(DEV)


def extract(ex, im):
    """MicKey_Extractor.forward (mickey_extractor.py:43-58): the crop, the backbone under no_grad, then the four heads."""
    B, _, H, W = im.shape
    f = 14
    im = im[:, :, :f * (H // f), :f * (W // f)]
    with torch.no_grad():
        feats = ex.dinov2_vitl14.forward_features(im.to(torch.float16))["x_norm_patchtokens"].permute(0, 2, 1).reshape(
            B, 1024, H // f, W // f).float()
    return feats, (ex.det_offset(feats), ex.depth_head(feats), ex.det_head(feats), ex.dsc_head(feats))


def correspondences(kpts, depth, scr, dsc):
    """get_abs_kpts_coordinates and prepare_kpts_dsc (compute_correspondences.py:20-43)."""
    B, _, H, W = kpts.shape
    x = torch.arange(W, device=kpts.device).view(1, 1, W).tile([B, H, 1])
    y = torch.arange(H, device=kpts.device).view(1, H, 1).tile([B, 1, W])
    kpts = (kpts + torch.concat([x.unsqueeze(1), y.unsqueeze(1)], dim=1)) * 14
    N = H * W
    return kpts.view(B, 2, N), depth.view(B, 1, N), scr.view(B, 1, N), dsc.view(B, dsc.shape[1], N)


def match(scores_fn, c0, c1):
    """The matcher, kp_matrix_scores and prepare_batch_for_loss (compute_correspondences.py:79-90, model.py:198-203)."""
    scores = scores_fn(c0[3], c1[3])
    kp_scores = torch.matmul(c0[2].transpose(2, 1).contiguous(), c1[2])
    return scores * kp_scores


def step_batch(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    from tests.common import K_TOY
    K = torch.tensor(K_TOY).expand(B, 3, 3).contiguous()
    T = torch.eye(4).expand(B, 4, 4).clone()
    T[:, :3, 3] = torch.tensor([0.3, -0.1, 0.2])
    ims = [torch.rand(B, 3, H, W, generator=g) for _ in range(2)]
    data = {"K_color0": K, "K_color1": K, "Kori_color0": K, "Kori_color1": K, "T_0to1": T}
    return [im.to(DEV) for im in ims], {k: v.to(DEV) for k, v in data.items()}


def fp64_step(model, sd0, feats, upstream, dtype):
    """The same step from the same backbone features, every head, the matcher and the outer product restated by the
    oracles in `dtype`, driven by the same upstream gradients.  Returns {name: gradient} and the total norm."""
    from oracle.mickey_oracle import dual_softmax as ds_oracle
    config = model.cfg["MICKEY"]
    leaves, sds = {}, {}
    for name in HEADS:
        sd = {}
        for n, (t, rg) in sd0[name].items():
            v = t.detach().to(dtype if t.is_floating_point() else t.dtype).clone()
            sd[n] = v.requires_grad_() if rg else v
            if rg:
                leaves[f"{name}.{n}"] = sd[n]
        sds[name] = sd
    mat = model.compute_matches.matcher.matching_mat
    dustbin = mat.dustbin_score.detach().to(dtype).clone().requires_grad_()
    leaves["matching_mat.dustbin_score"] = dustbin
    cs = []
    for f in feats:
        f = f.to(dtype)
        outs = [ho.head_chain(sds[n], n, config, f)[0] for n in ("det_offset", "depth_head", "det_head", "dsc_head")]
        cs.append(correspondences(*outs))
    final = match(lambda d0, d1: ds_oracle(d0, d1, mat.temperature, dustbin), cs[0], cs[1])
    torch.autograd.backward((torch.log(final + 1e-16), cs[0][0], cs[1][0], cs[0][1], cs[1][1]),
                            tuple(u.to(dtype) for u in upstream))
    grads = {n: t.grad for n, t in leaves.items()}
    return grads, float(torch.stack([g.double().norm() for g in grads.values()]).norm())


STEP_TENSOR_RATIO = 3.0
STEP_CASES = {"vitl_720x540_b8_curriculum": ("curriculum_learning", 8, 720, 540),
              "vitl_224x210_b2_overlap_warm_up": ("overlap_score_warm_up", 2, 224, 210)}


@pytest.mark.parametrize("case", list(STEP_CASES))
def test_training_step_backward_against_fp64(case):
    config, B, H, W = STEP_CASES[case]
    torch.manual_seed(0)
    model = converted_model(config)
    ex = model.compute_matches.extractor
    model.compute_matches.matcher.matching_mat.dustbin_score.grad = None
    sd0 = {n: {k: (t.detach().clone(), t.requires_grad) for k, t in getattr(ex, n).state_dict(keep_vars=True).items()}
           for n in HEADS}
    ims, data = step_batch(B, H, W, seed=B)
    feats, cs = [], []
    for im in ims:                                  # two extractor calls: separate batch statistics per image set
        f, outs = extract(ex, im)
        feats.append(f)
        cs.append(correspondences(*outs))
    final = match(model.compute_matches.matcher.matching_mat, cs[0], cs[1])
    batch = dict(data, final_scores=final, kps0=cs[0][0], kps1=cs[1][0], depth_kp0=cs[0][1], depth_kp1=cs[1][1])
    avg_loss, outputs, probs_grad, num_its = model.loss_fn(batch)
    assert num_its == 1
    avg_loss.backward()
    upstream = (probs_grad[0], outputs["kps0"].grad, outputs["kps1"].grad, outputs["depth0"].grad, outputs["depth1"].grad)
    assert all(u is not None and bool(torch.isfinite(u).all()) for u in upstream)
    # backward_step (model.py:124-137)
    torch.autograd.backward((torch.log(batch["final_scores"] + 1e-16), batch["kps0"], batch["kps1"], batch["depth_kp0"],
                             batch["depth_kp1"]), upstream)
    ours = {f"{n}.{k}": p.grad for n in HEADS for k, p in getattr(ex, n).named_parameters() if p.requires_grad}
    ours["matching_mat.dustbin_score"] = model.compute_matches.matcher.matching_mat.dustbin_score.grad
    assert all(g is not None for g in ours.values())
    total = float(torch.nn.utils.clip_grad_norm_(model.parameters(), max_norm=5))
    g64, t64 = fp64_step(model, sd0, feats, upstream, torch.float64)
    g32, t32 = fp64_step(model, sd0, feats, upstream, torch.float32)
    # clip_grad_norm_ scaled the gradients in place when the norm exceeded 5: compare the unclipped ones
    scale = min(1.0, 5.0 / (total + 1e-6))
    ours = {k: g / scale for k, g in ours.items()}
    errs = {k: (rel(ours[k], g64[k]), rel(g32[k], g64[k])) for k in g64}
    # what clip_grad_norm_ and the optimiser see of a head: all its parameters' gradients as one vector
    cat = lambda g, n: torch.cat([g[k].double().flatten() for k in g64 if k.startswith(n + ".")])
    groups = {f"{n} (all parameters)": (rel(cat(ours, n), cat(g64, n)), rel(cat(g32, n), cat(g64, n))) for n in HEADS}
    groups["clip_grad_norm_ total"] = (abs(total - t64) / t64, abs(t32 - t64) / t64)
    RESULTS[f"step {case}"] = {k: {"ours": a, "eager_fp32_tf32": b, "ratio": a / b if b else None}
                               for k, (a, b) in {**groups, **errs}.items()}
    out_dir = os.environ.get("MICKEY_TEST_RESULTS")
    if out_dir:
        with open(os.path.join(out_dir, "heads_training_ratios.json"), "w") as f:
            json.dump(RESULTS, f, indent=1)
    bad = {k: e for k, e in groups.items() if e[0] > RATIO * e[1] + FLOOR}
    assert not bad, f"{case} (ours, eager fp32) relative errors: {bad}"
    # each tensor alone is one draw of TF32 rounding noise through two image sets, four blocks and the matcher: held to
    # STEP_TENSOR_RATIO x the eager chain's error (DESIGN.md §6i has the spread)
    bad = {k: e for k, e in errs.items() if e[0] > STEP_TENSOR_RATIO * e[1] + FLOOR}
    assert not bad, f"{case} (ours, eager fp32) relative errors: {bad}"
