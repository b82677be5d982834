"""A converted training model's lifecycle without a GPU: the eval-mode head chain of oracle/heads_oracle.py against the
inference oracle's eval head, the checkpoint a converted model saves loading strictly into the inference model, resuming
from it, is_eval_model's flags, and the loss's cached grid after a first call under inference mode.  The live reference's
own on_save_checkpoint, on_load_checkpoint and is_eval_model run when its tree is present."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from mickey_b200.loss import MetricPoseLoss
from mickey_b200.model import build_model
from mickey_b200.training import HEADS, use_cuda_modules
from oracle import heads_oracle as ho
from oracle import mickey_oracle as mo
from tests.golden import make_training_tree as mtt
from tests.test_gpu_training_lifecycle import is_eval_model, on_save_checkpoint
from tests.test_heads_host import model_from_tree, needs_reference


# ---- the training oracle's eval chain is the inference oracle's eval head ---------------------------------------------
def seeded_cpu_head(name, config, seed):
    torch.manual_seed(seed)
    head = HEADS[name](config)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, b in head.named_buffers():
            if n.endswith("running_mean"):
                b.copy_(0.1 * torch.randn(b.shape, generator=g))
            elif n.endswith("running_var"):
                b.copy_(1 + 0.5 * torch.rand(b.shape, generator=g))
        for n, p in head.named_parameters():
            if "bn" in n:
                p.copy_((1 if n.endswith("weight") else 0) + 0.2 * torch.randn(p.shape, generator=g))
    return {n: t.detach().double() if t.is_floating_point() else t.detach() for n, t in head.state_dict().items()}


def inference_eval_head(sd, name, config, x):
    """oracle/mickey_oracle.py's head: head_trunk and the output activation, as its extractor() applies them."""
    kp, ds = config["KP_HEADS"], config["DSC_HEAD"]
    if name == "dsc_head":
        d = mo.head_trunk(sd, "", x, ds["POS_ENCODING"], False, kp["BN"])
        return mo.l2_normalize_channels(d) if ds["NORM_DSC"] else d
    t = mo.head_trunk(sd, "", x, kp["POS_ENCODING"], True, kp["BN"])
    if name == "det_head":
        return mo.score_activation(F.conv2d(t, sd["score.weight"]), kp["USE_SOFTMAX"])
    if name == "det_offset":
        return torch.sigmoid(F.conv2d(t, sd["xy_offset.weight"]))
    depth = F.conv2d(t, sd["depth.weight"])
    return kp["MAX_DEPTH"] * torch.sigmoid(depth) if kp["USE_DEPTHSIGMOID"] else depth


@pytest.mark.parametrize("shape", [(2, 9, 8), (1, 7, 7)], ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("name", list(HEADS))
def test_eval_head_chain_is_the_inference_oracle(name, shape):
    config = mtt.training_cfg()["MICKEY"]
    sd = seeded_cpu_head(name, config, seed=len(name))
    x = torch.randn(shape[0], 1024, *shape[1:], generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    before = {n: t.clone() for n, t in sd.items()}
    out, running = ho.head_chain(sd, name, config, x, train=False)
    ref = inference_eval_head(sd, name, config, x)
    assert running == {}
    assert all(torch.equal(sd[n], t) for n, t in before.items())
    assert out.shape == ref.shape
    assert float((out - ref).norm()) <= 1e-12 * float(ref.norm()) + 1e-300
    # the train-mode chain is a different function, so the identity above is not one any chain would meet (except the
    # score head's softmax over a single interior cell, which is 1 whatever the chain)
    if not (name == "det_head" and min(shape[1:]) <= 2 * ho.BORDER + 1):
        train_out = ho.head_chain(dict(sd), name, config, x)[0]
        assert float((train_out - ref).norm()) > 1e-3 * float(ref.norm())


# ---- the checkpoint of a converted model -------------------------------------------------------------------------------
def checkpoint_of(model):
    ckpt = {"state_dict": model.state_dict()}
    on_save_checkpoint(ckpt)
    return ckpt


def assert_loads_into_the_inference_model(state, model, monkeypatch):
    """build_model (mickey_b200/model.py:489-499) on the checkpoint `state`: a strict load, the same keys as the training
    model apart from the backbone's, and every tensor bit-equal to the training model's own after it."""
    monkeypatch.setenv("MICKEY_SYNTHETIC_BACKBONE", "1")            # no DINOv2 weights here; the backbone is not compared
    inf = build_model(mtt.training_cfg(), {"state_dict": dict(state)})
    loaded = inf.state_dict()
    own = {k: v for k, v in model.state_dict().items() if "dinov2" not in k}
    assert {k for k in loaded if "dinov2" not in k} == set(own)
    assert any("dinov2" in k for k in loaded)
    for k, v in own.items():
        assert loaded[k].dtype == v.dtype and torch.equal(loaded[k].cpu(), v.cpu()), k


@pytest.mark.parametrize("config", mtt.CONFIGS)
def test_converted_checkpoint_loads_into_the_inference_model(config, monkeypatch):
    model = use_cuda_modules(model_from_tree(config))
    state = checkpoint_of(model)["state_dict"]
    full = model.state_dict()
    assert set(state) == {k for k in full if "dinov2" not in k} and len(state) < len(full)
    assert_loads_into_the_inference_model(state, model, monkeypatch)


# ---- the live reference: its own checkpoint hooks and is_eval_model --------------------------------------------------
def live_converted(config, seed=None):
    model = use_cuda_modules(mtt.reference_training_model(mtt.training_cfg(config), variant="vits"))
    if seed is not None:                                              # values of a trained model: not the fresh init
        g = torch.Generator().manual_seed(seed)
        with torch.no_grad():
            for k, t in model.state_dict().items():
                if "dinov2" not in k:
                    t.copy_(torch.randn(t.shape, generator=g).to(t.dtype) if t.is_floating_point() else
                            torch.randint(0, 99, t.shape, generator=g).to(t.dtype))
    return model


@needs_reference
@pytest.mark.parametrize("config", mtt.CONFIGS)
def test_live_checkpoint_loads_into_the_inference_model_and_resumes(config, monkeypatch):
    model = live_converted(config, seed=3)
    ckpt = {"state_dict": model.state_dict()}
    model.on_save_checkpoint(ckpt)
    state = ckpt["state_dict"]
    assert state.keys() == checkpoint_of(model)["state_dict"].keys()
    assert_loads_into_the_inference_model(state, model, monkeypatch)
    # resuming: the reference's on_load_checkpoint fills the backbone from the model's own, then a strict load
    fresh = live_converted(config)
    backbone = fresh.compute_matches.extractor.dinov2_vitl14
    own = {k: v.clone() for k, v in fresh.state_dict().items() if "dinov2" in k}
    backbone._packed = object()                                     # stands for weights packed by an earlier forward
    resume = {"state_dict": dict(state)}
    fresh.on_load_checkpoint(resume)
    fresh.load_state_dict(resume["state_dict"], strict=True)
    assert backbone._packed is None
    after = fresh.state_dict()
    assert after.keys() == model.state_dict().keys()
    for k, v in after.items():
        want = own[k] if "dinov2" in k else state[k]
        assert v.dtype == want.dtype and torch.equal(v, want), k


def head_modules(model):
    return {f"compute_matches.extractor.{n}" for n in HEADS}


def in_heads(name, model):
    return any(name == h or name.startswith(h + ".") for h in head_modules(model))


def check_is_eval_model(model, switch):
    flags = {n: m.training for n, m in model.named_modules()}
    assert all(flags[n] for n in flags if in_heads(n, model))
    switch(model, True)
    after = {n: m.training for n, m in model.named_modules()}
    assert {n for n in flags if after[n] != flags[n]} == {n for n in flags if in_heads(n, model)}
    bns = [n for n, m in model.named_modules() if isinstance(m, nn.BatchNorm2d)]
    assert len(bns) == 32 and all(in_heads(n, model) and not after[n] for n in bns)
    switch(model, False)
    assert {n: m.training for n, m in model.named_modules()} == flags
    return after


def test_is_eval_model_restatement_switches_exactly_the_heads():
    check_is_eval_model(use_cuda_modules(model_from_tree()), is_eval_model)


@needs_reference
def test_live_is_eval_model_switches_exactly_the_heads_as_restated():
    model = live_converted("curriculum_learning")
    live = check_is_eval_model(model, lambda m, e: m.is_eval_model(e))
    restated = check_is_eval_model(model, is_eval_model)
    assert live == restated


# ---- the loss's cached grid after a first call under inference mode ------------------------------------------------------
def test_loss_grid_made_under_inference_mode_is_a_normal_tensor():
    """A validation before the first training step (Lightning's sanity check) makes the loss's VCRE grid under
    inference_mode; the training step's autograd then saves it for backward, which an inference tensor cannot be."""
    loss = MetricPoseLoss(mtt.training_cfg())
    with torch.inference_mode():
        grid = loss._vcre_grid(torch.device("cpu"))
    assert not grid.is_inference()
    assert loss._vcre_grid(torch.device("cpu")) is grid
    R = torch.eye(3, requires_grad=True)
    (R @ grid.T).sum().backward()
    torch.testing.assert_close(R.grad, grid.sum(0).expand(3, 3), rtol=1e-6, atol=1e-5)
