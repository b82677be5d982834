"""The heads' output layers and the whole-model swap without a GPU: the oracle's closed-form backward against fp64
autograd, an fp32 restatement of the kernels' arithmetic with an error model that rejects planted mutations, the argument
checks of mickey_b200.heads.head_out and of the C entry points, the drop-in heads' parameter trees and
mickey_b200.training.use_cuda_modules on a model built from the recorded reference tree (and on the live reference when
its tree is present)."""
import ctypes as C
import json

import numpy as np
import pytest
import torch
import torch.nn as nn

from mickey_b200 import _lib
from mickey_b200.head_transformer import sine_table
from mickey_b200.heads import KINDS, head_out
from mickey_b200.training import HEADS, use_cuda_modules
from oracle import heads_oracle as ho
from oracle import ref_harness
from tests.golden import make_training_tree as mtt

TREE = json.load(open(mtt.TREE))
EXTRACTOR = "compute_matches.extractor."


def layer_inputs(kind, B=2, C_=16, h=9, w=8, seed=0, dtype=torch.float64):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, C_, h, w, generator=g, dtype=dtype)
    k = 2 if kind == "offset" else 1
    W = None if kind == "desc" else torch.randn(k, C_, 1, 1, generator=g, dtype=dtype) * 2
    gk = C_ if kind == "desc" else k
    go = torch.randn(B, gk, h, w, generator=g, dtype=dtype)
    return x, W, go


@pytest.mark.parametrize("kind", list(KINDS))
def test_closed_form_backward_matches_fp64_autograd(kind):
    x, W, go = layer_inputs(kind)
    xr = x.clone().requires_grad_()
    Wr = None if W is None else W.clone().requires_grad_()
    out, norm = ho.output_forward(kind, xr, Wr, temperature=100.0 if kind == "score_softmax" else 1.0, max_depth=60.0)
    grads = torch.autograd.grad(out, [t for t in (xr, Wr) if t is not None], go)
    dx, dW = ho.output_backward(kind, x, W, out.detach(), None if norm is None else norm.detach(), go, temperature=100.0,
                                max_depth=60.0)
    assert (dx - grads[0]).abs().max() <= 1e-12 * max(1.0, grads[0].abs().max())
    if W is not None:
        assert (dW - grads[1]).abs().max() <= 1e-12 * max(1.0, grads[1].abs().max())


# ---- the kernels' arithmetic restated in fp32 numpy, with fp64 accumulation where the kernels use it --------------------
U32 = 2.0 ** -24


def restate(kind, x, W, go, eps=1e-16, T=100.0, md=60.0, mutation=None):
    """(out, dx, dW) as csrc/head_out.cu computes them; `mutation` plants one defect."""
    f = np.float32
    x, go = x.astype(f), go.astype(f)
    B, C_, h, w = x.shape
    mask = np.zeros((h, w), f)
    lo = 4 if mutation == "border" else 3
    mask[lo:h - 3, lo:w - 3] = 1
    if kind == "desc":
        n = np.sqrt((x.astype(np.float64) ** 2).sum(1, keepdims=True) + 1e-10).astype(f)
        y = (x / n).astype(f)
        yg = (y.astype(np.float64) * go).sum(1, keepdims=True).astype(f)
        if mutation == "projection":
            yg = np.zeros_like(yg)
        return y, ((go - y * yg) / n).astype(f), None
    Wm = W.reshape(W.shape[0], C_).astype(f)
    r = np.einsum("kc,bchw->bkhw", Wm, x).astype(f)               # fp32 dot products (FMA order aside)
    if kind == "score_softmax":
        shift = f(r.astype(np.float64).reshape(B, -1).mean(-1).astype(f)) + f(eps)
        e = (np.exp((r - shift.reshape(B, 1, 1, 1)) / f(T)) * mask).astype(f)
        p = (e / (e.astype(np.float64).sum((2, 3), keepdims=True).astype(f) + f(eps))).astype(f)
        gp = (go.astype(np.float64) * p).sum((2, 3), keepdims=True).astype(f)
        if mutation == "no_gp":
            gp = np.zeros_like(gp)
        dr = (p * (go - gp) / f(T)).astype(f)
        if mutation == "through_mean":              # the gradient also taken through the (undetached) mean
            dr = dr - dr.astype(np.float64).mean((2, 3), keepdims=True).astype(f)
        out = p
    else:
        s = (1 / (1 + np.exp(-r))).astype(f)
        if kind == "score_sigmoid":
            out = (s * mask).astype(f)
            # sigma' taken on the masked value p = sigma mask is the same thing: p (1 - p) is 0 wherever the mask is.  The
            # planted defect is the mask left out of the derivative instead.
            dr = go * out * (1 - out) * mask
            if mutation == "mask_dropped":
                dr = go * s * (1 - s)
        elif kind == "offset":
            out = s
            dr = go * s * (1 - s)
        elif kind == "depth":
            out, dr = r, go
        else:
            out = (f(md) * s).astype(f)
            # "scaled_derivative": sigma' taken on the scaled value MAX_DEPTH sigma instead of sigma
            dr = go * (out * (1 - (out if mutation == "scaled_derivative" else out / f(md))))
    dr = dr.astype(f)
    dx = np.einsum("bkhw,kc->bchw", dr, Wm).astype(f)
    P = B * h * w
    flat_dr = dr.transpose(1, 0, 2, 3).reshape(dr.shape[1], P).astype(np.float64)
    flat_x = x.transpose(1, 0, 2, 3).reshape(C_, P).astype(np.float64)
    if mutation == "last_slot":
        flat_dr = flat_dr[:, :P - P % 256 if P % 256 else P - 256]
        flat_x = flat_x[:, :flat_dr.shape[1]]
    dW = (flat_dr @ flat_x.T).astype(f).reshape(W.shape)
    return out, dx, dW


def within(ours, ref, scale):
    """The error model: every element within 64 u32 of the quantity's scale (fp32 roundings over at most a few dozen
    operations and the exp / sigmoid ulps), plus u32 of the element itself."""
    return np.all(np.abs(ours.astype(np.float64) - ref) <= 64 * U32 * scale + U32 * np.abs(ref))


def ref64(kind, x, W, go, eps=1e-16, T=100.0, md=60.0):
    xt, gt = torch.from_numpy(x).double(), torch.from_numpy(go).double()
    Wt = None if W is None else torch.from_numpy(W).double()
    out, norm = ho.output_forward(kind, xt, Wt, eps=eps, temperature=T, max_depth=md)
    dx, dW = ho.output_backward(kind, xt, Wt, out, norm, gt, temperature=T, max_depth=md)
    return [None if t is None else t.numpy() for t in (out, dx, dW)]


def scales(kind, x, W, go, ref):
    """The scale each result's rounding is charged against: |x| |W| summed like the value itself, and so on."""
    out, dx, dW = ref
    ax, ag = np.abs(x).astype(np.float64), np.abs(go).astype(np.float64)
    if kind == "desc":
        return np.abs(out).max(), np.abs(dx).max() + ag.max() / 1.0, None
    Wm = np.abs(W.reshape(W.shape[0], -1)).astype(np.float64)
    so = np.abs(out).max() + (np.einsum("kc,bchw->bkhw", Wm, ax).max() if kind == "depth" else 0)
    dr_scale = {"score_softmax": np.abs(out).max() * 2 * ag.max() / 100.0, "depth_sigmoid": 60.0 * ag.max()}.get(
        kind, ag.max())
    return so, dr_scale * Wm.sum(0).max() + np.abs(dx).max(), dr_scale * ax.sum((0, 2, 3)).max() + np.abs(dW).max()


# The softmax is invariant to a shift of r, so the gradient through the mean is sum_i dr_i / (h w) = sum g p (1 - sum p) /
# (T h w), with 1 - sum p = eps / (sum e + eps).  At the module's eps = 1e-16 that is far below any rounding, so a planted
# one passes the error model there.  With a loaded eps of order 1 it is not, and the error model rejects it: the detach
# is pinned by the loaded-eps case.
@pytest.mark.parametrize("eps", [1e-16, 0.5])
def test_gradient_through_the_mean(eps):
    x, W, go = (t.numpy().astype(np.float32) for t in layer_inputs("score_softmax", B=2, C_=64, h=17, w=19))
    ref = ref64("score_softmax", x, W, go, eps=eps)
    sc = scales("score_softmax", x, W, go, ref)
    assert all(within(o, r, s) for o, r, s in zip(restate("score_softmax", x, W, go, eps=eps), ref, sc))
    planted = restate("score_softmax", x, W, go, eps=eps, mutation="through_mean")
    assert all(within(o, r, s) for o, r, s in zip(planted, ref, sc)) == (eps < 1e-3)


MUTATIONS = {"no_gp": ["score_softmax"], "border": ["score_softmax", "score_sigmoid"],
             "mask_dropped": ["score_sigmoid"], "scaled_derivative": ["depth_sigmoid"], "projection": ["desc"],
             "last_slot": ["score_softmax", "score_sigmoid", "offset", "depth", "depth_sigmoid"]}


@pytest.mark.parametrize("kind", list(KINDS))
def test_fp32_restatement_within_the_error_model_and_mutations_rejected(kind):
    x, W, go = (t if t is None else t.numpy().astype(np.float32) for t in layer_inputs(kind, B=2, C_=64, h=17, w=19))
    ref = ref64(kind, x, W, go)
    sc = scales(kind, x, W, go, ref)
    for ours, r, s in zip(restate(kind, x, W, go), ref, sc):
        if r is not None:
            assert within(ours, r, s)
    for mutation, kinds in MUTATIONS.items():
        if kind not in kinds:
            continue
        mutated = restate(kind, x, W, go, mutation=mutation)
        assert not all(r is None or within(o, r, s) for o, r, s in zip(mutated, ref, sc)), mutation


# ---- argument checks ---------------------------------------------------------------------------------------------------
def test_head_out_rejects_bad_arguments_before_any_launch():
    x = torch.zeros(2, 64, 9, 9)
    W = torch.zeros(1, 64, 1, 1)
    eps = torch.tensor(1e-16)
    cases = [
        (dict(x=x, kind="softmax", weight=W), "kind must be"),
        (dict(x=x.numpy(), kind="depth", weight=W), "torch tensor"),
        (dict(x=x.double(), kind="depth", weight=W), "float32"),
        (dict(x=x[0], kind="depth", weight=W), "float32"),
        (dict(x=torch.zeros(0, 64, 9, 9), kind="depth", weight=W), "B, h, w >= 1"),
        (dict(x=torch.zeros(1, 4097, 1, 1), kind="desc"), "C <= 4096"),
        (dict(x=x, kind="desc", weight=W), "no weight"),
        (dict(x=x, kind="depth"), "needs a float32 weight"),
        (dict(x=x, kind="offset", weight=W), r"weight \[2, 64\]"),
        (dict(x=x, kind="depth", weight=W.double()), "needs a float32 weight"),
        (dict(x=x, kind="score_softmax", weight=W), "needs eps"),
        (dict(x=x, kind="score_softmax", weight=W, eps=torch.zeros(2)), "needs eps"),
        (dict(x=x, kind="score_softmax", weight=W, eps=nn.Parameter(eps.clone())), "must not require grad"),
        (dict(x=x, kind="score_softmax", weight=W, eps=eps, temperature=0.0), "temperature"),
        (dict(x=x, kind="score_softmax", weight=W, eps=eps, temperature=float("inf")), "temperature"),
        (dict(x=x, kind="depth_sigmoid", weight=W, max_depth=float("nan")), "max_depth"),
        (dict(x=x, kind="depth", weight=W), "CUDA device"),
    ]
    for kw, msg in cases:
        with pytest.raises(ValueError, match=msg):
            head_out(**kw)


def test_c_entry_points_reject_bad_arguments():
    lib = _lib.load()
    assert lib.mk_head_out_backward_ws_bytes(0, 8, 51, 38, 64) > 0
    assert lib.mk_head_out_backward_ws_bytes(5, 8, 51, 38, 128) == 0
    for args in ((6, 1, 4, 4, 64), (-1, 1, 4, 4, 64), (0, 0, 4, 4, 64), (0, 1, 0, 4, 64), (0, 1, 4, 4, 0),
                 (0, 1, 4, 4, 4097), (0, 1 << 13, 1 << 7, 1 << 7, 64)):
        assert lib.mk_head_out_backward_ws_bytes(*args) == -1, args
    fake = C.c_void_p(256)
    st = (C.c_longlong * 4)(64 * 16, 16, 4, 1)
    fwd = lambda kind, w, eps=fake, T=100.0, md=1.0, out=fake: lib.mk_head_out_forward(
        kind, fake, st, 1, 64, 4, 4, w, eps, T, md, out, None, None)
    for call in (lambda: fwd(7, fake), lambda: fwd(5, fake), lambda: fwd(3, None), lambda: fwd(0, fake, eps=None),
                 lambda: fwd(0, fake, T=0.0), lambda: fwd(4, fake, md=float("inf")), lambda: fwd(3, fake, out=None)):
        assert call() == -1
        assert lib.mk_last_error().decode().startswith("mk_head_out_forward")
    bwd = lambda kind, w, norm=None, gw=None, ws=fake, nbytes=1 << 30, md=1.0: lib.mk_head_out_backward(
        kind, fake, st, 1, 64, 4, 4, w, 100.0, md, fake, norm, fake, fake, gw, ws, nbytes, None)
    for call in (lambda: bwd(5, None), lambda: bwd(5, None, norm=fake, gw=fake), lambda: bwd(3, None),
                 lambda: bwd(3, fake, nbytes=16), lambda: bwd(3, fake, ws=C.c_void_p(260)), lambda: bwd(4, fake, md=0.0)):
        assert call() == -1
        assert lib.mk_last_error().decode().startswith("mk_head_out_backward")


# ---- the drop-in heads against the recorded reference tree -------------------------------------------------------------
def recorded(prefix):
    return [(n[len(prefix):], *rest) for n, *rest in TREE["state"] if n.startswith(prefix)]


@pytest.mark.parametrize("name", list(HEADS))
def test_head_parameter_trees_match_the_recorded_reference(name):
    head = HEADS[name](mtt.training_cfg()["MICKEY"])
    params = dict(head.named_parameters())
    ours = [(n, "param" if n in params else "buffer", list(t.shape), str(t.dtype).replace("torch.", ""),
             bool(t.requires_grad)) for n, t in head.state_dict(keep_vars=True).items()]
    assert ours == [tuple(e) for e in recorded(EXTRACTOR + name + ".")]


def model_from_tree(config="curriculum_learning", tree=TREE):
    """A stand-in for MicKeyTrainingModel with the recorded parameter and buffer tree (names, shapes, dtypes,
    requires_grad, training flags), seeded values, plain nn.Modules as its submodules, and the reference's config
    `config`.  The loss has a topK exactly when the reference's has one (loss_class.py:62-67)."""
    g = torch.Generator().manual_seed(0)
    root = nn.Module()

    def module(path):
        mod = root
        for part in path.split(".") if path else []:
            if not hasattr(mod, part):
                mod.add_module(part, nn.Module())
            mod = getattr(mod, part)
        return mod

    for n, kind, shape, dtype, rg in tree["state"] + tree["nonpersistent"]:
        path, _, leaf = n.rpartition(".")
        mod = module(path)
        dt = getattr(torch, dtype)
        v = (torch.randn(shape, generator=g) if dt.is_floating_point else torch.randint(0, 9, shape, generator=g)).to(dt)
        if n.endswith("posEnc.pe"):          # the transformers' sine table, not a state: the reference's own values
            v = sine_table()[None]
        if kind == "param":
            mod.register_parameter(leaf, nn.Parameter(v, requires_grad=rg))
        else:
            mod.register_buffer(leaf, v, persistent=[n, kind, shape, dtype, rg] in tree["state"])
    for n, flag in tree["training"].items():
        module(n).training = flag
    root.compute_matches.extractor.dinov2_vitl14.embed_dim = 1024
    root.compute_matches.matcher.matching_mat.temperature = 0.1
    if not hasattr(root, "loss_fn"):
        root.add_module("loss_fn", nn.Module())
    root.cfg = mtt.training_cfg(config)
    cl = root.cfg.LOSS_CLASS.CURRICULUM_LEARNING
    if cl.TRAIN_CURRICULUM or cl.TRAIN_WITH_TOPK:
        root.loss_fn.topK = cl.TOPK_INIT if cl.TRAIN_CURRICULUM else cl.TOPK
    return root


def snapshot(model):
    return {n: (t, t.dtype, t.device, t.requires_grad, t.detach().clone())
            for n, t in model.state_dict(keep_vars=True).items()}


def assert_kept(model, before, flags, topk):
    after = model.state_dict(keep_vars=True)
    assert list(after) == list(before)
    for n, (t, dt, dev, rg, val) in before.items():
        assert after[n] is t and t.dtype == dt and t.device == dev and t.requires_grad == rg and torch.equal(t, val), n
    assert {n: m.training for n, m in model.named_modules() if n in flags} == {
        n: f for n, f in flags.items() if n in dict(model.named_modules())}
    assert model.loss_fn.topK == topk


def check_swap(model):
    before = snapshot(model)
    flags = {n: m.training for n, m in model.named_modules()}
    topk = None                                                     # what the CUDA loss holds without top-K training
    if hasattr(model.loss_fn, "topK"):
        model.loss_fn.topK = topk = 45                              # curriculum state moved by an epoch end
    assert use_cuda_modules(model) is model
    assert not any(t.is_meta for t in model.state_dict().values())
    ex = model.compute_matches.extractor
    for name, cls in HEADS.items():
        assert type(getattr(ex, name)) is cls
    from mickey_b200.dinov2 import DinoVisionTransformer
    from mickey_b200.dual_softmax import dualSoftmax
    from mickey_b200.loss import MetricPoseLoss
    assert type(ex.dinov2_vitl14) is DinoVisionTransformer
    assert type(model.compute_matches.matcher.matching_mat) is dualSoftmax
    assert type(model.loss_fn) is MetricPoseLoss
    assert not any(b.is_meta for b in model.buffers())
    assert_kept(model, before, flags, topk)
    mods = {n: m for n, m in model.named_modules()}
    use_cuda_modules(model)                                         # a second call changes nothing
    assert {n: m for n, m in model.named_modules()} == mods
    assert_kept(model, before, flags, topk)
    # every trainable parameter of the extractor and matcher now belongs to a mickey_b200 module
    owners = [ex.dinov2_vitl14, model.compute_matches.matcher.matching_mat] + [getattr(ex, n) for n in HEADS]
    owned = {id(p) for m in owners for p in m.parameters()}
    assert all(id(p) in owned for p in model.compute_matches.parameters())


def check_rejected(model, reject):
    before = snapshot(model)
    mods = {n: m for n, m in model.named_modules()}
    reject(model.cfg)
    with pytest.raises(ValueError):
        use_cuda_modules(model)
    assert {n: m for n, m in model.named_modules()} == mods
    assert snapshot(model).keys() == before.keys()
    assert all(model.state_dict(keep_vars=True)[n] is t for n, (t, *_) in before.items())


def few_samples(cfg):
    cfg.LOSS_CLASS.SAMPLER.NUM_SAMPLES_MATCHES = 100               # not a multiple of 32: the CUDA loss rejects it


def fp32_backbone(cfg):
    cfg.MICKEY.DINOV2.FLOAT16 = False                               # the CUDA backbone runs in fp16 only


REJECTED = {"few_samples": few_samples, "fp32_backbone": fp32_backbone}


@pytest.mark.parametrize("config", mtt.CONFIGS)
def test_use_cuda_modules_on_the_recorded_tree(config):
    check_swap(model_from_tree(config))


@pytest.mark.parametrize("reject", list(REJECTED))
def test_use_cuda_modules_rejects_without_touching_the_recorded_tree(reject):
    check_rejected(model_from_tree(), REJECTED[reject])


def test_use_cuda_modules_rejects_a_head_tree_it_cannot_hold():
    model = model_from_tree()
    model.compute_matches.extractor.det_head.resblock1.conv1.register_parameter("bias", nn.Parameter(torch.zeros(512)))
    mods = {n: m for n, m in model.named_modules()}
    with pytest.raises(ValueError, match="det_head"):
        use_cuda_modules(model)
    assert {n: m for n, m in model.named_modules()} == mods


needs_reference = pytest.mark.skipif(not ref_harness.available(), reason="reference tree not present")


@needs_reference
def test_recorded_tree_is_the_live_reference():
    model = mtt.reference_training_model(mtt.training_cfg(), variant="vits")
    live = mtt.tree_of(model)
    keep = lambda entries: [e for e in entries if "dinov2" not in e[0]]
    assert keep(live["state"]) == keep(TREE["state"]) and live["topK"] == TREE["topK"]
    assert {n: f for n, f in live["training"].items() if "dinov2" not in n} == \
        {n: f for n, f in TREE["training"].items() if "dinov2" not in n}


@needs_reference
@pytest.mark.parametrize("config", mtt.CONFIGS)
def test_use_cuda_modules_on_the_live_reference_model(config):
    check_swap(mtt.reference_training_model(mtt.training_cfg(config), variant="vits"))


@needs_reference
@pytest.mark.parametrize("reject", list(REJECTED))
def test_use_cuda_modules_rejects_without_touching_the_live_reference_model(reject):
    check_rejected(mtt.reference_training_model(mtt.training_cfg(), variant="vits"), REJECTED[reject])


@needs_reference
@pytest.mark.parametrize("name", list(HEADS))
def test_heads_load_the_live_reference_state_both_ways(name):
    model = mtt.reference_training_model(mtt.training_cfg(), variant="vits")
    ref = getattr(model.compute_matches.extractor, name)
    ours = HEADS[name](mtt.training_cfg()["MICKEY"])
    ours.load_state_dict(ref.state_dict(), strict=True)
    ref.load_state_dict(ours.state_dict(), strict=True)
    for attr in ("tmp_softmax", "use_softmax", "use_depth_sigmoid", "max_depth", "norm_desc"):
        assert getattr(ours, attr, None) == getattr(ref, attr, None), attr


# ---- the reference's recorded heads, rebuilt without the reference and held to the fp64 chain ---------------------------
from tests.golden import make_heads_fixture as mhf  # noqa: E402

HEADS_FIXTURE = np.load(mhf.FIXTURE)


@pytest.mark.parametrize("case", list(mhf.CASES))
def test_reference_heads_fixture_against_the_fp64_chain(case):
    """Outputs and running statistics within 1e-5 of their scale; gradients within 5 % in norm over the recorded sample
    (fp32 rounding flips ReLU masks in four batch-normed blocks, so element-wise bounds do not fit them)."""
    head_name, _, _, seed = mhf.CASES[case]
    config = mhf.case_config(case)
    head = HEADS[head_name](config).train()
    x, gout = mhf.case_inputs(head, seed)
    assert mhf.checksum(head, x, gout) == pytest.approx(float(HEADS_FIXTURE[f"{case}/checksum"]), rel=1e-12)
    sd = {n: (t.detach().double().clone().requires_grad_() if t.requires_grad else
              t.detach().to(torch.float64 if t.is_floating_point() else t.dtype).clone())
          for n, t in head.state_dict(keep_vars=True).items()}
    out, running = ho.head_chain(sd, head_name, config, x.double())
    names = [n for n, p in head.named_parameters() if p.requires_grad]
    grads = torch.autograd.grad(out, [sd[n] for n in names], gout.double())
    ours = {"out": out.detach(), **dict(zip(names, grads)), **running}
    recorded_names = {k.split("/")[1] for k in HEADS_FIXTURE.files if k.startswith(case + "/") and k.endswith("/val")}
    assert recorded_names == set(ours)
    for name, v in ours.items():
        idx = torch.from_numpy(HEADS_FIXTURE[f"{case}/{name}/idx"]).long()
        ref = torch.from_numpy(HEADS_FIXTURE[f"{case}/{name}/val"]).double()
        mine = v.reshape(-1)[idx]
        if name == "out" or "running" in name:
            assert (mine - ref).abs().max() <= 1e-5 * v.abs().max(), name
            assert abs(float(v.sum()) - float(HEADS_FIXTURE[f"{case}/{name}/sum"])) <= 1e-5 * float(v.abs().sum()), name
        else:
            assert (mine - ref).norm() <= 0.05 * mine.norm() + 1e-12, name
