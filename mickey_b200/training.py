"""Move a reference MicKeyTrainingModel onto mickey_b200's CUDA modules in one call.

    from mickey_b200.training import use_cuda_modules

    model = MicKeyTrainingModel(cfg)
    use_cuda_modules(model)            # before trainer.fit, so that configure_optimizers collects the new modules' Parameters
    use_cuda_modules(model, solver=True)   # the same, and the validation's pose solver too
    use_cuda_modules(model, cuda_tail=True)   # the same, and the loss's differentiable tail in CUDA
    trainer.fit(model, datamodule)

See use_cuda_modules for what moves and what is kept.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .config import VARIANTS
from .dinov2 import DinoVisionTransformer
from .dual_softmax import dualSoftmax
from .heads import DeepResBlock_depth, DeepResBlock_desc, DeepResBlock_det, DeepResBlock_offset
from .loss import MetricPoseLoss
from .procrustes import e2eProbabilisticProcrustesSolver

HEADS = {"depth_head": DeepResBlock_depth, "det_offset": DeepResBlock_offset, "dsc_head": DeepResBlock_desc,
         "det_head": DeepResBlock_det}


def _check_trees(new: nn.Module, old: nn.Module, what: str):
    """Raises ValueError when the parameter and buffer trees of `new` and `old` differ in a name, their order or a shape."""
    new_p, old_p = dict(new.named_parameters()), dict(old.named_parameters())
    new_b, old_b = dict(new.named_buffers()), dict(old.named_buffers())
    for kind, a, b in (("parameters", new_p, old_p), ("buffers", new_b, old_b)):
        if list(a) != list(b):
            raise ValueError(f"{what}: the CUDA module's {kind} differ from the model's: only in the model "
                             f"{sorted(set(b) - set(a))}, only in the CUDA module {sorted(set(a) - set(b))}"
                             if set(a) != set(b) else f"{what}: the {kind} are registered in a different order")
        for n in a:
            if a[n].shape != b[n].shape:
                raise ValueError(f"{what}: {n} has shape {tuple(b[n].shape)} in the model and {tuple(a[n].shape)} in the "
                                 f"CUDA module")


def _transplant(new: nn.Module, old: nn.Module):
    """Hand `old`'s very Parameter and buffer objects to `new` under the same names, and each submodule's training flag
    (a submodule only `new` has takes its parent's), so values, dtypes, devices, requires_grad and any .grad stay exactly
    as they were."""
    for n, p in old.named_parameters():
        mod, _, leaf = n.rpartition(".")
        new.get_submodule(mod)._parameters[leaf] = p
    for n, b in old.named_buffers():
        mod, _, leaf = n.rpartition(".")
        new.get_submodule(mod)._buffers[leaf] = b
    flags = {n: m.training for n, m in old.named_modules()}
    for n, m in new.named_modules():                   # parents come before their children
        m.training = flags.setdefault(n, flags[n.rpartition(".")[0]])


def use_cuda_modules(model, solver: bool = False, cuda_tail: bool = False):
    """Replace, in place, the modules of the reference's MicKeyTrainingModel that have CUDA drop-ins, and return model:

        compute_matches.extractor.dinov2_vitl14      -> mickey_b200.dinov2.DinoVisionTransformer (the variant of its width)
        compute_matches.extractor.{det_head, det_offset, depth_head, dsc_head}
                                                     -> mickey_b200.heads.DeepResBlock_{det, offset, depth, desc}
        compute_matches.matcher.matching_mat         -> mickey_b200.dual_softmax.dualSoftmax
        loss_fn                                      -> mickey_b200.loss.MetricPoseLoss
        e2e_Procrustes (with solver=True)            -> mickey_b200.procrustes.e2eProbabilisticProcrustesSolver

    Each new module takes over the old one's Parameter and buffer objects, so model.state_dict() keeps its keys, shapes,
    dtypes and values bit for bit (BN running statistics, num_batches_tracked and an fp16 backbone under DINOV2.FLOAT16
    included), as do every requires_grad, every module's training flag and every device.  The loss keeps its topK, the
    curriculum state on_train_epoch_end moves, when the reference's loss has one (only with top-K or curriculum training).
    DINOV2.FLOAT16: False is rejected: the CUDA backbone runs in fp16 only.  model.e2e_Procrustes, the pose solver of the
    validation step and of the logging in backward_step, is replaced only with solver=True (it holds no parameters or
    buffers, so the state dict is the same either way); by default it stays the reference's.  With cuda_tail=True the loss
    runs its differentiable tail in CUDA (MetricPoseLoss(cfg, cuda_tail=True)); a loss that is already the drop-in gets the
    flag set.  Without it the loss keeps the autograd tail (or whatever an earlier call chose).

    Call it before trainer.fit, so that configure_optimizers collects the new modules' Parameters.  Every replacement is
    built and checked before the model is touched: a configuration a drop-in rejects raises ValueError and leaves the
    model unchanged.  A module that is already a drop-in is left as it is, so a second call changes nothing."""
    ex = model.compute_matches.extractor
    matcher = model.compute_matches.matcher
    cfg = model.cfg
    swaps = []                                   # (parent, name, new module, old module)

    # The backbone and the heads are built on the meta device: every tensor they hold is replaced by the model's own.
    old = ex.dinov2_vitl14
    if not isinstance(old, DinoVisionTransformer):
        if not cfg['MICKEY']['DINOV2']['FLOAT16']:
            raise ValueError("dinov2_vitl14: the CUDA backbone runs in fp16 only (DINOV2.FLOAT16: True); this model's "
                             "configuration has DINOV2.FLOAT16: False")
        width = {D: v for v, (D, _, _) in VARIANTS.items()}
        if old.embed_dim not in width:
            raise ValueError(f"dinov2_vitl14: no CUDA backbone of width {old.embed_dim} (have {sorted(width)})")
        with torch.device("meta"):
            swaps.append((ex, "dinov2_vitl14", DinoVisionTransformer(width[old.embed_dim]), old))
    for name, cls in HEADS.items():
        old = getattr(ex, name)
        if not isinstance(old, cls):
            with torch.device("meta"):
                swaps.append((ex, name, cls(cfg['MICKEY']), old))
    old = matcher.matching_mat
    if not isinstance(old, dualSoftmax):
        if cfg['FEATURE_MATCHER']['TYPE'] != 'DualSoftmax':
            raise ValueError(f"matching_mat: only the DualSoftmax matcher has a CUDA module, the model has "
                             f"{cfg['FEATURE_MATCHER']['TYPE']!r}")
        new = dualSoftmax(cfg['FEATURE_MATCHER']['DUAL_SOFTMAX'])
        new.temperature = old.temperature
        swaps.append((matcher, "matching_mat", new, old))
    old = model.loss_fn
    if not isinstance(old, MetricPoseLoss):
        new = MetricPoseLoss(cfg, cuda_tail=cuda_tail)
        if hasattr(old, "topK"):                 # the reference sets it only with top-K or curriculum training
            new.topK = old.topK
        swaps.append((model, "loss_fn", new, old))
    procrustes = None
    if solver and not isinstance(getattr(model, "e2e_Procrustes", None), e2eProbabilisticProcrustesSolver):
        procrustes = e2eProbabilisticProcrustesSolver(cfg)

    for parent, name, new, old in swaps:
        _check_trees(new, old, name)
    for parent, name, new, old in swaps:
        _transplant(new, old)
        setattr(parent, name, new)
    if procrustes is not None:
        model.e2e_Procrustes = procrustes
    if cuda_tail:
        model.loss_fn.cuda_tail = True
    return model
