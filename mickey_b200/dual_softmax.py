"""MicKey's dual-softmax matcher as a differentiable op: the forward and the backward in CUDA (csrc/matcher_grad.cu).

`dual_softmax(dsc0, dsc1, dustbin, temperature)` computes the reference's dualSoftmax.forward
(lib/models/MicKey/modules/utils/feature_matcher.py:64-83); given the keypoint scores it also returns kp_matrix_scores
(compute_correspondences.py:46-50) and their product, final_scores (model.py:201).  It is differentiable in the
descriptors, the dustbin logit and the keypoint scores.  Only the inputs and two [B, N] log-sum-exp vectors are saved for
the backward; no N x N tensor is kept.

`dualSoftmax(cfg)` is a drop-in for the reference's module, with the same parameter name, so a trained state dict's
`compute_matches.matcher.matching_mat.dustbin_score` loads unchanged.  INTEGRATION.md shows the swap in a training model.
"""
from __future__ import annotations

import math
from typing import Optional

import torch
import torch.nn as nn

from . import _lib

MAX_N = 8192
DESC_DIM = 128
UNIT_NORM_SQ = 1.0005      # squared norms up to this count as unit (|S| <= 1.001, mk_match's bound under NORM_DSC)


def _check_dsc(name, t):
    if not torch.is_tensor(t):
        raise ValueError(f"{name} must be a torch tensor, got {type(t).__name__}")
    if t.dim() != 3 or t.shape[1] != DESC_DIM:
        raise ValueError(f"{name} must be [B, {DESC_DIM}, N], got {tuple(t.shape)}")
    if t.dtype != torch.float32:
        raise ValueError(f"{name} must be float32, got {t.dtype}")
    if t.device.type != "cuda":
        raise ValueError(f"{name} must be on a CUDA device (mickey_b200 has no CPU path), got {t.device}")


def _check_scr(name, t, B, N, dev):
    if not torch.is_tensor(t):
        raise ValueError(f"{name} must be a torch tensor, got {type(t).__name__}")
    if tuple(t.shape) not in ((B, N), (B, 1, N)):
        raise ValueError(f"{name} must be [B, N] or [B, 1, N] = [{B}, {N}], got {tuple(t.shape)}")
    if t.dtype != torch.float32 or t.device != dev:
        raise ValueError(f"{name} must be float32 on {dev}, got {t.dtype} on {t.device}")


class _DualSoftmax(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dsc0, dsc1, dustbin, scr0, scr1, temperature, unit_norm):
        B, _, N = dsc0.shape
        dev = dsc0.device
        lib = _lib.load()
        d0, d1 = dsc0.contiguous(), dsc1.contiguous()
        s0 = None if scr0 is None else scr0.reshape(B, N).contiguous()
        s1 = None if scr1 is None else scr1.reshape(B, N).contiguous()
        db = None if dustbin is None else dustbin.reshape(1).contiguous()
        npad = -(-N // 128) * 128
        with torch.cuda.device(dev):
            scores = torch.empty(B, N, N, dtype=torch.float32, device=dev)
            kp = final = None
            if s0 is not None:
                kp = torch.empty_like(scores)
                final = torch.empty_like(scores)
            lse_r = torch.empty(B, npad, dtype=torch.float32, device=dev)
            lse_c = torch.empty(B, npad, dtype=torch.float32, device=dev)
            ws = _lib.workspace(lib.mk_dual_softmax_ws_bytes(B, N), dev, "mk_dual_softmax_ws_bytes")
            _lib.check(lib.mk_dual_softmax(_lib.ptr(d0), _lib.ptr(d1), _lib.ptr(s0), _lib.ptr(s1), _lib.ptr(db),
                                           float(temperature), B, N, int(unit_norm), _lib.ptr(scores), _lib.ptr(kp),
                                           _lib.ptr(final), N, _lib.ptr(lse_r), _lib.ptr(lse_c), _lib.ptr(ws), ws.numel(),
                                           _lib.stream(dev)), "mk_dual_softmax")
        ctx.save_for_backward(d0, d1, s0, s1, db, lse_r, lse_c)
        ctx.temperature = float(temperature)
        ctx.scr_shapes = (None if scr0 is None else scr0.shape, None if scr1 is None else scr1.shape)
        ctx.dustbin_shape = None if dustbin is None else dustbin.shape
        ctx.set_materialize_grads(False)
        if s0 is None:
            return scores
        return scores, kp, final

    @staticmethod
    def backward(ctx, *grads):
        d0, d1, s0, s1, db, lse_r, lse_c = ctx.saved_tensors
        gs, gk, gf = (tuple(grads) + (None, None))[:3]
        if gs is None and gk is None and gf is None:
            return (None,) * 7
        B, _, N = d0.shape
        dev = d0.device
        lib = _lib.load()
        views = [None if g is None else _lib.pitched(g.float()) for g in (gs, gk, gf)]
        (gs, ps), (gk, pk), (gf, pf) = [(None, 0) if v is None else v for v in views]
        with torch.cuda.device(dev):
            dd0 = torch.empty_like(d0)
            dd1 = torch.empty_like(d1)
            ds0 = None if s0 is None else torch.empty_like(s0)
            ds1 = None if s1 is None else torch.empty_like(s1)
            ddb = None if db is None else torch.empty(1, dtype=torch.float32, device=dev)
            ws = _lib.workspace(lib.mk_dual_softmax_backward_ws_bytes(B, N), dev, "mk_dual_softmax_backward_ws_bytes")
            _lib.check(lib.mk_dual_softmax_backward(
                _lib.ptr(d0), _lib.ptr(d1), _lib.ptr(s0), _lib.ptr(s1), _lib.ptr(db), ctx.temperature, B, N,
                _lib.ptr(lse_r), _lib.ptr(lse_c), _lib.ptr(gs), ps, _lib.ptr(gk), pk, _lib.ptr(gf), pf,
                _lib.ptr(dd0), _lib.ptr(dd1), _lib.ptr(ds0), _lib.ptr(ds1), _lib.ptr(ddb), _lib.ptr(ws), ws.numel(),
                _lib.stream(dev)), "mk_dual_softmax_backward")
        sh0, sh1 = ctx.scr_shapes
        return (dd0, dd1,
                None if ddb is None else ddb.reshape(ctx.dustbin_shape),
                None if ds0 is None else ds0.reshape(sh0),
                None if ds1 is None else ds1.reshape(sh1),
                None, None)


def _is_unit_norm(dsc0, dsc1) -> bool:
    """Every descriptor has norm <= 1 (up to rounding): the normalised descriptors of DSC_HEAD.NORM_DSC."""
    with torch.no_grad():
        m = torch.maximum(dsc0.square().sum(1).amax(), dsc1.square().sum(1).amax())
    return bool(m <= UNIT_NORM_SQ)


def dual_softmax(dsc0: torch.Tensor, dsc1: torch.Tensor, dustbin: Optional[torch.Tensor], temperature: float,
                 scr0: Optional[torch.Tensor] = None, scr1: Optional[torch.Tensor] = None, unit_norm: Optional[bool] = None):
    """The dual-softmax matcher with its CUDA backward.

    dsc0, dsc1: fp32 [B, 128, N] (CUDA, any strides); dustbin: the dustbin logit (a one-element tensor on the same device)
    or None; temperature > 0.  Returns scores [B, N, N], or with scr0 / scr1 ([B, N] or [B, 1, N]) the tuple
    (scores, kp_scores, final_scores).  Differentiable in dsc0, dsc1, dustbin, scr0 and scr1.

    unit_norm: whether every descriptor has norm <= 1; None checks it (one device-to-host copy).  It selects the same
    row / column partials as mk_match, so the outputs are bit-identical to the inference engine's on the same descriptors.
    """
    _check_dsc("dsc0", dsc0)
    _check_dsc("dsc1", dsc1)
    if dsc0.shape != dsc1.shape or dsc0.device != dsc1.device:
        raise ValueError(f"dsc0 and dsc1 must have one shape and device, got {tuple(dsc0.shape)} on {dsc0.device} and "
                         f"{tuple(dsc1.shape)} on {dsc1.device}")
    B, _, N = dsc0.shape
    dev = dsc0.device
    if B < 1 or not 2 <= N <= MAX_N:
        raise ValueError(f"dual_softmax needs B >= 1 and 2 <= N <= {MAX_N}, got B {B}, N {N}")
    try:
        T = float(temperature)
    except (TypeError, ValueError):
        raise ValueError(f"temperature must be a real number, got {temperature!r}") from None
    if not (math.isfinite(T) and T > 0 and math.isfinite(1.0 / T)):
        raise ValueError(f"temperature must be positive and finite, got {temperature!r}")
    if dustbin is not None:
        if not torch.is_tensor(dustbin) or dustbin.numel() != 1:
            raise ValueError("dustbin must be a one-element tensor or None")
        if dustbin.dtype != torch.float32 or dustbin.device != dev:
            raise ValueError(f"dustbin must be float32 on {dev}, got {dustbin.dtype} on {dustbin.device}")
    if (scr0 is None) != (scr1 is None):
        raise ValueError("scr0 and scr1 are given together or not at all")
    if scr0 is not None:
        _check_scr("scr0", scr0, B, N, dev)
        _check_scr("scr1", scr1, B, N, dev)
    if unit_norm is None:
        unit_norm = _is_unit_norm(dsc0, dsc1)
    return _DualSoftmax.apply(dsc0, dsc1, dustbin, scr0, scr1, T, bool(unit_norm))


class dualSoftmax(nn.Module):
    """Drop-in for the reference's dualSoftmax (feature_matcher.py:54-83): cfg is FEATURE_MATCHER.DUAL_SOFTMAX.
    forward(dsc0, dsc1) -> scores [B, N, N]; the backward runs in CUDA."""

    def __init__(self, cfg):
        super().__init__()
        self.temperature = cfg['TEMPERATURE']
        self.use_dustbin = False
        if cfg['USE_DUSTBIN']:
            self.dustbin_score = nn.Parameter(torch.tensor(1.))
            self.use_dustbin = True

    def forward(self, dsc0, dsc1):
        return dual_softmax(dsc0, dsc1, self.dustbin_score if self.use_dustbin else None, self.temperature)
