"""MicKey's four heads as trainable modules, every layer forward and backward in CUDA.

`head_out(x, kind, weight, ...)` is the heads' output layer (csrc/head_out.cu): the 1x1 convolution and activation of the
keypoint heads, or the descriptor head's L2 normalisation, in fp32, differentiable in x and the weight.

`DeepResBlock_det`, `DeepResBlock_offset`, `DeepResBlock_depth` and `DeepResBlock_desc(config, padding_mode='zeros')` are
drop-ins for the reference's classes (lib/models/MicKey/modules/mickey_extractor.py:67-251), built from `config` =
cfg['MICKEY'] as the reference builds them.  They hold the reference's submodules and parameters under the reference's
names (resblock1..4 as mickey_b200.resblock.BasicBlock, att_layer as mickey_b200.head_transformer.Transformer_self_att,
the output convolutions as nn.Conv2d, the det head's frozen eps / offset_par1 / offset_par2 / ones_kernel), so a head's
state_dict() loads with strict=True both ways.  forward(feature_volume) chains rb1 -> rb2 -> rb3 -> att_layer -> rb4 ->
the output layer and returns exactly what the reference head returns.  mickey_b200.training.use_cuda_modules moves a
whole training model onto these modules.
"""
from __future__ import annotations

import ctypes as C
import math

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from . import _lib
from .head_transformer import Transformer_self_att
from .resblock import BasicBlock

KINDS = {"score_softmax": 0, "score_sigmoid": 1, "offset": 2, "depth": 3, "depth_sigmoid": 4, "desc": 5}
DESC = KINDS["desc"]
MAX_C = 4096
MAX_PIXELS = 1 << 26          # B h w


def _strides(t):
    return (C.c_longlong * 4)(*t.stride())


def _outputs(kind, C_):
    return 2 if kind == KINDS["offset"] else C_ if kind == DESC else 1


def _forward(kind, x, weight, eps, temperature, max_depth, save):
    B, C_, h, w = x.shape
    dev = x.device
    lib = _lib.load()
    with torch.cuda.device(dev):
        out = torch.empty(B, _outputs(kind, C_), h, w, dtype=torch.float32, device=dev)
        norm = torch.empty(B, h, w, dtype=torch.float32, device=dev) if kind == DESC and save else None
        _lib.check(lib.mk_head_out_forward(kind, _lib.ptr(x), _strides(x), B, C_, h, w, _lib.ptr(weight), _lib.ptr(eps),
                                           temperature, max_depth, _lib.ptr(out), _lib.ptr(norm), _lib.stream(dev)),
                   "mk_head_out_forward")
    return out, norm


class _HeadOut(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, eps, kind, temperature, max_depth):
        out, norm = _forward(kind, x, weight, eps, temperature, max_depth, save=True)
        ctx.save_for_backward(x, weight, out, norm)      # x as given: the backward reads it in place
        ctx.args = (kind, temperature, max_depth)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        x, weight, out, norm = ctx.saved_tensors
        kind, temperature, max_depth = ctx.args
        need = ctx.needs_input_grad
        B, C_, h, w = x.shape
        dev = out.device
        lib = _lib.load()
        g = grad_out.float().contiguous()
        with torch.cuda.device(dev):
            gx = torch.empty(B, C_, h, w, dtype=torch.float32, device=dev) if need[0] else None
            gw = torch.empty_like(weight, memory_format=torch.contiguous_format) if need[1] else None
            ws = _lib.workspace(lib.mk_head_out_backward_ws_bytes(kind, B, h, w, C_), dev, "mk_head_out_backward_ws_bytes")
            _lib.check(lib.mk_head_out_backward(kind, _lib.ptr(x), _strides(x), B, C_, h, w, _lib.ptr(weight), temperature,
                                                max_depth, _lib.ptr(out), _lib.ptr(norm), _lib.ptr(g), _lib.ptr(gx),
                                                _lib.ptr(gw), _lib.ptr(ws), ws.numel(), _lib.stream(dev)),
                       "mk_head_out_backward")
        return gx, gw, None, None, None, None


def head_out(x: torch.Tensor, kind: str, weight=None, eps=None, temperature: float = 100.0,
             max_depth: float = 1.0) -> torch.Tensor:
    """The output layer `kind` of a head on x = rb4's output, fp32 [B, C, h, w] on CUDA with any strides.  Returns a fresh
    contiguous fp32 [B, k, h, w], differentiable in x and weight:

        "score_softmax"  weight [1, C]  e / (sum e + eps), e = exp((r - (mean r + eps)) / temperature) with 3 border cells
                                        zeroed, per image (remove_brd_and_softmax, mickey_extractor.py:112-124)
        "score_sigmoid"  weight [1, C]  sigmoid(r) with 3 border cells zeroed (:140)
        "offset"         weight [2, C]  sigmoid(r) (:173-176)
        "depth"          weight [1, C]  r (:216)
        "depth_sigmoid"  weight [1, C]  max_depth sigmoid(r) (:214)
        "desc"           no weight      x / sqrt(sum_c x^2 + 1e-10) (desc_l2norm, extractor_utils.py:6-10)

    r is the 1x1 convolution W x (weight [k, C] or the conv's [k, C, 1, 1]).  eps is the det head's device scalar
    Parameter (read on the device, never differentiated); the mean is detached as in the reference."""
    if kind not in KINDS:
        raise ValueError(f"kind must be one of {sorted(KINDS)}, got {kind!r}")
    k_id = KINDS[kind]
    if not torch.is_tensor(x):
        raise ValueError(f"x must be a torch tensor, got {type(x).__name__}")
    if x.dtype != torch.float32 or x.dim() != 4:
        raise ValueError(f"x must be float32 [B, C, h, w], got {x.dtype} {tuple(x.shape)}")
    B, C_, h, w = x.shape
    if B < 1 or h < 1 or w < 1 or not 1 <= C_ <= MAX_C:
        raise ValueError(f"x must have B, h, w >= 1 and 1 <= C <= {MAX_C}, got {tuple(x.shape)}")
    if B * h * w > MAX_PIXELS:
        raise ValueError(f"B h w must be at most {MAX_PIXELS}, got {B * h * w}")
    if k_id == DESC:
        if weight is not None:
            raise ValueError("the descriptor layer has no weight")
    else:
        k = _outputs(k_id, C_)
        if not torch.is_tensor(weight) or weight.dtype != torch.float32 or weight.device != x.device or \
                tuple(weight.shape) not in ((k, C_), (k, C_, 1, 1)):
            got = f"{weight.dtype} {tuple(weight.shape)} on {weight.device}" if torch.is_tensor(weight) else repr(weight)
            raise ValueError(f"{kind} needs a float32 weight [{k}, {C_}] or [{k}, {C_}, 1, 1] on {x.device}, got {got}")
        weight = weight.reshape(k, C_).contiguous()
    if k_id == KINDS["score_softmax"]:
        if not torch.is_tensor(eps) or eps.numel() != 1 or eps.dtype != torch.float32 or eps.device != x.device:
            got = f"{eps.dtype} {tuple(eps.shape)} on {eps.device}" if torch.is_tensor(eps) else repr(eps)
            raise ValueError(f"score_softmax needs eps as a one-element float32 tensor on {x.device}, got {got}")
        if eps.requires_grad:
            raise ValueError("eps must not require grad: the layer does not differentiate it")
        eps = eps.detach().reshape(1).contiguous()
        temperature = float(temperature)
        if not (math.isfinite(temperature) and temperature > 0):
            raise ValueError(f"temperature must be finite and > 0, got {temperature}")
    else:
        eps, temperature = None, 1.0
    max_depth = float(max_depth)
    if k_id == KINDS["depth_sigmoid"] and not (math.isfinite(max_depth) and max_depth != 0):
        raise ValueError(f"max_depth must be finite and non-zero, got {max_depth}")
    if x.device.type != "cuda":
        raise ValueError(f"x must be on a CUDA device (mickey_b200 has no CPU path), got {x.device}")
    if torch.is_grad_enabled() and (x.requires_grad or (weight is not None and weight.requires_grad)):
        return _HeadOut.apply(x, weight, eps, k_id, temperature, max_depth)
    with torch.no_grad():
        return _forward(k_id, x, weight, eps, temperature, max_depth, save=False)[0]


class _Head(nn.Module):
    """rb1 -> rb2 -> rb3 -> att_layer -> rb4, shared by the four heads (mickey_extractor.py:128-132 and the like)."""

    def _blocks(self, config, last_dim, padding_mode):
        bn = config['KP_HEADS']['BN']
        dims = config['KP_HEADS']['BLOCKS_DIM']
        cin = config['DINOV2']['CHANNEL_DIM']
        outs = [dims[0], dims[1], dims[2], last_dim]
        for i, (a, b) in enumerate(zip([cin] + outs[:3], outs)):
            setattr(self, f"resblock{i + 1}", BasicBlock(a, b, stride=1, bn=bn, padding_mode=padding_mode))

    def _trunk(self, feature_volume, relu=True):
        x = self.resblock1(feature_volume)
        x = self.resblock2(x)
        x = self.resblock3(x)
        x = self.att_layer(x)
        return self.resblock4(x, relu=relu)


class DeepResBlock_det(_Head):
    """Drop-in for the reference's keypoint-score head (mickey_extractor.py:67-142)."""

    def __init__(self, config, padding_mode='zeros'):
        super().__init__()
        self._blocks(config, config['KP_HEADS']['BLOCKS_DIM'][3], padding_mode)
        self.score = nn.Conv2d(config['KP_HEADS']['BLOCKS_DIM'][3], 1, kernel_size=1, stride=1, padding=0, bias=False)
        self.use_softmax = config['KP_HEADS']['USE_SOFTMAX']
        self.sigmoid = torch.nn.Sigmoid()
        self.logsigmoid = torch.nn.LogSigmoid()
        self.softmax = torch.nn.Softmax(dim=-1)
        self.tmp_softmax = 100
        self.eps = nn.Parameter(torch.tensor(1e-16), requires_grad=False)
        self.offset_par1 = nn.Parameter(torch.tensor(0.5), requires_grad=False)
        self.offset_par2 = nn.Parameter(torch.tensor(2.), requires_grad=False)
        self.ones_kernel = nn.Parameter(torch.ones((1, 1, 3, 3)), requires_grad=False)
        self.att_layer = Transformer_self_att(d_model=128, num_layers=3, add_posEnc=config['KP_HEADS']['POS_ENCODING'])

    def forward(self, feature_volume):
        x = self._trunk(feature_volume)
        if self.use_softmax:
            return head_out(x, "score_softmax", self.score.weight, eps=self.eps, temperature=self.tmp_softmax)
        return head_out(x, "score_sigmoid", self.score.weight)


class DeepResBlock_offset(_Head):
    """Drop-in for the reference's keypoint-offset head (mickey_extractor.py:145-178)."""

    def __init__(self, config, padding_mode='zeros'):
        super().__init__()
        self.sigmoid = torch.nn.Sigmoid()
        self._blocks(config, config['KP_HEADS']['BLOCKS_DIM'][3], padding_mode)
        self.xy_offset = nn.Conv2d(config['KP_HEADS']['BLOCKS_DIM'][3], 2, kernel_size=1, stride=1, padding=0, bias=False)
        self.att_layer = Transformer_self_att(d_model=128, num_layers=3, add_posEnc=config['KP_HEADS']['POS_ENCODING'])

    def forward(self, feature_volume):
        return head_out(self._trunk(feature_volume), "offset", self.xy_offset.weight)


class DeepResBlock_depth(_Head):
    """Drop-in for the reference's depth head (mickey_extractor.py:181-218)."""

    def __init__(self, config, padding_mode='zeros'):
        super().__init__()
        self.use_depth_sigmoid = config['KP_HEADS']['USE_DEPTHSIGMOID']
        self.max_depth = config['KP_HEADS']['MAX_DEPTH']
        self.sigmoid = torch.nn.Sigmoid()
        self._blocks(config, config['KP_HEADS']['BLOCKS_DIM'][3], padding_mode)
        self.depth = nn.Conv2d(config['KP_HEADS']['BLOCKS_DIM'][3], 1, kernel_size=1, stride=1, padding=0, bias=False)
        self.att_layer = Transformer_self_att(d_model=128, num_layers=3, add_posEnc=config['KP_HEADS']['POS_ENCODING'])

    def forward(self, feature_volume):
        x = self._trunk(feature_volume)
        if self.use_depth_sigmoid:
            return head_out(x, "depth_sigmoid", self.depth.weight, max_depth=self.max_depth)
        return head_out(x, "depth", self.depth.weight)


class DeepResBlock_desc(_Head):
    """Drop-in for the reference's descriptor head (mickey_extractor.py:221-251)."""

    def __init__(self, config, padding_mode='zeros'):
        super().__init__()
        self.norm_desc = config['DSC_HEAD']['NORM_DSC']
        self._blocks(config, config['DSC_HEAD']['LAST_DIM'], padding_mode)
        self.att_layer = Transformer_self_att(d_model=128, num_layers=3, add_posEnc=config['DSC_HEAD']['POS_ENCODING'])

    def forward(self, feature_volume):
        x = self._trunk(feature_volume, relu=False)
        return head_out(x, "desc") if self.norm_desc else x
