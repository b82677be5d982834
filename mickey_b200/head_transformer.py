"""The heads' linear-attention transformer as a trainable module: the forward and the backward in CUDA
(csrc/head_transformer.cu).

`Transformer_self_att(d_model=128, num_layers=3, add_posEnc=False)` is a drop-in for the reference's class
(lib/models/MicKey/modules/att_layers/transformer.py:44-103, EncoderLayer in transformer_utils.py:8-66): the same
parameter names and shapes, the same non-persistent `posEnc.pe` buffer and the same attributes, so a head's trained
`att_layer.state_dict()` loads with strict=True.  Its forward takes fp32 [B, 128, h, w] on CUDA (any strides) and returns
a fresh contiguous fp32 [B, 128, h, w], differentiable in the input and every parameter; the arithmetic is fp32
throughout, as the reference trains it.  Under torch.no_grad() it runs the forward only and keeps nothing.
INTEGRATION.md shows the swap in a training model.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from . import _lib

D_MODEL = 128
NHEADS = 8
PE_MAX = 256
MAX_B = 65535                 # the kernels' per-image grids (gridDim.y)
MAX_TOKENS = 65535 * 64       # the GEMMs' 64-token tiles (gridDim.y)
MAX_LAYERS = 1024
_NAMES = ("q_proj", "k_proj", "v_proj", "merge", "mlp0", "mlp2", "norm1_w", "norm1_b", "norm2_w", "norm2_b")


def _layer_table(params, num_layers):
    """params: 10 * num_layers tensors in _NAMES order per layer -> ctypes array of mk_htr_layer."""
    tab = (_lib.MkHtrLayer * num_layers)()
    for i in range(num_layers):
        for j, name in enumerate(_NAMES):
            setattr(tab[i], name, params[10 * i + j].data_ptr())
    return tab


def _aligned(t):
    """Contiguous and 16-byte aligned (the kernels read parameters as float4)."""
    t = t.contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()


def _forward(x, pe, params, num_layers, save):
    B, _, h, w = x.shape
    dev = x.device
    lib = _lib.load()
    with torch.cuda.device(dev):
        out = torch.empty(B, D_MODEL, h, w, dtype=torch.float32, device=dev)
        ws = _lib.workspace(lib.mk_head_transformer_ws_bytes(B, h, w, num_layers, int(save)), dev,
                            "mk_head_transformer_ws_bytes")
        _lib.check(lib.mk_head_transformer(_lib.ptr(x), _lib.ptr(pe), B, h, w, _layer_table(params, num_layers), num_layers,
                                           _lib.ptr(out), int(save), _lib.ptr(ws), ws.numel(), _lib.stream(dev)),
                   "mk_head_transformer")
    return out, ws


class _HeadTransformer(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, pe, num_layers, *params):
        params = [_aligned(p) for p in params]
        out, saved = _forward(x, pe, params, num_layers, save=True)
        ctx.save_for_backward(saved, *params)
        ctx.num_layers = num_layers
        ctx.shape = tuple(x.shape)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        saved, *params = ctx.saved_tensors
        L = ctx.num_layers
        B, _, h, w = ctx.shape
        dev = saved.device
        need = ctx.needs_input_grad
        lib = _lib.load()
        g = _aligned(grad_out.float())
        with torch.cuda.device(dev):
            gx = torch.empty(ctx.shape, dtype=torch.float32, device=dev) if need[0] else None
            grads = [torch.empty_like(p) if need[3 + i] else None for i, p in enumerate(params)]
            gtab = (_lib.MkHtrLayerGrads * L)()
            for i in range(L):
                for j, name in enumerate(_NAMES):
                    t = grads[10 * i + j]
                    setattr(gtab[i], name, None if t is None else t.data_ptr())
            ws = _lib.workspace(lib.mk_head_transformer_backward_ws_bytes(B, h, w, L), dev,
                                "mk_head_transformer_backward_ws_bytes")
            _lib.check(lib.mk_head_transformer_backward(_lib.ptr(saved), _lib.ptr(g), B, h, w, _layer_table(params, L), L,
                                                        _lib.ptr(gx), gtab, _lib.ptr(ws), ws.numel(), _lib.stream(dev)),
                       "mk_head_transformer_backward")
        return (gx, None, None, *grads)


def head_transformer(x: torch.Tensor, params, pe=None) -> torch.Tensor:
    """Transformer_self_att's forward on x fp32 [B, 128, h, w] (CUDA, any strides) with the layers' parameters `params`
    (10 per layer: q_proj, k_proj, v_proj, merge, mlp.0, mlp.2 weights, norm1 weight and bias, norm2 weight and bias) and
    the positional encoding pe ([1, 128, 256, 256], added as pe[:, :, :h, :w]) or None.  Returns a fresh contiguous fp32
    [B, 128, h, w], differentiable in x and params."""
    if not torch.is_tensor(x):
        raise ValueError(f"x must be a torch tensor, got {type(x).__name__}")
    if x.dtype != torch.float32:
        raise ValueError(f"x must be float32, got {x.dtype}")
    if x.dim() != 4 or x.shape[1] != D_MODEL:
        raise ValueError(f"x must be [B, {D_MODEL}, h, w], got {tuple(x.shape)}")
    B, _, h, w = x.shape
    if B < 1 or h < 1 or w < 1:
        raise ValueError(f"x must have B, h, w >= 1, got {tuple(x.shape)}")
    if len(params) == 0 or len(params) % 10 or len(params) > 10 * MAX_LAYERS:
        raise ValueError(f"params must hold 10 tensors per layer for 1 to {MAX_LAYERS} layers, got {len(params)}")
    num_layers = len(params) // 10
    for i, p in enumerate(params):
        shape = {3: (D_MODEL, D_MODEL), 4: (2 * D_MODEL, 2 * D_MODEL), 5: (D_MODEL, 2 * D_MODEL)}.get(
            i % 10, (D_MODEL, D_MODEL) if i % 10 < 3 else (D_MODEL,))
        if not torch.is_tensor(p) or p.dtype != torch.float32 or p.device != x.device or tuple(p.shape) != shape:
            got = f"{tuple(p.shape)} {p.dtype} on {p.device}" if torch.is_tensor(p) else type(p).__name__
            raise ValueError(f"layer {i // 10} {_NAMES[i % 10]} must be float32 {shape} on {x.device}, got {got}")
    if pe is not None:
        if h > PE_MAX or w > PE_MAX:
            raise ValueError(f"the positional encoding covers at most {PE_MAX} x {PE_MAX} positions, got {h} x {w}")
        if tuple(pe.shape) != (1, D_MODEL, PE_MAX, PE_MAX) or pe.dtype != torch.float32 or pe.device != x.device:
            raise ValueError(f"pe must be float32 [1, {D_MODEL}, {PE_MAX}, {PE_MAX}] on {x.device}, got "
                             f"{tuple(pe.shape)} {pe.dtype} on {pe.device}")
        pe = _aligned(pe)
    if B > MAX_B or B * h * w > MAX_TOKENS:
        raise ValueError(f"at most {MAX_B} images and {MAX_TOKENS} tokens per call, got B {B}, {B * h * w} tokens")
    if x.device.type != "cuda":
        raise ValueError(f"x must be on a CUDA device (mickey_b200 has no CPU path), got {x.device}")
    x = _aligned(x)
    if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params)):
        return _HeadTransformer.apply(x, pe, num_layers, *params)
    with torch.no_grad():
        return _forward(x, pe, [_aligned(p) for p in params], num_layers, save=False)[0]


def sine_table(d_model: int = D_MODEL, size: int = PE_MAX) -> torch.Tensor:
    """The heads' 2-D sine positional encoding [d_model, size, size]: for k < d_model / 4, with positions p = 1 .. size
    and f_k = exp(2k * -ln(10^4) / (d_model / 2)), channel 4k is sin(f_k x), 4k + 1 cos(f_k x), 4k + 2 sin(f_k y) and
    4k + 3 cos(f_k y).  Every angle is the fp32 product f_k * p, so the table equals the reference's buffer bit for bit."""
    f = (torch.arange(0, d_model // 2, 2, dtype=torch.float32) * (-math.log(10000.0) / (d_model // 2))).exp()
    p = torch.arange(1, size + 1, dtype=torch.float32)
    col = (f[:, None, None] * p[None, None, :]).expand(-1, size, size)     # varies along x
    row = (f[:, None, None] * p[None, :, None]).expand(-1, size, size)     # varies along y
    return torch.stack([col.sin(), col.cos(), row.sin(), row.cos()], 1).reshape(d_model, size, size)


class PositionEncodingSine(nn.Module):
    """Holds sine_table() as the non-persistent buffer `pe` [1, d_model, 256, 256], as the reference's module does."""

    def __init__(self, d_model):
        super().__init__()
        self.register_buffer("pe", sine_table(d_model)[None], persistent=False)


class EncoderLayer(nn.Module):
    """The parameters of the reference's EncoderLayer (transformer_utils.py:8-38) with linear attention: no biases."""

    def __init__(self, d_model, nhead):
        super().__init__()
        self.dim = d_model // nhead
        self.nhead = nhead
        self.q_proj = nn.Linear(d_model, d_model, bias=False)
        self.k_proj = nn.Linear(d_model, d_model, bias=False)
        self.v_proj = nn.Linear(d_model, d_model, bias=False)
        self.merge = nn.Linear(d_model, d_model, bias=False)
        self.mlp = nn.Sequential(nn.Linear(d_model * 2, d_model * 2, bias=False), nn.ReLU(True),
                                 nn.Linear(d_model * 2, d_model, bias=False))
        self.norm1 = nn.LayerNorm(d_model)
        self.norm2 = nn.LayerNorm(d_model)

    def params(self):
        return [self.q_proj.weight, self.k_proj.weight, self.v_proj.weight, self.merge.weight, self.mlp[0].weight,
                self.mlp[2].weight, self.norm1.weight, self.norm1.bias, self.norm2.weight, self.norm2.bias]


class Transformer_self_att(nn.Module):
    """Drop-in for the reference's Transformer_self_att with d_model = 128 (the heads' only size) and its 8 heads."""

    def __init__(self, d_model=D_MODEL, num_layers=3, add_posEnc=False):
        super().__init__()
        if d_model != D_MODEL:
            raise ValueError(f"Transformer_self_att runs d_model = {D_MODEL} only, got {d_model}")
        if int(num_layers) != num_layers or not 1 <= num_layers <= MAX_LAYERS:
            raise ValueError(f"num_layers must be an integer in [1, {MAX_LAYERS}], got {num_layers}")
        self.d_model = d_model
        self.nheads = NHEADS
        self.layer_names = ['self'] * int(num_layers)
        self.layers = nn.ModuleList([EncoderLayer(d_model, self.nheads) for _ in self.layer_names])
        self._reset_parameters()
        self.add_posEnc = add_posEnc
        self.posEnc = PositionEncodingSine(d_model)

    def _reset_parameters(self):
        for p in self.parameters():
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)

    def forward(self, feats):
        params = [p for layer in self.layers for p in layer.params()]
        return head_transformer(feats, params, self.posEnc.pe if self.add_posEnc else None)
