"""The heads' residual block as a trainable module: TF32 wgmma convolutions and batch norm, forward and backward in CUDA
(csrc/resblock.cu).

`BasicBlock(in_planes, planes, stride=1, bn=True, padding_mode='zeros')` is a drop-in for the reference's class
(lib/models/MicKey/modules/utils/extractor_utils.py:12-35): the same submodules (`conv1`, `bn1`, `conv2`, `bn2`, and
`shortcut.0` when the widths differ), real nn.Conv2d / nn.BatchNorm2d / nn.Identity modules, so a head's trained
`resblockK.state_dict()` loads with strict=True.  Its forward takes fp32 [B, in_planes, h, w] on CUDA (any strides) and
returns a fresh contiguous fp32 [B, planes, h, w], differentiable in the input and every parameter.

The convolutions run as TF32 tensor-core GEMMs with fp32 accumulation: the arithmetic torch uses for the reference's
convolutions under its default `torch.backends.cudnn.allow_tf32 = True`.  With that flag off the forward raises rather
than compute at a precision the caller turned off.  In train mode the batch norms normalise with batch statistics and
update the running statistics exactly as F.batch_norm does (also under torch.no_grad()); in eval mode they use the running
statistics.  INTEGRATION.md shows the swap in a training model.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from . import _lib

MAX_ROWS = 1 << 24            # B (h+2)(w+2): padded rows of the kernels' NHWC buffers
MAX_CHANNELS = 4096
TRAIN, RELU, SAVE, BN = 1, 2, 4, 8


def _strides(t):
    return (C.c_longlong * 4)(*t.stride())


def _params(w1, w2, wsc, bn1, bn2, mom1, mom2):
    p = _lib.MkResblockParams()
    p.w1, p.w2, p.wsc = w1.data_ptr(), w2.data_ptr(), None if wsc is None else wsc.data_ptr()
    if bn1 is not None:
        p.bn1_w, p.bn1_b, p.bn1_mean, p.bn1_var = (t.data_ptr() for t in bn1[:4])
        p.bn2_w, p.bn2_b, p.bn2_mean, p.bn2_var = (t.data_ptr() for t in bn2[:4])
        p.eps1, p.eps2 = float(bn1[4]), float(bn2[4])
        p.momentum1, p.momentum2 = float(mom1), float(mom2)
    return p


def _forward(x, w1, w2, wsc, bn1, bn2, mom1, mom2, flags):
    B, cin, h, w = x.shape
    cout = w1.shape[0]
    dev = x.device
    lib = _lib.load()
    with torch.cuda.device(dev):
        out = torch.empty(B, cout, h, w, dtype=torch.float32, device=dev)
        saved = _lib.workspace(lib.mk_resblock_saved_bytes(B, h, w, cin, cout), dev, "mk_resblock_saved_bytes")
        ws = _lib.workspace(lib.mk_resblock_ws_bytes(B, h, w, cin, cout), dev, "mk_resblock_ws_bytes")
        P = _params(w1, w2, wsc, bn1, bn2, mom1, mom2)
        _lib.check(lib.mk_resblock_forward(_lib.ptr(x), _strides(x), B, h, w, cin, cout, C.byref(P), flags, _lib.ptr(out),
                                           _lib.ptr(saved), saved.numel(), _lib.ptr(ws), ws.numel(), _lib.stream(dev)),
                   "mk_resblock_forward")
    return out, saved       # the scratch workspace is released here; only the saved region outlives the call


class _ResBlock(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w1, w2, wsc, g1, b1, g2, b2, bn1, bn2, mom1, mom2, flags):
        # bn1 / bn2: (weight, bias, running_mean, running_var, eps) or None; weight and bias are g1, b1 / g2, b2
        out, saved = _forward(x, w1, w2, wsc, bn1, bn2, mom1, mom2, flags | SAVE)
        B, cin, h, w = x.shape
        ctx.save_for_backward(saved, out, w1, w2, wsc, g1, g2)
        ctx.flags = flags
        ctx.shape = (B, cin, h, w)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        saved, out, w1, w2, wsc, g1, g2 = ctx.saved_tensors
        B, cin, h, w = ctx.shape
        cout = w1.shape[0]
        need = ctx.needs_input_grad
        dev = saved.device
        lib = _lib.load()
        g = grad_out.float()
        with torch.cuda.device(dev):
            names = ("dx", "w1", "w2", "wsc", "bn1_w", "bn1_b", "bn2_w", "bn2_b")
            like = (None, w1, w2, wsc, g1, g1, g2, g2)
            grads = [None] * 8
            G = _lib.MkResblockGrads()
            want = 0
            for i in range(8):
                if need[i]:
                    grads[i] = (torch.empty(ctx.shape, dtype=torch.float32, device=dev) if i == 0
                                else torch.empty_like(like[i], memory_format=torch.contiguous_format))
                    setattr(G, names[i], grads[i].data_ptr())
                    want |= 1 << i
            P = _lib.MkResblockParams()
            P.w1, P.w2, P.wsc = w1.data_ptr(), w2.data_ptr(), None if wsc is None else wsc.data_ptr()
            if g1 is not None:
                P.bn1_w, P.bn2_w = g1.data_ptr(), g2.data_ptr()
            ws = _lib.workspace(lib.mk_resblock_backward_ws_bytes(B, h, w, cin, cout), dev, "mk_resblock_backward_ws_bytes")
            _lib.check(lib.mk_resblock_backward(_lib.ptr(saved), _lib.ptr(g), _strides(g), _lib.ptr(out), B, h, w, cin, cout,
                                                C.byref(P), ctx.flags, want, C.byref(G), _lib.ptr(ws), ws.numel(),
                                                _lib.stream(dev)),
                       "mk_resblock_backward")
        return (*grads, None, None, None, None, None)


class BasicBlock(nn.Module):
    """Drop-in for the reference's BasicBlock (pre-activation residual block of the heads) with stride 1 and zero
    padding, the only configuration MicKey builds."""
    expansion = 1

    def __init__(self, in_planes, planes, stride=1, bn=True, padding_mode='zeros'):
        super().__init__()
        if stride != 1:
            raise ValueError(f"BasicBlock runs stride 1 only, got {stride}")
        if padding_mode != 'zeros':
            raise ValueError(f"BasicBlock runs padding_mode 'zeros' only, got {padding_mode!r}")
        for name, c in (("in_planes", in_planes), ("planes", planes)):
            if int(c) != c or c < 32 or c > MAX_CHANNELS or c % 32:
                raise ValueError(f"{name} must be a multiple of 32 in [32, {MAX_CHANNELS}], got {c}")
        self.conv1 = nn.Conv2d(in_planes, planes, kernel_size=3, stride=stride, padding=1, bias=False, padding_mode=padding_mode)
        self.bn1 = nn.BatchNorm2d(planes) if bn else nn.Identity()
        self.conv2 = nn.Conv2d(planes, planes, kernel_size=3, stride=1, padding=1, bias=False, padding_mode=padding_mode)
        self.bn2 = nn.BatchNorm2d(planes) if bn else nn.Identity()
        if stride != 1 or in_planes != self.expansion * planes:
            self.shortcut = nn.Sequential(nn.Conv2d(in_planes, self.expansion * planes, kernel_size=1, stride=stride, bias=False))

    def _check(self, x):
        if not torch.is_tensor(x):
            raise ValueError(f"x must be a torch tensor, got {type(x).__name__}")
        cin = self.conv1.in_channels
        if x.dtype != torch.float32 or x.dim() != 4 or x.shape[1] != cin:
            raise ValueError(f"x must be float32 [B, {cin}, h, w], got {x.dtype} {tuple(x.shape)}")
        B, _, h, w = x.shape
        if B < 1 or h < 1 or w < 1:
            raise ValueError(f"x must have B, h, w >= 1, got {tuple(x.shape)}")
        if B * (h + 2) * (w + 2) > MAX_ROWS:
            raise ValueError(f"B (h+2)(w+2) must be at most {MAX_ROWS}, got {B * (h + 2) * (w + 2)}")
        bns = [m for m in (self.bn1, self.bn2) if isinstance(m, nn.BatchNorm2d)]
        if len(bns) == 1 or any(not isinstance(m, (nn.BatchNorm2d, nn.Identity)) for m in (self.bn1, self.bn2)):
            raise ValueError("bn1 and bn2 must both be nn.BatchNorm2d or both nn.Identity, got "
                             f"{type(self.bn1).__name__} and {type(self.bn2).__name__}")
        for m in bns:
            if not m.affine or not m.track_running_stats:
                raise ValueError("BasicBlock needs batch norm with affine=True and track_running_stats=True")
        if bns and self.bn1.training != self.bn2.training:
            raise ValueError("bn1 and bn2 must both be in train mode or both in eval mode")
        if bns and self.bn1.training and B * h * w == 1:
            raise ValueError(f"expected more than 1 value per channel when training, got input size {tuple(x.shape)}")
        if x.device.type != "cuda":
            raise ValueError(f"x must be on a CUDA device (mickey_b200 has no CPU path), got {x.device}")
        for p in self.parameters():
            if p.device != x.device or p.dtype != torch.float32:
                raise ValueError(f"parameters must be float32 on {x.device}, got {p.dtype} on {p.device}")
        if not torch.backends.cudnn.allow_tf32:
            raise RuntimeError("BasicBlock computes its convolutions in TF32, and torch.backends.cudnn.allow_tf32 is False: "
                               "the reference's convolutions would then run in full fp32, which this module does not "
                               "implement")

    @staticmethod
    def _momentum(m):
        """F.batch_norm's exponential-average factor for this call: BatchNorm2d.forward's, after its num_batches_tracked
        update (the counter itself moves only once the call has been launched)."""
        return 1.0 / float(m.num_batches_tracked + 1) if m.momentum is None else m.momentum

    def _count_batch(self):
        for m in (self.bn1, self.bn2):
            m.num_batches_tracked.add_(1)

    def forward(self, x, relu=True):
        self._check(x)
        has_bn = isinstance(self.bn1, nn.BatchNorm2d)
        train = has_bn and self.bn1.training
        flags = (TRAIN if train else 0) | (RELU if relu else 0) | (BN if has_bn else 0)
        mom1 = mom2 = 0.0
        if train:
            mom1, mom2 = self._momentum(self.bn1), self._momentum(self.bn2)
        w1, w2 = self.conv1.weight.contiguous(), self.conv2.weight.contiguous()
        wsc = self.shortcut[0].weight.contiguous() if hasattr(self, "shortcut") else None
        if has_bn:
            g1, b1, g2, b2 = self.bn1.weight, self.bn1.bias, self.bn2.weight, self.bn2.bias
            bn1 = (g1, b1, self.bn1.running_mean, self.bn1.running_var, self.bn1.eps)
            bn2 = (g2, b2, self.bn2.running_mean, self.bn2.running_var, self.bn2.eps)
            for t in (g1, b1, g2, b2, *bn1[2:4], *bn2[2:4]):
                if not t.is_contiguous():
                    raise ValueError("batch-norm parameters and buffers must be contiguous")
        else:
            g1 = b1 = g2 = b2 = bn1 = bn2 = None
        params = [w1, w2, wsc, g1, b1, g2, b2]
        if torch.is_grad_enabled() and (x.requires_grad or any(p is not None and p.requires_grad for p in params)):
            out = _ResBlock.apply(x, *params, bn1, bn2, mom1, mom2, flags)
        else:
            with torch.no_grad():
                out = _forward(x, w1, w2, wsc, bn1, bn2, mom1, mom2, flags)[0]
        if train:
            self._count_batch()
        return out
