"""Functional restatement of the heads' residual block (BasicBlock) in train and eval mode, with a closed-form backward.

    z1 = conv3x3(x, w1);  a1 = relu(bn1(z1));  z2 = conv3x3(a1, w2);  s = conv1x1(x, wsc) or x
    out = act(bn2(z2) + s)                     act = relu, or the identity for relu=False (the descriptor head's rb4)

bn(z) = (z - mean) / sqrt(var + eps) * weight + bias, with the batch mean and biased variance over (B, h, w) in train mode
(the running statistics then move by the exponential-average factor, the unbiased variance into running_var) and the
running statistics in eval mode.  Device- and dtype-agnostic: it computes in the dtype of its inputs.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def _bn(z, p, train):
    """p: dict(weight, bias, running_mean, running_var, eps, factor) or None.  Returns (y, xhat, rstd, mean, var)."""
    if p is None:
        return z, None, None, None, None
    if train:
        mean = z.mean((0, 2, 3))
        var = z.var((0, 2, 3), unbiased=False)
    else:
        mean, var = p["running_mean"].to(z.dtype), p["running_var"].to(z.dtype)
    rstd = (var + p["eps"]).rsqrt()
    xhat = (z - mean[None, :, None, None]) * rstd[None, :, None, None]
    y = xhat * p["weight"][None, :, None, None] + p["bias"][None, :, None, None]
    return y, xhat, rstd, mean, var


def running_update(p, mean, var, count):
    """The running statistics after one train-mode call, as F.batch_norm leaves them (unbiased variance)."""
    f = p["factor"]
    rm = (1 - f) * p["running_mean"].to(mean.dtype) + f * mean
    rv = (1 - f) * p["running_var"].to(var.dtype) + f * var * count / (count - 1)
    return rm, rv


def block_forward(x, w1, w2, wsc, bn1, bn2, train=True, relu=True):
    """Returns (out, aux): aux holds the intermediates block_backward needs and the batch statistics."""
    z1 = F.conv2d(x, w1, padding=1)
    y1, xh1, rs1, m1, v1 = _bn(z1, bn1, train)
    a1 = F.relu(y1)
    z2 = F.conv2d(a1, w2, padding=1)
    y2, xh2, rs2, m2, v2 = _bn(z2, bn2, train)
    s = F.conv2d(x, wsc) if wsc is not None else x
    pre = y2 + s
    out = F.relu(pre) if relu else pre
    aux = dict(z1=z1, a1=a1, z2=z2, xh1=xh1, xh2=xh2, rs1=rs1, rs2=rs2, mean1=m1, var1=v1, mean2=m2, var2=v2, out=out)
    return out, aux


def _bn_backward(g, xhat, rstd, weight, train):
    """dz, dweight, dbias of y = xhat * weight + bias: dz = weight rstd / M (M g - sum g - xhat sum g xhat) in train mode,
    weight rstd g in eval mode."""
    sg = g.sum((0, 2, 3))
    sgx = (g * xhat).sum((0, 2, 3))
    k = (weight * rstd)[None, :, None, None]
    if train:
        M = g.numel() // g.shape[1]
        dz = k * (g - sg[None, :, None, None] / M - xhat * sgx[None, :, None, None] / M)
    else:
        dz = k * g
    return dz, sgx, sg


def block_backward(x, w1, w2, wsc, bn1, bn2, grad_out, aux, train=True, relu=True):
    """Closed-form gradients of block_forward: dict with dx, w1, w2, wsc, bn1_w, bn1_b, bn2_w, bn2_b (None where the
    block has no such parameter)."""
    gw = torch.nn.grad
    g = grad_out * (aux["out"] > 0) if relu else grad_out
    r = dict(wsc=None, bn1_w=None, bn1_b=None, bn2_w=None, bn2_b=None)
    if wsc is not None:
        r["wsc"] = gw.conv2d_weight(x, wsc.shape, g)
        dx_sc = gw.conv2d_input(x.shape, wsc, g)
    else:
        dx_sc = g
    if bn2 is not None:
        dz2, r["bn2_w"], r["bn2_b"] = _bn_backward(g, aux["xh2"], aux["rs2"], bn2["weight"], train)
    else:
        dz2 = g
    r["w2"] = gw.conv2d_weight(aux["a1"], w2.shape, dz2, padding=1)
    da1 = gw.conv2d_input(aux["a1"].shape, w2, dz2, padding=1) * (aux["a1"] > 0)
    if bn1 is not None:
        dz1, r["bn1_w"], r["bn1_b"] = _bn_backward(da1, aux["xh1"], aux["rs1"], bn1["weight"], train)
    else:
        dz1 = da1
    r["w1"] = gw.conv2d_weight(x, w1.shape, dz1, padding=1)
    r["dx"] = gw.conv2d_input(x.shape, w1, dz1, padding=1) + dx_sc
    return r


def bn_params(module, dtype=None, device=None):
    """The dict block_forward takes from an nn.BatchNorm2d (None for nn.Identity), with F.batch_norm's exponential-average
    factor for the module's next train-mode call."""
    if not isinstance(module, torch.nn.BatchNorm2d):
        return None
    cv = lambda t: t.detach().to(dtype=dtype or t.dtype, device=device or t.device).clone()
    nbt = int(module.num_batches_tracked) + 1
    return dict(weight=cv(module.weight), bias=cv(module.bias), running_mean=cv(module.running_mean),
                running_var=cv(module.running_var), eps=module.eps,
                factor=1.0 / nbt if module.momentum is None else module.momentum)
