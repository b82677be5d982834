"""Plain-torch restatement of the heads' output layers with a closed-form backward, and of a whole head in train or eval mode.

Output layers (x = rb4's output [B, C, h, w], W the 1x1 weight [k, C], r = W x, g the upstream gradient):
    score_softmax   remove_brd_and_softmax (mickey_extractor.py:98-124, 137-138): s = r - (mean r + eps) with the mean
                    detached, e = exp(s / T) mask, p = e / (sum e + eps);   dr = p (g - sum g p) / T
    score_sigmoid   remove_borders(sigmoid(r), 3) (:140);                    dr = g s (1 - s) mask, s = sigmoid(r)
    offset          sigmoid(r) (:173-176);                                   dr = g o (1 - o)
    depth           r, or MAX_DEPTH sigmoid(r) (:213-216);                   dr = g, or g MAX_DEPTH s (1 - s)
    desc            desc_l2norm (extractor_utils.py:6-10), y = x / n;        dx = (g - y (y . g)) / n
and for the convolution dx = dr^T W, dW = sum_{b, p} dr x^T.  mask zeroes 3 cells at each border.

head_chain restates a head's forward in train or eval mode: resblock1..3 (oracle/resblock_oracle.py), the transformer
(oracle/mickey_oracle.py head_transformer), resblock4 (relu=False for the descriptor head, :246) and the output layer, as
mickey_extractor.py:126-142 / 164-178 / 203-218 / 240-251 chain them.  Device- and dtype-agnostic: everything computes in
the dtype of its inputs.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import resblock_oracle as rbo
from oracle.mickey_oracle import head_transformer

BORDER = 3
KINDS = ("score_softmax", "score_sigmoid", "offset", "depth", "depth_sigmoid", "desc")


def border_mask(h, w, dtype=torch.float64, device=None):
    """remove_borders (mickey_extractor.py:98-110) as a [h, w] 0/1 mask."""
    m = torch.zeros(h, w, dtype=dtype, device=device)
    m[BORDER:h - BORDER, BORDER:w - BORDER] = 1
    return m


def conv1x1(x, W):
    return torch.einsum("kc,bchw->bkhw", W.reshape(W.shape[0], -1), x)


def output_forward(kind, x, W=None, eps=1e-16, temperature=100.0, max_depth=1.0):
    """The reference's output layer `kind` on x.  Returns (out, norm): norm is the descriptor's [B, 1, h, w] L2 norm,
    None for the other kinds."""
    if kind == "desc":
        n = x.pow(2).sum(dim=1, keepdim=True).add(1e-10).pow(0.5)
        return x / n, n
    r = conv1x1(x, W)
    B, _, h, w = r.shape
    mask = border_mask(h, w, r.dtype, r.device)
    if kind == "score_softmax":
        s = r - (r.reshape(B, -1).mean(-1).view(B, 1, 1, 1) + eps).detach()
        e = torch.exp(s / temperature) * mask
        return e / (e.sum((2, 3), keepdim=True) + eps), None
    if kind == "score_sigmoid":
        return torch.sigmoid(r) * mask, None
    if kind == "offset":
        return torch.sigmoid(r), None
    if kind == "depth":
        return r, None
    if kind == "depth_sigmoid":
        return max_depth * torch.sigmoid(r), None
    raise ValueError(kind)


def output_backward(kind, x, W, out, norm, g, temperature=100.0, max_depth=1.0):
    """Closed-form (dx, dW) of output_forward (dW None for the descriptor)."""
    if kind == "desc":
        return (g - out * (out * g).sum(1, keepdim=True)) / norm, None
    h, w = out.shape[2:]
    if kind == "score_softmax":
        dr = out * (g - (g * out).sum((2, 3), keepdim=True)) / temperature
    elif kind == "score_sigmoid":
        s = torch.sigmoid(conv1x1(x, W))
        dr = g * s * (1 - s) * border_mask(h, w, out.dtype, out.device)
    elif kind == "offset":
        dr = g * out * (1 - out)
    elif kind == "depth":
        dr = g
    else:
        s = out / max_depth
        dr = g * max_depth * s * (1 - s)
    Wm = W.reshape(W.shape[0], -1)
    dx = torch.einsum("bkhw,kc->bchw", dr, Wm)
    dW = torch.einsum("bkhw,bchw->kc", dr, x).reshape(W.shape)
    return dx, dW


def head_kind(head_name, config):
    """(output kind, name of the output convolution's weight in the head's state dict, final ReLU of rb4) for a head of
    MicKey_Extractor (det_head, det_offset, depth_head, dsc_head) under config = cfg['MICKEY']."""
    kp = config["KP_HEADS"]
    if head_name == "det_head":
        return ("score_softmax" if kp["USE_SOFTMAX"] else "score_sigmoid"), "score.weight", True
    if head_name == "det_offset":
        return "offset", "xy_offset.weight", True
    if head_name == "depth_head":
        return ("depth_sigmoid" if kp["USE_DEPTHSIGMOID"] else "depth"), "depth.weight", True
    return ("desc" if config["DSC_HEAD"]["NORM_DSC"] else None), None, False


def head_chain(sd, head_name, config, x, momentum=0.1, train=True):
    """A head's forward on feature_volume x from its state dict `sd` (tensors in the dtype and on the device to compute
    in; parameters may require grad).  Returns (out, running): in train mode running maps every BN running-statistics name
    to its value after the call, as F.batch_norm leaves it; with train=False batch norm uses the running statistics,
    nothing is updated and running is empty."""
    kind, wname, last_relu = head_kind(head_name, config)
    running = {}
    bn = config["KP_HEADS"]["BN"]
    for k in (1, 2, 3, 4):
        pre = f"resblock{k}."
        bns = []
        for j in (1, 2):
            if not bn:
                bns.append(None)
                continue
            b = f"{pre}bn{j}."
            nbt = int(sd[b + "num_batches_tracked"]) + 1
            bns.append(dict(weight=sd[b + "weight"], bias=sd[b + "bias"], running_mean=sd[b + "running_mean"],
                            running_var=sd[b + "running_var"], eps=1e-5, factor=momentum if momentum else 1.0 / nbt))
        wsc = sd.get(pre + "shortcut.0.weight")
        x, aux = rbo.block_forward(x, sd[pre + "conv1.weight"], sd[pre + "conv2.weight"], wsc, bns[0], bns[1], train=train,
                                   relu=last_relu or k < 4)
        for j, p in ((1, bns[0]), (2, bns[1])):
            if p is not None and train:
                m, v = aux[f"mean{j}"].detach(), aux[f"var{j}"].detach()
                count = x.numel() // x.shape[1]
                rm, rv = rbo.running_update(p, m, v, count)
                running[f"{pre}bn{j}.running_mean"], running[f"{pre}bn{j}.running_var"] = rm, rv
        if k == 3:
            x = head_transformer(sd, "att_layer.", x, _pos_enc(config, head_name))
    if kind is None:
        return x, running
    return output_forward(kind, x, sd.get(wname), eps=sd.get("eps", 1e-16),
                          max_depth=config["KP_HEADS"]["MAX_DEPTH"])[0], running


def _pos_enc(config, head_name):
    return config["DSC_HEAD" if head_name == "dsc_head" else "KP_HEADS"]["POS_ENCODING"]
