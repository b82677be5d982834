"""The dual-softmax matcher's backward in closed form (DESIGN.md §6e), in the dtype of its inputs.

Per pair, for i, j < N: s_ij = <d0_i, d1_j> / T; with the dustbin, s_iN = s_Nj = s_NN = alpha.  r_i / c_j are the
log-sum-exps of row i / column j over the augmented matrix, P = exp(s - r) (softmax(., 2)), Q = exp(s - c)
(softmax(., 1)), scores = P Q, kp_ij = sig0_i sig1_j, final = scores kp.  For upstream gradients Gs, Gk, Gf (any may be
None):
    w_ij = (Gs_ij + Gf_ij kp_ij) scores_ij,  h_ij = Gk_ij + Gf_ij scores_ij
    W_i = sum_j w_ij,  W'_j = sum_i w_ij,  dS_ij = 2 w_ij - P_ij W_i - Q_ij W'_j
    dd0_i = (1/T) sum_j dS_ij d1_j,  dd1_j = (1/T) sum_i dS_ij d0_i
    dsig0_i = sum_j h_ij sig1_j,  dsig1_j = sum_i h_ij sig0_i
    dalpha = -sum_pairs [ sum_i e^(alpha - r_i) W_i + sum_j e^(alpha - c_j) W'_j ]
This equals autograd of mickey_oracle.dual_softmax + kp_matrix_scores + the product (tests/test_matcher_grad_host.py).
"""
from __future__ import annotations

from typing import Optional

import torch
from torch import Tensor


def forward(dsc0: Tensor, dsc1: Tensor, temperature: float, dustbin: Optional[Tensor] = None,
            scr0: Optional[Tensor] = None, scr1: Optional[Tensor] = None) -> dict:
    """dsc [B, C, N], scr [B, N] or [B, 1, N].  Returns s, r, c, P, Q, scores, kp, final (kp / final None without scr)."""
    s = torch.matmul(dsc0.transpose(1, 2), dsc1) / temperature
    if dustbin is None:
        r = torch.logsumexp(s, 2)
        c = torch.logsumexp(s, 1)
    else:
        a = dustbin.reshape(()).to(s.dtype)
        B, N, _ = s.shape
        ab = a.expand(B, N, 1)
        r = torch.logsumexp(torch.cat([s, ab], 2), 2)
        c = torch.logsumexp(torch.cat([s, ab.transpose(1, 2)], 1), 1)
    P = torch.exp(s - r[:, :, None])
    Q = torch.exp(s - c[:, None, :])
    scores = P * Q
    out = dict(s=s, r=r, c=c, P=P, Q=Q, scores=scores, kp=None, final=None)
    if scr0 is not None:
        B, N = s.shape[0], s.shape[1]
        kp = scr0.reshape(B, N, 1) * scr1.reshape(B, 1, N)
        out.update(kp=kp, final=scores * kp)
    return out


def backward(fw: dict, dsc0: Tensor, dsc1: Tensor, temperature: float, dustbin: Optional[Tensor] = None,
             scr0: Optional[Tensor] = None, scr1: Optional[Tensor] = None, grad_scores: Optional[Tensor] = None,
             grad_kp: Optional[Tensor] = None, grad_final: Optional[Tensor] = None) -> dict:
    """The closed form above on the forward's intermediates `fw`.  Returns ddsc0, ddsc1 [B, C, N], dscr0, dscr1 [B, N]
    (None without scr), ddustbin (a 0-dim tensor, None without the dustbin) and the intermediates w, h, W, Wc, dS."""
    B, N = fw["s"].shape[0], fw["s"].shape[1]
    sc, P, Q = fw["scores"], fw["P"], fw["Q"]
    zero = torch.zeros_like(sc)
    kp = fw["kp"] if fw["kp"] is not None else torch.ones_like(sc)
    gs = grad_scores if grad_scores is not None else zero
    gk = grad_kp if grad_kp is not None else zero
    gf = grad_final if grad_final is not None else zero
    w = (gs + gf * kp) * sc
    h = gk + gf * sc
    W = w.sum(2)
    Wc = w.sum(1)
    dS = 2 * w - P * W[:, :, None] - Q * Wc[:, None, :]
    ddsc0 = torch.matmul(dsc1, dS.transpose(1, 2)) / temperature           # [B, C, N0]
    ddsc1 = torch.matmul(dsc0, dS) / temperature                           # [B, C, N1]
    out = dict(ddsc0=ddsc0, ddsc1=ddsc1, dscr0=None, dscr1=None, ddustbin=None, w=w, h=h, W=W, Wc=Wc, dS=dS)
    if scr0 is not None:
        out["dscr0"] = (h * scr1.reshape(B, 1, N)).sum(2)
        out["dscr1"] = (h * scr0.reshape(B, N, 1)).sum(1)
    if dustbin is not None:
        a = dustbin.reshape(()).to(sc.dtype)
        out["ddustbin"] = -((torch.exp(a - fw["r"]) * W).sum() + (torch.exp(a - fw["c"]) * Wc).sum())
    return out
