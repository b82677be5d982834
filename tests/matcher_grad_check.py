"""Element-wise bounds for the dual-softmax matcher's backward (csrc/matcher_grad.cu) against the fp64 closed form
(oracle/matcher_grad_oracle.py), and the planted mutations each bound must reject.

Notation as in DESIGN.md §6e; u = 2^-24; x = s log2(e) (log2-domain logits); k2 = log2(e) / T; A_ij = sum_c |d0_ic d1_jc|.
Every bound is written over sums of |terms|: dS_ij = 2 w_ij - P_ij W_i - Q_ij W'_j cancels by construction (softmax
gradients sum to zero along the normalised axis), so |dS| itself says nothing about the size of its rounding errors.

* logits in the backward (fp32 FMA over 128 channels):        e_x = k2 (C + 2) u A + u |x|
* the forward's log-sum-exps (hi + lo fp16 operands, 384 tensor-core products, ex2.approx, n-term fp32 sums, log2f):
      e_fwd = k2 (400 2^-23 A + 2^-24 (|d0_i|_1 + |d1_j|_1)),  e_lr_i = max_j e_fwd + 1.5 (N + 2) u + 2^-21 + 2 u |lr_i|
* P = exp2(x - lr), Q = exp2(x - lc) (exp2f: 2 ulp):           rho_P = ln2 (e_x + e_lr) + 2^-21 + 2u, rho_Q alike
  scores = P Q:                                                 rho_sc = rho_P + rho_Q + u
* w = (Gs + Gf kp) scores:                                      e_w = (|Gs| + |Gf| kp) scores (rho_sc + 5u)
* W_i, W'_j (n-term sums):                                      e_W = sum e_w + N u sum |w|
* dS:  e_dS = 2 e_w + P (rho_P |W| + e_W) + Q (rho_Q |W'| + e_W') + 3u (2|w| + P |W| + Q |W'|)
  plus 4 t (t = 2^-149, fp32's subnormal spacing: wide logits push P W and Q W' below the normal range)
* dd0_ic = (1/T) sum_j dS_ij d1_jc:  (1/T) [sum_j e_dS |d1_jc| + N u sum_j (|dS| + e_dS) |d1_jc| + N t] + 2u |dd0| + t;
  dd1 alike
* h = Gk + Gf scores:                 e_h = |Gf| scores (rho_sc + 2u) + u (|Gk| + |Gf| scores)
  dsig0_i = sum_j h_ij sig1_j:        sum_j e_h sig1_j + (N + 1) u sum_j |h sig1|
* dalpha, terms t = e^(alpha - r) W:  sum |t| (ln2 (e_l + u |alpha log2 e|) + 2^-21 + 3u) + e^(alpha - r) e_W, plus
                                      (2 N + 1) B u sum |t| for the sums, and t (|W| + 2) per term for underflow
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Callable, Dict, Optional

import torch

from oracle import matcher_grad_oracle as mgo

U = 2.0 ** -24
TINY = 2.0 ** -149                 # fp32's subnormal spacing: the absolute error of an operation whose result underflows
LN2 = math.log(2.0)
LOG2E = 1.0 / LN2
TILE = 64                          # keypoints per tile of the backward kernels


def reference(d0, d1, T, dust, s0, s1, gs, gk, gf):
    """fp64 forward + backward of the closed form on the given (fp32) inputs."""
    f = lambda t: None if t is None else t.double()
    fw = mgo.forward(f(d0), f(d1), T, f(dust), f(s0), f(s1))
    bw = mgo.backward(fw, f(d0), f(d1), T, f(dust), f(s0), f(s1), f(gs), f(gk), f(gf))
    return fw, bw


def bounds(d0, d1, T, dust, s0, s1, gs, gk, gf, fw, bw) -> Dict[str, torch.Tensor]:
    """Bound of every output of the fp32 backward (see the module docstring)."""
    d0, d1 = d0.double(), d1.double()
    B, C, N = d0.shape
    k2 = LOG2E / T
    a0, a1 = d0.abs(), d1.abs()
    A = torch.matmul(a0.transpose(1, 2), a1)
    x = fw["s"] * LOG2E
    lr, lc = fw["r"] * LOG2E, fw["c"] * LOG2E
    e_x = k2 * (C + 2) * U * A + U * x.abs()
    e_fwd = k2 * (400 * 2.0 ** -23 * A + 2.0 ** -24 * (a0.sum(1)[:, :, None] + a1.sum(1)[:, None, :]))
    e_lr = e_fwd.amax(2) + 1.5 * (N + 2) * U + 2.0 ** -21 + 2 * U * lr.abs()
    e_lc = e_fwd.amax(1) + 1.5 * (N + 2) * U + 2.0 ** -21 + 2 * U * lc.abs()
    P, Q, sc = fw["P"], fw["Q"], fw["scores"]
    rhoP = LN2 * (e_x + e_lr[:, :, None]) + 2.0 ** -21 + 2 * U
    rhoQ = LN2 * (e_x + e_lc[:, None, :]) + 2.0 ** -21 + 2 * U
    rho_sc = rhoP + rhoQ + U
    kp = fw["kp"] if fw["kp"] is not None else torch.ones_like(sc)
    z = torch.zeros_like(sc)
    gs_a = gs.double().abs() if gs is not None else z
    gk_a = gk.double().abs() if gk is not None else z
    gf_a = gf.double().abs() if gf is not None else z
    e_w = (gs_a + gf_a * kp) * sc * (rho_sc + 5 * U)
    wa = bw["w"].abs()
    W, Wc = bw["W"], bw["Wc"]
    e_W = e_w.sum(2) + N * U * wa.sum(2)
    e_Wc = e_w.sum(1) + N * U * wa.sum(1)
    e_dS = (2 * e_w + P * (rhoP * W.abs()[:, :, None] + e_W[:, :, None]) + Q * (rhoQ * Wc.abs()[:, None, :] + e_Wc[:, None, :])
            + 3 * U * (2 * wa + P * W.abs()[:, :, None] + Q * Wc.abs()[:, None, :]))
    e_dS = e_dS + 4 * TINY                              # each of the cell's operations may land in fp32's subnormal range
    dSa = bw["dS"].abs() + e_dS
    out = {
        "ddsc0": (torch.matmul(a1, e_dS.transpose(1, 2)) + N * U * torch.matmul(a1, dSa.transpose(1, 2)) + N * TINY) / T
                 + 2 * U * bw["ddsc0"].abs() + TINY,
        "ddsc1": (torch.matmul(a0, e_dS) + N * U * torch.matmul(a0, dSa) + N * TINY) / T + 2 * U * bw["ddsc1"].abs() + TINY,
    }
    if s0 is not None:
        s0a, s1a = s0.double().abs().reshape(B, N), s1.double().abs().reshape(B, N)
        ha = gk_a + gf_a * sc
        e_h = gf_a * sc * (rho_sc + 2 * U) + U * ha
        out["dscr0"] = (e_h * s1a[:, None, :]).sum(2) + (N + 1) * U * (ha * s1a[:, None, :]).sum(2)
        out["dscr1"] = (e_h * s0a[:, :, None]).sum(1) + (N + 1) * U * (ha * s0a[:, :, None]).sum(1)
    if dust is not None:
        al = float(dust.reshape(()))
        er = torch.exp(al - fw["r"])
        ec = torch.exp(al - fw["c"])
        ta, tc = (er * W).abs(), (ec * Wc).abs()
        ua = U * abs(al * LOG2E)
        b = ((ta * (LN2 * (e_lr + ua) + 2.0 ** -21 + 3 * U) + er * e_W).sum()
             + (tc * (LN2 * (e_lc + ua) + 2.0 ** -21 + 3 * U) + ec * e_Wc).sum()
             + (2 * N + 1) * B * U * (ta.sum() + tc.sum())
             + TINY * ((W.abs() + 2).sum() + (Wc.abs() + 2).sum()))      # e^(alpha - r) and the product may underflow
        out["ddustbin"] = b.reshape(())
    return out


def check(name: str, got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> float:
    """|got - ref| <= bound for every element; returns max(err / bound).  On failure, names the worst element as
    (pair, channel, keypoint, tile) for ddsc [B, 128, N], (pair, keypoint, tile) for dscr [B, N]."""
    got = got.detach().double().reshape(ref.shape)
    err = (got - ref).abs()
    bad = ~(err <= bound)
    ratio = float((err / bound.clamp_min(1e-300)).max()) if ref.numel() else 0.0
    if bool(bad.any()):
        r = torch.where(bad, err / bound.clamp_min(1e-300), torch.zeros_like(err))
        idx = [int(v) for v in torch.unravel_index(r.argmax(), r.shape)] if ref.dim() else []
        axis = "column" if name.endswith("1") else "row"
        if ref.dim() == 3:
            where = f"pair {idx[0]}, channel {idx[1]}, {axis} {idx[2]} (tile {idx[2] // TILE})"
        elif ref.dim() == 2:
            where = f"pair {idx[0]}, {axis} {idx[1]} (tile {idx[1] // TILE})"
        else:
            where = "scalar"
        raise AssertionError(f"{name}: {int(bad.sum())} of {ref.numel()} elements out of bounds; worst at {where}: got "
                             f"{float(got[tuple(idx)]):.9e}, fp64 {float(ref[tuple(idx)]):.9e}, bound "
                             f"{float(bound[tuple(idx)]):.3e}")
    return ratio


@dataclass
class Mutation:
    name: str
    output: str
    make: Callable[..., torch.Tensor]


def _rebackward(fw, d0, d1, T, dust, s0, s1, gs, gk, gf, dS_fn=None, Wc_fn=None):
    """ddsc0 / ddsc1 / dscr0 of the closed form with one intermediate replaced."""
    f = lambda t: None if t is None else t.double()
    bw = mgo.backward(fw, f(d0), f(d1), T, f(dust), f(s0), f(s1), f(gs), f(gk), f(gf))
    w, P, Q, W, Wc = bw["w"], fw["P"], fw["Q"], bw["W"], bw["Wc"]
    if Wc_fn is not None:
        Wc = Wc_fn(Wc)
    dS = dS_fn(w, P, Q, W, Wc) if dS_fn is not None else 2 * w - P * W[:, :, None] - Q * Wc[:, None, :]
    return torch.matmul(f(d1), dS.transpose(1, 2)) / T


def mutations(d0, d1, T, dust, s0, s1, gs, gk, gf, fw):
    """The bugs each bound must reject, as (name, output, mutated fp64 output)."""
    args = (d0, d1, T, dust, s0, s1, gs, gk, gf)
    B, _, N = d0.shape
    out = []
    # the contraction loop stops one tile early (the last, possibly partial, tile of j is never read)
    bw = mgo.backward(fw, *[None if t is None or isinstance(t, float) else t.double() for t in (d0, d1)], T,
                      *[None if t is None else t.double() for t in (dust, s0, s1, gs, gk, gf)])
    last = ((N - 1) // TILE) * TILE
    dS = bw["dS"].clone()
    dS[:, :, last:] = 0
    out.append(("last tile of the contraction dropped", "ddsc0", torch.matmul(d1.double(), dS.transpose(1, 2)) / T))
    # W' of the neighbouring column
    out.append(("W' of the neighbouring column", "ddsc0",
                _rebackward(fw, *args, Wc_fn=lambda Wc: torch.roll(Wc, -1, 1))))
    # the factor 2 on w dropped
    out.append(("factor 2 on w dropped", "ddsc0",
                _rebackward(fw, *args, dS_fn=lambda w, P, Q, W, Wc: w - P * W[:, :, None] - Q * Wc[:, None, :])))
    # Gf one row off (the row pitch taken as one row too many)
    if gf is not None:
        gsh = torch.zeros_like(gf)
        gsh[:, :-1] = gf[:, 1:]
        f = lambda t: None if t is None else t.double()
        m = mgo.backward(fw, f(d0), f(d1), T, f(dust), f(s0), f(s1), f(gs), f(gk), f(gsh))
        out.append(("Gf read one row off", "ddsc0", m["ddsc0"]))
    # the dustbin left out of one row's normaliser: the row where the dustbin's share times the row's |w| is largest
    if dust is not None:
        i = int((torch.exp(float(dust.reshape(())) - fw["r"][0]) * bw["w"][0].abs().sum(1)).argmax())
        fw2 = dict(fw)
        r = fw["r"].clone()
        r[:, i] = torch.logsumexp(fw["s"][:, i, :], 1)
        fw2["r"] = r
        fw2["P"] = torch.exp(fw["s"] - r[:, :, None])
        fw2["scores"] = fw2["P"] * fw["Q"]
        if fw["kp"] is not None:
            fw2["final"] = fw2["scores"] * fw["kp"]
        f = lambda t: None if t is None else t.double()
        m = mgo.backward(fw2, f(d0), f(d1), T, f(dust), f(s0), f(s1), f(gs), f(gk), f(gf))
        out.append(("dustbin left out of one row's normaliser", "ddsc0", m["ddsc0"]))
    return out


def rejected(ref: torch.Tensor, mutated: torch.Tensor, bound: torch.Tensor) -> bool:
    return bool(((mutated - ref).abs() > bound).any())


def case_inputs(B, N, T, dust_on, grads, scr=True, scale=None, pitch=None, seed=0, device="cpu"):
    """Seeded inputs: unit descriptors (or `scale` times Gaussian ones, with one dominant row and column), keypoint scores
    in (0, 1), a REINFORCE-shaped Gf (nonzero at 0.5 % of the cells, divided by final + 1e-16 as in the training step),
    dense Gs and Gk.  grads: a subset of "s", "k", "f".  With `pitch`, the gradients are [B, N, pitch][:, :, :N] views."""
    g = torch.Generator().manual_seed(seed)
    if scale is None:
        d0 = torch.nn.functional.normalize(torch.randn(B, 128, N, generator=g), dim=1)
        d1 = torch.nn.functional.normalize(torch.randn(B, 128, N, generator=g), dim=1)
    else:
        d0 = torch.randn(B, 128, N, generator=g) * scale
        d1 = torch.randn(B, 128, N, generator=g) * scale
        d0[0, :, min(7, N - 1)] *= 3.0
        d1[-1, :, min(9, N - 1)] *= 3.0
    s0 = torch.rand(B, N, generator=g) if scr else None
    s1 = torch.rand(B, N, generator=g) if scr else None
    dust = torch.tensor([1.0]) if dust_on else None

    def mat(fill):
        P = pitch or N
        t = torch.zeros(B, N, P)
        t[:, :, :N] = fill
        if P > N:
            t[:, :, N:] = float("nan")                    # padding must never be read
        return t[:, :, :N].to(device)

    gs = mat(torch.randn(B, N, N, generator=g)) if "s" in grads else None
    gk = mat(torch.randn(B, N, N, generator=g)) if "k" in grads and scr else None
    gf = None
    if "f" in grads:
        pg = torch.randn(B, N, N, generator=g) * (torch.rand(B, N, N, generator=g) < 0.005)
        fw = mgo.forward(d0.double(), d1.double(), T, None if dust is None else dust.double(),
                         None if s0 is None else s0.double(), None if s1 is None else s1.double())
        fin = fw["final"] if fw["final"] is not None else fw["scores"]
        gf = mat((pg.double() / (fin + 1e-16)).float())
    to = lambda t: None if t is None else t.to(device)
    return to(d0), to(d1), T, to(dust), to(s0), to(s1), gs, gk, gf
