"""The dual-softmax backward on the CPU: the closed form against autograd, against the live reference's recorded
gradients, the drop-in module's names, argument rejection and the workspace sizes."""
import ctypes as C
import itertools
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

from mickey_b200 import _lib
from mickey_b200.dual_softmax import dual_softmax, dualSoftmax
from oracle import matcher_grad_oracle as mgo
from oracle import mickey_oracle as mo
from tests import matcher_grad_check as mgc
from tests.golden import make_matcher_grad_fixture as fixture

SUBSETS = [s for n in (1, 2, 3) for s in itertools.combinations("skf", n)]


@pytest.mark.parametrize("dust", [True, False])
@pytest.mark.parametrize("subset", SUBSETS, ids=lambda s: "".join(s))
def test_closed_form_equals_fp64_autograd(dust, subset):
    """mickey_oracle.dual_softmax + kp + final + log(final + 1e-16) under fp64 autograd, for every subset of upstream
    gradients (Gs on scores, Gk on kp_scores, probs_grad on log(final + 1e-16))."""
    B, N, T = 2, 37, 0.1
    g = torch.Generator().manual_seed(7)
    d0 = torch.randn(B, 128, N, generator=g, dtype=torch.float64) * 0.2
    d1 = torch.randn(B, 128, N, generator=g, dtype=torch.float64) * 0.2
    s0 = torch.rand(B, 1, N, generator=g, dtype=torch.float64)
    s1 = torch.rand(B, 1, N, generator=g, dtype=torch.float64)
    alpha = torch.tensor(0.7, dtype=torch.float64)
    Gs, Gk = torch.randn(B, N, N, generator=g, dtype=torch.float64), torch.randn(B, N, N, generator=g, dtype=torch.float64)
    PG = torch.randn(B, N, N, generator=g, dtype=torch.float64) * (torch.rand(B, N, N, generator=g) < 0.1)
    leaves = [t.clone().requires_grad_() for t in (d0, d1, s0, s1, alpha)]
    x0, x1, y0, y1, a = leaves
    scores = mo.dual_softmax(x0, x1, T, a if dust else None)
    kp = torch.matmul(y0.transpose(2, 1), y1)
    final = scores * kp
    outs, ups = [], []
    if "s" in subset:
        outs.append(scores); ups.append(Gs)
    if "k" in subset:
        outs.append(kp); ups.append(Gk)
    if "f" in subset:
        outs.append(torch.log(final + 1e-16)); ups.append(PG)
    torch.autograd.backward(outs, ups)
    fw = mgo.forward(d0, d1, T, alpha if dust else None, s0, s1)
    gf = PG / (fw["final"] + 1e-16) if "f" in subset else None
    bw = mgo.backward(fw, d0, d1, T, alpha if dust else None, s0, s1, Gs if "s" in subset else None,
                      Gk if "k" in subset else None, gf)
    for got, leaf in ((bw["ddsc0"], x0), (bw["ddsc1"], x1), (bw["dscr0"], y0), (bw["dscr1"], y1)):
        ref = leaf.grad if leaf.grad is not None else torch.zeros_like(leaf)
        torch.testing.assert_close(got.reshape(ref.shape), ref, rtol=1e-12, atol=1e-14)
    if dust:
        ref = a.grad if a.grad is not None else torch.zeros_like(a)
        torch.testing.assert_close(bw["ddustbin"], ref, rtol=1e-12, atol=1e-14)


@pytest.mark.parametrize("case", list(fixture.CASES))
def test_closed_form_reproduces_the_live_reference(case):
    """The fp64 closed form against the reference's own fp32 autograd (tests/golden/reference_matcher_grad_small.npz),
    within the fp32 bounds of tests/matcher_grad_check.py."""
    feat, loss, up, dust = fixture.CASES[case]
    d0, d1, s0, s1, pg = fixture.inputs(feat, loss)
    z = np.load(fixture.FIXTURE)
    B, N = d0.shape[0], d0.shape[2]
    T = fixture.TEMPERATURE
    db = torch.tensor(1.0) if dust else None
    fw = mgo.forward(d0.double(), d1.double(), T, None if db is None else db.double(), s0.double(), s1.double())
    if up == "reinforce":
        gs, gk, gf = None, None, (pg.double() / (fw["final"] + 1e-16)).float()
    else:
        gs, gk = fixture.dense_grads(B, N, fixture.seed_of(case))
        gf = None
    fw, bw = mgc.reference(d0, d1, T, db, s0, s1, gs, gk, gf)
    bnd = mgc.bounds(d0, d1, T, db, s0, s1, gs, gk, gf, fw, bw)
    for k in ("ddsc0", "ddsc1", "dscr0", "dscr1"):
        mgc.check(f"{case}/{k}", torch.from_numpy(z[f"{case}/{k}"]), bw[k].reshape(z[f"{case}/{k}"].shape),
                  bnd[k].reshape(z[f"{case}/{k}"].shape))
    if dust:
        mgc.check(f"{case}/ddustbin", torch.tensor(float(z[f"{case}/ddustbin"])), bw["ddustbin"], bnd["ddustbin"])


@pytest.mark.parametrize("N,dust,T", [(129, True, 1.0), (257, False, 0.1), (850, True, 1.0), (850, True, 0.1)])
def test_bounds_hold_for_fp32_arithmetic_and_reject_the_mutations(N, dust, T):
    """The closed form evaluated in fp32 (torch, CPU) stays inside the bounds, and every planted mutation leaves them.
    The dustbin's share of a row is ~e / (1.5 N) at T = 0.1 and unit descriptors, below what the worst-case bound of the
    forward's split-operand logits can resolve; at T = 1 it is rejected."""
    args = mgc.case_inputs(2, N, T, dust, "skf", seed=N)
    d0, d1, T, db, s0, s1, gs, gk, gf = args
    fw, bw = mgc.reference(*args)
    bnd = mgc.bounds(*args, fw, bw)
    fw32 = mgo.forward(d0, d1, T, db, s0, s1)
    bw32 = mgo.backward(fw32, d0, d1, T, db, s0, s1, gs, gk, gf)
    for k in ("ddsc0", "ddsc1", "dscr0", "dscr1"):
        mgc.check(k, bw32[k], bw[k], bnd[k])
    if dust:
        mgc.check("ddustbin", bw32["ddustbin"], bw["ddustbin"], bnd["ddustbin"])
    muts = mgc.mutations(*args, fw)
    assert len(muts) == (5 if dust else 4)
    for name, out, mutated in muts:
        if "dustbin" in name and T != 1.0:
            continue
        assert mgc.rejected(bw[out], mutated, bnd[out]), name


def test_dualSoftmax_module_matches_the_reference_names():
    """Same attributes and parameter as feature_matcher.py's dualSoftmax; the released state-dict key loads."""
    m = dualSoftmax({"TEMPERATURE": 0.1, "USE_DUSTBIN": True})
    assert m.temperature == 0.1 and m.use_dustbin is True
    assert [n for n, _ in m.named_parameters()] == ["dustbin_score"]
    assert m.dustbin_score.shape == () and float(m.dustbin_score.detach()) == 1.0 and m.dustbin_score.requires_grad
    off = dualSoftmax({"TEMPERATURE": 0.1, "USE_DUSTBIN": False})
    assert off.use_dustbin is False and list(off.parameters()) == []
    root = nn.Module()
    root.compute_matches = nn.Module()
    root.compute_matches.matcher = nn.Module()
    root.compute_matches.matcher.matching_mat = m
    assert list(root.state_dict()) == [mo.DUSTBIN]
    root.load_state_dict({mo.DUSTBIN: torch.tensor(0.25)})
    assert float(m.dustbin_score.detach()) == 0.25


def test_python_arguments_are_rejected_before_any_launch():
    d = torch.zeros(1, 128, 8)
    with pytest.raises(ValueError, match="128"):
        dual_softmax(torch.zeros(1, 64, 8), d, None, 0.1)
    with pytest.raises(ValueError, match="float32"):
        dual_softmax(d.double(), d.double(), None, 0.1)
    with pytest.raises(ValueError, match="CUDA"):
        dual_softmax(d, d, None, 0.1)


def test_c_arguments_are_rejected_before_any_launch():
    lib = _lib.load()
    p = C.c_void_p(256)                     # never dereferenced: every call below fails its argument check first
    ws = lib.mk_dual_softmax_ws_bytes(2, 100)
    bws = lib.mk_dual_softmax_backward_ws_bytes(2, 100)

    def fwd(B=2, N=100, T=0.1, scr=(p, p), outs=(p, p, p), pitch=0, wsb=ws):
        return lib.mk_dual_softmax(p, p, scr[0], scr[1], None, T, B, N, 1, *outs, pitch, p, p, p, wsb, None)

    def bwd(B=2, N=100, T=0.1, scr=(p, p), g=(p, None, p), pitches=(0, 0, 0), dscr=(p, p), dd=p, dust=None, wsb=bws):
        return lib.mk_dual_softmax_backward(p, p, scr[0], scr[1], dust, T, B, N, p, p, g[0], pitches[0], g[1], pitches[1],
                                            g[2], pitches[2], p, p, dscr[0], dscr[1], dd, p, wsb, None)

    for rc in (fwd(B=0), fwd(N=1), fwd(N=8193), fwd(T=0.0), fwd(T=float("nan")), fwd(scr=(p, None)),
               fwd(outs=(None, None, None)), fwd(outs=(p, p, None)), fwd(outs=(p, p, p), scr=(None, None)),
               fwd(pitch=99), fwd(wsb=ws - 1),
               bwd(B=0), bwd(N=1), bwd(T=-1.0), bwd(g=(None, None, None)), bwd(scr=(None, None), g=(None, p, None)),
               bwd(dscr=(None, p)), bwd(dust=p, dd=None), bwd(pitches=(99, 0, 0)), bwd(wsb=bws - 1)):
        assert rc == -1
    assert lib.mk_dual_softmax_ws_bytes(0, 100) == 0 and lib.mk_dual_softmax_backward_ws_bytes(1, 8193) == 0


@pytest.mark.parametrize("B,N", [(1, 2), (3, 129), (8, 1938), (24, 850), (1, 4176)])
def test_workspaces_hold_no_NxN_intermediate(B, N):
    """Forward: the split operands and the forward's own (max, sum) slots; backward: (W, dsig) slots per 64-wide tile,
    i.e. 16 B * N^2 / 64 per pair, plus O(N) vectors.  Neither is as large as one fp32 N x N matrix."""
    lib = _lib.load()
    nt = -(-N // 64)
    np_ = nt * 64
    npad = -(-N // 128) * 128
    slots_b = B * (2 * nt * np_ * 8 + 4 * np_ * 4)
    assert lib.mk_dual_softmax_backward_ws_bytes(B, N) <= slots_b + 5 * 256
    slots_f = B * (2 * N * 384 * 2 + 2 * N * 4 + (npad // 64 + npad // 32) * npad * 8)
    assert lib.mk_dual_softmax_ws_bytes(B, N) <= slots_f + 4 * 256
    if N >= 850:
        assert lib.mk_dual_softmax_backward_ws_bytes(B, N) < B * N * N * 4 // 2
