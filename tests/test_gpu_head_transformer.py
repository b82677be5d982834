"""The heads' transformer on the GPU (mickey_b200.head_transformer, csrc/head_transformer.cu): every output and gradient
element by element against the fp64 restatement of tests/head_transformer_check.py, determinism, batch invariance and
autograd behaviour."""
import pytest
import torch

from mickey_b200.head_transformer import Transformer_self_att
from tests import head_transformer_check as hc
from tests.elementwise import record

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _module(num_layers, pe_on, params):
    m = Transformer_self_att(128, num_layers, pe_on).to(DEV)
    with torch.no_grad():
        for p, v in zip([p for l in m.layers for p in l.params()], params):
            p.copy_(v)
    return m


def _run(m, x, go, need_x=True, need_w=True):
    for p in m.parameters():
        p.grad = None
        p.requires_grad_(need_w)
    xx = x.clone().requires_grad_(need_x)
    out = m(xx)
    out.backward(go)
    return out, xx.grad, [p.grad for l in m.layers for p in l.params()]


SHAPES = [  # B, h, w, layers, pe
    (8, 38, 51, 3, True),         # curriculum_learning: 720x540 -> 51 x 38
    (24, 25, 34, 3, False),       # warm-up: 476x350 -> 34 x 25
    (2, 7, 7, 3, True),
    (3, 1, 1, 1, False),          # N = 1
    (2, 1, 2, 3, True),           # N = 2
    (2, 9, 7, 1, True),           # N = 63
    (2, 8, 8, 3, False),          # N = 64
    (2, 5, 13, 1, False),         # N = 65
    (1, 127, 1, 3, True),         # N = 127
    (2, 16, 8, 1, False),         # N = 128
    (2, 3, 43, 3, False),         # N = 129
    (1, 58, 72, 3, True),         # N = 4176
    (2, 256, 1, 1, True),
    (2, 1, 256, 3, True),
]


@pytest.mark.parametrize("B,h,w,L,pe_on", SHAPES)
def test_against_fp64(B, h, w, L, pe_on):
    x, params, go = hc.case_inputs(B, h, w, L, seed=B * 1000 + h * 7 + w, device=DEV)
    m = _module(L, pe_on, params)
    out, dx, grads = _run(m, x, go)
    ref = hc.restate(x, params, m.posEnc.pe if pe_on else None, go)
    geometry = f"B{B}_{h}x{w}_L{L}_{'pe' if pe_on else 'nope'}"
    record("head_transformer.out", geometry, hc.check("out", out, *ref["out"]))
    record("head_transformer.dx", geometry, hc.check("dx", dx, *ref["dx"]))
    for i, g in enumerate(grads):
        record(f"head_transformer.{hc.param_key(i)}", geometry, hc.check(hc.param_key(i), g, *ref[hc.param_key(i)]))
    for mut in hc.MUTATIONS:
        # not observable: no PE, the next position outside the 256-wide table, one image, or one token (with N = 1,
        # msg = v (phi(q).phi(k)) / (phi(q).phi(k) + eps) does not depend on q or k, so elu' carries no gradient)
        if (mut == "pe_next" and (not pe_on or w == 256) or mut == "kv_neighbour" and B < 2
                or mut in ("out_chunk", "elu_one") and h * w < 2):
            continue
        assert hc.rejected(ref, hc.restate(x, params, m.posEnc.pe if pe_on else None, go, mutation=mut)), mut


@pytest.mark.parametrize("need_x,need_w", [(True, False), (False, True), (True, True)])
def test_gradient_subsets(need_x, need_w):
    B, h, w, L = 2, 9, 11, 3
    x, params, go = hc.case_inputs(B, h, w, L, seed=7, device=DEV)
    m = _module(L, True, params)
    out, dx, grads = _run(m, x, go, need_x, need_w)
    ref = hc.restate(x, params, m.posEnc.pe, go)
    hc.check("out", out, *ref["out"])
    assert (dx is not None) == need_x
    if need_x:
        hc.check("dx", dx, *ref["dx"])
    for i, g in enumerate(grads):
        assert (g is not None) == need_w
        if need_w:
            hc.check(hc.param_key(i), g, *ref[hc.param_key(i)])
    _, dx_all, grads_all = _run(m, x, go, True, True)
    if need_x:
        assert torch.equal(dx, dx_all)
    if need_w:
        assert all(torch.equal(a, b) for a, b in zip(grads, grads_all))


def test_frozen_parameter_gets_no_gradient():
    x, params, go = hc.case_inputs(2, 6, 5, 3, seed=3, device=DEV)
    m = _module(3, False, params)
    m.layers[1].mlp[0].weight.requires_grad_(False)
    xx = x.clone().requires_grad_()
    m(xx).backward(go)
    assert m.layers[1].mlp[0].weight.grad is None
    assert m.layers[0].q_proj.weight.grad is not None and xx.grad is not None


def test_deterministic_and_batch_invariant():
    B, h, w, L = 4, 13, 11, 3
    x, params, go = hc.case_inputs(B, h, w, L, seed=11, device=DEV)
    m = _module(L, True, params)
    o1, d1, g1 = _run(m, x, go)
    o2, d2, g2 = _run(m, x, go)
    assert torch.equal(o1, o2) and torch.equal(d1, d2) and all(torch.equal(a, b) for a, b in zip(g1, g2))
    for b in range(B):
        ob, db, _ = _run(m, x[b:b + 1], go[b:b + 1])
        assert torch.equal(ob, o1[b:b + 1]), b
        assert torch.equal(db, d1[b:b + 1]), b


def test_autograd_accumulates_strided_and_no_grad():
    B, h, w, L = 2, 10, 12, 3
    x, params, go = hc.case_inputs(B, h, w, L, seed=5, device=DEV)
    m = _module(L, True, params)
    _, _, g1 = _run(m, x, go)
    g1 = [g.clone() for g in g1]
    m(x).backward(go)             # accumulates into .grad
    for p, g in zip([p for l in m.layers for p in l.params()], g1):
        assert torch.equal(p.grad, g + g)
    # strided input (channels-last) gives the bits of its contiguous copy
    xs = x.to(memory_format=torch.channels_last)
    assert not xs.is_contiguous()
    with torch.no_grad():
        ref = m(x)
        assert torch.equal(m(xs), ref)
    out = m(x.clone().requires_grad_())
    assert torch.equal(out.detach(), ref) and out.is_contiguous() and out.dtype == torch.float32


def test_head_chain_conv_gradients():
    """conv -> Transformer_self_att -> conv, built from torch.nn layers and backpropagated in fp32 on the GPU; the same
    chain runs in fp64 on the CPU through the restatement.  Both convolutions' weight gradients must agree within the
    transformer's bounds pushed through them plus the convolutions' own roundings.  cuDNN is off so that the convolutions
    are plain im2col GEMMs in fp32 (no TF32, no Winograd), whose rounding is K u sum |a b| like every other contraction."""
    B, h, w, L = 2, 12, 10, 3
    x, params, _ = hc.case_inputs(B, h, w, L, seed=21, device=DEV)
    g = torch.Generator().manual_seed(22)
    c1 = torch.nn.Conv2d(128, 128, 3, padding=1, bias=False)
    c2 = torch.nn.Conv2d(128, 16, 3, padding=1, bias=False)
    gy = torch.randn(B, 16, h, w, generator=g)
    m = _module(L, True, params)
    cudnn = torch.backends.cudnn.enabled
    torch.backends.cudnn.enabled = False
    try:
        g1, g2 = c1.to(DEV), c2.to(DEV)
        g2(m(g1(x))).backward(gy.to(DEV))
        gw1, gw2 = g1.weight.grad.double().cpu(), g2.weight.grad.double().cpu()
    finally:
        torch.backends.cudnn.enabled = cudnn
    # fp64 chain
    W1, W2 = c1.weight.detach().double().cpu(), c2.weight.detach().double().cpu()
    x64, gy64 = x.double().cpu(), gy.double()
    conv = torch.nn.functional.conv2d
    t64 = conv(x64, W1, padding=1)
    e_t = (9 * 128 + 2) * hc.U * conv(x64.abs(), W1.abs(), padding=1)               # conv1's fp32 rounding
    go64 = torch.nn.grad.conv2d_input(t64.shape, W2, gy64, padding=1)                # the gradient conv2 passes back
    e_go = (9 * 16 + 2) * hc.U * torch.nn.grad.conv2d_input(t64.shape, W2.abs(), gy64.abs(), padding=1)
    ref = hc.restate(t64, params, m.posEnc.pe, go64, x_err=e_t, grad_err=e_go)
    out, e_out = ref["out"]
    dx, e_dx = ref["dx"]
    n = 9 * B * h * w + 2
    cw = torch.nn.grad.conv2d_weight
    want2 = cw(out, W2.shape, gy64, padding=1)
    bound2 = cw(e_out, W2.shape, gy64.abs(), padding=1) + n * hc.U * cw(out.abs(), W2.shape, gy64.abs(), padding=1)
    want1 = cw(x64, W1.shape, dx, padding=1)
    bound1 = cw(x64.abs(), W1.shape, e_dx, padding=1) + n * hc.U * cw(x64.abs(), W1.shape, dx.abs(), padding=1)
    for name, got, want, bound in (("conv2.weight", gw2, want2, bound2), ("conv1.weight", gw1, want1, bound1)):
        err = (got - want).abs()
        assert bool((err <= bound).all()), (name, float((err / bound).max()))
        record(f"head_chain.{name}", "B2_12x10_L3_pe", float((err / bound).max()))
