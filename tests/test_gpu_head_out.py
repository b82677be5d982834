"""The heads' output layers on the GPU (mickey_b200.heads.head_out, csrc/head_out.cu).

- Every kind at the training shapes, one interior cell, no interior cell, single rows and columns and a map above 4096
  cells: the output, dx and dW element by element against the fp64 oracle (oracle/heads_oracle.py).  The bound charges
  each element the fp32 rounding of the terms that form it: 2^-16 of the quantity's largest magnitude plus 2^-20 of
  itself.  Where no cell is interior the score layers' output and gradients are exactly zero.
- NCHW, strided and channels_last inputs give the same bits; runs repeat bit for bit; an image's output and dx are the
  same alone and inside a batch; gradient subsets, a frozen weight, accumulation into .grad, no_grad and a loaded eps.
"""
import pytest
import torch

from mickey_b200.heads import KINDS, head_out
from oracle import heads_oracle as ho

pytestmark = pytest.mark.gpu
DEV = "cuda"
SHAPES = [(8, 51, 38), (24, 34, 25), (1, 7, 7), (2, 5, 9), (2, 9, 6), (1, 1, 40), (1, 40, 1), (1, 70, 65)]
MD = 60.0


def inputs(kind, B, h, w, seed=0, C_=None):
    C_ = C_ or (128 if kind == "desc" else 64)
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(B, C_, h, w, generator=g, device=DEV)
    k = 2 if kind == "offset" else 1
    W = None if kind == "desc" else torch.randn(k, C_, 1, 1, generator=g, device=DEV) / C_ ** 0.5 * 4
    go = torch.randn(B, C_ if kind == "desc" else k, h, w, generator=g, device=DEV)
    return x, W, go


def run(kind, x, W, go, eps=None):
    x = x.detach().requires_grad_()
    Wp = None if W is None else W.detach().clone().requires_grad_()
    e = torch.tensor(1e-16, device=DEV) if eps is None else eps
    out = head_out(x, kind, Wp, eps=e, max_depth=MD)
    out.backward(go)
    return out.detach(), x.grad, None if Wp is None else Wp.grad


def fp64(kind, x, W, go, eps=1e-16):
    X, G = x.double(), go.double()
    Wd = None if W is None else W.double()
    out, norm = ho.output_forward(kind, X, Wd, eps=eps, max_depth=MD)
    dx, dW = ho.output_backward(kind, X, Wd, out, norm, G, max_depth=MD)
    return out, dx, dW


def assert_close(ours, ref, what):
    bound = 2.0 ** -16 * ref.abs().max() + 2.0 ** -20 * ref.abs()
    err = (ours.double() - ref).abs()
    assert bool((err <= bound).all()), f"{what}: max err {err.max():.3e}, bound at that element {bound.flatten()[err.argmax()]:.3e}"


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("kind", list(KINDS))
def test_against_fp64(kind, shape):
    B, h, w = shape
    x, W, go = inputs(kind, B, h, w)
    ours = run(kind, x, W, go)
    ref = fp64(kind, x, W, go)
    no_interior = kind.startswith("score") and (h <= 6 or w <= 6)
    for o, r, name in zip(ours, ref, ("out", "dx", "dW")):
        if r is None:
            assert o is None
            continue
        assert o.shape == r.shape, name
        if no_interior:
            assert bool((o == 0).all()), name
        else:
            assert_close(o, r, f"{kind} {shape} {name}")


def layouts(x):
    B, C_, h, w = x.shape
    wide = torch.zeros(B, 2 * C_, h, w + 3, device=DEV)
    wide[:, ::2, :, 1:w + 1] = x
    return {"nchw": x.contiguous(), "strided": wide[:, ::2, :, 1:w + 1], "channels_last":
            x.contiguous(memory_format=torch.channels_last)}


@pytest.mark.parametrize("kind", list(KINDS))
def test_layouts_determinism_and_batch_invariance(kind):
    x, W, go = inputs(kind, 8, 51, 38, seed=1)
    base = run(kind, x, W, go)
    for name, xl in layouts(x).items():
        assert not (name == "strided" and xl.is_contiguous())
        for a, b in zip(run(kind, xl, W, go), base):
            assert a is None or torch.equal(a, b), name
    for a, b in zip(run(kind, x, W, go), base):
        assert a is None or torch.equal(a, b)
    alone = run(kind, x[3:4], W, go[3:4])
    assert torch.equal(alone[0], base[0][3:4]) and torch.equal(alone[1], base[1][3:4])


@pytest.mark.parametrize("kind", ["score_softmax", "offset", "depth_sigmoid"])
def test_gradient_subsets_frozen_weight_accumulation_and_no_grad(kind):
    x, W, go = inputs(kind, 2, 20, 17, seed=2)
    out, dx, dW = run(kind, x, W, go)
    eps = torch.tensor(1e-16, device=DEV)
    # x only: a frozen weight gets no gradient
    xr = x.clone().requires_grad_()
    Wf = W.clone()
    head_out(xr, kind, Wf, eps=eps, max_depth=MD).backward(go)
    assert torch.equal(xr.grad, dx) and Wf.grad is None
    # the weight only
    Wr = W.clone().requires_grad_()
    head_out(x, kind, Wr, eps=eps, max_depth=MD).backward(go)
    assert torch.equal(Wr.grad, dW)
    # accumulation into .grad, as torch's own layers do
    head_out(x, kind, Wr, eps=eps, max_depth=MD).backward(go)
    assert torch.equal(Wr.grad, dW + dW)
    # through the 1x1 conv's own Parameter [k, C, 1, 1]
    conv = torch.nn.Conv2d(64, W.shape[0], 1, bias=False).to(DEV)
    with torch.no_grad():
        conv.weight.copy_(W)
    head_out(x, kind, conv.weight, eps=eps, max_depth=MD).backward(go)
    assert torch.equal(conv.weight.grad, dW)
    with torch.no_grad():
        y = head_out(x, kind, Wr, eps=eps, max_depth=MD)
    assert torch.equal(y, out) and not y.requires_grad


def test_a_loaded_eps_is_honoured():
    x, W, go = inputs("score_softmax", 2, 20, 17, seed=3)
    eps = torch.tensor(0.5, device=DEV)
    ours = run("score_softmax", x, W, go, eps=eps)
    ref = fp64("score_softmax", x, W, go, eps=0.5)
    for o, r, name in zip(ours, ref, ("out", "dx", "dW")):
        assert_close(o, r, name)
    assert not torch.allclose(ours[0], run("score_softmax", x, W, go)[0], rtol=1e-3, atol=0)
