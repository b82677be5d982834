"""The heads' residual block on the GPU (mickey_b200.resblock, csrc/resblock.cu).

- The TF32 convolution GEMM alone (mk_op_conv_tf32) in its three forms, element by element against fp64 on TF32-exact
  operands, within the fp32-accumulation bound K 2^-23 sum|a||b|, with planted layout mutations that the bound rejects.
- The whole block against the fp64 oracle, forward and backward, next to torch's own cuDNN TF32 run of the same block:
  every output, gradient and running statistic within 2x the reference's own relative error (or 2e-3).
- Behaviour: determinism, strides and channels_last, gradient subsets, accumulation, no_grad, eval mode, allow_tf32 off.
"""
import ctypes as C

import pytest
import torch
import torch.nn as nn

from mickey_b200 import _lib
from mickey_b200.resblock import BasicBlock
from oracle import resblock_oracle as ro

pytestmark = pytest.mark.gpu
DEV = "cuda"
U23 = 2.0 ** -23


def tf32(t):
    """Round fp32 to TF32 (10 explicit mantissa bits), to nearest with ties away from zero, as cvt.rna.tf32.f32."""
    i = t.contiguous().view(torch.int32)
    sign = i & torch.tensor(-0x80000000, dtype=torch.int32, device=t.device)
    mag = ((i & 0x7FFFFFFF) + 0x1000) & ~0x1FFF
    return (sign | mag).view(torch.float32)


def padded_nhwc(x):
    """[B, C, h, w] -> padded NHWC [B (h+2)(w+2), C] with a zero ring."""
    B, Cc, h, w = x.shape
    return torch.nn.functional.pad(x, (1, 1, 1, 1)).permute(0, 2, 3, 1).reshape(-1, Cc).contiguous()


def unpad(rows, B, h, w):
    Cc = rows.shape[1]
    return rows.reshape(B, h + 2, w + 2, Cc)[:, 1:h + 1, 1:w + 1].permute(0, 3, 1, 2)


def channel_major(x):
    """[B, C, h, w] -> [C, Rp]: the padded NHWC rows transposed, zero beyond R."""
    p = padded_nhwc(x)
    R = p.shape[0]
    Rp = (R + 3) // 4 * 4
    out = torch.zeros(p.shape[1], Rp, dtype=p.dtype, device=p.device)
    out[:, :R] = p.t()
    return out


def op_conv(mode, a, b, B, h, w, cin, cout, taps, out_shape):
    lib = _lib.load()
    nb = int(lib.mk_op_conv_tf32_ws_bytes(mode, B, h, w, cin, cout, taps))
    assert nb > 0
    ws = torch.empty(nb, dtype=torch.uint8, device=DEV)
    out = torch.full(out_shape, float("nan"), dtype=torch.float32, device=DEV)
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(lib.mk_op_conv_tf32(mode, _lib.ptr(a), _lib.ptr(b), _lib.ptr(out), B, h, w, cin, cout, taps, _lib.ptr(ws),
                                   nb, s), "mk_op_conv_tf32")
    torch.cuda.synchronize()
    return out


def _bound_check(got, ref, bound, mutants):
    err = (got.double() - ref).abs()
    ratio = (err / bound).max().item()
    assert torch.isfinite(got).all()
    assert ratio <= 1.0, f"max err / bound = {ratio}"
    for name, m in mutants.items():
        r = ((m - ref).abs() / bound).max().item()
        assert r > 1.0, f"planted mutation '{name}' is not rejected (max |mut - ref| / bound = {r})"
    return ratio


GEMM_CASES = [  # B, h, w, cin, cout, taps
    (2, 15, 14, 64, 128, 9),
    (2, 7, 7, 128, 64, 9),
    (1, 1, 1, 32, 32, 9),
    (3, 5, 1, 96, 64, 9),          # w = 1, channels not a multiple of 64
    (2, 9, 12, 256, 128, 1),
    (1, 70, 70, 64, 64, 9),        # N > 4096 pixels
]


@pytest.mark.parametrize("B,h,w,cin,cout,taps", GEMM_CASES)
def test_conv_gemm_forms_against_fp64(B, h, w, cin, cout, taps):
    g = torch.Generator(device="cpu").manual_seed(B * 1000 + h * 10 + w + cin + taps)
    k = 3 if taps == 9 else 1
    pad = 1 if taps == 9 else 0
    x = tf32(torch.randn(B, cin, h, w, generator=g).to(DEV))
    W = tf32((torch.randn(cout, cin, k, k, generator=g) / (cin * taps) ** 0.5).to(DEV))
    dz = tf32(torch.randn(B, cout, h, w, generator=g).to(DEV))
    conv = torch.nn.functional.conv2d
    gw = torch.nn.grad
    K = cin * taps
    # forward
    got = unpad(op_conv(0, padded_nhwc(x), W, B, h, w, cin, cout, taps, (B * (h + 2) * (w + 2), cout)), B, h, w)
    ref = conv(x.double(), W.double(), padding=pad)
    bound = K * U23 * conv(x.double().abs(), W.double().abs(), padding=pad) + 1e-30
    mut = {"K chunk dropped": conv(x.double() * (torch.arange(cin, device=DEV) >= 32).double()[None, :, None, None],
                                   W.double(), padding=pad)}
    if taps == 9 and w > 1:
        mut["tap one row off"] = conv(torch.roll(x.double(), 1, 3), W.double(), padding=pad)
    _bound_check(got, ref, bound, mut)
    # dgrad
    got = unpad(op_conv(1, padded_nhwc(dz), W, B, h, w, cin, cout, taps, (B * (h + 2) * (w + 2), cin)), B, h, w)
    ref = gw.conv2d_input(x.shape, W.double(), dz.double(), padding=pad)
    bound = cout * taps * U23 * gw.conv2d_input(x.shape, W.double().abs(), dz.double().abs(), padding=pad) + 1e-30
    mut = {"taps not flipped": gw.conv2d_input(x.shape, W.double().flip(2, 3), dz.double(), padding=pad)} if taps == 9 and h * w > 1 else {}
    if B > 1:
        mut["image boundary"] = gw.conv2d_input(x.shape, W.double(), torch.roll(dz.double(), 1, 0), padding=pad)
    _bound_check(got, ref, bound, mut)
    # wgrad
    got = op_conv(2, channel_major(dz), channel_major(x), B, h, w, cin, cout, taps, (cout, cin, k, k))
    ref = gw.conv2d_weight(x.double(), W.shape, dz.double(), padding=pad)
    npix = B * h * w
    bound = npix * U23 * gw.conv2d_weight(x.double().abs(), W.shape, dz.double().abs(), padding=pad) + 1e-30
    half = dz.double().clone()
    half[-1, :, -1, :] = 0                                     # the last rows of pixels: the last wgrad slot's share
    mut = {"last pixel rows dropped": gw.conv2d_weight(x.double(), W.shape, half, padding=pad)}
    _bound_check(got, ref, bound, mut)


def _blocks(cin, cout, bn, seed):
    torch.manual_seed(seed)
    ours = BasicBlock(cin, cout, bn=bn).to(DEV)
    with torch.no_grad():
        for m in ours.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.2, 0.2)
                m.running_mean.uniform_(-0.1, 0.1)
                m.running_var.uniform_(0.5, 2.0)
    return ours


def _params_of(m, dtype):
    cv = lambda t: None if t is None else t.detach().to(dtype)
    wsc = m.shortcut[0].weight if hasattr(m, "shortcut") else None
    return cv(m.conv1.weight), cv(m.conv2.weight), cv(wsc), ro.bn_params(m.bn1, dtype), ro.bn_params(m.bn2, dtype)


def _oracle(m, x, go, train, relu, dtype):
    w1, w2, wsc, bn1, bn2 = _params_of(m, dtype)
    out, aux = ro.block_forward(x.to(dtype), w1, w2, wsc, bn1, bn2, train, relu)
    grads = ro.block_backward(x.to(dtype), w1, w2, wsc, bn1, bn2, go.to(dtype), aux, train, relu)
    run = None
    if train and bn1 is not None:
        M = x.shape[0] * x.shape[2] * x.shape[3]
        run = ro.running_update(bn1, aux["mean1"], aux["var1"], M) + ro.running_update(bn2, aux["mean2"], aux["var2"], M)
    return out, grads, run


def _cudnn_reference(m, x, go, train, relu):
    """The same block in eager torch on the GPU in fp32 (cuDNN, default TF32 flags), through autograd."""
    w1, w2, wsc = [None if p is None else p.clone().requires_grad_() for p in _params_of(m, torch.float32)[:3]]
    bns = []
    for mod in (m.bn1, m.bn2):
        if isinstance(mod, nn.BatchNorm2d):
            bns.append((mod.weight.detach().clone().requires_grad_(), mod.bias.detach().clone().requires_grad_(),
                        mod.running_mean.clone(), mod.running_var.clone(), mod.eps,
                        ro.bn_params(mod)["factor"]))
        else:
            bns.append(None)
    xx = x.clone().requires_grad_()
    F = torch.nn.functional

    def bn(z, b):
        return z if b is None else F.batch_norm(z, b[2], b[3], b[0], b[1], train, b[5], b[4])
    a1 = F.relu(bn(F.conv2d(xx, w1, padding=1), bns[0]))
    pre = bn(F.conv2d(a1, w2, padding=1), bns[1]) + (F.conv2d(xx, wsc) if wsc is not None else xx)
    out = F.relu(pre) if relu else pre
    out.backward(go)
    grads = dict(dx=xx.grad, w1=w1.grad, w2=w2.grad, wsc=None if wsc is None else wsc.grad,
                 bn1_w=None if bns[0] is None else bns[0][0].grad, bn1_b=None if bns[0] is None else bns[0][1].grad,
                 bn2_w=None if bns[1] is None else bns[1][0].grad, bn2_b=None if bns[1] is None else bns[1][1].grad)
    run = (bns[0][2], bns[0][3], bns[1][2], bns[1][3]) if train and bns[0] is not None else None
    return out.detach(), grads, run


def _ours(m, x, go, relu):
    for p in m.parameters():
        p.grad = None
    xx = x.clone().requires_grad_()
    out = m(xx, relu=relu)
    out.backward(go)
    wsc = m.shortcut[0].weight.grad if hasattr(m, "shortcut") else None
    bn = isinstance(m.bn1, nn.BatchNorm2d)
    grads = dict(dx=xx.grad, w1=m.conv1.weight.grad, w2=m.conv2.weight.grad, wsc=wsc,
                 bn1_w=m.bn1.weight.grad if bn else None, bn1_b=m.bn1.bias.grad if bn else None,
                 bn2_w=m.bn2.weight.grad if bn else None, bn2_b=m.bn2.bias.grad if bn else None)
    return out.detach(), grads


def _rel(a, ref):
    return ((a.double() - ref).norm() / ref.norm().clamp_min(1e-300)).item()


BLOCK_SHAPES = [(1024, 512), (512, 256), (256, 128), (128, 64), (128, 128)]
TRAIN_GEOMS = [(8, 38, 51), (24, 25, 34)]
EDGE_GEOMS = [(2, 1, 1), (1, 1, 7), (3, 7, 1), (2, 7, 7), (2, 15, 14), (1, 70, 70)]


def _compare(cin, cout, B, h, w, train, relu, bn=True, record=None, floor=2e-3):
    m = _blocks(cin, cout, bn, seed=cin + cout + B + h)
    if not train:
        m.eval()
    g = torch.Generator(device="cpu").manual_seed(B * 31 + h * 7 + w)
    x = torch.randn(B, cin, h, w, generator=g).to(DEV)
    go = torch.randn(B, cout, h, w, generator=g).to(DEV)
    o64, g64, r64 = _oracle(m, x, go, train, relu, torch.float64)
    o32, g32, r32 = _cudnn_reference(m, x, go, train, relu)
    out, grads = _ours(m, x, go, relu)
    ratios = {}

    def gate(name, ours, theirs, ref):
        e_ours, e_ref = _rel(ours, ref), _rel(theirs, ref)
        ratios[name] = (e_ours, e_ref)
        assert e_ours <= max(2 * e_ref, floor), f"{name}: rel err {e_ours:.3e}, cuDNN TF32 {e_ref:.3e}"
    gate("out", out, o32, o64)
    for k, v in g64.items():
        if v is None:
            assert grads[k] is None
            continue
        gate(k, grads[k], g32[k], v)
    if r64 is not None:
        mine = (m.bn1.running_mean, m.bn1.running_var, m.bn2.running_mean, m.bn2.running_var)
        for name, a, b, ref in zip(("rm1", "rv1", "rm2", "rv2"), mine, r32, r64):
            gate(name, a, b, ref)
    if record is not None:
        record[(cin, cout, B, h, w, train, relu)] = ratios
    return ratios


@pytest.mark.parametrize("cin,cout", BLOCK_SHAPES)
@pytest.mark.parametrize("B,h,w", TRAIN_GEOMS)
def test_block_training_shapes_against_fp64_and_cudnn(cin, cout, B, h, w):
    r = _compare(cin, cout, B, h, w, train=True, relu=(cin, cout) != (128, 128))
    print("\nratios", cin, cout, B, h, w, {k: f"{a:.2e}/{b:.2e}" for k, (a, b) in r.items()})


@pytest.mark.parametrize("B,h,w", EDGE_GEOMS)
@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("relu", [True, False])
def test_block_edge_geometries(B, h, w, train, relu):
    _compare(128, 64, B, h, w, train, relu)
    _compare(64, 64, B, h, w, train, relu)


def test_block_without_batch_norm():
    # At this size cuDNN picks full-fp32 algorithms, so its error is no TF32 yardstick.  TF32 rounding flips ReLU masks
    # of values near zero, which moves the gradients by a few percent (cuDNN's own TF32 runs above show 1-3 %); the
    # convolution arithmetic itself is checked element by element by test_conv_gemm_forms_against_fp64.
    _compare(128, 64, 2, 9, 11, train=True, relu=True, bn=False, floor=6e-2)
    _compare(64, 64, 2, 9, 11, train=True, relu=False, bn=False, floor=6e-2)


def test_deterministic_and_layout_independent():
    m = _blocks(256, 128, True, 5)
    x = torch.randn(4, 256, 13, 17, device=DEV)
    go = torch.randn(4, 128, 13, 17, device=DEV)
    state = {k: v.clone() for k, v in m.state_dict().items()}
    runs = []
    for variant in ("contig", "contig", "channels_last", "strided"):
        m.load_state_dict(state)
        xi = x.clone()
        if variant == "channels_last":
            xi = xi.contiguous(memory_format=torch.channels_last)
        elif variant == "strided":
            xi = torch.randn(4, 256, 13, 34, device=DEV)[..., ::2]
            xi.copy_(x)
        xi.requires_grad_()
        for p in m.parameters():
            p.grad = None
        out = m(xi)
        out.backward(go.contiguous(memory_format=torch.channels_last) if variant == "channels_last" else go)
        runs.append([out, xi.grad] + [p.grad for p in m.parameters()] + [b.clone() for b in m.buffers()])
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert torch.equal(a, b)


def test_gradient_subsets_accumulation_and_modes():
    m = _blocks(128, 64, True, 7)
    x = torch.randn(2, 128, 9, 10, device=DEV)
    go = torch.randn(2, 64, 9, 10, device=DEV)
    # full run for reference values
    out_full, g_full = _ours(m, x, go, True)
    m2 = _blocks(128, 64, True, 7)
    # frozen conv1 weight and an input that needs no gradient: no dX, no conv1 grad, the rest equal
    m2.conv1.weight.requires_grad_(False)
    out = m2(x)
    out.backward(go)
    assert m2.conv1.weight.grad is None
    assert torch.equal(m2.conv2.weight.grad, g_full["w2"])
    assert torch.equal(m2.shortcut[0].weight.grad, g_full["wsc"])
    assert torch.equal(m2.bn1.weight.grad, g_full["bn1_w"])
    # accumulation
    m3 = _blocks(128, 64, True, 7)
    for _ in range(2):
        m3(x).backward(go)
    assert torch.allclose(m3.conv2.weight.grad, 2 * g_full["w2"], rtol=1e-6, atol=0)
    # no_grad in train mode updates the running statistics; eval leaves them
    m4 = _blocks(128, 64, True, 7)
    rm = m4.bn1.running_mean.clone()
    with torch.no_grad():
        y = m4(x)
    assert not y.requires_grad and not torch.equal(rm, m4.bn1.running_mean)
    assert int(m4.bn1.num_batches_tracked) == 1
    m4.eval()
    before = [b.clone() for b in m4.buffers()]
    m4(x)
    for a, b in zip(before, m4.buffers()):
        assert torch.equal(a, b)


def test_momentum_none_is_cumulative_average():
    m = _blocks(64, 64, True, 9)
    ref = _blocks(64, 64, True, 9)
    for mod in (m.bn1, m.bn2, ref.bn1, ref.bn2):
        mod.momentum = None
    xs = [torch.randn(2, 64, 6, 5, device=DEV) for _ in range(3)]
    for x in xs:
        with torch.no_grad():
            m(x)
        w1, w2, wsc, bn1, bn2 = _params_of(ref, torch.float64)
        _, aux = ro.block_forward(x.double(), w1, w2, wsc, bn1, bn2, True, True)
        for mod, mean, var in ((ref.bn1, aux["mean1"], aux["var1"]), (ref.bn2, aux["mean2"], aux["var2"])):
            rm, rv = ro.running_update(ro.bn_params(mod, torch.float64), mean, var, 60)
            mod.running_mean.copy_(rm)
            mod.running_var.copy_(rv)
            mod.num_batches_tracked += 1
    for a, b in ((m.bn1.running_var, ref.bn1.running_var), (m.bn2.running_mean, ref.bn2.running_mean)):
        assert _rel(a, b.double()) < 5e-3


def test_allow_tf32_off_raises():
    m = _blocks(64, 64, True, 1)
    x = torch.randn(1, 64, 4, 4, device=DEV)
    old = torch.backends.cudnn.allow_tf32
    try:
        torch.backends.cudnn.allow_tf32 = False
        with pytest.raises(RuntimeError, match="allow_tf32"):
            m(x)
    finally:
        torch.backends.cudnn.allow_tf32 = old
