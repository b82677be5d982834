"""The residual block stage by stage on the GPU, element by element against fp64.  Each stage starts from the module's
own intermediates: the forward's saved region (pre-BN z1 / z2, batch statistics, BN1-apply + ReLU) and the backward's
workspace (g, dz2, dA1, dz1, the data gradients), located with mk_resblock_layout.  So no stage inherits an earlier
stage's error.  Bounds: TF32 operands are exact (the kernels round them; the references use the same rounded values), a
GEMM carries K 2^-23 sum|a||b| of fp32 accumulation, element-wise fp32 arithmetic a few 2^-24 of its operands, and each
TF32 rounding 2^-11.  Every check plants mutations of its reference and asserts that the bound rejects them."""
import ctypes as C
import math

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from mickey_b200 import _lib
from mickey_b200.resblock import BasicBlock
from tests.test_gpu_resblock import padded_nhwc, tf32, unpad

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
GW = torch.nn.grad


def check(got, ref, bound, mutants=None, what=""):
    got, ref = got.double(), ref.double()
    assert torch.isfinite(got).all(), what
    r = ((got - ref).abs() / bound).max().item()
    assert r <= 1.0, f"{what}: max err / bound = {r}"
    for name, m in (mutants or {}).items():
        rm = ((m.double() - ref).abs() / bound).max().item()
        assert rm > 1.0, f"{what}: planted '{name}' not rejected ({rm})"
    return r


def f32_at(buf, off, shape):
    n = math.prod(shape)
    return buf[off:off + 4 * n].view(torch.float32).view(shape)


def wgrad_last_slot_rows(R, cout, cin):
    """Padded rows the last weight-gradient slot covers (the kernels' slot plan)."""
    bn = 128 if cin >= 128 else 64
    tiles = -(-cout // 128) * -(-cin // bn)
    kch = -(-R // 32)
    s = min(max(1, min(32, -(-264 // tiles))), kch)
    cps = -(-kch // s)
    slots = -(-kch // cps)
    return (slots - 1) * cps * 32, R


def conv_bound(a, w, pad, K):
    return K * 2 * U * F.conv2d(a.abs(), w.abs(), padding=pad) + 1e-300


def bn_bwd_ref(g, z, mean, rstd, gamma, train):
    xh = (z - mean[None, :, None, None]) * rstd[None, :, None, None]
    M = g.shape[0] * g.shape[2] * g.shape[3]
    sg, sgx = g.sum((0, 2, 3)), (g * xh).sum((0, 2, 3))
    k = (gamma * rstd)[None, :, None, None]
    a = (sg / M)[None, :, None, None] if train else torch.zeros_like(k)
    b = (sgx / M)[None, :, None, None] if train else torch.zeros_like(k)
    dz = k * (g - a - xh * b)
    bound = 2.0 ** -11 * dz.abs() + 8 * U * k.abs() * (g.abs() + a.abs() + xh.abs() * b.abs()) + 1e-300
    return dz, bound, k * (g - xh * b), sg, sgx, xh


def run_stages(cin, cout, B, h, w, train, relu, bn=True, seed=0):
    torch.manual_seed(seed)
    m = BasicBlock(cin, cout, bn=bn).to(DEV)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, nn.BatchNorm2d):
                mod.weight.uniform_(0.5, 1.5); mod.bias.uniform_(-0.2, 0.2)
                mod.running_mean.uniform_(-0.1, 0.1); mod.running_var.uniform_(0.5, 2.0)
    if not train:
        m.eval()
    g = torch.Generator(device="cpu").manual_seed(seed + B + h + w)
    x = torch.randn(B, cin, h, w, generator=g).to(DEV).requires_grad_()
    go = torch.randn(B, cout, h, w, generator=g).to(DEV)
    run0 = [b.clone() for b in (m.bn1.running_mean, m.bn1.running_var, m.bn2.running_mean, m.bn2.running_var)] if bn else None
    out = m(x, relu=relu)
    saved, out_s, w1, w2, wsc, g1, g2 = out.grad_fn.saved_tensors
    lib = _lib.load()
    so, bo = (C.c_longlong * 6)(), (C.c_longlong * 6)()
    _lib.check(lib.mk_resblock_layout(B, h, w, cin, cout, so, bo), "mk_resblock_layout")
    R = B * (h + 2) * (w + 2)
    Rp = (R + 3) // 4 * 4
    nhwc = lambda buf, off, c: unpad(f32_at(buf, off, (R, c)), B, h, w).double()
    z1, z2, a1 = nhwc(saved, so[0], cout), nhwc(saved, so[1], cout), nhwc(saved, so[2], cout)
    st = f32_at(saved, so[5], (4, cout)).double()
    x32 = tf32(x.detach()).double()
    W1, W2 = tf32(w1.detach()).double(), tf32(w2.detach()).double()
    Wsc = tf32(wsc.detach()).double() if wsc is not None else None
    gam = [None if t is None else t.detach().double() for t in (g1, g2)]
    bet = [m.bn1.bias.detach().double(), m.bn2.bias.detach().double()] if bn else [None, None]
    M = B * h * w

    # ---- forward stages ----
    def off_by_one(t, W):             # a tap read one padded row off, along a dimension longer than 1
        if h * w == 1:
            return {}
        return {"tap one row off": F.conv2d(torch.roll(t, 1, 3 if w > 1 else 2), W, padding=1)}
    check(z1, F.conv2d(x32, W1, padding=1), conv_bound(x32, W1, 1, 9 * cin),
          {**off_by_one(x32, W1),
           "K chunk dropped": F.conv2d(x32 * (torch.arange(cin, device=DEV) >= 32).double()[None, :, None, None], W1, padding=1)},
          "z1")
    check(z2, F.conv2d(a1, W2, padding=1), conv_bound(a1, W2, 1, 9 * cout), off_by_one(a1, W2), "z2")
    ys = []
    for i, (z, nb) in enumerate(((z1, m.bn1), (z2, m.bn2))):
        mean, rstd = st[2 * i], st[2 * i + 1]
        if bn and train:
            mu, var = z.mean((0, 2, 3)), z.var((0, 2, 3), unbiased=False)
            ring = F.pad(z, (1, 1, 1, 1))                          # the pad ring counted in the statistics
            mu_r, var_r = ring.mean((0, 2, 3)), ring.var((0, 2, 3), unbiased=False)
            check(mean, mu, 2 * U * mu.abs() + 2.0 ** -30 * z.abs().mean((0, 2, 3)) + 1e-300, {"pad ring in mean": mu_r},
                  f"mean{i + 1}")
            rs = (var + nb.eps).rsqrt()
            check(rstd, rs, 2 * U * rs + 1e-300, {"pad ring in var": (var_r + nb.eps).rsqrt()}, f"rstd{i + 1}")
            f = nb.momentum
            rm0, rv0 = run0[2 * i].double(), run0[2 * i + 1].double()
            rm_ref = f * mu + (1 - f) * rm0
            rv_ref = f * var * M / (M - 1) + (1 - f) * rv0
            check(nb.running_mean, rm_ref, 4 * U * (f * mu.abs() + (1 - f) * rm0.abs()) + 1e-300, None, f"running_mean{i + 1}")
            check(nb.running_var, rv_ref, 4 * U * (f * var.abs() * M / (M - 1) + (1 - f) * rv0.abs()) + 1e-300,
                  {"biased variance": f * var + (1 - f) * rv0}, f"running_var{i + 1}")
        elif bn:
            assert torch.equal(mean, nb.running_mean.double())
            check(rstd, (nb.running_var.double() + nb.eps).rsqrt(), 2 * U * rstd.abs(), None, f"rstd{i + 1}")
            assert torch.equal(nb.running_var, run0[2 * i + 1]) and torch.equal(nb.running_mean, run0[2 * i])
        if bn:
            c = lambda t: t[None, :, None, None]
            zc = (z - c(mean)) * c(rstd)
            y = zc * c(gam[i]) + c(bet[i])
            yb = 6 * U * ((z - c(mean)).abs() * c(rstd) * c(gam[i]).abs() + c(bet[i]).abs())
        else:
            y, yb = z, torch.zeros_like(z)
        ys.append((y, yb))
    y1, yb1 = ys[0]
    a1_ref = F.relu(y1)
    check(a1, a1_ref, 2.0 ** -11 * y1.abs() + yb1 + 1e-300,
          {"ReLU mask shifted by one channel": y1 * (torch.roll(y1, 1, 1) > 0)}, "BN1-apply + ReLU")
    y2, yb2 = ys[1]
    if Wsc is not None:
        s = F.conv2d(x32, Wsc)
        sb = conv_bound(x32, Wsc, 0, cin) + U * s.abs()
    else:
        s, sb = x.detach().double(), torch.zeros_like(y2)
    pre = y2 + s
    check(out.detach(), F.relu(pre) if relu else pre, yb2 + sb + 2 * U * pre.abs() + 1e-300,
          {"ReLU mask shifted by one channel": pre * (torch.roll(pre, 1, 1) > 0)} if relu else None, "out")

    # ---- backward stages, from the backward's own workspace ----
    flags = (1 if (bn and train) else 0) | (2 if relu else 0) | (8 if bn else 0)
    P = _lib.MkResblockParams()
    P.w1, P.w2, P.wsc = w1.data_ptr(), w2.data_ptr(), None if wsc is None else wsc.data_ptr()
    if bn:
        P.bn1_w, P.bn2_w = g1.data_ptr(), g2.data_ptr()
    nws = int(lib.mk_resblock_backward_ws_bytes(B, h, w, cin, cout))
    s_ = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    gstr = (C.c_longlong * 4)(*go.stride())

    def backward(want):
        ws = torch.zeros(nws, dtype=torch.uint8, device=DEV)
        grads = {"dx": torch.empty_like(x), "w1": torch.empty_like(w1), "w2": torch.empty_like(w2),
                 "wsc": None if wsc is None else torch.empty_like(wsc),
                 "bn1_w": None if not bn else torch.empty_like(g1), "bn1_b": None if not bn else torch.empty_like(g1),
                 "bn2_w": None if not bn else torch.empty_like(g2), "bn2_b": None if not bn else torch.empty_like(g2)}
        G = _lib.MkResblockGrads()
        for i, k in enumerate(("dx", "w1", "w2", "wsc", "bn1_w", "bn1_b", "bn2_w", "bn2_b")):
            if want >> i & 1:
                setattr(G, k, grads[k].data_ptr())
        _lib.check(lib.mk_resblock_backward(_lib.ptr(saved), _lib.ptr(go), gstr, _lib.ptr(out_s), B, h, w, cin, cout,
                                            C.byref(P), flags, want, C.byref(G), _lib.ptr(ws), nws, s_), "backward")
        torch.cuda.synchronize()
        return ws, grads

    full = 1 | 2 | 4 | (8 if wsc is not None else 0) | (0xF0 if bn else 0)
    ws2, _ = backward(4)                           # dW2 only: dz^T holds dz2
    dz2 = unpad(f32_at(ws2, bo[2], (cout, Rp))[:, :R].t(), B, h, w).double()
    ws, gr = backward(full)
    gf = nhwc(ws, bo[0], cout)
    g_ref = go.double() * (out.detach() > 0) if relu else go.double()
    assert torch.equal(gf, g_ref)
    if bn:
        dz2_ref, bnd, no_mean, sg, sgx, _ = bn_bwd_ref(gf, z2, st[2], st[3], gam[1], train)
        check(dz2, dz2_ref, bnd, {"mean term dropped": no_mean} if train else None, "dz2")
        check(gr["bn2_b"], sg, 2 * U * sg.abs() + 2.0 ** -30 * gf.abs().sum((0, 2, 3)) + 1e-300, None, "dbeta2")
        check(gr["bn2_w"], sgx, 2 * U * sgx.abs() + 2.0 ** -30 * (gf.abs() * z2.abs()).sum((0, 2, 3)) * st[3] + 1e-300,
              None, "dgamma2")
    else:
        check(dz2, tf32(gf.float()).double(), 2.0 ** -11 * gf.abs() + 1e-300, None, "dz2")
    da1 = nhwc(ws, bo[3], cout)
    check(da1, GW.conv2d_input(a1.shape, W2, dz2, padding=1),
          9 * cout * 2 * U * GW.conv2d_input(a1.shape, W2.abs(), dz2.abs(), padding=1) + 1e-300,
          {"taps not flipped": GW.conv2d_input(a1.shape, W2.flip(2, 3), dz2, padding=1)} if h * w > 1 else None, "dA1")
    dz1 = nhwc(ws, bo[1], cout)
    g1m = da1 * (a1 > 0)
    if bn:
        dz1_ref, bnd, no_mean, sg1, sgx1, _ = bn_bwd_ref(g1m, z1, st[0], st[1], gam[0], train)
        shifted = bn_bwd_ref(da1 * (torch.roll(a1, 1, 1) > 0), z1, st[0], st[1], gam[0], train)[0]
        # with two values per channel the train-mode BN backward is identically zero: nothing upstream can show in dz1
        muts = {} if train and M <= 2 else {"ReLU mask shifted by one channel": shifted,
                                            **({"mean term dropped": no_mean} if train else {})}
        check(dz1, dz1_ref, bnd, muts, "dz1")
        check(gr["bn1_b"], sg1, 2 * U * sg1.abs() + 2.0 ** -30 * g1m.abs().sum((0, 2, 3)) + 1e-300, None, "dbeta1")
    else:
        check(dz1, tf32(g1m.float()).double(), 2.0 ** -11 * g1m.abs() + 1e-300,
              {"ReLU mask shifted by one channel": da1 * (torch.roll(a1, 1, 1) > 0)}, "dz1")
    # weight gradients: pixel slots folded in order; the last slot's rows dropped must be rejected
    npix = M + 32
    lo, hi = wgrad_last_slot_rows(R, cout, cout)

    def drop_rows(t, lo, hi):
        p = padded_nhwc(t)
        p[lo:hi] = 0
        return unpad(p, B, h, w)

    def slot_mutant(name, a, d, shape, lo, hi):
        # only where the last slot holds interior pixels (a slot of ring rows contributes zero anyway)
        if torch.equal(drop_rows(torch.ones_like(d[:, :1]), lo, hi), torch.ones_like(d[:, :1])):
            return {}
        return {name: GW.conv2d_weight(a, shape, drop_rows(d, lo, hi), padding=1)}
    wb = lambda a, d, shape, pad: npix * 2 * U * GW.conv2d_weight(a.abs(), shape, d.abs(), padding=pad) + 1e-300
    check(gr["w2"], GW.conv2d_weight(a1, W2.shape, dz2, padding=1), wb(a1, dz2, W2.shape, 1),
          slot_mutant("last wgrad slot dropped", a1, dz2, W2.shape, lo, hi), "dW2")
    lo, hi = wgrad_last_slot_rows(R, cout, cin)
    check(gr["w1"], GW.conv2d_weight(x32, W1.shape, dz1, padding=1), wb(x32, dz1, W1.shape, 1),
          slot_mutant("last wgrad slot dropped", x32, dz1, W1.shape, lo, hi), "dW1")
    dxc = nhwc(ws, bo[4], cin)
    check(dxc, GW.conv2d_input(x.shape, W1, dz1, padding=1),
          9 * cout * 2 * U * GW.conv2d_input(x.shape, W1.abs(), dz1.abs(), padding=1) + 1e-300, None, "conv1 dgrad")
    if Wsc is not None:
        gt = tf32(gf.float()).double()
        check(gr["wsc"], GW.conv2d_weight(x32, Wsc.shape, gt), wb(x32, gt, Wsc.shape, 0), None, "dWsc")
        dxs = nhwc(ws, bo[5], cin)
        check(dxs, GW.conv2d_input(x.shape, Wsc, gt), cout * 2 * U * GW.conv2d_input(x.shape, Wsc.abs(), gt.abs()) + 1e-300,
              None, "shortcut dgrad")
        other = dxs
    else:
        other = gf
    check(gr["dx"], dxc + other, U * (dxc + other).abs() + 1e-300, {"shortcut dropped": dxc}, "dX")
    # the module's own backward gives the same bits as this call
    out.backward(go)
    assert torch.equal(x.grad, gr["dx"]) and torch.equal(m.conv1.weight.grad, gr["w1"])


@pytest.mark.parametrize("cin,cout", [(1024, 512), (512, 256), (256, 128), (128, 64), (128, 128)])
@pytest.mark.parametrize("B,h,w", [(8, 38, 51), (24, 25, 34)])
def test_stages_training_shapes(cin, cout, B, h, w):
    run_stages(cin, cout, B, h, w, train=True, relu=(cin, cout) != (128, 128))


EDGES = [(2, 1, 1), (1, 1, 7), (3, 7, 1), (2, 7, 7), (1, 3, 75), (1, 70, 70)]   # (1, 3, 75): R = 385 = 3 * 128 + 1


@pytest.mark.parametrize("B,h,w", EDGES)
@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("relu", [True, False])
def test_stages_edge_geometries(B, h, w, train, relu):
    run_stages(128, 64, B, h, w, train, relu)
    run_stages(64, 64, B, h, w, train, relu, seed=1)


def test_stages_without_batch_norm():
    run_stages(128, 64, 2, 9, 11, True, True, bn=False)
    run_stages(64, 64, 2, 9, 11, True, False, bn=False)
