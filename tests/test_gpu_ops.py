"""GPU unit tests of the individual CUDA kernels (through the operator-level C ABI) against plain
fp32 torch math on the same inputs.  The wgmma GEMM is additionally cross-checked against the SIMT
debug kernel, which shares its epilogues, to separate descriptor bugs from epilogue bugs."""
import ctypes as C
import os
import math

import pytest
import torch
import torch.nn.functional as F

from mickey_b200 import _lib
from tests.common import rel_err
from tests.gpu_util import gemm, stream

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


@pytest.mark.parametrize("impl", ["simt", "tc"])
@pytest.mark.parametrize("M,N,K", [(300, 256, 192), (128, 128, 64), (1000, 384, 1536), (77, 64, 128)])
def test_gemm_store_h_bias_gelu(impl, M, N, K):
    a = _rand(M, K, seed=1).half()
    w = _rand(N, K, scale=0.05, seed=2).half()
    bias = _rand(N, scale=0.1, seed=3)
    out = torch.zeros(M, N, dtype=torch.float16, device=DEV)
    gemm("STORE_H", a, w, M, N, K, impl=impl, bias=bias, act=1, out_h=out, out_h_ld=N)
    ref = F.gelu(a.float() @ w.float().t() + bias)
    assert rel_err(out, ref) < 2e-3


def test_persistent_gemm_large_grids():
    """Grids of several waves of one-tile CTAs (two resident per SM): bias+GELU store, fp32 residual, grouped LayerNorm
    epilogue and a 3x3 conv, all against torch."""
    for M, N, K in ((4000, 1536, 384),      # 384 one-tile CTAs
                    (20000, 1536, 768),     # 157 x 12 tiles, K = 12 chunks
                    (9000, 640, 1536)):     # 71 x 5 tiles, K = 24 chunks
        a, w, bias = _rand(M, K, seed=40).half(), _rand(N, K, scale=0.05, seed=41).half(), _rand(N, scale=0.1, seed=42)
        out = torch.zeros(M, N, dtype=torch.float16, device=DEV)
        gemm("STORE_H", a, w, M, N, K, bias=bias, act=1, out_h=out, out_h_ld=N)
        assert rel_err(out, F.gelu(a.float() @ w.float().t() + bias)) < 2e-3, (M, N, K)
    M, N, K = 30000, 768, 768                                   # 235 x 6 tiles, fp32 residual
    a, w = _rand(M, K, seed=43).half(), _rand(N, K, scale=0.05, seed=44).half()
    bias, gamma, x = _rand(N, scale=0.1, seed=45), _rand(N, seed=46), _rand(M, N, seed=47)
    ref = x + gamma * (a.float() @ w.float().t() + bias)
    gemm("RESID_F", a, w, M, N, K, bias=bias, gamma=gamma, out_f=x, out_f_ld=N)
    assert rel_err(x, ref) < 1e-5
    M, N, K = 9000, 768, 768                                    # 71 x 6 = 426 tiles, K = 12 chunks
    a, w = _rand(M, K, seed=43).half(), _rand(N, K, scale=0.05, seed=44).half()
    bias, gamma, x = _rand(N, scale=0.1, seed=45), _rand(N, seed=46), _rand(M, N, seed=47)
    ref = x + gamma * (a.float() @ w.float().t() + bias)
    gemm("RESID_F", a, w, M, N, K, bias=bias, gamma=gamma, out_f=x, out_f_ld=N)
    assert rel_err(x, ref) < 1e-5
    R, G, K = 80000, 4, 256                                     # 625 x 1 x 4 = 2500 tiles, LayerNorm epilogue
    a, w = _rand(R, G * K, seed=48).half(), _rand(G * 128, K, scale=0.1, seed=49).half()
    gamma, beta, x32 = _rand(G * 128, seed=50), _rand(G * 128, seed=51), _rand(R, G * 128, seed=52)
    x_ref = x32.clone()
    out_h = torch.zeros(R, G * 256, dtype=torch.float16, device=DEV)
    gemm("LN", a, w, R, 128, K, groups=G, a_col_group_off=K, b_row_group_off=128, gamma=gamma, beta=beta, ln_group_off=128,
         eps=1e-5, out_f=x32, out_f_ld=G * 128, out_f_group_off=128, out_h=out_h, out_h_ld=G * 256, out_h_group_off=256)
    for g in range(G):
        acc = a[:, g * K:(g + 1) * K].float() @ w[g * 128:(g + 1) * 128].float().t()
        ref = x_ref[:, g * 128:(g + 1) * 128] + F.layer_norm(acc, (128,), gamma[g * 128:(g + 1) * 128], beta[g * 128:(g + 1) * 128], 1e-5)
        assert rel_err(x32[:, g * 128:(g + 1) * 128], ref) < 1e-4, g
        assert rel_err(out_h[:, g * 256:g * 256 + 128], ref) < 1e-3, g
    _conv_case(6, 51, 38, 128, 128, 2)                          # 100 x 1 x 2 groups, 128-wide tiles
    _conv_case(16, 51, 38, 128, 256, 2)                         # 265 x 2 x 2 groups


def _conv_case(n_img, gh, gw, cin, cout, Gc):
    h2, w2 = gh + 2, gw + 2
    xc = _rand(n_img, Gc * cin, gh, gw, seed=53).half()
    wt = _rand(Gc * cout, cin, 3, 3, scale=0.05, seed=54).half()
    xp = torch.zeros(n_img, h2, w2, Gc * cin, dtype=torch.float16, device=DEV)
    xp[:, 1:-1, 1:-1] = xc.permute(0, 2, 3, 1)
    wp = wt.permute(0, 2, 3, 1).reshape(Gc * cout, 9 * cin).contiguous()
    Rr = n_img * h2 * w2
    o32 = torch.full((Rr, Gc * cout), 7.0, device=DEV)
    taps = [(ky - 1) * w2 + (kx - 1) for ky in range(3) for kx in range(3)]
    gemm("CONV", xp.reshape(Rr, Gc * cin), wp, Rr, cout, taps=taps, chunks_per_tap=cin // 64, groups=Gc, a_col_group_off=cin,
         b_row_group_off=cout, act=2, pad_h2=h2, pad_w2=w2, out_f=o32, out_f_ld=Gc * cout, out_f_group_off=cout)
    got = o32.reshape(n_img, h2, w2, Gc * cout)
    for g in range(Gc):
        ref = F.relu(F.conv2d(xc[:, g * cin:(g + 1) * cin].float(), wt[g * cout:(g + 1) * cout].float(), padding=1))
        assert rel_err(got[:, 1:-1, 1:-1, g * cout:(g + 1) * cout].permute(0, 3, 1, 2), ref) < 1e-5, g
    ring = got.clone(); ring[:, 1:-1, 1:-1] = 0
    assert float(ring.abs().max()) == 0.0


@pytest.mark.parametrize("impl", ["simt", "tc"])
def test_gemm_resid_layerscale(impl):
    M, N, K = 515, 384, 384
    a = _rand(M, K, seed=4).half()
    w = _rand(N, K, scale=0.05, seed=5).half()
    bias, gamma = _rand(N, scale=0.1, seed=6), _rand(N, seed=7)
    x = _rand(M, N, seed=8)
    ref = x + gamma * (a.float() @ w.float().t() + bias)
    gemm("RESID_F", a, w, M, N, K, impl=impl, bias=bias, gamma=gamma, out_f=x, out_f_ld=N)
    assert rel_err(x, ref) < 1e-5


@pytest.mark.parametrize("impl", ["simt", "tc"])
def test_gemm_grouped_store_f(impl):
    """4 groups reading column slices of one A matrix and row slices of one stacked B (head layout)."""
    R, G, K, N = 333, 4, 128, 384
    a = _rand(R, G * 256, seed=9).half()
    w = _rand(G * N, K, scale=0.1, seed=10).half()
    out = torch.zeros(R, G * N, device=DEV)
    gemm("STORE_F", a, w, R, N, K, impl=impl, groups=G, a_col_group_off=256, b_row_group_off=N,
         out_f=out, out_f_ld=G * N, out_f_group_off=N)
    for g in range(G):
        ref = a[:, g * 256:g * 256 + K].float() @ w[g * N:(g + 1) * N].float().t()
        assert rel_err(out[:, g * N:(g + 1) * N], ref) < 1e-5, g


@pytest.mark.parametrize("impl", ["simt", "tc"])
@pytest.mark.parametrize("cin,cout", [(128, 64), (192, 128)])
def test_conv3x3_as_shifted_gemm(impl, cin, cout):
    """3x3 conv (pad 1) + bias + fp16 residual + ReLU over a zero-padded NHWC image == F.conv2d."""
    n_img, gh, gw = 3, 9, 7
    h2, w2 = gh + 2, gw + 2
    x = _rand(n_img, cin, gh, gw, seed=11).half()
    wt = _rand(cout, cin, 3, 3, scale=0.05, seed=12).half()
    bias = _rand(cout, scale=0.1, seed=13)
    res = _rand(n_img, cout, gh, gw, seed=14).half()
    xp = torch.zeros(n_img, h2, w2, cin, dtype=torch.float16, device=DEV)
    xp[:, 1:-1, 1:-1] = x.permute(0, 2, 3, 1)
    rp = torch.zeros(n_img, h2, w2, cout, dtype=torch.float16, device=DEV)
    rp[:, 1:-1, 1:-1] = res.permute(0, 2, 3, 1)
    wp = wt.permute(0, 2, 3, 1).reshape(cout, 9 * cin).contiguous()
    R = n_img * h2 * w2
    out = torch.full((R, cout), 7.0, dtype=torch.float16, device=DEV)
    out32 = torch.full((R, cout), 7.0, device=DEV)
    taps = [(ky - 1) * w2 + (kx - 1) for ky in range(3) for kx in range(3)]
    gemm("CONV", xp.reshape(R, cin), wp, R, cout, impl=impl, taps=taps, chunks_per_tap=cin // 64, bias=bias, act=2,
         res_h=rp.reshape(R, cout), res_h_ld=cout, pad_h2=h2, pad_w2=w2, out_h=out, out_h_ld=cout,
         out_f=out32, out_f_ld=cout)
    ref = F.relu(F.conv2d(x.float(), wt.float(), padding=1) + bias.view(1, -1, 1, 1) + res.float())
    got = out32.reshape(n_img, h2, w2, cout)
    assert rel_err(got[:, 1:-1, 1:-1].permute(0, 3, 1, 2), ref) < 1e-5
    ring = got.clone(); ring[:, 1:-1, 1:-1] = 0
    assert float(ring.abs().max()) == 0.0          # pad ring is written as zeros
    assert rel_err(out.float(), out32) < 1e-3


@pytest.mark.parametrize("impl", ["simt", "tc"])
def test_gemm_layernorm_epilogue(impl):
    R, G, K = 260, 2, 256
    a = _rand(R, G * K, seed=15).half()
    w = _rand(G * 128, K, scale=0.1, seed=16).half()
    gamma, beta = _rand(G * 128, seed=17), _rand(G * 128, seed=18)
    x32 = _rand(R, G * 128, seed=19)
    x_ref = x32.clone()
    out_h = torch.zeros(R, G * 256, dtype=torch.float16, device=DEV)
    gemm("LN", a, w, R, 128, K, impl=impl, groups=G, a_col_group_off=K, b_row_group_off=128, gamma=gamma, beta=beta,
         ln_group_off=128, eps=1e-5, out_f=x32, out_f_ld=G * 128, out_f_group_off=128, out_h=out_h, out_h_ld=G * 256,
         out_h_group_off=256)
    for g in range(G):
        acc = a[:, g * K:(g + 1) * K].float() @ w[g * 128:(g + 1) * 128].float().t()
        ref = x_ref[:, g * 128:(g + 1) * 128] + F.layer_norm(acc, (128,), gamma[g * 128:(g + 1) * 128],
                                                               beta[g * 128:(g + 1) * 128], 1e-5)
        assert rel_err(x32[:, g * 128:(g + 1) * 128], ref) < 1e-4, g
        assert rel_err(out_h[:, g * 256:g * 256 + 128], ref) < 1e-3, g


@pytest.mark.parametrize("D", [384, 768, 1024])
def test_layernorm(D):
    lib = _lib.load()
    rows = 777
    x, w, b = _rand(rows, D, seed=20) * 3 + 1, _rand(D, seed=21), _rand(D, seed=22)
    out = torch.zeros(rows, D, dtype=torch.float16, device=DEV)
    _lib.check(lib.mk_op_layernorm(_lib.ptr(x), _lib.ptr(w), _lib.ptr(b), _lib.ptr(out), rows, D, 1e-6, 0, 0, 0, stream()))
    assert rel_err(out, F.layer_norm(x, (D,), w, b, 1e-6)) < 1e-3


def test_layernorm_scatter_to_padded_grid():
    lib = _lib.load()
    n_img, gh, gw, D = 2, 5, 4, 384
    T = gh * gw + 1
    x, w, b = _rand(n_img * T, D, seed=23), _rand(D, seed=24), _rand(D, seed=25)
    out = torch.zeros(n_img, gh + 2, gw + 2, D, dtype=torch.float16, device=DEV)
    _lib.check(lib.mk_op_layernorm(_lib.ptr(x), _lib.ptr(w), _lib.ptr(b), _lib.ptr(out), n_img * T, D, 1e-6, 1, gh, gw, stream()))
    ref = F.layer_norm(x, (D,), w, b, 1e-6).reshape(n_img, T, D)[:, 1:].reshape(n_img, gh, gw, D)
    assert rel_err(out[:, 1:-1, 1:-1], ref) < 1e-3
    assert float(out[:, 0].abs().max()) == 0 and float(out[:, :, 0].abs().max()) == 0


@pytest.mark.parametrize("impl", [2, 1], ids=["mma", "tcgen05"])
@pytest.mark.parametrize("T,heads,scale", [(211, 6, 1.5), (1939, 6, 1.5), (64, 12, 1.5), (300, 6, 6.0)])
def test_attention(T, heads, scale, impl):
    """impl 2: the mma.sync kernel; impl 1: the TMA / asynchronous tensor-core kernel (wgmma on sm_90a; its test id
    `tcgen05` is the one it had when the library targeted sm_100a).  scale 6.0 makes the logits span > 2^8, so that the
    running maximum moves and O is rescaled across key tiles."""
    lib = _lib.load()
    n_img, D = 2, heads * 64
    qkv = (_rand(n_img * T, 3 * D, seed=26) * scale).half()
    out = torch.zeros(n_img * T, D, dtype=torch.float16, device=DEV)
    _lib.check(lib.mk_op_attention(_lib.ptr(qkv), _lib.ptr(out), n_img, T, D, heads, impl, stream()))
    q, k, v = qkv.float().reshape(n_img, T, 3, heads, 64).permute(2, 0, 3, 1, 4)
    ref = (torch.softmax(q @ k.transpose(-1, -2) * 0.125, -1) @ v).transpose(1, 2).reshape(n_img * T, D)
    assert rel_err(out, ref) < 2e-3


def test_gemm_2sm():
    """Large GEMMs with N % 256 == 0 (and one small one): bias+GELU, fp32 residual, fp32 store and plain fp16 store;
    rows beyond M stay untouched."""
    for M, N, K in ((20000, 1536, 768), (40000, 512, 1024), (256, 256, 768)):
        a, w, bias = _rand(M, K, seed=70).half(), _rand(N, K, scale=0.05, seed=71).half(), _rand(N, scale=0.1, seed=72)
        out = torch.zeros(M, N, dtype=torch.float16, device=DEV)
        gemm("STORE_H", a, w, M, N, K, bias=bias, act=1, out_h=out, out_h_ld=N)
        assert rel_err(out, F.gelu(a.float() @ w.float().t() + bias)) < 2e-3, (M, N, K)
    M, N, K = 30000, 768, 768
    a, w = _rand(M, K, seed=73).half(), _rand(N, K, scale=0.05, seed=74).half()
    bias, gamma, x = _rand(N, scale=0.1, seed=75), _rand(N, seed=76), _rand(M, N, seed=77)
    ref = x + gamma * (a.float() @ w.float().t() + bias)
    gemm("RESID_F", a, w, M, N, K, bias=bias, gamma=gamma, out_f=x, out_f_ld=N)
    assert rel_err(x, ref) < 1e-5
    # fp32 store (head linear-attention q, k, v) and the plain fp16 store without bias; rows beyond M stay untouched
    out_f = torch.full((M + 8, N), 7.0, device=DEV)
    gemm("STORE_F", a, w, M, N, K, out_f=out_f, out_f_ld=N)
    assert rel_err(out_f[:M], a.float() @ w.float().t()) < 1e-5
    assert bool((out_f[M:] == 7.0).all())
    out_h = torch.full((M + 8, N), 7.0, dtype=torch.float16, device=DEV)
    gemm("STORE_H", a, w, M, N, K, out_h=out_h, out_h_ld=N)
    assert rel_err(out_h[:M], a.float() @ w.float().t()) < 1e-3
    assert bool((out_h[M:] == 7.0).all())


def test_patch_gather_and_patch_epilogue():
    lib = _lib.load()
    n_img, H, W, D = 2, 70, 56, 384
    gh, gw = H // 14, W // 14
    N = gh * gw
    img = torch.rand(n_img, 3, H, W, device=DEV)
    wt = _rand(D, 3, 14, 14, scale=0.05, seed=27)
    posb, clspos = _rand(N, D, seed=28), _rand(D, seed=29)
    P = torch.zeros(n_img * N, 640, dtype=torch.float16, device=DEV)
    X = torch.zeros(n_img * (N + 1), D, device=DEV)
    _lib.check(lib.mk_op_patch_gather(_lib.ptr(img), _lib.ptr(P), n_img, H, W, 640, _lib.ptr(X), _lib.ptr(clspos), D, stream()))
    wp = F.pad(wt.reshape(D, 588), (0, 52)).half().contiguous()
    gemm("PATCH", P, wp, n_img * N, D, 640, aux=posb, tok_per_img=N, out_f=X, out_f_ld=D)
    ref = F.conv2d(img.half().float(), wt.half().float(), stride=14).flatten(2).transpose(1, 2) + posb[None]
    Xr = X.reshape(n_img, N + 1, D)
    assert rel_err(Xr[:, 1:], ref) < 1e-5
    assert rel_err(Xr[:, 0], clspos[None].expand(n_img, -1)) < 1e-7


def test_linear_attention():
    lib = _lib.load()
    n_img, G, gh, gw = 2, 4, 6, 5
    h2, w2 = gh + 2, gw + 2
    R = n_img * h2 * w2
    qkv = _rand(R, G * 384, seed=30)
    kv = torch.zeros(n_img, G, 8, 272, device=DEV)
    kvp = torch.zeros(n_img, G, (h2 * w2 + 31) // 32, 8, 272, device=DEV)
    msg = torch.zeros(R, G * 128, dtype=torch.float16, device=DEV)
    _lib.check(lib.mk_op_linattn(_lib.ptr(qkv), _lib.ptr(kvp), _lib.ptr(kv), _lib.ptr(msg), n_img, G, h2, w2, 1e-6, stream()))
    t = qkv.reshape(n_img, h2, w2, G, 3, 8, 16)[:, 1:-1, 1:-1].reshape(n_img, gh * gw, G, 3, 8, 16)
    for g in range(G):
        q, k, v = t[:, :, g, 0], t[:, :, g, 1], t[:, :, g, 2]
        Q, K = F.elu(q) + 1, F.elu(k) + 1
        L = gh * gw
        KV = torch.einsum("bshd,bshv->bhdv", K, v / L)
        Z = 1 / (torch.einsum("blhd,bhd->blh", Q, K.sum(1)) + 1e-6)
        ref = torch.einsum("blhd,bhdv,blh->blhv", Q, KV, Z) * L
        got = msg.reshape(n_img, h2, w2, G, 8, 16)[:, 1:-1, 1:-1, g].reshape(n_img, L, 8, 16)
        assert rel_err(got, ref) < 2e-3, g


def _matcher(d0, d1, s0, s1, T, dust, lean=False, pitch=None, bound=0.0):
    """The three launches of the matcher through the operator-level ABI: EPI_LSE (row + column partials from one pass
    over S), mk_op_matcher_reduce, EPI_DUAL."""
    lib = _lib.load()
    B, N, _ = d0.shape
    npad = (N + 127) // 128 * 128

    def split(d, role):
        hi = d.half()
        lo = (d - hi.float()).half()
        return torch.cat([hi, lo, hi] if role == 0 else [hi, hi, lo], dim=-1).reshape(B * N, 384).contiguous()

    a0, a1 = split(d0, 0), split(d1, 1)
    pr = torch.full((B, npad // 64, npad, 2), float("nan"), device=DEV)
    pc = torch.full((B, npad // 32, npad, 2), float("nan"), device=DEV)
    lr, lc = torch.full((B, npad), float("nan"), device=DEV), torch.full((B, npad), float("nan"), device=DEV)
    common = dict(groups=B, a_row_group_off=N, b_row_group_off=N, n_valid=N, inv_temp=1 / T, part_ld=npad)
    gemm("LSE", a0, a1, N, N, 384, part_row=pr, part_col=pc, lse_bound=bound, **common)
    _lib.check(lib.mk_op_matcher_reduce(_lib.ptr(pr), _lib.ptr(pc), _lib.ptr(dust), B, N, npad, _lib.ptr(lr), _lib.ptr(lc), stream()))
    # pitch None: the reference's contiguous [B, N, N] (st.global path); otherwise [B, N, pitch][:, :, :N] views: with
    # pitch % 4 == 0 the outputs leave through TMA tensor stores.  The pad columns must stay untouched (-7).
    def out():
        return torch.zeros(B, N, N, device=DEV) if pitch is None else torch.full((B, N, pitch), -7.0, device=DEV)[:, :, :N]
    fin = out()
    common["out_pitch"] = fin.stride(1)
    if lean:
        gemm("DUAL", a0, a1, N, N, 384, lse_r=lr, lse_c=lc, scr0=s0, scr1=s1, final_scores=fin, **common)
        return None, None, fin, lr, lc
    sc, kp = out(), out()
    gemm("DUAL", a0, a1, N, N, 384, lse_r=lr, lse_c=lc, scr0=s0, scr1=s1, scores=sc, kp_scores=kp, final_scores=fin, **common)
    if pitch is not None:
        # the pad stays untouched, except that a tensor store clips at 16-byte granularity: columns N .. round_up(N, 4)
        # may receive zeros (the values the kernel computes for columns beyond n_valid)
        n4 = (N + 3) // 4 * 4
        for t in ((fin,) if lean else (sc, kp, fin)):
            assert bool((t._base[:, :, n4:] == -7.0).all()), "pad columns were written"
            assert bool(((t._base[:, :, N:n4] == -7.0) | (t._base[:, :, N:n4] == 0.0)).all())
    return sc, kp, fin, lr, lc


def _dual_softmax_ref(d0, d1, T, dust):
    S = torch.einsum("bnd,bmd->bnm", d0.double(), d1.double()) / T
    if dust is None:
        return torch.softmax(S, 1) * torch.softmax(S, 2), S
    B, N, _ = S.shape
    full = torch.full((B, N + 1, N + 1), float(dust), dtype=torch.float64, device=S.device)
    full[:, :N, :N] = S
    return (torch.softmax(full, 1) * torch.softmax(full, 2))[:, :N, :N], S


@pytest.mark.parametrize("B,N", [(2, 300), (1, 1938), (3, 1938), (1, 128), (2, 129)])
def test_matcher_epilogues_vs_dual_softmax(B, N):
    """EPI_LSE + reduce + EPI_DUAL on split-fp16 descriptors == softmax(dim1)*softmax(dim2) with dustbin
    (N = 1938: the full BASELINE size; B = 3 gives 768 tiles, several waves; 128 / 129: tile-boundary cases)."""
    T = 0.1
    d0 = F.normalize(_rand(B, N, 128, seed=31), dim=-1)
    d1 = F.normalize(_rand(B, N, 128, seed=32), dim=-1)
    s0, s1 = torch.rand(B, N, device=DEV), torch.rand(B, N, device=DEV)
    dust = torch.tensor([1.0], device=DEV)
    sc, kp, fin, lr, lc = _matcher(d0, d1, s0, s1, T, dust)
    ref, S = _dual_softmax_ref(d0, d1, T, 1.0)
    # the two log-sum-exp vectors (log2 domain) of the dustbin-augmented logits
    lse_r = torch.logsumexp(torch.cat([S, torch.full_like(S[:, :, :1], 1.0)], 2), 2) / math.log(2)
    lse_c = torch.logsumexp(torch.cat([S, torch.full_like(S[:, :1, :], 1.0)], 1), 1) / math.log(2)
    assert float((lr[:, :N].double() - lse_r).abs().max()) < 1e-4 and float((lc[:, :N].double() - lse_c).abs().max()) < 1e-4
    assert rel_err(sc, ref) < 1e-4
    assert rel_err(kp, s0[:, :, None] * s1[:, None, :]) < 1e-6
    assert rel_err(fin, ref * s0[:, :, None].double() * s1[:, None, :].double()) < 1e-4
    # lean mode (scores / kp_scores NULL): final_scores is bit-identical
    _, _, fin2, _, _ = _matcher(d0, d1, s0, s1, T, dust, lean=True)
    assert torch.equal(fin, fin2)
    # normalised descriptors: the fixed-shift partials (one exponential per cell) give the same vectors
    sc5, _, fin5, lr5, lc5 = _matcher(d0, d1, s0, s1, T, dust, bound=1.001)
    assert float((lr5[:, :N] - lr[:, :N]).abs().max()) < 1e-5 and float((lc5[:, :N] - lc[:, :N]).abs().max()) < 1e-5
    assert rel_err(sc5, ref) < 1e-4 and rel_err(fin5, fin) < 1e-5
    # padded row pitch (16-byte aligned rows) -> TMA tensor stores: bit-identical to the st.global path, pad untouched
    pitch = (N + 31) // 32 * 32
    sc3, kp3, fin3, _, _ = _matcher(d0, d1, s0, s1, T, dust, pitch=pitch)
    assert torch.equal(sc3, sc) and torch.equal(kp3, kp) and torch.equal(fin3, fin)
    _, _, fin4, _, _ = _matcher(d0, d1, s0, s1, T, dust, lean=True, pitch=pitch + 4)
    assert torch.equal(fin4, fin)


@pytest.mark.parametrize("scale,T,use_dust", [(6.0, 0.1, True), (6.0, 0.1, False), (1.0, 0.01, False), (40.0, 1.0, True)])
def test_matcher_wide_logit_range(scale, T, use_dust):
    """Un-normalised descriptors / small temperatures (NORM_DSC: False, TEMPERATURE): logits span thousands, far beyond
    what one global shift can hold in fp32 (exp underflows below -87).  The reference's softmaxes subtract true row /
    column maxima (F.softmax); so do the epilogues: every output is finite and matches fp64 wherever it is not negligible."""
    B, N = 2, 500
    d0, d1 = _rand(B, N, 128, seed=41) * scale, _rand(B, N, 128, seed=42) * scale
    d0[0, 7] *= 3.0                                       # one dominant row
    d1[1, 9] *= 3.0                                       # one dominant column
    s0, s1 = torch.rand(B, N, device=DEV), torch.rand(B, N, device=DEV)
    dust = torch.tensor([1.0], device=DEV) if use_dust else None
    sc, kp, fin, lr, lc = _matcher(d0, d1, s0, s1, T, dust)
    assert bool(torch.isfinite(sc).all()) and bool(torch.isfinite(fin).all()) and bool(torch.isfinite(lr[:, :N]).all())
    # split-fp16 operands carry ~2^-22 relative error per product term: compare against the SAME rounded operands in fp64
    def rounded(d):
        hi = d.half().double()
        return hi + (d.double() - hi).half().double()
    ref, S = _dual_softmax_ref(rounded(d0), rounded(d1), T, 1.0 if use_dust else None)
    assert float(S.abs().max()) > 500                     # the regime this test is about
    # absolute error of a logit ~ |s| * 2^-21 -> relative error of exp(2s - ...) ~ 2 * that
    tol = 4 * float(S.abs().max()) * 2.0 ** -21 + 1e-4
    big = ref > 1e-6
    assert float(((sc.double() - ref).abs() / ref.clamp_min(1e-300))[big].max()) < tol
    assert float((sc.double() - ref).abs().max()) < tol
    if not use_dust:                                      # without a dustbin every row / column of a softmax sums to <= 1 and the maxima carry mass
        assert float(sc.sum(-1).max()) <= 1 + 4 * tol and float(sc.max()) > 0.1


def _philox4x32_7(c0, c1, c2, c3, seed):
    """numpy restatement of the device generator (ransac.cu Philox): counters are uint32 arrays."""
    import numpy as np
    M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
    a, b = seed & 0xffffffff, seed >> 32
    c0, c1, c2, c3 = (np.asarray(x, dtype=np.uint32).copy() for x in np.broadcast_arrays(c0, c1, c2, c3))
    for _ in range(7):
        p0, p1 = M0 * c0.astype(np.uint64), M1 * c2.astype(np.uint64)
        hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), (p0 & np.uint64(0xffffffff)).astype(np.uint32)
        hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), (p1 & np.uint64(0xffffffff)).astype(np.uint32)
        c0, c1, c2, c3 = hi1 ^ c1 ^ np.uint32(a), lo1, hi0 ^ c3 ^ np.uint32(b), lo0
        a, b = (a + 0x9E3779B9) & 0xffffffff, (b + 0xBB67AE85) & 0xffffffff
    return c0, c1, c2, c3


@pytest.mark.parametrize("mode,N", [("spread", 120), ("few_nonzero", 120), ("spread", 121)])
def test_outer_sampler_is_topk_of_the_race(mode, N):
    """The kernel's draw must be exactly 'the n_s largest p / Exp(1) keys' of its own counter-based noise: the host
    regenerates every cell's key for a stream (numpy Philox) and takes the top n_s by brute force.  Device log / divide
    are approximate, so a handful of keys at the boundary may differ."""
    import numpy as np
    lib = _lib.load()
    B, IM, n_s, seed = 2, 10, 2048, 0x1234567887654321      # N = 121: N*N is not a multiple of 4 (scalar load path)
    cells = N * N
    g = torch.Generator().manual_seed(3)
    p = torch.rand(B, cells, generator=g) ** 6 * 1e-3
    if mode == "few_nonzero":
        p[:, torch.randperm(cells, generator=g)[: cells - 2100]] = 0      # 2100 nonzero cells: every one is a candidate
    ws_bytes = lib.mk_op_sample_workspace_bytes(B, IM)
    ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=DEV)
    idx = torch.full((B * IM, n_s), -1, dtype=torch.int32, device=DEV)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    _lib.check(lib.mk_op_sample(_lib.ptr(p.to(DEV)), B, N, 0, IM, n_s, seed, _lib.ptr(ws), ws_bytes, _lib.ptr(idx), _lib.ptr(status), stream()))
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    idx = idx.cpu().numpy().reshape(B, IM, n_s)
    e = np.arange(cells, dtype=np.uint32)
    for b in range(B):
        pb = p[b].numpy().astype(np.float64)
        for s in (0, 7, 9):
            sg, j = divmod(s, 8)
            w = _philox4x32_7(e, np.uint32(0x5bd1e995), np.uint32(sg), np.uint32(b), seed)[j >> 1]
            prefix = (w >> np.uint32((j & 1) * 16)) & np.uint32(0xffff)
            low = _philox4x32_7(e, np.uint32(0x2545F491), np.uint32(s), np.uint32(b), seed)[0]
            u = (prefix.astype(np.float64) + (low.astype(np.float64) + 0.5) * 2.0 ** -32) * 2.0 ** -16
            key = np.where(pb > 0, pb / -np.log1p(-np.minimum(u, 0.99999994)), 0.0)
            want = np.argsort(-key, kind="stable")[:n_s]
            got = idx[b, s]
            assert len(set(got.tolist())) == n_s
            missing = set(want.tolist()) - set(got.tolist())
            assert len(missing) <= 3, (mode, b, s, len(missing))
            assert np.all(got[1:] > got[:-1])   # canonical order of a draw: ascending cell index


@pytest.mark.parametrize("N,pitch", [(150, 160), (150, 152), (151, 153), (149, 149), (1938, 1952)])
def test_outer_sampler_does_not_depend_on_the_row_pitch(N, pitch):
    """final_scores as a padded-pitch view ([N, pitch][:, :N], what the matcher's TMA path writes; 16-byte 4-cell slots
    per row), as an odd pitch (scalar path) and contiguous (flat 16-byte loads when N*N % 4 == 0): the logical cell index
    does not depend on the layout, so the same seed gives the identical draw; garbage in the pad columns is never read."""
    lib = _lib.load()
    B, IM, n_s = 2, 8, 2048
    g = torch.Generator().manual_seed(3)
    p = (torch.rand(B, N, N, generator=g) * 1e-6).to(DEV)
    p[p < 2e-7] = 0
    padded = torch.full((B, N, pitch), 1e3, device=DEV)           # a pad that would dominate every draw if it were read
    padded[:, :, :N] = p
    ws_bytes = lib.mk_op_sample_workspace_bytes(B, IM)
    ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=DEV)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    out = []
    for t, pt in ((p.contiguous(), 0), (padded, pitch)):
        idx = torch.full((B * IM, n_s), -1, dtype=torch.int32, device=DEV)
        _lib.check(lib.mk_op_sample(_lib.ptr(t), B, N, pt, IM, n_s, 4321, _lib.ptr(ws), ws_bytes, _lib.ptr(idx), _lib.ptr(status), stream()))
        torch.cuda.synchronize()
        assert int(status.item()) == 0
        out.append(idx.clone())
    assert torch.equal(out[0], out[1])
    assert int(out[0].max()) < N * N and float(p.reshape(B, -1)[0][out[0][0].long()].min()) > 0


def test_outer_sampler_properties():
    """Exponential-race sampler: distinct cells, never a zero-probability cell, heavy cells (almost) always
    drawn, light cells drawn in proportion to their mass."""
    lib = _lib.load()
    B, N, IM, n_s = 1, 150, 8, 2048
    cells = N * N
    g = torch.Generator().manual_seed(0)
    p = torch.rand(B, cells, generator=g) * 1e-6
    zero = torch.rand(B, cells, generator=g) < 0.3
    p[zero] = 0
    heavy = torch.randperm(cells, generator=g)[:500]
    p[0, heavy] = 1.0
    p = p.to(DEV)
    ws_bytes = lib.mk_op_sample_workspace_bytes(B, IM)
    ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=DEV)
    idx = torch.full((B * IM, n_s), -1, dtype=torch.int32, device=DEV)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    _lib.check(lib.mk_op_sample(_lib.ptr(p), B, N, 0, IM, n_s, 1234, _lib.ptr(ws), ws_bytes, _lib.ptr(idx), _lib.ptr(status), stream()))
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    idx = idx.long().cpu()
    pc = p.cpu()[0]
    heavy_set = set(heavy.tolist())
    for s in range(IM):
        row = idx[s]
        assert row.min() >= 0 and row.max() < cells
        assert len(set(row.tolist())) == n_s                      # without replacement
        assert float(pc[row].min()) > 0                           # zero cells are never drawn
        assert len(heavy_set & set(row.tolist())) == 500          # P(miss) ~ 1e-6 * cells / 1 per heavy cell
    # streams differ from each other
    assert len(set(idx[0].tolist()) & set(idx[1].tolist())) < n_s
    # light cells: inclusion frequency ~ proportional to p (two mass classes, ratio 2)
    p2 = torch.full((1, cells), 1e-6)
    p2[0, : cells // 2] = 2e-6
    p2 = p2.to(DEV)
    _lib.check(lib.mk_op_sample(_lib.ptr(p2), 1, N, 0, IM, n_s, 99, _lib.ptr(ws), ws_bytes, _lib.ptr(idx := torch.zeros(IM, n_s, dtype=torch.int32, device=DEV)), _lib.ptr(status), stream()))
    torch.cuda.synchronize()
    frac_heavy = float((idx.long() < cells // 2).float().mean())
    assert abs(frac_heavy - 2 / 3) < 0.03, frac_heavy
    # same seed -> same draw (counter-based generator), different seed -> different draw
    idx_b = torch.zeros(IM, n_s, dtype=torch.int32, device=DEV)
    _lib.check(lib.mk_op_sample(_lib.ptr(p2), 1, N, 0, IM, n_s, 99, _lib.ptr(ws), ws_bytes, _lib.ptr(idx_b), _lib.ptr(status), stream()))
    torch.cuda.synchronize()
    assert torch.equal(idx, idx_b)
