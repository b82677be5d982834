"""The CUDA DINOv2 backbone for training (mickey_b200/dinov2.py, mk_backbone_features) on the GPU, with seeded synthetic
weights: the channel-major final norm element by element against fp64 from the workspace's own residual stream, bit
equality with the inference path's X and F, the whole backbone against the fp32 oracle, the drop-in's tensor semantics,
batch invariance and the weight lifecycle."""
import ctypes as C

import pytest
import torch

from mickey_b200 import _lib
from mickey_b200.config import VARIANTS, mickey_cfg
from mickey_b200.dinov2 import DinoVisionTransformer
from mickey_b200.engine import Engine
from mickey_b200.weights import BACKBONE, synthetic_state_dict
from oracle import mickey_oracle as mo
from tests import elementwise as ew

pytestmark = pytest.mark.gpu
DEV = "cuda"
FP16_RULE = 1.5              # DESIGN §2: at most 1.5x the error of the reference's fp16 backbone


def _full_sd(variant):
    return synthetic_state_dict(mickey_cfg(variant, 2, 8), seed=3)


def _backbone_sd(sd):
    return {k[len(BACKBONE):]: v for k, v in sd.items() if k.startswith(BACKBONE)}


_SD = {}


def sd_of(variant):
    if variant not in _SD:
        _SD[variant] = _full_sd(variant)
    return _SD[variant]


def module(variant, sd=None):
    m = DinoVisionTransformer(variant)
    m.load_state_dict(_backbone_sd(sd if sd is not None else sd_of(variant)), strict=True)
    return m.to(DEV)


def images(B, H, W, seed=11):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, 3, H, W, generator=g).to(DEV, torch.float16)


@pytest.fixture(scope="module")
def vitl():
    return module("vitl")


# ---------------------------------------------------------------------------------------------------------------
# 1. the final norm, element by element, from the workspace's own X
# ---------------------------------------------------------------------------------------------------------------
CASES = {"vitl_720x540": ("vitl", 8, 714, 532), "vitl_warmup": ("vitl", 24, 476, 350),
         "vits_min": ("vits", 2, 98, 98), "vits_t2304": ("vits", 2, 658, 686)}


@pytest.mark.parametrize("case", list(CASES))
def test_final_norm_elementwise(case, vitl):
    variant, B, H, W = CASES[case]
    m = vitl if variant == "vitl" else module(variant)
    D = VARIANTS[variant][0]
    gh, gw = H // 14, W // 14
    N, T = gh * gw, gh * gw + 1
    got = m.forward_features(images(B, H, W))["x_norm_patchtokens"]
    torch.cuda.synchronize()
    assert got.shape == (B, N, D) and got.dtype == torch.float32
    X = m.ws_view("X", torch.float32, (B, T, D)).double()
    w, b = m.norm.weight.double(), m.norm.bias.double()
    ref, bound = ew.ln_bound(X[:, 1:], 0.0, w, b, 1e-6)
    bound = bound + ew.out_rounding(ref, False)
    with_cls, _ = ew.ln_bound(X[0:1, :N], 0.0, w, b, 1e-6)
    muts = [ew.Mutation("token of the neighbouring image", (0, slice(7, 8)), ref[1, 7:8]),
            ew.Mutation("cls row included (tokens shifted by one)", (0,), with_cls[0]),
            ew.Mutation("token-major instead of channel-major", (0,), ref[0].reshape(-1).reshape(D, N).t()),
            ew.Mutation("32 channels of the next token", (0, slice(7, 8), slice(32, 64)), ref[0, 8:9, 32:64])]
    where = ew.Where(lambda idx: (int(idx[0]) * N + int(idx[1]), 0, int(idx[2])), ew.Rows("patches", N))
    ratio = ew.check(f"{case} out", got, ref, bound, where, muts)
    ew.record("backbone_final_norm", case, ratio)
    print(f"\n[{case}] final norm (channel-major fp32): max err/bound {ratio:.3g}, {len(muts)} mutations rejected")


# ---------------------------------------------------------------------------------------------------------------
# 2. the same X and, rounded to fp16, the same F as the inference path
# ---------------------------------------------------------------------------------------------------------------
def test_bit_equal_to_the_inference_path(vitl):
    n, H, W = 16, 714, 532
    D, N, T = 1024, 1938, 1939
    x = images(n, H, W, seed=5)
    out = vitl.forward_features(x)["x_norm_patchtokens"]
    X_bb = vitl.ws_view("X", torch.float32, (n, T, D)).clone()
    eng = Engine(mickey_cfg("vitl", 2, 8), "cuda:0")
    eng.load_state_dict(sd_of("vitl"))
    eng.extract(x.float())
    torch.cuda.synchronize()
    X_inf = eng.ws_view("X", torch.float32, (n, T, D))
    Fm = eng.ws_view("F", torch.float16, (n, H // 14 + 2, W // 14 + 2, D))
    assert torch.equal(X_bb, X_inf)
    assert torch.equal(out.half(), Fm[:, 1:-1, 1:-1].reshape(n, N, D))


# ---------------------------------------------------------------------------------------------------------------
# 3. end to end against the oracle (fp32), next to the reference's fp16 backbone
# ---------------------------------------------------------------------------------------------------------------
def test_end_to_end_against_the_fp32_oracle(vitl):
    B, H, W = 8, 714, 532
    x = images(B, H, W, seed=7)
    got = vitl.forward_features(x)["x_norm_patchtokens"]
    sd = {k: v.to(DEV) for k, v in sd_of("vitl").items() if k.startswith(BACKBONE)}
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            ref32 = mo.vit_forward_features(sd, x.float())
            ref16 = mo.vit_forward_features({k: v.half() for k, v in sd.items()}, x).float()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    rel = lambda a: float((a.double() - ref32.double()).norm() / ref32.double().norm())   # noqa: E731
    e_ours, e_16 = rel(got), rel(ref16)
    ew.record("backbone_rel_frobenius", "vitl_720x540_ours", e_ours)
    ew.record("backbone_rel_frobenius", "vitl_720x540_oracle_fp16", e_16)
    print(f"\nViT-L B=8 714x532: relative Frobenius error vs fp32 oracle: ours {e_ours:.3e}, fp16 oracle {e_16:.3e}")
    assert e_ours <= FP16_RULE * e_16, (e_ours, e_16)


# ---------------------------------------------------------------------------------------------------------------
# 4. drop-in semantics
# ---------------------------------------------------------------------------------------------------------------
def test_dropin_tensor_semantics():
    m = module("vits")
    B, C_, H, W = 2, 384, 720, 540
    big = images(B, H, W, seed=9)
    x = big[:, :, :14 * (H // 14), :14 * (W // 14)]          # the extractor's crop (mickey_extractor.py:46)
    h, w = H // 14, W // 14
    raw = m.forward_features(x.to(torch.float16))["x_norm_patchtokens"]
    feats = raw.permute(0, 2, 1).reshape(B, C_, h, w).float()  # mickey_extractor.py:49-51
    assert feats.is_contiguous() and feats.dtype == torch.float32 and feats.shape == (B, C_, h, w)
    assert feats.data_ptr() == raw.data_ptr() and raw.untyped_storage().nbytes() == B * C_ * h * w * 4
    for grad in (True, False):
        with torch.set_grad_enabled(grad):
            assert not m.forward_features(x)["x_norm_patchtokens"].requires_grad
    keep = raw.clone()
    other = m.forward_features(images(B, 14 * h, 14 * w, seed=10))["x_norm_patchtokens"]
    s0, s1 = raw.data_ptr(), other.data_ptr()
    n = raw.untyped_storage().nbytes()
    assert s0 + n <= s1 or s1 + n <= s0, "two calls alias"
    torch.cuda.synchronize()
    assert torch.equal(raw, keep), "the first call's features changed after the second call"
    assert not x.is_contiguous()
    assert torch.equal(m.forward_features(x)["x_norm_patchtokens"], m.forward_features(x.contiguous())["x_norm_patchtokens"])


# ---------------------------------------------------------------------------------------------------------------
# 5. batch invariance and determinism
# ---------------------------------------------------------------------------------------------------------------
def test_batch_invariance_and_determinism(vitl):
    x = images(24, 476, 350, seed=13)
    full = vitl.forward_features(x)["x_norm_patchtokens"]
    again = vitl.forward_features(x)["x_norm_patchtokens"]
    assert torch.equal(full, again)
    for k in (0, 13, 23):
        alone = vitl.forward_features(x[k:k + 1])["x_norm_patchtokens"]
        assert torch.equal(alone[0], full[k]), k


# ---------------------------------------------------------------------------------------------------------------
# 6. weight lifecycle
# ---------------------------------------------------------------------------------------------------------------
def test_weight_lifecycle():
    x = images(2, 224, 196, seed=15)
    m = module("vits")
    m.forward_features(x)
    sd_new = synthetic_state_dict(mickey_cfg("vits", 2, 8), seed=4)
    m.load_state_dict(_backbone_sd(sd_new))
    fresh = module("vits", sd_new)
    after = m.forward_features(x)["x_norm_patchtokens"]
    assert torch.equal(after, fresh.forward_features(x)["x_norm_patchtokens"])
    assert not torch.equal(after, module("vits").forward_features(x)["x_norm_patchtokens"])
    # the reference's FLOAT16 cast: fp16 parameters pack with their fp16 values
    half = module("vits").to(torch.float16)
    assert all(p.dtype == torch.float16 for p in half.parameters())
    rounded = module("vits", {k: (v.half().float() if k.startswith(BACKBONE) else v) for k, v in sd_of("vits").items()})
    got = half.forward_features(x)["x_norm_patchtokens"]
    assert torch.equal(got, rounded.forward_features(x)["x_norm_patchtokens"])
    assert not torch.equal(got, module("vits").forward_features(x)["x_norm_patchtokens"])
    # train() / eval() change nothing
    assert torch.equal(half.train().forward_features(x)["x_norm_patchtokens"], half.eval().forward_features(x)["x_norm_patchtokens"])


def test_streams():
    """A call on another stream than the last one waits for it: the shared workspace is never raced."""
    m = module("vits")
    x0, x1 = images(4, 476, 350, seed=21), images(4, 476, 350, seed=22)
    ref0 = m.forward_features(x0)["x_norm_patchtokens"].clone()
    ref1 = m.forward_features(x1)["x_norm_patchtokens"].clone()
    s = torch.cuda.Stream()
    a = m.forward_features(x0)["x_norm_patchtokens"]
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        b = m.forward_features(x1)["x_norm_patchtokens"]
    torch.cuda.current_stream().wait_stream(s)
    c = m.forward_features(x0)["x_norm_patchtokens"]
    torch.cuda.synchronize()
    assert torch.equal(a, ref0) and torch.equal(b, ref1) and torch.equal(c, ref0)


# ---------------------------------------------------------------------------------------------------------------
# C ABI on a live handle: the workspace is the six backbone buffers, and the handle-dependent rejections
# ---------------------------------------------------------------------------------------------------------------
def _handle(variant):
    lib = _lib.load()
    D, depth, heads = VARIANTS[variant]
    cfg = _lib.MkConfig()
    cfg.embed_dim, cfg.depth, cfg.heads, cfg.down_factor = D, depth, heads, 14
    h = C.c_void_p()
    _lib.check(lib.mk_create(0, C.byref(cfg), C.byref(h)), "mk_create")
    return lib, h


@pytest.mark.parametrize("variant,n,H,W", [("vitl", 8, 714, 532), ("vitl", 24, 476, 350), ("vits", 3, 98, 98)])
def test_backbone_workspace_is_the_six_buffers(variant, n, H, W):
    lib, h = _handle(variant)
    try:
        D = VARIANTS[variant][0]
        N = (H // 14) * (W // 14)
        M = n * (N + 1)
        a = lambda b: (b + 255) // 256 * 256                                    # noqa: E731
        sizes = [n * N * 640 * 2, M * D * 4, M * D * 2, M * 3 * D * 2, M * D * 2, M * 4 * D * 2]
        got = lib.mk_backbone_ws_bytes(h, n, H, W)
        print(f"\n{variant} n={n} {H}x{W}: backbone workspace {got / 1e9:.3f} GB, "
              f"extraction workspace {lib.mk_workspace_bytes_for(h, n, 0, H, W) / 1e9:.3f} GB")
        assert got == sum(a(s) for s in sizes)
        assert got < lib.mk_workspace_bytes_for(h, n, 0, H, W)
    finally:
        lib.mk_destroy(h)


def test_handle_dependent_rejections():
    lib, h = _handle("vits")
    p = C.c_void_p(256)                     # never dereferenced: every call below fails its check first
    try:
        need = lib.mk_backbone_ws_bytes(h, 2, 98, 98)
        call = lambda H=98, W=98, wsb=need: lib.mk_backbone_features(h, p, 2, H, W, p, p, wsb, None)   # noqa: E731
        assert call() == -1 and b"not finalized" in lib.mk_last_error()
        _lib.check(lib.mk_finalize(h, 98, 98), "mk_finalize")
        assert call(H=112) == -1 and b"geometry" in lib.mk_last_error()
        assert call(wsb=need - 1) == -1 and b"workspace too small" in lib.mk_last_error()
    finally:
        lib.mk_destroy(h)
