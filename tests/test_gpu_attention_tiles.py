"""The wgmma attention kernel's tiling: persistent CTAs that run several (image, head, 192-query) tiles each, with the
TMA ring's stage and phase carried from tile to tile, and an output that leaves through a TMA store clipped at T in
every image."""
import pytest
import torch

from mickey_b200 import _lib
from tests.common import rel_err
from tests.gpu_util import stream

pytestmark = pytest.mark.gpu
DEV = "cuda"
TC = 1          # impl 1: the wgmma / TMA kernel


def _qkv(n_img, T, heads, seed, scale=1.5):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(n_img * T, 3 * heads * 64, generator=g) * scale).half().to(DEV)


def _attention(qkv, out, n_img, T, heads):
    lib = _lib.load()
    _lib.check(lib.mk_op_attention(_lib.ptr(qkv), _lib.ptr(out), n_img, T, heads * 64, heads, TC, stream()))


def _ref(qkv, n_img, T, heads):
    q, k, v = qkv.float().reshape(n_img, T, 3, heads, 64).permute(2, 0, 3, 1, 4)
    return (torch.softmax(q @ k.transpose(-1, -2) * 0.125, -1) @ v).transpose(1, 2).reshape(n_img * T, heads * 64)


@pytest.mark.parametrize("n_img,T,heads", [(16, 1939, 12),     # 11 x 12 x 16 = 2112 tiles: 16 per CTA on 132 SMs
                                           (3, 1939, 6),       # 198 tiles: some CTAs run two
                                           (5, 193, 12),       # one valid row in every second 192-query tile
                                           (7, 64, 6)])
def test_batched_equals_per_image(n_img, T, heads):
    """A multi-image, multi-head call is byte-equal to one call per image on the same rows."""
    D = heads * 64
    qkv = _qkv(n_img, T, heads, seed=100 + T)
    out = torch.zeros(n_img * T, D, dtype=torch.float16, device=DEV)
    _attention(qkv, out, n_img, T, heads)
    for i in range(n_img):
        one = torch.zeros(T, D, dtype=torch.float16, device=DEV)
        _attention(qkv[i * T:(i + 1) * T].contiguous(), one, 1, T, heads)
        assert torch.equal(out[i * T:(i + 1) * T], one), i


@pytest.mark.parametrize("T", [1, 64, 193, 1939])
def test_rows_past_the_output_are_untouched(T):
    """Every image is clipped at T: sentinel rows after the n_img * T output rows keep their bytes, and every image's
    rows match torch."""
    n_img, heads = 3, 6
    D = heads * 64
    qkv = _qkv(n_img, T, heads, seed=200 + T)
    pad = 256
    buf = torch.full(((n_img * T + pad), D), -7.25, dtype=torch.float16, device=DEV)
    _attention(qkv, buf, n_img, T, heads)
    assert bool((buf[n_img * T:] == -7.25).all())
    ref = _ref(qkv, n_img, T, heads)
    for i in range(n_img):
        assert rel_err(buf[i * T:(i + 1) * T], ref[i * T:(i + 1) * T]) < 2e-3, i


def test_deterministic():
    n_img, T, heads = 16, 1939, 12
    qkv = _qkv(n_img, T, heads, seed=300)
    a = torch.empty(n_img * T, heads * 64, dtype=torch.float16, device=DEV)
    b = torch.empty_like(a)
    _attention(qkv, a, n_img, T, heads)
    _attention(qkv, b, n_img, T, heads)
    assert torch.equal(a, b)
