"""Host side of the CUDA DINOv2 backbone (mickey_b200/dinov2.py, mk_backbone_features): the module's parameter tree
against the reference's, every rejected input, the C argument checks and the pack_backbone split.  No GPU needed."""
import ctypes as C

import pytest
import torch

from mickey_b200 import _lib
from mickey_b200.config import VARIANTS, mickey_cfg
from mickey_b200.dinov2 import DinoVisionTransformer
from mickey_b200.engine import KPAD, pack_backbone, pack_weights
from mickey_b200.weights import BACKBONE, synthetic_state_dict
from oracle import ref_harness


def _shapes(sd):
    return {k: tuple(v.shape) for k, v in sd.items()}


@pytest.fixture(scope="module")
def synthetic():
    return {v: synthetic_state_dict(mickey_cfg(v, 2, 8), seed=1) for v in VARIANTS}


@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_state_dict_matches_the_synthetic_backbone(variant, synthetic):
    m = DinoVisionTransformer(variant)
    want = {k[len(BACKBONE):]: v for k, v in synthetic[variant].items() if k.startswith(BACKBONE)}
    assert _shapes(m.state_dict()) == _shapes(want)
    assert all(not p.requires_grad for p in m.parameters())
    m.load_state_dict(want, strict=True)
    assert m._packed is None                        # packing waits for the first forward_features
    assert torch.equal(m.blocks[3].mlp.fc2.weight, want["blocks.3.mlp.fc2.weight"])


@pytest.mark.skipif(not ref_harness.available(), reason="reference tree not present")
@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_state_dict_matches_the_live_reference(variant, synthetic):
    cfg = mickey_cfg(variant, 2, 8)
    ref = ref_harness.build_reference_model(cfg, synthetic[variant], variant=variant)   # weights supplied: no download
    ref_vit = ref.compute_matches.extractor.dinov2_vitl14
    ours = DinoVisionTransformer(variant)
    assert list(ours.state_dict()) == list(ref_vit.state_dict())
    assert _shapes(ours.state_dict()) == _shapes(ref_vit.state_dict())
    assert [n for n, _ in ours.named_parameters()] == [n for n, _ in ref_vit.named_parameters()]


def _x(*shape, dtype=torch.float16):
    return torch.zeros(*shape, dtype=dtype)


@pytest.mark.parametrize("call,exc,match", [
    (lambda m: m.forward_features(_x(1, 3, 98, 98), masks=torch.zeros(1, 49, dtype=torch.bool)), NotImplementedError, "masks"),
    (lambda m: m.forward_features([_x(1, 3, 98, 98)]), NotImplementedError, "list"),
    (lambda m: m.forward_features_list([_x(1, 3, 98, 98)], [None]), NotImplementedError, "list"),
    (lambda m: m.forward_features(_x(1, 3, 98, 98, dtype=torch.float32)), ValueError, "fp32 backbone"),
    (lambda m: m.forward_features(_x(1, 3, 98, 98, dtype=torch.bfloat16)), ValueError, "float16"),
    (lambda m: m.forward_features(_x(1, 3, 98, 99)), ValueError, "multiples of the patch size"),
    (lambda m: m.forward_features(_x(1, 3, 100, 98)), ValueError, "multiples of the patch size"),
    (lambda m: m.forward_features(_x(1, 3, 84, 98)), ValueError, "at least 98"),
    (lambda m: m.forward_features(_x(1, 4, 98, 98)), ValueError, r"\[B, 3, H, W\]"),
    (lambda m: m.forward_features(_x(3, 98, 98)), ValueError, r"\[B, 3, H, W\]"),
    (lambda m: m.forward_features(_x(0, 3, 98, 98)), ValueError, "at least one image"),
    (lambda m: m.forward_features(_x(1, 3, 98, 98)), ValueError, "CUDA"),
    (lambda m: m.forward_features(None), ValueError, "torch tensor"),
    (lambda m: m(_x(1, 3, 98, 98)), NotImplementedError, "forward_features"),
], ids=["masks", "list", "forward_features_list", "fp32", "bf16", "W", "H", "small", "channels", "3d", "empty", "cpu",
        "not_a_tensor", "forward"])
def test_python_rejections_come_before_any_launch(call, exc, match):
    m = DinoVisionTransformer("vits")
    with pytest.raises(exc, match=match):
        call(m)
    assert m._packed is None                        # no handle, no packing, nothing launched


def test_c_arguments_are_rejected_before_any_launch():
    lib = _lib.load()
    p = C.c_void_p(256)                     # never dereferenced: every call below fails its argument check first
    ws = 1 << 40

    def call(h=p, img=p, n=2, H=98, W=98, out=p, w=p, wsb=ws):
        return lib.mk_backbone_features(h, img, n, H, W, out, w, wsb, None)

    for rc in (call(h=None), call(img=None), call(out=None), call(w=None), call(n=0), call(n=-3), call(H=99), call(W=112 + 7),
               call(H=84), call(W=70), call(H=0, W=0)):
        assert rc == -1
    assert b"mk_backbone_features" in lib.mk_last_error()
    for args in ((None, 2, 98, 98), (p, 0, 98, 98), (p, 2, 99, 98), (p, 2, 98, 84)):
        assert lib.mk_backbone_ws_bytes(*args) == -1


def test_pack_weights_is_pack_backbone_plus_the_heads():
    """The split leaves pack_weights' output unchanged: the backbone's entries are pack_backbone's, in the same order and
    first, and each one is the state-dict tensor in the kernels' layout."""
    cfg = mickey_cfg("vits", 2, 8)
    sd = synthetic_state_dict(cfg, seed=2)
    full = pack_weights(sd, cfg, "cpu")
    bb = pack_backbone(sd, "vits", "cpu")
    assert list(full)[:len(bb)] == list(bb)
    for k, v in bb.items():
        assert full[k].dtype == v.dtype and torch.equal(full[k], v), k
    D, depth, _ = VARIANTS["vits"]
    assert len(bb) == 1 + 14 * depth + 2
    pw = sd[BACKBONE + "patch_embed.proj.weight"].reshape(D, 588)
    assert torch.equal(bb["patch.w"][:, :588], pw.half()) and not bb["patch.w"][:, 588:].any()
    assert bb["patch.w"].shape == (D, KPAD)
    names = {"ln1.w": "norm1.weight", "ln1.b": "norm1.bias", "ln2.w": "norm2.weight", "ln2.b": "norm2.bias",
             "qkv.w": "attn.qkv.weight", "qkv.b": "attn.qkv.bias", "proj.w": "attn.proj.weight", "proj.b": "attn.proj.bias",
             "fc1.w": "mlp.fc1.weight", "fc1.b": "mlp.fc1.bias", "fc2.w": "mlp.fc2.weight", "fc2.b": "mlp.fc2.bias",
             "ls1": "ls1.gamma", "ls2": "ls2.gamma"}
    for i in (0, depth - 1):
        for q, r in names.items():
            got, want = bb[f"blk{i}.{q}"], sd[f"{BACKBONE}blocks.{i}.{r}"]
            dt = torch.float16 if q.endswith(".w") and not q.startswith("ln") else torch.float32
            assert got.dtype == dt and torch.equal(got, want.to(dt)), (i, q)
    assert torch.equal(bb["norm.w"], sd[BACKBONE + "norm.weight"]) and torch.equal(bb["norm.b"], sd[BACKBONE + "norm.bias"])
    # the module's own tree (no prefix) packs to the same tensors
    m = DinoVisionTransformer("vits")
    m.load_state_dict({k[len(BACKBONE):]: v for k, v in sd.items() if k.startswith(BACKBONE)})
    mine = pack_backbone(dict(m.named_parameters()), "vits", "cpu", prefix="")
    assert list(mine) == list(bb) and all(torch.equal(mine[k], bb[k]) for k in bb)
