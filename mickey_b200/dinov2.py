"""MicKey's frozen DINOv2 backbone in CUDA: a drop-in for the reference's DinoVisionTransformer in a training model.

The reference freezes the backbone (mickey_extractor.py:27-28) and runs it under torch.no_grad (:48-51), so training
needs its forward pass only.  `DinoVisionTransformer(variant)` has the reference's parameters, names and shapes
(dinov2.py:95-152 with block_chunks = 0), every one with requires_grad=False, so state dicts and checkpoints load and
save unchanged and optimisers skip them.  `forward_features` runs the patch embedding, every block and the final norm
in libmickey_b200.so (mk_backbone_features, the kernels of the inference engine) and hands back the features in the
layout the extractor turns into the heads' input.  INTEGRATION.md shows the swap in a training model.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.nn as nn

from . import _lib
from .config import VARIANTS
from .engine import PATCH, pack_backbone, position_tables, raw_positions

POS_GRID = 37               # img_size 518 / patch 14 (mickey_extractor.py:18-22)
MIN_SIDE = 7 * PATCH        # the smallest image the engine accepts
MAX_GEOMETRIES = 4          # image sizes whose position tables are kept at once


class _Params(nn.Module):
    """A node of the parameter tree: holds frozen parameters under the reference's names."""

    def __init__(self, **shapes):
        super().__init__()
        for name, shape in shapes.items():
            self.register_parameter(name, nn.Parameter(torch.zeros(shape), requires_grad=False))


class _Block(nn.Module):
    def __init__(self, D):
        super().__init__()
        self.norm1 = _Params(weight=(D,), bias=(D,))
        self.attn = nn.Module()
        self.attn.qkv = _Params(weight=(3 * D, D), bias=(3 * D,))
        self.attn.proj = _Params(weight=(D, D), bias=(D,))
        self.ls1 = _Params(gamma=(D,))
        self.norm2 = _Params(weight=(D,), bias=(D,))
        self.mlp = nn.Module()
        self.mlp.fc1 = _Params(weight=(4 * D, D), bias=(4 * D,))
        self.mlp.fc2 = _Params(weight=(D, 4 * D), bias=(D,))
        self.ls2 = _Params(gamma=(D,))


class _Packed(_lib.Handle):
    """The C handle, the packed weights, the per-geometry tables and the workspace of one device.  Kept in the module's
    __dict__, outside the state dict."""

    def __init__(self, module: "DinoVisionTransformer", device: torch.device):
        D, depth, heads = VARIANTS[module.variant]
        cfg = _lib.MkConfig()
        cfg.embed_dim, cfg.depth, cfg.heads, cfg.down_factor = D, depth, heads, PATCH
        super().__init__(device, cfg)
        with torch.no_grad():
            sd = dict(module.named_parameters())
            self.packed = pack_backbone(sd, module.variant, device, prefix="")
            self.raw_pos = raw_positions(sd, device, prefix="")
        for name, t in self.packed.items():
            self.register(name, t)
        self.tables: Dict[tuple, Dict[str, torch.Tensor]] = {}
        self.geo = None
        self.ws = None
        self.n_img = 0
        self.stream = torch.cuda.current_stream(device)

    def buffers(self):
        yield from self.packed.values()
        for tb in self.tables.values():
            yield from tb.values()
        if self.ws is not None:
            yield self.ws

    def on_stream(self, stream):
        """The workspace is reused by every call: a call on another stream waits for the last one's, and the buffers are
        recorded for the new stream so that a block freed later is reused only after its work there."""
        if stream != self.stream:
            stream.wait_stream(self.stream)
            for t in self.buffers():
                t.record_stream(stream)
            self.stream = stream

    def use_geometry(self, H, W):
        if self.geo == (H, W):
            return
        tb = self.tables.get((H, W))
        if tb is None:
            tb = position_tables(self.raw_pos, H, W)
            if len(self.tables) >= MAX_GEOMETRIES:
                del self.tables[next(iter(self.tables))]
            self.tables[(H, W)] = tb
        for n, t in tb.items():
            self.register(n, t)
        _lib.check(self.lib.mk_finalize(self.h, H, W), "mk_finalize")
        self.geo = (H, W)

    def workspace(self, n_img, H, W):
        nbytes = int(self.lib.mk_backbone_ws_bytes(self.h, n_img, H, W))
        if self.ws is None or not 0 <= nbytes <= self.ws.numel():
            self.ws = None
            self.ws = _lib.workspace(nbytes, self.device, f"mk_backbone_ws_bytes({n_img}, {H}, {W})")
        return self.ws


class DinoVisionTransformer(nn.Module):
    """Drop-in for the reference's frozen DinoVisionTransformer (vit_small / vit_base / vit_large with patch 14,
    img_size 518, block_chunks 0) in MicKey's extractor.

    Parameters carry the reference's names and shapes (mask_token included) and never require grad.  The weights are
    packed for the kernels at the first forward_features and again after load_state_dict or a move / cast (.to, .half,
    .cuda); fp16 parameters (the extractor's `.to(float16)` under DINOV2.FLOAT16) pack with their fp16 values.  train()
    and eval() change nothing: the backbone has no dropout or batch statistics.
    """

    def __init__(self, variant: str = "vitl"):
        super().__init__()
        if variant not in VARIANTS:
            raise ValueError(f"variant must be one of {sorted(VARIANTS)}, got {variant!r}")
        D, depth, _ = VARIANTS[variant]
        self.variant = variant
        self.embed_dim = self.num_features = D
        self.patch_size = PATCH
        self.n_blocks = depth
        self.cls_token = nn.Parameter(torch.zeros(1, 1, D), requires_grad=False)
        self.pos_embed = nn.Parameter(torch.zeros(1, 1 + POS_GRID * POS_GRID, D), requires_grad=False)
        self.patch_embed = nn.Module()
        self.patch_embed.proj = _Params(weight=(D, 3, PATCH, PATCH), bias=(D,))
        self.blocks = nn.ModuleList(_Block(D) for _ in range(depth))
        self.norm = _Params(weight=(D,), bias=(D,))
        self.mask_token = nn.Parameter(torch.zeros(1, D), requires_grad=False)
        self._packed: Optional[_Packed] = None

    # -- repacking ---------------------------------------------------------------------------------------------
    def _load_from_state_dict(self, *args, **kwargs):
        # runs whenever a load covers this module, called on it or on a model that holds it
        self._packed = None
        super()._load_from_state_dict(*args, **kwargs)

    def _apply(self, fn, *args, **kwargs):
        self._packed = None
        return super()._apply(fn, *args, **kwargs)

    def _state(self, device) -> _Packed:
        if self._packed is None or self._packed.device != device:
            self._packed = None
            self._packed = _Packed(self, device)
        return self._packed

    # -- forward -----------------------------------------------------------------------------------------------
    def forward_features_list(self, x_list, masks_list):
        raise NotImplementedError("mickey_b200's DinoVisionTransformer takes one batch tensor; list inputs are not supported")

    def forward_features(self, x, masks=None):
        """x: CUDA fp16 [B, 3, H, W] (any strides; H, W multiples of 14, at least 98) -> {"x_norm_patchtokens": [B, N, D]}.

        The value is a [B, N, D] fp32 view of a fresh channel-major [B, D, N] buffer, so the extractor's
        `.permute(0, 2, 1).reshape(B, C, h, w).float()` is that buffer without a copy.  The reference's other keys
        (x_norm_clstoken, x_norm_regtokens, x_prenorm, masks) are not produced.  Runs on the current CUDA stream; the
        result never requires grad.  Every argument is checked before anything is launched."""
        if masks is not None:
            raise NotImplementedError("forward_features(masks=...) is not supported: MicKey never masks tokens")
        if isinstance(x, (list, tuple)):
            raise NotImplementedError("forward_features on a list of batches is not supported")
        if not torch.is_tensor(x):
            raise ValueError(f"x must be a torch tensor, got {type(x).__name__}")
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"x must be [B, 3, H, W], got {tuple(x.shape)}")
        B, _, H, W = x.shape
        if B < 1:
            raise ValueError("x must hold at least one image")
        if x.dtype == torch.float32:
            raise ValueError("fp32 input asks for an fp32 backbone (DINOV2.FLOAT16: False), which mickey_b200 does not "
                             "have; run the backbone in fp16 (DINOV2.FLOAT16: True)")
        if x.dtype != torch.float16:
            raise ValueError(f"x must be float16, got {x.dtype}")
        if H % PATCH or W % PATCH:
            raise ValueError(f"image {H}x{W}: height and width must be multiples of the patch size {PATCH}")
        if H < MIN_SIDE or W < MIN_SIDE:
            raise ValueError(f"image {H}x{W}: height and width must be at least {MIN_SIDE}")
        if x.device.type != "cuda":
            raise ValueError(f"x must be on a CUDA device (mickey_b200 has no CPU path), got {x.device}")
        dev = x.device
        for name, p in self.named_parameters():
            if p.device != dev:
                raise ValueError(f"parameter {name} is on {p.device}, the input on {dev}: move the module first")
        D = self.embed_dim
        N = (H // PATCH) * (W // PATCH)
        with torch.cuda.device(dev), torch.no_grad():
            st = self._state(dev)
            st.on_stream(torch.cuda.current_stream(dev))
            st.use_geometry(H, W)
            ws = st.workspace(B, H, W)
            images = x.to(torch.float32, memory_format=torch.contiguous_format)
            out = torch.empty(B, D, N, dtype=torch.float32, device=dev)
            _lib.check(st.lib.mk_backbone_features(st.h, _lib.ptr(images), B, H, W, _lib.ptr(out), _lib.ptr(ws),
                                                   ws.numel(), _lib.stream(dev)), "mk_backbone_features")
            st.n_img = B
        return {"x_norm_patchtokens": out.permute(0, 2, 1)}

    def forward(self, *args, **kwargs):
        raise NotImplementedError("only forward_features is provided: MicKey's extractor never calls the backbone's head")

    def ws_view(self, name: str, dtype, shape):
        """Typed view of a named backbone buffer ("X", "XN", ...) of the last call's workspace (tests, debugging).  The
        offsets are mk_workspace_offset's, which name the buffers for an even image count."""
        st = self._packed
        if st is None or st.geo is None or st.n_img % 2:
            raise _lib.MickeyB200Error("ws_view needs a previous forward_features call on an even number of images")
        H, W = st.geo
        return st.workspace_view(st.ws, st.n_img // 2, H, W, name, dtype, shape)
