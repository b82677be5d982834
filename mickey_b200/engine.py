"""Device-side pipeline driver: packs a reference-named state dict into the layouts the CUDA kernels
consume, owns the workspace, and calls the C ABI (include/mickey_b200.h) on the current CUDA stream.

PyTorch is plumbing here (device memory, streams); all arithmetic of the hot path happens inside
libmickey_b200.so.  The only torch arithmetic in this file is weight preparation at load time:
fp16 casts, BatchNorm folding into the conv weights, stacking the four heads, the bicubic resize of
the position embedding (same torch call as the reference, dinov2.py:165-189) and the sine table.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import math
import weakref
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from . import _lib
from .config import VARIANTS, backbone_variant
from .weights import BACKBONE, DUSTBIN, EXTRACTOR

HEAD_ORDER = ("depth_head", "det_offset", "det_head", "dsc_head")     # group order inside the kernels
KPAD = 640
PATCH = 14


def nn_pitch(N: int) -> int:
    """Row pitch (floats) of the N x N outputs the engine allocates: N rounded up to 32, so that every row starts on a
    128-byte line and the matcher's outputs can leave through TMA tensor stores (N = 1938 rows are only 8-byte aligned).
    The tensors handed out are the [.., :N] views."""
    return (N + 31) // 32 * 32


def nn_empty(B: int, N: int, device):
    """fp32 [B, N, N] view of a [B, N, nn_pitch(N)] buffer."""
    return torch.empty(B, N, nn_pitch(N), device=device)[:, :, :N]


def make_mk_config(cfg) -> _lib.MkConfig:
    variant = backbone_variant(cfg)
    D, depth, heads = VARIANTS[variant]
    m, p = cfg["MICKEY"], cfg["PROCRUSTES"]
    if cfg["FEATURE_MATCHER"]["TYPE"] != "DualSoftmax":
        # the reference's Sinkhorn branch is unreachable (feature_matcher.py:50 vs :125, SURVEY.md §2 row 5)
        raise NotImplementedError("only FEATURE_MATCHER.TYPE == 'DualSoftmax' is supported")
    c = _lib.MkConfig()
    c.embed_dim, c.depth, c.heads = D, depth, heads
    c.down_factor = int(m["DINOV2"]["DOWN_FACTOR"])
    for i, v in enumerate(m["KP_HEADS"]["BLOCKS_DIM"]):
        c.block_dims[i] = int(v)
    c.desc_dim = int(m["DSC_HEAD"]["LAST_DIM"])
    c.use_softmax = int(bool(m["KP_HEADS"]["USE_SOFTMAX"]))
    c.depth_sigmoid = int(bool(m["KP_HEADS"]["USE_DEPTHSIGMOID"]))
    c.max_depth = float(m["KP_HEADS"]["MAX_DEPTH"])
    c.kp_pos_enc = int(bool(m["KP_HEADS"]["POS_ENCODING"]))
    c.dsc_pos_enc = int(bool(m["DSC_HEAD"]["POS_ENCODING"]))
    c.norm_dsc = int(bool(m["DSC_HEAD"]["NORM_DSC"]))
    c.temperature = float(cfg["FEATURE_MATCHER"]["DUAL_SOFTMAX"]["TEMPERATURE"])
    c.use_dustbin = int(bool(cfg["FEATURE_MATCHER"]["DUAL_SOFTMAX"]["USE_DUSTBIN"]))
    c.it_matches, c.it_ransac = int(p["IT_MATCHES"]), int(p["IT_RANSAC"])
    c.num_sampled, c.num_corr, c.num_refine = int(p["NUM_SAMPLED_MATCHES"]), int(p["NUM_CORR_3D_3D"]), int(p["NUM_REFINEMENTS"])
    c.th_inlier, c.th_soft_inlier = float(p["TH_INLIER"]), float(p["TH_SOFT_INLIER"])
    if c.down_factor != PATCH:
        raise NotImplementedError("DOWN_FACTOR must be 14 (DINOv2 patch size)")
    return c


# ---------------------------------------------------------------------------------------------------------
# weight packing
# ---------------------------------------------------------------------------------------------------------
def _fold_conv3x3(w: torch.Tensor, bn: Optional[Dict[str, torch.Tensor]]):
    """[cout, cin, 3, 3] (+ eval BatchNorm) -> ([cout, 9*cin] with column = (ky*3+kx)*cin + ci, shift[cout])."""
    cout, cin = w.shape[:2]
    w = w.float()
    if bn is not None:
        scale = bn["weight"].float() / torch.sqrt(bn["running_var"].float() + 1e-5)
        shift = bn["bias"].float() - bn["running_mean"].float() * scale
    else:
        scale = torch.ones(cout, device=w.device)
        shift = torch.zeros(cout, device=w.device)
    wp = (w * scale.view(-1, 1, 1, 1)).permute(0, 2, 3, 1).reshape(cout, 9 * cin)
    return wp, shift


def _h16(t):
    return t.to(torch.float16).contiguous()


def _f32(t):
    return t.to(torch.float32).contiguous()


def pack_backbone(sd: Dict[str, torch.Tensor], variant: str, device, prefix: str = BACKBONE) -> Dict[str, torch.Tensor]:
    """The DINOv2 backbone's tensors of a state dict (fp32 or fp16; names `prefix` + the reference's module names) ->
    {packed name: device tensor}: the patch embedding, every block and the final norm.  The size-dependent tables
    (position embedding, cls token, patch bias) are built per image geometry by whoever finalizes the handle."""
    D, depth, _ = VARIANTS[variant]
    out: Dict[str, torch.Tensor] = {}

    def g(name):
        return sd[name].detach().to(device)

    h16, f32 = _h16, _f32
    b = prefix
    pw = g(b + "patch_embed.proj.weight").float().reshape(D, 3 * PATCH * PATCH)
    out["patch.w"] = h16(F.pad(pw, (0, KPAD - pw.shape[1])))
    for i in range(depth):
        p, q = f"{b}blocks.{i}.", f"blk{i}."
        out[q + "ln1.w"], out[q + "ln1.b"] = f32(g(p + "norm1.weight")), f32(g(p + "norm1.bias"))
        out[q + "ln2.w"], out[q + "ln2.b"] = f32(g(p + "norm2.weight")), f32(g(p + "norm2.bias"))
        out[q + "qkv.w"], out[q + "qkv.b"] = h16(g(p + "attn.qkv.weight")), f32(g(p + "attn.qkv.bias"))
        out[q + "proj.w"], out[q + "proj.b"] = h16(g(p + "attn.proj.weight")), f32(g(p + "attn.proj.bias"))
        out[q + "fc1.w"], out[q + "fc1.b"] = h16(g(p + "mlp.fc1.weight")), f32(g(p + "mlp.fc1.bias"))
        out[q + "fc2.w"], out[q + "fc2.b"] = h16(g(p + "mlp.fc2.weight")), f32(g(p + "mlp.fc2.bias"))
        out[q + "ls1"], out[q + "ls2"] = f32(g(p + "ls1.gamma")), f32(g(p + "ls2.gamma"))
    out["norm.w"], out["norm.b"] = f32(g(b + "norm.weight")), f32(g(b + "norm.bias"))
    return out


def pack_weights(sd: Dict[str, torch.Tensor], cfg, device) -> Dict[str, torch.Tensor]:
    """state dict with reference names (fp32 or fp16) -> {packed name: device tensor}."""
    use_bn = bool(cfg["MICKEY"]["KP_HEADS"]["BN"])
    out = pack_backbone(sd, backbone_variant(cfg), device)

    def g(name):
        return sd[name].detach().to(device)

    h16, f32 = _h16, _f32

    def bn_of(prefix):
        if not use_bn:
            return None
        return {k: g(prefix + k) for k in ("weight", "bias", "running_mean", "running_var")}

    def block(head, r):
        rp = f"{EXTRACTOR}{head}.resblock{r}."
        w1, s1 = _fold_conv3x3(g(rp + "conv1.weight"), bn_of(rp + "bn1."))
        w2, s2 = _fold_conv3x3(g(rp + "conv2.weight"), bn_of(rp + "bn2."))
        sc = sd.get(rp + "shortcut.0.weight")
        sc = None if sc is None else sc.detach().to(device).float().reshape(sc.shape[0], sc.shape[1])
        return w1, s1, w2, s2, sc

    for r in (1, 2, 3):
        parts = [block(hd, r) for hd in HEAD_ORDER]
        assert all(p[4] is not None for p in parts), "resblocks 1-3 change width and must have a shortcut conv"
        out[f"rb{r}.c1.w"], out[f"rb{r}.c1.b"] = h16(torch.cat([p[0] for p in parts])), f32(torch.cat([p[1] for p in parts]))
        out[f"rb{r}.c2.w"], out[f"rb{r}.c2.b"] = h16(torch.cat([p[2] for p in parts])), f32(torch.cat([p[3] for p in parts]))
        out[f"rb{r}.sc.w"] = h16(torch.cat([p[4] for p in parts]))
    kparts = [block(hd, 4) for hd in HEAD_ORDER[:3]]
    out["rb4k.c1.w"], out["rb4k.c1.b"] = h16(torch.cat([p[0] for p in kparts])), f32(torch.cat([p[1] for p in kparts]))
    out["rb4k.c2.w"], out["rb4k.c2.b"] = h16(torch.cat([p[2] for p in kparts])), f32(torch.cat([p[3] for p in kparts]))
    out["rb4k.sc.w"] = h16(torch.cat([p[4] for p in kparts]))
    d = block("dsc_head", 4)
    if d[4] is not None:
        raise NotImplementedError("descriptor head with LAST_DIM != 128 (shortcut conv in resblock4) is not supported")
    out["rb4d.c1.w"], out["rb4d.c1.b"], out["rb4d.c2.w"], out["rb4d.c2.b"] = h16(d[0]), f32(d[1]), h16(d[2]), f32(d[3])

    for l in range(3):
        def lw(name):
            return [g(f"{EXTRACTOR}{hd}.att_layer.layers.{l}.{name}").float() for hd in HEAD_ORDER]
        qkv = [torch.cat([q_, k_, v_]) for q_, k_, v_ in zip(lw("q_proj.weight"), lw("k_proj.weight"), lw("v_proj.weight"))]
        out[f"att{l}.qkv.w"] = h16(torch.cat(qkv))
        out[f"att{l}.merge.w"] = h16(torch.cat(lw("merge.weight")))
        out[f"att{l}.mlp0.w"] = h16(torch.cat(lw("mlp.0.weight")))
        out[f"att{l}.mlp2.w"] = h16(torch.cat(lw("mlp.2.weight")))
        out[f"att{l}.n1.w"], out[f"att{l}.n1.b"] = f32(torch.cat(lw("norm1.weight"))), f32(torch.cat(lw("norm1.bias")))
        out[f"att{l}.n2.w"], out[f"att{l}.n2.b"] = f32(torch.cat(lw("norm2.weight"))), f32(torch.cat(lw("norm2.bias")))

    out["out.depth.w"] = f32(g(EXTRACTOR + "depth_head.depth.weight").reshape(-1))
    out["out.xy.w"] = f32(g(EXTRACTOR + "det_offset.xy_offset.weight").reshape(-1))
    out["out.score.w"] = f32(g(EXTRACTOR + "det_head.score.weight").reshape(-1))
    if DUSTBIN in sd:
        out["dustbin"] = f32(g(DUSTBIN).reshape(1))
    return out


def interpolate_pos_embed(pos_embed: torch.Tensor, gh: int, gw: int) -> torch.Tensor:
    """Resize the square position-embedding grid to (gh, gw) exactly as the reference does
    (dinov2.py:165-189: bicubic, scale_factor with the +0.1 trick).  Returns [1 + gh*gw, D] fp32."""
    pe = pos_embed.float()
    n = pe.shape[1] - 1
    gs = int(math.sqrt(n))
    dim = pe.shape[-1]
    if gh * gw == n and gh == gw:
        return pe[0]
    grid = pe[:, 1:].reshape(1, gs, gs, dim).permute(0, 3, 1, 2)
    grid = F.interpolate(grid, scale_factor=((gh + 0.1) / gs, (gw + 0.1) / gs), mode="bicubic")
    assert grid.shape[-2:] == (gh, gw)
    return torch.cat([pe[0, :1], grid.permute(0, 2, 3, 1).reshape(gh * gw, dim)], dim=0)


def raw_positions(sd: Dict[str, torch.Tensor], device, prefix: str = BACKBONE):
    """(pos_embed, cls_token, patch-embedding bias) of a state dict, fp32 on `device`: the inputs of position_tables."""
    return tuple(sd[prefix + n].detach().to(device).float() for n in ("pos_embed", "cls_token", "patch_embed.proj.bias"))


def position_tables(raw, H: int, W: int) -> Dict[str, torch.Tensor]:
    """The backbone's size-dependent tables for H x W images, from raw_positions(): "patch.posb" (the position embedding
    resized to the patch grid plus the patch-embedding bias) and "patch.clspos" (the cls token plus its position)."""
    pos, cls, pbias = raw
    with torch.no_grad():
        full = interpolate_pos_embed(pos, H // PATCH, W // PATCH)
        return {"patch.posb": (full[1:] + pbias[None]).contiguous(), "patch.clspos": (cls.reshape(-1) + full[0]).contiguous()}


def sine_table_padded(gh: int, gw: int, d_model: int = 128) -> torch.Tensor:
    """2-D sine position encoding (att_layers/transformer.py:25-36, positions start at 1) laid out on
    the zero-padded token grid: [(gh+2)*(gw+2), d_model], zeros on the pad ring."""
    y = torch.arange(1, gh + 1, dtype=torch.float32).view(gh, 1).expand(gh, gw)
    x = torch.arange(1, gw + 1, dtype=torch.float32).view(1, gw).expand(gh, gw)
    div = torch.exp(torch.arange(0, d_model // 2, 2).float() * (-math.log(10000.0) / (d_model // 2)))
    pe = torch.zeros(gh, gw, d_model)
    pe[..., 0::4] = torch.sin(x[..., None] * div)
    pe[..., 1::4] = torch.cos(x[..., None] * div)
    pe[..., 2::4] = torch.sin(y[..., None] * div)
    pe[..., 3::4] = torch.cos(y[..., None] * div)
    out = torch.zeros(gh + 2, gw + 2, d_model)
    out[1:-1, 1:-1] = pe
    return out.reshape(-1, d_model).contiguous()


def _version_of(t):
    """t's version counter, which in-place torch ops on t or its views advance; None for inference tensors (no counter)."""
    try:
        return t._version
    except RuntimeError:
        return None


# ---------------------------------------------------------------------------------------------------------
class Engine(_lib.Handle):
    """One C handle + packed weights + workspace for a fixed (cfg, device)."""
    MAX_GEOMETRIES = 4          # image geometries whose tables / workspace / graphs are kept alive at once

    def __init__(self, cfg, device, side_stream: bool = False):
        """side_stream=True gives the engine its own CUDA stream for forward(): two such engines (see
        MickeyRelativePose.pipeline_depth) keep two steps in flight, so the many kernels of one step that cannot fill
        132 SMs at B=1 share the GPU with the next step's."""
        self.cfg = cfg
        device = torch.device(device)
        if device.type != "cuda":
            raise _lib.MickeyB200Error("mickey_b200 runs on a CUDA device only (sm_90a); there is no CPU path")
        self.mkcfg = make_mk_config(cfg)
        super().__init__(device, self.mkcfg)
        self.packed: Dict[str, torch.Tensor] = {}
        self.stream = torch.cuda.Stream(device=self.device) if side_stream else None
        self.assume_inputs_ready = False
        self._raw_pos = None
        self.geo = None
        self.ws = None
        self.ws_pairs = 0
        # Per-geometry state (size-dependent tables, workspace, captured graphs) stays alive while graphs that baked
        # its pointers may still be replayed; a weight (re)load drops all of it.
        self._geo_state: Dict[tuple, dict] = {}
        self._graphs, self._slot = {}, {}
        self._copy_stream = None
        self._pairs_ws = None
        self._loc_ws = None
        # set when the engine takes new blocks on the caller's stream (weights, tables, workspace, buffer sets): that stream
        # may still have work queued on those blocks (writes of the weights and tables, or pending kernels of tensors freed
        # there), so the streams that use them next wait on it once
        self._caller_pending = False
        self._last_ent = None           # buffer set of the last forward() call (release())

    # -- streams -----------------------------------------------------------------------------------------------
    # Engine buffers (packed weights, per-geometry tables, workspaces, the static buffer sets) are allocated on the
    # caller's stream.  When the engine has a side stream they are also used there, so each one is passed to
    # record_stream for it: when a buffer is dropped (batch growth, geometry eviction, weight reload) the caching
    # allocator hands its block out again only after the side stream's work queued so far has finished.
    def _own(self, t):
        if t is not None and self.stream is not None:
            t.record_stream(self.stream)
        return t

    def _buffers(self):
        yield from self.packed.values()
        yield self.ws
        yield self._pairs_ws
        yield self._loc_ws
        for gs in self._geo_state.values():
            yield from (gs[n] for n in ("patch.posb", "patch.clspos", "head.pe", "ws"))
        for ent in self._graphs.values():
            yield from ent["st"].values()

    def use_side_stream(self):
        """Give the engine its own stream from now on (MickeyRelativePose.pipeline_depth > 1).  Buffers allocated
        before, and the graphs captured on the caller's stream, stay valid: the buffers are recorded for the new stream."""
        if self.stream is None:
            self.stream = torch.cuda.Stream(device=self.device)
            for t in self._buffers():
                self._own(t)
            self._caller_pending = True

    @contextlib.contextmanager
    def _ordered(self):
        """Handle calls outside forward() (the staged stages, feature banks, solve) run on the caller's stream.  They
        share the handle's device RNG word and forward()'s workspace with the graph replays queued on the side stream,
        so they run after that stream's queued work, and the side stream's later work runs after them."""
        if self.stream is None:
            yield
            return
        caller = torch.cuda.current_stream()
        caller.wait_stream(self.stream)
        try:
            yield
        finally:
            self.stream.wait_stream(caller)

    # -- weights ---------------------------------------------------------------------------------------------
    def load_state_dict(self, sd: Dict[str, torch.Tensor], share_with: "Engine" = None):
        """share_with: another engine on the same device whose packed weight tensors are registered here too
        (one copy of the weights in HBM for all pipeline slots)."""
        if share_with is not None:
            self.packed = {k: v for k, v in share_with.packed.items() if k not in ("patch.posb", "patch.clspos", "head.pe")}
            self._raw_pos = share_with._raw_pos
        else:
            with torch.no_grad():
                self.packed = pack_weights(sd, self.cfg, self.device)
                self._raw_pos = raw_positions(sd, self.device)
        for name, t in self.packed.items():
            self.register(name, self._own(t))
        self._caller_pending = True
        # captured graphs hold raw pointers of the previous packed weights and tables: none of them may be replayed
        self._graphs.clear()
        self._slot.clear()
        self._geo_state.clear()
        self.geo = None
        self.ws = None
        self.ws_pairs = 0

    def prepare(self, n_pairs: int, H: int, W: int):
        """Size-dependent tables + workspace for images cropped to (H, W) (multiples of 14)."""
        self._use_geometry(H, W)
        if self.ws is None or self.ws_pairs < n_pairs:
            nbytes = self.lib.mk_workspace_bytes(self.h, n_pairs, H, W)
            self.ws = self._own(_lib.workspace(nbytes, self.device, "mk_workspace_bytes"))
            self.ws_pairs = n_pairs
            self._caller_pending = True
        return self.ws

    def _use_geometry(self, H: int, W: int):
        """Register the size-dependent tables of (H, W) and finalize the handle for it (kept per geometry)."""
        assert self.packed, "load_state_dict first"
        if self.geo != (H, W):
            if self.geo is not None:                       # park the outgoing geometry's workspace with its state
                self._geo_state[self.geo].update(ws=self.ws, ws_pairs=self.ws_pairs)
            gs = self._geo_state.get((H, W))
            if gs is None:
                gs = position_tables(self._raw_pos, H, W)
                gs.update({"head.pe": sine_table_padded(H // PATCH, W // PATCH).to(self.device), "ws": None, "ws_pairs": 0})
                for n in ("patch.posb", "patch.clspos", "head.pe"):
                    self._own(gs[n])
                self._caller_pending = True
                if len(self._geo_state) >= self.MAX_GEOMETRIES:      # evict the oldest geometry together with its graphs
                    old = next(iter(self._geo_state))
                    del self._geo_state[old]
                    for k in [k for k in self._graphs if (k[1], k[2]) == old]:
                        del self._graphs[k]
                self._geo_state[(H, W)] = gs
            for n in ("patch.posb", "patch.clspos", "head.pe"):
                self.packed[n] = gs[n]
                self.register(n, gs[n])
            _lib.check(self.lib.mk_finalize(self.h, H, W), "mk_finalize")
            self.geo = (H, W)
            self.ws, self.ws_pairs = gs["ws"], gs["ws_pairs"]

    @property
    def launch_count(self) -> int:
        """Kernel launches issued by the library (eager calls) ..."""
        return int(self.lib.mk_launch_count(self.h))

    @property
    def total_kernel_launches(self) -> int:
        """... plus the kernel nodes executed by CUDA-graph replays of mk_forward."""
        return self.launch_count + getattr(self, "graph_launches", 0)

    def ws_view(self, name: str, dtype, shape):
        """Typed view of a named intermediate buffer of the last call's workspace (debugging / tests)."""
        H, W = self.geo
        return self.workspace_view(self.ws, self.ws_pairs, H, W, name, dtype, shape)

    def profile(self, enable: bool):
        _lib.check(self.lib.mk_profile_enable(self.h, int(enable)), "mk_profile_enable")

    def profile_read(self) -> Dict[str, tuple]:
        """{kernel class: (launch scopes, total device ms)} measured with CUDA events on the launch stream."""
        buf = C.create_string_buffer(1 << 16)
        _lib.check(self.lib.mk_profile_read(self.h, buf, len(buf)), "mk_profile_read")
        out = {}
        for line in buf.value.decode().splitlines():
            tag, n, ms = line.split()
            out[tag] = (int(n), float(ms))
        return out

    def _ws_for(self, n_pairs, H, W):
        # the workspace layout depends on n_pairs: carve exactly for this call's batch
        self.prepare(n_pairs, H, W)
        if self.ws_pairs != n_pairs:
            nbytes = self.lib.mk_workspace_bytes(self.h, n_pairs, H, W)
            if self.ws.numel() < nbytes:
                self.ws = self._own(_lib.workspace(nbytes, self.device, "mk_workspace_bytes"))
                self._caller_pending = True
            self.ws_pairs = n_pairs
        return self.ws

    # -- stages ------------------------------------------------------------------------------------------------
    @staticmethod
    def _image_batch(images: torch.Tensor):
        """fp32 [n, 3, H, W] or uint8 [n, H, W, 3] (RGB as decoded, SURVEY.md §8 f1) -> (contiguous images, u8, n, H, W)."""
        u8 = images.dtype == torch.uint8
        if u8:
            assert images.dim() == 4 and images.shape[-1] == 3, "uint8 images must be [n, H, W, 3] (HWC, RGB)"
            images = images.contiguous()
            n_img, H, W, _ = images.shape
        else:
            images = images.float().contiguous()
            n_img, _, H, W = images.shape
        return images, u8, n_img, H, W

    def _nn_outputs(self, B, N, lean):
        """(scores, kp_scores, final_scores) of B pairs as nn_empty views; scores and kp_scores are None when lean."""
        dev = self.device
        return (None if lean else nn_empty(B, N, dev)), (None if lean else nn_empty(B, N, dev)), nn_empty(B, N, dev)

    def _solver_outputs(self, B):
        dev, c = self.device, self.mkcfg
        return {"pose": torch.empty(B, 13, device=dev), "best_set": torch.empty(B, dtype=torch.int32, device=dev),
                "inlier_mask": torch.empty(B, c.num_sampled, device=dev),
                "sampled_idx": torch.empty(B * c.it_matches, c.num_sampled, dtype=torch.int32, device=dev),
                "status": torch.zeros(1, dtype=torch.int32, device=dev)}

    def _outputs(self, n_img, n_pairs, N, lean=False, scr_dsc=True):
        """Fresh outputs of a call on n_img images and n_pairs pairs, keyed as forward() returns them: kps, depth and (with
        scr_dsc) scr, dsc per image; when n_pairs > 0, the matcher's and the solver's outputs."""
        dev = self.device
        out = {"kps": torch.empty(n_img, 2, N, device=dev), "depth": torch.empty(n_img, 1, N, device=dev)}
        if scr_dsc:
            out.update(scr=torch.empty(n_img, 1, N, device=dev), dsc=torch.empty(n_img, self.mkcfg.desc_dim, N, device=dev))
        if n_pairs:
            out["scores"], out["kp_scores"], out["final_scores"] = self._nn_outputs(n_pairs, N, lean)
            out.update(self._solver_outputs(n_pairs))
        return out

    @staticmethod
    def _output_args(out):
        """The trailing outputs of mk_forward / mk_forward_u8 (with scr, dsc) or mk_forward_pairs, in the header's order."""
        p, f = _lib.ptr, out["final_scores"]
        return (*(p(out[k]) for k in ("kps", "depth", "scr", "dsc", "scores", "kp_scores") if k in out), p(f), f.stride(1),
                *(p(out[k]) for k in ("pose", "best_set", "inlier_mask", "sampled_idx", "status")))

    @staticmethod
    def _forward_seed(seed):
        return (int(seed) & (2 ** 64 - 1)) or 1         # a seed of 0 would continue the device-side sequence

    def _intrinsics(self, K):
        return K.to(self.device, torch.float32).contiguous()

    def extract(self, images: torch.Tensor):
        """images fp32 [2B, 3, H, W] (image0 batch then image1 batch) -> kps, depth, scr, dsc.
        H, W need not be multiples of 14: the patch gather reads only the top-left 14*(H//14) x 14*(W//14) crop
        (reference mickey_extractor.py:46), so no cropped copy is made."""
        images, u8, n_img, H, W = self._image_batch(images)
        assert n_img % 2 == 0
        B, N = n_img // 2, (H // PATCH) * (W // PATCH)
        ws = self._ws_for(B, H, W)
        feats = tuple(self._outputs(n_img, 0, N).values())          # kps, depth, scr, dsc
        fn = self.lib.mk_extract_u8 if u8 else self.lib.mk_extract
        with self._ordered():
            _lib.check(fn(self.h, _lib.ptr(images), B, H, W, *map(_lib.ptr, feats), _lib.ptr(ws), ws.numel(), _lib.stream()),
                       "mk_extract")
        return feats

    # -- feature banks: extract images once, then match / solve any pairs among them ------------------------------
    def _bank_ws(self, n_img, n_pairs, H, W):
        """Workspace of extract_images / forward_pairs.  It is separate from forward()'s, whose buffer sets and captured
        graphs hold that workspace's address; it grows to the largest call seen."""
        nbytes = self.lib.mk_workspace_bytes_for(self.h, n_img, n_pairs, H, W)
        if self._pairs_ws is None or self._pairs_ws.numel() < nbytes:
            self._pairs_ws = None
            self._pairs_ws = _lib.workspace(nbytes, self.device, "mk_workspace_bytes_for")
        return self._pairs_ws

    def extract_images(self, images: torch.Tensor):
        """Any number n >= 1 of images, fp32 [n, 3, H, W] or uint8 [n, H, W, 3] -> kps [n,2,N], depth [n,1,N], scr [n,1,N],
        dsc [n,128,N]: per image, bit-identical to what extract() gives for that image (mk_extract_images / _u8)."""
        images, u8, n_img, H, W = self._image_batch(images)
        if n_img < 1:
            raise _lib.MickeyB200Error("extract_images needs at least one image")
        N = (H // PATCH) * (W // PATCH)
        self._use_geometry(H, W)
        ws = self._bank_ws(n_img, 0, H, W)
        feats = tuple(self._outputs(n_img, 0, N).values())          # kps, depth, scr, dsc
        fn = self.lib.mk_extract_images_u8 if u8 else self.lib.mk_extract_images
        with self._ordered():
            _lib.check(fn(self.h, _lib.ptr(images), n_img, H, W, *map(_lib.ptr, feats), _lib.ptr(ws), ws.numel(),
                          _lib.stream()), "mk_extract_images")
        return feats

    def forward_pairs(self, bank0, idx0, bank1, idx1, K0, K1, seed: int, image_size, lean: bool = False):
        """Match and solve the pairs (bank0[idx0[p]], bank1[idx1[p]]) in one C call (mk_forward_pairs).

        bank = (kps, depth, scr, dsc) as extract_images returns it, extracted at image_size = (H, W); idx0 / idx1 int32
        device tensors [P] that the caller has range-checked; K0 / K1 [P, 3, 3].  Returns fresh tensors: kps [2P,2,N] and
        depth [2P,1,N] (image-0 rows first), scores / kp_scores (None when lean), final_scores, pose [P,13], best_set,
        inlier_mask, sampled_idx, status."""
        H, W = image_size
        self._use_geometry(H, W)
        P, N = idx0.numel(), bank0[0].shape[-1]
        ws = self._bank_ws(0, P, H, W)
        out = self._outputs(2 * P, P, N, lean, scr_dsc=False)
        K0, K1 = self._intrinsics(K0), self._intrinsics(K1)
        p = _lib.ptr
        with self._ordered():
            _lib.check(self.lib.mk_forward_pairs(
                self.h, *(p(t) for t in bank0), bank0[0].shape[0], *(p(t) for t in bank1), bank1[0].shape[0], p(idx0), p(idx1),
                p(K0), p(K1), P, C.c_ulonglong(self._forward_seed(seed)), *self._output_args(out), p(ws), ws.numel(),
                _lib.stream()), "mk_forward_pairs")
        return out

    def match(self, B: int, N: int, lean: bool = False):
        """lean: only final_scores (the matrix the solver reads) is materialised; scores / kp_scores come back as None."""
        scores, kp_scores, final = self._nn_outputs(B, N, lean)
        with self._ordered():
            _lib.check(self.lib.mk_match(self.h, B, _lib.ptr(scores), _lib.ptr(kp_scores), _lib.ptr(final), final.stride(1),
                                         _lib.ptr(self.ws), self.ws.numel(), _lib.stream()), "mk_match")
        return scores, kp_scores, final

    # -- whole path in one C call, optionally replayed from a CUDA graph -------------------------------------------
    def _static_buffers(self, B, H, W, u8=False, lean=False):
        dev = self.device
        images = torch.empty(2 * B, H, W, 3, dtype=torch.uint8, device=dev) if u8 else torch.empty(2 * B, 3, H, W, device=dev)
        return {"images": images, "K0": torch.empty(B, 3, 3, device=dev), "K1": torch.empty(B, 3, 3, device=dev),
                **self._outputs(2 * B, B, (H // PATCH) * (W // PATCH), lean)}

    def _call_forward(self, st, B, H, W, seed):
        fn = self.lib.mk_forward_u8 if st["images"].dtype == torch.uint8 else self.lib.mk_forward
        _lib.check(fn(self.h, _lib.ptr(st["images"]), _lib.ptr(st["K0"]), _lib.ptr(st["K1"]), B, H, W, C.c_ulonglong(seed),
                      *self._output_args(st), _lib.ptr(self.ws), self.ws.numel(), _lib.stream()), "mk_forward")

    def forward(self, image0, image1, K0, K1, seed: int, use_graph: bool = True, lean: bool = False):
        """Whole hot path (extract -> match -> solve) for a batch of pairs.

        Returns the dict of STATIC output tensors of this (B, H, W) geometry.  Two buffer sets alternate, so the
        tensors of one call stay valid until the call after the next one with the same geometry on this engine.  That
        window is in stream order when this engine's work waits on the caller's stream (no side stream, or device
        inputs without assume_inputs_ready), or for reads the caller announced with release().  Otherwise it holds in
        host order only: reads of a call's outputs queued on the caller's stream must have completed (synchronise that
        stream) before the call that reuses the buffer set is issued; waiting on the caller's stream instead would
        serialise the pipeline, since the caller waits on every call's completion.  Host (pinned)
        inputs are copied H2D on a side stream into the other buffer set while the previous call is still
        computing; device inputs are copied D2D on the main stream, after the caller's stream has produced them
        (unless assume_inputs_ready).  Inputs of another floating dtype (fp64 K, say) are converted by those copies."""
        B = image0.shape[0]
        u8 = image0.dtype == torch.uint8                 # [B, H, W, 3] RGB straight from the decoder (mk_forward_u8)
        if u8:
            if image0.dim() != 4 or image0.shape[-1] != 3 or image1.dtype != torch.uint8:
                raise _lib.MickeyB200Error("uint8 images must both be [B, H, W, 3] (HWC, RGB)")
            H, W = image0.shape[1], image0.shape[2]
        else:
            H, W = image0.shape[-2], image0.shape[-1]
        if image1.shape != image0.shape:
            raise _lib.MickeyB200Error(f"image0 {tuple(image0.shape)} and image1 {tuple(image1.shape)} must have the same shape: "
                                       "both images of a batch go through one extraction call")
        self._ws_for(B, H, W)
        ent = self._buffer_set((B, H, W), (bool(u8), bool(lean)), self.ws, lambda: self._static_buffers(B, H, W, u8, lean))
        st = ent["st"]
        return self._issue(ent, (image0, image1, K0, K1), (st["images"][:B], st["images"][B:], st["K0"], st["K1"]),
                           lambda s: self._call_forward(st, B, H, W, s), seed, use_graph)

    def _buffer_set(self, shape, fmt, ws, make):
        """The static buffer set of a forward() / localize() call of shape (n, H, W) and format fmt: two sets alternate per
        (shape, fmt); a set (with its graph) is rebuilt when the workspace ws it was captured with has moved."""
        if self._copy_stream is None:
            self._copy_stream = torch.cuda.Stream(device=self.device)
        slot = self._slot.get((*shape, fmt), 0)
        self._slot[(*shape, fmt)] = slot ^ 1
        key = (*shape, slot, fmt)
        ent = self._graphs.get(key)
        if ent is None or ent["ws_ptr"] != ws.data_ptr():
            ent = {"st": {k: self._own(t) for k, t in make().items()}, "graph": None,
                   "launches": 0, "ws_ptr": ws.data_ptr(), "calls": 0, "done": None, "readers": set()}
            self._graphs[key] = ent
            self._caller_pending = True
        return ent

    def _issue(self, ent, ops, dst, call, seed, use_graph, before=None):
        """Issue one call of buffer set ent: copy the inputs ops into dst, run before() (on the engine's stream, after
        those copies), then call(seed) eagerly or from the set's graph.  Returns the set's static tensors."""
        st = ent["st"]
        caller = torch.cuda.current_stream()
        main = self.stream if self.stream is not None else caller
        fresh, self._caller_pending = self._caller_pending, False
        if self.stream is not None:
            if ent.get("released") is not None:
                main.wait_event(ent["released"])        # the caller's reads of this set's previous outputs
                ent["released"] = None
            if caller.cuda_stream not in ent["readers"]:
                # the caller reads the outputs on its own stream: a dropped buffer set is reused only after that
                ent["readers"].add(caller.cuda_stream)
                for t in st.values():
                    if t is not None:
                        t.record_stream(caller)
            on_device = any(t.device.type != "cpu" for t in ops)
            if fresh or (on_device and not self.assume_inputs_ready):
                main.wait_stream(caller)                # device inputs may still be being produced on the caller's stream
        with torch.cuda.stream(main):
            self._forward_on(main, ent, dst, ops, call, seed, use_graph, caller if fresh else None, before)
        if self.stream is not None:
            caller.wait_event(ent["done"])              # outputs are safe to consume on the caller's stream
        self._last_ent = ent
        return st

    def release(self):
        """The caller's stream has queued every read of the outputs the last forward() returned.  The call that reuses
        that buffer set waits for those reads (an event on the caller's stream), not for the caller's stream as a whole,
        so steps stay in flight.  Without a side stream the caller's stream orders everything and this does nothing."""
        if self.stream is not None and self._last_ent is not None:
            ev = torch.cuda.Event()
            ev.record()
            self._last_ent["released"] = ev

    def _forward_on(self, main, ent, dst, ops, call, seed, use_graph, caller_pending, before):
        if any(t.device.type == "cpu" for t in ops):
            cs = self._copy_stream
            if caller_pending is not None:
                cs.wait_stream(caller_pending)          # new input buffers: blocks the caller's stream may still be using
            if ent["done"] is not None:
                cs.wait_event(ent["done"])              # the graph that last read this input buffer has finished
            with torch.cuda.stream(cs):
                for d, s in zip(dst, ops):
                    if s.device.type == "cpu":
                        d.copy_(s, non_blocking=True)
            main.wait_stream(cs)
        for d, s in zip(dst, ops):                      # device operands: in order behind the caller's stream (see forward)
            if s.device.type != "cpu":
                d.copy_(s, non_blocking=True)
        if before is not None:
            before()
        seed = self._forward_seed(seed)
        if not use_graph:
            call(seed)
        elif ent["graph"] is None and ent["calls"] == 0:
            # first call of this buffer set runs eagerly (one-time lazy initialisation inside the library:
            # function attributes, TMA descriptors); the second call is captured, later calls replay
            l0 = self.launch_count
            call(seed)
            ent["launches"] = self.launch_count - l0
            ent["calls"] = 1
        else:
            _lib.check(self.lib.mk_set_seed(self.h, C.c_ulonglong(seed), _lib.stream()), "mk_set_seed")
            if ent["graph"] is None:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    call(0)                                 # seed 0 = continue the device-side sequence
                ent["graph"] = g
            ent["graph"].replay()
            self.graph_replays = getattr(self, "graph_replays", 0) + 1
            self.graph_launches = getattr(self, "graph_launches", 0) + ent["launches"]
        if ent["done"] is None:
            ent["done"] = torch.cuda.Event()
        ent["done"].record(main)

    # -- localization against cached references: only the queries are extracted (mk_localize) ---------------------------
    REF_KEYS = ("ref.kps", "ref.depth", "ref.scr", "ref.dsc")

    def _localize_ws(self, P, H, W):
        """Workspace of localize(), apart from forward()'s and the feature banks': localize()'s buffer sets and graphs hold
        its address.  It grows to the largest call seen; a set captured on an outgrown workspace is rebuilt."""
        nbytes = self.lib.mk_workspace_bytes_for(self.h, P, P, H, W)
        if self._loc_ws is None or self._loc_ws.numel() < nbytes:
            self._loc_ws = self._own(_lib.workspace(nbytes, self.device, "mk_workspace_bytes_for"))
            self._caller_pending = True
        return self._loc_ws

    def _localize_buffers(self, P, H, W, n_ref, u8, lean):
        dev, D, N = self.device, self.mkcfg.desc_dim, (H // PATCH) * (W // PATCH)
        queries = torch.empty(P, H, W, 3, dtype=torch.uint8, device=dev) if u8 else torch.empty(P, 3, H, W, device=dev)
        ref = (torch.empty(n_ref, 2, N, device=dev), torch.empty(n_ref, 1, N, device=dev), torch.empty(n_ref, 1, N, device=dev),
               torch.empty(n_ref, D, N, device=dev))
        out = self._outputs(2 * P, P, N, lean, scr_dsc=False)
        return {"queries": queries, "ref_idx": torch.empty(P, dtype=torch.int32, device=dev),
                "K0": torch.empty(P, 3, 3, device=dev), "K1": torch.empty(P, 3, 3, device=dev), **dict(zip(self.REF_KEYS, ref)),
                "kps": out.pop("kps"), "depth": out.pop("depth"), "scr": torch.empty(P, 1, N, device=dev),
                "dsc": torch.empty(P, D, N, device=dev), **out}

    def _call_localize(self, st, ws, n_ref, P, H, W, seed):
        fn = self.lib.mk_localize_u8 if st["queries"].dtype == torch.uint8 else self.lib.mk_localize
        p = _lib.ptr
        _lib.check(fn(self.h, *(p(st[k]) for k in self.REF_KEYS), n_ref, p(st["ref_idx"]), p(st["queries"]), p(st["K0"]),
                      p(st["K1"]), P, H, W, C.c_ulonglong(seed), *self._output_args(st), p(ws), ws.numel(), _lib.stream()),
                   "mk_localize")

    def localize(self, ref_bank, ref_idx, queries, K0, K1, seed: int, use_graph: bool = True, lean: bool = False):
        """Pose P queries against cached references in one C call (mk_localize): pair p = (reference ref_idx[p], query p).

        ref_bank = (kps, depth, scr, dsc) of n_ref references as extract_images returns them (fp32, contiguous, on the
        engine's device), extracted at the queries' token grid; ref_idx int [P] in [0, n_ref) (host or device); queries
        fp32 [P, 3, H, W] or uint8 [P, H, W, 3] RGB, K0 / K1 [P, 3, 3], host (pinned) or device, as forward() takes them.
        Returns the static tensors of this call's buffer set, with forward()'s lifetime rules: kps [2P,2,N] and depth
        [2P,1,N] (reference rows first), the queries' scr [P,1,N] and dsc [P,128,N], scores / kp_scores (None when lean),
        final_scores, pose, best_set, inlier_mask, sampled_idx, status.

        A captured graph must not read the caller's tensors, which may be freed or changed before a replay: each buffer set
        holds a copy of the reference bank (its reference slot), refreshed on the engine's stream whenever the bank's
        tensors are not the objects last copied (held by weak reference, so a new tensor at a freed one's address is
        still new) or their version counters moved (an in-place torch op on them or a view of them).  Writes that bypass
        the version counter (through .data or a raw pointer) are not seen: pass new tensors after such writes."""
        u8 = queries.dtype == torch.uint8
        if u8:
            if queries.dim() != 4 or queries.shape[-1] != 3:
                raise _lib.MickeyB200Error("uint8 queries must be [P, H, W, 3] (HWC, RGB)")
            P, H, W = queries.shape[:3]
        else:
            P, H, W = queries.shape[0], queries.shape[-2], queries.shape[-1]
        n_ref = ref_bank[0].shape[0]
        self._use_geometry(H, W)
        ws = self._localize_ws(P, H, W)
        ent = self._buffer_set((P, H, W), ("localize", bool(u8), bool(lean), n_ref), ws,
                               lambda: self._localize_buffers(P, H, W, n_ref, u8, lean))
        st = ent["st"]
        src = tuple(ref_bank)
        seen = ent.get("ref_src")
        stale = seen is None or any(r() is not t or v is None or v != _version_of(t) for (r, v), t in zip(seen, src))
        if stale:
            # the slot's copies read the caller's tensors: like new engine blocks, they wait for the caller's stream
            self._caller_pending = True

        def refresh():
            if stale:
                for k, t in zip(self.REF_KEYS, src):
                    st[k].copy_(t, non_blocking=True)
                    if self.stream is not None:
                        t.record_stream(self.stream)        # the caller may drop t before this copy has run
                ent["ref_src"] = tuple((weakref.ref(t), _version_of(t)) for t in src)

        return self._issue(ent, (queries, ref_idx, K0, K1), (st["queries"], st["ref_idx"], st["K0"], st["K1"]),
                           lambda s: self._call_localize(st, ws, n_ref, P, H, W, s), seed, use_graph, before=refresh)

    def solve(self, final_scores, kps, depth, K0, K1, seed: int, outer_idx=None, inner_idx=None):
        """kps [2B,2,N], depth [2B,1,N] as produced by extract (image0 rows first).  final_scores [B,N,N] may be a padded
        view (last dim contiguous, rows `stride(1)` floats apart) or any tensor (made contiguous).  Returns the solver's
        outputs (_solver_outputs) and hyp_scores [B, IT_MATCHES * IT_RANSAC].  A seed of 0 continues the device-side
        sequence."""
        B, N, _ = final_scores.shape
        final_scores, pitch = _lib.pitched(final_scores)
        dev, c = self.device, self.mkcfg
        out = self._solver_outputs(B)
        out["hyp_scores"] = torch.empty(B, c.it_matches * c.it_ransac, device=dev)
        outer_idx, inner_idx = (None if i is None else i.to(dev, torch.int32).contiguous() for i in (outer_idx, inner_idx))
        K0, K1 = self._intrinsics(K0), self._intrinsics(K1)
        p = _lib.ptr
        with self._ordered():
            _lib.check(self.lib.mk_solve_pose(
                self.h, p(final_scores), pitch, p(kps), p(depth), p(K0), p(K1), B, N, C.c_ulonglong(seed & (2 ** 64 - 1)),
                p(outer_idx), p(inner_idx), p(out["pose"]), p(out["best_set"]), p(out["inlier_mask"]), p(out["sampled_idx"]),
                p(out["hyp_scores"]), p(out["status"]), p(self.ws), self.ws.numel(), _lib.stream()), "mk_solve_pose")
        return out
