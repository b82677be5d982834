"""Host-side mirror of the reference's model surface for the inference hot path.

Same names, arguments, data-dict keys and error behaviour as
    lib/models/builder.py:5-20            build_model(cfg, checkpoint)
    lib/models/MicKey/compute_pose.py:6-60 MickeyRelativePose
    .../modules/compute_correspondences.py ComputeCorrespondences
    .../modules/utils/probabilisticProcrustes.py e2eProbabilisticProcrustesSolver
so that demo_inference.py / submission.py run against it unchanged — but every stage executes inside
libmickey_b200.so (hand-written sm_90a CUDA).  The nn.Module tree below only *stores* the parameters
under the reference's state-dict names (so a real mickey.ckpt loads with strict=True); it has no
forward arithmetic of its own.
"""
from __future__ import annotations

import operator
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn

from ._lib import MickeyB200Error
from .config import backbone_variant
from .engine import Engine, PATCH
from .matches import mutual_matches
from .weights import synthetic_state_dict

_BUFFER_SUFFIXES = ("running_mean", "running_var", "num_batches_tracked")


@dataclass
class MickeyFeatures:
    """Extractor outputs of n images (MickeyRelativePose.extract_features): a feature bank that pose_from_features pairs
    by index.  kps [n,2,N] (pixels), depth [n,1,N], scr [n,1,N], dsc [n,128,N], fp32, in the data-dict layouts;
    grid = (gh, gw) token grid (N = gh * gw); image_size = (H, W) of the images they were extracted from."""
    kps: torch.Tensor
    depth: torch.Tensor
    scr: torch.Tensor
    dsc: torch.Tensor
    grid: Tuple[int, int]
    image_size: Tuple[int, int]

    def __len__(self) -> int:
        return self.kps.shape[0]

    @property
    def device(self) -> torch.device:
        return self.kps.device

    def tensors(self):
        return self.kps, self.depth, self.scr, self.dsc

    @staticmethod
    def cat(banks: Sequence["MickeyFeatures"]) -> "MickeyFeatures":
        """One bank holding the images of `banks` in order (all of one geometry)."""
        first = banks[0]
        for b in banks[1:]:
            if b.grid != first.grid or b.image_size != first.image_size:
                raise MickeyB200Error(f"cannot join banks of geometry {b.image_size} and {first.image_size}")
        if len(banks) == 1:
            return first
        return MickeyFeatures(*(torch.cat(ts) for ts in zip(*(b.tensors() for b in banks))), first.grid, first.image_size)


def _host_indices(idx, name: str) -> List[int]:
    if torch.is_tensor(idx):
        if idx.dtype.is_floating_point or idx.dtype.is_complex or idx.dtype == torch.bool:
            raise MickeyB200Error(f"{name} must hold integers, got {idx.dtype}")
        return [int(v) for v in idx.detach().reshape(-1).cpu().tolist()]
    out = []
    for v in idx:
        try:
            if isinstance(v, bool):
                raise TypeError
            out.append(operator.index(v))
        except TypeError:
            raise MickeyB200Error(f"{name} must hold integers, got {v!r}") from None
    return out


def validate_pairs(feats0: MickeyFeatures, idx0, feats1: MickeyFeatures, idx1) -> Tuple[List[int], List[int]]:
    """Host-side checks of a pose_from_features request, before anything is launched: integer indices inside their
    banks, as many idx0 as idx1 (at least one pair), both banks of one geometry (the solver needs N x N square) and on
    one device.  Returns the indices as host lists."""
    i0, i1 = _host_indices(idx0, "idx0"), _host_indices(idx1, "idx1")
    if len(i0) != len(i1):
        raise MickeyB200Error(f"idx0 has {len(i0)} entries and idx1 {len(i1)}: one index of each bank per pair")
    if not i0:
        raise MickeyB200Error("pose_from_features needs at least one pair")
    for name, idx, bank in (("idx0", i0, feats0), ("idx1", i1, feats1)):
        bad = [v for v in idx if not 0 <= v < len(bank)]
        if bad:
            raise MickeyB200Error(f"{name} {bad[:4]} outside its bank of {len(bank)} images")
    if feats0.grid != feats1.grid:
        raise MickeyB200Error(f"banks of token grids {feats0.grid} and {feats1.grid}: both must come from one geometry")
    for b in (feats0, feats1):
        _check_bank(b)
    devs = {t.device for b in (feats0, feats1) for t in b.tensors()}
    if len(devs) != 1:
        raise MickeyB200Error(f"bank tensors on several devices: {sorted(map(str, devs))}")
    return i0, i1


def _check_bank(b: MickeyFeatures):
    if tuple(b.grid) != (b.image_size[0] // PATCH, b.image_size[1] // PATCH):
        raise MickeyB200Error(f"bank grid {b.grid} is not the token grid of its image size {b.image_size}")
    N = b.grid[0] * b.grid[1]
    if tuple(b.kps.shape[1:]) != (2, N) or tuple(b.dsc.shape[2:]) != (N,) or b.depth.shape[-1] != N or b.scr.shape[-1] != N:
        raise MickeyB200Error(f"bank tensors {tuple(b.kps.shape)} / {tuple(b.dsc.shape)} do not match its grid {b.grid}")
    if any(t.shape[0] != len(b) for t in b.tensors()):
        raise MickeyB200Error("bank tensors hold different image counts")


def validate_localize(reference: MickeyFeatures, ref_idx, queries, K_color0, K_color1) -> List[int]:
    """Host-side checks of a localize request, before anything is launched, with validate_pairs' rules: at least one
    query, fp32 [P, 3, H, W] or uint8 [P, H, W, 3]; integer ref_idx, one per query, inside the reference bank; the bank's
    token grid equal to the queries' (the solver needs N x N square); the bank on one device, and the queries there or on
    the host; K_color0 / K_color1 of shape [P, 3, 3].  Returns ref_idx as a host list."""
    idx = _host_indices(ref_idx, "ref_idx")
    if not torch.is_tensor(queries) or queries.dim() != 4:
        raise MickeyB200Error("queries must be a [P, 3, H, W] float or [P, H, W, 3] uint8 tensor")
    if queries.dtype == torch.uint8:
        if queries.shape[-1] != 3:
            raise MickeyB200Error(f"uint8 queries must be [P, H, W, 3] (HWC, RGB), got {tuple(queries.shape)}")
        P, H, W = queries.shape[:3]
    else:
        if not queries.dtype.is_floating_point or queries.shape[1] != 3:
            raise MickeyB200Error(f"float queries must be [P, 3, H, W], got {tuple(queries.shape)} {queries.dtype}")
        P, H, W = queries.shape[0], queries.shape[2], queries.shape[3]
    if P < 1:
        raise MickeyB200Error("localize needs at least one query")
    if len(idx) != P:
        raise MickeyB200Error(f"ref_idx has {len(idx)} entries for {P} queries: one reference per query")
    bad = [v for v in idx if not 0 <= v < len(reference)]
    if bad:
        raise MickeyB200Error(f"ref_idx {bad[:4]} outside the reference bank of {len(reference)} images")
    _check_bank(reference)
    if tuple(reference.grid) != (H // PATCH, W // PATCH):
        raise MickeyB200Error(f"reference grid {tuple(reference.grid)} differs from the queries' token grid "
                              f"{(H // PATCH, W // PATCH)} ({H} x {W} images)")
    devs = {t.device for t in reference.tensors()}
    if len(devs) != 1:
        raise MickeyB200Error(f"reference tensors on several devices: {sorted(map(str, devs))}")
    if queries.device.type != "cpu" and queries.device != reference.device:
        raise MickeyB200Error(f"queries on {queries.device}, reference on {reference.device}")
    K0, K1 = torch.as_tensor(K_color0), torch.as_tensor(K_color1)
    if tuple(K0.shape) != (P, 3, 3) or tuple(K1.shape) != (P, 3, 3):
        raise MickeyB200Error(f"K_color0 {tuple(K0.shape)} / K_color1 {tuple(K1.shape)} must be [{P}, 3, 3]")
    return idx


def synthetic_backbone_allowed() -> bool:
    """Benchmarks and tests run on seeded random-init weights (BASELINE.json: there is no network for the DINOv2
    download the reference performs, mickey_extractor.py:15-17); they opt in with MICKEY_SYNTHETIC_BACKBONE=1.
    Anyone else loading a real mickey.ckpt (which omits the frozen DINOv2 tensors) without supplying DINOv2 weights
    would silently get poses from a random backbone, so that is an error."""
    import os
    return os.environ.get("MICKEY_SYNTHETIC_BACKBONE", "0") == "1"


def _set_correspondences(data, kps, depth, scr, dsc, grid, down_factor, scores=None, kp_scores=None):
    """The data-dict keys ComputeCorrespondences sets (compute_correspondences.py:52-92) for n pairs: kps [2n,2,N] and
    depth [2n,1,N] hold the image-0 rows first; scr = (scr0, scr1) and dsc = (dsc0, dsc1), [n,.,N] each; scores and
    kp_scores are left out when None (lean outputs).  Every tensor stored is the given tensor or a view of it."""
    gh, gw = grid
    n = kps.shape[0] // 2
    data["kps0_shape"], data["kps1_shape"], data["down_factor"] = [gh, gw], [gh, gw], down_factor
    data["depth0_map"], data["depth1_map"] = depth[:n].reshape(n, 1, gh, gw), depth[n:].reshape(n, 1, gh, gw)
    data["kps0"], data["kps1"] = kps[:n], kps[n:]
    data["depth_kp0"], data["depth_kp1"] = depth[:n], depth[n:]
    data["scr0"], data["scr1"] = scr
    data["dsc0"], data["dsc1"] = dsc
    if scores is not None:
        data["scores"], data["kp_scores"] = scores, kp_scores


def _pose_views(pose):
    """R [B,3,3], t [B,1,3] and the soft inlier count [B,1]: views of the solver's pose [B,13] = R row-major | t | inliers."""
    B = pose.shape[0]
    return pose[:, :9].reshape(B, 3, 3), pose[:, 9:12].reshape(B, 1, 3), pose[:, 12:13]


def _inlier_list(solver, final_scores, kps0, kps1, depth_kp0, depth_kp1):
    """The reference's inlier list (probabilisticProcrustes.py:305-327) from the solver's winning sampled set and its
    hard-inlier mask: per pair, the rows [x0, y0, x1, y1, score, d0, d1] of the set's inlier cells, sorted by score
    descending.  solver: best_set [B], sampled_idx [B*IT_MATCHES, S], inlier_mask [B, S] and status of the solver call.
    Any zero-pose status bit (bits 0-2 from the solver, bit 3 from mk_forward_pairs' index check) gives every pair an
    empty [0, 5] tensor."""
    B, N = kps0.shape[0], final_scores.shape[-1]
    if int(solver["status"].item()) & 15:
        return [torch.zeros([0, 5]) for _ in range(B)]
    cells = solver["sampled_idx"].long()[solver["best_set"].long()]           # [B, S]
    mask = solver["inlier_mask"] > 0.5
    i0, i1 = torch.div(cells, N, rounding_mode="trunc"), cells % N
    bidx = torch.arange(B, device=cells.device)[:, None].expand_as(cells)
    w = final_scores[bidx, i0, i1]
    rows = torch.cat([kps0[bidx, :, i0], kps1[bidx, :, i1], w[..., None], depth_kp0[bidx, :, i0], depth_kp1[bidx, :, i1]], dim=-1)
    out = []
    for b in range(B):
        rb = rows[b][mask[b]]
        out.append(rb[torch.argsort(rb[:, 4], descending=True)])
    return out


class _ParamTree(nn.Module):
    """A module whose only job is to hold tensors under dotted names."""

    def add(self, dotted: str, tensor: torch.Tensor):
        parts = dotted.split(".")
        node = self
        for p in parts[:-1]:
            if p not in node._modules:
                node.add_module(p, _ParamTree())
            node = node._modules[p]
        leaf = parts[-1]
        if leaf in _BUFFER_SUFFIXES:
            node.register_buffer(leaf, tensor.clone())
        else:
            node.register_parameter(leaf, nn.Parameter(tensor.clone(), requires_grad=False))

    def eval(self):            # the reference calls .eval()/.train() on the heads; nothing to switch here
        return super().eval()


class featureMatcher(_ParamTree):
    """Holds the matcher's parameters (matching_mat.dustbin_score) under the reference's names and offers its
    get_matches_list (reference feature_matcher.py:19-46), CUDA-backed (mickey_b200.matches)."""

    def get_matches_list(self, scores, min_conf=0.0):
        """MicKey's correspondences of one pair: scores [1, N, N] fp32 on the GPU (e.g. data['final_scores'][b:b+1]), any
        strides.  Returns int64 [M, 2] (i, j) on its device, sorted by scores[0, i, j] descending, equal scores by ascending
        i.  Like the reference, the last row and column are not candidates.  B != 1 is a ValueError (the reference supports
        batch size 1 only; MickeyRelativePose.mutual_matches takes a batch)."""
        if torch.is_tensor(scores) and scores.dim() == 3 and scores.shape[0] != 1:
            raise ValueError(f"get_matches_list supports batch size 1 (as the reference does), got {tuple(scores.shape)}; "
                             "use MickeyRelativePose.mutual_matches for a batch")
        return mutual_matches(scores, min_conf)[0][0]


REFERENCE_SAMPLED_MATCHES = 2048


def check_sampled_matches(n):
    """The drop-in solvers accept PROCRUSTES.NUM_SAMPLED_MATCHES = 2048 only.  The reference's estimate_pose_vectorized
    reshapes its point tensors to 2048 samples per set (probabilisticProcrustes.py:271-272), so under any other value it
    raises inside its try and returns the zero pose on every call; the CUDA solver (mk_solve_pose, mk_procrustes_solve)
    would return real poses instead.  Such a configuration is rejected rather than silently generalised."""
    if n != REFERENCE_SAMPLED_MATCHES:
        raise ValueError(f"PROCRUSTES.NUM_SAMPLED_MATCHES must be {REFERENCE_SAMPLED_MATCHES}, got {n}: the reference "
                         "reshapes its sampled sets to 2048 entries (probabilisticProcrustes.py:271-272) and returns the "
                         "zero pose on every call under any other value")


class e2eProbabilisticProcrustesSolver:
    """Test-time metric pose solver (reference probabilisticProcrustes.py:5-20, 183-348), CUDA-backed."""

    def __init__(self, cfg, owner: "MickeyRelativePose"):
        p = cfg.PROCRUSTES
        self.it_RANSAC = p.IT_RANSAC
        self.it_matches = p.IT_MATCHES
        self.num_samples_matches = p.NUM_SAMPLED_MATCHES
        self.num_corr_3d_3d = p.NUM_CORR_3D_3D
        self.num_refinements = p.NUM_REFINEMENTS
        self.th_inlier = p.TH_INLIER
        self.th_soft_inlier = p.TH_SOFT_INLIER
        check_sampled_matches(self.num_samples_matches)
        self._owner = owner

    def estimate_pose_vectorized(self, batch, return_inliers=False, outer_idx=None, inner_idx=None, seed=None):
        eng = self._owner._engine()
        final = batch["final_scores"].detach().float()      # a padded-pitch view goes to the kernels as it is
        kps = torch.cat([batch["kps0"], batch["kps1"]], 0).detach().float().contiguous()
        depth = torch.cat([batch["depth_kp0"], batch["depth_kp1"]], 0).detach().float().contiguous()
        if seed is None:
            seed = int(torch.randint(1, 2 ** 62, (1,)).item())     # follows torch.manual_seed like the reference
        res = eng.solve(final, kps, depth, batch["K_color0"], batch["K_color1"], seed, outer_idx=outer_idx, inner_idx=inner_idx)
        R, t, inliers = (v.contiguous() for v in _pose_views(res["pose"]))
        batch["_solver"] = res
        if not return_inliers:
            return R, t, inliers
        return R, t, inliers, _inlier_list(res, final, batch["kps0"], batch["kps1"], batch["depth_kp0"], batch["depth_kp1"])


class ComputeCorrespondences(nn.Module):
    """Extraction + matching (reference compute_correspondences.py:6-92), CUDA-backed."""

    def __init__(self, cfg, owner: "MickeyRelativePose"):
        super().__init__()
        object.__setattr__(self, "_owner", owner)
        self.dsc_dim = cfg["MICKEY"]["DSC_HEAD"]["LAST_DIM"]
        self.down_factor = cfg["MICKEY"]["DINOV2"]["DOWN_FACTOR"]
        self.extractor = _ParamTree()
        self.matcher = featureMatcher()

    def forward(self, data):
        eng = self._owner._engine()
        im0, im1 = data["image0"], data["image1"]
        B = im0.shape[0]
        if im0.shape != im1.shape:
            raise ValueError(f"image0 {tuple(im0.shape)} and image1 {tuple(im1.shape)} must have the same shape (both images "
                             "of a batch are extracted in one call)")
        images = torch.cat([im0, im1], dim=0)
        kps, depth, scr, dsc = eng.extract(images)
        H, W = eng.geo
        scores, kp_scores, final = eng.match(B, kps.shape[-1], lean=bool(getattr(self._owner, "lean_outputs", False)))
        _set_correspondences(data, kps, depth, (scr[:B], scr[B:]), (dsc[:B], dsc[B:]), (H // PATCH, W // PATCH),
                             self.down_factor, scores, kp_scores)
        data["_final_scores_fused"] = final
        return data["kps0"], data["dsc0"], data["kps1"], data["dsc1"]


class MickeyRelativePose(nn.Module):
    """Metric relative pose between two images (reference compute_pose.py:6-60)."""

    def __init__(self, cfg, dinov2_weights=None):
        """dinov2_weights: optional DINOv2 state dict (native names: 'cls_token', 'blocks.0.attn.qkv.weight', ...)
        or a path to one — the stand-in for the reference's download (mickey_extractor.py:15-17; there is no network
        here).  Also read from $MICKEY_DINOV2_WEIGHTS.  Without it the backbone keeps seeded random-init values."""
        super().__init__()
        if cfg.MODEL is not None and cfg.MODEL != "MicKey":
            raise NotImplementedError()
        self.cfg = cfg
        self.variant = backbone_variant(cfg)
        self.compute_matches = ComputeCorrespondences(cfg, self)
        self.e2e_Procrustes = e2eProbabilisticProcrustesSolver(cfg, self)
        # parameter storage under the reference's names; values are placeholders until a checkpoint loads
        # (the reference downloads DINOv2 here, mickey_extractor.py:15-17 — there is no network on the box)
        for name, t in synthetic_state_dict(cfg, seed=0).items():
            assert name.startswith("compute_matches.")
            self.compute_matches.__getattr__(name.split(".")[1]).add(".".join(name.split(".")[2:]), t)
        import os
        dinov2_weights = dinov2_weights or os.environ.get("MICKEY_DINOV2_WEIGHTS")
        self.__dict__["_backbone_is_synthetic"] = dinov2_weights is None
        if dinov2_weights is not None:
            if isinstance(dinov2_weights, str):
                dinov2_weights = torch.load(dinov2_weights, map_location="cpu")
            own = self.state_dict()
            pre = "compute_matches.extractor.dinov2_vitl14."
            missing = [k for k in own if k.startswith(pre) and k[len(pre):] not in dinov2_weights]
            if missing:
                raise KeyError(f"DINOv2 weights lack {missing[:3]} ...")
            super().load_state_dict({**own, **{pre + k: v for k, v in dinov2_weights.items() if pre + k in own}})
        self.__dict__["_eng"] = None
        self.__dict__["_eng_version"] = -1
        self.__dict__["_param_version"] = 0
        self.is_eval_model(True)

    # -- checkpoint plumbing (compute_pose.py:39-48, builder.py:11-13) ---------------------------------------
    def on_load_checkpoint(self, checkpoint):
        """compute_pose.py:39-48: the checkpoint's (absent) DINOv2 tensors are filled from the module's own backbone.
        The reference's own backbone is the downloaded pretrained DINOv2; here it must have been supplied
        (`dinov2_weights=` / $MICKEY_DINOV2_WEIGHTS) unless synthetic weights were explicitly allowed."""
        if self.__dict__.get("_backbone_is_synthetic", True) and not synthetic_backbone_allowed():
            raise RuntimeError(
                "MickeyRelativePose holds seeded RANDOM DINOv2 weights: the reference downloads the pretrained ViT at this "
                "point (mickey_extractor.py:15-17) and there is no network here.  Pass dinov2_weights= (or set "
                "$MICKEY_DINOV2_WEIGHTS to a dinov2_vit*14_pretrain.pth), or set MICKEY_SYNTHETIC_BACKBONE=1 to run on "
                "synthetic weights on purpose (benchmarks / tests).")
        own = self.compute_matches.state_dict()
        for k in own:
            if "dinov2" in k:
                checkpoint["state_dict"]["compute_matches." + k] = own[k]

    def load_state_dict(self, state_dict, strict=True, **kw):
        res = super().load_state_dict(state_dict, strict=strict, **kw)
        self.__dict__["_param_version"] += 1
        return res

    def _apply(self, fn, *a, **k):
        res = super()._apply(fn, *a, **k)
        self.__dict__["_param_version"] += 1
        return res

    def is_eval_model(self, is_eval):
        return None        # BatchNorm is folded at load time: always eval semantics

    def _engine_pool(self):
        """pipeline_depth engines (default 1).  With depth 2, consecutive forward() calls alternate between two engines
        that own separate workspaces, CUDA graphs, RNG state and streams but share one copy of the packed weights."""
        depth = int(getattr(self, "pipeline_depth", 1))
        first = self._engine()
        pool = self.__dict__.setdefault("_pool", [])
        if len(pool) != depth - 1 or self.__dict__.get("_pool_version") != self._eng_version or (pool and pool[0].device != first.device):
            pool.clear()
            for _ in range(depth - 1):
                e = Engine(self.cfg, first.device, side_stream=True)
                e.load_state_dict(None, share_with=first)
                pool.append(e)
            self.__dict__["_pool_version"] = self._eng_version
        if depth > 1:
            first.use_side_stream()
        engines = [first] + pool
        for e in engines:
            e.assume_inputs_ready = bool(getattr(self, "assume_inputs_ready", False))
        return engines

    def _engine(self) -> Engine:
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("mickey_b200 runs on CUDA only: move the model to an H100 with .cuda() "
                               "(there is no CPU fallback)")
        if self._eng is None or self._eng.device != dev:
            self.__dict__["_eng"] = Engine(self.cfg, dev)
            self.__dict__["_eng_version"] = -1
        if self._eng_version != self._param_version:
            self._eng.load_state_dict(self.state_dict())
            self.__dict__["_eng_version"] = self._param_version
        return self._eng

    # -- the hot path ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, data, return_inliers=False):
        """One C call (mk_forward) per batch, replayed from a CUDA graph after the first two calls.
        `self.static_outputs = True` hands out the engine's static output buffers directly (they are overwritten by the
        forward after the next one of the same geometry on the same engine; with pipeline_depth > 1 under
        assume_inputs_ready or with host inputs, reads of them must have completed before that call is issued, see
        Engine.forward); the default clones them so that every call returns fresh
        tensors like the reference does.  `self.lean_outputs = True` skips data['scores'] / data['kp_scores'] (the solver
        only reads final_scores): 17 instead of 47 MB of N x N traffic per 720x540 pair."""
        if getattr(self, "staged", False):
            return self.forward_staged(data, return_inliers)
        pool = self._engine_pool()
        turn = self.__dict__.get("_turn", 0)
        self.__dict__["_turn"] = turn + 1
        eng = pool[turn % len(pool)]
        im0, im1 = data["image0"], data["image1"]
        B = im0.shape[0]
        seed = int(torch.randint(1, 2 ** 62, (1,)).item())
        # uint8 [B,H,W,3] goes to the ingest kernel as it is (mickey_b200.io); other dtypes (fp64 K, say) are converted by
        # the engine's copies into its fp32 input buffers, on the stream that also reads them
        st = eng.forward(im0, im1, data["K_color0"], data["K_color1"], seed,
                         use_graph=getattr(self, "use_graph", True), lean=bool(getattr(self, "lean_outputs", False)))
        static = getattr(self, "static_outputs", False)
        keep = (lambda t: t) if static else (lambda t: None if t is None else t.clone())   # None: lean_outputs
        H, W = eng.geo
        kps, depth, scr, dsc = keep(st["kps"]), keep(st["depth"]), keep(st["scr"]), keep(st["dsc"])
        _set_correspondences(data, kps, depth, (scr[:B], scr[B:]), (dsc[:B], dsc[B:]), (H // PATCH, W // PATCH),
                             self.compute_matches.down_factor, keep(st["scores"]), keep(st["kp_scores"]))
        data["final_scores"] = keep(st["final_scores"])
        R, t, inliers = _pose_views(keep(st["pose"]))
        if return_inliers:
            data["inliers_list"] = _inlier_list(st, data["final_scores"], data["kps0"], data["kps1"], data["depth_kp0"],
                                                data["depth_kp1"])
        if not static:
            eng.release()                                # every read of the static buffers above is queued
        data["R"], data["t"], data["inliers"] = R, t, inliers
        return R, t

    @torch.no_grad()
    def forward_staged(self, data, return_inliers=False):
        """The same path as three C calls (mk_extract / mk_match / mk_solve_pose), mirroring the reference's
        structure (compute_pose.py:20-37); used by the stage-wise tests."""
        self.compute_matches(data)
        # final_scores = scores * kp_scores (compute_pose.py:23) is produced by the matcher kernel's epilogue
        data["final_scores"] = data.pop("_final_scores_fused")
        if return_inliers:
            R, t, inliers, inliers_list = self.e2e_Procrustes.estimate_pose_vectorized(data, return_inliers=True)
            data["inliers_list"] = inliers_list
        else:
            R, t, inliers = self.e2e_Procrustes.estimate_pose_vectorized(data, return_inliers=False)
        data.pop("_solver", None)
        data["R"] = R
        data["t"] = t
        data["inliers"] = inliers
        return R, t

    # -- feature banks: extract each image once, pose for any (i, j) among them --------------------------------------
    @torch.no_grad()
    def extract_features(self, images: torch.Tensor) -> MickeyFeatures:
        """Features of n images, float [n, 3, H, W] in [0, 1] or uint8 [n, H, W, 3] RGB, in one extraction call.  Each
        image's features are bit-identical to what forward() computes for it, whatever role it plays there."""
        eng = self._engine()
        if images.dtype != torch.uint8:
            images = images.float()
        kps, depth, scr, dsc = eng.extract_images(images.to(eng.device))
        H, W = eng.geo
        return MickeyFeatures(kps, depth, scr, dsc, (H // PATCH, W // PATCH), (H, W))

    @torch.no_grad()
    def pose_from_features(self, feats0: MickeyFeatures, idx0, feats1: MickeyFeatures, idx1, K_color0, K_color1,
                           return_inliers: bool = False) -> dict:
        """Relative pose of the P pairs (feats0[idx0[p]], feats1[idx1[p]]) from features extract_features computed.

        idx0 / idx1: host lists or tensors of P image indices (validated on the host: MickeyB200Error before anything is
        launched).  K_color0 / K_color1: [P, 3, 3] intrinsics of each pair.  Returns the data dict forward() fills for
        those pairs (kps0/1, depth_kp0/1, scr0/1, dsc0/1, depth0/1_map, kps0/1_shape, down_factor, scores, kp_scores
        (absent under lean_outputs), final_scores, R, t, inliers, and inliers_list with return_inliers).  One seed is
        drawn from the torch RNG as in forward(), so under the same seed the poses equal forward() on the explicit pairs."""
        i0, i1 = validate_pairs(feats0, idx0, feats1, idx1)
        P = len(i0)
        K0, K1 = torch.as_tensor(K_color0), torch.as_tensor(K_color1)
        if tuple(K0.shape) != (P, 3, 3) or tuple(K1.shape) != (P, 3, 3):
            raise MickeyB200Error(f"K_color0 {tuple(K0.shape)} / K_color1 {tuple(K1.shape)} must be [{P}, 3, 3]")
        eng = self._engine()
        if feats0.device != eng.device:
            raise MickeyB200Error(f"features on {feats0.device}, model on {eng.device}")
        seed = int(torch.randint(1, 2 ** 62, (1,)).item())
        dev = eng.device
        t0 = torch.tensor(i0, dtype=torch.int32).to(dev, non_blocking=True)
        t1 = torch.tensor(i1, dtype=torch.int32).to(dev, non_blocking=True)
        bank0 = tuple(t.float().contiguous() for t in feats0.tensors())
        bank1 = tuple(t.float().contiguous() for t in feats1.tensors())
        st = eng.forward_pairs(bank0, t0, bank1, t1, K0.float(), K1.float(), seed, feats0.image_size,
                               lean=bool(getattr(self, "lean_outputs", False)))
        data = {}
        _set_correspondences(data, st["kps"], st["depth"],
                             (bank0[2].index_select(0, t0.long()), bank1[2].index_select(0, t1.long())),
                             (bank0[3].index_select(0, t0.long()), bank1[3].index_select(0, t1.long())),
                             feats0.grid, self.compute_matches.down_factor, st["scores"], st["kp_scores"])
        data["final_scores"] = st["final_scores"]
        data["R"], data["t"], data["inliers"] = _pose_views(st["pose"])
        if return_inliers:
            data["inliers_list"] = _inlier_list(st, data["final_scores"], data["kps0"], data["kps1"], data["depth_kp0"],
                                                data["depth_kp1"])
        return data

    # -- localization: queries against cached references, the queries alone extracted -----------------------------------
    @torch.no_grad()
    def localize(self, reference: MickeyFeatures, ref_idx, queries, K_color0, K_color1, return_inliers: bool = False) -> dict:
        """Relative pose of P pairs (reference[ref_idx[p]], queries[p]) in one C call (mk_localize): only the queries are
        extracted, the references' features come from extract_features.

        queries: float [P, 3, H, W] in [0, 1] or uint8 [P, H, W, 3] RGB, on the model's device or on the host (pinned
        host frames are copied on a side stream, overlapped with the previous call); ref_idx: host list or tensor of P
        indices into `reference`, whose token grid must be the queries'; K_color0 / K_color1: [P, 3, 3].  Everything is
        validated on the host (MickeyB200Error before anything is launched or a seed drawn).  Returns the data dict
        pose_from_features returns for the same pairs, with the same keys and lean_outputs behaviour; one seed is drawn
        from the torch RNG as in forward(), so under the same seed every output equals forward() on the explicit pairs.
        Like forward(), it replays a CUDA graph from the third call of a shape on, follows pipeline_depth,
        assume_inputs_ready and static_outputs, and keeps its own copy of the reference bank for the graph to read
        (Engine.localize: refreshed when other tensors are passed or theirs change in place)."""
        idx = validate_localize(reference, ref_idx, queries, K_color0, K_color1)
        dev = next(self.parameters()).device
        if reference.device != dev:
            raise MickeyB200Error(f"reference on {reference.device}, model on {dev}")
        pool = self._engine_pool()
        turn = self.__dict__.get("_turn", 0)
        self.__dict__["_turn"] = turn + 1
        eng = pool[turn % len(pool)]
        seed = int(torch.randint(1, 2 ** 62, (1,)).item())
        bank = tuple(t.float().contiguous() for t in reference.tensors())
        ridx = torch.tensor(idx, dtype=torch.int32).pin_memory()
        if queries.dtype != torch.uint8:
            queries = queries.float()
        st = eng.localize(bank, ridx, queries, K_color0, K_color1, seed, use_graph=getattr(self, "use_graph", True),
                          lean=bool(getattr(self, "lean_outputs", False)))
        static = getattr(self, "static_outputs", False)
        keep = (lambda t: t) if static else (lambda t: None if t is None else t.clone())   # None: lean_outputs
        gidx = st["ref_idx"]                             # ref_idx on the device, in the engine's buffer set
        data = {}
        _set_correspondences(data, keep(st["kps"]), keep(st["depth"]), (bank[2].index_select(0, gidx), keep(st["scr"])),
                             (bank[3].index_select(0, gidx), keep(st["dsc"])), reference.grid, self.compute_matches.down_factor,
                             keep(st["scores"]), keep(st["kp_scores"]))
        data["final_scores"] = keep(st["final_scores"])
        data["R"], data["t"], data["inliers"] = _pose_views(keep(st["pose"]))
        if return_inliers:
            data["inliers_list"] = _inlier_list(st, data["final_scores"], data["kps0"], data["kps1"], data["depth_kp0"],
                                                data["depth_kp1"])
        if not static:
            eng.release()                                # every read of the static buffers above is queued
        return data

    @torch.no_grad()
    def mutual_matches(self, scores, min_conf: float = 0.0):
        """get_matches_list (reference feature_matcher.py:19-46) of every pair of scores [B, N, N] fp32 on the GPU, e.g.
        data['final_scores'] after forward(): a list of B int64 [M_b, 2] tensors (i, j) and a list of their B fp32 [M_b]
        scores, each sorted by score descending, equal scores by ascending i.  Two kernel launches for the whole batch and
        one device-to-host copy of the counts."""
        return mutual_matches(scores, min_conf)


def build_model(cfg, checkpoint=""):
    """Mirror of reference lib/models/builder.py:5-20.  `checkpoint` may be a path (torch.load) or an
    already loaded dict {'state_dict': ...}."""
    if cfg.MODEL == "MicKey":
        model = MickeyRelativePose(cfg)
        ckpt = checkpoint if isinstance(checkpoint, dict) else torch.load(checkpoint, map_location="cpu")
        model.on_load_checkpoint(ckpt)
        model.load_state_dict(ckpt["state_dict"])
        if torch.cuda.is_available():
            model = model.cuda()
        model.eval()
        return model
    raise NotImplementedError()
