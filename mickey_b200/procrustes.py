"""MicKey's metric pose solver for callers without an inference engine: a drop-in for the reference's
e2eProbabilisticProcrustesSolver (lib/models/MicKey/modules/utils/probabilisticProcrustes.py:5-20, 183-348) on
mk_procrustes_solve, the handle-free entry of the CUDA solver that MickeyRelativePose runs.

The training model calls the solver in validation_step (lib/models/MicKey/model.py:66-89) and, with return_inliers, in
the logging of backward_step (:164).  The reference's estimate_pose_vectorized materialises a [B * IT_MATCHES, N * N]
copy of final_scores for torch.multinomial and [B * IT_MATCHES * IT_RANSAC, NUM_SAMPLED_MATCHES, 3] point tensors,
several GB at the validation shapes; here the whole solve runs in a workspace of a few MB and reads final_scores in place.

    from mickey_b200.procrustes import e2eProbabilisticProcrustesSolver
    model.e2e_Procrustes = e2eProbabilisticProcrustesSolver(model.cfg)   # or mickey_b200.training.use_cuda_modules(model, solver=True)
"""
from __future__ import annotations

import math

import torch

from . import _lib
from .model import _inlier_list, _pose_views, check_sampled_matches

# include/mickey_b200.h, mk_procrustes_solve's sizes
MAX_GRID, INT_MAX = 65535, 2 ** 31 - 1
STATUS_ZERO = 1 | 2 | 4          # the status bits that give the zero result


class e2eProbabilisticProcrustesSolver:
    """Drop-in for the reference class, built from cfg.PROCRUSTES: the same attributes, and estimate_pose_vectorized with
    the reference's results, computed by the CUDA solver.  It holds no parameters, buffers or state across calls."""

    def __init__(self, cfg):
        p = cfg.PROCRUSTES
        self.it_RANSAC = p.IT_RANSAC
        self.it_matches = p.IT_MATCHES
        self.num_samples_matches = p.NUM_SAMPLED_MATCHES
        self.num_corr_3d_3d = p.NUM_CORR_3D_3D
        self.num_refinements = p.NUM_REFINEMENTS
        self.th_inlier = p.TH_INLIER
        self.th_soft_inlier = p.TH_SOFT_INLIER
        # the kernels' limits, checked here so that an unsupported configuration fails at construction
        if not 1 <= self.it_matches <= MAX_GRID:
            raise ValueError(f"PROCRUSTES.IT_MATCHES must be in [1, {MAX_GRID}], got {self.it_matches}")
        if not (self.it_RANSAC >= 1 and self.it_matches * self.it_RANSAC <= INT_MAX):
            raise ValueError(f"PROCRUSTES.IT_RANSAC must be >= 1 with IT_MATCHES * IT_RANSAC < 2^31, got {self.it_RANSAC}")
        check_sampled_matches(self.num_samples_matches)      # 2048 only: the reference's own limit, inside the kernels'
        if self.num_corr_3d_3d != 3:
            raise ValueError(f"PROCRUSTES.NUM_CORR_3D_3D must be 3, got {self.num_corr_3d_3d}")
        if self.num_refinements < 0:
            raise ValueError(f"PROCRUSTES.NUM_REFINEMENTS must be >= 0, got {self.num_refinements}")
        for name in ("th_inlier", "th_soft_inlier"):
            v = getattr(self, name)
            if not (math.isfinite(v) and v > 0):
                raise ValueError(f"PROCRUSTES.{name.upper()} must be finite and positive, got {v}")

    def estimate_pose_vectorized(self, batch, return_inliers=False, outer_idx=None, inner_idx=None, seed=None):
        """The pose of every pair of batch: final_scores [B, N, N] fp32 (any strides; it may require grad), kps0 / kps1
        [B, 2, N], depth_kp0 / depth_kp1 [B, 1, N] and K_color0 / K_color1 [B, 3, 3], on one CUDA device, all read
        detached: no autograd graph is built and no .grad is touched, under no_grad, inference_mode or grad mode alike.

        Returns R [B, 3, 3], t [B, 1, 3] and best_inliers, the soft inlier count, [B, 1] as the reference's
        soft_inlier_counting_3d returns it, and with return_inliers the per-pair inlier lists of the reference
        ([M_b, 7] rows x0, y0, x1, y1, score, d0, d1, sorted by score descending, on final_scores' device).  Where the
        reference takes its except branch or ends with num_valid_h == 0 (:331-342: a NaN, inf or negative cell, a pair
        whose scores sum to zero or hold fewer than NUM_SAMPLED_MATCHES cells, a non-finite hypothesis), the result is
        its zero result for the whole batch: R and t zero, best_inliers zeros [B], and B empty [0, 5] tensors on the CPU
        (the reference's torch.zeros([0, 5])).

        One seed is drawn from the torch RNG per call (so results follow torch.manual_seed); `seed` overrides it, and
        outer_idx [B * IT_MATCHES, NUM_SAMPLED_MATCHES] / inner_idx [B * IT_MATCHES * IT_RANSAC, 3] replace the two
        draws.  batch['_solver'] receives the solver's outputs: pose, best_set, inlier_mask, sampled_idx, hyp_scores
        and status."""
        fs = batch["final_scores"].detach()
        if fs.dim() != 3 or fs.shape[1] != fs.shape[2] or fs.device.type != "cuda":
            raise ValueError(f"final_scores must be a CUDA [B, N, N] tensor, got {tuple(fs.shape)} on {fs.device} "
                             "(mickey_b200 has no CPU path)")
        B, N = fs.shape[0], fs.shape[1]
        IM, IR, S = self.it_matches, self.it_RANSAC, self.num_samples_matches
        dev = fs.device
        fs, pitch = _lib.pitched(fs.float())
        f32 = lambda t: t.detach().to(dev, torch.float32).contiguous()
        kps = f32(torch.cat([batch["kps0"].detach(), batch["kps1"].detach()], 0))
        depth = f32(torch.cat([batch["depth_kp0"].detach(), batch["depth_kp1"].detach()], 0))
        K0, K1 = f32(batch["K_color0"]), f32(batch["K_color1"])
        oi, ii = (None if i is None else i.to(dev, torch.int32).contiguous() for i in (outer_idx, inner_idx))
        if oi is not None and tuple(oi.shape) != (B * IM, S):
            raise ValueError(f"outer_idx must be [B*IT_MATCHES, NUM_SAMPLED_MATCHES] = [{B * IM}, {S}], got {tuple(oi.shape)}")
        if ii is not None and tuple(ii.shape) != (B * IM * IR, 3):
            raise ValueError(f"inner_idx must be [B*IT_MATCHES*IT_RANSAC, 3] = [{B * IM * IR}, 3], got {tuple(ii.shape)}")
        if seed is None:
            seed = int(torch.randint(1, 2 ** 62, (1,)).item())     # follows torch.manual_seed like the reference
        lib = _lib.load()
        with torch.cuda.device(dev):
            res = {"pose": torch.empty(B, 13, device=dev), "best_set": torch.empty(B, dtype=torch.int32, device=dev),
                   "inlier_mask": torch.empty(B, S, device=dev),
                   "sampled_idx": torch.empty(B * IM, S, dtype=torch.int32, device=dev),
                   "hyp_scores": torch.empty(B, IM * IR, device=dev), "status": torch.zeros(1, dtype=torch.int32, device=dev)}
            ws = _lib.workspace(lib.mk_procrustes_ws_bytes(B, N, IM, IR, S), dev, "mk_procrustes_ws_bytes")
            p = _lib.ptr
            _lib.check(lib.mk_procrustes_solve(
                p(fs), pitch, p(kps), p(depth), p(K0), p(K1), B, N, IM, IR, S, self.num_corr_3d_3d, self.num_refinements,
                self.th_inlier, self.th_soft_inlier, seed & (2 ** 64 - 1), p(oi), p(ii), p(res["pose"]), p(res["best_set"]),
                p(res["inlier_mask"]), p(res["sampled_idx"]), p(res["hyp_scores"]), p(res["status"]), p(ws), ws.numel(),
                _lib.stream(dev)), "mk_procrustes_solve")
        batch["_solver"] = res
        R, t, inliers = (v.contiguous() for v in _pose_views(res["pose"]))   # the kernel wrote the zero pose on failure
        if int(res["status"].item()) & STATUS_ZERO:
            inliers = inliers.reshape(B)
        if not return_inliers:
            return R, t, inliers
        kps0, kps1 = kps[:B], kps[B:]
        return R, t, inliers, _inlier_list(res, fs, kps0, kps1, depth[:B], depth[B:])
