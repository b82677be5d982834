"""MicKey's training loss, MetricPoseLoss (reference lib/models/MicKey/modules/loss/loss_class.py), on the GPU.

The parts that are expensive and not differentiated run in CUDA (csrc/loss.cu): the two torch.multinomial draws, the
refinement search of every hypothesis (:163-196) and the dense REINFORCE gradient over the N x N match probabilities
(:251-261, :299-316).  The small differentiable tail runs in autograd, exactly where the reference keeps gradients: one
weighted Procrustes per hypothesis on its final inlier mask, the soft inlier score, the VCRE / POSE_ERR loss, the score
softmax with the null hypothesis, the baseline and the curriculum top-K.  So `avg_loss.backward()` fills the kps / depth
leaves of `outputs` through torch's own SVD backward, as in the reference.  MetricPoseLoss(cfg, cuda_tail=True) runs that
tail in CUDA instead (csrc/loss_tail.cu, LossTail): the same arithmetic in fp64 and a closed-form backward with no SVD.

Only `RANSAC_vectorized` is restated: the reference hard-codes `use_RANSAC_vectorized = True`.

Edge behaviour follows the reference:
- A NaN, inf or negative cell anywhere in final_scores (:126-131), a matrix torch.multinomial rejects (:269-276) or a set
  whose scores sum to zero: no search; baseline, losses and gradients are zero and num_valid_h = 0.
- A NaN or inf in any hypothesis's R or t (:213-223) gives the same zero result.  The rank check is off, as
  `RANSAC_vectorized` passes `check_rank=False`.
- With top-K and B > 1 the zero result gives avg_loss = 0 / 0 = NaN; the reference's `backward_step` tests num_valid_h
  first.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib

STATUS_PRECHECK, STATUS_INNER = 16, 32          # include/mickey_b200.h MK_LOSS_STATUS_*
STATUS_SKIP = 1 | 2 | STATUS_PRECHECK | STATUS_INNER
LOSS_MAX_S, LOSS_MAX_C = 2048, 16              # csrc/ops.h: largest NUM_SAMPLES_MATCHES and NUM_CORR_3d3d


def vcre_grid(device=None) -> torch.Tensor:
    """The virtual-correspondence grid of lib/benchmarks/reprojection.py:32-56 (7 x 4 x 7 points, step 0.3 m, 1.8 m in
    front of the camera), [196, 3] fp64, in np.meshgrid's 'xy' order."""
    step = 0.3
    x = (torch.arange(7, dtype=torch.float64) - 3.0) * step
    y = (torch.arange(4, dtype=torch.float64) - 1.5) * step
    z = torch.arange(7, dtype=torch.float64) * step + 1.8
    yy, xx, zz = torch.meshgrid(y, x, z, indexing="ij")          # shape (4, 7, 7), as np.meshgrid(x, y, z)
    return torch.stack([xx.reshape(-1), yy.reshape(-1), zz.reshape(-1)], -1).to(device)


# ---- the differentiable tail: restatements of the reference's helpers --------------------------------------------
def backproject_3d(uv, depth, K):
    """training_utils.py:7-22: uv [B, n, 2], depth [B, n, 1], K [B, 3, 3] -> [B, n, 3]."""
    uv1 = torch.cat([uv, torch.ones_like(uv[..., :1])], -1)
    return depth * (torch.linalg.inv(K) @ uv1.transpose(2, 1)).transpose(2, 1)


def weighted_procrustes(A, B, w, eps=1e-16):
    """solvers.py:3-54 with use_weights=True, use_mask=True, check_rank=False: returns (R, t)."""
    W1 = torch.abs(w).sum(1, keepdim=True)
    w_norm = (w / (W1 + eps)).unsqueeze(-1)
    a_mean = (w_norm * A).sum(1, keepdim=True)
    b_mean = (w_norm * B).sum(1, keepdim=True)
    H = (A - a_mean).transpose(1, 2) @ (w.unsqueeze(-1) * (B - b_mean))
    U, _, V = torch.svd(H)
    Z = torch.eye(3, dtype=A.dtype, device=A.device).unsqueeze(0).repeat(A.shape[0], 1, 1)
    Z[:, -1, -1] = torch.sign(torch.linalg.det(U @ V.transpose(1, 2)))
    R = V @ Z @ U.transpose(1, 2)
    return R, b_mean - a_mean @ R.transpose(1, 2)


def soft_inlier_counting_3d(X0, X1, R, t, th):
    """training_utils.py:55-61."""
    d = ((((R @ X0.transpose(2, 1)).transpose(2, 1) + t - X1) ** 2.0).sum(-1) + 1e-6) ** 0.5
    return torch.sigmoid(5.0 / th * (th - d)).sum(-1).view(X0.shape[0], 1)


def rot_angle_loss(R, Rgt):
    """loss_utils.py:95-110."""
    cosine = (torch.diagonal(R.transpose(1, 2) @ Rgt, dim1=-2, dim2=-1).sum(-1) - 1) / 2
    return torch.acos(torch.clip(cosine, -0.99999, 0.99999)).abs().unsqueeze(-1)


def trans_l1_loss(t, tgt):
    """loss_utils.py:85-93."""
    return torch.abs(t - tgt).sum(-1)


def project_2d(XYZ, K):
    """training_utils.py:24-35."""
    xyz = (K @ XYZ.transpose(2, 1)).transpose(2, 1)
    return (xyz / (xyz[:, :, 2:3] + 1e-16))[:, :, :2]


def vcre_loss(R, t, Rgt, tgt, K, grid, H=720):
    """lib/utils/metrics.py:56-80 (Tgt given as Rgt [B, 3, 3], tgt [B, 1, 3])."""
    eye = grid.to(R.dtype).unsqueeze(0).expand(R.shape[0], -1, -1)
    uv_gt = project_2d(eye, K)
    tmp = R @ eye.transpose(2, 1) + t.transpose(2, 1)
    res = (Rgt.transpose(2, 1) @ tmp - Rgt.transpose(2, 1) @ tgt.transpose(2, 1)).transpose(2, 1)
    uv_pred = project_2d(res, K)
    d = ((torch.clip(uv_gt, 0, H) - torch.clip(uv_pred, 0, H)) ** 2.0).sum(-1)
    return ((d + 1e-6) ** 0.5).mean(-1).view(R.shape[0], 1)


def compute_vcre_loss(R, t, Rgt, tgt, K0, K1, grid, soft_clipping):
    """loss_utils.py:40-66."""
    R_inv = R.transpose(2, 1)
    t_inv = (-1 * R_inv @ t.transpose(2, 1)).transpose(2, 1)
    Rgt_inv = Rgt.transpose(2, 1)
    tgt_inv = (-1 * Rgt_inv @ tgt.transpose(2, 1)).transpose(2, 1)
    loss = (vcre_loss(R_inv, t_inv, Rgt_inv, tgt_inv, K1, grid) + vcre_loss(R, t, Rgt, tgt, K0, grid)) / 2.0
    if soft_clipping:
        loss = torch.tanh(loss / 80)
    return loss, rot_angle_loss(R, Rgt), trans_l1_loss(t, tgt)


def compute_pose_loss(R, t, Rgt, tgt, K0, K1, grid, soft_clipping):
    """loss_utils.py:26-38."""
    loss_rot, loss_trans = rot_angle_loss(R, Rgt), trans_l1_loss(t, tgt)
    if soft_clipping:
        return torch.tanh(loss_rot / 0.9) + torch.tanh(loss_trans / 0.9), loss_rot, loss_trans
    return loss_rot + loss_trans, loss_rot, loss_trans


def unpack_mask(bits: torch.Tensor, S: int) -> torch.Tensor:
    """uint32 words [H, S/32] as written by mk_loss_search (int32 storage) -> {0, 1} fp32 [H, S]."""
    sh = torch.arange(32, device=bits.device, dtype=torch.int64)
    return ((bits.to(torch.int64).unsqueeze(-1) >> sh) & 1).reshape(bits.shape[0], S).float()


class LossParams:
    """The LOSS_CLASS keys of the reference config (curriculum_learning.yaml:55-87) that MetricPoseLoss reads."""

    def __init__(self, cfg):
        lc = cfg.LOSS_CLASS
        g = lc.GENERATE_HYPOTHESES
        self.loss_type, self.soft_clipping = lc.LOSS_FUNCTION, bool(lc.SOFT_CLIPPING)
        if self.loss_type not in ("VCRE", "POSE_ERR"):
            raise ValueError(f"LOSS_CLASS.LOSS_FUNCTION must be VCRE or POSE_ERR, got {self.loss_type!r}")
        sub = lc.VCRE if self.loss_type == "VCRE" else lc.POSE_ERR
        self.max_loss_null = float(sub.MAX_LOSS_SOFTVALUE if self.soft_clipping else sub.MAX_LOSS_VALUE)
        self.n_sample = int(lc.SAMPLER.NUM_SAMPLES_MATCHES)
        self.score_temperature = float(g.SCORE_TEMPERATURE)
        self.it_matches, self.it_ransac = int(g.IT_MATCHES), int(g.IT_RANSAC)
        self.inlier_3d_th, self.inlier_ref_th = float(g.INLIER_3D_TH), float(g.INLIER_REF_TH)
        self.num_ref_steps, self.num_corr = int(g.NUM_REF_STEPS), int(g.NUM_CORR_3d3d)
        self.add_null_hypothesis = bool(lc.NULL_HYPOTHESIS.ADD_NULL_HYPOTHESIS)
        self.th_outliers = float(lc.NULL_HYPOTHESIS.TH_OUTLIERS)
        cl = lc.CURRICULUM_LEARNING
        self.train_w_top = bool(cl.TRAIN_WITH_TOPK or cl.TRAIN_CURRICULUM)
        self.topK = cl.TOPK_INIT if cl.TRAIN_CURRICULUM else (cl.TOPK if cl.TRAIN_WITH_TOPK else None)
        # mk_loss_search's limits, checked here so that an unsupported config fails at construction, not at the first
        # forward: the inlier masks are 32-bit words, one bit per set entry
        if not (0 < self.n_sample <= LOSS_MAX_S and self.n_sample % 32 == 0):
            raise ValueError(f"SAMPLER.NUM_SAMPLES_MATCHES must be a multiple of 32 up to {LOSS_MAX_S}, got {self.n_sample}")
        if not (1 <= self.num_corr <= min(LOSS_MAX_C, self.n_sample)):
            raise ValueError(f"GENERATE_HYPOTHESES.NUM_CORR_3d3d must be in [1, {LOSS_MAX_C}] and <= NUM_SAMPLES_MATCHES, "
                             f"got {self.num_corr}")


def loss_search(fs, kps0, d0, kps1, d1, K0, K1, p: LossParams, seed: int, outer_idx=None, inner_idx=None):
    """mk_loss_search on a batch.  Returns (sampled int32 [B*IM, S], inner int32 [B*IM*IR, C], inliers_final {0,1} fp32
    [B*IM*IR, S], status int).  final_scores may be a view with contiguous rows and pairs N row pitches apart."""
    sampled, inner, bits, status = _loss_search_bits(fs, kps0, d0, kps1, d1, K0, K1, p, seed, outer_idx, inner_idx)
    return sampled, inner, unpack_mask(bits, p.n_sample), status


def _loss_search_bits(fs, kps0, d0, kps1, d1, K0, K1, p: LossParams, seed: int, outer_idx=None, inner_idx=None):
    """loss_search with inliers_final as the kernel writes it: int32 bit words [B*IM*IR, S/32]."""
    B, N = fs.shape[0], fs.shape[1]
    IM, IR, S, Cn = p.it_matches, p.it_ransac, p.n_sample, p.num_corr
    fs, pitch = _lib.pitched(fs)
    dev = fs.device
    f32 = lambda t: t.detach().to(dev, torch.float32).contiguous()
    kps0, d0, kps1, d1, K0, K1 = (f32(t) for t in (kps0, d0, kps1, d1, K0, K1))
    lib = _lib.load()
    sampled = torch.empty(B * IM, S, dtype=torch.int32, device=dev)
    inner = torch.empty(B * IM * IR, Cn, dtype=torch.int32, device=dev)
    bits = torch.empty(B * IM * IR, S // 32, dtype=torch.int32, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    ws = _lib.workspace(lib.mk_loss_search_ws_bytes(B, IM), dev, "mk_loss_search_ws_bytes")
    oi = None if outer_idx is None else outer_idx.to(dev, torch.int32).contiguous()
    ii = None if inner_idx is None else inner_idx.to(dev, torch.int32).contiguous()
    if oi is not None and tuple(oi.shape) != (B * IM, S):
        raise ValueError(f"outer_idx must be [B*IM, S] = [{B * IM}, {S}], got {tuple(oi.shape)}")
    if ii is not None and tuple(ii.shape) != (B * IM * IR, Cn):
        raise ValueError(f"inner_idx must be [B*IM*IR, C] = [{B * IM * IR}, {Cn}], got {tuple(ii.shape)}")
    _lib.check(lib.mk_loss_search(_lib.ptr(fs), pitch, _lib.ptr(kps0), _lib.ptr(d0), _lib.ptr(kps1), _lib.ptr(d1), _lib.ptr(K0),
                                  _lib.ptr(K1), B, N, IM, IR, S, Cn, p.num_ref_steps, p.inlier_ref_th, seed, _lib.ptr(oi),
                                  _lib.ptr(ii), _lib.ptr(sampled), _lib.ptr(inner), _lib.ptr(bits), _lib.ptr(status),
                                  _lib.ptr(ws), ws.numel(), _lib.stream(dev)), "mk_loss_search")
    return sampled, inner, bits, int(status.item())


def loss_gradient(sampled, loss_value, baseline, mask_topk, B, N, IM, S):
    """mk_loss_gradient: the dense probs_grad fp32 [B, N, N]."""
    dev = sampled.device
    lib = _lib.load()
    f32 = lambda t: t.detach().to(dev, torch.float32).contiguous()
    lv, bl, mk = f32(loss_value).reshape(-1), f32(baseline).reshape(-1), f32(mask_topk).reshape(-1)
    grad = torch.empty(B, N, N, dtype=torch.float32, device=dev)
    ws = _lib.workspace(lib.mk_loss_gradient_ws_bytes(B, IM, S), dev, "mk_loss_gradient_ws_bytes")
    _lib.check(lib.mk_loss_gradient(_lib.ptr(sampled.to(torch.int32).contiguous()), _lib.ptr(lv), _lib.ptr(bl), _lib.ptr(mk),
                                    B, N, IM, S, _lib.ptr(grad), _lib.ptr(ws), ws.numel(), _lib.stream(dev)), "mk_loss_gradient")
    return grad


class LossTail(torch.autograd.Function):
    """The differentiable tail in CUDA (mk_loss_tail_forward / mk_loss_tail_backward): (loss_value, loss_rot, loss_trans)
    fp32 [B*IM] and the status word int32 [1] from the search's drawn cells and inlier bit words, differentiable in the
    kps / depth leaves.  The forward's saved state lives in a workspace allocated per call and kept on ctx only when a
    backward can follow, so calls that interleave never share state and no_grad / inference_mode keep nothing."""

    @staticmethod
    def forward(ctx, kps0, depth0, kps1, depth1, sampled, bits, K0, K1, Kori0, Kori1, T, grid, p: LossParams, save: bool):
        B, N = kps0.shape[0], kps0.shape[2]
        IM, IR, S = p.it_matches, p.it_ransac, p.n_sample
        dev = kps0.device
        kps0, depth0, kps1, depth1 = (t.contiguous() for t in (kps0, depth0, kps1, depth1))
        lib = _lib.load()
        ws = _lib.workspace(lib.mk_loss_tail_ws_bytes(B, N, IM, IR, S), dev, "mk_loss_tail_ws_bytes")
        out = torch.empty(3, B * IM, dtype=torch.float32, device=dev)
        status = torch.empty(1, dtype=torch.int32, device=dev)
        args = [_lib.ptr(t) for t in (sampled, bits, kps0, depth0, kps1, depth1, K0, K1, Kori0, Kori1, T, grid)]
        args += [B, N, IM, IR, S, 0 if p.loss_type == "VCRE" else 1, int(p.soft_clipping), int(p.add_null_hypothesis),
                 p.inlier_3d_th, p.score_temperature]
        _lib.check(lib.mk_loss_tail_forward(*args, p.th_outliers * p.n_sample, p.max_loss_null, _lib.ptr(out[0]),
                                            _lib.ptr(out[1]), _lib.ptr(out[2]), _lib.ptr(status), _lib.ptr(ws), ws.numel(),
                                            _lib.stream(dev)), "mk_loss_tail_forward")
        ctx.mark_non_differentiable(status)
        if save:
            ctx.save_for_backward(kps0, depth0, kps1, depth1, sampled, bits, K0, K1, Kori0, Kori1, T, grid)
            ctx.p, ctx.ws = p, ws
        return out[0], out[1], out[2], status

    @staticmethod
    def backward(ctx, g_value, g_rot, g_trans, _g_status):
        if not hasattr(ctx, "ws"):
            raise RuntimeError("LossTail: the forward ran without saving its state (save=False)")
        kps0, depth0, kps1, depth1, sampled, bits, K0, K1, Kori0, Kori1, T, grid = ctx.saved_tensors
        p, ws = ctx.p, ctx.ws
        B, N = kps0.shape[0], kps0.shape[2]
        dev = kps0.device
        g = [t.to(torch.float32).contiguous() for t in (g_value, g_rot, g_trans)]
        dk0, dk1 = torch.empty_like(kps0), torch.empty_like(kps1)
        dd0, dd1 = torch.empty_like(depth0), torch.empty_like(depth1)
        lib = _lib.load()
        args = [_lib.ptr(t) for t in (sampled, bits, kps0, depth0, kps1, depth1, K0, K1, Kori0, Kori1, T, grid)]
        args += [B, N, p.it_matches, p.it_ransac, p.n_sample, 0 if p.loss_type == "VCRE" else 1, int(p.soft_clipping),
                 int(p.add_null_hypothesis), p.inlier_3d_th, p.score_temperature]
        _lib.check(lib.mk_loss_tail_backward(*args, *(_lib.ptr(t) for t in g), _lib.ptr(dk0), _lib.ptr(dk1), _lib.ptr(dd0),
                                             _lib.ptr(dd1), _lib.ptr(ws), ws.numel(), _lib.stream(dev)),
                   "mk_loss_tail_backward")
        return dk0, dd0, dk1, dd1, None, None, None, None, None, None, None, None, None, None


class MetricPoseLoss(torch.nn.Module):
    """Drop-in for the reference MetricPoseLoss(cfg): `forward(batch)` returns (avg_loss, outputs, [probs_grad],
    num_valid_h) with the reference's keys.  batch: final_scores [B, N, N], kps0/kps1 [B, 2, N], depth_kp0/depth_kp1
    [B, 1, N], K_color0/1 and Kori_color0/1 [B, 3, 3], T_0to1 [B, 4, 4], all on one CUDA device.  `topK` is settable
    (the training model raises it every epoch).  One seed is drawn from the torch RNG per call; `seed`, `outer_idx` and
    `inner_idx` override the draws (the parity tests inject the reference's).  After a call, `last_loss_value` [B*IM]
    and `last_baseline` [B] hold the REINFORCE iteration losses and baselines (detached).

    cuda_tail=True (also settable later) runs the differentiable tail in CUDA (LossTail) instead of autograd: the same
    values to fp32 rounding, gradients through a closed-form, SVD-free backward, bit-identical from run to run."""

    def __init__(self, cfg, cuda_tail: bool = False):
        super().__init__()
        self.p = LossParams(cfg)
        self.topK = self.p.topK
        self.cuda_tail = bool(cuda_tail)
        self._grid = {}

    def _vcre_grid(self, dev):
        if dev not in self._grid:
            # a normal tensor even when the first call is a validation under inference mode (Lightning's default, and its
            # sanity check runs before the first training step): autograd cannot save an inference tensor for backward
            with torch.inference_mode(False):
                self._grid[dev] = vcre_grid(dev).float()
        return self._grid[dev]

    def forward(self, batch, seed=None, outer_idx=None, inner_idx=None):
        p = self.p
        fs = batch["final_scores"].detach()
        if fs.dim() != 3 or fs.shape[1] != fs.shape[2] or fs.dtype != torch.float32 or fs.device.type != "cuda":
            raise ValueError(f"final_scores must be a CUDA float32 [B, N, N] tensor, got {tuple(fs.shape)} {fs.dtype} "
                             f"on {fs.device} (mickey_b200 has no CPU path)")
        B, N = fs.shape[0], fs.shape[1]
        IM, IR, S = p.it_matches, p.it_ransac, p.n_sample
        dev = fs.device
        kps0, depth0 = batch["kps0"].detach().requires_grad_(), batch["depth_kp0"].detach().requires_grad_()
        kps1, depth1 = batch["kps1"].detach().requires_grad_(), batch["depth_kp1"].detach().requires_grad_()
        Rgt, tgt = batch["T_0to1"][:, :3, :3], batch["T_0to1"][:, :3, 3:].transpose(1, 2)
        K0, K1 = batch["K_color0"].float(), batch["K_color1"].float()
        if seed is None:
            seed = int(torch.randint(1, 2 ** 62, (1,)).item())     # follows torch.manual_seed like the reference
        sampled, _, bits, status = _loss_search_bits(fs, kps0, depth0, kps1, depth1, K0, K1, p, seed, outer_idx, inner_idx)

        outputs = {"kps0": kps0, "kps1": kps1, "depth0": depth0, "depth1": depth1}
        baseline = torch.zeros(B, device=dev)
        losses_rot = torch.zeros(B, 1, device=dev)
        losses_trans = torch.zeros(B, 1, device=dev)
        loss_value = None
        num_valid_h = 0
        if not status & STATUS_SKIP:
            if self.cuda_tail:
                tail = self._cuda_tail(batch, sampled, bits, kps0, depth0, kps1, depth1, K0, K1)
            else:
                tail = self._tail(batch, sampled, unpack_mask(bits, S), kps0, depth0, kps1, depth1, K0, K1, Rgt, tgt, B, N)
            if tail is not None:
                loss_value, loss_rot, loss_trans = tail
                losses_rot = loss_rot.reshape(B, IM).sum(-1).unsqueeze(-1)
                losses_trans = loss_trans.reshape(B, IM).sum(-1).unsqueeze(-1)
                baseline = loss_value.reshape(B, IM).sum(-1)
                num_valid_h = 1
        # RANSAC_vectorized (:287-329)
        baseline = baseline / IM
        losses_trans = losses_trans / IM
        losses_rot = losses_rot / IM
        if p.train_w_top and B > 1:
            select_top_b = np.maximum(int(B * self.topK / 100), 1)
            topk_loss = baseline[torch.argsort(baseline)[select_top_b]]
            mask_topk = (baseline < topk_loss).float()
            avg_loss = (mask_topk * baseline).sum() / mask_topk.sum()
        else:
            avg_loss = torch.mean(baseline)
            mask_topk = torch.ones(B, device=dev)
        if loss_value is None:
            gradients = torch.zeros(B, N, N, device=dev)
        else:
            gradients = loss_gradient(sampled, loss_value, baseline, mask_topk, B, N, IM, S)
        self.last_loss_value = None if loss_value is None else loss_value.detach()      # per outer iteration [B*IM]
        self.last_baseline = baseline.detach()
        outputs["avg_loss_rot"] = torch.mean(losses_rot)
        outputs["avg_loss_trans"] = torch.mean(losses_trans)
        outputs["avg_rot_errs"] = torch.mean(torch.rad2deg(torch.as_tensor(losses_rot)))
        outputs["avg_t_errs"] = torch.mean(losses_trans)
        outputs["mask_topk"] = mask_topk
        return avg_loss, outputs, [gradients], num_valid_h

    def _cuda_tail(self, batch, sampled, bits, kps0, depth0, kps1, depth1, K0, K1):
        """_tail's values and gradients through LossTail, or None for the same invalid-pose early return."""
        dev = kps0.device
        f32 = lambda t: t.detach().to(dev, torch.float32).contiguous()
        leaves = (kps0, depth0, kps1, depth1)
        if any(t.dtype != torch.float32 or t.device != dev for t in leaves):
            raise ValueError("cuda_tail: kps0, kps1, depth_kp0 and depth_kp1 must be float32 tensors on one CUDA device")
        save = torch.is_grad_enabled() and any(t.requires_grad for t in leaves)
        loss_value, loss_rot, loss_trans, status = LossTail.apply(
            *leaves, sampled, bits, f32(K0), f32(K1), f32(batch["Kori_color0"]), f32(batch["Kori_color1"]),
            f32(batch["T_0to1"]), self._vcre_grid(dev), self.p, save)
        if int(status.item()):
            return None
        return loss_value, loss_rot, loss_trans

    def _tail(self, batch, sampled, inl, kps0, depth0, kps1, depth1, K0, K1, Rgt, tgt, B, N):
        """:140-152 and :199-248 in autograd.  Returns (loss_value [B*IM], loss_rot [B*IM], loss_trans [B*IM]) or None
        for the invalid-pose early return (:213-223)."""
        p = self.p
        IM, IR, S = p.it_matches, p.it_ransac, p.n_sample
        dev = kps0.device
        cell = sampled.long()
        i0, i1 = torch.div(cell, N, rounding_mode="trunc"), cell % N
        bidx = torch.arange(B, device=dev).repeat_interleave(IM).unsqueeze(1).expand(-1, S)
        X = backproject_3d(kps0[bidx, :2, i0], depth0[bidx, :2, i0], K0.repeat_interleave(IM, 0))
        Y = backproject_3d(kps1[bidx, :2, i1], depth1[bidx, :2, i1], K1.repeat_interleave(IM, 0))
        X_v = X.unsqueeze(1).expand(-1, IR, -1, -1).reshape(B * IM * IR, S, 3)
        Y_v = Y.unsqueeze(1).expand(-1, IR, -1, -1).reshape(B * IM * IR, S, 3)
        R, t = weighted_procrustes(X_v, Y_v, inl)
        if not (bool(torch.isfinite(R).all()) and bool(torch.isfinite(t).all())):
            return None
        score_k = soft_inlier_counting_3d(X_v, Y_v, R, t, p.inlier_3d_th)
        rep = IM * IR
        Rgt_v, tgt_v = Rgt.repeat_interleave(rep, 0), tgt.repeat_interleave(rep, 0)
        Kori0, Kori1 = batch["Kori_color0"].repeat_interleave(rep, 0), batch["Kori_color1"].repeat_interleave(rep, 0)
        loss_fn = compute_vcre_loss if p.loss_type == "VCRE" else compute_pose_loss
        loss_value_k, loss_rot_k, loss_trans_k = loss_fn(R, t, Rgt_v, tgt_v, Kori0, Kori1, self._vcre_grid(dev),
                                                         p.soft_clipping)
        loss_value_k = loss_value_k.reshape(B * IM, IR)
        loss_rot_k, loss_trans_k = loss_rot_k.reshape(B * IM, IR), loss_trans_k.reshape(B * IM, IR)
        score_k = score_k.reshape(B * IM, IR)
        sm = torch.softmax(score_k / p.score_temperature, -1)
        loss_rot, loss_trans = (loss_rot_k * sm).sum(-1), (loss_trans_k * sm).sum(-1)
        if p.add_null_hypothesis:
            null_score = torch.full((B * IM, 1), p.th_outliers * p.n_sample, device=dev)
            null_loss = torch.full((B * IM, 1), p.max_loss_null, device=dev)
            loss_value_k = torch.cat([loss_value_k, null_loss], -1)
            score_k = torch.cat([score_k, null_score], -1)
        loss_value = (loss_value_k * torch.softmax(score_k / p.score_temperature, -1)).sum(-1)
        return loss_value, loss_rot, loss_trans
