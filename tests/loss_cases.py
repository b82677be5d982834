"""Batches and configurations of the training-loss fixture (tests/golden/make_loss_fixture.py) and its tests.

A batch takes the small golden features (final_scores, kps0, kps1 of the ViT-S / ViT-B cases at 196 x 210 / 208) and
plants a geometry in them: depths in [1.5, 4] m, a pose T_0to1 (12 degrees, 0.35 m) and, for the best-scoring cell of
every row, a keypoint / depth in image 1 that T_0to1 maps the image-0 point to (plus 2 cm of depth noise), with that
cell's score raised 200-fold.  So the high-probability cells are mostly consistent, hypotheses gather inliers and the
refinement runs.  K_color and Kori_color are one planted pinhole matrix.
"""
import math
import os

import numpy as np
import torch

from mickey_b200.config import default_cfg

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIXTURE = os.path.join(GOLDEN, "reference_loss_small.npz")
IM, IR = 4, 8          # a small hypothesis budget keeps the fixture small; every other key is the released config

# case -> (golden features, pairs taken from it, LOSS_FUNCTION, SOFT_CLIPPING, ADD_NULL_HYPOTHESIS, top-K)
CASES = {
    "vits_vcre": ("vits_small", [0, 1], "VCRE", True, True, False),
    "vitb_vcre": ("vitb_small", [0, 0], "VCRE", True, True, False),
    "vits_vcre_hard": ("vits_small", [0, 1], "VCRE", False, True, False),
    "vits_pose": ("vits_small", [0, 1], "POSE_ERR", True, True, False),
    "vitb_pose_hard_nonull": ("vitb_small", [0, 0], "POSE_ERR", False, False, False),
    "vits_vcre_nonull": ("vits_small", [0, 1], "VCRE", True, False, False),
    "vits_topk_b4": ("vits_small", [0, 1, 1, 0], "VCRE", True, True, True),
}


WARMUP_FIXTURE = os.path.join(GOLDEN, "reference_loss_warmup_small.npz")
# The reference's warm-up configs (64 samples per set, no null hypothesis; top-K from 30 % in the curriculum one, none in
# the overlap-score one), as they are apart from the hypothesis budget.
# case -> (golden features, pairs taken from it, reference config, LOSS_FUNCTION, SOFT_CLIPPING)
WARMUP_CASES = {
    "warm_curriculum_vits_topk_b4": ("vits_small", [0, 1, 1, 0], "curriculum_learning_warm_up", "VCRE", True),
    "warm_curriculum_vitb_pose": ("vitb_small", [0, 0], "curriculum_learning_warm_up", "POSE_ERR", True),
    "warm_overlap_vits_vcre": ("vits_small", [0, 1], "overlap_score_warm_up", "VCRE", True),
    "warm_overlap_vitb_pose_hard": ("vitb_small", [0, 0], "overlap_score_warm_up", "POSE_ERR", False),
}


def reference_cfg(name, it_matches=None, it_ransac=None):
    """The reference config tests/golden/reference_cfg_<name>.yaml, with the hypothesis budget replaced when given."""
    cfg = default_cfg()
    cfg.merge_from_file(os.path.join(GOLDEN, f"reference_cfg_{name}.yaml"))
    g = cfg.LOSS_CLASS.GENERATE_HYPOTHESES
    if it_matches is not None:
        g.IT_MATCHES = it_matches
    if it_ransac is not None:
        g.IT_RANSAC = it_ransac
    return cfg


def warmup_cfg(name):
    _, _, ref, loss, soft = WARMUP_CASES[name]
    cfg = reference_cfg(ref, IM, IR)
    cfg.LOSS_CLASS.LOSS_FUNCTION, cfg.LOSS_CLASS.SOFT_CLIPPING = loss, soft
    return cfg


def loss_cfg(loss="VCRE", soft=True, null=True, topk=False, it_matches=IM, it_ransac=IR):
    cfg = default_cfg()
    cfg.merge_from_file(os.path.join(GOLDEN, "reference_cfg_curriculum_learning.yaml"))
    lc = cfg.LOSS_CLASS
    lc.LOSS_FUNCTION, lc.SOFT_CLIPPING = loss, soft
    lc.NULL_HYPOTHESIS.ADD_NULL_HYPOTHESIS = null
    lc.CURRICULUM_LEARNING.TRAIN_CURRICULUM = topk
    lc.CURRICULUM_LEARNING.TRAIN_WITH_TOPK = topk
    lc.GENERATE_HYPOTHESES.IT_MATCHES, lc.GENERATE_HYPOTHESES.IT_RANSAC = it_matches, it_ransac
    return cfg


def case_cfg(name):
    if name in WARMUP_CASES:
        return warmup_cfg(name)
    _, _, loss, soft, null, topk = CASES[name]
    return loss_cfg(loss, soft, null, topk)


def planted_pose(deg=12.0, t=(0.25, -0.1, 0.22)):
    a = math.radians(deg)
    ax = torch.tensor([0.3, 1.0, 0.2], dtype=torch.float64)
    ax = ax / ax.norm()
    Kx = torch.tensor([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]], dtype=torch.float64)
    R = torch.eye(3, dtype=torch.float64) + math.sin(a) * Kx + (1 - math.cos(a)) * Kx @ Kx
    T = torch.eye(4, dtype=torch.float64)
    T[:3, :3], T[:3, 3] = R, torch.tensor(t, dtype=torch.float64)
    return T


def plant(fs, kps0, kps1, seed=0, K=None):
    """fp32 batch dict of the loss from final_scores [B, N, N] and kps [B, 2, N] (see the module docstring)."""
    g = torch.Generator().manual_seed(seed)
    B, N = fs.shape[0], fs.shape[1]
    if K is None:
        K = torch.tensor([[160.0, 0, 98.0], [0, 160.0, 105.0], [0, 0, 1]], dtype=torch.float64)
    T = planted_pose()
    d0 = 1.5 + 2.5 * torch.rand(B, 1, N, generator=g, dtype=torch.float64)
    d1 = 1.5 + 2.5 * torch.rand(B, 1, N, generator=g, dtype=torch.float64)
    k0, k1 = kps0.double().clone(), kps1.double().clone()
    fs = fs.clone()
    for b in range(B):
        uv1 = torch.cat([k0[b], torch.ones(1, N, dtype=torch.float64)], 0)
        X0 = d0[b] * (torch.linalg.inv(K) @ uv1)                                   # [3, N]
        X1 = T[:3, :3] @ X0 + T[:3, 3:]
        j = fs[b].double().argmax(1)
        seen = set()
        for i in range(N):
            jj = int(j[i])
            if jj in seen:
                continue
            seen.add(jj)
            z = float(X1[2, i]) + 0.02 * float(torch.randn(1, generator=g, dtype=torch.float64))
            p = K @ (X1[:, i] / X1[2, i])
            k1[b, :, jj] = p[:2]
            d1[b, 0, jj] = z
            fs[b, i, jj] *= 200.0
    Kb = K.float().unsqueeze(0).repeat(B, 1, 1)
    return {"final_scores": fs.float().contiguous(), "kps0": k0.float(), "kps1": k1.float(), "depth_kp0": d0.float(),
            "depth_kp1": d1.float(), "K_color0": Kb.clone(), "K_color1": Kb.clone(), "Kori_color0": Kb.clone(),
            "Kori_color1": Kb.clone(), "T_0to1": T.float().unsqueeze(0).repeat(B, 1, 1)}


def case_batch(name):
    src, pairs, *_ = CASES[name] if name in CASES else WARMUP_CASES[name]
    z = np.load(os.path.join(GOLDEN, f"{src}.npz"))
    take = lambda k: torch.from_numpy(z[k][pairs])
    return plant(take("final_scores"), take("kps0"), take("kps1"), seed=len(pairs))
