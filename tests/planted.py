"""Planted-pose problem generator for the solver (size-independent property test)."""
import math

import torch

from tests.common import K_TOY


def _rot(axis, deg):
    axis = torch.tensor(axis, dtype=torch.float64)
    axis = axis / axis.norm()
    a = math.radians(deg)
    Kx = torch.tensor([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]], dtype=torch.float64)
    return torch.eye(3, dtype=torch.float64) + math.sin(a) * Kx + (1 - math.cos(a)) * (Kx @ Kx)


def planted_problem(n_side=(20, 16), batch=1, outlier_frac=0.4, seed=0, diag_weight=1.0, off_weight=1e-6, noise=0.0):
    """Keypoint i in image 0 corresponds to keypoint i in image 1: Y_i = R X_i + t exactly for the
    inlier fraction; the rest get a corrupted depth.  final_scores is diagonal-heavy so the sampler
    picks (i, i) cells almost always.  Returns tensors shaped like the model's data dict.

    noise > 0 moves every Y_i by an isotropic Gaussian of that standard deviation (metres) before it is projected:
    a hypothesis from three points is then off by more than the threshold far from them, and each refinement of the
    solver adds the points its better fit brings inside (the inlier set grows over several refinements)."""
    g = torch.Generator().manual_seed(seed)
    h, w = n_side
    N = h * w
    K = torch.tensor(K_TOY, dtype=torch.float64)
    Kinv = torch.linalg.inv(K)
    Rs, ts, k0s, k1s, d0s, d1s, fs = [], [], [], [], [], [], []
    for b in range(batch):
        R = _rot([0.2 + 0.1 * b, 1.0, 0.3], 12.0 + 3 * b)
        t = torch.tensor([0.4, -0.15, 0.25], dtype=torch.float64) * (1 + 0.2 * b)
        uv0 = torch.stack([torch.rand(N, generator=g, dtype=torch.float64) * 520 + 10,
                           torch.rand(N, generator=g, dtype=torch.float64) * 700 + 10], 0)       # [2,N]
        d0 = torch.rand(N, generator=g, dtype=torch.float64) * 4 + 2
        X = d0 * (Kinv @ torch.cat([uv0, torch.ones(1, N, dtype=torch.float64)], 0))            # [3,N]
        Y = R @ X + t[:, None]
        if noise > 0:
            Y = Y + noise * torch.randn(3, N, generator=g, dtype=torch.float64)
        d1 = Y[2].clone()
        proj = K @ (Y / Y[2:3])
        uv1 = proj[:2]
        n_out = int(outlier_frac * N)
        bad = torch.randperm(N, generator=g)[:n_out]
        d1[bad] = d1[bad] * (1.5 + torch.rand(n_out, generator=g, dtype=torch.float64))
        f = torch.full((N, N), off_weight, dtype=torch.float64)
        f[torch.arange(N), torch.arange(N)] = diag_weight
        f = f / f.sum()
        Rs.append(R); ts.append(t.view(1, 3)); k0s.append(uv0); k1s.append(uv1)
        d0s.append(d0.view(1, N)); d1s.append(d1.view(1, N)); fs.append(f)
    st = lambda xs: torch.stack(xs).float()
    return {"R": st(Rs), "t": st(ts), "kps0": st(k0s), "kps1": st(k1s), "depth0": st(d0s),
            "depth1": st(d1s), "final_scores": st(fs), "K": K.float()[None].repeat(batch, 1, 1), "N": N}
