"""Submission writer (SURVEY.md §8 f2): the reference's `predict` / `save_submission` (submission.py:17-68) with the
per-pair work moved to the device.

The reference loops over the pairs of a batch on the host: `R.cpu().numpy()`, `t.cpu().numpy()`,
`data['inliers'][i].item()` (three blocking D2H copies per pair), `mat2quat`, a NaN/Inf test, then formats
`<query image> qw qx qy qz tx ty tz inliers` (:24-29).  Here one kernel (`mk_pose_to_submission`, csrc/io_ops.cu)
converts every rotation of the batch to its quaternion in fp64 and evaluates the filter, ONE copy brings the packed
[B, 9] block to the host, and the lines are formatted with the reference's own formatter settings, so the text is the
same as the Python writer's (quaternions agree to ~1e-15; a fp32 eigen-solver, as transforms3d runs on fp32 input,
differs in the 7th digit).
"""
from __future__ import annotations

from collections import defaultdict
from dataclasses import dataclass
from pathlib import Path
from zipfile import ZipFile

import numpy as np
import torch

from . import _lib


@dataclass
class Pose:
    """submission.py:17-29 (same fields, same text)."""
    image_name: str
    q: np.ndarray
    t: np.ndarray
    inliers: float

    def __str__(self) -> str:
        formatter = {'float': lambda v: f'{v:.6f}'}
        max_line_width = 1000
        q_str = np.array2string(self.q, formatter=formatter, max_line_width=max_line_width)[1:-1]
        t_str = np.array2string(self.t, formatter=formatter, max_line_width=max_line_width)[1:-1]
        return f'{self.image_name} {q_str} {t_str} {self.inliers}'


def pack_poses(R: torch.Tensor, t: torch.Tensor, inliers: torch.Tensor) -> torch.Tensor:
    B = R.shape[0]
    return torch.cat([R.reshape(B, 9), t.reshape(B, 3), inliers.reshape(B, 1)], dim=1).float().contiguous()


def poses_to_records(packed: torch.Tensor) -> np.ndarray:
    """packed [B, 13] fp32 on the GPU (R | t | inliers) -> host float64 [B, 9] = qw qx qy qz tx ty tz inliers valid:
    one kernel + one D2H copy for the whole batch."""
    if packed.device.type != "cuda":
        raise _lib.MickeyB200Error("poses_to_records runs on the GPU (there is no CPU path)")
    lib = _lib.load()
    B = packed.shape[0]
    out = torch.empty(B, 9, dtype=torch.float64, device=packed.device)
    with torch.cuda.device(packed.device):
        _lib.check(lib.mk_pose_to_submission(_lib.ptr(packed), B, _lib.ptr(out), _lib.stream()), "mk_pose_to_submission")
    return out.cpu().numpy()


def records_to_poses(records: np.ndarray, image_names) -> list:
    """Host formatting objects for the valid rows (the reference skips frames with NaN/Inf, submission.py:50-52)."""
    poses = []
    for rec, name in zip(records, image_names):
        if rec[8] == 0.0:
            continue
        poses.append(Pose(image_name=name, q=rec[0:4].copy(), t=rec[4:7].astype(np.float32), inliers=float(np.float32(rec[7]))))
    return poses


def predict(loader, model, to_device=None, shard=None):
    """Mirror of submission.py:32-61.  `to_device(data, model)` defaults to the reference's data_to_model_device;
    `shard=(rank, world)` makes this process take every world-th batch (see lib/datasets/sampler.py for the
    pair-level sharding used by tools/run_submission.py)."""
    if to_device is None:
        from lib.utils.data import data_to_model_device as to_device
    results_dict = defaultdict(list)
    for i_batch, data in enumerate(loader):
        if shard is not None and i_batch % shard[1] != shard[0]:
            continue
        data = to_device(data, model)
        with torch.no_grad():
            R_batched, t_batched = model(data)
        recs = poses_to_records(pack_poses(R_batched, t_batched, data['inliers']))
        scenes, queries = data['scene_id'], data['pair_names'][1]
        for rec, scene, query in zip(recs, scenes, queries):
            for pose in records_to_poses(rec[None], [query]):
                results_dict[scene].append(pose)
    return results_dict


def save_submission(results_dict: dict, output_path: Path):
    """submission.py:64-68."""
    with ZipFile(output_path, 'w') as zf:
        for scene, poses in results_dict.items():
            poses_str = '\n'.join((str(pose) for pose in poses))
            zf.writestr(f'pose_{scene}.txt', poses_str.encode('utf-8'))
