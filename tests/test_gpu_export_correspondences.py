"""tools/export_correspondences.py on a small synthetic Map-free tree: one file per scene with one entry per query, whose
matches are model.mutual_matches of that pair and whose coordinates / depths are the matched keypoints'."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.common import ROOT
from tools.make_synthetic_mapfree import make_tree

pytestmark = pytest.mark.gpu


def test_export_matches_mutual_matches(tmp_path):
    from mickey_b200.config import CfgNode, mickey_cfg
    cfg = mickey_cfg("vits", 2, 8)
    (tmp_path / "model.yaml").write_text(CfgNode({k: cfg[k] for k in ("MODEL", "MICKEY", "FEATURE_MATCHER", "PROCRUSTES")}).dump())
    make_tree(str(tmp_path / "data"), "val", scenes=2, queries=11, seed=3, width=196, height=224)
    cmd = [sys.executable, os.path.join(ROOT, "tools", "export_correspondences.py"), "--variant", "vits", "--config",
           str(tmp_path / "model.yaml"), "--data_root", str(tmp_path / "data"), "--split", "val", "--batch_size", "4",
           "--workers", "0", "--uint8", "-o", str(tmp_path / "out")]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=str(tmp_path), env=dict(os.environ, PYTHONPATH=ROOT), timeout=900)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    summary = json.loads(r.stdout.strip().splitlines()[-1])
    assert summary["pairs"] == 6 and sorted(os.listdir(tmp_path / "out")) == ["s00000.npz", "s00001.npz"]

    # the same batches through the model in this process
    sys.path.insert(0, os.path.join(ROOT, "compat"))
    os.environ.setdefault("MICKEY_SYNTHETIC_BACKBONE", "1")
    from config.default import cfg as base
    from lib.datasets.datamodules import DataModule
    from mickey_b200.model import build_model
    from mickey_b200.weights import synthetic_checkpoint
    c = base.clone()
    c.merge_from_file(os.path.join(ROOT, "config", "datasets", "mapfree.yaml"))
    c.merge_from_file(str(tmp_path / "model.yaml"))
    c.DATASET.DATA_ROOT = str(tmp_path / "data")
    c.TRAINING.BATCH_SIZE, c.TRAINING.NUM_WORKERS = 4, 0
    model = build_model(c, synthetic_checkpoint(c, seed=0, with_backbone=True))
    files = {s: np.load(tmp_path / "out" / f"{s}.npz") for s in ("s00000", "s00001")}
    seen = {s: 0 for s in files}
    for data in DataModule(c, drop_last_val=False, uint8_images=True).val_dataloader():
        for k in ("image0", "image1", "K_color0", "K_color1"):
            data[k] = data[k].cuda()
        with torch.no_grad():
            model(data)
            lists, scores = model.mutual_matches(data["final_scores"])
        for b, ij in enumerate(lists):
            scene, q = data["scene_id"][b], seen[data["scene_id"][b]]
            f = files[scene]
            assert str(f["queries"][q]) == data["pair_names"][1][b] and str(f["reference"]) == data["pair_names"][0][b]
            ij = ij.cpu()
            assert np.array_equal(f[f"q{q}_ij"], ij.numpy()) and len(ij) > 0
            kps0, kps1 = data["kps0"][b].cpu(), data["kps1"][b].cpu()
            assert np.array_equal(f[f"q{q}_pts0"], kps0[:, ij[:, 0]].t().numpy())
            assert np.array_equal(f[f"q{q}_pts1"], kps1[:, ij[:, 1]].t().numpy())
            assert np.array_equal(f[f"q{q}_depth1"], data["depth_kp1"][b, 0].cpu()[ij[:, 1]].numpy())
            assert np.array_equal(f[f"q{q}_scores"], scores[b].cpu().numpy())
            assert np.array_equal(f["depth_map0"][q], data["depth0_map"][b, 0].cpu().numpy())
            seen[scene] += 1
    for s, f in files.items():
        assert seen[s] == len(f["queries"]) == f["depth_map1"].shape[0] == 3
