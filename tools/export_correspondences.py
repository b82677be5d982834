"""Export MicKey's correspondences and depths for a Map-free split: the "MicKey correspondences and depth files" the
reference README (README.md:70-76) offers for download, made here for any checkpoint and split.

    python tools/export_correspondences.py --split val --data_root data --checkpoint mickey.ckpt --uint8 -o corr/
    python -m torch.distributed.run --nproc-per-node 8 tools/export_correspondences.py ...     # pairs sharded by rank

Every pair goes through model(data) (the same loader and batches as tools/run_submission.py), then
model.mutual_matches(final_scores, --min_conf), i.e. the reference's get_matches_list, per pair.

Output: one <scene>.npz per scene (<scene>.rank<r>.npz with several ranks: each rank writes the queries it ran).
  reference             str, the scene's reference image (image0 of every pair)
  queries               str [Q], the query images (image1), in loader order
  depth_map0            float32 [Q, h, w]  metric depth of the reference image on the token grid (h, w = H/14, W/14)
  depth_map1            float32 [Q, h, w]  metric depth of each query
  and for query q, with M_q matches sorted by score (descending, equal scores by ascending i):
  q<q>_ij               int32 [M_q, 2]     keypoint indices (i into the reference's, j into the query's N = h * w keypoints)
  q<q>_pts0, q<q>_pts1  float32 [M_q, 2]   pixel coordinates (x, y) of the matched keypoints: kps0[i], kps1[j]
  q<q>_depth0, q<q>_depth1  float32 [M_q]  their metric depths depth_kp0[i], depth_kp1[j]
  q<q>_scores           float32 [M_q]      final_scores[i, j]
Pixel coordinates are in the resized image the model ran on (config DATASET resize).  This is the project's own layout;
it is not the file format of the Map-free benchmark's correspondence loaders.
"""
import argparse
import json
import os
import sys
from collections import defaultdict
from pathlib import Path

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "compat")] if __import__("importlib").util.find_spec("transforms3d") is None else [ROOT]

from mickey_b200.config import mickey_cfg                               # noqa: E402
from mickey_b200.model import build_model                               # noqa: E402
from mickey_b200.weights import synthetic_checkpoint                    # noqa: E402


def batch_records(model, data, min_conf):
    """The per-query records of one batch that model(data) has run on, as numpy arrays."""
    lists, scores = model.mutual_matches(data["final_scores"], min_conf)
    out = []
    for b, (ij, sc) in enumerate(zip(lists, scores)):
        i, j = ij[:, 0], ij[:, 1]
        out.append({"ij": ij.int(), "pts0": data["kps0"][b][:, i].t(), "pts1": data["kps1"][b][:, j].t(),
                    "depth0": data["depth_kp0"][b, 0, i], "depth1": data["depth_kp1"][b, 0, j], "scores": sc,
                    "depth_map0": data["depth0_map"][b, 0], "depth_map1": data["depth1_map"][b, 0]})
    return [{k: v.detach().float().cpu().numpy() if k != "ij" else v.cpu().numpy() for k, v in r.items()} for r in out]


def write_scene(path, reference, queries, recs):
    arrays = {"reference": np.array(reference), "queries": np.array(queries),
              "depth_map0": np.stack([r["depth_map0"] for r in recs]), "depth_map1": np.stack([r["depth_map1"] for r in recs])}
    for q, r in enumerate(recs):
        for k in ("ij", "pts0", "pts1", "depth0", "depth1", "scores"):
            arrays[f"q{q}_{k}"] = r[k]
    np.savez_compressed(path, **arrays)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default=None, help="model YAML (reference format); default: built-in MicKey config of --variant")
    ap.add_argument("--variant", default="vitl", choices=["vits", "vitb", "vitl"])
    ap.add_argument("--checkpoint", default="synthetic", help="mickey.ckpt, or 'synthetic' for seeded random-init weights")
    ap.add_argument("--data_root", default=None)
    ap.add_argument("--split", choices=("val", "test"), default="val")
    ap.add_argument("--batch_size", type=int, default=8)
    ap.add_argument("--workers", type=int, default=4)
    ap.add_argument("--uint8", action="store_true", help="uint8 HWC batches + fused ingest kernel (a quarter of the H2D bytes)")
    ap.add_argument("--min_conf", type=float, default=0.0, help="get_matches_list's min_conf: keep matches with exp(score) > it")
    ap.add_argument("--output_root", "-o", type=Path, default=Path("correspondences/"))
    args = ap.parse_args()

    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if args.checkpoint == "synthetic":
        os.environ.setdefault("MICKEY_SYNTHETIC_BACKBONE", "1")

    from config.default import cfg
    from lib.datasets.datamodules import DataModule
    cfg.merge_from_file(os.path.join(ROOT, "config", "datasets", "mapfree.yaml"))
    if args.config:
        cfg.merge_from_file(args.config)
    else:
        cfg.merge_from_other_cfg({k: v for k, v in mickey_cfg(args.variant).items() if k in ("MODEL", "MICKEY", "FEATURE_MATCHER", "PROCRUSTES")})
    if args.data_root:
        cfg.DATASET.DATA_ROOT = args.data_root
    cfg.TRAINING.BATCH_SIZE, cfg.TRAINING.NUM_WORKERS = args.batch_size, args.workers
    dm = DataModule(cfg, drop_last_val=False, uint8_images=args.uint8, pin_memory=True)    # shards the pairs by rank
    loader = dm.val_dataloader() if args.split == "val" else dm.test_dataloader()
    ckpt = synthetic_checkpoint(cfg, seed=0, with_backbone=True) if args.checkpoint == "synthetic" else args.checkpoint
    model = build_model(cfg, ckpt)

    scenes = defaultdict(lambda: {"reference": None, "queries": [], "recs": []})
    n = 0
    for data in loader:
        for k in ("image0", "image1", "K_color0", "K_color1"):
            data[k] = data[k].to(dev, non_blocking=True)
        with torch.no_grad():
            model(data)
            recs = batch_records(model, data, args.min_conf)
        for b, r in enumerate(recs):
            sc = scenes[data["scene_id"][b]]
            sc["reference"] = data["pair_names"][0][b]
            sc["queries"].append(data["pair_names"][1][b])
            sc["recs"].append(r)
            n += 1
    args.output_root.mkdir(parents=True, exist_ok=True)
    files = []
    for scene, sc in scenes.items():
        path = args.output_root / (f"{scene}.npz" if world == 1 else f"{scene}.rank{rank}.npz")
        write_scene(path, sc["reference"], sc["queries"], sc["recs"])
        files.append(str(path))
    print(json.dumps({"rank": rank, "pairs": n, "scenes": len(files), "files": files, "min_conf": args.min_conf}), flush=True)


if __name__ == "__main__":
    main()
