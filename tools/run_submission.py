"""BASELINE config 5 — Map-free val/test submission on N GPUs (one process per GPU, torchrun):

    python tools/make_synthetic_mapfree.py --root data --split val --scenes 8 --queries 40
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29520 \
        tools/run_submission.py --variant vitl --split val --output_root results/ --uint8

What the reference does in one process (submission.py:71-96) is sharded here by PAIR: every rank builds the same pair
list, takes its contiguous slice (lib/datasets/sampler.py), runs the CUDA hot path on its batches and joins ONE
all-gather of the packed [batch, 13] poses per step (ranks whose slice is exhausted contribute an empty block).  Rank 0
converts the gathered poses to submission records on its GPU (mk_pose_to_submission, one D2H per step), writes
`submission.zip` with the reference's `pose_<scene>.txt` line format, and grades the poses against the tree's ground
truth with the reference's pose-error definitions (lib/utils/metrics.py:12-53).  `--evaluate` also grades the written zip
as the Map-free benchmark does (mickey_b200/mapfree_eval.py) and adds its numbers under "mapfree_metrics".  With
random-init weights the poses are noise — the run proves the plumbing and gives pairs/s end to end from JPEG files.

Every val/test pair of a scene has the same image0, the scene's reference image.  `--share-reference` reads and extracts
each reference once (ReferenceBank), extracts only the query images of a step and poses the batch from the two feature
banks (model.pose_from_features).  The loader then leaves image0 out of its items.  `--localize` (implies
`--share-reference`) poses each batch in one call, model.localize: only the queries are extracted, matched against the
cached references of the batch's one or two scenes, replayed from a CUDA graph.  Every path draws one seed per batch, so
under the same `--seed` they write the same submission.
"""
import argparse
import json
import os
import sys
import time
from collections import defaultdict
from pathlib import Path

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "compat")] if __import__("importlib").util.find_spec("transforms3d") is None else [ROOT]

from mickey_b200 import dist as mkdist                                  # noqa: E402
from mickey_b200 import submission as mksub                             # noqa: E402
from mickey_b200.config import mickey_cfg                               # noqa: E402
from mickey_b200.model import MickeyFeatures, build_model               # noqa: E402
from mickey_b200.weights import synthetic_checkpoint                    # noqa: E402


def pose_errors(R, t, T_gt):
    """Rotation angle (deg) and translation Euclidean error (m) as in lib/utils/metrics.py:12-53 (numpy, fp64)."""
    Rgt, tgt = T_gt[:, :3, :3], T_gt[:, :3, 3]
    cos = np.clip((np.einsum("bij,bij->b", R, Rgt) - 1) / 2, -1, 1)      # trace(R^T Rgt)
    return np.rad2deg(np.arccos(cos)), np.linalg.norm(t - tgt, axis=-1)


class ReferenceBank:
    """Features of the reference images the current batch uses.  A reference is read (`load(scene_root, name)`) and
    extracted (`extract(image) -> features`) when its first pair arrives, and dropped when a batch no longer uses it: the
    loader walks each rank's pairs scene by scene, so a scene's reference is extracted once per rank."""

    def __init__(self, load, extract):
        self.load, self.extract = load, extract
        self.cache = {}
        self.extracted = 0

    def lookup(self, keys):
        """keys: (scene_root, image0 name) of every pair of the batch -> (features of each distinct reference in order of
        first use, index of every pair's reference in that list)."""
        order = list(dict.fromkeys(keys))
        for k in order:
            if k not in self.cache:
                self.cache[k] = self.extract(self.load(*k))
                self.extracted += 1
        for k in [k for k in self.cache if k not in order]:
            del self.cache[k]
        pos = {k: i for i, k in enumerate(order)}
        return [self.cache[k] for k in order], [pos[k] for k in keys]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default=None, help="model YAML (reference format); default: built-in MicKey config of --variant")
    ap.add_argument("--variant", default="vitl", choices=["vits", "vitb", "vitl"])
    ap.add_argument("--checkpoint", default="synthetic", help="mickey.ckpt, or 'synthetic' for seeded random-init weights")
    ap.add_argument("--data_root", default=None)
    ap.add_argument("--split", choices=("val", "test"), default="val")
    ap.add_argument("--batch_size", type=int, default=0, help="default: the reference's 12 (val) / 8 (test)")
    ap.add_argument("--workers", type=int, default=4)
    ap.add_argument("--uint8", action="store_true", help="uint8 HWC batches + fused ingest kernel (a quarter of the H2D bytes)")
    ap.add_argument("--share-reference", action="store_true",
                    help="extract each scene's reference image once and pose every pair from feature banks")
    ap.add_argument("--localize", action="store_true",
                    help="with --share-reference: extract only the queries and pose each batch in one call (model.localize)")
    ap.add_argument("--seed", type=int, default=None,
                    help="seed the torch RNG that the solver's per-batch seeds come from (a reproducible submission)")
    ap.add_argument("--output_root", "-o", type=Path, default=Path("results/"))
    ap.add_argument("--evaluate", action="store_true",
                    help="grade the written submission.zip as the Map-free benchmark does (summary key mapfree_metrics)")
    args = ap.parse_args()

    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=dev)
    if args.checkpoint == "synthetic":
        os.environ.setdefault("MICKEY_SYNTHETIC_BACKBONE", "1")

    from config.default import cfg
    from lib.datasets.datamodules import DataModule
    cfg.merge_from_file(os.path.join(ROOT, "config", "datasets", "mapfree.yaml"))            # submission.py:73-74
    if args.config:
        cfg.merge_from_file(args.config)
    else:
        cfg.merge_from_other_cfg({k: v for k, v in mickey_cfg(args.variant).items() if k in ("MODEL", "MICKEY", "FEATURE_MATCHER", "PROCRUSTES")})
    if args.data_root:
        cfg.DATASET.DATA_ROOT = args.data_root
    cfg.TRAINING.BATCH_SIZE = args.batch_size or (12 if args.split == "val" else 8)           # submission.py:77-84
    cfg.TRAINING.NUM_WORKERS = args.workers
    BS = cfg.TRAINING.BATCH_SIZE

    share = args.share_reference or args.localize
    dm = DataModule(cfg, drop_last_val=False, uint8_images=args.uint8, pin_memory=True, skip_image0=share)
    loader = dm.val_dataloader() if args.split == "val" else dm.test_dataloader()
    n_pairs = len(loader.dataset)
    n_steps, step_rows = mkdist.step_plan(n_pairs, world, BS)
    ckpt = synthetic_checkpoint(cfg, seed=0, with_backbone=True) if args.checkpoint == "synthetic" else args.checkpoint
    model = build_model(cfg, ckpt)

    # names / ground truth of every pair in global order, from the scene indices (no image is read for this)
    names, scenes, T_gt = [], [], []
    if rank == 0:
        for sc in loader.dataset.datasets:
            for pr in sc.pairs:
                a, b = sc.get_pair_path(pr)
                names.append(b); scenes.append(sc.scene_root.stem)
                T_gt.append(np.zeros((4, 4)) if sc.test_scene else sc.relative_pose(a, b)[0])

    gathered = [[] for _ in range(world)]                       # rank 0: records per source rank, in step order
    h2d = 0
    refs = None
    if share:
        scene_of = {str(sc.scene_root): sc for sc in loader.dataset.datasets}

        def extract_reference(image):
            nonlocal h2d
            h2d += image.numel() * image.element_size()
            return model.extract_features(image[None].to(dev))
        refs = ReferenceBank(lambda root, name: scene_of[root].image(name), extract_reference)
    if args.seed is not None:
        torch.manual_seed(args.seed)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    it = iter(loader)
    for step in range(n_steps):
        rows = step_rows[step]
        mine = torch.zeros(BS, 13, device=dev)
        if rows[rank] > 0:
            data = next(it)
            for k in ("image1", "K_color0", "K_color1") if share else ("image0", "image1", "K_color0", "K_color1"):
                data[k] = data[k].to(dev, non_blocking=True)
                h2d += data[k].numel() * data[k].element_size()
            with torch.no_grad():
                if args.localize:
                    banks, idx0 = refs.lookup(list(zip(data["scene_root"], data["pair_names"][0])))
                    data = model.localize(MickeyFeatures.cat(banks), idx0, data["image1"], data["K_color0"], data["K_color1"])
                    R, t = data["R"], data["t"]
                elif share:
                    banks, idx0 = refs.lookup(list(zip(data["scene_root"], data["pair_names"][0])))
                    queries = model.extract_features(data["image1"])
                    data = model.pose_from_features(MickeyFeatures.cat(banks), idx0, queries, range(len(queries)),
                                                    data["K_color0"], data["K_color1"])
                    R, t = data["R"], data["t"]
                else:
                    R, t = model(data)
            mine[:rows[rank]] = mksub.pack_poses(R, t, data["inliers"])
        allp = mkdist.gather_poses(mine)                        # the ONE collective of the step ([world*BS, 13])
        if rank == 0:
            recs = mksub.poses_to_records(allp)                 # quaternions + NaN filter on the GPU, one D2H
            for r in range(world):
                if rows[r]:
                    gathered[r].append(recs[r * BS:r * BS + rows[r]])
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0

    if rank == 0:
        recs = np.concatenate([np.concatenate(g) for g in gathered if g], axis=0)
        assert recs.shape[0] == n_pairs, (recs.shape, n_pairs)
        results = defaultdict(list)
        for rec, scene, name in zip(recs, scenes, names):
            for pose in mksub.records_to_poses(rec[None], [name]):
                results[scene].append(pose)
        args.output_root.mkdir(parents=True, exist_ok=True)
        mksub.save_submission(results, args.output_root / "submission.zip")
        summary = {"pairs": n_pairs, "gpus": world, "batch_size": BS, "steps": n_steps, "wall_s": wall, "pairs_per_s": n_pairs / wall,
                   "uint8_ingest": bool(args.uint8), "share_reference": share, "localize": bool(args.localize), "h2d_bytes_rank0": h2d, "valid_poses": int(recs[:, 8].sum()),
                   "scenes": len(results), "zip": str(args.output_root / "submission.zip")}
        if share:
            summary["references_extracted_rank0"] = refs.extracted
        if args.split == "val":
            from transforms3d.quaternions import quat2mat
            ok = recs[:, 8] > 0
            Rm = np.stack([quat2mat(q) for q in recs[ok, :4]]) if ok.any() else np.zeros((0, 3, 3))
            r_err, t_err = pose_errors(Rm, recs[ok, 4:7], np.stack(T_gt)[ok].astype(np.float64))
            summary.update(median_R_err_deg=float(np.median(r_err)) if ok.any() else None,
                           median_t_err_m=float(np.median(t_err)) if ok.any() else None)
        if args.evaluate:
            from mickey_b200.mapfree_eval import evaluate_submission
            summary["mapfree_metrics"], _ = evaluate_submission(cfg.DATASET.DATA_ROOT, args.output_root / "submission.zip",
                                                                args.split)
        print(json.dumps(summary), flush=True)
    if world > 1:
        import torch.distributed as dist
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
