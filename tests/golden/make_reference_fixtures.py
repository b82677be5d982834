"""Generate the reference fixtures of the CPU tests that compare with the unmodified reference (nianticlabs/mickey):

    MICKEY_REFERENCE_ROOT=<reference checkout> python tests/golden/make_reference_fixtures.py

  reference_pose_lines.json     submission.py's Pose dataclass: text of a few records
  reference_cfg_*.yaml          config/MicKey/*.yaml merged into the reference's own config/default.py, re-dumped
  reference_stagewise_vits.npz  compute_matches() of the reference, in float64, on the seeded ViT-S case of test_oracle_golden.py
  reference_mapfree_items.json  the reference's MapFreeDataset on the generated tree of test_datasets.py (arrays as sha256)
"""
import hashlib
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_harness  # noqa: E402

REF = ref_harness.REF_ROOT
POSES = [("seq1/frame_00010.jpg", [0.5, -0.5, 0.5, 0.5], [1.25, -0.125, 3.0], 12.5),
         ("s00460/seq1/frame_00000.jpg", [0.9998, 0.0101, -0.0152, 0.0043], [-0.0312, 0.00021, 1.98765], 301.0),
         ("a.jpg", [1.0, 0.0, 0.0, 0.0], [1e-7, -12345.678901, 0.5], 0.0)]


def _swap_lib(path):
    """Import the reference's `lib` / `config` packages instead of this repository's."""
    for k in [k for k in sys.modules if k.split(".")[0] in ("lib", "config")]:
        del sys.modules[k]
    sys.path.insert(0, path)


def pose_lines():
    src = open(os.path.join(REF, "submission.py")).read()
    ns = {}
    exec("from dataclasses import dataclass\nimport numpy as np\n" + src[src.index("@dataclass"):src.index("def predict")], ns)
    out = []
    for name, q, t, inl in POSES:
        p = ns["Pose"](image_name=name, q=np.array(q), t=np.array(t, dtype=np.float32), inliers=inl)
        out.append({"image_name": name, "q": q, "t": t, "inliers": inl, "line": str(p)})
    return out


def stagewise():
    """Evaluated in float64, so that the stored stage outputs do not depend on the CPU that runs the comparison."""
    from mickey_b200.config import mickey_cfg
    from mickey_b200.weights import synthetic_state_dict
    from tests.common import float64_eval, synthetic_pair, to_float64
    cfg = mickey_cfg("vits", 2, 8, float16=False)
    sd = synthetic_state_dict(cfg, seed=2)
    model = ref_harness.build_reference_model(cfg, sd, variant="vits").double()
    for m in model.modules():
        if hasattr(m, "amp_dtype"):
            m.amp_dtype = torch.float64                    # the backbone's input cast (mickey_extractor.py:49)
    ref = to_float64(synthetic_pair(1, 154, 140, seed=9))
    with torch.no_grad(), float64_eval():
        model.compute_matches(ref)
    return {k: ref[k].numpy() for k in ("kps0", "depth_kp0", "scr0", "dsc0", "scores", "kp_scores")}


def digest(v):
    a = np.ascontiguousarray(v.numpy() if torch.is_tensor(v) else np.asarray(v))
    return {"dtype": str(a.dtype), "shape": list(a.shape), "sha256": hashlib.sha256(a.tobytes()).hexdigest()}


def mapfree_items():
    import tempfile
    sys.path.insert(0, os.path.join(ROOT, "compat"))
    from tools.make_synthetic_mapfree import make_tree
    from config.default import cfg as our_cfg
    d = tempfile.mkdtemp()
    make_tree(d, "val", scenes=3, queries=11, seed=2, width=200, height=260, frame_step=2)
    cfg = our_cfg.clone()
    cfg.merge_from_file(os.path.join(ROOT, "config", "datasets", "mapfree.yaml"))
    cfg.DATASET.DATA_ROOT = d
    cfg.TRAINING.BATCH_SIZE, cfg.TRAINING.NUM_WORKERS = 4, 0
    _swap_lib(REF)
    import lib.datasets.mapfree as ref_mapfree
    assert ref_mapfree.__file__.startswith(REF)
    ds = ref_mapfree.MapFreeDataset(cfg, "val")
    items = []
    for i in range(len(ds)):
        b = ds[i]
        item = {}
        for k, v in b.items():
            if torch.is_tensor(v) or isinstance(v, np.ndarray):
                item[k] = {"array": digest(v)}
            elif isinstance(v, str) and v.startswith(d):
                item[k] = {"path": os.path.relpath(v, d)}          # paths inside the generated tree, relative to it
            else:
                item[k] = list(v) if isinstance(v, tuple) else v
        items.append(item)
    return items


def reference_cfgs():
    _swap_lib(REF)
    from config.default import cfg as ref_cfg
    out = {}
    for f in ("curriculum_learning.yaml", "overlap_score.yaml", "curriculum_learning_warm_up.yaml",
              "overlap_score_warm_up.yaml"):
        c = ref_cfg.clone()
        c.merge_from_file(os.path.join(REF, "config", "MicKey", f))
        out[f] = c.dump()
    return out


if __name__ == "__main__":
    assert ref_harness.available(), "set MICKEY_REFERENCE_ROOT to a reference checkout"
    with open(os.path.join(HERE, "reference_pose_lines.json"), "w") as f:
        json.dump(pose_lines(), f, indent=1)
    np.savez_compressed(os.path.join(HERE, "reference_stagewise_vits.npz"), **stagewise())
    items = mapfree_items()
    with open(os.path.join(HERE, "reference_mapfree_items.json"), "w") as f:
        json.dump(items, f, indent=1)
    for name, text in reference_cfgs().items():
        with open(os.path.join(HERE, "reference_cfg_" + name), "w") as f:
            f.write(text)
