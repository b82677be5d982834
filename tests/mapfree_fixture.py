"""The recorded Map-free grading fixture (tests/golden/reference_mapfree_eval.json, made by
tests/golden/make_mapfree_eval_fixture.py): its val tree and submission zips written back to disk, and the graded frames
of a zip as mk_mapfree_frame_metrics takes them."""
import json
import os
import zipfile
from pathlib import Path

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
with open(os.path.join(HERE, "golden", "reference_mapfree_eval.json")) as _f:
    FIX = json.load(_f)
GRADED_ZIPS = [z for z, rec in FIX["zips"].items() if rec.get("output")]


def write_tree(root: Path) -> Path:
    """<root>/val/<scene>/{intrinsics.txt, poses.txt} -> root."""
    for scene, files in FIX["scenes"].items():
        d = Path(root) / FIX["split"] / scene
        d.mkdir(parents=True, exist_ok=True)
        for name, text in files.items():
            (d / name).write_text(text)
    return Path(root)


def write_zip(root: Path, name: str) -> Path:
    path = Path(root) / f"{name}.zip"
    with zipfile.ZipFile(path, "w") as zf:
        for member, text in FIX["zips"][name]["files"].items():
            zf.writestr(member, text.encode("utf-8"))
    return path


def graded_frames(root: Path, name: str):
    """[(scene, frames)] of zip `name` in the fixture's scene order, frames as mapfree_eval._scene_frames collects them
    (scenes without a file in the zip are left out)."""
    from mickey_b200 import mapfree_eval as mfe
    zp = write_zip(root, name)
    out = []
    with zipfile.ZipFile(zp) as zf:
        for scene in FIX["scene_order"]:
            frames, _ = mfe._scene_frames(Path(root) / FIX["split"], zf, scene)
            if frames is not None and len(frames["confidence"]):
                out.append((scene, frames))
    return out


def reference_values(name: str, scene: str) -> np.ndarray:
    """The benchmark's [n, 3] trans_err, rot_err, reproj_err of one scene of zip `name`."""
    res = FIX["zips"][name]["scenes"][scene]["results"]
    return np.array([res["trans_err"], res["rot_err"], res["reproj_err"]], dtype=np.float64).T.reshape(-1, 3)
