"""tools/run_submission.py --share-reference (each scene's reference extracted once, pairs posed from feature banks)
writes the same submission.zip as the paired path, byte for byte: under one --seed both paths draw the same seed per
batch."""
import json
import os
import subprocess
import sys
import zipfile

import pytest

from tests.common import ROOT
from tools.make_synthetic_mapfree import make_tree

pytestmark = pytest.mark.gpu


def _run(tmp_path, out, *extra):
    cmd = [sys.executable, os.path.join(ROOT, "tools", "run_submission.py"), "--variant", "vits", "--config",
           str(tmp_path / "model.yaml"), "--checkpoint", "synthetic", "--data_root", str(tmp_path / "data"), "--split", "val",
           "--batch_size", "4", "--workers", "0", "--seed", "7", "-o", str(tmp_path / out), *extra]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=str(tmp_path), env=dict(os.environ, PYTHONPATH=ROOT), timeout=900)
    assert r.returncode == 0, (r.stdout + r.stderr)[-3000:]
    summary = json.loads(r.stdout.strip().splitlines()[-1])
    with zipfile.ZipFile(tmp_path / out / "submission.zip") as z:
        return summary, {n: z.read(n) for n in z.namelist()}


def test_share_reference_writes_the_same_submission(tmp_path):
    from mickey_b200.config import CfgNode, mickey_cfg
    cfg = mickey_cfg("vits", 2, 8)
    (tmp_path / "model.yaml").write_text(CfgNode({k: cfg[k] for k in ("MODEL", "MICKEY", "FEATURE_MATCHER", "PROCRUSTES")}).dump())
    # 2 scenes x 3 pairs in batches of 4: the first batch straddles both scenes' references
    make_tree(str(tmp_path / "data"), "val", scenes=2, queries=11, seed=3, width=196, height=224)
    s_paired, paired = _run(tmp_path, "paired")
    s_shared, shared = _run(tmp_path, "shared", "--share-reference")
    assert s_paired["pairs"] == s_shared["pairs"] == 6 and s_shared["references_extracted_rank0"] == 2
    assert sorted(paired) == ["pose_s00000.txt", "pose_s00001.txt"]
    assert paired == shared
    assert all(len(v.decode().split("\n")) == 3 for v in paired.values())
