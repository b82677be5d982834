"""tools/run_submission.py --localize (only the queries extracted, each batch posed against the cached references of its
scenes in one call) writes the same submission.zip as --share-reference and as the paired path, byte for byte: under one
--seed every path draws the same seed per batch."""
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


@pytest.mark.parametrize("uint8", [False, True])
def test_localize_writes_the_same_submission(tmp_path, uint8):
    from mickey_b200.config import CfgNode, mickey_cfg
    cfg = mickey_cfg("vits", 2, 8)
    (tmp_path / "model.yaml").write_text(CfgNode({k: cfg[k] for k in ("MODEL", "MICKEY", "FEATURE_MATCHER", "PROCRUSTES")}).dump())
    # 3 scenes x 3 pairs in batches of 4: batches straddle two scenes' references, and the last one holds one pair
    make_tree(str(tmp_path / "data"), "val", scenes=3, queries=11, seed=5, width=196, height=224)
    u8 = ["--uint8"] if uint8 else []
    s_paired, paired = _run(tmp_path, "paired", *u8)
    s_shared, shared = _run(tmp_path, "shared", "--share-reference", *u8)
    s_loc, loc = _run(tmp_path, "localize", "--localize", *u8)
    assert s_paired["pairs"] == s_loc["pairs"] == 9 and s_loc["references_extracted_rank0"] == 3
    assert s_loc["localize"] and s_loc["share_reference"] and not s_shared["localize"]
    assert sorted(loc) == ["pose_s00000.txt", "pose_s00001.txt", "pose_s00002.txt"]
    assert loc == shared == paired
