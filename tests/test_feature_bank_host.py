"""CPU tests of the feature-bank path's host side: index validation of pose_from_features, the reference cache of
tools/run_submission.py --share-reference, and the dataset option that leaves image0 out of each item."""
import os
import sys

import numpy as np
import pytest
import torch

from tests.common import ROOT

sys.path.insert(0, os.path.join(ROOT, "compat")) if __import__("importlib").util.find_spec("transforms3d") is None else None

from config.default import cfg as _cfg                              # noqa: E402
from lib.datasets.datamodules import DataModule                      # noqa: E402
from lib.datasets.mapfree import MapFreeDataset                      # noqa: E402
from mickey_b200._lib import MickeyB200Error                         # noqa: E402
from mickey_b200.model import MickeyFeatures, validate_pairs         # noqa: E402
from tools.make_synthetic_mapfree import make_tree                   # noqa: E402
from tools.run_submission import ReferenceBank                       # noqa: E402


def _bank(n, grid=(3, 4), device="cpu"):
    N = grid[0] * grid[1]
    z = lambda *s: torch.zeros(*s, device=device)                    # noqa: E731
    return MickeyFeatures(z(n, 2, N), z(n, 1, N), z(n, 1, N), z(n, 128, N), grid, (grid[0] * 14, grid[1] * 14))


def test_validate_pairs_accepts_host_lists_and_tensors():
    a, b = _bank(1), _bank(5)
    assert validate_pairs(a, [0, 0, 0], b, [4, 0, 2]) == ([0, 0, 0], [4, 0, 2])
    assert validate_pairs(a, torch.zeros(2, dtype=torch.int64), b, range(2)) == ([0, 0], [0, 1])
    assert validate_pairs(b, np.array([3, 1], dtype=np.int32), b, (np.int64(1), 3)) == ([3, 1], [1, 3])
    assert validate_pairs(b, torch.tensor([[1], [2]], dtype=torch.int32), b, [0, 4]) == ([1, 2], [0, 4])


@pytest.mark.parametrize("i0,i1", [([1], [0]), ([0], [5]), ([-1], [0]), ([0, 0], [1]), ([], []), ([0.0], [1]), ([True], [1]),
                                   (torch.tensor([0.0]), [1]), (torch.tensor([True]), [1]), (["0"], [1])])
def test_validate_pairs_rejects_bad_indices(i0, i1):
    with pytest.raises(MickeyB200Error):
        validate_pairs(_bank(1), i0, _bank(5), i1)


def test_validate_pairs_rejects_mixed_geometry_shapes_and_devices():
    with pytest.raises(MickeyB200Error, match="geometry"):
        validate_pairs(_bank(2), [0], _bank(2, grid=(4, 3)), [1])
    broken = _bank(2)
    broken.dsc = torch.zeros(2, 128, 7)
    with pytest.raises(MickeyB200Error):
        validate_pairs(broken, [0], _bank(2), [1])
    short = _bank(2)
    short.scr = torch.zeros(1, 1, 12)
    with pytest.raises(MickeyB200Error):
        validate_pairs(short, [0], _bank(2), [1])
    odd = _bank(2)
    odd.image_size = (28, 56)
    with pytest.raises(MickeyB200Error, match="token grid"):
        validate_pairs(odd, [0], odd, [1])
    with pytest.raises(MickeyB200Error, match="devices"):
        validate_pairs(_bank(2), [0], _bank(2, device="meta"), [1])


def test_features_cat_keeps_order_and_checks_geometry():
    a, b = _bank(1), _bank(2)
    a.kps.fill_(1.0)
    b.kps.fill_(2.0)
    ab = MickeyFeatures.cat([a, b])
    assert len(ab) == 3 and ab.kps[:, 0, 0].tolist() == [1.0, 2.0, 2.0] and ab.grid == a.grid
    assert MickeyFeatures.cat([a]) is a
    with pytest.raises(MickeyB200Error):
        MickeyFeatures.cat([a, _bank(1, grid=(4, 3))])


def test_reference_bank_extracts_each_reference_once():
    loads, extracted = [], []

    def load(root, name):
        loads.append((root, name))
        return f"img:{root}/{name}"

    def extract(image):
        extracted.append(image)
        return f"feat:{image}"

    refs = ReferenceBank(load, extract)
    r0, r1, r2 = ("s0", "seq0/frame_00000.jpg"), ("s1", "seq0/frame_00000.jpg"), ("s2", "seq0/frame_00000.jpg")
    banks, idx = refs.lookup([r0, r0, r0])
    assert banks == ["feat:img:s0/seq0/frame_00000.jpg"] and idx == [0, 0, 0]
    banks, idx = refs.lookup([r0, r1, r1, r1])                          # a batch that straddles two scenes
    assert len(banks) == 2 and banks[0] == "feat:img:s0/seq0/frame_00000.jpg" and idx == [0, 1, 1, 1]
    banks, idx = refs.lookup([r1, r1])
    assert banks == ["feat:img:s1/seq0/frame_00000.jpg"] and idx == [0, 0]
    assert list(refs.cache) == [r1]                                      # s0's features are dropped with its last pair
    banks, idx = refs.lookup([r1, r2, r2])
    assert idx == [0, 1, 1]
    assert loads == [r0, r1, r2] and refs.extracted == 3 and len(extracted) == 3


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    d = tmp_path_factory.mktemp("mapfree_bank")
    make_tree(str(d), "val", scenes=2, queries=11, seed=4, width=200, height=260)
    return str(d)


def _cfg_for(tree, bs=4):
    cfg = _cfg.clone()
    cfg.merge_from_file(os.path.join(ROOT, "config", "datasets", "mapfree.yaml"))
    cfg.DATASET.DATA_ROOT = tree
    cfg.TRAINING.BATCH_SIZE, cfg.TRAINING.NUM_WORKERS = bs, 0
    return cfg


def _same(a, b):
    if torch.is_tensor(a):
        return torch.equal(a, b)
    if isinstance(a, np.ndarray):
        return np.array_equal(a, b)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return a == b


@pytest.mark.parametrize("u8", [False, True])
def test_skip_image0_items_equal_default_items_without_image0(tree, u8):
    cfg = _cfg_for(tree)
    full, lean = MapFreeDataset(cfg, "val", uint8_images=u8), MapFreeDataset(cfg, "val", uint8_images=u8, skip_image0=True)
    assert len(full) == len(lean) == 6
    for i in range(len(full)):
        a, b = full[i], lean[i]
        assert "image0" not in b and set(a) - set(b) == {"image0"}
        assert all(_same(a[k], b[k]) for k in b), i
        scene = lean.datasets[0 if i < 3 else 1]
        assert _same(scene.image(b["pair_names"][0]), a["image0"])        # what the driver reads once per scene
    dl_full = DataModule(cfg, drop_last_val=False, uint8_images=u8).val_dataloader()
    dl_lean = DataModule(cfg, drop_last_val=False, uint8_images=u8, skip_image0=True).val_dataloader()
    for a, b in zip(dl_full, dl_lean):
        assert "image0" not in b and all(_same(a[k], b[k]) for k in b)
