"""Map-free relocalisation scenes as a torch Dataset (the reference's lib/datasets/mapfree.py:10-194), rebuilt around a
parsed scene index so that a scene can be enumerated and sharded without touching its images.

On-disk format (one directory per scene under <DATA_ROOT>/<split>/):
    intrinsics.txt   `<frame> fx fy cx cy W H`                       (mapfree.py:31-50)
    poses.txt        `<frame> qw qx qy qz tx ty tz`  world-to-camera  (mapfree.py:52-69)
    overlaps.npz     optional (train): idxs [P,4] = (seqA, imA, seqB, imB), overlaps [P]   (mapfree.py:83-93)
    seq0/frame_00000.jpg (reference image), seq1/frame_XXXXX.jpg (queries)
val / test pairs = (seq0 frame 0, every SAMPLE_FACTOR-th seq1 frame of poses.txt)       (mapfree.py:94-103)

`uint8_images=True` returns the images as uint8 [h, w, 3] (what cv2 hands over) for the fused ingest kernel
(mk_forward_u8); the default returns the reference's float [3, h, w] tensors.  `skip_image0=True` leaves `image0` out of
every item: a caller that extracts each scene's reference image once (tools/run_submission.py --share-reference) reads
it itself, once per scene, instead of the loader decoding it once per pair.
"""
from pathlib import Path

import numpy as np
import torch
import torch.utils.data as data
from transforms3d.quaternions import qinverse, qmult, rotate_vector, quat2mat

from lib.datasets.utils import correct_intrinsic_scale
from mickey_b200.io import read_color_image_u8, to_float_chw

SAMPLE_FACTOR = {"train": 1, "val": 5, "test": 5}


def _rows(path: Path):
    with path.open("r") as f:
        for line in f:
            if "#" in line or not line.strip():
                continue
            parts = line.strip().split(" ")
            yield parts[0], np.array([float(x) for x in parts[1:]])


class MapFreeScene(data.Dataset):
    def __init__(self, scene_root, resize, sample_factor=1, overlap_limits=None, transforms=None, test_scene=False,
                 uint8_images=False, skip_image0=False):
        super().__init__()
        self.scene_root = Path(scene_root)
        self.resize = resize
        self.sample_factor = sample_factor
        self.transforms = transforms
        self.test_scene = test_scene
        self.uint8_images = uint8_images
        self.skip_image0 = skip_image0
        self.poses = self.read_poses(self.scene_root)
        self.K, self.K_ori = self.read_intrinsics(self.scene_root, resize)
        self.pairs = self.load_pairs(self.scene_root, overlap_limits, sample_factor)

    # ---- scene index -------------------------------------------------------------------------------------------
    @staticmethod
    def read_intrinsics(scene_root: Path, resize=None):
        K_scaled, K_native = {}, {}
        for name, v in _rows(Path(scene_root) / "intrinsics.txt"):
            fx, fy, cx, cy, W, H = v
            K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], dtype=np.float32)
            K_native[name] = K
            K_scaled[name] = K if resize is None else correct_intrinsic_scale(K, resize[0] / W, resize[1] / H)
        return K_scaled, K_native

    @staticmethod
    def read_poses(scene_root: Path):
        """frame -> (q [qw qx qy qz], t [tx ty tz]) with X_cam = R(q) X_world + t."""
        return {name: (v[:4], v[4:]) for name, v in _rows(Path(scene_root) / "poses.txt")}

    def load_pairs(self, scene_root: Path, overlap_limits=None, sample_factor=1):
        """[P, 4] = (seqA, imA, seqB, imB).  Train scenes: pairs of overlaps.npz inside the overlap window; val/test:
        the seq0 keyframe against every sample_factor-th seq1 frame listed in poses.txt."""
        npz = Path(scene_root) / "overlaps.npz"
        if npz.exists():
            z = np.load(npz, allow_pickle=True)
            idxs, overlaps = z["idxs"], z["overlaps"]
            if overlap_limits is not None:
                lo, hi = overlap_limits
                return idxs[(overlaps > lo) & (overlaps < hi)].copy()
            return None                                   # the reference returns None here as well (mapfree.py:83-93)
        queries = [int(name[-9:-4]) for name in self.poses if "seq0" not in name]
        pairs = np.zeros((len(self.poses) - 1, 4), dtype=np.uint16)
        pairs[:, 2] = 1
        pairs[:, 3] = np.array(queries, dtype=np.uint16)
        return pairs[::sample_factor]

    @staticmethod
    def get_pair_path(pair):
        seqA, imgA, seqB, imgB = pair
        return f"seq{seqA}/frame_{imgA:05}.jpg", f"seq{seqB}/frame_{imgB:05}.jpg"

    def __len__(self):
        return len(self.pairs)

    # ---- one pair ----------------------------------------------------------------------------------------------
    def image(self, rel):
        """One image of the scene as the items carry it (resized; uint8 HWC or float CHW)."""
        u8 = read_color_image_u8(self.scene_root / rel, self.resize)
        if self.uint8_images:
            return u8
        img = to_float_chw(u8)
        return self.transforms(img) if self.transforms else img

    def relative_pose(self, nameA, nameB):
        """4x4 transform camera A -> camera B and the camera centres (mapfree.py:121-137)."""
        (qA, tA), (qB, tB) = self.poses[nameA], self.poses[nameB]
        cA, cB = rotate_vector(-tA, qinverse(qA)), rotate_vector(-tB, qinverse(qB))
        qAB = qmult(qB, qinverse(qA))
        T = np.eye(4, dtype=np.float32)
        T[:3, :3] = quat2mat(qAB)
        T[:3, 3] = tB - rotate_vector(tA, qAB)
        return T, (qA, cA), (qB, cB)

    def __getitem__(self, index):
        nameA, nameB = self.get_pair_path(self.pairs[index])
        if self.test_scene:                               # no ground truth in the test split
            T = np.zeros([4, 4])
            (qA, cA), (qB, cB) = (np.zeros([4]), np.zeros([3])), (np.zeros([4]), np.zeros([3]))
        else:
            T, (qA, cA), (qB, cB) = self.relative_pose(nameA, nameB)
        item = {} if self.skip_image0 else {"image0": self.image(nameA)}
        item.update({
            "image1": self.image(nameB),
            "T_0to1": torch.from_numpy(T),
            "abs_q_0": qA, "abs_c_0": cA, "abs_q_1": qB, "abs_c_1": cB,
            "K_color0": self.K[nameA], "Kori_color0": self.K_ori[nameA],
            "K_color1": self.K[nameB], "Kori_color1": self.K_ori[nameB],
            "dataset_name": "Mapfree", "scene_id": self.scene_root.stem, "scene_root": str(self.scene_root),
            "pair_id": index * self.sample_factor, "pair_names": (nameA, nameB),
        })
        return item


class MapFreeDataset(data.ConcatDataset):
    def __init__(self, cfg, mode, transforms=None, uint8_images=False, skip_image0=False):
        assert mode in SAMPLE_FACTOR, "Invalid dataset mode"
        root = Path(cfg.DATASET.DATA_ROOT) / mode
        scenes = cfg.DATASET.SCENES
        if scenes is None:
            scenes = sorted(s.name for s in root.iterdir() if s.is_dir())
        if cfg.DEBUG:
            scenes = scenes[:30] if mode == "train" else scenes[:10] if mode == "val" else scenes
        window = (cfg.DATASET.MIN_OVERLAP_SCORE, cfg.DATASET.MAX_OVERLAP_SCORE)
        size = (cfg.DATASET.WIDTH, cfg.DATASET.HEIGHT)
        super().__init__([MapFreeScene(root / s, size, SAMPLE_FACTOR[mode], window, transforms, mode == "test", uint8_images,
                                       skip_image0)
                          for s in scenes])
