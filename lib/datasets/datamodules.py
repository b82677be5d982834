"""DataModule with the reference's surface for inference (lib/datasets/datamodules.py:12-67): val_dataloader() /
test_dataloader() over the Map-free scenes, batch size and workers from cfg.TRAINING.  Additions for the H100 path:
`uint8_images` (uint8 HWC batches for the fused ingest kernel), `skip_image0` (items without the reference image, which
the caller reads once per scene), `pin_memory`, and rank-sharding of the pair list when
torch.distributed is initialised (one process per GPU).  The training loader (scene-balanced sampler, colour jitter)
belongs to the training side, which is out of scope here."""
from torch.utils.data import DataLoader

from lib.datasets.mapfree import MapFreeDataset
from lib.datasets.sampler import ShardedSequentialSampler


class DataModule:
    def __init__(self, cfg, drop_last_val=True, uint8_images=False, pin_memory=False, shard=True, skip_image0=False):
        self.cfg = cfg
        self.drop_last_val = drop_last_val
        self.uint8_images = uint8_images
        self.skip_image0 = skip_image0
        self.pin_memory = pin_memory
        self.shard = shard
        datasets = {"MapFree": MapFreeDataset}
        assert cfg.DATASET.DATA_SOURCE in datasets, "invalid DATA_SOURCE, this dataset is not implemented"
        self.dataset_type = datasets[cfg.DATASET.DATA_SOURCE]

    def _loader(self, mode):
        dataset = self.dataset_type(self.cfg, mode, uint8_images=self.uint8_images, skip_image0=self.skip_image0)
        sampler = ShardedSequentialSampler(dataset) if self.shard else None
        return DataLoader(dataset, batch_size=self.cfg.TRAINING.BATCH_SIZE, num_workers=self.cfg.TRAINING.NUM_WORKERS,
                          sampler=sampler, shuffle=False, drop_last=self.drop_last_val, pin_memory=self.pin_memory)

    def val_dataloader(self):
        return self._loader("val")

    def test_dataloader(self):
        return self._loader("test")

    def train_dataloader(self):
        raise NotImplementedError("training is outside the inference hot path (SURVEY.md §2 row 8)")
