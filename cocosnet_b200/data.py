"""Data for train.py / test.py, in the reference's batch-dict schema (data/pix2pix_dataset.py:138-144): label, image,
ref, label_ref, self_ref, path.

create_dataloader reads the real ADE20k, CelebA-HQ and DeepFashion datasets (cocosnet_b200/datasets.py) when
--dataroot is an existing directory.  Otherwise -- and for celebahqedge, flickr and synthetic, which have no reader --
it serves SyntheticDataset: blocky random label maps and uniform-noise images, which is also what bench.py and the
tests feed the model (synthetic_batch).
"""
import os
import random

import numpy as np
import torch
import torch.utils.data


def blocky_labels(rng, n_classes, size, block=16):
    lab = rng.integers(0, n_classes, size=(size // block, size // block))
    return np.repeat(np.repeat(lab, block, axis=0), block, axis=1)


class SyntheticDataset(torch.utils.data.Dataset):
    def __init__(self, opt, length=64, seed=1234):
        self.opt = opt
        self.length = max(length, 12)  # reference train.py:27 touches dataset[11]
        self.seed = seed
        self.real_reference_probability = 1 if opt.phase == "test" else getattr(opt, "real_reference_probability", 0.7)
        self.hard_reference_probability = 0 if opt.phase == "test" else getattr(opt, "hard_reference_probability", 0.2)

    def __len__(self):
        return self.length

    def _label(self, rng):
        opt, s = self.opt, self.opt.crop_size
        mode = opt.dataset_mode
        if mode == "deepfashion":  # 3-ch stick figure + 17 distance maps, float in [0,1]
            return torch.from_numpy(rng.uniform(0, 1, (20, s, s)).astype(np.float32))
        if mode == "celebahqedge":
            return torch.from_numpy(rng.integers(0, 2, (15, s, s)).astype(np.float32))
        if mode == "celebahq":  # ids interleaved with a {0,1} glasses channel; class 16 (= -3) must be absent
            ids = blocky_labels(rng, 16, s)
            glasses = (blocky_labels(rng, 2, s) > 0).astype(np.int64)
            return torch.from_numpy(np.stack([ids, glasses]).astype(np.float32))
        n = opt.label_nc + (1 if opt.contain_dontcare_label else 0)
        return torch.from_numpy(blocky_labels(rng, n, s)[None].astype(np.float32))

    def __getitem__(self, index):
        rng = np.random.default_rng(self.seed + index)
        s = self.opt.crop_size
        img = lambda: torch.from_numpy(rng.uniform(-1, 1, (3, s, s)).astype(np.float32))  # noqa: E731
        return {"label": self._label(rng), "image": img(), "path": "synthetic_%d" % index,
                "self_ref": torch.ones(3, s, s) if index % 2 == 0 else torch.zeros(3, s, s),  # self-reference flag
                "ref": img(), "label_ref": self._label(rng)}


def synthetic_batch(opt, batch, seed=1234, pin=False):
    ds = SyntheticDataset(opt, length=max(batch, 12), seed=seed)
    items = [ds[i] for i in range(batch)]
    out = {k: torch.stack([it[k] for it in items]) for k in ("label", "image", "ref", "label_ref", "self_ref")}
    out["path"] = [it["path"] for it in items]
    if pin:
        out = {k: (v.pin_memory() if torch.is_tensor(v) else v) for k, v in out.items()}
    return out


def create_dataloader(opt, seed=0):
    """Global batches of opt.batchSize (data/__init__.py:40-60).  The shuffle order comes from a generator seeded
    identically on every rank, so with one process per GPU all ranks draw the SAME global batch and
    trainer.shard_batch() hands each its contiguous slice -- DataParallel.scatter's split of one batch.

    A real reader (when opt.dataroot is a directory and the mode has one) decodes in opt.nThreads workers.  Its
    random draws (crops, flips, references) then agree on every rank too: the DataLoader seeds each worker's `random`
    from the same generator, and this process's `random` -- which the DeepFashion reference lists draw from while they
    are read, and which serves every item when opt.nThreads is 0 -- is seeded from `seed` before the reader is built.
    The synthetic data is generated in the main process from per-item seeds."""
    from .datasets import READERS
    gen = torch.Generator()
    gen.manual_seed(seed)
    if opt.dataset_mode in READERS and os.path.isdir(opt.dataroot):
        random.seed(seed)
        ds = READERS[opt.dataset_mode](opt)
        print("dataset [%s] of size %d was created" % (type(ds).__name__, len(ds)))
        return torch.utils.data.DataLoader(ds, batch_size=opt.batchSize, shuffle=not opt.serial_batches,
                                           num_workers=int(opt.nThreads), drop_last=opt.isTrain, generator=gen)
    ds = SyntheticDataset(opt)
    print("dataset [%s] of size %d was created" % (type(ds).__name__, len(ds)))
    return torch.utils.data.DataLoader(ds, batch_size=opt.batchSize, shuffle=not opt.serial_batches,
                                       num_workers=0, drop_last=opt.isTrain, generator=gen)


def seeded_vgg_state_dict(seed=7):
    """Deterministic stand-in for models/vgg19_conv.pth (pix2pix_model.py:30 loads it; not redistributable and not in
    the reference tree): He-normal conv weights, zero bias.  Same recipe as oracle/ref_harness.py uses for the
    reference side of the goldens."""
    from .nets import VGG19_feature_color_torchversion
    g = torch.Generator().manual_seed(seed)
    sd = VGG19_feature_color_torchversion().state_dict()
    for key, v in sd.items():
        if key.endswith("weight"):
            v.copy_(torch.randn(v.shape, generator=g) * (2.0 / v[0].numel()) ** 0.5)
        else:
            v.zero_()
    return sd
