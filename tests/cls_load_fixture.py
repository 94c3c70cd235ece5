"""The dataset behind tests/golden/cls_load.npz, duck-typed on the attributes the reference's ClassificationDataset
exposes to the classification loader.  The images come from the fixture's arrays through `decode` (no image codec)."""
import json
import os
from pathlib import Path

import numpy as np

from oracle import cls_load_ref as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cls_load.npz")
IMG_SIZE = 32  # meta['img_size'] of the fixture


def load():
    return np.load(GOLDEN)


def meta(z):
    return json.loads(str(z["meta"]))


class ClsDataset:
    def __init__(self, z, size=IMG_SIZE):
        m = meta(z)
        assert m["img_size"] == IMG_SIZE
        self.root = Path("datasets/fixture/val")
        self.classes = m["classes"]
        self.samples = [[str(self.root / f), j, (self.root / f).with_suffix(".npy"), None] for f, j in zip(m["files"], m["labels"])]
        self.src = [z[f"src{i}"] for i in range(len(self.samples))]
        self.torch_transforms = R.classify_transforms(size)
        self.album_transforms = None
        self.cache_ram = self.cache_disk = False

    def __len__(self):
        return len(self.samples)


def decode(ds, i):
    """The loader's decode step over the fixture's arrays (load_cls_image's contract)."""
    return ds.src[i]


def expected(z, items):
    """(images (B, 3, 32, 32) float32, labels (B,) int64) the reference yielded for dataset items `items`."""
    labels = meta(z)["labels"]
    return np.stack([z[f"img{i}"] for i in items], 0), np.array([labels[i] for i in items], np.int64)
