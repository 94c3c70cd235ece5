"""The datasets behind tests/golden/val_load.npz, duck-typed on the attributes the reference's LoadImagesAndLabels[AndMasks]
exposes to the validation loaders.  The source images come from the fixture through `decode` (no image codec): the
originals, or with `cache=True` the RAM cache load_image fills (oracle/val_load_ref.load_resize, which the fixture's
generator checked against the reference's load_image)."""
import json
import os

import numpy as np

from oracle import val_load_ref as V

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "val_load.npz")
IMG_SIZE = 64  # meta['img_size'] of the fixture


def load():
    return np.load(GOLDEN)


def meta(z):
    return json.loads(str(z["meta"]))


def runs(z):
    return sorted(meta(z)["runs"])


class ValDataset:
    def __init__(self, z, run, cache=False):
        m = meta(z)["runs"][run]
        order = m["order"]
        n = len(order)
        self.run, self.order, self.batch_size = run, order, m["batch"]
        self.src = [z[f"src{k}"] for k in order]
        self.labels = [z[f"labels{k}"] for k in order]
        self.segments = []
        for k in order:
            if f"segs{k}" in z.files:
                self.segments.append(np.split(z[f"segs{k}"], np.cumsum(z[f"seglen{k}"])[:-1]))
            else:
                self.segments.append([])
        self.img_size = IMG_SIZE
        self.augment, self.image_weights, self.rect, self.mosaic = False, False, m["rect"], False
        self.batch = np.floor(np.arange(n) / m["batch"]).astype(int)
        if self.rect:
            self.batch_shapes = z[f"{run}.batch_shapes"]
        self.indices = np.arange(n)
        self.n = n
        self.im_files = [f"im{k}.png" for k in order]
        self.im_hw0 = [s.shape[:2] for s in self.src]
        assert meta(z)["img_size"] == IMG_SIZE
        self.ims = [V.load_resize(s, IMG_SIZE) for s in self.src] if cache else [None] * n
        if m["overlap"] is not None:
            self.overlap, self.downsample_ratio = m["overlap"], m["ratio"]
        self.n_batches = m["batches"]

    def __len__(self):
        return self.n


def decode(ds, i):
    """The loader's decode step over the fixture's arrays (load_val_image's contract)."""
    if ds.ims[i] is not None:
        return ds.ims[i], tuple(ds.im_hw0[i]), True
    return ds.src[i], tuple(ds.src[i].shape[:2]), False


def expected(z, run, bi):
    """(imgs, targets, shapes, masks or None) the reference yielded for batch bi of `run`."""
    key = "det.rect" if run.startswith("seg.") else run
    masks = z[f"{run}.masks{bi}"] if f"{run}.masks{bi}" in z.files else None
    return z[f"{key}.imgs{bi}"], z[f"{run}.targets{bi}"], json.loads(str(z[f"{run}.shapes{bi}"])), masks


def as_json(shapes):
    return json.loads(json.dumps([[list(a), [list(b), list(c)]] for a, (b, c) in shapes]))
