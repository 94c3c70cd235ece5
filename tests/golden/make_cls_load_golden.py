"""Generate tests/golden/cls_load.npz by running the UNMODIFIED reference's classification dataloader
(utils/dataloaders.py create_classification_dataloader -> ClassificationDataset + InfiniteDataLoader) through
tests/golden/refshim.py, and pin oracle/cls_load_ref.py to it.

Runs only where the reference tree, cv2 and torchvision exist:
    python tests/golden/make_cls_load_golden.py
An ImageFolder of seeded synthetic PNGs (lossless) in 3 classes at imgsz 32, sized so that CenterCrop takes every path:
a non-integer shrink, m = 2 * size and 3 * size, m = size, enlargements, 1-pixel sides, odd h - m and w - m (the // 2
floors), portrait, landscape and square.  Albumentations is not installed, so augment=True yields classify_transforms too.
For augment in (True, False), cache in (False, "ram", "disk") and workers in (0, 2), the loader is driven as
classify/train.py drives it: one next(iter(loader)), then three full passes.
Hard asserts while generating: every batch tensor equals the oracle's transform of its image bit for bit, every label is
the item's class, and all runs draw the same index stream (the order depends on neither workers, cache nor augment).
The fixture stores each image's source and expected tensor once, plus the recorded index stream.
"""
from __future__ import annotations

import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import cv2  # noqa: E402
import refshim  # noqa: E402
import torch  # noqa: E402

from oracle import cls_load_ref as R  # noqa: E402

IMG_SIZE = 32
BATCH = 5
# (h, w) per class: non-integer shrink, m = 2s (odd w - m), m = 3s portrait, m = s (odd w - m), enlargement (odd w - m),
# 1-pixel sides, odd h - m portrait, square, tall and wide strips
SHAPES = [[(50, 75), (64, 81), (120, 96), (32, 45)],
          [(20, 27), (1, 40), (40, 1), (77, 50)],
          [(33, 33), (65, 64), (9, 100), (100, 7), (47, 47)]]


def synth_image(h, w, seed):
    """Seeded uint8 BGR image: wrapping integer ramps with a sprinkle of random pixels (low entropy keeps the fixture
    small; noisy images are covered by the oracle's sweep against cv2 and the kernel's sweep against the oracle)."""
    rs = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    a, k = rs.randint(1, 9, 3), int(rs.randint(1, 5))
    im = np.stack([(a[c] * (xx + k * yy) + 40 * c) % 256 for c in range(3)], -1).astype(np.uint8)
    hit = rs.rand(h, w) < 0.02
    im[hit] = rs.randint(0, 256, (int(hit.sum()), 3))
    return im


def gen():
    assert "RANK" not in os.environ, "the recorded stream is the single-process one (RANK -1)"
    refshim.install()
    from utils.dataloaders import create_classification_dataloader

    store, meta = {}, {"img_size": IMG_SIZE, "batch": BATCH, "runs": {}}
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, "val")
        seed = 900
        for c, shapes in enumerate(SHAPES):
            os.makedirs(os.path.join(root, f"class{c}"))
            for k, (h, w) in enumerate(shapes):
                cv2.imwrite(os.path.join(root, f"class{c}", f"im{k}.png"), synth_image(h, w, seed))
                seed += 1
        stream = None
        for augment in (False, True):
            for cache in (False, "ram", "disk"):
                for workers in (0, 2):
                    for f in os.listdir(root):
                        for g in os.listdir(os.path.join(root, f)):
                            if g.endswith(".npy"):
                                os.remove(os.path.join(root, f, g))
                    loader = create_classification_dataloader(root, imgsz=IMG_SIZE, batch_size=BATCH, augment=augment, cache=cache, rank=-1,
                                                              workers=workers)
                    ds = loader.dataset
                    assert ds.album_transforms is None and loader.num_workers == workers
                    if "files" not in meta:
                        meta["files"] = [os.path.relpath(s[0], root) for s in ds.samples]
                        meta["labels"] = [int(s[1]) for s in ds.samples]
                        meta["classes"] = list(ds.classes)
                        for i, s in enumerate(ds.samples):
                            src = cv2.imread(s[0])
                            store[f"src{i}"] = src
                            want = ds.torch_transforms(src).numpy()
                            assert np.array_equal(R.transform(src, IMG_SIZE).view(np.uint32), want.view(np.uint32)), (i, src.shape)
                            store[f"img{i}"] = want
                    assert [os.path.relpath(s[0], root) for s in ds.samples] == meta["files"]
                    index = {store[f"img{i}"].tobytes(): i for i in range(len(ds.samples))}
                    assert len(index) == len(ds.samples), "the expected tensors must be distinct"

                    def record(batch):
                        images, labels = batch
                        assert images.dtype == torch.float32 and labels.dtype == torch.int64
                        got = [index[x.numpy().tobytes()] for x in images]  # KeyError: a tensor the oracle does not reproduce
                        assert labels.tolist() == [meta["labels"][i] for i in got]
                        return got

                    run = dict(first=record(next(iter(loader))), passes=[[record(b) for b in loader] for _ in range(3)])
                    assert all(len(p) == len(loader) for p in run["passes"])
                    if cache == "disk":
                        assert all(os.path.exists(str(s[2])) for s in ds.samples)
                    stream = stream or run
                    assert run == stream, (augment, cache, workers)
                    meta["runs"][f"augment{int(augment)}.cache_{cache}.workers{workers}"] = run
                    print(f"augment={augment} cache={cache} workers={workers}: {len(loader)} batches per pass, oracle == reference")
                    del loader, ds  # its worker processes stop before the next run clears the .npy files
    meta["stream"] = stream
    store["meta"] = np.array(json.dumps(meta))
    out = os.path.join(HERE, "cls_load.npz")
    np.savez_compressed(out, **store)
    print("written", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    gen()
