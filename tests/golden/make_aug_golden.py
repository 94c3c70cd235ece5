"""Generate tests/golden/aug.npz and aug_signatures.json by running the UNMODIFIED reference's training dataloader
(reference utils/dataloaders.py LoadImagesAndLabels.__getitem__ + collate_fn, augment=True, num_workers=0) through
tests/golden/refshim.py, and pin oracle/aug_ref.py against it and against the installed cv2.

Runs only where the reference tree and cv2 exist:
    python tests/golden/make_aug_golden.py
Hard asserts, while generating:
  * aug_ref.warp_affine == cv2.warpAffine on 400 random affine maps (rotation, shear, scale 0.1-1.9, non-square sources);
  * aug_ref.bgr2hsv / hsv2bgr == cv2.cvtColor over their entire uint8 domains (rows of 32 and of 37 pixels);
  * the oracle reproduces every reference batch byte for byte (images) and bit for bit (targets) -- and its draws
    consume the random streams exactly as the reference does (the next draw after each batch agrees).
The fixture holds the `load_image` outputs of a small synthetic dataset (seeded images of mixed shapes written as PNG
to a temporary directory), its labels, the seeds and the expected batches, at img_size 128.
"""
from __future__ import annotations

import hashlib
import inspect
import json
import os
import random
import sys
import tempfile
from pathlib import Path

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import cv2  # noqa: E402
import refshim  # noqa: E402
import torch  # noqa: E402

from oracle import aug_ref  # noqa: E402

IMG_SIZE = 128
BATCH = 4
N_BATCHES = 2
# original (h, w) of the synthetic images; load_image resizes the long side to IMG_SIZE
SHAPES = [(96, 128), (128, 96), (100, 150), (40, 200), (200, 30), (128, 128), (70, 90)]

def load_hyps():
    """scratch-low, scratch-high (mixup 0.1, scale 0.9) and a hyp with mosaic 0.5, rotation, shear and flipud."""
    import yaml

    def hyp(name):
        with open(os.path.join(refshim.REFERENCE_ROOT, "data", "hyps", f"hyp.{name}.yaml")) as f:
            return yaml.safe_load(f)

    low = hyp("scratch-low")
    return {"low": low, "high": hyp("scratch-high"), "mixed": dict(low, mosaic=0.5, degrees=30.0, shear=10.0, flipud=0.5, scale=0.6, mixup=0.5)}


SEEDS = {"low": 11, "high": 12, "mixed": 13}


def synth_labels(rs, n):
    """Float32 (n, 5) normalised class + xywh labels (some touch the image border); image 5 has none."""
    xy = rs.uniform(0.05, 0.95, (n, 2))
    wh = rs.uniform(0.03, 0.6, (n, 2))
    return np.concatenate((rs.randint(0, 80, (n, 1)), xy, wh), 1).astype(np.float32)


def check_warp():
    rng = np.random.default_rng(0)
    for t in range(400):
        h, w = int(rng.integers(1, 300)), int(rng.integers(1, 300))
        im = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        draws = (0.0, 0.0, float(rng.uniform(-180, 180)), float(rng.uniform(0.1, 1.9)), float(rng.uniform(-20, 20)),
                 float(rng.uniform(-20, 20)), float(rng.uniform(0.3, 0.7)), float(rng.uniform(0.3, 0.7)))
        border = [-int(rng.integers(0, 100))] * 2 if t % 2 else [0, 0]
        M = aug_ref.affine(draws, (h, w), border)
        dsize = (w + 2 * border[1], h + 2 * border[0])
        if dsize[0] <= 0 or dsize[1] <= 0:
            continue
        ref = cv2.warpAffine(im, M[:2], dsize=dsize, borderValue=(114, 114, 114))
        assert np.array_equal(ref, aug_ref.warp_affine(im, M[:2], dsize)), ("warp", t)
        assert np.array_equal(cv2.invertAffineTransform(M[:2]), aug_ref.invert_affine(M[:2])), ("invert", t)
    print("warpAffine: oracle == cv2 on 400 maps")


def check_hsv():
    B, G, R = np.meshgrid(np.arange(256), np.arange(256), np.arange(256), indexing="ij")
    bgr = np.stack([B, G, R], -1).astype(np.uint8).reshape(-1, 3)
    H, S, V = np.meshgrid(np.arange(180), np.arange(256), np.arange(256), indexing="ij")
    hsv = np.stack([H, S, V], -1).astype(np.uint8).reshape(-1, 3)
    digests = {}
    for width in (32, 37):
        n = (len(bgr) // width) * width
        a = bgr[:n].reshape(-1, width, 3)
        ref = cv2.cvtColor(a, cv2.COLOR_BGR2HSV)
        assert np.array_equal(ref, aug_ref.bgr2hsv(a)), ("bgr2hsv", width)
        n = (len(hsv) // width) * width
        a = hsv[:n].reshape(-1, width, 3)
        ref = cv2.cvtColor(a, cv2.COLOR_HSV2BGR)
        assert np.array_equal(ref, aug_ref.hsv2bgr(a)), ("hsv2bgr", width)
    digests["bgr2hsv"] = hashlib.sha256(aug_ref.bgr2hsv(bgr.reshape(-1, 32, 3)).tobytes()).hexdigest()
    digests["hsv2bgr_simd"] = hashlib.sha256(aug_ref.hsv2bgr(hsv.reshape(-1, 32, 3)).tobytes()).hexdigest()
    digests["hsv2bgr_tail"] = hashlib.sha256(aug_ref.hsv2bgr(hsv.reshape(-1, 1, 3)).tobytes()).hexdigest()
    assert np.array_equal(cv2.cvtColor(hsv.reshape(-1, 1, 3), cv2.COLOR_HSV2BGR), aug_ref.hsv2bgr(hsv.reshape(-1, 1, 3)))
    print("cvtColor: oracle == cv2 over both uint8 domains")
    return digests


def make_dataset(tmp, hyp, LoadImagesAndLabels, Albumentations):
    """A LoadImagesAndLabels instance over PNG files, its attributes set as __init__ sets them for augment=True,
    rect=False, cache_images=False (the constructor's file scan and label cache are not part of the arithmetic)."""
    rs = np.random.RandomState(5)
    from oracle import pre_ref

    files, labels = [], []
    for k, (h, w) in enumerate(SHAPES):
        f = os.path.join(tmp, f"im{k}.png")
        cv2.imwrite(f, pre_ref.synth_image(h, w, 100 + k))
        files.append(f)
        labels.append(np.zeros((0, 5), np.float32) if k == 5 else synth_labels(rs, 1 + k % 4 * 3))
    ds = LoadImagesAndLabels.__new__(LoadImagesAndLabels)
    n = len(files)
    ds.img_size, ds.augment, ds.hyp, ds.image_weights, ds.rect = IMG_SIZE, True, hyp, False, False
    ds.mosaic = True
    ds.mosaic_border = [-IMG_SIZE // 2, -IMG_SIZE // 2]
    ds.stride = 32
    ds.albumentations = Albumentations(size=IMG_SIZE)
    assert ds.albumentations.transform is None
    ds.im_files = files
    ds.label_files = [f.replace(".png", ".txt") for f in files]
    ds.labels = labels
    ds.segments = [[] for _ in range(n)]
    ds.shapes = np.array([(w, h) for h, w in SHAPES])
    ds.n = n
    ds.indices = np.arange(n)
    ds.ims = [None] * n
    ds.npy_files = [Path(f).with_suffix(".npy") for f in files]
    return ds


def gen_aug():

    HYPS = load_hyps()

    def xyxy2xywhn(x, w=640, h=640, clip=False, eps=0.0):
        if clip:
            x = refshim.clip_boxes(x, (h - eps, w - eps))
        y = np.empty_like(x, dtype=np.float32)
        y[..., 0] = ((x[..., 0] + x[..., 2]) / 2) / w
        y[..., 1] = ((x[..., 1] + x[..., 3]) / 2) / h
        y[..., 2] = (x[..., 2] - x[..., 0]) / w
        y[..., 3] = (x[..., 3] - x[..., 1]) / h
        return y

    def xywhn2xyxy(x, w=640, h=640, padw=0, padh=0):
        y = np.empty_like(x, dtype=np.float32)
        y[..., 0] = w * (x[..., 0] - x[..., 2] / 2) + padw
        y[..., 1] = h * (x[..., 1] - x[..., 3] / 2) + padh
        y[..., 2] = w * (x[..., 0] + x[..., 2] / 2) + padw
        y[..., 3] = h * (x[..., 1] + x[..., 3] / 2) + padh
        return y

    # ultralytics.utils.ops box conversions the reference's dataloader imports (public package behaviour)
    refshim._REAL["ultralytics.utils.ops"].update(xyxy2xywhn=xyxy2xywhn, xywhn2xyxy=xywhn2xyxy)
    refshim.install()
    from utils import augmentations as ref_aug
    from utils.dataloaders import LoadImagesAndLabels

    check_warp()
    digests = check_hsv()
    store = {}
    with tempfile.TemporaryDirectory() as tmp:
        for tag, hyp in HYPS.items():
            ds = make_dataset(tmp, hyp, LoadImagesAndLabels, ref_aug.Albumentations)
            if tag == "low":
                for k in range(ds.n):
                    im, hw0, hw = ds.load_image(k)
                    store[f"src{k}"] = im
                    store[f"hw0_{k}"] = np.array(hw0)
                    store[f"labels{k}"] = ds.labels[k]
            seed = SEEDS[tag]
            random.seed(seed)
            np.random.seed(seed)
            loader = torch.utils.data.DataLoader(ds, batch_size=BATCH, shuffle=False, num_workers=0, collate_fn=LoadImagesAndLabels.collate_fn)
            ref_batches = [(imgs.numpy(), targets.numpy()) for imgs, targets, _, _ in loader]
            assert len(ref_batches) == N_BATCHES
            next_ref = (random.random(), np.random.random())
            random.seed(seed)
            np.random.seed(seed)
            for bi, (ri, rt) in enumerate(ref_batches):
                idx = list(range(bi * BATCH, min((bi + 1) * BATCH, ds.n)))
                imgs, targets, params = aug_ref.get_batch(ds, idx)
                assert np.array_equal(imgs, ri), (tag, bi, "images", np.argwhere(imgs != ri)[:5])
                assert targets.dtype == rt.dtype and targets.shape == rt.shape and np.array_equal(targets.view(np.uint32), rt.view(np.uint32)), (tag, bi)
                store[f"{tag}.imgs{bi}"] = ri
                store[f"{tag}.targets{bi}"] = rt
                store[f"{tag}.mosaic{bi}"] = np.array([p["mosaic"] for p in params])
                store[f"{tag}.mixup{bi}"] = np.array([p["mosaic"] and len(p["m"]) == 2 for p in params])
                store[f"{tag}.draws{bi}"] = np.array([aug_ref.draw_vector(p) for p in params])
            assert (random.random(), np.random.random()) == next_ref, (tag, "draw count")
            print(f"hyp {tag}: {len(ref_batches)} batches, oracle == reference; mosaic {[bool(x) for k in store if k.startswith(tag + '.mosaic') for x in store[k]]}")
            store[f"{tag}.seed"] = np.array(seed)
    store["hyps"] = np.array(json.dumps(HYPS))
    np.savez_compressed(f"{HERE}/aug.npz", **store)
    sig = {name: [(n, repr(q.default) if q.default is not inspect._empty else None, str(q.kind))
                  for n, q in inspect.signature(getattr(ref_aug, name)).parameters.items()]
           for name in ("random_perspective", "augment_hsv", "mixup")}
    sig["hsv_digest"] = digests
    with open(f"{HERE}/aug_signatures.json", "w") as f:
        json.dump(sig, f, indent=1, sort_keys=True)
    print("written", f"{HERE}/aug.npz", os.path.getsize(f"{HERE}/aug.npz"), "bytes")


if __name__ == "__main__":
    gen_aug()
