"""Generate tests/golden/seg_aug.npz by running the UNMODIFIED reference's segmentation training dataloader
(reference utils/segment/dataloaders.py LoadImagesAndLabelsAndMasks.__getitem__ + collate_fn, augment=True,
num_workers=0) through tests/golden/refshim.py, with ultralytics' polygon masks from tests/golden/seg_refshim.py,
and pin oracle/seg_aug_ref.py against it.

Runs only where the reference tree and cv2 exist:
    python tests/golden/make_seg_aug_golden.py
Hard asserts, while generating, for hyps scratch-low, scratch-med (mixup 0.1) and a mosaic-0.5 / rotation / shear /
flipud hyp, each with overlap True and False and downsample_ratio 1 and 4:
  * the oracle reproduces every reference batch: images byte for byte, targets bit for bit, masks in value, shape and
    dtype -- replaying, in overlap mode, the order the reference's own np.argsort(-areas) returned on this host;
  * its draws consume the random streams exactly as the reference does.
The fixture stores the batches under the engine's rule for equal areas (label order), and `meta` records every image
where that order differs from this host's argsort.  The synthetic polygons include concave, self-intersecting, partly
and wholly outside ones, and an image without labels; img_size 128.
"""
from __future__ import annotations

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
import seg_refshim  # noqa: E402
import torch  # noqa: E402

from oracle import seg_aug_ref  # noqa: E402

IMG_SIZE = 128
BATCH = 4
N_BATCHES = 2
SHAPES = [(96, 128), (128, 96), (100, 150), (40, 200), (200, 30), (128, 128), (70, 90)]
SEEDS = {"low": 21, "med": 22, "mixed": 23}


def load_hyps():
    import yaml

    def hyp(name):
        with open(os.path.join(refshim.REFERENCE_ROOT, "data", "hyps", f"hyp.{name}.yaml")) as f:
            return yaml.safe_load(f)

    low = hyp("scratch-low")
    return {"low": low, "med": hyp("scratch-med"), "mixed": dict(low, mosaic=0.5, degrees=30.0, shear=10.0, flipud=0.5, scale=0.6, mixup=0.5)}


def synth_polygon(rs, kind):
    """One float32 normalised polygon: 0 star (concave), 1 random order (self-intersecting), 2 partly outside [0, 1],
    3 wholly outside, 4 a thin sliver, 5 a few points."""
    c = rs.uniform(0.15, 0.85, 2)
    if kind == 0:
        n = int(rs.randint(5, 12)) * 2
        t = np.linspace(0, 2 * np.pi, n, endpoint=False)
        rad = np.where(np.arange(n) % 2, rs.uniform(0.03, 0.08), rs.uniform(0.12, 0.3))
        pts = c + np.stack([np.cos(t), np.sin(t)], 1) * rad[:, None]
    elif kind == 1:
        pts = c + rs.uniform(-0.25, 0.25, (int(rs.randint(4, 9)), 2))
    elif kind == 2:
        pts = rs.uniform(-0.2, 0.5, 2) + rs.uniform(0, 0.6, (int(rs.randint(3, 8)), 2))
    elif kind == 3:
        pts = np.array([1.05, 0.3]) + rs.uniform(0, 0.3, (5, 2))
    elif kind == 4:
        pts = np.array([c, c + [0.4, 0.01], c + [0.4, 0.02]])
    else:
        pts = c + rs.uniform(-0.1, 0.1, (3, 2))
    return pts.astype(np.float32)


def synth_labels(rs, n, k):
    """n polygons and their labels (class, segments2boxes xywh) for image k."""
    segs = [synth_polygon(rs, (k + j) % 6) for j in range(n)]
    boxes = []
    for s in segs:
        x, y = s.T
        x1, y1, x2, y2 = x.min(), y.min(), x.max(), y.max()
        boxes.append([(x1 + x2) / 2, (y1 + y2) / 2, x2 - x1, y2 - y1])
    lab = np.concatenate((rs.randint(0, 80, (n, 1)), np.array(boxes)), 1).astype(np.float32)
    return lab, segs


def make_dataset(tmp, hyp, overlap, ratio, cls, Albumentations):
    rs = np.random.RandomState(6)
    from oracle import pre_ref

    files, labels, segments = [], [], []
    for k, (h, w) in enumerate(SHAPES):
        f = os.path.join(tmp, f"im{k}.png")
        cv2.imwrite(f, pre_ref.synth_image(h, w, 200 + k))
        files.append(f)
        if k == 5:
            labels.append(np.zeros((0, 5), np.float32))
            segments.append([])
        else:
            lab, segs = synth_labels(rs, 2 + k % 4 * 2, k)
            labels.append(lab)
            segments.append(segs)
    ds = cls.__new__(cls)
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
    ds.segments = segments
    ds.shapes = np.array([(w, h) for h, w in SHAPES])
    ds.n = n
    ds.indices = np.arange(n)
    ds.ims = [None] * n
    ds.npy_files = [Path(f).with_suffix(".npy") for f in files]
    ds.overlap, ds.downsample_ratio = overlap, ratio
    return ds


def gen():
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

    # ultralytics.utils.ops box conversions the reference's dataloader imports (as in make_aug_golden.py)
    refshim._REAL["ultralytics.utils.ops"].update(xyxy2xywhn=xyxy2xywhn, xywhn2xyxy=xywhn2xyxy)
    seg_refshim.register(refshim)
    refshim.install()
    from utils import augmentations as ref_aug
    from utils.segment.dataloaders import LoadImagesAndLabelsAndMasks

    store, meta = {}, {"order_differs": []}
    with tempfile.TemporaryDirectory() as tmp:
        for tag, hyp in HYPS.items():
            for overlap in (True, False):
                for ratio in (1, 4):
                    run = f"{tag}.o{int(overlap)}.r{ratio}"
                    ds = make_dataset(tmp, hyp, overlap, ratio, LoadImagesAndLabelsAndMasks, ref_aug.Albumentations)
                    if "src0" not in store:
                        for k in range(ds.n):
                            im, hw0, _ = ds.load_image(k)
                            store[f"src{k}"] = im
                            store[f"hw0_{k}"] = np.array(hw0)
                            store[f"labels{k}"] = ds.labels[k]
                            for j, s in enumerate(ds.segments[k]):
                                store[f"seg{k}_{j}"] = s
                    seed = SEEDS[tag]
                    random.seed(seed)
                    np.random.seed(seed)
                    seg_refshim.OVERLAP_ORDERS.clear()
                    loader = torch.utils.data.DataLoader(ds, batch_size=BATCH, shuffle=False, num_workers=0,
                                                         collate_fn=LoadImagesAndLabelsAndMasks.collate_fn)
                    ref = [(im.numpy(), t.numpy(), m.numpy()) for im, t, _, _, m in loader]
                    assert len(ref) == N_BATCHES
                    next_ref = (random.random(), np.random.random())
                    orders = list(seg_refshim.OVERLAP_ORDERS)
                    random.seed(seed)
                    np.random.seed(seed)
                    states = []
                    for bi, (ri, rt, rm) in enumerate(ref):
                        idx = list(range(bi * BATCH, min((bi + 1) * BATCH, ds.n)))
                        states.append((random.getstate(), np.random.get_state()))
                        imgs, targets, masks, params = seg_aug_ref.get_batch(ds, idx, overlap, ratio, order=lambda areas: orders.pop(0))
                        assert np.array_equal(imgs, ri), (run, bi, "images")
                        assert targets.shape == rt.shape and np.array_equal(targets.view(np.uint32), rt.view(np.uint32)), (run, bi, "targets")
                        assert masks.dtype == rm.dtype and masks.shape == rm.shape and np.array_equal(masks, rm), (run, bi, "masks", masks.dtype, rm.dtype)
                    assert not orders and (random.random(), np.random.random()) == next_ref, (run, "draw count")
                    # the fixture: the same draws under the engine's rule for equal areas
                    for bi, (rs_, ns_) in enumerate(states):
                        random.setstate(rs_)
                        np.random.set_state(ns_)
                        idx = list(range(bi * BATCH, min((bi + 1) * BATCH, ds.n)))
                        imgs, targets, masks, params = seg_aug_ref.get_batch(ds, idx, overlap, ratio)
                        if not (np.array_equal(targets, ref[bi][1]) and masks.dtype == ref[bi][2].dtype and np.array_equal(masks, ref[bi][2])):
                            meta["order_differs"].append([run, bi])
                        if f"{tag}.imgs{bi}" in store:  # the images do not depend on the mask options
                            assert np.array_equal(store[f"{tag}.imgs{bi}"], imgs), (run, bi)
                        store[f"{tag}.imgs{bi}"] = imgs
                        store[f"{run}.targets{bi}"] = targets
                        store[f"{run}.masks{bi}"] = masks
                        store[f"{run}.mosaic{bi}"] = np.array([p["mosaic"] for p in params])
                        store[f"{run}.mixup{bi}"] = np.array([p["mosaic"] and len(p["m"]) == 2 for p in params])
                    store[f"{run}.seed"] = np.array(seed)
                    print(f"{run}: oracle == reference, mask dtypes {[str(b[2].dtype) for b in ref]}, targets {[len(b[1]) for b in ref]}")
    meta["runs"] = sorted({k.rsplit(".", 1)[0] for k in store if k.endswith(".seed")})
    store["hyps"] = np.array(json.dumps(HYPS))
    store["meta"] = np.array(json.dumps(meta))
    np.savez_compressed(f"{HERE}/seg_aug.npz", **store)
    print("order differs:", meta["order_differs"])
    print("written", f"{HERE}/seg_aug.npz", os.path.getsize(f"{HERE}/seg_aug.npz"), "bytes")


if __name__ == "__main__":
    gen()
