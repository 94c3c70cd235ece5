"""Generate tests/golden/val_load.npz by running the UNMODIFIED reference's validation dataloaders
(utils/dataloaders.py LoadImagesAndLabels and utils/segment/dataloaders.py LoadImagesAndLabelsAndMasks, __getitem__ +
collate_fn with augment=False, num_workers=0) through tests/golden/refshim.py, and pin oracle/val_load_ref.py to them.

Runs only where the reference tree and cv2 exist:
    python tests/golden/make_val_load_golden.py
The images are seeded synthetic PNGs (lossless), img_size 64, sized so that load_image takes every path: INTER_AREA
with integer factors 2 and 3 and with non-integer factors, INTER_LINEAR enlargements, the r == 1 copy and 1-pixel
edges.  Runs:
  * det.rect  : rect=True, pad=0.5, batch 4 (the val loader's settings);
  * det.square: rect=False (every image letterboxed into 64 x 64);
  * det.again : rect=True, pad=-0.5, batch 2, so that letterbox resizes the load_image result a second time;
  * seg.o{0,1}.r{1,4}: the rect=True images with polygons, overlap on and off, mask ratio 1 and 4, one image without
    labels and one with 300 (an int32 overlap plane).
Hard asserts while generating: the oracle reproduces every reference batch (images byte for byte, targets bit for bit,
shapes, masks in value, shape and dtype -- replaying, in overlap mode, the order this host's np.argsort returned).  The
fixture stores the masks and targets under the engine's rule for equal areas (label order); `meta` lists the batches
where that differs from this host's argsort.
"""
from __future__ import annotations

import json
import os
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

from oracle import pre_ref, seg_aug_ref  # noqa: E402
from oracle import val_load_ref as V  # noqa: E402

IMG_SIZE = 64  # small sizes keep the fixture small; the GPU tests sweep 333, 640 and 1280 against the oracle
# (h, w): area x2, area x3, area non-integer (r 0.64, and 1366 x 768 scaled), linear, copy, 1-pixel edges, odd enlargement
SHAPES = [(128, 96), (144, 192), (100, 75), (96, 171), (40, 30), (64, 48), (1, 100), (100, 1), (7, 5), (48, 64), (30, 50), (75, 125)]
RUNS = {"det.rect": dict(rect=True, pad=0.5, batch=4), "det.square": dict(rect=False, pad=0.0, batch=4),
        "det.again": dict(rect=True, pad=-0.5, batch=2)}
CROWD = 3  # image with 300 polygons
EMPTY = 7  # image without labels


def synth_image(h, w, seed):
    """Seeded uint8 BGR image: per-channel integer ramps that wrap around (so the interpolation weights and the edges
    matter) with a sprinkle of random pixels.  Low entropy keeps the stored sources and batches small; the arithmetic
    on noisy images is covered by the size sweeps against cv2 and the oracle."""
    rs = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    a, k = rs.randint(1, 9, 3), int(rs.randint(1, 5))  # each row is the previous one shifted by k pixels
    im = np.stack([(a[c] * (xx + k * yy) + 40 * c) % 256 for c in range(3)], -1).astype(np.uint8)
    hit = rs.rand(h, w) < 0.005
    im[hit] = rs.randint(0, 256, (int(hit.sum()), 3))
    return im


def synth_polygon(rs, max_points=16):
    n = int(rs.randint(3, max_points))
    t = np.sort(rs.uniform(0, 2 * np.pi, n))
    c, rad = rs.uniform(-0.1, 1.1, 2), rs.uniform(0.02, 0.5) * rs.uniform(0.3, 1.0, n)
    return (c + np.stack([np.cos(t), np.sin(t)], 1) * rad[:, None]).astype(np.float32)


def synth_labels(rs, k):
    n = 0 if k == EMPTY else (300 if k == CROWD else int(rs.randint(1, 9)))
    segs = [synth_polygon(rs, 6 if k == CROWD else 16) for _ in range(n)]
    if k == 0 and n >= 2:
        segs[1] = segs[0].copy()  # two equal areas: the overlap order's tie rule
    boxes = []
    for s in segs:
        x, y = np.clip(s, 0, 1).T
        boxes.append([(x.min() + x.max()) / 2, (y.min() + y.max()) / 2, x.max() - x.min(), y.max() - y.min()])
    lab = np.concatenate((rs.randint(0, 80, (n, 1)), np.array(boxes).reshape(-1, 4)), 1).astype(np.float32)
    return lab, segs


def rect_batches(shapes_wh, batch_size, img_size, stride, pad):
    """LoadImagesAndLabels.__init__'s aspect-ratio sort and batch shapes (utils/dataloaders.py:565-612)."""
    n = len(shapes_wh)
    bi = np.floor(np.arange(n) / batch_size).astype(int)
    nb = bi[-1] + 1
    s = np.asarray(shapes_wh)
    ar = s[:, 1] / s[:, 0]
    irect = ar.argsort()
    ar = ar[irect]
    shapes = [[1, 1]] * nb
    for i in range(nb):
        ari = ar[bi == i]
        mini, maxi = ari.min(), ari.max()
        if maxi < 1:
            shapes[i] = [maxi, 1]
        elif mini > 1:
            shapes[i] = [1, 1 / mini]
    return irect, bi, np.ceil(np.array(shapes) * img_size / stride + pad).astype(int) * stride


def make_dataset(cls, files, labels, segments, opts, seg=None):
    n = len(files)
    ds = cls.__new__(cls)
    ds.img_size, ds.augment, ds.hyp, ds.image_weights, ds.rect = IMG_SIZE, False, None, False, opts["rect"]
    ds.mosaic, ds.mosaic_border, ds.stride = False, [-IMG_SIZE // 2, -IMG_SIZE // 2], 32
    shapes_wh = [cv2.imread(f).shape[1::-1] for f in files]
    order = list(range(n))
    ds.batch = np.floor(np.arange(n) / opts["batch"]).astype(int)
    if opts["rect"]:
        irect, ds.batch, ds.batch_shapes = rect_batches(shapes_wh, opts["batch"], IMG_SIZE, 32, opts["pad"])
        order = [int(i) for i in irect]
    ds.im_files = [files[i] for i in order]
    ds.label_files = [f.replace(".png", ".txt") for f in ds.im_files]
    ds.labels = [labels[i] for i in order]
    ds.segments = [segments[i] for i in order]
    ds.shapes = np.array([shapes_wh[i] for i in order])
    ds.n = n
    ds.indices = np.arange(n)
    ds.ims = [None] * n
    ds.npy_files = [Path(f).with_suffix(".npy") for f in ds.im_files]
    if seg is not None:
        ds.overlap, ds.downsample_ratio = seg
    return ds, order


def oracle_batch(store, ds, order, idx, seg=None):
    items = []
    for i in idx:
        k = order[i]
        im = V.load_resize(store[f"src{k}"], IMG_SIZE)
        shape = ds.batch_shapes[ds.batch[i]] if ds.rect else IMG_SIZE  # as __getitem__ passes it to letterbox
        hw0 = store[f"src{k}"].shape[:2]
        if seg is None:
            items.append(V.get_item(im, hw0, ds.labels[i], shape))
        else:
            items.append(V.get_item(im, hw0, ds.labels[i], shape, ds.segments[i], seg[0], seg[1]))
    return V.get_batch(items)


def gen():
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

    refshim._REAL["ultralytics.utils.ops"].update(xyxy2xywhn=xyxy2xywhn, xywhn2xyxy=xywhn2xyxy)
    seg_refshim.register(refshim)
    refshim.install()
    from utils.dataloaders import LoadImagesAndLabels
    from utils.segment.dataloaders import LoadImagesAndLabelsAndMasks

    rs = np.random.RandomState(8)
    store, meta = {}, {"order_differs": [], "runs": {}, "img_size": IMG_SIZE}
    with tempfile.TemporaryDirectory() as tmp:
        files, labels, segments = [], [], []
        for k, (h, w) in enumerate(SHAPES):
            f = os.path.join(tmp, f"im{k}.png")
            cv2.imwrite(f, synth_image(h, w, 500 + k))
            files.append(f)
            store[f"src{k}"] = cv2.imread(f)
            lab, segs = synth_labels(rs, k)
            labels.append(lab)
            segments.append(segs)
            store[f"labels{k}"] = lab
            if segs:
                store[f"segs{k}"] = np.concatenate(segs, 0)
                store[f"seglen{k}"] = np.array([len(s) for s in segs])
        runs = [(name, opts, None) for name, opts in RUNS.items()]
        runs += [(f"seg.o{int(o)}.r{r}", RUNS["det.rect"], (o, r)) for o in (True, False) for r in (1, 4)]
        for name, opts, seg in runs:
            cls = LoadImagesAndLabels if seg is None else LoadImagesAndLabelsAndMasks
            ds, order = make_dataset(cls, files, labels, segments, opts, seg)
            for i, k in enumerate(order):
                im, hw0, hw = ds.load_image(i)
                assert np.array_equal(im, V.load_resize(store[f"src{k}"], IMG_SIZE)), (name, k, "load_image")
            seg_refshim.OVERLAP_ORDERS.clear()
            loader = torch.utils.data.DataLoader(ds, batch_size=opts["batch"], shuffle=False, num_workers=0, collate_fn=cls.collate_fn)
            batches = list(loader)
            orders = list(seg_refshim.OVERLAP_ORDERS)
            meta["runs"][name] = dict(rect=opts["rect"], pad=opts["pad"], batch=opts["batch"], order=order, batches=len(batches),
                                      overlap=None if seg is None else seg[0], ratio=None if seg is None else seg[1])
            if opts["rect"]:
                store[f"{name}.batch_shapes"] = ds.batch_shapes
            for bi, batch in enumerate(batches):
                idx = list(range(bi * opts["batch"], min((bi + 1) * opts["batch"], ds.n)))
                imgs, targets, paths, shapes = (x.numpy() if torch.is_tensor(x) else x for x in batch[:4])
                assert list(paths) == [ds.im_files[i] for i in idx]
                if seg is None:
                    oi, ot, osh = oracle_batch(store, ds, order, idx)
                else:
                    masks = batch[4].numpy()
                    host_orders = [orders.pop(0) for i in idx if len(ds.labels[i])] if seg[0] else []
                    replay = list(host_orders)
                    old = seg_aug_ref.overlap_order
                    seg_aug_ref.overlap_order = lambda areas: replay.pop(0)
                    try:
                        oi, ot, osh, om = oracle_batch(store, ds, order, idx, seg)
                    finally:
                        seg_aug_ref.overlap_order = old
                    assert om.dtype == masks.dtype and om.shape == masks.shape and np.array_equal(om, masks), (name, bi, "masks")
                    assert ot.shape == targets.shape and np.array_equal(ot.view(np.uint32), targets.view(np.uint32)), (name, bi, "targets")
                    ei, et, esh, em = oracle_batch(store, ds, order, idx, seg)  # the engine's rule for equal areas
                    if not (np.array_equal(et, ot) and np.array_equal(em, om)):
                        meta["order_differs"].append([name, bi])
                    ot, om = et, em
                    store[f"{name}.masks{bi}"] = om
                assert np.array_equal(oi, imgs), (name, bi, "images")
                assert ot.shape == targets.shape, (name, bi, ot.shape, targets.shape)
                if seg is None:
                    assert np.array_equal(ot.view(np.uint32), targets.view(np.uint32)), (name, bi, "targets")
                assert osh == tuple(shapes), (name, bi, osh, shapes)
                key = "det.rect" if seg is not None else name
                if f"{key}.imgs{bi}" in store:
                    assert np.array_equal(store[f"{key}.imgs{bi}"], imgs)
                store[f"{key}.imgs{bi}"] = imgs
                store[f"{name}.targets{bi}"] = ot
                store[f"{name}.shapes{bi}"] = np.array(json.dumps(osh))
            print(f"{name}: oracle == reference over {len(batches)} batches")
    store["meta"] = np.array(json.dumps(meta))
    np.savez_compressed(f"{HERE}/val_load.npz", **store)
    print("order differs:", meta["order_differs"])
    print("written", f"{HERE}/val_load.npz", os.path.getsize(f"{HERE}/val_load.npz"), "bytes")


if __name__ == "__main__":
    gen()
