"""Time the device segmentation augmentation of one training batch against the reference's per-image CPU cost.

    python tools/seg_aug_bench.py [--iters 30] [--out results.json]

Workload (yolov5s-seg training shapes): an in-RAM synthetic dataset of 64 images with COCO-like shapes (long side 640,
as load_image returns it) and Poisson(7.3) polygons per image (12-point star-like outlines); batch 16 at 640,
mask_ratio 4, overlap masks, hyp.scratch-low.  The engine's time runs from the host load_image outputs to device imgs +
targets + masks: the host part (random draws, load_image, table / label / polygon packing), then the rest (staging copy,
H2D, kernels, the label-count read, the mask composition), each ended by a device synchronise.  The CPU comparison runs
the reference's per-image arithmetic single-threaded through cv2 and numpy (mosaic, warpAffine, HSV, the segment path,
polygons2masks_overlap with cv2.fillPoly + cv2.resize) when cv2 is importable.  One JSON document is printed (and
written to --out), with the GPU's name and power limit from the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import random
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.aug_bench import HYP_LOW, SHAPES, gpu_info, split_at_staging  # noqa: E402
from yolov5_b200.utils.segment.dataloaders import DeviceSegAugmentLoader  # noqa: E402

S = 640
RATIO = 4


class RamSegDataset:
    def __init__(self, n, hyp, seed=0):
        rs = np.random.RandomState(seed)
        self.ims = [rs.randint(0, 256, SHAPES[k % len(SHAPES)] + (3,), dtype=np.uint8) for k in range(n)]
        self.labels, self.segments = [], []
        for _ in range(n):
            m = rs.poisson(7.3)
            segs = []
            for _ in range(m):
                c, r = rs.uniform(0.1, 0.9, 2), rs.uniform(0.02, 0.25)
                t = np.sort(rs.uniform(0, 2 * np.pi, 12))
                segs.append(np.clip(c + np.stack([np.cos(t), np.sin(t)], 1) * (r * rs.uniform(0.4, 1, 12))[:, None], 0, 1).astype(np.float32))
            boxes = [[(s[:, 0].min() + s[:, 0].max()) / 2, (s[:, 1].min() + s[:, 1].max()) / 2, np.ptp(s[:, 0]), np.ptp(s[:, 1])] for s in segs]
            self.labels.append(np.concatenate((rs.randint(0, 80, (m, 1)), np.array(boxes).reshape(-1, 4)), 1).astype(np.float32))
            self.segments.append(segs)
        self.img_size, self.augment, self.rect, self.mosaic = S, True, False, True
        self.mosaic_border = [-S // 2, -S // 2]
        self.hyp = hyp
        self.indices = np.arange(n)
        self.n = n
        self.im_files = [f"im{k}.jpg" for k in range(n)]
        self.albumentations = None
        self.overlap, self.downsample_ratio = True, RATIO

    def __len__(self):
        return len(self.ims)

    def load_image(self, i):
        return self.ims[i], self.ims[i].shape[:2], self.ims[i].shape[:2]


def time_engine(ds, batch, iters, dev):
    loader = DeviceSegAugmentLoader(ds, batch, device=dev)
    idx = list(range(batch))
    for _ in range(3):
        loader.collate(idx)
    torch.cuda.synchronize()
    total, dev_part, host_part = [], [], []
    with split_at_staging() as staged:
        for _ in range(iters):
            t0 = time.perf_counter()
            imgs, targets, _, _, masks = loader.collate(idx)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            total.append(t1 - t0)
            host_part.append(staged.t - t0)
            dev_part.append(t1 - staged.t)
    med = lambda v: float(np.median(v)) * 1e3  # noqa: E731
    return dict(batch_ms=med(total), host_draw_pack_ms=med(host_part), staging_h2d_kernels_masks_ms=med(dev_part),
                img_per_s=batch / (med(total) / 1e3), nt=int(targets.shape[0]), masks=list(masks.shape), masks_dtype=str(masks.dtype))


def time_cpu_reference(ds, n_img):
    """The reference's per-image work on one core: mosaic + warpAffine + HSV + flips, and the segment / mask path."""
    try:
        import cv2
    except ImportError:
        return "not run: cv2 is not importable"
    cv2.setNumThreads(1)
    from oracle import aug_ref, seg_aug_ref

    t0 = time.perf_counter()
    for i in range(n_img):
        p = seg_aug_ref.sample_params(ds, i)
        md = p["m"][0]
        img4 = np.full((2 * S, 2 * S, 3), 114, np.uint8)
        ims = [ds.load_image(k) for k in md["indices"]]
        labels4, segs4 = [], []
        for (im, _, (h, w)), (x1a, y1a, x2a, y2a, x1b, y1b), k in zip(ims, aug_ref.placements(md["xc"], md["yc"], S, [x[2] for x in ims]), md["indices"]):
            img4[y1a:y2a, x1a:x2a] = im[y1b:y1b + (y2a - y1a), x1b:x1b + (x2a - x1a)]
            lab = ds.labels[k].copy()
            if lab.size:
                lab[:, 1:] = aug_ref.xywhn2xyxy(lab[:, 1:], w, h, x1a - x1b, y1a - y1b)
                segs4 += [seg_aug_ref.xyn2xy(x, w, h, x1a - x1b, y1a - y1b) for x in ds.segments[k]]
            labels4.append(lab)
        labels4 = np.concatenate(labels4, 0)
        for x in (labels4[:, 1:], *segs4):
            np.clip(x, 0, 2 * S, out=x)
        M = aug_ref.affine(md["persp"], img4.shape[:2], ds.mosaic_border)
        img = cv2.warpAffine(img4, M[:2], dsize=(S, S), borderValue=(114, 114, 114))
        polys, new = [], np.zeros((len(segs4), 4))
        for j, s in enumerate(segs4):  # resample_segments, xy @ M.T, segment2box
            s = np.concatenate((s, s[0:1]), 0)
            x = np.linspace(0, len(s) - 1, 1000)
            xy = np.ones((1000, 3))
            xy[:, :2] = np.concatenate([np.interp(x, np.arange(len(s)), s[:, c]) for c in range(2)]).reshape(2, -1).T
            xy = (xy @ M.T)[:, :2]
            new[j] = seg_aug_ref.segment2box(xy, S, S)
            polys.append(xy)
        keep = aug_ref.box_candidates(labels4[:, 1:5].T * md["persp"][3], new.T, area_thr=0.01) if len(segs4) else []
        ms = []
        for xy, k in zip(polys, keep):
            if k:
                mk = cv2.fillPoly(np.zeros((S, S), np.uint8), [np.asarray(xy, np.int32).reshape(-1, 1, 2)], 1)
                ms.append(cv2.resize(mk, (S // RATIO, S // RATIO)))
        if ms:
            order = np.argsort(-np.asarray([m.sum() for m in ms]))
            v = np.zeros((S // RATIO, S // RATIO), np.uint8)
            for q, j in enumerate(order):
                v = np.clip(v + ms[j] * (q + 1), 0, q + 1)
        if p["hsv"] is not None:
            lut = aug_ref.hsv_luts(p["hsv"])
            hh, ss, vv = cv2.split(cv2.cvtColor(img, cv2.COLOR_BGR2HSV))
            img = cv2.cvtColor(cv2.merge((cv2.LUT(hh, lut[0]), cv2.LUT(ss, lut[1]), cv2.LUT(vv, lut[2]))), cv2.COLOR_HSV2BGR)
        if p["fliplr"]:
            img = np.fliplr(img)
        np.ascontiguousarray(img.transpose(2, 0, 1)[::-1])
    dt = time.perf_counter() - t0
    return dict(img_per_s_per_core=n_img / dt, ms_per_img=dt / n_img * 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    ap.add_argument("--iters", type=int, default=30)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("seg_aug_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    res = dict(gpu=gpu_info(), iters=a.iters, img_size=S, mask_ratio=RATIO, overlap=True, results={})
    ds = RamSegDataset(64, HYP_LOW)
    random.seed(0)
    np.random.seed(0)
    res["results"]["scratch-low B=16"] = time_engine(ds, 16, a.iters, dev)
    random.seed(0)
    np.random.seed(0)
    res["results"]["cpu reference"] = time_cpu_reference(ds, 32)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
