"""Time the device augmentation of one training batch against the reference's per-image CPU arithmetic.

    python tools/aug_bench.py [--iters 30] [--out results.json]

Workload: an in-RAM synthetic dataset of 64 images with COCO-like shapes (the long side already resized to s = 640, as
load_image returns it) and Poisson(7.3) labels per image; batches of 16 and 64 under hyp.scratch-low and
hyp.scratch-high (mixup 0.1, scale 0.9).  The engine's time runs from the host load_image outputs to device imgs +
targets: the host part (random draws, load_image, table and label packing), then the rest (copy into the pinned staging
buffer, H2D copy, letterbox for non-mosaic items, gather and label kernels, label-count read), each timed with a device
synchronise at its end.  The result is printed as one JSON document (also written to --out when given).  The CPU comparison runs oracle/aug_ref.py's per-image path through cv2 (warpAffine, cvtColor,
LUT) single-threaded when cv2 is importable; without cv2 it reports that the comparison was not run.
"""
from __future__ import annotations

import argparse
import contextlib
import json
import os
import random
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from yolov5_b200.utils import dataloaders as D  # noqa: E402
from yolov5_b200.utils.dataloaders import DeviceAugmentLoader  # noqa: E402

S = 640
SHAPES = [(480, 640), (640, 480), (427, 640), (640, 427), (360, 640), (640, 640), (512, 640), (640, 512)]
HYP_LOW = dict(lr0=0.01, hsv_h=0.015, hsv_s=0.7, hsv_v=0.4, degrees=0.0, translate=0.1, scale=0.5, shear=0.0, perspective=0.0,
               flipud=0.0, fliplr=0.5, mosaic=1.0, mixup=0.0, copy_paste=0.0)
HYPS = {"scratch-low": HYP_LOW, "scratch-high": dict(HYP_LOW, scale=0.9, mixup=0.1, copy_paste=0.1)}


class RamDataset:
    def __init__(self, n, hyp, seed=0):
        rs = np.random.RandomState(seed)
        self.ims = [rs.randint(0, 256, SHAPES[k % len(SHAPES)] + (3,), dtype=np.uint8) for k in range(n)]
        self.labels = []
        for _ in range(n):
            m = rs.poisson(7.3)
            self.labels.append(np.concatenate((rs.randint(0, 80, (m, 1)), rs.uniform(0.1, 0.9, (m, 2)), rs.uniform(0.02, 0.5, (m, 2))), 1).astype(np.float32))
        self.segments = [[] for _ in range(n)]
        self.img_size, self.augment, self.rect, self.mosaic = S, True, False, True
        self.mosaic_border = [-S // 2, -S // 2]
        self.hyp = hyp
        self.indices = np.arange(n)
        self.im_files = [f"im{k}.jpg" for k in range(n)]
        self.albumentations = None

    def __len__(self):
        return len(self.ims)

    def load_image(self, i):
        return self.ims[i], self.ims[i].shape[:2], self.ims[i].shape[:2]


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


@contextlib.contextmanager
def split_at_staging():
    """Split host packing from the device work at the staging hand-off: while active, each stage_upload call first
    synchronises the device and records the time in `.t` of the yielded wrapper."""
    real = D.stage_upload

    def staged(*a):
        torch.cuda.synchronize()
        staged.t = time.perf_counter()
        return real(*a)

    D.stage_upload = staged
    try:
        yield staged
    finally:
        D.stage_upload = real


def time_engine(ds, batch, iters, dev):
    loader = DeviceAugmentLoader(ds, batch, device=dev)
    idx = list(range(batch))
    for _ in range(3):
        loader.collate(idx)
    torch.cuda.synchronize()
    total, dev_part, host_part = [], [], []
    with split_at_staging() as staged:
        for _ in range(iters):
            t0 = time.perf_counter()
            imgs, targets, _, _ = loader.collate(idx)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            total.append(t1 - t0)
            host_part.append(staged.t - t0)
            dev_part.append(t1 - staged.t)
    med = lambda v: float(np.median(v)) * 1e3  # noqa: E731
    return dict(batch_ms=med(total), host_draw_pack_ms=med(host_part), staging_h2d_kernels_count_ms=med(dev_part),
                img_per_s=batch / (med(total) / 1e3), nt=int(targets.shape[0]))


def time_cpu_reference(ds, n_img):
    try:
        import cv2
    except ImportError:
        return "not run: cv2 is not importable"
    cv2.setNumThreads(1)
    from oracle import aug_ref

    t0 = time.perf_counter()
    for i in range(n_img):
        p = aug_ref.sample_params(ds, i)
        md = p["m"][0]
        img4 = np.full((2 * S, 2 * S, 3), 114, np.uint8)
        ims = [ds.load_image(k) for k in md["indices"]]
        for (im, _, (h, w)), (x1a, y1a, x2a, y2a, x1b, y1b) in zip(ims, aug_ref.placements(md["xc"], md["yc"], S, [x[2] for x in ims])):
            img4[y1a:y2a, x1a:x2a] = im[y1b:y1b + (y2a - y1a), x1b:x1b + (x2a - x1a)]
        M = aug_ref.affine(md["persp"], img4.shape[:2], ds.mosaic_border)
        img = cv2.warpAffine(img4, M[:2], dsize=(S, S), borderValue=(114, 114, 114))
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
        raise SystemExit("aug_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    res = dict(gpu=gpu_info(), iters=a.iters, img_size=S, results={})
    for name, hyp in HYPS.items():
        ds = RamDataset(64, hyp)
        for b in (16, 64):
            random.seed(0)
            np.random.seed(0)
            res["results"][f"{name} B={b}"] = time_engine(ds, b, a.iters, dev)
        random.seed(0)
        np.random.seed(0)
        res["results"][f"{name} cpu reference"] = time_cpu_reference(ds, 32)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
