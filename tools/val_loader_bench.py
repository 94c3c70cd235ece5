"""Validation dataloader throughput: DeviceValLoader (host decode threads + y5_val_letterbox) against the reference's
host pipeline (per item: cv2.imread, load_image's cv2.resize INTER_AREA / INTER_LINEAR, letterbox's copyMakeBorder,
HWC->CHW BGR->RGB; collate_fn; torch DataLoader with `--ref-workers` persistent worker processes, then the upload), on
the same host.  Both loaders are timed on their second pass over the data.

    python tools/val_loader_bench.py [--n 256] [--batch 32] [--workers 8] [--ref-workers 8]

Data: JPEGs written to a temporary directory -- COCO-val-like sizes (longest side 640, the other 240..640) and a
1920 x 1080 set -- at img_size 640 and 1280, rect batches with pad 0.5.  Prints one JSON line per (set, img_size) with
images/s of both loaders (each batch on the device, synchronised at the end), the new loader's host time per batch
(what the consumer waits for between batches), its device time per batch (the upload and y5_val_letterbox, timed
alone with CUDA events), and the GPU model and power limit.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
        return out.strip().splitlines()[0]
    except (OSError, IndexError):
        return torch.cuda.get_device_name(0)


class Dataset:
    """The attributes the val loaders read, for a directory of JPEGs (rect batches as LoadImagesAndLabels builds them)."""

    def __init__(self, files, shapes_wh, img_size, batch_size, pad=0.5, stride=32):
        import cv2  # noqa: F401  (the decode step needs it)

        s = np.asarray(shapes_wh, np.float64)
        ar = s[:, 1] / s[:, 0]
        irect = ar.argsort()
        self.im_files = [files[i] for i in irect]
        ar = ar[irect]
        n = len(files)
        self.batch = np.floor(np.arange(n) / batch_size).astype(int)
        nb = self.batch[-1] + 1
        shapes = [[1, 1]] * nb
        for i in range(nb):
            ari = ar[self.batch == i]
            if ari.max() < 1:
                shapes[i] = [ari.max(), 1]
            elif ari.min() > 1:
                shapes[i] = [1, 1 / ari.min()]
        self.batch_shapes = np.ceil(np.array(shapes) * img_size / stride + pad).astype(int) * stride
        self.img_size, self.augment, self.image_weights, self.rect = img_size, False, False, True
        self.indices = np.arange(n)
        self.labels = [np.zeros((0, 5), np.float32)] * n
        self.ims = [None] * n
        self.npy_files = None

    def __len__(self):
        return len(self.im_files)

    def __getitem__(self, i):  # the reference's host work for one item
        import cv2

        im = cv2.imread(self.im_files[i])
        h0, w0 = im.shape[:2]
        r = self.img_size / max(h0, w0)
        if r != 1:
            im = cv2.resize(im, (math.ceil(w0 * r), math.ceil(h0 * r)), interpolation=cv2.INTER_LINEAR if r > 1 else cv2.INTER_AREA)
        H, W = (int(v) for v in self.batch_shapes[self.batch[i]])
        h, w = im.shape[:2]
        r = min(H / h, W / w, 1.0)
        new = round(w * r), round(h * r)
        if new != (w, h):
            im = cv2.resize(im, new, interpolation=cv2.INTER_LINEAR)
        dw, dh = (W - new[0]) / 2, (H - new[1]) / 2
        top, bottom, left, right = round(dh - 0.1), round(dh + 0.1), round(dw - 0.1), round(dw + 0.1)
        im = cv2.copyMakeBorder(im, top, bottom, left, right, cv2.BORDER_CONSTANT, value=(114, 114, 114))
        return torch.from_numpy(np.ascontiguousarray(im.transpose((2, 0, 1))[::-1])), torch.zeros(0, 6), self.im_files[i], None

    @staticmethod
    def collate_fn(batch):
        im, label, path, shapes = zip(*batch)
        return torch.stack(im, 0), torch.cat(label, 0), path, shapes


def make_set(tmp, name, n, rs):
    import cv2

    files, shapes = [], []
    for k in range(n):
        if name == "coco":
            long, short = 640, int(rs.randint(240, 641))
            h, w = (long, short) if rs.rand() < 0.3 else (short, long)
        else:
            h, w = 1080, 1920
        yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
        im = np.stack([127 + 120 * np.sin(xx / (9 + c) + yy / (13 - c) + k) for c in range(3)], -1)
        im = np.clip(im + rs.uniform(-20, 20, (h, w, 3)), 0, 255).astype(np.uint8)
        f = os.path.join(tmp, f"{name}{k}.jpg")
        cv2.imwrite(f, im, [cv2.IMWRITE_JPEG_QUALITY, 90])
        files.append(f)
        shapes.append((w, h))
    return files, shapes


def run_new(ds, batch, workers, dev):
    from yolov5_b200.utils.dataloaders import DeviceValLoader

    loader = DeviceValLoader(ds, batch, device=dev, workers=workers)
    host = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    it = iter(loader)
    while True:
        t = time.perf_counter()
        try:
            imgs = next(it)[0]
        except StopIteration:
            break
        host.append(time.perf_counter() - t)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    # device time of one batch: the upload, then y5_val_letterbox, each timed alone with CUDA events
    from yolov5_b200.utils.dataloaders import ValBatchLayout, _Staging, load_val_image

    pos = list(range(min(batch, len(ds))))
    lay = ValBatchLayout(ds, pos, [load_val_image(ds, p) for p in pos])
    staging = _Staging(2)
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    up, kern = [], []
    for _ in range(10):
        e[0].record()
        buf = lay.upload(staging, dev)
        e[1].record()
        lay.letterbox(buf, torch.uint8, dev)
        e[2].record()
        torch.cuda.synchronize()
        up.append(e[0].elapsed_time(e[1]))
        kern.append(e[1].elapsed_time(e[2]))
    return len(ds) / wall, 1e3 * float(np.median(host)), float(np.median(up)), float(np.median(kern)), imgs


def run_ref(ds, batch, workers, dev):
    loader = torch.utils.data.DataLoader(ds, batch_size=batch, shuffle=False, num_workers=workers, pin_memory=True, collate_fn=Dataset.collate_fn,
                                         persistent_workers=workers > 0)
    for _ in loader:  # warm-up epoch: worker processes started, as in a training run's second validation
        pass
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for imgs, *_ in loader:
        imgs = imgs.to(dev, non_blocking=True)
    torch.cuda.synchronize()
    return len(ds) / (time.perf_counter() - t0), imgs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=256)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--ref-workers", type=int, default=8)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    rs = np.random.RandomState(0)
    info = gpu_info()
    with tempfile.TemporaryDirectory() as tmp:
        for name in ("coco", "1080p"):
            files, shapes = make_set(tmp, name, a.n, rs)
            for s in (640, 1280):
                ds = Dataset(files, shapes, s, a.batch)
                run_new(ds, a.batch, a.workers, dev)  # warm-up: thread pool, pinned buffers, allocator
                ips, host_ms, up_ms, kern_ms, got = run_new(ds, a.batch, a.workers, dev)
                ref_ips, want = run_ref(ds, a.batch, a.ref_workers, dev)
                same = bool(torch.equal(got, want))  # the last batch of both loaders
                print(json.dumps(dict(set=name, img_size=s, images=len(ds), batch=a.batch, new_img_s=round(ips, 1), new_host_ms_per_batch=round(host_ms, 2),
                                      new_upload_ms_per_batch=round(up_ms, 3), new_kernel_ms_per_batch=round(kern_ms, 3), ref_img_s=round(ref_ips, 1), workers=a.workers,
                                      ref_workers=a.ref_workers, last_batch_equal=same, cpus=os.cpu_count(), gpu=info)), flush=True)


if __name__ == "__main__":
    main()
