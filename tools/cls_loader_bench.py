"""Classification dataloader throughput: DeviceClassifyLoader (host decode threads + y5_cls_batch) against the reference's
host pipeline, on the same host, at imgsz 224.  The baseline does each item's work with the libraries the reference calls
(cv2.imread, CenterCrop's cv2.resize of the center square, ToTensor's CPU `/= 255`, torchvision's Normalize) in a torch
DataLoader with `--ref-workers` persistent worker processes and pin_memory, then `.to(device)`, with OpenCV
single-threaded as the reference sets it.  Both loaders are timed on their second pass.  It also prints the per-item host
cost of decode and transform on one thread, so the baseline's split is visible.

    python tools/cls_loader_bench.py [--n 1024] [--workers 8] [--ref-workers 8]

Data: N seeded ImageNet-like JPEGs written to a temporary directory in ImageFolder layout (10 classes; sides 300..600,
aspect ratios 0.6..1.7, about 500 x 375 on average).  For batch 64 (classify/train.py) and 128 (classify/val.py) it prints
one JSON line per arm with images/s (the pass, every batch on the device, synchronised at the end), host time per batch
(what the consumer waits for in next()), the staging + host-to-device copy per batch and, for the new loader, the
y5_cls_batch kernel per batch (CUDA events).  At batch 64 it also times yolov5s-cls's engine training step fed by each
loader (the batches/s a training pass reaches), and checks that the two arms' last batches are equal.  The GPU model and
power limit are printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import cls_load_ref as R  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
        return out.strip().splitlines()[0]
    except (OSError, IndexError):
        return torch.cuda.get_device_name(0)


class Dataset:
    """The attributes DeviceClassifyLoader reads, over an ImageFolder tree, and the reference's __getitem__ (no cache)."""

    def __init__(self, root, size):
        from pathlib import Path

        self.root = Path(root)
        self.classes = sorted(os.listdir(root))
        self.samples = [[str(self.root / c / f), j, (self.root / c / f).with_suffix(".npy"), None]
                        for j, c in enumerate(self.classes) for f in sorted(os.listdir(self.root / c))]
        self.torch_transforms = R.classify_transforms(size)  # what DeviceClassifyLoader checks; __getitem__ does not call it
        self.size = size
        self.normalize = self.torch_transforms.transforms[2]  # torchvision's Normalize(IMAGENET_MEAN, IMAGENET_STD)
        self.album_transforms = None
        self.cache_ram = self.cache_disk = False

    def __len__(self):
        return len(self.samples)

    def __getitem__(self, i):
        """The reference's per-item work: cv2.imread, CenterCrop (cv2.resize INTER_LINEAR of the center square), ToTensor
        (BGR -> RGB, CHW, float32 /= 255 on the CPU tensor) and torchvision's Normalize -- the same libraries the reference
        calls, not the oracle's numpy restatement (whose resize is far slower than cv2's)."""
        import cv2

        f, j = self.samples[i][:2]
        im = cv2.imread(f)
        h, w = im.shape[:2]
        m = min(h, w)
        top, left = (h - m) // 2, (w - m) // 2
        im = cv2.resize(im[top: top + m, left: left + m], (self.size, self.size), interpolation=cv2.INTER_LINEAR)
        x = torch.from_numpy(np.ascontiguousarray(im.transpose((2, 0, 1))[::-1])).float()
        x /= 255.0
        return self.normalize(x), j


def make_set(root, n, rs):
    import cv2

    for k in range(n):
        area = rs.uniform(300 * 300, 600 * 450)
        ar = rs.uniform(0.6, 1.7)
        h, w = int(min(600, max(300, (area / ar) ** 0.5))), int(min(600, max(300, (area * ar) ** 0.5)))
        yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
        im = np.stack([127 + 120 * np.sin(xx / (9 + c) + yy / (13 - c) + k) for c in range(3)], -1)
        im = np.clip(im + rs.uniform(-25, 25, (h, w, 3)), 0, 255).astype(np.uint8)
        d = os.path.join(root, f"class{k % 10}")
        os.makedirs(d, exist_ok=True)
        cv2.imwrite(os.path.join(d, f"im{k}.jpg"), im, [cv2.IMWRITE_JPEG_QUALITY, 90])


def timed_pass(batches, step=None):
    """Drain one pass -> (images/s, median host ms per batch, last batch)."""
    host, n, last = [], 0, None
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    it = iter(batches)
    while True:
        t = time.perf_counter()
        try:
            x, y = next(it)
        except StopIteration:
            break
        host.append(time.perf_counter() - t)
        if step is not None:
            step(x, y)
        n += len(y)
        last = (x, y)
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t0), 1e3 * float(np.median(host)), last


def device_times(loader, items):
    """Median ms of (staging + H2D copy, y5_cls_batch) for one batch, timed alone with CUDA events."""
    from yolov5_b200.utils import dataloaders as D

    loaded = [loader.decode(loader.dataset, i) for i in items]
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    up, kern = [], []
    real = D.stage_upload

    def marked(*a):
        e[0].record()
        real(*a)
        e[1].record()

    D.stage_upload = marked
    try:
        for _ in range(10):
            loader.collate(items, loaded)
            e[2].record()
            torch.cuda.synchronize()
            up.append(e[0].elapsed_time(e[1]))
            kern.append(e[1].elapsed_time(e[2]))
    finally:
        D.stage_upload = real
    return float(np.median(up)), float(np.median(kern))


def ref_h2d_ms(x_host, dev):
    e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ts = []
    for _ in range(10):
        e[0].record()
        x_host.to(dev, non_blocking=True)
        e[1].record()
        torch.cuda.synchronize()
        ts.append(e[0].elapsed_time(e[1]))
    return float(np.median(ts))


def train_step_fn(dev):
    from oracle import cls_ref
    from yolov5_b200.cfg import model_cfg
    from yolov5_b200.models.yolo import ClassificationModel, DetectionModel
    from yolov5_b200.utils.torch_utils import ModelEMA, smart_optimizer, smartCrossEntropyLoss

    m = ClassificationModel(model=DetectionModel("yolov5s"), nc=10)
    m.load_state_dict(cls_ref.synth_state_dict(model_cfg("yolov5s"), 10, seed=0))
    m = m.to(dev).train()
    opt = smart_optimizer(m, "Adam", 1e-3, 0.9, 5e-5)
    ema = ModelEMA(m)
    scaler = torch.amp.GradScaler("cuda")
    crit = smartCrossEntropyLoss(label_smoothing=0.1)

    def step(x, y):  # classify/train.py:219-233
        x, y = x.to(dev, non_blocking=True), y.to(dev)
        with torch.autocast("cuda"):
            loss = crit(m(x), y)
        scaler.scale(loss).backward()
        opt.fused_step(scaler, 10.0, ema, m)
        opt.zero_grad(set_to_none=True)

    return step


def item_costs(ds, k=64):
    """Median ms per item on one thread: cv2.imread, then the reference's transform (__getitem__ minus the decode)."""
    import cv2

    dec, tr = [], []
    for i in range(min(k, len(ds))):
        t0 = time.perf_counter()
        cv2.imread(ds.samples[i][0])
        t1 = time.perf_counter()
        ds[i]
        tr.append(time.perf_counter() - t1 - (t1 - t0))
        dec.append(t1 - t0)
    return 1e3 * float(np.median(dec)), 1e3 * float(np.median(tr))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1024)
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--ref-workers", type=int, default=8)
    a = ap.parse_args()
    import cv2

    from yolov5_b200.utils.dataloaders import DeviceClassifyLoader

    cv2.setNumThreads(0)  # as the reference's utils/general.py sets it on import: no OpenCV threads inside DataLoader workers
    dev = torch.device("cuda:0")
    info = gpu_info()
    with tempfile.TemporaryDirectory() as tmp:
        make_set(tmp, a.n, np.random.RandomState(0))
        ds = Dataset(tmp, 224)
        sides = np.array([cv2.imread(s[0]).shape[:2] for s in ds.samples])
        for i in range(8):  # the baseline's items are the reference's transform (pinned by the oracle)
            want = torch.from_numpy(R.transform(cv2.imread(ds.samples[i][0]), 224))
            assert torch.equal(ds[i][0].view(torch.int32), want.view(torch.int32)), i
        decode_ms, transform_ms = item_costs(ds)
        print(json.dumps(dict(per_item_one_thread_ms=dict(imread=round(decode_ms, 3), reference_transform=round(transform_ms, 3)), mean_hw=[round(float(v)) for v in sides.mean(0)],
                              cpus=os.cpu_count(), gpu=info)), flush=True)
        step = train_step_fn(dev)
        x0 = torch.zeros(64, 3, 224, 224, device=dev)
        y0 = torch.zeros(64, dtype=torch.int64, device=dev)
        for _ in range(3):
            step(x0, y0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(20):
            step(x0, y0)
        torch.cuda.synchronize()
        step_ms = (time.perf_counter() - t0) / 20 * 1e3
        for batch in (64, 128):
            new = DeviceClassifyLoader(ds, batch, shuffle=False, device=dev, workers=a.workers)
            ref = torch.utils.data.DataLoader(ds, batch_size=batch, shuffle=False, num_workers=a.ref_workers, pin_memory=True,
                                              persistent_workers=a.ref_workers > 0)
            res = {}
            for name, loader in (("device", new), ("reference", ref)):
                def on_device(it):
                    for x, y in it:
                        yield x.to(dev, non_blocking=True), y.to(dev)

                src = loader if name == "device" else on_device(loader)
                timed_pass(src)  # first pass: threads / worker processes started, pinned buffers, allocator
                src = loader if name == "device" else on_device(loader)
                ips, host_ms, last = timed_pass(src)
                r = dict(img_s=round(ips, 1), host_ms_per_batch=round(host_ms, 2))
                if name == "device":
                    up, kern = device_times(new, list(range(batch)))
                    r.update(stage_h2d_ms_per_batch=round(up, 3), kernel_ms_per_batch=round(kern, 3))
                else:
                    xh = next(iter(loader))[0]
                    r.update(h2d_ms_per_batch=round(ref_h2d_ms(xh, dev), 3))
                if batch == 64:
                    src = loader if name == "device" else on_device(loader)
                    tips, _, _ = timed_pass(src, step)
                    r.update(train_img_s=round(tips, 1))
                res[name] = (r, last)
            same = bool(torch.equal(res["device"][1][0], res["reference"][1][0]) and torch.equal(res["device"][1][1], res["reference"][1][1]))
            out = dict(batch=batch, imgsz=224, images=len(ds), mean_hw=[round(float(v)) for v in sides.mean(0)], device=res["device"][0],
                       reference=res["reference"][0], last_batch_equal=same, workers=a.workers, ref_workers=a.ref_workers, cpus=os.cpu_count(), gpu=info)
            if batch == 64:
                out["train_step_ms_resident_batch"] = round(step_ms, 2)
            print(json.dumps(out), flush=True)
            del ref


if __name__ == "__main__":
    main()
