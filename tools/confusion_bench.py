"""Confusion-matrix timing: ConfusionMatrix.process_batch_padded (one y5_confusion_batch launch per batch) against the
reference's per-image process_batch expressions on torch-cuda (oracle/confusion_ref.py process_batch_torch: device IoU and
candidate search, one `.cpu()` of the matches per image, then counts indexed by 0-d CUDA tensors, each a device read).

    python tools/confusion_bench.py [--batch 32] [--images 5000] [--repeat 5]

Batches are COCO-val-like (oracle/confusion_ref.py synth_batch over tools/ap_bench.py's stats): 300 rows per image,
80 classes, Poisson(7.3) labels, fp16-rounded confidences, in native pixels as val_batch_metrics hands them over.  Arms:
- engine per batch: CUDA events around process_batch_padded, the update alone (it never syncs);
- engine per batch + read: the update, then reading `matrix` (the one sync), host clock;
- reference per batch: val.py's per-image calls for one batch, host clock up to the last count;
- a pass over --images images in batches of --batch (a pool of 8 distinct batches reused), each arm ending with the
  matrix on the host; the reference's pass takes seconds and is timed once.
Every arm's matrix is compared with the reference arm's.  Prints one JSON line with the GPU, its power limit, the run
count and the median (and min) ms of each arm.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import confusion_ref  # noqa: E402
from yolov5_b200.utils.metrics import ConfusionMatrix  # noqa: E402

NC = 80


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def stat(ms):
    return {"median_ms": round(float(np.median(ms)), 4), "min_ms": round(float(np.min(ms)), 4), "runs": len(ms)}


def make_pool(n, batch, dev):
    pool = []
    for k in range(n):
        rows, count, lab6 = confusion_ref.synth_batch(batch, 300, NC, 7.3, seed=100 + k)
        pool.append(tuple(torch.from_numpy(x).to(dev) for x in (rows, count, lab6)))
    return pool


def reference_batch(matrix, rows, count, lab6):
    """val.py:282-309 per image, plots=True, on the batch's device tensors (count read on the host, as val.py's npr is)."""
    cnt = count.tolist()
    for si in range(rows.shape[0]):
        labels = lab6[lab6[:, 0] == si, 1:]
        nl, npr = labels.shape[0], cnt[si]
        if npr == 0:
            if nl:
                confusion_ref.process_batch_torch(matrix, None, labels[:, 0], NC)
            continue
        if nl:
            confusion_ref.process_batch_torch(matrix, rows[si, :npr, :6], labels, NC)
    return matrix


def host_ms(fn, repeat):
    fn()
    out = []
    for _ in range(repeat):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append(1000 * (time.perf_counter() - t0))
    return out


def event_ms(fn, repeat, inner=50):
    fn()
    out = []
    for _ in range(repeat):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(inner):
            fn()
        e1.record()
        e1.synchronize()
        out.append(e0.elapsed_time(e1) / inner)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--images", type=int, default=5000)
    ap.add_argument("--repeat", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("confusion_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    pool = make_pool(8, a.batch, dev)
    rows, count, lab6 = pool[0]
    res = {"gpu": gpu_info(), "host_cpus": os.cpu_count(), "batch": a.batch, "rows_per_image": 300, "classes": NC,
           "labels_per_batch": int(lab6.shape[0])}

    cm = ConfusionMatrix(NC)
    res["engine_update_per_batch"] = stat(event_ms(lambda: cm.process_batch_padded(rows, count, lab6), a.repeat))

    def engine_read():
        c = ConfusionMatrix(NC)
        c.process_batch_padded(rows, count, lab6)
        return c.matrix

    res["engine_update_and_read_per_batch"] = stat(host_ms(engine_read, a.repeat))
    res["reference_per_batch"] = stat(host_ms(lambda: reference_batch(np.zeros((NC + 1, NC + 1)), rows, count, lab6), a.repeat))
    res["equal_per_batch"] = bool(np.array_equal(engine_read(), reference_batch(np.zeros((NC + 1, NC + 1)), rows, count, lab6)))

    n_batches = -(-a.images // a.batch)
    sizes = [min(a.batch, a.images - k * a.batch) for k in range(n_batches)]

    def engine_pass():
        c = ConfusionMatrix(NC)
        for k, s in enumerate(sizes):
            r, n, l = pool[k % len(pool)]
            c.process_batch_padded(r[:s], n[:s], l if s == a.batch else l[l[:, 0] < s])
        return c.matrix

    def reference_pass():
        m = np.zeros((NC + 1, NC + 1))
        for k, s in enumerate(sizes):
            r, n, l = pool[k % len(pool)]
            reference_batch(m, r[:s], n[:s], l if s == a.batch else l[l[:, 0] < s])
        return m

    res["pass_images"] = a.images
    res["engine_pass"] = stat(host_ms(engine_pass, a.repeat))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    want = reference_pass()  # seconds per pass: timed once, after the per-batch arm has warmed the same expressions up
    res["reference_pass"] = stat([1000 * (time.perf_counter() - t0)])
    res["equal_pass"] = bool(np.array_equal(engine_pass(), want))
    res["speedup_per_batch"] = round(res["reference_per_batch"]["median_ms"] / res["engine_update_and_read_per_batch"]["median_ms"], 1)
    res["speedup_pass"] = round(res["reference_pass"]["median_ms"] / res["engine_pass"]["median_ms"], 1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
