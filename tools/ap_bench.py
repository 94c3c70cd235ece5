"""Validation AP timing: the engine's ap_per_class / ap_per_class_box_and_mask / ap_per_class_batch (csrc/ap_metrics.cu)
against numpy on the host.

    python tools/ap_bench.py [--images 5000 1000] [--repeat 5]

Stats are COCO-val-like (oracle/ap_ref.py synth_stats): 300 rows per image (what conf_thres 0.001 and max_det 300 keep on a
real model), 80 classes, Poisson(7.3) labels per image, fp16-rounded confidences, 10 nested IoU thresholds.  Arms:
- engine, CUDA tensors in: device events around the call, up to the numpy result on the host;
- engine, numpy in: host wall time, the upload included (the reference's calling convention);
- engine, ap_per_class_batch on the padded (images, 300, ...) tensors a batched val loop holds;
- engine, box + mask (ap_per_class_box_and_mask, one sort for both);
- host: oracle/ap_ref.py with numpy's default argsort, standing in for the reference's numpy expressions (same operations,
  one core), detection and box + mask (two calls, as the reference makes them).
Prints one JSON line with the GPU, its power limit and the median (and min) ms of each arm.
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
from oracle import ap_ref  # noqa: E402
from yolov5_b200.utils import metrics  # noqa: E402
from yolov5_b200.utils.segment.metrics import ap_per_class_box_and_mask  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


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


def event_ms(fn, repeat):
    fn()
    out = []
    for _ in range(repeat):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()  # returns numpy arrays: the results have been read back when it returns
        e1.record()
        e1.synchronize()
        out.append(e0.elapsed_time(e1))
    return out


def stat(ms):
    return {"median_ms": round(float(np.median(ms)), 3), "min_ms": round(float(np.min(ms)), 3)}


def run(n_img, repeat, dev):
    stats = ap_ref.synth_stats(n_img, 300, 80, 7.3, 10, seed=n_img, ties=True, min_det=300)
    tp, conf, pc, tc = ap_ref.concat_stats(stats)
    tp_m = tp & (np.random.RandomState(1).rand(*tp.shape) < 0.8)
    d = [torch.from_numpy(x).to(dev) for x in (tp, conf, pc, tc, tp_m)]
    correct = d[0].view(n_img, 300, 10)
    rows = torch.zeros(n_img, 300, 6, device=dev)
    rows[..., 4], rows[..., 5] = d[1].view(n_img, 300), d[2].view(n_img, 300)
    count = torch.full((n_img,), 300, dtype=torch.int32, device=dev)
    res = {"images": n_img, "rows": int(len(conf)), "classes": int(len(np.unique(tc))), "labels": int(len(tc))}
    res["engine_cuda_in"] = stat(event_ms(lambda: metrics.ap_per_class(d[0], d[1], d[2], d[3]), repeat))
    res["engine_numpy_in"] = stat(host_ms(lambda: metrics.ap_per_class(tp, conf, pc, tc), repeat))
    res["engine_batch"] = stat(event_ms(lambda: metrics.ap_per_class_batch(correct, rows, count, d[3]), repeat))
    res["engine_box_mask"] = stat(event_ms(lambda: ap_per_class_box_and_mask(d[4], d[0], d[1], d[2], d[3]), repeat))
    t0 = time.perf_counter()
    want = ap_ref.ap_per_class(tp, conf, pc, tc, stable=False)
    host = [1000 * (time.perf_counter() - t0)]
    for _ in range(max(1, repeat // 2)):
        t0 = time.perf_counter()
        ap_ref.ap_per_class(tp, conf, pc, tc, stable=False)
        host.append(1000 * (time.perf_counter() - t0))
    res["host_numpy_default_argsort"] = stat(host)
    t0 = time.perf_counter()
    ap_ref.ap_per_class(tp, conf, pc, tc, stable=False)
    ap_ref.ap_per_class(tp_m, conf, pc, tc, stable=False)
    res["host_numpy_box_mask"] = stat([1000 * (time.perf_counter() - t0)])
    got = metrics.ap_per_class(tp, conf, pc, tc)
    stable = ap_ref.ap_per_class(tp, conf, pc, tc)
    res["equal_to_oracle_stable_order"] = all(np.array_equal(a, b) for a, b in zip(got, stable))
    res["map50_95_engine_minus_default_argsort"] = float(got[5].mean() - want[5].mean())
    res["speedup_cuda_in_vs_host"] = round(res["host_numpy_default_argsort"]["median_ms"] / res["engine_cuda_in"]["median_ms"], 1)
    res["speedup_box_mask_vs_host"] = round(res["host_numpy_box_mask"]["median_ms"] / res["engine_box_mask"]["median_ms"], 1)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, nargs="+", default=[5000, 1000])
    ap.add_argument("--repeat", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ap_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    out = {"gpu": gpu_info(), "host_cpus": os.cpu_count(), "runs": [run(n, a.repeat, dev) for n in a.images]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
