"""Wide Detect head timing on the GPU: yolov5l with nc = 365 (Objects365, no = 370 outputs per anchor: three 128-column N tiles
per anchor in the head GEMM) against the same model at nc = 80, and the reference's expressions on torch-cuda.

    python tools/wide_head_bench.py [--batch 64] [--size 640] [--min-seconds 1.0] [--nc 365,80] [--no-reference]

Per nc: the engine's forward, forward + non_max_suppression (conf 0.25, iou 0.45, max_det 300), and the head GEMM of each level
alone (y5_detect_plan_run_to on the level's input as the forward left it) with its algorithmic bytes (read M * Cin * 2, write
2 * M * na * no * 2: raw and z) and the bandwidth they imply.  The reference arm is oracle/model_ref.forward(fused=True) in the
same dtype with cuDNN (the reference's own expressions evaluated by torch).  Prints one JSON line with the GPU's name and power
limit read in the same run.  CUDA-event timing after warm-up, each timed window at least --min-seconds long.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import model_ref  # noqa: E402
from yolov5_b200 import _lib  # noqa: E402
from yolov5_b200.cfg import model_cfg  # noqa: E402
from yolov5_b200.models.yolo import DetectionModel  # noqa: E402
from yolov5_b200.utils.general import non_max_suppression  # noqa: E402


def timed(fn, min_seconds, warmup=3):
    """mean ms per call over a window of at least `min_seconds` (device events)."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    n = 1
    while True:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        if ms >= 1000 * min_seconds:
            return ms / n
        n = max(n * 2, int(n * 1.2 * 1000 * min_seconds / max(ms, 1e-3)))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def head_levels(m, x, min_seconds):
    """Time each level's head GEMM alone; the level inputs are the static buffers the last forward filled."""
    with _lib.on(x.device):
        prog = m._program(x)
    lib, st = _lib.lib(), C.c_void_p(_lib.stream_ptr(x.device))
    det = m.model[-1]
    z = torch.empty(prog.B, prog.z_rows, det.no, dtype=prog.dtype, device=x.device)
    out = []
    for i, (plan, shape) in enumerate(zip(prog.head_ops, prog.det_shapes)):
        raw = torch.empty(shape, dtype=prog.dtype, device=x.device)
        B, na, ny, nx, no = shape
        cin = det.m[i].in_channels
        M = B * ny * nx

        def run():
            _lib.check(lib.y5_detect_plan_run_to(plan, raw.data_ptr(), z.data_ptr(), st), "detect")

        ms = timed(run, min_seconds)
        nbytes = M * cin * 2 + 2 * M * na * no * 2
        out.append({"level": i, "ny": ny, "nx": nx, "cin": cin, "M": M, "ms": round(ms, 4), "bytes": nbytes,
                    "GB_per_s": round(nbytes / ms / 1e6, 1)})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--nc", default="365,80", help="comma-separated class counts")
    ap.add_argument("--no-reference", action="store_true", help="skip the torch-cuda reference arm")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("wide_head_bench.py: needs a CUDA device")
    dev, dt = torch.device("cuda:0"), torch.bfloat16
    torch.backends.cudnn.benchmark = True
    res = {"gpu": gpu_info(), "model": "yolov5l", "batch": a.batch, "size": a.size, "dtype": "bf16", "runs": {}}
    x = torch.from_numpy(np.random.RandomState(0).uniform(0, 1, (a.batch, 3, a.size, a.size)).astype(np.float32)).to(dev, dt)
    for nc in (int(v) for v in a.nc.split(",")):
        cfg = dict(model_cfg("yolov5l"), nc=nc)
        sd = model_ref.synth_state_dict(cfg, seed=0, head_bias="hot")
        m = DetectionModel("yolov5l", nc=nc)
        m.load_state_dict(sd)
        m = m.to(dev, dt).eval()
        r = {"no": 5 + nc}
        r["forward_ms"] = round(timed(lambda: m(x), a.min_seconds), 3)
        r["forward_nms_ms"] = round(timed(lambda: non_max_suppression(m(x)[0], 0.25, 0.45, max_det=300), a.min_seconds), 3)
        r["head_levels"] = head_levels(m, x, a.min_seconds)
        r["head_ms"] = round(sum(lv["ms"] for lv in r["head_levels"]), 4)
        del m
        if a.no_reference:
            res["runs"][f"nc{nc}"] = r
            continue
        sd_d = {k: (v.to(dev, dt) if v.is_floating_point() else v.to(dev)) for k, v in sd.items()}

        def ref_forward():
            with torch.no_grad():
                return model_ref.forward(cfg, sd_d, x, fused=True)

        r["torch_reference_forward_ms"] = round(timed(ref_forward, a.min_seconds, warmup=2), 3)
        del sd_d
        torch.cuda.empty_cache()
        res["runs"][f"nc{nc}"] = r
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
