"""Cost of the Conv activation on an H100: SiLU vs LeakyReLU(0.1), measured in the same run, alternating the two.

    python tools/activation_bench.py [--rounds 3] [--fwd-iters 50] [--train-steps 10]

  forward: yolov5s, 32 x 3 x 640 x 640 fp16, eval (the engine's CUDA-graph replay), uint8 images resident on the GPU;
  training: yolov5m, 16 x 3 x 640 x 640 uint8 images, fp16 autocast forward (batch-statistics BN) + ComputeLoss + backward +
            the fused SGD step, eager.
Both models carry the same seeded weights; only Conv.default_act differs.  Each round times SiLU then LeakyReLU with CUDA events
after a warm-up; the medians over rounds are printed, with the card's name and power limit.  Prints one JSON line.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import loss_ref, model_ref  # noqa: E402
from yolov5_b200.cfg import HYP_SCRATCH_LOW, model_cfg  # noqa: E402
from yolov5_b200.models.common import Conv  # noqa: E402
from yolov5_b200.models.yolo import DetectionModel  # noqa: E402
from yolov5_b200.utils.loss import ComputeLoss  # noqa: E402
from yolov5_b200.utils.torch_utils import smart_optimizer  # noqa: E402

ACTS = {"silu": nn.SiLU, "leaky0.1": lambda: nn.LeakyReLU(0.1)}


def build(name, act, dev, train):
    Conv.default_act = ACTS[act]()
    try:
        m = DetectionModel(name)
    finally:
        Conv.default_act = nn.SiLU()
    m.load_state_dict(model_ref.synth_state_dict(model_cfg(name), seed=1))
    if train:
        m = m.to(dev).train()
        m.hyp = dict(HYP_SCRATCH_LOW)
    else:
        m = m.half().to(dev).eval()
    return m


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--fwd-iters", type=int, default=50)
    ap.add_argument("--train-steps", type=int, default=10)
    ap.add_argument("--fwd-batch", type=int, default=32)
    ap.add_argument("--train-batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=640)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("activation_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()

    img = torch.from_numpy(np.random.RandomState(0).randint(0, 256, (a.fwd_batch, 3, a.size, a.size)).astype(np.uint8)).to(dev)
    fwd = {act: build("yolov5s", act, dev, False) for act in ACTS}
    timg = torch.from_numpy(np.random.RandomState(1).randint(0, 256, (a.train_batch, 3, a.size, a.size)).astype(np.uint8)).to(dev)
    tgt = torch.from_numpy(loss_ref.synth_targets(a.train_batch, seed=2)).float().to(dev)
    train = {}
    for act in ACTS:
        m = build("yolov5m", act, dev, True)
        opt = smart_optimizer(m, "SGD", 0.01, 0.937, 5e-4)
        train[act] = (m, ComputeLoss(m), opt, torch.amp.GradScaler("cuda"))

    def fwd_fn(act):
        m = fwd[act]
        return lambda: m(img)

    def train_fn(act):
        m, loss_fn, opt, scaler = train[act]

        def step():
            with torch.autocast("cuda", dtype=torch.float16):
                p = m(timg)
            loss, _ = loss_fn(p, tgt)
            scaler.scale(loss).backward()
            opt.fused_step(scaler=scaler, max_norm=10.0)
            opt.zero_grad()
        return step

    res = {f"{k}_{act}": [] for k in ("fwd_ms", "train_ms") for act in ACTS}
    for _ in range(a.rounds):
        for act in ACTS:
            res[f"fwd_ms_{act}"].append(timed(fwd_fn(act), a.fwd_iters, 5))
        for act in ACTS:
            res[f"train_ms_{act}"].append(timed(train_fn(act), a.train_steps, 3))
    med = {k: statistics.median(v) for k, v in res.items()}
    out = dict(gpu=gpu, fwd="yolov5s %dx3x%d^2 fp16 eval" % (a.fwd_batch, a.size), train="yolov5m %dx3x%d^2 fp16 AMP step" % (a.train_batch, a.size),
               rounds=a.rounds, **{k: round(v, 3) for k, v in med.items()}, all=res)
    for act in ACTS:
        out[f"fwd_img_s_{act}"] = round(a.fwd_batch / med[f"fwd_ms_{act}"] * 1e3, 1)
        out[f"train_img_s_{act}"] = round(a.train_batch / med[f"train_ms_{act}"] * 1e3, 1)
    out["fwd_leaky_vs_silu"] = round(med["fwd_ms_leaky0.1"] / med["fwd_ms_silu"], 4)
    out["train_leaky_vs_silu"] = round(med["train_ms_leaky0.1"] / med["train_ms_silu"], 4)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
