"""yolov5s-transformer on the device: forward against yolov5s, the attention kernels alone, the AMP training step, and the
reference's expressions on torch-cuda for the same model.  Prints the card and its power limit with the numbers.

    python tools/transformer_bench.py [--iters 30]
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import loss_ref, model_ref, transformer_ref  # noqa: E402
from yolov5_b200 import _lib  # noqa: E402
from yolov5_b200.cfg import HYP_SCRATCH_LOW, model_cfg  # noqa: E402
from yolov5_b200.models.yolo import DetectionModel  # noqa: E402


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def model(name, dev, dtype=None, train=False):
    cfg = model_cfg(name)
    sd = (transformer_ref if "transformer" in name else model_ref).synth_state_dict(cfg, seed=1)
    m = DetectionModel(cfg)
    m.load_state_dict(sd)
    m = m.to(dev)
    if train:
        m.hyp = dict(HYP_SCRATCH_LOW)
        return m.train(), cfg, sd
    return m.to(dtype).eval(), cfg, sd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"card: {card}")
    # forward: engine yolov5s-transformer vs yolov5s, and the reference's expressions on torch-cuda
    for b, s in ((32, 640), (8, 1280)):
        x = torch.rand(b, 3, s, s, device=dev, dtype=torch.float16)
        res = {}
        for name in ("yolov5s", "yolov5s-transformer"):
            m, cfg, sd = model(name, dev, torch.float16)
            with torch.no_grad():
                res[name] = timed(lambda: m(x), a.iters)
            if name == "yolov5s-transformer":
                sd_d = {k: (v.to(dev, torch.float16) if v.is_floating_point() else v.to(dev)) for k, v in sd.items()}
                with torch.no_grad():
                    res["torch-cuda reference expressions"] = timed(lambda: transformer_ref.forward(cfg, sd_d, x, fused=True), max(3, a.iters // 3))
            del m
        print(f"forward {b}x{s}^2 fp16: " + ", ".join(f"{k} {v:.2f} ms" for k, v in res.items()))
    # the attention kernels alone at the P5 shapes (4 heads of 64: yolov5s-transformer)
    lib = _lib.lib()
    for b, L in ((32, 400), (8, 1600)):
        heads, dh = 4, 64
        c = heads * dh
        qkv = torch.randn(b * L, 3 * c, device=dev, dtype=torch.float16)
        o = torch.empty(b * L, c, device=dev, dtype=torch.float16)
        do = torch.randn_like(o)
        dqkv = torch.empty_like(qkv)
        lse = torch.empty(b * heads * L, device=dev)
        delta = torch.empty_like(lse)
        es, p = 2, qkv.data_ptr()
        st = C.c_void_p(_lib.stream_ptr(dev))

        def fwd():
            lib.y5_attention_fwd(p, p + c * es, p + 2 * c * es, 3 * c, o.data_ptr(), c, lse.data_ptr(), b, L, heads, dh, dh ** -0.5, 0, st)

        def bwd():
            d = dqkv.data_ptr()
            lib.y5_attention_bwd(p, p + c * es, p + 2 * c * es, 3 * c, o.data_ptr(), c, do.data_ptr(), c, lse.data_ptr(), delta.data_ptr(), d,
                                 d + c * es, d + 2 * c * es, 3 * c, b, L, heads, dh, dh ** -0.5, 0, st)

        flops = 4 * b * heads * L * L * dh
        tf, tb = timed(fwd, 200), timed(bwd, 200)
        print(f"attention B={b} L={L} heads={heads} dh={dh} fp16: fwd {tf * 1e3:.1f} us ({flops / tf / 1e9:.0f} TFLOP/s), "
              f"bwd {tb * 1e3:.1f} us ({2.5 * flops / tb / 1e9:.0f} TFLOP/s at 2.5x the forward's FLOPs)")
    # AMP training step at 16x640^2, eager and graphed
    from yolov5_b200.utils.loss import ComputeLoss
    from yolov5_b200.utils.torch_utils import GraphedTrainStep, smart_optimizer

    for name in ("yolov5s", "yolov5s-transformer"):
        m, _, _ = model(name, dev, train=True)
        opt = smart_optimizer(m, "SGD", lr=0.01, momentum=0.937, decay=5e-4)
        img = torch.from_numpy(np.random.RandomState(0).randint(0, 256, (16, 3, 640, 640)).astype(np.uint8)).to(dev)
        tgt = torch.from_numpy(loss_ref.synth_targets(16, seed=1)).float().to(dev)
        loss_fn, scaler = ComputeLoss(m), torch.amp.GradScaler("cuda")

        def eager():
            with torch.autocast("cuda", dtype=torch.float16):
                p = m(img)
            loss, _ = loss_fn(p, tgt)
            scaler.scale(loss).backward()
            opt.fused_step(scaler=scaler, max_norm=10.0, model=m)
            opt.zero_grad()

        te = timed(eager, max(5, a.iters // 3))
        step = GraphedTrainStep(m, loss_fn, opt, batch=16, size=640)
        tg = timed(lambda: step(img, tgt), max(5, a.iters // 3))
        print(f"AMP train step {name} 16x640^2: eager {te:.1f} ms, graphed {tg:.1f} ms")
        del m, step


if __name__ == "__main__":
    main()
