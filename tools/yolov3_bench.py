"""yolov3, yolov3-spp and yolov3-tiny on the device: the fp16 forward against the same network written as torch expressions on
torch-cuda (the reference's nn.Module forward: conv + folded BN + SiLU, max_pool2d, cat, upsample, the head convs), the pool
kernels alone with their achieved bytes/s, and the AMP training step, eager and graphed.  Prints the card and its power limit.

    python tools/yolov3_bench.py [--iters 30]
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
import torch.nn.functional as F  # noqa: E402

from oracle import loss_ref  # noqa: E402
from yolov5_b200 import _lib  # noqa: E402
from yolov5_b200.cfg import HYP_SCRATCH_LOW  # noqa: E402
from yolov5_b200.engine import fold_conv_bn  # noqa: E402
from yolov5_b200.models import common as mc  # noqa: E402
from yolov5_b200.models.yolo import Detect, DetectionModel  # noqa: E402

NAMES = ("yolov3", "yolov3-spp", "yolov3-tiny")


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


def torch_forward(model, x):
    """The network as torch-cuda expressions, BatchNorm folded, in x's dtype: the raw head maps."""
    cache = model.__dict__.setdefault("_bench_folded", {})

    def conv(m, t):
        if id(m) not in cache:
            w, b = fold_conv_bn(m.conv, m.bn)
            cache[id(m)] = (w.to(t.dtype), b.to(t.dtype))
        w, b = cache[id(m)]
        return F.silu(F.conv2d(t, w, b, m.conv.stride, m.conv.padding))

    def run(m, t):
        if isinstance(m, mc.Conv):
            return conv(m, t)
        if isinstance(m, mc.Bottleneck):
            y = conv(m.cv2, conv(m.cv1, t))
            return t + y if m.add else y
        if isinstance(m, mc.SPP):
            a = conv(m.cv1, t)
            return conv(m.cv2, torch.cat([a] + [p(a) for p in m.m], 1))
        if isinstance(m, torch.nn.Sequential):
            for s in m:
                t = run(s, t)
            return t
        if isinstance(m, mc.Concat):
            return torch.cat(t, 1)
        return m(t)  # nn.Upsample, nn.MaxPool2d, nn.ZeroPad2d

    ys, t = [], x
    for m in model.model:
        if m.f != -1:
            t = ys[m.f] if isinstance(m.f, int) else [t if j == -1 else ys[j] for j in m.f]
        if isinstance(m, Detect):
            return [F.conv2d(xi, c.weight.to(x.dtype), c.bias.to(x.dtype)).sigmoid() for xi, c in zip(t, m.m)]
        t = run(m, t)
        ys.append(t if m.i in model.save else None)


def model(name, dev, dtype=None, train=False):
    torch.manual_seed(0)
    m = DetectionModel(name).to(dev)
    if train:
        m.hyp = dict(HYP_SCRATCH_LOW)
        return m.train()
    return m.to(dtype).eval()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"card: {card}")
    x = torch.rand(32, 3, 640, 640, device=dev, dtype=torch.float16)
    for name in NAMES:
        m = model(name, dev, torch.float16)
        with torch.no_grad():
            te = timed(lambda: m(x), a.iters)
            tt = timed(lambda: torch_forward(m, x), max(3, a.iters // 3))
        print(f"forward {name} 32x640^2 fp16: engine {te:.2f} ms, torch-cuda expressions {tt:.2f} ms")
        del m
    lib, st = _lib.lib(), C.c_void_p(_lib.stream_ptr(dev))
    # the pool kernels at yolov3-tiny's and yolov3-spp's 32x640^2 shapes; bytes: each input and output element once
    for label, mode, (b, h, w, c) in (("MaxPool2d(2,2) 32x640x640x16", _lib.POOL_K2S2, (32, 640, 640, 16)),
                                      ("MaxPool2d(2,2) 32x80x80x128", _lib.POOL_K2S2, (32, 80, 80, 128)),
                                      ("ZeroPad2d+MaxPool2d(2,1) 32x20x20x512", _lib.POOL_K2S1_ZPAD, (32, 20, 20, 512))):
        xin = torch.randn(b, h, w, c, device=dev, dtype=torch.float16)
        ho, wo = (h // 2, w // 2) if mode == _lib.POOL_K2S2 else (h, w)
        y = torch.empty(b, ho, wo, c, device=dev, dtype=torch.float16)
        dy, dx = torch.randn_like(y), torch.empty_like(xin)
        tf = timed(lambda: lib.y5_maxpool2d(xin.data_ptr(), c, y.data_ptr(), c, b, h, w, c, mode, 0, st), 200)
        tb = timed(lambda: lib.y5_maxpool2d_bwd(xin.data_ptr(), c, dy.data_ptr(), c, dx.data_ptr(), c, b, h, w, c, mode, 0, st), 200)
        nf, nb = 2 * (b * h * w * c + b * ho * wo * c), 2 * (2 * b * h * w * c + b * ho * wo * c)
        print(f"{label} fp16: fwd {tf * 1e3:.1f} us ({nf / tf / 1e6:.0f} GB/s), bwd {tb * 1e3:.1f} us ({nb / tb / 1e6:.0f} GB/s)")
    b, h, w, c = 16, 20, 20, 256  # yolov3-spp's SPP at 16x640^2 training
    cat = torch.randn(b, h, w, 4 * c, device=dev, dtype=torch.float16)
    dcat, da = torch.randn_like(cat), torch.empty(b, h, w, c, device=dev, dtype=torch.float16)
    ws = torch.empty(lib.y5_spp_bwd_workspace_bytes(b, h, w, c), dtype=torch.uint8, device=dev)
    ts = timed(lambda: lib.y5_spp_pool_bwd(cat.data_ptr(), 4 * c, dcat.data_ptr(), 4 * c, da.data_ptr(), c, b, h, w, c, 5, 0, ws.data_ptr(), st), 200)
    nbytes = 2 * (b * h * w * c * 6) + ws.numel() * 2  # a, dcat (4 slices), da; the arg-max codes written and read once
    print(f"SPP backward {b}x{h}x{w}x{c} k=5 fp16: {ts * 1e3:.1f} us ({nbytes / ts / 1e6:.0f} GB/s counting each byte once)")
    # AMP training step at 16x640^2, eager and graphed
    from yolov5_b200.utils.loss import ComputeLoss
    from yolov5_b200.utils.torch_utils import GraphedTrainStep, smart_optimizer

    for name in NAMES:
        m = model(name, dev, train=True)
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
