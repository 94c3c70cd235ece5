"""yolov5s-ghost on the device: the fp16 forward against yolov5s and against the same network written as the reference's torch
expressions on torch-cuda (conv + folded BN + act, cuDNN's depthwise conv, cat, upsample, the head convs; channels_last); each
depthwise 5x5 conv alone at the model's 32x640^2 shapes (forward, data gradient, weight gradient) with its achieved bytes/s next
to cuDNN's depthwise conv on the same shapes; the sum of the forward kernels against the bandwidth floor of those layers; and
the 16x640^2 AMP training step, eager and graphed.  Prints the card and its power limit.

    python tools/ghost_bench.py [--iters 30]
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

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet: the floor below is bytes / this rate, not a measured figure


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


def torch_forward(model, x, shapes=None):
    """The network as the reference's torch-cuda expressions, BatchNorm folded, in x's dtype: the raw head maps.  `shapes` (a list)
    collects the (B, c, H, W) input of every depthwise conv."""
    cache = model.__dict__.setdefault("_bench_folded", {})

    def conv(m, t):
        if id(m) not in cache:
            w, b = fold_conv_bn(m.conv, m.bn)
            cache[id(m)] = (w.to(t.dtype).contiguous(memory_format=torch.channels_last), b.to(t.dtype))
        w, b = cache[id(m)]
        if m.conv.groups > 1 and shapes is not None:
            shapes.append(tuple(t.shape))
        return m.act(F.conv2d(t, w, b, m.conv.stride, m.conv.padding, groups=m.conv.groups))

    def run(m, t):
        if isinstance(m, mc.Conv):
            return conv(m, t)
        if isinstance(m, mc.GhostConv):
            y = conv(m.cv1, t)
            return torch.cat((y, conv(m.cv2, y)), 1)
        if isinstance(m, mc.GhostBottleneck):
            return run(m.conv[2], run(m.conv[0], t)) + t
        if isinstance(m, mc.Bottleneck):
            y = conv(m.cv2, conv(m.cv1, t))
            return t + y if m.add else y
        if isinstance(m, mc.C3):
            a = conv(m.cv1, t)
            for bt in m.m:
                a = run(bt, a)
            return conv(m.cv3, torch.cat((a, conv(m.cv2, t)), 1))
        if isinstance(m, mc.SPPF):
            a = conv(m.cv1, t)
            y1 = m.m(a)
            y2 = m.m(y1)
            return conv(m.cv2, torch.cat((a, y1, y2, m.m(y2)), 1))
        if isinstance(m, mc.Concat):
            return torch.cat(t, 1)
        return m(t)  # nn.Upsample

    ys, t = [], x.contiguous(memory_format=torch.channels_last)
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


def depthwise_kernels(shapes, dev, iters):
    """Each depthwise conv of the model alone, NHWC fp16, ours and cuDNN's (channels_last); bytes count each input, output and
    residual element once (the two-output GhostBottleneck form is timed as the forward of the plain form)."""
    lib, st = _lib.lib(), C.c_void_p(_lib.stream_ptr(dev))
    tot = {"fwd": 0.0, "dgrad": 0.0, "wgrad": 0.0, "cudnn fwd": 0.0, "cudnn dgrad": 0.0, "cudnn wgrad": 0.0}
    floor_bytes = 0
    seen = {}
    for s in shapes:
        seen[s] = seen.get(s, 0) + 1
    print("depthwise 5x5 conv alone, fp16 NHWC (B, c, H, W) x count: time us (GB/s counting each byte once)")
    for (b, c, h, w), n in seen.items():
        x = torch.randn(b, h, w, c, device=dev, dtype=torch.float16)
        y, dy, dx = torch.empty_like(x), torch.randn_like(x), torch.empty_like(x)
        wt = (torch.randn(c, 25, device=dev) * 0.2).half()
        bias = torch.zeros(c, device=dev)
        dw = torch.empty(c, 25, device=dev)
        ix, iy, idy, idx = x.data_ptr(), y.data_ptr(), dy.data_ptr(), dx.data_ptr()
        t = {
            "fwd": timed(lambda: lib.y5_dwconv_fwd(ix, c, wt.data_ptr(), bias.data_ptr(), iy, c, None, 0, None, 0, None, 0, b, h, w, c, 5, 1,
                                                   _lib.ACT_SILU, 0.0, 0, 0, st), iters),
            "dgrad": timed(lambda: lib.y5_dwconv_fwd(idy, c, wt.data_ptr(), None, idx, c, None, 0, None, 0, None, 0, b, h, w, c, 5, 1,
                                                     _lib.ACT_NONE, 0.0, 1, 0, st), iters),
            "wgrad": timed(lambda: lib.y5_dwconv_wgrad(ix, c, idy, c, dw.data_ptr(), b, h, w, c, 5, 1, 0, st), iters),
        }
        xc, dyc = x.permute(0, 3, 1, 2), dy.permute(0, 3, 1, 2)  # channels_last views of the same bytes
        wc = wt.view(c, 1, 5, 5)
        t["cudnn fwd"] = timed(lambda: F.silu(F.conv2d(xc, wc, bias.half(), 1, 2, groups=c)), iters)
        t["cudnn dgrad"] = timed(lambda: torch.ops.aten.convolution_backward(dyc, xc, wc, None, [1, 1], [2, 2], [1, 1], False, [0, 0], c,
                                                                             [True, False, False]), iters)
        t["cudnn wgrad"] = timed(lambda: torch.ops.aten.convolution_backward(dyc, xc, wc, None, [1, 1], [2, 2], [1, 1], False, [0, 0], c,
                                                                             [False, True, False]), iters)
        nbytes = 2 * 2 * b * h * w * c  # one input and one output map (wgrad: x and dy)
        floor_bytes += n * nbytes
        for k, v in t.items():
            tot[k] += n * v
        print(f"  ({b}, {c}, {h}, {w}) x{n}: " + ", ".join(f"{k} {v * 1e3:.1f} ({nbytes / v / 1e6:.0f})" for k, v in t.items()))
    floor_us = floor_bytes / HBM_BYTES_PER_S * 1e6
    print(f"all {len(shapes)} depthwise convs: {floor_bytes / 1e6:.0f} MB, floor at 3.35 TB/s {floor_us:.0f} us")
    for k, v in tot.items():
        print(f"  {k}: {v * 1e3:.0f} us total, {100 * floor_us / (v * 1e3):.0f} % of the floor's rate")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"card: {card}")
    x = torch.rand(32, 3, 640, 640, device=dev, dtype=torch.float16)
    shapes = []
    for name in ("yolov5s", "yolov5s-ghost"):
        m = model(name, dev, torch.float16)
        with torch.no_grad():
            te = timed(lambda: m(x), a.iters)
            line = f"forward {name} 32x640^2 fp16: engine {te:.2f} ms"
            if name == "yolov5s-ghost":
                torch_forward(m, x, shapes)
                tt = timed(lambda: torch_forward(m, x), max(3, a.iters // 3))
                line += f", reference expressions on torch-cuda (channels_last, cuDNN depthwise) {tt:.2f} ms"
        print(line)
        del m
    torch.backends.cudnn.benchmark = True
    depthwise_kernels(shapes, dev, 100)
    from yolov5_b200.utils.loss import ComputeLoss
    from yolov5_b200.utils.torch_utils import GraphedTrainStep, smart_optimizer

    m = model("yolov5s-ghost", dev, train=True)
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
    print(f"AMP train step yolov5s-ghost 16x640^2: eager {te:.1f} ms, graphed {tg:.1f} ms")


if __name__ == "__main__":
    main()
