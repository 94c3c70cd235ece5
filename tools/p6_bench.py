"""The P6 models at 1280 on the device: yolov5s6 and yolov5x6 fp16 forward, and forward + NMS (detect.py's regime, as bench.py
times it), at batch 8 and 32; the yolov5s6 AMP training step at 8 x 1280, eager and GraphedTrainStep.  Each workload is also run
as the reference's expressions on torch-cuda in the same process: the oracle's functional forward (F.conv2d / silu / max_pool2d
/ cat / interpolate) with channels_last weights and activations and cudnn.benchmark, the reference's NMS loop with
torchvision.ops.nms, and for training the forward under torch.autocast with the reference's loss as torch ops, GradScaler,
clip_grad_norm_ and torch.optim.SGD.  Weights are bench.py's seeded synthetic ones (Detect biases calibrated so NMS sees
~2 % of the anchors), images its blocky synthetic ones.

Every number is the median of --runs timed windows (engine and torch windows alternate), each window --iters calls after
warm-up; the min-max spread over the windows is printed beside it, with the card's name and power limit.

    python tools/p6_bench.py [--runs 5] [--iters 20]
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torchvision  # noqa: E402

from bench import NMS_KW, bench_state_dict, synth_images_u8  # noqa: E402
from oracle import loss_ref, model_ref  # noqa: E402
from yolov5_b200.cfg import HYP_SCRATCH_LOW, model_cfg  # noqa: E402
from yolov5_b200.models.yolo import DetectionModel  # noqa: E402
from yolov5_b200.utils.general import nms_device  # noqa: E402

SIZE = 1280
BALANCE4 = (4.0, 1.0, 0.25, 0.06)


def window(fn, iters):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def compare(label, fns, runs, iters, warmup=3):
    """fns: {arm: callable}; warms every arm up, then alternates `runs` timed windows of the arms; prints median [min-max] ms."""
    for fn in fns.values():
        for _ in range(warmup):
            fn()
    ts = {k: [] for k in fns}
    for _ in range(runs):
        for k, fn in fns.items():
            ts[k].append(window(fn, iters))
    parts = [f"{k} {np.median(v):.2f} ms [{min(v):.2f}-{max(v):.2f}]" for k, v in ts.items()]
    print(f"{label}: " + ", ".join(parts), flush=True)


def ref_nms(pred, conf_thres=0.25, iou_thres=0.45, max_det=300, max_nms=30000, max_wh=7680):
    """The reference's non_max_suppression (utils/general.py), single-label, no masks, on torch-cuda."""
    xc = pred[..., 4] > conf_thres
    out = []
    for xi, x in enumerate(pred):
        x = x[xc[xi]].float()
        x[:, 5:] *= x[:, 4:5]
        box = torch.cat((x[:, :2] - x[:, 2:4] / 2, x[:, :2] + x[:, 2:4] / 2), 1)
        conf, j = x[:, 5:].max(1, keepdim=True)
        x = torch.cat((box, conf, j.float()), 1)[conf.view(-1) > conf_thres]
        x = x[x[:, 4].argsort(descending=True)[:max_nms]]
        i = torchvision.ops.nms(x[:, :4] + x[:, 5:6] * max_wh, x[:, 4], iou_thres)[:max_det]
        out.append(x[i])
    return out


def torch_forward(cfg, sd_cl):
    return lambda x: model_ref.forward(cfg, sd_cl, x, fused=True)[0]


def inference(name, dev, runs, iters):
    cfg = model_cfg(name)
    sd = bench_state_dict(cfg)
    m = DetectionModel(name)
    m.load_state_dict(sd)
    m = m.to(dev).half().eval()
    sd_cl = {k: (v.to(dev, torch.float16).contiguous(memory_format=torch.channels_last) if v.dim() == 4 else
                 (v.to(dev, torch.float16) if v.is_floating_point() else v.to(dev))) for k, v in sd.items()}
    ref = torch_forward(cfg, sd_cl)
    for bs in (8, 32):
        x = (torch.from_numpy(synth_images_u8(bs, SIZE, 1)).to(dev).half() / 255).contiguous()
        xc = x.contiguous(memory_format=torch.channels_last)
        with torch.no_grad():
            z = m(x)[0]
            cand = int((z[..., 4] > NMS_KW["conf_thres"]).sum()) // bs
            compare(f"{name} {bs}x{SIZE}^2 fp16 forward", {"engine": lambda: m(x), "torch-cuda reference": lambda: ref(xc)}, runs, iters)
            compare(f"{name} {bs}x{SIZE}^2 fp16 forward + NMS ({cand} rows/img above conf {NMS_KW['conf_thres']})",
                    {"engine": lambda: nms_device(m(x)[0], **NMS_KW), "torch-cuda reference": lambda: ref_nms(ref(xc), **NMS_KW)}, runs, iters)
        del x, xc, z
        torch.cuda.empty_cache()
    del m, sd_cl


def training(name, bs, dev, runs, iters):
    from yolov5_b200.utils.loss import ComputeLoss
    from yolov5_b200.utils.torch_utils import GraphedTrainStep, smart_optimizer

    cfg = model_cfg(name)
    sd = model_ref.synth_state_dict(cfg, seed=0)
    img = torch.from_numpy(synth_images_u8(bs, SIZE, 2)).to(dev)
    tgt = torch.from_numpy(loss_ref.synth_targets(bs, seed=3)).float().to(dev)
    hyp = dict(HYP_SCRATCH_LOW)
    m = DetectionModel(name)
    m.load_state_dict(sd)
    m = m.to(dev).train()
    m.hyp = hyp
    opt = smart_optimizer(m, "SGD", lr=1e-3, momentum=0.937, decay=5e-4)
    loss_fn, scaler = ComputeLoss(m), torch.amp.GradScaler("cuda")

    def eager():
        with torch.autocast("cuda", dtype=torch.float16):
            p = m(img)
        loss, _ = loss_fn(p, tgt)
        scaler.scale(loss).backward()
        opt.fused_step(scaler=scaler, max_norm=10.0, model=m)
        opt.zero_grad()

    graphed = GraphedTrainStep(m, loss_fn, opt, batch=bs, size=SIZE)
    params = {k: (torch.nn.Parameter(v.to(dev).contiguous(memory_format=torch.channels_last) if v.dim() == 4 else v.to(dev))
                  if v.is_floating_point() and "running" not in k and "anchors" not in k else v.to(dev)) for k, v in sd.items()}
    plist = [q for q in params.values() if isinstance(q, torch.nn.Parameter)]
    anchors = params[[k for k in params if k.endswith(".anchors")][0]]
    opt_r = torch.optim.SGD(plist, lr=1e-3, momentum=0.937, nesterov=True, foreach=True)
    sc_r = torch.amp.GradScaler("cuda")

    def step_ref():
        x = (img.half() / 255).contiguous(memory_format=torch.channels_last)
        with torch.autocast("cuda", dtype=torch.float16):
            p = model_ref.forward(cfg, params, x, training=True, bn_batch_stats=True)
            loss, _ = loss_ref.compute_loss_torch([q.float() for q in p], tgt, anchors, hyp, balance=BALANCE4)
        opt_r.zero_grad(set_to_none=True)
        sc_r.scale(loss).backward()
        sc_r.unscale_(opt_r)
        torch.nn.utils.clip_grad_norm_(plist, max_norm=10.0)
        sc_r.step(opt_r)
        sc_r.update()

    compare(f"{name} {bs}x{SIZE}^2 AMP training step",
            {"engine eager": eager, "engine GraphedTrainStep": lambda: graphed(img, tgt), "torch-cuda reference": step_ref},
            runs, max(3, iters // 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("p6_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(f"card: {card}; torch {torch.__version__}, cuDNN {torch.backends.cudnn.version()}; {a.runs} windows x {a.iters} calls per number",
          flush=True)
    torch.backends.cudnn.benchmark = True
    for name in ("yolov5s6", "yolov5x6"):
        inference(name, dev, a.runs, a.iters)
    training("yolov5s6", 8, dev, a.runs, a.iters)


if __name__ == "__main__":
    main()
