"""Segmentation-loss timing on the GPU: the engine's ComputeLoss (liby5b200 seg-loss kernels) vs the reference's own
torch expressions on the same GPU, at yolov5s-seg training shapes.

    python tools/seg_loss_bench.py [--batch 16] [--size 640] [--min-seconds 1.0]

Heads (B, 3, 80|40|20, 80|40|20, 117) and proto (B, 32, 160, 160) channels_last, fp16; COCO-shaped labels
(loss_ref.synth_targets) and overlap masks painted from the boxes at image size.  Prints one JSON line: the GPU and
its power limit, loss forward+backward time of both arms, the engine's launches per forward+backward, and the eager
yolov5s-seg training step (forward + seg loss + backward + FusedSGD.fused_step).  CUDA-event timing after warm-up,
each timed window at least --min-seconds long.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import loss_ref, model_ref  # noqa: E402
from tests import seg_loss_ref  # noqa: E402
from yolov5_b200 import _lib  # noqa: E402
from yolov5_b200.cfg import HYP_SCRATCH_LOW, model_cfg  # noqa: E402
from yolov5_b200.models.yolo import SegmentationModel  # noqa: E402
from yolov5_b200.utils.segment.loss import ComputeLoss  # noqa: E402
from yolov5_b200.utils.torch_utils import FusedSGD  # noqa: E402


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
            return ms / n, n
        n = max(n * 2, int(n * 1.2 * 1000 * min_seconds / max(ms, 1e-3)))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("seg_loss_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    bs, sz = args.batch, args.size
    cfg = model_cfg("yolov5s-seg")
    sd = model_ref.synth_state_dict(cfg, seed=7)
    m = SegmentationModel("yolov5s-seg")
    m.load_state_dict(sd)
    m.hyp = dict(HYP_SCRATCH_LOW)
    m = m.to(dev).train()
    anchors = sd["model.24.anchors"]
    tg_np = loss_ref.synth_targets(bs, seed=8)
    masks_np = seg_loss_ref.overlap_masks(tg_np, bs, sz, sz)
    tg, masks = torch.from_numpy(tg_np).to(dev), torch.from_numpy(masks_np).to(dev)
    rs = np.random.RandomState(9)
    p = [torch.from_numpy(rs.normal(0, 1.5, (bs, 3, sz // s, sz // s, 117)).astype(np.float32)).to(dev, torch.float16).requires_grad_(True)
         for s in (8, 16, 32)]
    proto = torch.from_numpy(rs.normal(0, 0.5, (bs, 32, sz // 4, sz // 4)).astype(np.float32)).to(dev, torch.float16)
    proto = proto.contiguous(memory_format=torch.channels_last).requires_grad_(True)
    crit = ComputeLoss(m, overlap=True)

    def engine():
        for a in p + [proto]:
            a.grad = None
        loss, _ = crit((p, proto), tg, masks)
        loss.backward()

    def reference():
        for a in p + [proto]:
            a.grad = None
        with torch.autocast("cuda", dtype=torch.float16):
            loss, _ = seg_loss_ref.compute_seg_loss_torch(p, proto, tg, masks, anchors, HYP_SCRATCH_LOW, True)
        loss.backward()

    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    engine()
    torch.cuda.synchronize()
    launches = _lib.launch_count() - n0
    eng_ms, eng_n = timed(engine, args.min_seconds)
    ref_ms, ref_n = timed(reference, args.min_seconds)

    g = torch.Generator().manual_seed(10)
    img = (torch.rand(bs, 3, sz, sz, generator=g) * 255).to(torch.uint8).to(dev)
    opt = FusedSGD([q for q in m.parameters() if q.requires_grad], lr=0.01, momentum=0.937, nesterov=True)

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.float16):
            pred = m(img)
        loss, _ = crit(pred, tg, masks)
        loss.backward()
        opt.fused_step()

    step_ms, step_n = timed(step, args.min_seconds)
    print(json.dumps(dict(
        gpu=gpu_info(), batch=bs, size=sz, dtype="fp16", targets=int(tg.shape[0]),
        seg_loss_fwd_bwd_ms=dict(engine=round(eng_ms, 4), torch_reference=round(ref_ms, 4), speedup=round(ref_ms / eng_ms, 2),
                                 iters=dict(engine=eng_n, torch_reference=ref_n)),
        engine_launches_per_fwd_bwd=int(launches),
        train_step_ms=dict(engine_eager=round(step_ms, 3), iters=step_n))))


if __name__ == "__main__":
    main()
