"""Training-step timing on an H100: engine (yolov5_b200 train path) vs torch autocast execution of the same model.

    python tools/train_bench.py [--model yolov5s] [--batch 16] [--size 640] [--dtype fp16] [--steps 10]

Both arms: uint8 images resident on the GPU -> forward (batch-stat BN) -> ComputeLoss (liby5b200 loss kernel for both, it
is <1 % of the step) -> backward -> SGD(momentum, nesterov) step.  CUDA-event timing, 3 warm-up steps.
"""
import argparse
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import loss_ref, model_ref  # reference arm only
from yolov5_b200.cfg import HYP_SCRATCH_LOW, model_cfg
from yolov5_b200.models.yolo import DetectionModel
from yolov5_b200.utils.loss import ComputeLoss


def timed(fn, steps, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def graphed(step, steps):
    """Capture one whole training step (forward, loss, backward, optimizer) in a CUDA graph and time its replays."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            step()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    return timed(g.replay, steps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="yolov5s")
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--dtype", default="fp16")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--skip-reference", action="store_true")
    ap.add_argument("--train-only", action="store_true", help="skip the forward-only leg (for ncu launch lists of the step)")
    ap.add_argument("--graph", action="store_true", help="also time both arms with the whole step captured in a CUDA graph")
    ap.add_argument("--profile", action="store_true", help="print the engine arm's top CUDA kernels (torch profiler)")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    dt = torch.float16 if a.dtype == "fp16" else torch.bfloat16
    cfg = model_cfg(a.model)
    sd = model_ref.synth_state_dict(cfg, seed=0)
    img = torch.randint(0, 256, (a.batch, 3, a.size, a.size), dtype=torch.uint8, device=dev)
    targets = torch.from_numpy(loss_ref.synth_targets(a.batch, seed=1)).float().to(dev)

    m = DetectionModel(a.model)
    m.load_state_dict(sd)
    m = m.to(dev).train()
    m.hyp = dict(HYP_SCRATCH_LOW)
    loss_fn = ComputeLoss(m)
    opt = torch.optim.SGD(m.parameters(), lr=1e-4, momentum=0.937, nesterov=True, foreach=True)

    def step_engine():
        with torch.autocast("cuda", dtype=dt):
            p = m(img)
        loss, _ = loss_fn(p, targets)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()

    def fwd_engine():
        with torch.autocast("cuda", dtype=dt), torch.no_grad():
            m(img)

    t_step = timed(step_engine, a.steps)
    t_fwd = float("nan") if a.train_only else timed(fwd_engine, a.steps)
    print(f"engine   {a.model} bs{a.batch} {a.size} {a.dtype}: step {t_step:.2f} ms ({a.batch / t_step * 1e3:.0f} img/s), forward only {t_fwd:.2f} ms")
    if a.graph:
        t_g = graphed(step_engine, a.steps)
        print(f"engine   whole step in a CUDA graph: {t_g:.2f} ms ({a.batch / t_g * 1e3:.0f} img/s)")
    if a.profile:
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
            for _ in range(3):
                step_engine()
            torch.cuda.synchronize()
        print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=25, max_name_column_width=60))
        t0 = time.perf_counter()
        for _ in range(3):
            step_engine()
        host = (time.perf_counter() - t0) / 3 * 1e3
        torch.cuda.synchronize()
        print(f"host-side issue time per step: {host:.2f} ms")
    if a.skip_reference:
        return
    # reference arm: the same expressions through torch (NCHW, cuDNN, autocast), same loss kernel, same optimizer
    params = {k: (torch.nn.Parameter(v.to(dev)) if v.is_floating_point() and "running" not in k and "anchors" not in k else v.to(dev))
              for k, v in sd.items()}
    opt_r = torch.optim.SGD([p for p in params.values() if isinstance(p, torch.nn.Parameter)], lr=1e-4, momentum=0.937, nesterov=True, foreach=True)

    def step_ref():
        x = img.to(dt) / 255
        with torch.autocast("cuda", dtype=dt):
            p = model_ref.forward(cfg, params, x, training=True, bn_batch_stats=True)
        loss, _ = loss_fn(p, targets)
        opt_r.zero_grad(set_to_none=True)
        loss.backward()
        opt_r.step()

    if a.graph:
        t_rg = graphed(step_ref, a.steps)
        print(f"torch AMP whole step in a CUDA graph: {t_rg:.2f} ms ({a.batch / t_rg * 1e3:.0f} img/s)   engine/torch = {t_rg / t_g:.2f}x")
    t_ref = timed(step_ref, a.steps)
    print(f"torch AMP {a.model} bs{a.batch} {a.size} {a.dtype}: step {t_ref:.2f} ms ({a.batch / t_ref * 1e3:.0f} img/s)   engine/torch = {t_ref / t_step:.2f}x")


if __name__ == "__main__":
    main()
