"""Timing of the step after backward with `--optimizer Adam | AdamW` on yolov5m's parameter set (21.2 M fp32 parameters plus
the BN buffers the EMA tracks), seeded gradients, on the GPU:

  fused      FusedAdam / FusedAdamW.fused_step(scaler, 10.0, ema, model): y5_adam_step, three launches
  reference  train.py:413-421 on the same GPU: torch.optim.Adam / AdamW (foreach, torch's CUDA default) in the reference's
             three groups, scaler.unscale_, clip_grad_norm_, scaler.step, scaler.update and the reference's ModelEMA.update loop
  sgd        FusedSGD.fused_step (y5_opt_step), for context

    python tools/optim_bench.py [--optimizer AdamW] [--min-seconds 1.0]

Prints one JSON line: the GPU and its power limit, ms per step of each arm, and the largest weight difference between fused
and reference after one step from the same state (they must agree to rtol 1e-5).  CUDA-event timing after warm-up, each timed
window at least --min-seconds long.  The reference arm also copies the saved gradients back after each step (one 85 MB
copy, where train.py would run the next backward).  The fused step's algorithmic traffic is 36 B per parameter (read g, p, exp_avg,
exp_avg_sq, ema; write p, exp_avg, exp_avg_sq, ema) plus 4 B of the gradient-norm pass.
"""
import argparse
import json
import os
import subprocess
import sys
from copy import deepcopy

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from yolov5_b200.models.yolo import DetectionModel  # noqa: E402
from yolov5_b200.utils.torch_utils import ModelEMA, smart_optimizer  # noqa: E402


def gpu_name():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def torch_optimizer(model, name, lr, momentum, decay):
    """The reference's smart_optimizer groups on torch.optim.Adam / AdamW."""
    g = [], [], []
    for v in model.modules():
        for p_name, p in v.named_parameters(recurse=False):
            if p_name == "bias":
                g[2].append(p)
            elif p_name == "weight" and isinstance(v, torch.nn.BatchNorm2d):
                g[1].append(p)
            else:
                g[0].append(p)
    if name == "Adam":
        opt = torch.optim.Adam(g[2], lr=lr, betas=(momentum, 0.999))
    else:
        opt = torch.optim.AdamW(g[2], lr=lr, betas=(momentum, 0.999), weight_decay=0.0)
    opt.add_param_group({"params": g[0], "weight_decay": decay})
    opt.add_param_group({"params": g[1], "weight_decay": 0.0})
    return opt


def reference_ema_update(ema, model):
    """The reference's ModelEMA.update (utils/torch_utils.py:359-368)."""
    ema.updates += 1
    d = ema.decay(ema.updates)
    msd = model.state_dict()
    for k, v in ema.ema.state_dict().items():
        if v.dtype.is_floating_point:
            v *= d
            v += (1 - d) * msd[k].detach()


def time_ms(fn, min_seconds):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    n, total = 4, 0.0
    while True:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n):
            fn()
        b.record()
        b.synchronize()
        total = a.elapsed_time(b)
        if total >= 1000 * min_seconds:
            return total / n
        n *= 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--optimizer", default="AdamW", choices=["Adam", "AdamW"])
    ap.add_argument("--min-seconds", type=float, default=1.0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("optim_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    base = DetectionModel("yolov5m").to(dev).train()
    n_params = sum(p.numel() for p in base.parameters())
    grads = [torch.randn_like(p) * 1024.0 for p in base.parameters()]  # as a scaled backward leaves them (scale 1024)

    def setup(kind):
        m = deepcopy(base)
        opt = (torch_optimizer(m, args.optimizer, 0.001, 0.937, 5e-4) if kind == "reference"
               else smart_optimizer(m, "SGD" if kind == "sgd" else args.optimizer, 0.001, 0.937, 5e-4))
        scaler = torch.amp.GradScaler("cuda", init_scale=1024.0, growth_interval=10**9)
        scaler.scale(torch.zeros(1, device=dev))
        for p, g in zip(m.parameters(), grads):
            p.grad = g.clone()
        return m, opt, scaler, ModelEMA(m)

    def fused_step(m, opt, scaler, ema):
        return lambda: opt.fused_step(scaler=scaler, max_norm=10.0, ema=ema, model=m)

    def reference_step(m, opt, scaler, ema):
        ps = list(m.parameters())
        saved = [p.grad.clone() for p in ps]

        def step():
            scaler.unscale_(opt)
            torch.nn.utils.clip_grad_norm_(ps, max_norm=10.0)
            scaler.step(opt)
            scaler.update()
            reference_ema_update(ema, m)
            for p, g in zip(ps, saved):  # train.py zeroes the gradients; keep the same ones for the next timed step
                p.grad.copy_(g)
        return step

    # agreement after one step from the same state
    fa, ra = setup("fused"), setup("reference")
    fused_step(*fa)()
    reference_step(*ra)()
    worst = 0.0
    for a, b in zip(fa[0].parameters(), ra[0].parameters()):
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-7), float((a - b).abs().max())
        worst = max(worst, float((a - b).abs().max()))
    del fa, ra
    torch.cuda.empty_cache()

    out = {"gpu": gpu_name(), "optimizer": args.optimizer, "params": n_params}
    for kind, make in (("fused", fused_step), ("reference", reference_step), ("sgd", fused_step)):
        state = setup(kind)
        out[f"{kind}_ms"] = round(time_ms(make(*state), args.min_seconds), 4)
        del state
        torch.cuda.empty_cache()
    out["fused_algorithmic_GB"] = round(40 * n_params / 1e9, 3)
    out["fused_GBps"] = round(40 * n_params / 1e9 / (out["fused_ms"] / 1e3), 1)
    out["max_abs_weight_diff_after_one_step"] = worst
    out["speedup_vs_reference"] = round(out["reference_ms"] / out["fused_ms"], 2)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
