"""Timing of YOLOv5 classification (yolov5s-cls: the yolov5s backbone cut at layer 10 + Classify, nc = 1000) on one GPU:

  eval   classify/val.py's default batch: 128 x 3 x 224 x 224 fp16 images into model.half()
         engine     ClassificationModel.forward (one CUDA-graph replay of conv_gemm / pool kernels + a fresh logits tensor)
         torch      the same expressions (oracle/cls_ref.py on oracle/model_ref.py's building blocks, BN folded) in fp16 on torch-cuda
  train  classify/train.py's defaults: 64 x 224 x 224, fp16 AMP, CE(label_smoothing=0.1), Adam(lr 1e-3, betas (0.9, 0.999)) in the
         reference's three groups, GradScaler, clip_grad_norm_(10), ModelEMA
         engine     autocast forward (train_ops), y5_cross_entropy, scaled backward, FusedAdam.fused_step(scaler, 10.0, ema, model)
         torch      the oracle expressions under autocast with batch-statistics BN, nn.CrossEntropyLoss, GradScaler,
                    torch.optim.Adam (foreach), clip_grad_norm_ and a per-tensor EMA loop (reference utils/torch_utils.py:359-368)

    python tools/cls_bench.py [--min-seconds 1.0]

Prints one JSON line: the GPU and its power limit, ms per call of each arm and images/s.  CUDA-event timing after warm-up, each
timed window at least --min-seconds long.  The torch arms run with torch's defaults (cuDNN picks its algorithms, TF32 allowed).
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import cls_ref  # noqa: E402
from yolov5_b200.cfg import model_cfg  # noqa: E402
from yolov5_b200.models.yolo import ClassificationModel, DetectionModel  # noqa: E402
from yolov5_b200.utils.torch_utils import ModelEMA, smart_optimizer, smartCrossEntropyLoss  # noqa: E402


def gpu_name():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def fold_state_dict(sd):
    """state_dict with every conv's BatchNorm folded into conv weight + bias (a fused model's state_dict)."""
    from oracle import model_ref

    out = {k: v for k, v in sd.items() if ".bn." not in k}
    for k in sd:
        if k.endswith(".bn.weight"):
            p = k[: -len(".bn.weight")]
            eps = cls_ref.HEAD_BN_EPS if p.endswith(".conv") and f"{p[: -len('.conv')]}.linear.weight" in sd else model_ref.BN_EPS
            out[f"{p}.conv.weight"], out[f"{p}.conv.bias"] = model_ref.fold_bn(
                sd[f"{p}.conv.weight"], *(sd[f"{p}.bn.{q}"] for q in ("weight", "bias", "running_mean", "running_var")), eps=eps)
    return out


def time_ms(fn, min_seconds):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    n = 2
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
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--eval-batch", type=int, default=128)
    ap.add_argument("--train-batch", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("cls_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    cfg = model_cfg("yolov5s")
    sd = cls_ref.synth_state_dict(cfg, 1000, seed=0)
    g = torch.Generator().manual_seed(1)
    out = {"gpu": gpu_name(), "model": "yolov5s-cls", "nc": 1000}

    # ---------------------------------------------------------------- eval
    x = torch.rand(args.eval_batch, 3, 224, 224, generator=g).to(dev, torch.float16)
    m = ClassificationModel(model=DetectionModel("yolov5s"), nc=1000)
    m.load_state_dict(sd)
    m = m.to(dev).half().eval()
    sd_h = {k: v.to(dev, torch.float16) for k, v in fold_state_dict(sd).items()}  # BN folded once, like model.fuse().half()
    with torch.no_grad():
        y_e, y_t = m(x), cls_ref.forward(cfg, sd_h, x)
        out["eval_max_abs_logit_diff"] = round(float((y_e.float() - y_t.float()).abs().max()), 4)
        out["eval_engine_ms"] = round(time_ms(lambda: m(x), args.min_seconds), 3)
        out["eval_torch_ms"] = round(time_ms(lambda: cls_ref.forward(cfg, sd_h, x), args.min_seconds), 3)
    out["eval_batch"] = args.eval_batch
    out["eval_engine_img_per_s"] = round(args.eval_batch / out["eval_engine_ms"] * 1e3)
    out["eval_torch_img_per_s"] = round(args.eval_batch / out["eval_torch_ms"] * 1e3)
    del m, sd_h, x, y_e, y_t
    torch.cuda.empty_cache()

    # ---------------------------------------------------------------- train
    xt = torch.rand(args.train_batch, 3, 224, 224, generator=g).to(dev)
    lab = torch.randint(0, 1000, (args.train_batch,), generator=g).to(dev)

    mt = ClassificationModel(model=DetectionModel("yolov5s"), nc=1000)
    mt.load_state_dict(sd)
    mt = mt.to(dev).train()
    opt = smart_optimizer(mt, "Adam", 1e-3, 0.9, 5e-5)
    ema = ModelEMA(mt)
    scaler = torch.amp.GradScaler("cuda")
    crit = smartCrossEntropyLoss(label_smoothing=0.1)

    def engine_step():
        with torch.autocast("cuda"):
            loss = crit(mt(xt), lab)
        scaler.scale(loss).backward()
        opt.fused_step(scaler, 10.0, ema, mt)
        opt.zero_grad(set_to_none=True)

    params = {k: v.to(dev).clone().requires_grad_(v.is_floating_point() and "running" not in k) for k, v in sd.items()}
    leaves = [v for v in params.values() if v.requires_grad]
    groups = ([v for k, v in params.items() if v.requires_grad and k.endswith(".bias")],
              [v for k, v in params.items() if v.requires_grad and ".bn.weight" in k],
              [v for k, v in params.items() if v.requires_grad and not k.endswith(".bias") and ".bn.weight" not in k])
    topt = torch.optim.Adam(groups[0], lr=1e-3, betas=(0.9, 0.999), foreach=True)
    topt.add_param_group({"params": groups[2], "weight_decay": 5e-5})
    topt.add_param_group({"params": groups[1], "weight_decay": 0.0})
    tema = {k: v.detach().clone() for k, v in params.items() if v.is_floating_point()}
    tscaler = torch.amp.GradScaler("cuda")
    tcrit = torch.nn.CrossEntropyLoss(label_smoothing=0.1)
    tcount = [0]

    def torch_step():
        with torch.autocast("cuda"):
            loss = tcrit(cls_ref.forward(cfg, params, xt, bn_batch_stats=True), lab)
        tscaler.scale(loss).backward()
        tscaler.unscale_(topt)
        torch.nn.utils.clip_grad_norm_(leaves, max_norm=10.0)
        tscaler.step(topt)
        tscaler.update()
        topt.zero_grad()
        tcount[0] += 1
        d = 0.9999 * (1 - torch.e ** (-tcount[0] / 2000))
        with torch.no_grad():
            for k, v in tema.items():
                v *= d
                v += (1 - d) * params[k].detach()

    out["train_batch"] = args.train_batch
    out["train_engine_ms"] = round(time_ms(engine_step, args.min_seconds), 3)
    out["train_torch_ms"] = round(time_ms(torch_step, args.min_seconds), 3)
    out["train_engine_img_per_s"] = round(args.train_batch / out["train_engine_ms"] * 1e3)
    out["train_torch_img_per_s"] = round(args.train_batch / out["train_torch_ms"] * 1e3)
    out["eval_speedup"] = round(out["eval_torch_ms"] / out["eval_engine_ms"], 2)
    out["train_speedup"] = round(out["train_torch_ms"] / out["train_engine_ms"], 2)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
