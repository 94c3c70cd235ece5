"""Cost of --sync-bn: one eager smart_DDP training step on two GPUs, with BatchNorm and with SyncBatchNorm.

    torchrun --nproc-per-node 2 tools/syncbn_bench.py [--model yolov5m] [--batch 8] [--size 640] [--steps 20]

Three legs, each uint8 images resident on the GPU -> autocast fp16 forward -> ComputeLoss -> scaled backward (DDP's bucketed
gradient all-reduce) -> optimizer step:
  * engine, BatchNorm2d;
  * engine, torch.nn.SyncBatchNorm.convert_sync_batchnorm: two all-reduces per BN layer per step (79 layers in yolov5m);
  * the reference's expressions on torch-cuda (cuDNN convolutions, GradScaler) with torch's own SyncBatchNorm.
Rank 0 prints one JSON line: ms per step of each leg (CUDA events, after warm-up), the GPU and its power limit.
With fewer than two GPUs it says so and exits.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import loss_ref, model_ref  # reference leg only  # noqa: E402
from yolov5_b200.cfg import HYP_SCRATCH_LOW, model_cfg  # noqa: E402
from yolov5_b200.models.yolo import DetectionModel  # noqa: E402
from yolov5_b200.utils.loss import ComputeLoss  # noqa: E402
from yolov5_b200.utils.torch_utils import smart_DDP, smart_optimizer  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, steps, warmup):
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


class _SyncBNFunctional:
    """model_ref's `F` with batch_norm routed through one torch.nn.SyncBatchNorm per layer (keyed by its weight)"""

    def __init__(self, functional):
        self._f, self._bn = functional, {}

    def __getattr__(self, name):
        return getattr(self._f, name)

    def batch_norm(self, x, running_mean, running_var, weight, bias, training=False, eps=1e-5):
        bn = self._bn.get(id(weight))
        if bn is None:
            bn = self._bn[id(weight)] = nn.SyncBatchNorm(weight.numel(), eps=eps, momentum=0.03).to(weight.device)
            bn.weight, bn.bias = weight, bias
        return bn(x)


class _RefNet(nn.Module):
    """the reference's expressions (oracle/model_ref.py) over a state_dict of Parameters, as a module DDP can wrap"""

    def __init__(self, cfg, sd, dev):
        super().__init__()
        self.cfg, self.keys = cfg, list(sd)
        train = {k: v for k, v in sd.items() if v.is_floating_point() and "running" not in k and "anchors" not in k}
        self.p = nn.ParameterDict({k.replace(".", "__"): nn.Parameter(v.to(dev)) for k, v in train.items()})
        self.fixed = {k: v.to(dev) for k, v in sd.items() if k not in train}

    def forward(self, x):
        sd = {k: self.p[k.replace(".", "__")] if k.replace(".", "__") in self.p else self.fixed[k] for k in self.keys}
        return model_ref.forward(self.cfg, sd, x, training=True, bn_batch_stats=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="yolov5m")
    ap.add_argument("--batch", type=int, default=8, help="images per GPU")
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if torch.cuda.device_count() < 2 or int(os.environ.get("WORLD_SIZE", "1")) < 2:
        print("syncbn_bench: needs 2 GPUs (run with torchrun --nproc-per-node 2)")
        return
    import torch.distributed as dist

    rank = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", device_id=dev)
    cfg = model_cfg(a.model)
    sd = model_ref.synth_state_dict(cfg, seed=0)
    img = torch.randint(0, 256, (a.batch, 3, a.size, a.size), dtype=torch.uint8, device=dev)
    targets = torch.from_numpy(loss_ref.synth_targets(a.batch, seed=1 + rank)).float().to(dev)
    world = dist.get_world_size()
    out = {"gpu": gpu_info(), "model": a.model, "batch_per_gpu": a.batch, "size": a.size, "world": world, "dtype": "fp16"}

    for leg, sync in (("engine_bn_ms", False), ("engine_syncbn_ms", True)):
        m = DetectionModel(a.model)
        m.load_state_dict(sd)
        if sync:
            m = nn.SyncBatchNorm.convert_sync_batchnorm(m)
        m = m.to(dev).train()
        m.hyp = dict(HYP_SCRATCH_LOW)
        net, loss_fn = smart_DDP(m), ComputeLoss(m)
        opt = smart_optimizer(m, "SGD", lr=1e-4, momentum=0.937, decay=5e-4)
        scaler = torch.amp.GradScaler("cuda")

        def step():
            with torch.autocast("cuda", dtype=torch.float16):
                p = net(img)
            loss, _ = loss_fn(p, targets)
            scaler.scale(loss * world).backward()
            opt.fused_step(scaler=scaler, max_norm=10.0)
            opt.zero_grad(set_to_none=True)

        out[leg] = round(timed(step, a.steps, a.warmup), 3)
        del net, m, opt

    # reference leg: torch's own SyncBatchNorm inside the reference's expressions, cuDNN, GradScaler, torch SGD
    m = DetectionModel(a.model)
    m.load_state_dict(sd)
    m.hyp = dict(HYP_SCRATCH_LOW)
    loss_fn = ComputeLoss(m.to(dev))
    model_ref.F = _SyncBNFunctional(model_ref.F)
    ref = _RefNet(cfg, sd, dev)
    net = nn.parallel.DistributedDataParallel(ref, device_ids=[rank], output_device=rank)
    opt = torch.optim.SGD(ref.parameters(), lr=1e-4, momentum=0.937, nesterov=True, foreach=True)
    scaler = torch.amp.GradScaler("cuda")

    def step_ref():
        x = img.half() / 255
        with torch.autocast("cuda", dtype=torch.float16):
            p = net(x)
        loss, _ = loss_fn(p, targets)
        scaler.scale(loss * world).backward()
        scaler.unscale_(opt)
        torch.nn.utils.clip_grad_norm_(ref.parameters(), max_norm=10.0)
        scaler.step(opt)
        scaler.update()
        opt.zero_grad(set_to_none=True)

    out["reference_syncbn_ms"] = round(timed(step_ref, a.steps, a.warmup), 3)
    out["syncbn_over_bn"] = round(out["engine_syncbn_ms"] / out["engine_bn_ms"], 3)
    if rank == 0:
        print(json.dumps(out))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
