"""Generate the YOLOv3 fixtures in tests/golden/ by running the UNMODIFIED reference (/root/reference) through refshim.

Runs only in the build container (the GPU box has no /root/reference):
    python tests/golden/make_yolov3_golden.py

For each of models/hub/yolov3.yaml, yolov3-spp.yaml and yolov3-tiny.yaml, at the reduced scale of small_cfg (width 1/16 with
channel_multiple 16, so every channel count, Bottleneck hidden widths included, stays a multiple of 8; depth 1/3; nc 3):
  ref_<name>_tiny.pt   a checkpoint pickled BY THE REFERENCE, as train.py writes them (BatchNorm statistics made non-trivial)
  <name>_golden.npz    the YAML's digest; the parameter count and state_dict keys of the FULL-size reference model; its Detect
                       strides and (reordered, scaled) anchors; the small model's fp32 eval forward (z and raw maps) on a seeded
                       96x128 image; and, for yolov3-spp and yolov3-tiny, one training step of the small model with the checkpoint's weights (batch-statistics
                       BN, ComputeLoss with hyp.scratch-low, fp32) on seeded uint8 images and labels: the loss, its items and
                       every parameter's gradient

Only inputs derived from seeds go in; no existing fixture is touched.
"""
from __future__ import annotations

import json
import os
import sys
from copy import deepcopy

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import refshim  # noqa: E402

refshim.install()

import torch  # noqa: E402
import yaml  # noqa: E402

from make_golden import cfg_digest, synth_image  # noqa: E402
from oracle.loss_ref import synth_targets  # noqa: E402
from yolov5_b200.cfg import HYP_SCRATCH_LOW  # noqa: E402

torch.set_num_threads(8)
REF = refshim.REFERENCE_ROOT
NAMES = ("yolov3", "yolov3-spp", "yolov3-tiny")
TRAINED = ("yolov3-spp", "yolov3-tiny")
X_SHAPE, X_SEED = (1, 3, 96, 128), 301
TRAIN_SHAPE, TRAIN_SEED, TARGET_SEED = (4, 3, 128, 128), 302, 303


def ref_cfg(name: str) -> dict:
    with open(f"{REF}/models/hub/{name}.yaml", encoding="ascii", errors="ignore") as f:
        return yaml.safe_load(f)


def small_cfg(name: str) -> dict:
    """The same topology, narrow and shallow enough to commit as a pickled checkpoint."""
    cfg = ref_cfg(name)
    cfg.update(nc=3, depth_multiple=0.33, width_multiple=0.0625, channel_multiple=16)
    return cfg


def train_images() -> torch.Tensor:
    return torch.from_numpy(np.random.RandomState(TRAIN_SEED).randint(0, 256, TRAIN_SHAPE).astype(np.uint8))


def gen(name: str) -> None:
    from models.yolo import DetectionModel
    from utils.loss import ComputeLoss

    full = DetectionModel(ref_cfg(name))
    det = full.model[-1]
    store = {"digest": np.array(cfg_digest(ref_cfg(name))), "n_params": np.array(sum(p.numel() for p in full.parameters())),
             "keys": np.array(json.dumps(list(full.state_dict().keys()))), "stride": det.stride.numpy(), "anchors": det.anchors.numpy()}
    del full
    cfg = small_cfg(name)
    torch.manual_seed(311)
    m = DetectionModel(deepcopy(cfg), ch=3)
    g = torch.Generator().manual_seed(312)
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.weight.data = torch.rand(mod.weight.shape, generator=g) + 0.5
            mod.bias.data = torch.randn(mod.bias.shape, generator=g) * 0.1
            mod.running_mean = torch.randn(mod.running_mean.shape, generator=g) * 0.1
            mod.running_var = torch.rand(mod.running_var.shape, generator=g) + 0.5
    m.names = {0: "a", 1: "b", 2: "c"}
    store["small_cfg"] = np.array(json.dumps(cfg))
    store["small_keys"] = np.array(json.dumps(list(m.state_dict().keys())))
    store["x_shape"], store["x_seed"] = np.array(X_SHAPE), np.array(X_SEED)
    m.eval()
    with torch.no_grad():
        z, raws = m(synth_image(X_SHAPE, X_SEED))
    store["z"] = z.numpy()
    for i, r in enumerate(raws):
        store[f"raw{i}"] = r.numpy()
    torch.save({"epoch": -1, "best_fitness": None, "model": deepcopy(m).half(), "ema": None, "updates": 0, "optimizer": None, "opt": {},
                "date": "fixture"}, f"{HERE}/ref_{name}_tiny.pt")
    if name in TRAINED:
        tm = deepcopy(m).half().float().train()  # the checkpoint's fp16-rounded weights
        tm.hyp = dict(HYP_SCRATCH_LOW)
        targets = torch.from_numpy(synth_targets(TRAIN_SHAPE[0], seed=TARGET_SEED, nc=3))
        pred = tm(train_images().float() / 255)
        loss, items = ComputeLoss(tm)(pred, targets)
        loss.backward()
        store["train_shape"], store["train_seeds"] = np.array(TRAIN_SHAPE), np.array([TRAIN_SEED, TARGET_SEED])
        store["loss"], store["items"] = loss.detach().numpy(), items.numpy()
        for k, p in tm.named_parameters():
            store[f"grad:{k}"] = p.grad.numpy()
    np.savez_compressed(f"{HERE}/{name.replace('-', '_')}_golden.npz", **store)
    print(f"{name}: {int(store['n_params'])} parameters, small model {sum(p.numel() for p in m.parameters())}, "
          f"checkpoint {os.path.getsize(f'{HERE}/ref_{name}_tiny.pt') / 1e6:.2f} MB, strides {store['stride'].tolist()}")


if __name__ == "__main__":
    for n in NAMES:
        gen(n)
