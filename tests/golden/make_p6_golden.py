"""Generate the P6 fixtures in tests/golden/ by running the UNMODIFIED reference (/root/reference) through refshim.

Runs only in the build container (the GPU box has no /root/reference):
    python tests/golden/make_p6_golden.py

  p6_golden.npz    for each of models/hub/yolov5{n,s,m,l,x}6.yaml (prefix "<size>:"): the YAML's digest, the FULL-size reference
                   model's parameter count, state_dict keys with their shapes, Detect strides and (reordered, scaled) anchors.
                   For a reduced yolov5s6 (width 1/16 with channel_multiple 16, so every channel count, C3 hidden widths included,
                   stays a multiple of 8; depth 1/3; nc 3): its fp32 eval forward (z and the four raw maps) and its fp32 TTA
                   forward (augment=True) on a seeded 128x192 image, and one training step with the checkpoint's weights
                   (batch-statistics BN, ComputeLoss with hyp.scratch-low, fp32) on seeded uint8 images: the targets, the loss,
                   its items and every parameter's gradient
  ref_p6_tiny.pt   that reduced model's checkpoint pickled BY THE REFERENCE, as train.py writes them (BatchNorm statistics made
                   non-trivial)

The training targets are COCO128-shaped labels plus one large box per image: synthetic labels alone never reach the P6 anchors
(436-925 pixels) at a 256-pixel training size, and the fourth level's loss and gradients are what this fixture is for.
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
SIZES = "nsmlx"
X_SHAPE, X_SEED = (1, 3, 128, 192), 601
TRAIN_SHAPE, TRAIN_SEED, TARGET_SEED = (4, 3, 256, 256), 602, 603


def ref_cfg(size: str) -> dict:
    with open(f"{REF}/models/hub/yolov5{size}6.yaml", encoding="ascii", errors="ignore") as f:
        return yaml.safe_load(f)


def small_cfg() -> dict:
    cfg = ref_cfg("s")
    cfg.update(nc=3, depth_multiple=0.33, width_multiple=0.0625, channel_multiple=16)
    return cfg


def train_targets() -> np.ndarray:
    """synth_targets plus one box of 0.55-0.9 x 0.6-0.95 of the image per image (matches the P6 anchors)."""
    tg = synth_targets(TRAIN_SHAPE[0], seed=TARGET_SEED, nc=3)
    rs = np.random.RandomState(TARGET_SEED + 1)
    n = TRAIN_SHAPE[0]
    big = np.stack([np.arange(n), rs.randint(0, 3, n), rs.uniform(0.45, 0.55, n), rs.uniform(0.45, 0.55, n),
                    rs.uniform(0.55, 0.9, n), rs.uniform(0.6, 0.95, n)], 1)
    return np.concatenate((tg, big), 0).astype(np.float32)


def full_model_data(store: dict) -> None:
    from models.yolo import DetectionModel

    for s in SIZES:
        full = DetectionModel(ref_cfg(s))
        det = full.model[-1]
        store[f"{s}:digest"] = np.array(cfg_digest(ref_cfg(s)))
        store[f"{s}:n_params"] = np.array(sum(p.numel() for p in full.parameters()))
        store[f"{s}:keys"] = np.array(json.dumps([[k, list(v.shape)] for k, v in full.state_dict().items()]))
        store[f"{s}:stride"], store[f"{s}:anchors"] = det.stride.numpy(), det.anchors.numpy()
        print(f"yolov5{s}6: {int(store[f'{s}:n_params'])} parameters, strides {det.stride.tolist()}")
        del full


def small_model_data(store: dict) -> None:
    from models.yolo import DetectionModel
    from utils.loss import ComputeLoss

    cfg = small_cfg()
    torch.manual_seed(611)
    m = DetectionModel(deepcopy(cfg), ch=3)
    g = torch.Generator().manual_seed(612)
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
    torch.save({"epoch": -1, "best_fitness": None, "model": deepcopy(m).half(), "ema": None, "updates": 0, "optimizer": None, "opt": {},
                "date": "fixture"}, f"{HERE}/ref_p6_tiny.pt")
    em = deepcopy(m).half().float().eval()  # the checkpoint's fp16-rounded weights, as the tests load them
    x = synth_image(X_SHAPE, X_SEED)
    with torch.no_grad():
        z, raws = em(x)
        store["z_aug"] = em(x, augment=True)[0].numpy()
    store["z"] = z.numpy()
    for i, r in enumerate(raws):
        store[f"raw{i}"] = r.numpy()
    tm = deepcopy(m).half().float().train()
    tm.hyp = dict(HYP_SCRATCH_LOW)
    targets = train_targets()
    imgs = torch.from_numpy(np.random.RandomState(TRAIN_SEED).randint(0, 256, TRAIN_SHAPE).astype(np.uint8))
    pred = tm(imgs.float() / 255)
    loss, items = ComputeLoss(tm)(pred, torch.from_numpy(targets))
    loss.backward()
    store["train_shape"], store["train_seed"], store["targets"] = np.array(TRAIN_SHAPE), np.array(TRAIN_SEED), targets
    store["loss"], store["items"] = loss.detach().numpy(), items.numpy()
    for k, p in tm.named_parameters():
        store[f"grad:{k}"] = p.grad.numpy()
    print(f"small model: {sum(p.numel() for p in m.parameters())} parameters, checkpoint "
          f"{os.path.getsize(f'{HERE}/ref_p6_tiny.pt') / 1e6:.2f} MB, z {tuple(z.shape)}, loss {float(loss):.5f}")


if __name__ == "__main__":
    out = {}
    full_model_data(out)
    small_model_data(out)
    np.savez_compressed(f"{HERE}/p6_golden.npz", **out)
    print(f"p6_golden.npz {os.path.getsize(f'{HERE}/p6_golden.npz') / 1e6:.2f} MB")
