"""Generate the LeakyReLU fixtures in tests/golden/ by running the UNMODIFIED reference (/root/reference) through refshim.

Runs only in the build container (the GPU box has no /root/reference):
    python tests/golden/make_leaky_golden.py

  leaky_forward.npz  the reference's models/hub/yolov5s-LeakyReLU.yaml (`activation: nn.LeakyReLU(0.1)`) scaled to yolov5n
                     (width_multiple 0.25): its fused eval forward (z and the raw head maps) on model_ref.synth_state_dict weights
                     and a seeded image, as make_golden.py's model fixture; the oracle (oracle/model_ref.py run with the model
                     dict's activation by tests/act_ref.py) is checked against it while generating (hard assert)
  ref_leaky_tiny.pt  a checkpoint pickled BY THE REFERENCE whose Conv modules carry LeakyReLU(0.1), as train.py writes them, and
  ref_leaky_tiny_forward.npz  its eval forward on a seeded image

Only inputs derived from seeds go in; no existing fixture is touched.  The reference sets the class attribute
Conv.default_act while parsing such a model; it is restored to nn.SiLU() afterwards.
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

from make_golden import synth_image, tiny_cfg  # noqa: E402
from oracle import model_ref  # noqa: E402
from tests.act_ref import forward as oracle_forward  # noqa: E402

torch.set_num_threads(8)
REF = refshim.REFERENCE_ROOT
SHAPE, SEED_W, SEED_X = (2, 3, 96, 128), 30, 130


def leaky_cfg() -> dict:
    """models/hub/yolov5s-LeakyReLU.yaml with yolov5n's width multiple (depth 0.33 is already yolov5n's)."""
    with open(f"{REF}/models/hub/yolov5s-LeakyReLU.yaml", encoding="ascii", errors="ignore") as f:
        cfg = yaml.safe_load(f)
    assert cfg["activation"] == "nn.LeakyReLU(0.1)" and cfg["depth_multiple"] == 0.33
    cfg["width_multiple"] = 0.25
    return cfg


def restore_default_act():
    from models.common import Conv

    Conv.default_act = torch.nn.SiLU()


def gen_forward():
    from models.yolo import DetectionModel

    cfg = leaky_cfg()
    sd = model_ref.synth_state_dict(cfg, seed=SEED_W)
    try:
        m = DetectionModel(deepcopy(cfg))
        mf = DetectionModel(deepcopy(cfg))
    finally:
        restore_default_act()
    acts = {type(c.act) for c in m.modules() if type(c).__name__ == "Conv"}
    assert acts == {torch.nn.LeakyReLU}, acts
    for mm in (m, mf):
        r = mm.load_state_dict(sd, strict=True)
        assert not r.missing_keys and not r.unexpected_keys
        mm.eval()
    mf = mf.fuse()
    x = synth_image(SHAPE, SEED_X)
    store = {}
    with torch.no_grad():
        for tag, mm, fused in (("bn", m, False), ("fused", mf, True)):
            z_r, raw_r = mm(x)
            z_o, raw_o = oracle_forward(cfg, sd, x, fused=fused)
            d = (z_r - z_o).abs().max().item()
            print(f"yolov5n-LeakyReLU {tag}: z max|ref-oracle| = {d:.3e}  (|z|max {z_r.abs().max():.1f})")
            assert torch.allclose(z_r, z_o, rtol=1e-4, atol=1e-4), (tag, d)
            for a, b in zip(raw_r, raw_o):
                assert torch.allclose(a, b, rtol=1e-4, atol=1e-4)
            if fused:  # the engine's form; the BatchNorm form is only checked against the oracle
                store["z"] = z_r.numpy()
                for l, a in enumerate(raw_r):
                    store[f"raw{l}"] = a.numpy()
    store["shape"] = np.array(SHAPE)
    store["seed"] = np.array([SEED_W, SEED_X])
    store["cfg"] = np.array(json.dumps(cfg))
    np.savez_compressed(f"{HERE}/leaky_forward.npz", **store)


def gen_ckpt():
    """As make_golden.gen_ckpt, with `activation: nn.LeakyReLU(0.1)` in the model dict."""
    from models.yolo import DetectionModel

    cfg = tiny_cfg()
    cfg["activation"] = "nn.LeakyReLU(0.1)"
    torch.manual_seed(6)
    try:
        m = DetectionModel(cfg, ch=3)
    finally:
        restore_default_act()
    g = torch.Generator().manual_seed(7)
    for mod in m.modules():  # non-trivial BatchNorm statistics so the fold matters
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.weight.data = torch.rand(mod.weight.shape, generator=g) + 0.5
            mod.bias.data = torch.randn(mod.bias.shape, generator=g) * 0.1
            mod.running_mean = torch.randn(mod.running_mean.shape, generator=g) * 0.1
            mod.running_var = torch.rand(mod.running_var.shape, generator=g) + 0.5
    m.names = {0: "a", 1: "b", 2: "c"}
    m.eval()
    x = synth_image((1, 3, 64, 96), 8)
    with torch.no_grad():
        z = m(x)[0].numpy()
    torch.save({"epoch": -1, "best_fitness": None, "model": deepcopy(m).half(), "ema": None, "updates": 0, "optimizer": None, "opt": {},
                "date": "fixture"}, f"{HERE}/ref_leaky_tiny.pt")
    np.savez_compressed(f"{HERE}/ref_leaky_tiny_forward.npz", z=z, keys=np.array(json.dumps(list(m.state_dict().keys()))),
                        cfg=np.array(json.dumps(cfg)))
    print(f"reference-pickled LeakyReLU checkpoint: {sum(p.numel() for p in m.parameters())} parameters, "
          f"{os.path.getsize(f'{HERE}/ref_leaky_tiny.pt') / 1e6:.2f} MB")


if __name__ == "__main__":
    gen_forward()
    gen_ckpt()
