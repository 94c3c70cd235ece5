"""Generate the C3TR fixtures in tests/golden/ by running the UNMODIFIED reference (/root/reference) through refshim.

Runs only in the build container (the GPU box has no /root/reference):
    python tests/golden/make_transformer_golden.py

  transformer_forward_w50.npz, transformer_forward_w25.npz
                             the reference's models/hub/yolov5s-transformer.yaml at width 0.5 (head dim 64) and 0.25 (head dim
                             32), one file per width: its fused eval forward (z and the raw head maps) on
                             oracle/transformer_ref.synth_state_dict weights and a seeded 96x128 image, the state_dict key list
                             and the YAML's digest; the oracle (oracle/transformer_ref.py) is checked against every output while
                             generating (hard assert)
  ref_transformer_tiny.pt    a checkpoint pickled BY THE REFERENCE with a C3TR (tiny_transformer_cfg: narrow layers around a
                             C3TR of 128 channels, four heads of 32), as train.py writes them, and
  ref_transformer_tiny_forward.npz  its eval forward on a seeded image

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
from oracle import transformer_ref  # noqa: E402
from yolov5_b200.cfg import model_cfg  # noqa: E402

torch.set_num_threads(8)
REF = refshim.REFERENCE_ROOT
SHAPE, SEED_W, SEED_X = (1, 3, 96, 128), 40, 140
WIDTHS = (0.5, 0.25)


def transformer_cfg() -> dict:
    with open(f"{REF}/models/hub/yolov5s-transformer.yaml", encoding="ascii", errors="ignore") as f:
        return yaml.safe_load(f)


def gen_forward():
    from models.yolo import DetectionModel

    base = transformer_cfg()
    x = synth_image(SHAPE, SEED_X)
    for wm in WIDTHS:
        store = {"shape": np.array(SHAPE), "seed": np.array([SEED_W, SEED_X]), "width": np.array(wm), "digest": np.array(cfg_digest(base))}
        cfg = deepcopy(base)
        cfg["width_multiple"] = wm
        sd = transformer_ref.synth_state_dict(cfg, seed=SEED_W)
        m = DetectionModel(deepcopy(cfg))
        assert list(m.state_dict().keys()) == list(sd.keys())
        r = m.load_state_dict(sd, strict=True)
        assert not r.missing_keys and not r.unexpected_keys
        m = m.eval().fuse()
        sd64 = {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}
        with torch.no_grad():
            z_r, raw_r = m(x)
            z_o, raw_o = transformer_ref.forward(cfg, sd64, x.double(), fused=True)
        d = (z_r.double() - z_o).abs().max().item()
        print(f"yolov5s-transformer width {wm}: z max|ref-oracle| = {d:.3e}  (|z|max {z_r.abs().max():.1f})")
        assert torch.allclose(z_r.double(), z_o, rtol=1e-4, atol=1e-4), (wm, d)
        for a, b in zip(raw_r, raw_o):
            assert torch.allclose(a.double(), b, rtol=1e-4, atol=1e-4)
        store["z"] = z_r.numpy()
        for l, a in enumerate(raw_r):
            store[f"raw{l}"] = a.numpy()
        store["keys"] = np.array(json.dumps(list(sd.keys())))
        np.savez_compressed(f"{HERE}/transformer_forward_w{int(wm * 100)}.npz", **store)


def tiny_transformer_cfg() -> dict:
    """yolov5 v6 topology with narrow layers (as make_golden.tiny_cfg, narrower still) and layer 8 a C3TR(128, e=1.0): c_ = 128,
    four heads of 32, the smallest head dim the kernels take.  Small enough to commit as a pickled checkpoint."""
    cfg = json.loads(json.dumps(model_cfg("yolov5s")))
    cm = {64: 16, 128: 16, 256: 16, 512: 32, 1024: 32}
    for part in ("backbone", "head"):
        for row in cfg[part]:
            if row[2] in ("Conv", "C3", "SPPF") and isinstance(row[3][0], int):
                row[3][0] = cm[row[3][0]]
    cfg.update(nc=3, depth_multiple=0.33, width_multiple=1.0)
    cfg["backbone"][8] = [-1, 3, "C3TR", [128, True, 1, 1.0]]  # args [c2, shortcut, g, e], as the reference's parse_model reads them
    return cfg


def gen_ckpt():
    from models.yolo import DetectionModel

    cfg = tiny_transformer_cfg()
    torch.manual_seed(9)
    m = DetectionModel(cfg, ch=3)
    g = torch.Generator().manual_seed(10)
    for mod in m.modules():  # non-trivial BatchNorm statistics and attention biases
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.weight.data = torch.rand(mod.weight.shape, generator=g) + 0.5
            mod.bias.data = torch.randn(mod.bias.shape, generator=g) * 0.1
            mod.running_mean = torch.randn(mod.running_mean.shape, generator=g) * 0.1
            mod.running_var = torch.rand(mod.running_var.shape, generator=g) + 0.5
        elif isinstance(mod, torch.nn.MultiheadAttention):
            mod.in_proj_bias.data = torch.randn(mod.in_proj_bias.shape, generator=g) * 0.1
            mod.out_proj.bias.data = torch.randn(mod.out_proj.bias.shape, generator=g) * 0.1
    m.names = {0: "a", 1: "b", 2: "c"}
    m.eval()
    x = synth_image((1, 3, 64, 96), 11)
    with torch.no_grad():
        z = m(x)[0].numpy()
    torch.save({"epoch": -1, "best_fitness": None, "model": deepcopy(m).half(), "ema": None, "updates": 0, "optimizer": None, "opt": {},
                "date": "fixture"}, f"{HERE}/ref_transformer_tiny.pt")
    np.savez_compressed(f"{HERE}/ref_transformer_tiny_forward.npz", z=z, keys=np.array(json.dumps(list(m.state_dict().keys()))),
                        cfg=np.array(json.dumps(cfg)))
    print(f"reference-pickled C3TR checkpoint: {sum(p.numel() for p in m.parameters())} parameters, "
          f"{os.path.getsize(f'{HERE}/ref_transformer_tiny.pt') / 1e6:.2f} MB")


if __name__ == "__main__":
    gen_forward()
    gen_ckpt()
