"""Generate tests/golden/wide_head.npz: the UNMODIFIED reference (/root/reference) with Detect / Segment heads wider than one
128-column N tile of the head GEMM.

    python tests/golden/make_wide_head_golden.py

Cases: yolov5n with nc = 365 (Objects365's class count, no = 370 outputs per anchor) and yolov5n-seg with nc = 100 (no = 137,
the 32 mask columns straddle the first 128), on oracle/model_ref.synth_state_dict weights with the hot head bias (the decoded
output holds NMS candidates) and a seeded image.  The reference is imported through refshim.py, as make_golden.py does; while
generating, oracle/model_ref.forward is checked against the reference output (hard assert), which pins the oracle at these
widths.  The fixture holds z samples and sums only.
"""
from __future__ import annotations

import copy
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import refshim  # noqa: E402

refshim.install()

import torch  # noqa: E402

from oracle import model_ref  # noqa: E402
from yolov5_b200.cfg import model_cfg  # noqa: E402

torch.set_num_threads(8)
REF = refshim.REFERENCE_ROOT

# name, nc, image shape, weight seed, image seed
CASES = [("yolov5n", 365, (1, 3, 128, 160), 40, 140), ("yolov5n-seg", 100, (1, 3, 128, 160), 41, 141)]
SAMPLE = 7  # every 7th z row is stored


def wide_cfg(name: str, nc: int) -> dict:
    cfg = copy.deepcopy(model_cfg(name))
    cfg["nc"] = nc
    return cfg


def synth_image(shape, seed):
    return torch.from_numpy(np.random.RandomState(seed).uniform(0, 1, shape).astype(np.float32))


def ref_model(name, nc, sd):
    from models.yolo import DetectionModel, SegmentationModel

    sub = "models/segment/" if name.endswith("-seg") else "models/"
    cls = SegmentationModel if name.endswith("-seg") else DetectionModel
    m = cls(f"{REF}/{sub}{name}.yaml", nc=nc)
    missing = m.load_state_dict(sd, strict=True)
    assert not missing.missing_keys and not missing.unexpected_keys
    return m.eval()


def main():
    store = {}
    for name, nc, shape, sw, sx in CASES:
        cfg = wide_cfg(name, nc)
        sd = model_ref.synth_state_dict(cfg, seed=sw, head_bias="hot")
        x = synth_image(shape, sx)
        seg = name.endswith("-seg")
        with torch.no_grad():
            m = ref_model(name, nc, sd)
            assert m.model[-1].no > 128, (name, m.model[-1].no)
            for tag, r, o in (("bn", m(x), model_ref.forward(cfg, sd, x)), ("fused", m.fuse()(x), model_ref.forward(cfg, sd, x, fused=True))):
                z_r, z_o = r[0], o[0]
                d = (z_r - z_o).abs().max().item()
                assert torch.allclose(z_r, z_o, rtol=1e-4, atol=1e-4), (name, tag, d)
                raw_r, raw_o = (r[2], o[2]) if seg else (r[1], o[1])
                for a, b in zip(raw_r, raw_o):
                    assert a.shape[-1] == 5 + nc + (32 if seg else 0)
                    assert torch.allclose(a, b, rtol=1e-4, atol=1e-4), (name, tag)
                if seg:
                    assert torch.allclose(r[1], o[1], rtol=1e-4, atol=1e-4), (name, tag, "proto")
                print(f"{name} nc={nc} {tag}: z {tuple(z_r.shape)} max|ref-oracle| = {d:.3e}; "
                      f"obj*cls > 0.25 rows: {int(((z_r[..., 4:5] * z_r[..., 5 : 5 + nc]).amax(-1) > 0.25).sum())}")
        store[f"{name}.z_sample"] = z_r[:, ::SAMPLE].numpy()
        store[f"{name}.z_sum"] = np.array([z_r.double().sum().item(), z_r.double().abs().sum().item()])
        store[f"{name}.z_shape"] = np.array(z_r.shape)
        store[f"{name}.case"] = np.array([nc, *shape, sw, sx])
    store["sample"] = np.array(SAMPLE)
    np.savez_compressed(f"{HERE}/wide_head.npz", **store)
    print("written", f"{HERE}/wide_head.npz", f"{os.path.getsize(f'{HERE}/wide_head.npz') / 1e3:.0f} kB")


if __name__ == "__main__":
    main()
