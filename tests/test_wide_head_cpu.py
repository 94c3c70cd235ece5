"""CPU: oracle/model_ref's forward with Detect / Segment heads wider than 128 outputs per anchor (yolov5n at nc = 365,
yolov5n-seg at nc = 100) equals the reference's output stored in tests/golden/wide_head.npz.  The GPU tests of these widths
(test_wide_head_gpu.py) measure the engine against this oracle."""
import copy
import os

import numpy as np
import pytest
import torch

from oracle import model_ref
from yolov5_b200.cfg import model_cfg

G = os.path.join(os.path.dirname(__file__), "golden")
NAMES = ["yolov5n", "yolov5n-seg"]


def wide_case(name):
    """(cfg with the fixture's nc, state_dict, image) of a wide_head.npz case."""
    g = np.load(os.path.join(G, "wide_head.npz"))
    nc, b, c, h, w, sw, sx = (int(v) for v in g[f"{name}.case"])
    cfg = copy.deepcopy(model_cfg(name))
    cfg["nc"] = nc
    sd = model_ref.synth_state_dict(cfg, seed=sw, head_bias="hot")
    x = torch.from_numpy(np.random.RandomState(sx).uniform(0, 1, (b, c, h, w)).astype(np.float32))
    return cfg, sd, x


@pytest.mark.parametrize("fused", [False, True], ids=["bn", "fused"])
@pytest.mark.parametrize("name", NAMES)
def test_oracle_wide_head_equals_reference(name, fused):
    g = np.load(os.path.join(G, "wide_head.npz"))
    cfg, sd, x = wide_case(name)
    with torch.no_grad():
        z = model_ref.forward(cfg, sd, x, fused=fused)[0]
    nm = 32 if name.endswith("-seg") else 0
    assert tuple(z.shape) == tuple(g[f"{name}.z_shape"]) and z.shape[-1] == 5 + cfg["nc"] + nm > 128
    s = int(g["sample"])
    np.testing.assert_allclose(z[:, ::s].numpy(), g[f"{name}.z_sample"], rtol=1e-4, atol=1e-4)
    sums = np.array([z.double().sum().item(), z.double().abs().sum().item()])
    np.testing.assert_allclose(sums, g[f"{name}.z_sum"], rtol=1e-5)
