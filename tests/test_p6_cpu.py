"""CPU: the P6 models (reference models/hub/yolov5{n,s,m,l,x}6.yaml) without a GPU -- the built-in names against the reference
YAMLs' digests; parameter counts, state_dict keys and shapes, Detect strides and anchors against the reference's models; the
four-level loss balance; the reference-pickled checkpoint through compat."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from yolov5_b200.cfg import model_cfg, model_names

G = os.path.join(os.path.dirname(__file__), "golden")
SIZES = "nsmlx"


def _fixture():
    return np.load(os.path.join(G, "p6_golden.npz"))


@pytest.mark.parametrize("size", SIZES)
def test_builtin_names_match_reference_yaml(size):
    name = f"yolov5{size}6"
    cfg = model_cfg(name)
    assert hashlib.sha256(json.dumps(cfg, sort_keys=True).encode()).hexdigest() == str(_fixture()[f"{size}:digest"])
    assert model_cfg(f"{name}.yaml") == cfg == model_cfg(f"models/hub/{name}.yaml")
    assert cfg["head"][-1] == [[23, 26, 29, 32], 1, "Detect", ["nc", "anchors"]]


def test_model_names_unchanged():
    assert model_names() == [f"yolov5{k}" for k in SIZES] + [f"yolov5{k}-seg" for k in SIZES]
    with pytest.raises(KeyError):
        model_cfg("yolov5q6")
    with pytest.raises(KeyError):
        model_cfg("yolov5s7")


@pytest.mark.parametrize("size", SIZES)
def test_parameters_keys_strides_anchors_match_reference(size):
    from yolov5_b200.models.yolo import DetectionModel

    f = _fixture()
    m = DetectionModel(f"yolov5{size}6")
    assert sum(p.numel() for p in m.parameters()) == int(f[f"{size}:n_params"])
    assert [[k, list(v.shape)] for k, v in m.state_dict().items()] == json.loads(str(f[f"{size}:keys"]))
    det = m.model[-1]
    assert det.nl == 4 and det.stride.tolist() == [8.0, 16.0, 32.0, 64.0] == f[f"{size}:stride"].tolist()
    assert int(m.stride.max()) == 64
    assert torch.equal(det.anchors, torch.from_numpy(f[f"{size}:anchors"]))
    px = torch.tensor(model_cfg(f"yolov5{size}6")["anchors"], dtype=torch.float32).view(4, 3, 2)
    assert torch.equal(det.anchors, px / torch.tensor([8.0, 16.0, 32.0, 64.0]).view(4, 1, 1))  # already ascending: no flip


def test_small_model_keys_match_reference():
    from yolov5_b200.models.yolo import DetectionModel

    f = _fixture()
    small = DetectionModel(json.loads(str(f["small_cfg"])))
    assert list(small.state_dict().keys()) == json.loads(str(f["small_keys"]))
    assert all(mod.out_channels % 8 == 0 for mod in small.modules() if isinstance(mod, torch.nn.Conv2d))


def test_four_level_loss_balance():
    from yolov5_b200.cfg import HYP_SCRATCH_LOW
    from yolov5_b200.models.yolo import DetectionModel
    from yolov5_b200.utils.loss import ComputeLoss

    m = DetectionModel("yolov5n6")
    m.hyp = dict(HYP_SCRATCH_LOW)
    crit = ComputeLoss(m)
    assert crit.nl == 4 and crit.balance[:4] == [4.0, 1.0, 0.25, 0.06]


def test_reference_checkpoint_loads_through_compat():
    from yolov5_b200 import compat

    assert compat.install()
    ck = torch.load(os.path.join(G, "ref_p6_tiny.pt"), map_location="cpu", weights_only=False)
    m = ck["model"]
    assert type(m).__module__ == "yolov5_b200.models.yolo"
    assert list(m.state_dict().keys()) == json.loads(str(_fixture()["small_keys"]))
    assert m.model[-1].nl == 4 and m.stride.tolist() == [8.0, 16.0, 32.0, 64.0]
