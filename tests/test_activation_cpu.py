"""CPU: Conv activations beyond SiLU (the model dict's `activation:` key, reference models/yolo.py:383-388).

A model built from the reference's models/hub/yolov5s-LeakyReLU.yaml (its dict is stored in tests/golden/leaky_forward.npz) has
the reference's state_dict keys and LeakyReLU(0.1) in every Conv; a checkpoint pickled by the reference with LeakyReLU Conv modules
loads through attempt_load; activations outside SiLU / ReLU / LeakyReLU / Identity are refused with their name; the ABI's
activation code and the new BN entry points are mirrored in _lib.  Every test that builds from such a dict puts
Conv.default_act back to nn.SiLU()."""
import ctypes
import json
import os
import re

import numpy as np
import pytest
import torch
from torch import nn

from oracle import model_ref
from yolov5_b200 import _lib
from yolov5_b200.engine import act_spec
from yolov5_b200.models.common import Conv

G = os.path.join(os.path.dirname(__file__), "golden")
HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "y5b200.h")


@pytest.fixture
def restore_act():
    yield
    Conv.default_act = nn.SiLU()


def _leaky_cfg():
    return json.loads(str(np.load(os.path.join(G, "leaky_forward.npz"))["cfg"]))


def test_leaky_yaml_builds_with_reference_keys_and_leaky_convs(restore_act):
    from yolov5_b200.models.yolo import DetectionModel

    cfg = _leaky_cfg()
    assert cfg["activation"] == "nn.LeakyReLU(0.1)"
    m = DetectionModel(cfg)
    convs = [c for c in m.modules() if isinstance(c, Conv)]
    assert convs and all(type(c.act) is nn.LeakyReLU and c.act.negative_slope == 0.1 for c in convs)
    # oracle/model_ref.param_shapes is the reference's key order (pinned by tests/golden/model_forward.npz)
    assert list(m.state_dict().keys()) == list(model_ref.param_shapes(cfg).keys())
    m.load_state_dict(model_ref.synth_state_dict(cfg, seed=30))
    assert [float(s) for s in m.stride] == [8.0, 16.0, 32.0]
    Conv.default_act = nn.SiLU()
    assert type(DetectionModel("yolov5n").model[0].act) is nn.SiLU  # once restored, later models are SiLU again


def test_segment_and_classification_models_from_a_leaky_dict(restore_act):
    from yolov5_b200.cfg import model_cfg
    from yolov5_b200.models.yolo import ClassificationModel, DetectionModel, SegmentationModel

    cfg = model_cfg("yolov5n-seg")
    cfg["activation"] = "nn.ReLU()"
    m = SegmentationModel(cfg)
    assert {type(c.act) for c in m.modules() if isinstance(c, Conv)} == {nn.ReLU}
    Conv.default_act = nn.SiLU()
    det = DetectionModel(_leaky_cfg())
    cls = ClassificationModel(model=det, nc=10, cutoff=10)
    assert {type(c.act) for c in cls.modules() if isinstance(c, Conv)} == {nn.LeakyReLU}


def test_reference_pickled_leaky_checkpoint_loads():
    from yolov5_b200 import compat
    from yolov5_b200.models import yolo
    from yolov5_b200.models.experimental import attempt_load

    try:
        ref = np.load(os.path.join(G, "ref_leaky_tiny_forward.npz"))
        m = attempt_load(os.path.join(G, "ref_leaky_tiny.pt"), device="cpu", fuse=False)
        assert type(m) is yolo.DetectionModel and list(m.state_dict().keys()) == json.loads(str(ref["keys"]))
        convs = [c for c in m.modules() if isinstance(c, Conv)]
        assert convs and all(type(c.act) is nn.LeakyReLU and act_spec(c.act) == (_lib.ACT_LEAKY, pytest.approx(0.1)) for c in convs)
        fused = attempt_load(os.path.join(G, "ref_leaky_tiny.pt"), device="cpu")
        assert not hasattr(fused.model[0], "bn") and type(fused.model[0].act) is nn.LeakyReLU
    finally:
        compat.uninstall()
    assert Conv.default_act.__class__ is nn.SiLU  # loading a pickle does not touch the class default


def test_act_spec_and_refusals(restore_act):
    from yolov5_b200 import train_ops
    from yolov5_b200.models.yolo import DetectionModel

    assert act_spec(nn.SiLU()) == (_lib.ACT_SILU, 0.0) and act_spec(nn.Identity()) == (_lib.ACT_NONE, 0.0)
    assert act_spec(nn.ReLU()) == (_lib.ACT_LEAKY, 0.0) and act_spec(nn.LeakyReLU(0.01)) == (_lib.ACT_LEAKY, 0.01)
    for bad in (nn.Hardswish(), nn.GELU(), nn.LeakyReLU(float("inf")), nn.ReLU6()):
        with pytest.raises(NotImplementedError, match=type(bad).__name__):
            act_spec(bad)
    cfg = _leaky_cfg()
    cfg["activation"] = "nn.Hardswish()"
    m = DetectionModel(cfg)  # builds (parameters are activation independent) ...
    with pytest.raises(NotImplementedError, match="Hardswish"):  # ... but the engine's lowerings refuse it, by name
        train_ops.conv_module(m.model[0], torch.zeros(1, 3, 32, 32), stem=2)


def test_abi_activation_code_and_slope_argument(built_lib):
    src = open(HEADER).read()
    codes = dict(re.findall(r"#define (Y5_ACT_\w+) (\d+)", src))
    assert {k: int(v) for k, v in codes.items()} == {"Y5_ACT_NONE": _lib.ACT_NONE, "Y5_ACT_SILU": _lib.ACT_SILU, "Y5_ACT_LEAKY": _lib.ACT_LEAKY}
    assert [f for f, _ in _lib.ConvDesc._fields_][-1] == "act_slope" and _lib.ConvDesc().act_slope == 0.0  # zero default: today's descs
    lib = built_lib
    P = None
    # the activation is checked before anything touches the device: a bad code or a non-finite slope is refused on any machine
    args = (P, 64, P, 64, 10, 64, _lib.Y5_F16, P, P, P, P)
    tail = (P, P, 1e-3, 0.03, P, P, P, 0, P)
    sync_tail = (P, 4096, *tail[2:])  # a non-NULL row count: SyncBatchNorm's forward
    assert lib.y5_bn_act_fwd(*args, 3, 0.0, *tail) == -2 and b"activation code 3" in lib.y5_last_error()
    assert lib.y5_bn_act_fwd(*args, _lib.ACT_LEAKY, float("nan"), *tail) == -1 and b"slope" in lib.y5_last_error()
    assert lib.y5_bn_act_fwd(*args, _lib.ACT_LEAKY, float("inf"), *sync_tail) == -1 and b"slope" in lib.y5_last_error()
    bargs = (P, 64, P, 64, P, 64, 10, 64, _lib.Y5_F16, P, P, P, P)
    assert lib.y5_bn_act_bwd(*bargs, 7, 0.0, P, P, P, P) == -2
    assert lib.y5_bn_act_bwd_reduce(*bargs, _lib.ACT_LEAKY, float("nan"), P, P, P, P) == -1
    assert lib.y5_bn_act_bwd(*bargs, _lib.ACT_LEAKY, 0.1, P, P, P, P) == -1 and b"null" in lib.y5_last_error().lower()
