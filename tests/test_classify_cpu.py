"""CPU: the classification surface -- ClassificationModel / Classify / smartCrossEntropyLoss / reshape_classifier_output with the
reference's signatures and state_dict keys, a checkpoint pickled by the reference loading into the engine's classes, the oracle
(oracle/cls_ref.py) against the reference's outputs (tests/golden/cls.npz, make_cls_golden.py), and the refused options."""
import inspect
import json
import os
import pickle

import numpy as np
import pytest
import torch

from oracle import cls_ref
from tests.golden import make_cls_golden as mk
from yolov5_b200.cfg import model_cfg

G = os.path.join(os.path.dirname(__file__), "golden")
NC = mk.NC
_tiny_cfg = mk.tiny_cfg


def _golden():
    return np.load(os.path.join(G, "cls.npz"))


def _cls_model(name_or_cfg="yolov5n", nc=NC):
    from yolov5_b200.models.yolo import ClassificationModel, DetectionModel

    return ClassificationModel(model=DetectionModel(name_or_cfg), nc=nc)


def test_signatures_match_the_reference():
    from yolov5_b200.models.common import Classify
    from yolov5_b200.models.yolo import ClassificationModel
    from yolov5_b200.utils.torch_utils import reshape_classifier_output, smartCrossEntropyLoss

    with open(os.path.join(G, "cls_signatures.json")) as f:
        ref = json.load(f)
    ours = {"Classify.__init__": Classify.__init__, "ClassificationModel.__init__": ClassificationModel.__init__,
            "ClassificationModel._from_detection_model": ClassificationModel._from_detection_model,
            "ClassificationModel._from_yaml": ClassificationModel._from_yaml, "smartCrossEntropyLoss": smartCrossEntropyLoss,
            "reshape_classifier_output": reshape_classifier_output}
    assert sorted(ref) == sorted(ours)
    for name, fn in ours.items():
        mine = [[n, repr(p.default) if p.default is not inspect._empty else None, str(p.kind)] for n, p in inspect.signature(fn).parameters.items()]
        assert mine == ref[name], (name, mine, ref[name])


@pytest.mark.parametrize("name", ["yolov5n", "yolov5s"])
def test_state_dict_keys_and_shapes_equal_the_reference(name):
    m = _cls_model(name, 1000)
    want = cls_ref.param_shapes(model_cfg(name), 1000)
    assert list(m.state_dict()) == list(want)
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == {k: tuple(v) for k, v in want.items()}
    head = m.model[-1]
    assert (head.i, head.f, head.type) == (9, -1, "models.common.Classify") and m.save == [] and m.nc == 1000
    assert isinstance(head.pool, torch.nn.AdaptiveAvgPool2d) and isinstance(head.drop, torch.nn.Dropout) and head.drop.inplace
    assert [float(s) for s in m.stride] == [8.0, 16.0, 32.0]
    assert head.conv.bn.eps == 1e-5 and m.model[8].cv1.bn.eps == 1e-3  # the head BN keeps torch's defaults, as in the reference
    from yolov5_b200.models.yolo import ClassificationModel

    assert ClassificationModel(cfg="x.yaml").model is None


def test_tiny_model_keys_equal_the_reference_pickle_and_golden():
    g = _golden()
    m = _cls_model(_tiny_cfg())
    assert list(m.state_dict()) == json.loads(str(g["ckpt.keys"]))
    assert {k: list(v.shape) for k, v in m.state_dict().items()} == json.loads(str(g["ckpt.shapes"]))


def test_reference_pickled_checkpoint_loads_through_compat_and_attempt_load():
    from yolov5_b200 import compat
    from yolov5_b200.models import common, yolo
    from yolov5_b200.models.experimental import attempt_load

    try:
        assert compat.install()
        from models.yolo import ClassificationModel  # classify/train.py:40

        assert ClassificationModel is yolo.ClassificationModel
        import models.common as mcm

        assert mcm.Classify is common.Classify
        ck = torch.load(os.path.join(G, "ref_cls_tiny.pt"), map_location="cpu", weights_only=False)
        m = ck["model"]
        assert type(m) is yolo.ClassificationModel and type(m.model[-1]) is common.Classify
        assert next(m.parameters()).dtype == torch.float16 and m.nc == NC
        twin = _cls_model(_tiny_cfg())
        twin.load_state_dict(m.float().state_dict())
        fused = attempt_load(os.path.join(G, "ref_cls_tiny.pt"), device="cpu")
        head = fused.model[-1]
        assert type(fused) is yolo.ClassificationModel and not fused.training
        assert not hasattr(head.conv, "bn") and head.conv.conv.bias is not None  # fuse() folds Classify.conv too
        assert next(fused.parameters()).dtype == torch.float32
        pickle.loads(pickle.dumps(fused))
    finally:
        compat.uninstall()


def test_reshape_classifier_output_replaces_the_linear_and_drops_the_caches():
    from yolov5_b200.models.common import _param_version
    from yolov5_b200.utils.torch_utils import reshape_classifier_output

    m = _cls_model(_tiny_cfg())
    _param_version(m)  # the tensor list behind the program cache key
    m.__dict__["_y5_programs"] = {"stale": None}
    old = m.model[-1].linear
    reshape_classifier_output(m, NC)  # same class count: untouched
    assert m.model[-1].linear is old
    reshape_classifier_output(m, 7)
    assert m.model[-1].linear.out_features == 7 and m.model[-1].linear.in_features == 1280
    assert "_y5_programs" not in m.__dict__ and "_y5_tensors" not in m.__dict__
    assert any(t is m.model[-1].linear.weight for t in (m.__dict__.setdefault("_y5_tensors", list(m.parameters()))))

    class Plain(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.body = torch.nn.Conv2d(3, 8, 1)
            self.fc = torch.nn.Linear(8, 5)

    p = Plain()
    reshape_classifier_output(p, 3)
    assert p.fc.out_features == 3 and p.fc.in_features == 8


def test_oracle_matches_the_reference_golden():
    g = _golden()
    cfg = model_cfg("yolov5n")
    sd = cls_ref.synth_state_dict(cfg, NC, seed=mk.EVAL["seed"])
    x = mk.image(mk.EVAL["shape"], mk.EVAL["x_seed"])
    with torch.no_grad():
        y = cls_ref.forward(cfg, sd, x)
    assert np.allclose(y.numpy(), g["eval.logits"], rtol=1e-5, atol=1e-5)
    with torch.no_grad():  # BN folded (what attempt_load's fuse() computes) gives the same logits
        yf = cls_ref.forward(cfg, sd, x, fused=True)
    assert np.allclose(yf.numpy(), g["eval.logits"], rtol=1e-4, atol=1e-4)
    tcfg = mk.tiny_cfg()
    sd = cls_ref.synth_state_dict(tcfg, NC, seed=mk.TRAIN["seed"])
    params = {k: v.clone().requires_grad_(v.is_floating_point() and "running" not in k) for k, v in sd.items()}
    y = cls_ref.forward(tcfg, params, mk.image(mk.TRAIN["shape"], mk.TRAIN["x_seed"]), bn_batch_stats=True)
    loss = cls_ref.cross_entropy(y, mk.labels(mk.TRAIN["shape"][0], mk.TRAIN["label_seed"]), mk.TRAIN["eps"])
    loss.backward()
    assert np.allclose(y.detach().numpy(), g["train.logits"], rtol=1e-4, atol=1e-5)
    assert abs(float(loss.detach()) - float(g["train.loss"])) <= 1e-5 * float(g["train.loss"])
    keys = [k[len("train.grad."):] for k in g.files if k.startswith("train.grad.")]
    assert sorted(keys) == sorted(k for k, v in params.items() if v.requires_grad)  # every parameter's gradient is pinned
    for k in keys:
        entries, norm = mk.grad_record(params[k].grad.numpy())
        assert np.allclose(entries, g[f"train.grad.{k}"], rtol=1e-3, atol=1e-6), k
        assert abs(norm - float(g[f"train.gradnorm.{k}"])) <= 1e-4 * float(g[f"train.gradnorm.{k}"]) + 1e-9, k
    for b, nc, eps, seed in mk.CE:
        t = f"ce.{nc}.{eps}"
        z, lab = mk.ce_case(b, nc, seed)
        z = z.double()
        assert abs(float(cls_ref.cross_entropy(z, lab, eps)) - float(g[f"{t}.loss"])) <= 1e-5 * float(g[f"{t}.loss"]), t
        assert np.allclose(cls_ref.cross_entropy_grad(z, lab, eps).numpy(), g[f"{t}.grad"], rtol=1e-4, atol=1e-7), t


def test_cross_entropy_module_is_a_torch_cross_entropy_loss():
    from yolov5_b200.utils.loss import CrossEntropyLoss
    from yolov5_b200.utils.torch_utils import smartCrossEntropyLoss

    crit = smartCrossEntropyLoss(label_smoothing=0.1)
    assert isinstance(crit, torch.nn.CrossEntropyLoss) and isinstance(crit, CrossEntropyLoss)
    assert crit.label_smoothing == 0.1 and crit.reduction == "mean" and crit.ignore_index == -100
    assert smartCrossEntropyLoss().label_smoothing == 0.0


def test_refused_inputs_and_options():
    from yolov5_b200.utils.loss import CrossEntropyLoss

    z, lab = torch.zeros(4, NC), torch.zeros(4, dtype=torch.long)
    with pytest.raises(RuntimeError, match="CUDA"):
        CrossEntropyLoss(label_smoothing=0.1)(z, lab)
    for kw in (dict(weight=torch.ones(NC)), dict(reduction="sum"), dict(reduction="none"), dict(ignore_index=3)):
        with pytest.raises(NotImplementedError):
            CrossEntropyLoss(**kw)(z, lab)
    with pytest.raises(NotImplementedError, match="probabilit"):
        CrossEntropyLoss()(z, torch.zeros(4, NC))
    m = _cls_model(_tiny_cfg())
    with pytest.raises(RuntimeError, match="CUDA"):
        m.eval()(torch.zeros(1, 3, 64, 64))
    with pytest.raises(RuntimeError, match="ClassificationModel"):
        m.model[-1](torch.zeros(1, 128, 2, 2))


def test_dropout_in_training_is_refused_before_any_launch():
    from yolov5_b200.train_ops import _classify

    m = _cls_model(_tiny_cfg())
    head = m.model[-1]
    head.drop.p = 0.2  # classify/train.py --dropout 0.2
    head.train()
    with pytest.raises(NotImplementedError, match="Dropout"):
        _classify(head, torch.zeros(1, 128, 2, 2))
    with pytest.raises(NotImplementedError, match="Concat"):
        _classify(head, [torch.zeros(1, 64, 2, 2), torch.zeros(1, 64, 2, 2)])
