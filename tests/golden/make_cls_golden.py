"""Generate tests/golden/cls.npz, cls_signatures.json and ref_cls_tiny.pt by running the UNMODIFIED reference's
classification model (models/yolo.py ClassificationModel, models/common.py Classify) and loss (utils/torch_utils.py
smartCrossEntropyLoss) through tests/golden/refshim.py.

Runs only where the reference tree exists:
    python tests/golden/make_cls_golden.py
Weights come from oracle/cls_ref.synth_state_dict and inputs from the seeds below (`image`, `labels`, `ce_case`, which the
tests call), so cls.npz holds only the reference's outputs.  Gradients with more than GRAD_SAMPLE elements are stored as a
fixed seeded sample of their entries plus their full L2 norm (`grad_record`), which keeps the fixture small.  While
generating, the oracle (oracle/cls_ref.py) is checked against the reference on every entry (hard assert).
"""
from __future__ import annotations

import inspect
import json
import os
import sys
from copy import deepcopy

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from oracle import cls_ref  # noqa: E402
from yolov5_b200.cfg import model_cfg  # noqa: E402

NC = 10
EVAL = dict(model="yolov5n", seed=31, shape=(2, 3, 64, 64), x_seed=32)        # eval logits, random BN statistics
TRAIN = dict(seed=33, shape=(4, 3, 64, 64), x_seed=34, label_seed=35, eps=0.1)  # tiny_cfg(): training logits, loss, gradients
CKPT = dict(seed=36, shape=(2, 3, 64, 64), x_seed=37)                          # reference-pickled tiny model + its logits
CE = [(16, 10, 0.0, 40), (16, 10, 0.1, 41), (8, 1000, 0.0, 42), (8, 1000, 0.1, 43)]  # (batch, nc, eps, seed)


def tiny_cfg():
    """yolov5n's topology at width_multiple 0.125 (every channel count still a multiple of 8)."""
    cfg = model_cfg("yolov5n")
    cfg["width_multiple"] = 0.125
    return cfg


def image(shape, seed):
    return torch.from_numpy(np.random.RandomState(seed).uniform(0, 1, shape).astype(np.float32))


def labels(n, seed):
    return torch.from_numpy(np.random.RandomState(seed).randint(0, NC, n).astype(np.int64))


def ce_case(b, nc, seed):
    rs = np.random.RandomState(seed)
    return torch.from_numpy((rs.normal(0, 3, (b, nc))).astype(np.float32)), torch.from_numpy(rs.randint(0, nc, b).astype(np.int64))


GRAD_SAMPLE = 2048  # gradients with more elements are pinned by this many seeded entries plus their full L2 norm


def grad_sample_index(numel):
    """flat indices of a gradient's pinned entries: all of them up to GRAD_SAMPLE, else a fixed sorted sample"""
    if numel <= GRAD_SAMPLE:
        return np.arange(numel)
    return np.sort(np.random.RandomState(numel).choice(numel, GRAD_SAMPLE, replace=False))


def grad_record(g):
    """(pinned entries, float64 L2 norm) of a gradient tensor, as cls.npz stores them"""
    flat = np.asarray(g, dtype=np.float32).reshape(-1)
    return flat[grad_sample_index(flat.size)], np.float64(np.linalg.norm(flat.astype(np.float64)))


def ref_cls_model(cfg, sd):
    """reference ClassificationModel(model=DetectionModel(cfg), nc=NC) loaded with `sd` (strict)."""
    from models.yolo import ClassificationModel, DetectionModel

    m = ClassificationModel(model=DetectionModel(deepcopy(cfg)), nc=NC)
    m.load_state_dict(sd, strict=True)
    return m


def main():
    sys.path.insert(0, HERE)
    import refshim

    refshim.install()
    from models.common import Classify
    from models.yolo import ClassificationModel
    from utils.torch_utils import reshape_classifier_output, smartCrossEntropyLoss

    store = {}
    # eval logits (running BN statistics) of yolov5n-cls
    cfg = model_cfg(EVAL["model"])
    sd = cls_ref.synth_state_dict(cfg, NC, seed=EVAL["seed"])
    m = ref_cls_model(cfg, sd).eval()
    assert list(m.state_dict()) == list(cls_ref.param_shapes(cfg, NC)), "state_dict keys / order differ from the oracle's"
    print(f"reference yolov5n-cls: {len(m.state_dict())} state_dict entries, {sum(p.numel() for p in m.parameters())} parameters")
    x = image(EVAL["shape"], EVAL["x_seed"])
    with torch.no_grad():
        y = m(x)
        yo = cls_ref.forward(cfg, sd, x)
    assert y.shape == (EVAL["shape"][0], NC) and torch.allclose(y, yo, rtol=1e-5, atol=1e-5), (y - yo).abs().max()
    store["eval.logits"] = y.numpy()

    # training forward + CE(eps) + backward of the tiny model
    tcfg = tiny_cfg()
    sd = cls_ref.synth_state_dict(tcfg, NC, seed=TRAIN["seed"])
    m = ref_cls_model(tcfg, sd).train()
    x, lab = image(TRAIN["shape"], TRAIN["x_seed"]), labels(TRAIN["shape"][0], TRAIN["label_seed"])
    y = m(x)
    loss = smartCrossEntropyLoss(label_smoothing=TRAIN["eps"])(y, lab)
    loss.backward()
    params = {k: v.clone().requires_grad_(v.is_floating_point() and "running" not in k) for k, v in sd.items()}
    yo = cls_ref.forward(tcfg, params, x, bn_batch_stats=True)
    lo = cls_ref.cross_entropy(yo, lab, TRAIN["eps"])
    lo.backward()
    assert torch.allclose(y, yo, rtol=1e-4, atol=1e-5) and torch.allclose(loss, lo, rtol=1e-5), (loss, lo)
    for k, p in m.named_parameters():
        assert torch.allclose(p.grad, params[k].grad, rtol=1e-3, atol=1e-6), (k, (p.grad - params[k].grad).abs().max())
        store[f"train.grad.{k}"], store[f"train.gradnorm.{k}"] = grad_record(p.grad.numpy())
    store["train.logits"], store["train.loss"] = y.detach().numpy(), loss.detach().numpy()

    # cross-entropy cases
    for b, nc, eps, seed in CE:
        z, lab = ce_case(b, nc, seed)
        z.requires_grad_(True)
        crit = smartCrossEntropyLoss(label_smoothing=eps)
        loss = crit(z, lab)
        loss.backward()
        z64 = z.detach().double()
        assert abs(float(loss) - float(cls_ref.cross_entropy(z64, lab, eps))) <= 1e-5 * abs(float(loss)), (nc, eps)
        assert torch.allclose(z.grad.double(), cls_ref.cross_entropy_grad(z64, lab, eps), rtol=1e-4, atol=1e-7), (nc, eps)
        tag = f"ce.{nc}.{eps}"
        store[f"{tag}.loss"], store[f"{tag}.grad"] = loss.detach().numpy(), z.grad.numpy()

    # a checkpoint pickled by the reference, in classify/train.py's format ({"model": deepcopy(ema).half(), ...})
    sd = cls_ref.synth_state_dict(tcfg, NC, seed=CKPT["seed"])
    sd = {k: v.half().float() if v.is_floating_point() else v for k, v in sd.items()}  # the fp16 checkpoint holds these values
    m = ref_cls_model(tcfg, sd).eval()
    m.names = [f"class{i}" for i in range(NC)]
    x = image(CKPT["shape"], CKPT["x_seed"])
    with torch.no_grad():
        y = m(x)
    torch.save({"model": deepcopy(m).half(), "ema": None, "updates": 0, "optimizer": None, "date": "fixture"}, f"{HERE}/ref_cls_tiny.pt")
    store["ckpt.logits"] = y.numpy()
    store["ckpt.keys"] = np.array(json.dumps(list(m.state_dict())))
    store["ckpt.shapes"] = np.array(json.dumps({k: list(v.shape) for k, v in m.state_dict().items()}))

    np.savez_compressed(f"{HERE}/cls.npz", **store)
    sig = {}
    for name, obj in (("Classify.__init__", Classify.__init__), ("ClassificationModel.__init__", ClassificationModel.__init__),
                      ("ClassificationModel._from_detection_model", ClassificationModel._from_detection_model),
                      ("ClassificationModel._from_yaml", ClassificationModel._from_yaml),
                      ("smartCrossEntropyLoss", smartCrossEntropyLoss), ("reshape_classifier_output", reshape_classifier_output)):
        sig[name] = [(n, repr(q.default) if q.default is not inspect._empty else None, str(q.kind)) for n, q in inspect.signature(obj).parameters.items()]
    with open(f"{HERE}/cls_signatures.json", "w") as f:
        json.dump(sig, f, indent=1, sort_keys=True)
    print("written", f"{HERE}/cls.npz", os.path.getsize(f"{HERE}/cls.npz"), "bytes;", f"{HERE}/ref_cls_tiny.pt",
          os.path.getsize(f"{HERE}/ref_cls_tiny.pt"), "bytes; oracle == reference")


if __name__ == "__main__":
    main()
