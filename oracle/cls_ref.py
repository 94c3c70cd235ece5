"""ORACLE (test infrastructure, never on the product path): CPU restatement of the YOLOv5 classification model and loss.

Reference lines restated (paths relative to the reference tree):
  models/yolo.py:343-372       ClassificationModel._from_detection_model: backbone cut at `cutoff`, last layer -> Classify
  models/common.py:1120-1140   Classify: Conv(c1, 1280) -> AdaptiveAvgPool2d(1) -> flatten -> Dropout -> Linear(1280, nc)
  utils/torch_utils.py:52-57   smartCrossEntropyLoss -> nn.CrossEntropyLoss(label_smoothing=eps), reduction 'mean'

Driven by a state_dict with the reference's key names (model.{i}.* for the backbone, model.{cutoff-1}.conv.* and
model.{cutoff-1}.linear.* for the head) plus the detection model dict.  Pinned by tests/golden/cls.npz, written by
tests/golden/make_cls_golden.py from the unmodified reference.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from . import model_ref

C_HEAD = 1280  # Classify's hidden width (efficientnet_b0 size)
HEAD_BN_EPS = 1e-5  # Classify.conv.bn keeps nn.BatchNorm2d's default (see _head_conv)


def head_in_channels(cfg: dict, cutoff: int = 10) -> int:
    """Input channels of the layer Classify replaces (models/yolo.py:361): that layer's conv / cv1 input."""
    layers, _ = model_ref.parse_layers(cfg)
    return layers[cutoff - 1]["c1"]


def param_shapes(cfg: dict, nc: int, cutoff: int = 10) -> dict:
    """state_dict key -> shape of ClassificationModel(model=DetectionModel(cfg), nc, cutoff), in the reference's key order."""
    out = {k: v for k, v in model_ref.param_shapes(cfg).items() if int(k.split(".")[1]) < cutoff - 1}
    p = f"model.{cutoff - 1}"
    out[f"{p}.conv.conv.weight"] = (C_HEAD, head_in_channels(cfg, cutoff), 1, 1)
    for q in ("weight", "bias", "running_mean", "running_var"):
        out[f"{p}.conv.bn.{q}"] = (C_HEAD,)
    out[f"{p}.conv.bn.num_batches_tracked"] = ()
    out[f"{p}.linear.weight"] = (nc, C_HEAD)
    out[f"{p}.linear.bias"] = (nc,)
    return out


def synth_state_dict(cfg: dict, nc: int, seed: int = 0, cutoff: int = 10) -> dict:
    """Seeded weights: the backbone as model_ref.synth_state_dict draws it, the head conv / BN the same way, the Linear
    U(-1/sqrt(1280), 1/sqrt(1280)) for weight and bias (nn.Linear's bound)."""
    sd = {k: v for k, v in model_ref.synth_state_dict(cfg, seed=seed).items() if int(k.split(".")[1]) < cutoff - 1}
    rs = np.random.RandomState(seed + 1000)
    for k, shp in param_shapes(cfg, nc, cutoff).items():
        if k in sd:
            continue
        if k.endswith("num_batches_tracked"):
            v = np.zeros((), np.int64)
        elif ".bn." in k:
            v = rs.uniform(0.5, 1.5, shp) if k.endswith(("weight", "running_var")) else rs.normal(0.0, 0.1, shp)
        elif ".linear." in k:
            v = rs.uniform(-1, 1, shp) / math.sqrt(C_HEAD)
        else:
            v = rs.uniform(-1, 1, shp) / math.sqrt(shp[1])
        sd[k] = torch.from_numpy(np.asarray(v, dtype=np.int64 if k.endswith("tracked") else np.float32).copy())
    return sd


def _head_conv(sd, p, x, bn_batch_stats, fused):
    """Classify.conv: 1x1 conv -> BN -> SiLU.  Its BatchNorm is created after initialize_weights ran (models/yolo.py:362), so it
    keeps torch's defaults eps = 1e-5, momentum = 0.1 instead of the backbone's 1e-3 / 0.03."""
    w = sd[f"{p}.conv.weight"]
    if f"{p}.bn.weight" not in sd:  # fused state_dict: conv with bias
        return F.silu(F.conv2d(x, w, sd[f"{p}.conv.bias"]))
    g, b, m, v = (sd[f"{p}.bn.{q}"] for q in ("weight", "bias", "running_mean", "running_var"))
    if fused:
        w2, b2 = model_ref.fold_bn(w, g, b, m, v, eps=HEAD_BN_EPS)
        return F.silu(F.conv2d(x, w2, b2))
    y = F.conv2d(x, w)
    y = F.batch_norm(y, None, None, g, b, training=True, eps=HEAD_BN_EPS) if bn_batch_stats else F.batch_norm(y, m, v, g, b, eps=HEAD_BN_EPS)
    return F.silu(y)


def forward(cfg: dict, sd: dict, x: torch.Tensor, cutoff: int = 10, bn_batch_stats: bool = False, fused: bool = False) -> torch.Tensor:
    """(B, nc) logits.  bn_batch_stats: every BatchNorm normalises with batch statistics (model.train(), dropout_p = 0)."""
    layers, _ = model_ref.parse_layers(cfg)
    prev, model_ref._BN_BATCH_STATS = model_ref._BN_BATCH_STATS, bool(bn_batch_stats)
    try:
        ys = []
        for L in layers[: cutoff - 1]:
            f, kind, p = L["f"], L["kind"], f"model.{L['i']}"
            if f != -1:
                x = ys[f] if isinstance(f, int) else [x if j == -1 else ys[j] for j in f]
            if kind == "Conv":
                a = L["args"]
                x = model_ref.conv_block(sd, p, x, a[0] if a else 1, a[1] if len(a) > 1 else 1, a[2] if len(a) > 2 else None, fused)
            elif kind == "C3":
                x = model_ref.c3(sd, p, x, L["n"], L["args"][0] if L["args"] else True, fused)
            elif kind == "SPPF":
                x = model_ref.sppf(sd, p, x, L["args"][0] if L["args"] else 5, fused)
            else:
                raise NotImplementedError(kind)
            ys.append(x)
        p = f"model.{cutoff - 1}"
        h = _head_conv(sd, f"{p}.conv", x, bn_batch_stats, fused)
        pooled = h.mean((2, 3))  # AdaptiveAvgPool2d(1) + flatten(1)
        return F.linear(pooled, sd[f"{p}.linear.weight"], sd[f"{p}.linear.bias"])
    finally:
        model_ref._BN_BATCH_STATS = prev


def cross_entropy(logits: torch.Tensor, labels: torch.Tensor, eps: float = 0.0) -> torch.Tensor:
    """mean_i[(1 - eps) (-log p_{i,y_i}) + (eps / nc) sum_c (-log p_{i,c})] in the logits' dtype (use float64 for a reference)."""
    nc = logits.shape[1]
    nlp = -torch.log_softmax(logits, 1)
    return ((1 - eps) * nlp.gather(1, labels.view(-1, 1)).squeeze(1) + (eps / nc) * nlp.sum(1)).mean()


def cross_entropy_grad(logits: torch.Tensor, labels: torch.Tensor, eps: float = 0.0) -> torch.Tensor:
    """d loss / d logits = (softmax - q) / B,  q = (1 - eps) onehot + eps / nc."""
    b, nc = logits.shape
    q = torch.full_like(logits, eps / nc)
    q[torch.arange(b), labels] += 1 - eps
    return (torch.softmax(logits, 1) - q) / b
