"""Segmentation validation AP on the device (reference utils/segment/metrics.py:17-64): box and mask AP from one sort."""
from __future__ import annotations

from ..metrics import _ap_flat, _box_and_mask


def ap_per_class_box_and_mask(tp_m, tp_b, conf, pred_cls, target_cls, plot=False, save_dir=".", names=()):
    """Reference signature: tp_m / tp_b (n, niou) mask / box true positives, conf, pred_cls (n,), target_cls (m,), numpy
    arrays or CUDA tensors -> {"boxes": {"p", "r", "ap", "f1", "ap_class"}, "masks": {...}} as numpy arrays, each equal to
    ap_per_class of its tp matrix.  The predictions are sorted once for both.  plot=True raises NotImplementedError."""
    if plot:
        raise NotImplementedError("y5b200: ap_per_class_box_and_mask(plot=True): plotting is not ported (validation runs with plots=False)")
    return _box_and_mask(*_ap_flat([tp_b, tp_m], conf, pred_cls, target_cls, 1e-16))
