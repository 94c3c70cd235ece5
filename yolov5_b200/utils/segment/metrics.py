"""Segmentation validation AP on the device (reference utils/segment/metrics.py:17-64): box and mask AP from one sort.  The
host bookkeeping segment/val.py and segment/train.py import from here, `fitness`, `Metric`, `Metrics` and `KEYS`, works on
the numpy arrays that AP returns."""
from __future__ import annotations

import numpy as np

from ..metrics import _ap_flat, _box_and_mask


def ap_per_class_box_and_mask(tp_m, tp_b, conf, pred_cls, target_cls, plot=False, save_dir=".", names=()):
    """Reference signature: tp_m / tp_b (n, niou) mask / box true positives, conf, pred_cls (n,), target_cls (m,), numpy
    arrays or CUDA tensors -> {"boxes": {"p", "r", "ap", "f1", "ap_class"}, "masks": {...}} as numpy arrays, each equal to
    ap_per_class of its tp matrix.  The predictions are sorted once for both.  plot=True raises NotImplementedError."""
    if plot:
        raise NotImplementedError("y5b200: ap_per_class_box_and_mask(plot=True): plotting is not ported (validation runs with plots=False)")
    return _box_and_mask(*_ap_flat([tp_b, tp_m], conf, pred_cls, target_cls, 1e-16))


def fitness(x):
    """Reference utils/segment/metrics.py fitness: per row of [P, R, mAP@0.5, mAP@0.5:0.95] for boxes then masks (numpy,
    host), 0.1 * mAP@0.5 + 0.9 * mAP@0.5:0.95 of each group, summed over the eight weighted columns in column order."""
    return np.sum(np.asarray(x)[:, :8] * np.array([0.0, 0.0, 0.1, 0.9] * 2), axis=1)


class Metric:
    """Reference utils/segment/metrics.py Metric: one task's per-class results as ap_per_class_box_and_mask returns them
    (p, r, f1 (nc,), all_ap (nc, 10), ap_class_index (nc,)), and the means segment/val.py and segment/train.py print and
    log.  Every mean is 0.0 and every per-class array [] before the first update or when no class has labels."""

    def __init__(self) -> None:
        self.p = []
        self.r = []
        self.f1 = []
        self.all_ap = []
        self.ap_class_index = []

    @property
    def ap50(self):
        """AP at IoU 0.5 per class, (nc,) or []."""
        return self.all_ap[:, 0] if len(self.all_ap) else []

    @property
    def ap(self):
        """AP averaged over the IoU thresholds 0.5:0.95 per class, (nc,) or []."""
        return self.all_ap.mean(1) if len(self.all_ap) else []

    @property
    def mp(self):
        """Precision averaged over the classes."""
        return self.p.mean() if len(self.p) else 0.0

    @property
    def mr(self):
        """Recall averaged over the classes."""
        return self.r.mean() if len(self.r) else 0.0

    @property
    def map50(self):
        """AP at IoU 0.5 averaged over the classes."""
        return self.all_ap[:, 0].mean() if len(self.all_ap) else 0.0

    @property
    def map(self):
        """AP averaged over the classes and the thresholds 0.5:0.95."""
        return self.all_ap.mean() if len(self.all_ap) else 0.0

    def mean_results(self):
        """(mp, mr, map50, map)."""
        return self.mp, self.mr, self.map50, self.map

    def class_result(self, i):
        """(p, r, ap50, ap) of the i-th class with results (index into ap_class_index, not a class id)."""
        return self.p[i], self.r[i], self.ap50[i], self.ap[i]

    def get_maps(self, nc):
        """(nc,) float64: each class's AP@0.5:0.95, and map for the classes without results."""
        maps = np.full(nc, self.map, dtype=np.float64)
        ap = self.ap
        for i, c in enumerate(self.ap_class_index):
            maps[c] = ap[i]
        return maps

    def update(self, results):
        """results = (p, r, all_ap, f1, ap_class_index), the values of one ap_per_class_box_and_mask entry in its order."""
        self.p, self.r, self.all_ap, self.f1, self.ap_class_index = results


class Metrics:
    """Reference utils/segment/metrics.py Metrics: a Metric for boxes and one for masks, fed by ap_per_class_box_and_mask;
    results concatenate box then mask."""

    def __init__(self) -> None:
        self.metric_box = Metric()
        self.metric_mask = Metric()

    def update(self, results):
        """results = ap_per_class_box_and_mask's dict {"boxes": {...}, "masks": {...}}."""
        self.metric_box.update(list(results["boxes"].values()))
        self.metric_mask.update(list(results["masks"].values()))

    def mean_results(self):
        """Box (mp, mr, map50, map) followed by the mask's: 8 values."""
        return self.metric_box.mean_results() + self.metric_mask.mean_results()

    def class_result(self, i):
        """Box (p, r, ap50, ap) of result i followed by the mask's."""
        return self.metric_box.class_result(i) + self.metric_mask.class_result(i)

    def get_maps(self, nc):
        """Box per-class mAPs plus the mask's, element by element (nc,)."""
        return self.metric_box.get_maps(nc) + self.metric_mask.get_maps(nc)

    @property
    def ap_class_index(self):
        """The classes with results (the box and mask entries share them)."""
        return self.metric_box.ap_class_index


# the columns of segment/train.py's results.csv: 4 training losses, box and mask P / R / mAP@0.5 / mAP@0.5:0.95, 4 validation
# losses and the 3 learning rates
KEYS = [f"train/{k}_loss" for k in ("box", "seg", "obj", "cls")] + [
    f"metrics/{k}({t})" for t in "BM" for k in ("precision", "recall", "mAP_0.5", "mAP_0.5:0.95")] + [
    f"val/{k}_loss" for k in ("box", "seg", "obj", "cls")] + [f"x/lr{i}" for i in range(3)]
