"""Generate tests/golden/confusion.npz by running the UNMODIFIED reference's ConfusionMatrix (utils/metrics.py:129-221),
`fitness` (utils/metrics.py:19) and segment `fitness` / `Metric` / `Metrics` (utils/segment/metrics.py) through
tests/golden/refshim.py on torch-cpu tensors.

Runs only where the reference tree exists:
    python tests/golden/make_confusion_golden.py
Every case is one ConfusionMatrix fed a list of process_batch calls; it stores the calls' inputs, the reference's matrix
(`.reference`, the host's default numpy argsort) and the matrix under the stable order the engine defines (`.stable`,
oracle/confusion_ref.py).  While generating, the oracle run with the reference's own sort must reproduce `.reference` on every
case (hard assert); `meta` records the cases where the two orders give different matrices (equal IoUs between classes).
"""
from __future__ import annotations

import inspect
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import confusion_ref  # noqa: E402

F = np.float32


def _coco_calls(seed, n_img, nc=80):
    rows, count, lab6 = confusion_ref.synth_batch(n_img, 300, nc, 7.3, seed=seed)
    calls = []
    for b in range(n_img):  # val.py's branching: no rows -> detections=None, no labels -> no call
        lab = lab6[lab6[:, 0] == b, 1:]
        if count[b] == 0 and len(lab):
            calls.append((None, lab[:, 0]))
        elif len(lab):
            calls.append((rows[b, :count[b], :6], lab))
    return calls


def _tie_calls():
    """Duplicate boxes and duplicate labels of different classes: equal IoUs decide which class is counted."""
    box = [10, 10, 110, 60]
    dup_dets = np.array([box + [0.9, 1], box + [0.8, 2], box + [0.7, 3]], F)
    one_label = np.array([[5] + box], F)
    dup_labels = np.array([[4] + box, [6] + box, [7] + box], F)
    near = np.array([[4, 10, 10, 110, 62], [6, 10, 8, 110, 60]], F)  # both IoU 50/52 with `box`
    many = np.concatenate([np.array([[c, 10 * c, 0, 10 * c + 40, 40]], F) for c in range(8)] * 3)  # 24 labels, 8 distinct boxes
    many_dets = np.concatenate([np.array([[10 * c, 0, 10 * c + 40, 40, 0.5 + 0.01 * c, (c + 1) % 8]], F) for c in range(8)] * 3)
    return [(dup_dets, one_label), (dup_dets[:1], dup_labels), (dup_dets, dup_labels), (dup_dets[:2], near), (many_dets, many)]


def cases():
    out = {}
    out["coco_a"] = (80, 0.25, 0.45, _coco_calls(1, 24))
    out["coco_b"] = (80, 0.25, 0.45, _coco_calls(2, 16))
    empty5 = np.zeros((0, 5), F)
    empty6 = np.zeros((0, 6), F)
    lab = np.array([[3, 0, 0, 50, 50], [7, 100, 100, 200, 160]], F)
    far = np.array([[300, 300, 400, 400, 0.9, 3], [0, 0, 50, 50, 0.2, 3]], F)  # no overlap; the overlapping one is below conf
    out["no_detections"] = (10, 0.25, 0.45, [(empty6, lab)])
    out["no_labels"] = (10, 0.25, 0.45, [(far, empty5)])
    out["no_match"] = (10, 0.25, 0.45, [(far, lab)])  # labels background, no detection counted
    # conf exactly 0.25 is dropped; IoU exactly fp32(0.45) (9 / 20) is no candidate; fp32 just above either is kept
    g = np.array([[2, 0, 0, 20, 1]], F)
    at = np.array([[0, 0, 9, 1, 0.9, 2], [0, 0, 20, 1, 0.25, 1]], F)
    above = np.array([[0, 0, 20, 1, np.nextafter(F(0.25), F(1)), 1]], F)
    out["thresholds"] = (5, 0.25, 0.45, [(at, g), (above, g)])
    out["thresholds_other"] = (5, 0.3, 0.6, [(np.array([[0, 0, 20, 1, 0.3, 1], [0, 0, 12, 1, F(0.3) * F(1.0000001), 1]], F), g)])
    out["ties"] = (8, 0.25, 0.45, _tie_calls())
    out["detections_none"] = (80, 0.25, 0.45, [(None, np.array([0, 5, 5, 79], F)), (None, np.zeros(0, F))])
    out["nc1"] = (1, 0.25, 0.45, _nc1_calls())
    return out


def _nc1_calls():
    calls = []
    for d, lab in _coco_calls(3, 6, nc=1):
        if d is not None:
            d = d.copy()
            d[:, 5] = 0
        calls.append((d, lab))
    return calls


def _run(cm_cls, nc, conf, iou, calls):
    import torch

    cm = cm_cls(nc=nc, conf=conf, iou_thres=iou)
    for d, lab in calls:
        cm.process_batch(None if d is None else torch.from_numpy(d), torch.from_numpy(lab))
    return cm.matrix


def _metric_inputs():
    rs = np.random.RandomState(7)
    out = {"fitness_x": rs.rand(5, 7), "seg_fitness_x": rs.rand(4, 12)}
    nc_res = 6
    for t in ("boxes", "masks"):
        out[f"{t}_p"], out[f"{t}_r"], out[f"{t}_f1"] = rs.rand(nc_res), rs.rand(nc_res), rs.rand(nc_res)
        out[f"{t}_ap"] = np.sort(rs.rand(nc_res, 10), 1)[:, ::-1].copy()
    out["ap_class"] = np.array([0, 2, 3, 7, 11, 12])
    return out


def metrics_record(fitness, seg_fitness, metrics_cls, x):
    """Outputs of fitness, segment fitness and a Metrics fed the fixed results (the same calls for reference and engine)."""
    out = {"fitness": np.asarray(fitness(x["fitness_x"])), "seg_fitness": np.asarray(seg_fitness(x["seg_fitness_x"]))}
    m = metrics_cls()
    out["empty_mean_results"] = np.array(m.mean_results(), np.float64)
    out["empty_maps"] = np.asarray(m.get_maps(15))
    res = {t: {"p": x[f"{t}_p"], "r": x[f"{t}_r"], "ap": x[f"{t}_ap"], "f1": x[f"{t}_f1"], "ap_class": x["ap_class"]} for t in ("boxes", "masks")}
    m.update(res)
    out["mean_results"] = np.array(m.mean_results(), np.float64)
    out["class_results"] = np.array([m.class_result(i) for i in range(len(x["ap_class"]))], np.float64)
    out["maps"] = np.asarray(m.get_maps(15))
    out["ap_class_index"] = np.asarray(m.ap_class_index)
    for t, metric in (("box", m.metric_box), ("mask", m.metric_mask)):
        for k in ("ap50", "ap", "mp", "mr", "map50", "map"):
            out[f"{t}_{k}"] = np.asarray(getattr(metric, k), np.float64)
    return out


SIGNATURES = [("utils.metrics", "ConfusionMatrix.__init__"), ("utils.metrics", "ConfusionMatrix.process_batch"),
              ("utils.metrics", "ConfusionMatrix.plot"), ("utils.metrics", "ConfusionMatrix.print"), ("utils.metrics", "fitness"),
              ("utils.segment.metrics", "fitness"), ("utils.segment.metrics", "Metric.__init__"), ("utils.segment.metrics", "Metric.update"),
              ("utils.segment.metrics", "Metric.mean_results"), ("utils.segment.metrics", "Metric.class_result"),
              ("utils.segment.metrics", "Metric.get_maps"), ("utils.segment.metrics", "Metrics.__init__"),
              ("utils.segment.metrics", "Metrics.update"), ("utils.segment.metrics", "Metrics.mean_results"),
              ("utils.segment.metrics", "Metrics.class_result"), ("utils.segment.metrics", "Metrics.get_maps")]


def signatures():
    import importlib

    out = {}
    for mod, qual in SIGNATURES:
        obj = importlib.import_module(mod)
        for part in qual.split("."):
            obj = getattr(obj, part)
        out[f"{mod}:{qual}"] = [(n, repr(p.default) if p.default is not inspect._empty else None, str(p.kind))
                                for n, p in inspect.signature(obj).parameters.items()]
    return out


def main():
    sys.path.insert(0, HERE)
    import refshim

    refshim.install()
    from utils.metrics import ConfusionMatrix, fitness
    from utils.segment import metrics as seg

    store, meta = {}, {"cases": {}}
    for tag, (nc, conf, iou, calls) in cases().items():
        store[f"{tag}.params"] = np.array([nc, conf, iou], np.float64)
        for k, (d, lab) in enumerate(calls):
            if d is not None:
                store[f"{tag}.{k}.det"] = d
            store[f"{tag}.{k}.lab"] = lab
        ref = _run(ConfusionMatrix, nc, conf, iou, calls)
        stable = np.zeros((nc + 1, nc + 1))
        default = np.zeros((nc + 1, nc + 1))
        for d, lab in calls:
            confusion_ref.process_batch(stable, d, lab, nc, conf, iou, stable=True)
            confusion_ref.process_batch(default, d, lab, nc, conf, iou, stable=False)
        assert np.array_equal(default, ref), (tag, "oracle with the reference's sort != reference")
        store[f"{tag}.reference"] = ref
        store[f"{tag}.stable"] = stable
        meta["cases"][tag] = dict(nc=nc, calls=len(calls), total=float(ref.sum()), default_equals_stable=bool(np.array_equal(ref, stable)))
        print(f"confusion {tag}: {meta['cases'][tag]}")
    x = _metric_inputs()
    for k, v in x.items():
        store[f"metrics.in.{k}"] = v
    ref_m = metrics_record(fitness, seg.fitness, seg.Metrics, x)
    ours = metrics_record(confusion_ref.fitness, confusion_ref.seg_fitness, seg.Metrics, x)
    for k, v in ref_m.items():
        store[f"metrics.out.{k}"] = v
    assert np.array_equal(ours["fitness"], ref_m["fitness"]) and np.array_equal(ours["seg_fitness"], ref_m["seg_fitness"])
    maps = 0
    for t, group in (("box", "boxes"), ("mask", "masks")):
        s = confusion_ref.metric_summary(x[f"{group}_p"], x[f"{group}_r"], x[f"{group}_ap"], x["ap_class"], 15)
        for k in ("ap50", "ap", "mp", "mr", "map50", "map"):
            assert np.array_equal(np.asarray(s[k], np.float64), ref_m[f"{t}_{k}"]), (t, k)
        maps = maps + s["maps"]
    assert np.array_equal(maps, ref_m["maps"])
    meta["signatures"] = signatures()
    meta["keys"] = list(seg.KEYS)
    store["meta"] = np.array(json.dumps(meta, sort_keys=True))
    np.savez_compressed(f"{HERE}/confusion.npz", **store)
    print("written", f"{HERE}/confusion.npz", os.path.getsize(f"{HERE}/confusion.npz"), "bytes")


if __name__ == "__main__":
    main()
