"""numpy restatement of the reference's ConfusionMatrix.process_batch (utils/metrics.py:139-183), of val.py's per-image calls
to it (val.py:282-309, segment/val.py:263-297), and of the host bookkeeping `fitness` (utils/metrics.py:19-22) and
`Metric` / `Metrics` / segment `fitness` (utils/segment/metrics.py).

Order of equal IoUs.  The reference sorts its candidate list twice with `argsort()[::-1]` (numpy's default kind), whose order
among equal values depends on the array's length and the host.  The defined order here, and in the engine, is numpy's stable
sort of the negated IoU: equal IoUs keep the (label, detection) scan order, so a detection keeps the first of its equally
good labels and a label the first of its equally good detections.  `stable=False` runs the reference's own expression
instead (what tests/golden/make_confusion_golden.py checks against the unmodified reference on the host that wrote it).

Also: `process_batch_torch`, the reference's per-image expressions on torch tensors (device IoU, `.cpu()` of the matches,
counts indexed by 0-d tensors) as a timing baseline, and `synth_batch`, COCO-like padded rows and labels for the tests and
tools/confusion_bench.py."""
from __future__ import annotations

import numpy as np

from . import ap_ref, nms_ref


def _descending(v, stable):
    if stable:
        return np.argsort(-v, kind="stable")
    return v.argsort()[::-1]


def _match(iou, iou_thres, stable):
    """(label, detection) index pairs kept by the two np.unique passes of process_batch (utils/metrics.py:160-169)."""
    li, di = np.nonzero(iou > np.float32(iou_thres))
    if li.size > 1:
        m = np.stack((li.astype(np.float32), di.astype(np.float32), iou[li, di]), 1)  # float32, as torch.cat promotes
        m = m[_descending(m[:, 2], stable)]
        m = m[np.unique(m[:, 1], return_index=True)[1]]  # each detection: its first (best) label
        m = m[_descending(m[:, 2], stable)]
        m = m[np.unique(m[:, 0], return_index=True)[1]]  # each label: its first (best) detection
        li, di = m[:, 0].astype(int), m[:, 1].astype(int)
    return li, di


def process_batch(matrix, detections, labels, nc, conf=0.25, iou_thres=0.45, stable=True):
    """Add one process_batch call into `matrix` ((nc+1, nc+1), in place).  detections (N,6) float32 [x1,y1,x2,y2,conf,cls]
    or None, labels (M,5) float32 [cls,x1,y1,x2,y2] (with detections=None: (M,) classes)."""
    if detections is None:
        for gc in np.asarray(labels, np.float32).astype(np.int32):
            matrix[nc, gc] += 1
        return matrix
    det = np.asarray(detections, np.float32)
    lab = np.asarray(labels, np.float32).reshape(-1, 5)
    det = det[det[:, 4] > np.float32(conf)]
    gt_cls = lab[:, 0].astype(np.int32)
    det_cls = det[:, 5].astype(np.int32)
    iou = nms_ref.box_iou(lab[:, 1:], det[:, :4]) if len(lab) and len(det) else np.zeros((len(lab), len(det)), np.float32)
    li, di = _match(iou, iou_thres, stable)
    for i, gc in enumerate(gt_cls):
        hit = di[li == i]
        matrix[det_cls[hit[0]] if li.size and hit.size == 1 else nc, gc] += 1
    if li.size:
        for d in np.setdiff1d(np.arange(len(det)), di):
            matrix[det_cls[d], nc] += 1
    return matrix


def val_loop(matrix, rows, count, labels6, nc, conf=0.25, iou_thres=0.45, stable=True):
    """val.py's per-image calls for a padded batch: rows (B, max_det, >=6) in native pixels, count (B,), labels6 (nt,6)
    [img, cls, x1,y1,x2,y2].  An image without rows and with labels: process_batch(None, classes); with rows and labels:
    process_batch(rows[:, :6], labels); without labels: no call."""
    rows, labels6 = np.asarray(rows, np.float32), np.asarray(labels6, np.float32).reshape(-1, 6)
    for si in range(rows.shape[0]):
        lab = labels6[labels6[:, 0] == si, 1:]
        pred = rows[si, :int(count[si]), :6]
        if len(pred) == 0:
            if len(lab):
                process_batch(matrix, None, lab[:, 0], nc, conf, iou_thres, stable)
            continue
        if len(lab):
            process_batch(matrix, pred, lab, nc, conf, iou_thres, stable)
    return matrix


def process_batch_torch(matrix, detections, labels, nc, conf=0.25, iou_thres=0.45):
    """The reference's per-image expressions on torch tensors (a timing baseline): IoU, candidate search and the float32
    match table on the tensors' device, one `.cpu()` of the matches, then the counts indexed by 0-d tensors of the
    detections' device (each index a device read)."""
    import torch

    if detections is None:
        for gc in labels.int():
            matrix[nc, gc] += 1
        return matrix
    det = detections[detections[:, 4] > conf]
    gt_cls = labels[:, 0].int()
    det_cls = det[:, 5].int()
    a, b = labels[:, 1:].unsqueeze(1), det[:, :4].unsqueeze(0)
    inter = (torch.min(a[..., 2:], b[..., 2:]) - torch.max(a[..., :2], b[..., :2])).clamp(0).prod(2)
    iou = inter / ((a[..., 2:] - a[..., :2]).prod(2) + (b[..., 2:] - b[..., :2]).prod(2) - inter + 1e-7)
    li, di = torch.where(iou > iou_thres)
    if li.shape[0]:
        m = torch.cat((torch.stack((li, di), 1), iou[li, di][:, None]), 1).cpu().numpy()
        if m.shape[0] > 1:
            m = m[_descending(m[:, 2], False)]
            m = m[np.unique(m[:, 1], return_index=True)[1]]
            m = m[_descending(m[:, 2], False)]
            m = m[np.unique(m[:, 0], return_index=True)[1]]
    else:
        m = np.zeros((0, 3))
    m0, m1 = m[:, 0].astype(int), m[:, 1].astype(int)
    for i, gc in enumerate(gt_cls):
        hit = m1[m0 == i]
        if m.shape[0] and hit.size == 1:
            matrix[det_cls[hit[0]], gc] += 1
        else:
            matrix[nc, gc] += 1
    if m.shape[0]:
        for i, dc in enumerate(det_cls):
            if not any(m1 == i):
                matrix[dc, nc] += 1
    return matrix


def synth_batch(n_img, max_det=300, nc=80, mean_labels=7.3, seed=0, size=640.0, extra_cols=0):
    """COCO-like padded validation rows and labels in native pixels: ap_ref.synth_stats' classes, fp16-rounded confidences
    and Poisson(mean_labels) labels per image, boxes drawn so that some detections overlap a label (jittered copies, of
    its class or another) and the rest fall anywhere.  Returns rows (n_img, max_det, 6 + extra_cols) float32 (padding
    rows random), count (n_img,) int32, labels6 (nt, 6) float32 [img, cls, x1,y1,x2,y2] in image order."""
    rs = np.random.RandomState(seed + 1)
    stats = ap_ref.synth_stats(n_img, max_det, nc, mean_labels, 1, seed, ties=True)

    def boxes(k):
        c = rs.rand(k, 2) * size
        wh = (rs.rand(k, 2) ** 2 * 0.5 + 0.02) * size
        return np.clip(np.concatenate((c - wh / 2, c + wh / 2), 1), 0, size).astype(np.float32)

    rows = (rs.rand(n_img, max_det, 6 + extra_cols) * size).astype(np.float32)
    count = np.zeros(n_img, np.int32)
    labels = []
    for b, (correct, conf, pc, tc) in enumerate(stats):
        lb = boxes(len(tc))
        labels.append(np.concatenate((np.full((len(tc), 1), b, np.float32), tc[:, None], lb), 1))
        n = len(conf)
        db = boxes(n)
        near = rs.rand(n) < 0.6
        if len(tc):
            src = np.where(correct[:, 0], -1, rs.randint(0, len(tc), n))
            for d in np.nonzero(near)[0]:
                same = np.nonzero(tc == pc[d])[0] if src[d] < 0 else []
                j = rs.choice(same) if len(same) else rs.randint(0, len(tc))
                w = np.array([lb[j, 2] - lb[j, 0], lb[j, 3] - lb[j, 1]] * 2, np.float32)
                jitter = 0.03 if src[d] < 0 else 0.15  # true positives sit tighter than the rest
                db[d] = np.clip(lb[j] + (rs.randn(4) * jitter * w).astype(np.float32), 0, size)
        rows[b, :n, :4] = db
        rows[b, :n, 4] = conf
        rows[b, :n, 5] = pc
        count[b] = n
    lab6 = np.concatenate(labels, 0) if labels else np.zeros((0, 6), np.float32)
    return rows, count, lab6.astype(np.float32)


def fitness(x):
    """utils/metrics.py:19: 0.1 * mAP@0.5 + 0.9 * mAP@0.5:0.95 per row of [P, R, mAP@0.5, mAP@0.5:0.95, ...]."""
    x = np.asarray(x)
    return np.sum(x[:, :4] * np.array([0.0, 0.0, 0.1, 0.9]), axis=1)


def seg_fitness(x):
    """utils/segment/metrics.py fitness: the same weights on the box and the mask groups of [P, R, mAP50, mAP] x 2."""
    x = np.asarray(x)
    return np.sum(x[:, :8] * np.array([0.0, 0.0, 0.1, 0.9] * 2), axis=1)


def metric_summary(p, r, all_ap, ap_class, nc):
    """Every quantity segment Metric derives from (p, r, all_ap, f1, ap_class) after update(), as a dict of numpy values;
    an empty result (no classes) gives the reference's defaults ([] per class, 0.0 means)."""
    p, r, all_ap = np.asarray(p), np.asarray(r), np.asarray(all_ap)
    has = len(all_ap) > 0
    ap = all_ap.mean(1) if has else np.zeros(0)
    mean_ap = all_ap.mean() if has else 0.0
    maps = np.full(nc, mean_ap, np.float64)
    for i, c in enumerate(ap_class):
        maps[c] = ap[i]
    return {"ap50": all_ap[:, 0] if has else np.zeros(0), "ap": ap, "mp": p.mean() if len(p) else 0.0, "mr": r.mean() if len(r) else 0.0,
            "map50": all_ap[:, 0].mean() if has else 0.0, "map": mean_ap, "maps": maps}
