"""ORACLE (test infrastructure, never on the product path): process_batch(masks=True) of segment/val.py.

reference utils/metrics.py:239-265 with ultralytics' mask_iou (not under the reference tree; restated from its public
definition, parity unpinned like box_iou):
- ``expand_gt``: the overlap expansion, the bilinear resize and the strict > 0.5 in the reference's own torch expressions (CPU).
- ``mask_iou_exact``: integer intersections and unions, then the reference's single fp32 rounding.
- ``match``: the matching rule of oracle.post_ref.process_batch (first label in scan order on equal IoU) on a given IoU
  matrix; ``replay_reference_sort=True`` runs the reference's own `argsort()[::-1]` instead, whose order inside equal-IoU runs
  depends on numpy's sort (not stable) -- the fixture generator uses it to check the oracle against the reference exactly.
- ``case_inputs``: the seeded inputs of tests/golden/mask_val.npz (tests/golden/make_mask_val_golden.py).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from tests.seg_loss_ref import paint_masks

# tag: (overlap, nl, gt (h, w), pred (h, w), detections, seed, variant)
CASES = {
    "ov_sorted": (True, 8, (160, 160), (160, 160), 40, 1, "sorted"),
    "ov_unsorted": (True, 9, (160, 160), (160, 160), 40, 2, "shuffled"),
    "nonov": (False, 8, (160, 160), (160, 160), 40, 3, "shuffled"),
    "down640": (False, 7, (640, 640), (160, 160), 30, 4, "shuffled"),
    "up160": (False, 6, (160, 160), (640, 640), 24, 5, "shuffled"),
    "rect": (False, 7, (480, 640), (120, 160), 30, 6, "shuffled"),
    "odd_ratio": (False, 6, (100, 150), (160, 160), 24, 7, "shuffled"),
    "ov_resize": (True, 8, (640, 640), (160, 160), 36, 8, "shuffled"),
    "ov_index_oob": (True, 6, (160, 160), (160, 160), 30, 9, "oob"),
    "empty": (False, 6, (160, 160), (160, 160), 24, 10, "empty"),
    "nl1": (True, 1, (160, 160), (160, 160), 12, 11, "sorted"),
    "dup": (False, 6, (160, 160), (160, 160), 30, 12, "dup"),
}
IOUV = np.linspace(0.5, 0.95, 10).astype(np.float32)


def case_inputs(tag):
    """(detections (n,6) fp32 [x1,y1,x2,y2,conf,cls], labels (nl,5) fp32 [cls,x1,y1,x2,y2], pred_masks (n,h,w) fp32 0/1,
    gt_masks fp32: (1,H,W) label indices with overlap, else (nl,H,W) 0/1, overlap)."""
    overlap, nl, (gh, gw), (ph, pw), n, seed, variant = CASES[tag]
    rs = np.random.RandomState(seed)
    xy = rs.uniform(0.2, 0.8, (nl, 2))
    wh = rs.uniform(0.15, 0.45, (nl, 2))
    boxes = np.concatenate((xy, wh), 1).astype(np.float32)  # xywhn
    cls = np.sort(rs.randint(0, 4, nl)) if variant == "sorted" else rs.randint(0, 4, nl)
    if variant == "dup":  # labels 1 and 4 repeat labels 0 and 3: same polygon, same class
        boxes[1], cls[1], boxes[4], cls[4] = boxes[0], cls[0], boxes[3], cls[3]
    if overlap:
        gt = paint_masks((gh, gw), boxes, np.arange(1, nl + 1))[None]
        if variant == "oob":  # values above nl and a non-integer value match no label
            gt[0, : gh // 8, : gw // 8] = nl + 3
            gt[0, -gh // 8:, -gw // 8:] = 2.5
    else:
        holes = rs.uniform(size=(nl, gh, gw)) > 0.15
        gt = np.stack([paint_masks((gh, gw), boxes[i:i + 1], [1.0]) * holes[i] for i in range(nl)])
        if variant == "dup":
            gt[1], gt[4] = gt[0], gt[3]
        if variant == "empty":
            gt[2] = 0
    gt = gt.astype(np.float32)
    owner = rs.randint(0, nl, n)
    jitter = rs.normal(0, 0.03, (n, 4)).astype(np.float32)
    pb = boxes[owner] + jitter
    pred = np.stack([paint_masks((ph, pw), pb[i:i + 1], [1.0]) * (rs.uniform(size=(ph, pw)) > rs.choice([0.0, 0.05, 0.3]))
                     for i in range(n)]).astype(np.float32)
    if variant == "empty":
        pred[::5] = 0
    dcls = np.where(rs.uniform(size=n) < 0.85, cls[owner], rs.randint(0, 4, n)).astype(np.float32)
    xyxy = np.concatenate((pb[:, :2] - pb[:, 2:] / 2, pb[:, :2] + pb[:, 2:] / 2), 1) * np.array([pw, ph, pw, ph], np.float32)
    det = np.concatenate((xyxy, rs.uniform(0.001, 1, (n, 1)), dcls[:, None]), 1).astype(np.float32)
    lxyxy = np.concatenate((boxes[:, :2] - boxes[:, 2:] / 2, boxes[:, :2] + boxes[:, 2:] / 2), 1) * np.array([pw, ph, pw, ph], np.float32)
    labels = np.concatenate((cls[:, None].astype(np.float32), lxyxy), 1).astype(np.float32)
    return det, labels, pred, gt, overlap


def expand_gt(gt_masks: np.ndarray, nl: int, overlap: bool, out_hw):
    """(nl, oh, ow) fp32 0/1 gt masks as process_batch builds them, and the interpolated values before `gt_(0.5)` (None when
    the shapes already agree)."""
    g = torch.from_numpy(np.asarray(gt_masks, np.float32))
    if overlap:
        index = torch.arange(nl).view(nl, 1, 1) + 1
        g = torch.where(g.repeat(nl, 1, 1) == index, 1.0, 0.0)
    if tuple(g.shape[1:]) == tuple(out_hw):
        return g.numpy(), None
    v = F.interpolate(g[None], tuple(out_hw), mode="bilinear", align_corners=False)[0]
    return (v > 0.5).float().numpy(), v.numpy()


def mask_iou_exact(m1: np.ndarray, m2: np.ndarray, eps: float = 1e-7) -> np.ndarray:
    """(N, n) x (M, n) 0/1 -> (N, M) fp32: integer intersections and unions, then fl(inter / fl(union + eps))."""
    a = np.asarray(m1).reshape(m1.shape[0], -1).astype(np.int64)
    b = np.asarray(m2).reshape(m2.shape[0], -1).astype(np.int64)
    inter = a @ b.T
    union = a.sum(1)[:, None] + b.sum(1)[None] - inter
    return inter.astype(np.float32) / (union.astype(np.float32) + np.float32(eps))


def match(iou: np.ndarray, label_cls: np.ndarray, det_cls: np.ndarray, iouv: np.ndarray, replay_reference_sort: bool = False) -> np.ndarray:
    """correct (N, len(iouv)) bool from iou (M labels, N detections)."""
    n = iou.shape[1]
    correct = np.zeros((n, len(iouv)), bool)
    same = label_cls[:, None] == det_cls[None, :]
    for t, thr in enumerate(iouv):
        li, di = np.nonzero((iou >= thr) & same)
        if li.size == 0:
            continue
        if replay_reference_sort:  # utils/metrics.py:258-263 verbatim on the same float32 array
            matches = np.concatenate((np.stack((li, di), 1).astype(np.float32), iou[li, di][:, None]), 1)
            if li.size > 1:
                matches = matches[matches[:, 2].argsort()[::-1]]
                matches = matches[np.unique(matches[:, 1], return_index=True)[1]]
                matches = matches[np.unique(matches[:, 0], return_index=True)[1]]
            correct[matches[:, 1].astype(int), t] = True
            continue
        order = np.argsort(-iou[li, di], kind="stable")  # oracle.post_ref.process_batch's rule
        li, di = li[order], di[order]
        _, first = np.unique(di, return_index=True)
        li, di = li[first], di[first]
        _, first = np.unique(li, return_index=True)
        correct[di[first], t] = True
    return correct


def process_batch_masks(detections, labels, iouv, pred_masks, gt_masks, overlap, replay_reference_sort=False):
    """(correct (N, niou) bool, iou (nl, N) fp32, gt 0/1 masks at the prediction size, their pre-threshold values or None)."""
    nl = labels.shape[0]
    gt, vals = expand_gt(gt_masks, nl, overlap, pred_masks.shape[1:])
    iou = mask_iou_exact(gt.reshape(nl, -1), np.asarray(pred_masks).reshape(pred_masks.shape[0], -1))
    return match(iou, labels[:, 0], detections[:, 5], iouv, replay_reference_sort), iou, gt, vals


def pack_bits(masks: np.ndarray) -> np.ndarray:
    """The engine's bit rows (y5_mask_pack) of (n, h, w) 0/1 masks as int32 words: np.packbits little-endian, zero padded to
    a multiple of 256 pixels."""
    n = masks.shape[0]
    flat = np.asarray(masks).reshape(n, int(np.prod(masks.shape[1:]))) != 0
    px = flat.shape[1]
    padded = np.zeros((n, (px + 255) // 256 * 256), bool)
    padded[:, :px] = flat
    return np.packbits(padded, axis=1, bitorder="little").view("<i4")


def process_batch_torch(detections, labels, iouv, pred_masks=None, gt_masks=None, overlap=False, masks=False):
    """The reference's process_batch (utils/metrics.py:224-265) in its own torch expressions on any device, with mask_iou
    and box_iou restated: the torch-cuda arm of tools/seg_val_bench.py."""
    if masks:
        if overlap:
            nl = len(labels)
            index = torch.arange(nl, device=gt_masks.device).view(nl, 1, 1) + 1
            gt_masks = gt_masks.repeat(nl, 1, 1)
            gt_masks = torch.where(gt_masks == index, 1.0, 0.0)
        if gt_masks.shape[1:] != pred_masks.shape[1:]:
            gt_masks = F.interpolate(gt_masks[None], pred_masks.shape[1:], mode="bilinear", align_corners=False)[0]
            gt_masks = gt_masks.gt_(0.5)
        m1, m2 = gt_masks.view(gt_masks.shape[0], -1), pred_masks.view(pred_masks.shape[0], -1)
        inter = torch.matmul(m1, m2.T).clamp_(0)
        iou = inter / ((m1.sum(1)[:, None] + m2.sum(1)[None]) - inter + 1e-7)
    else:
        (a1, a2), (b1, b2) = labels[:, 1:].float().unsqueeze(1).chunk(2, 2), detections[:, :4].float().unsqueeze(0).chunk(2, 2)
        inter = (torch.min(a2, b2) - torch.max(a1, b1)).clamp_(0).prod(2)
        iou = inter / ((a2 - a1).prod(2) + (b2 - b1).prod(2) - inter + 1e-7)
    correct = np.zeros((detections.shape[0], iouv.shape[0])).astype(bool)
    correct_class = labels[:, 0:1] == detections[:, 5]
    for i in range(len(iouv)):
        x = torch.where((iou >= iouv[i]) & correct_class)
        if x[0].shape[0]:
            matches = torch.cat((torch.stack(x, 1), iou[x[0], x[1]][:, None]), 1).cpu().numpy()
            if x[0].shape[0] > 1:
                matches = matches[matches[:, 2].argsort()[::-1]]
                matches = matches[np.unique(matches[:, 1], return_index=True)[1]]
                matches = matches[np.unique(matches[:, 0], return_index=True)[1]]
            correct[matches[:, 1].astype(int), i] = True
    return torch.tensor(correct, dtype=torch.bool, device=iouv.device)
