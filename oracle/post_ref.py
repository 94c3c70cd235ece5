"""ORACLE (test infrastructure, never on the product path): CPU restatement of the steps right after NMS -- the rows
SURVEY.md section 8(f) ranks next: mask post-processing and device-side metric matching.  numpy, float32 unless noted.

Only tests/ (and later __graft_entry__.smoke() / bench.py's baseline legs) may import this.  The CUDA kernels for these
rows are not built yet; this file and tests/golden/post.npz are the checker they will be held to.

Pinned: tests/golden/post.npz holds outputs of the real reference (tests/golden/make_golden.py post, through
tests/golden/refshim.py); tests/test_oracle_golden.py checks this file against them.  `box_iou` / `clip_boxes` come from
the absent `ultralytics` package in the reference: pinned only to the shim's restatement.

Reference lines restated (paths relative to /root/reference):
  utils/segment/general.py:10-22   crop_mask                      -> crop_mask
  utils/segment/general.py:25-52   process_mask                   -> process_mask
  utils/segment/general.py:55-76   process_mask_native            -> process_mask_native
  utils/general.py:613-626         scale_boxes (+ clip_boxes)     -> scale_boxes
  utils/metrics.py:224-265         process_batch (box branch)     -> process_batch
"""
from __future__ import annotations

import numpy as np

from . import nms_ref


def crop_mask(masks: np.ndarray, boxes: np.ndarray) -> np.ndarray:
    """Zero everything outside each mask's xyxy box (half-open on the right/bottom).  masks (n,h,w), boxes (n,4)."""
    n, h, w = masks.shape
    xs = np.arange(w, dtype=boxes.dtype)[None, None, :]
    ys = np.arange(h, dtype=boxes.dtype)[None, :, None]
    x1, y1, x2, y2 = (boxes[:, i][:, None, None] for i in range(4))
    keep = (xs >= x1) & (xs < x2) & (ys >= y1) & (ys < y2)
    return masks * keep


def bilinear_resize(x: np.ndarray, out_hw) -> np.ndarray:
    """F.interpolate(mode='bilinear', align_corners=False) on the last two dims; fp32 arithmetic like torch's CPU kernel
    (source index max(0, (dst + 0.5) * in/out - 0.5), neighbour clamped to the last row/column)."""
    n, h, w = x.shape
    oh, ow = out_hw

    def axis(inp, out):
        scale = np.float32(inp) / np.float32(out)
        src = np.maximum((np.arange(out, dtype=np.float32) + np.float32(0.5)) * scale - np.float32(0.5), np.float32(0))
        i0 = np.minimum(src.astype(np.int64), inp - 1)
        i1 = np.minimum(i0 + 1, inp - 1)
        lam = (src - i0.astype(np.float32)).astype(np.float32)
        return i0, i1, lam

    y0, y1, ly = axis(h, oh)
    x0, x1, lx = axis(w, ow)
    x = x.astype(np.float32)
    one = np.float32(1)
    top = x[:, y0][:, :, x0] * (one - lx)[None, None, :] + x[:, y0][:, :, x1] * lx[None, None, :]
    bot = x[:, y1][:, :, x0] * (one - lx)[None, None, :] + x[:, y1][:, :, x1] * lx[None, None, :]
    return (top * (one - ly)[None, :, None] + bot * ly[None, :, None]).astype(np.float32)


def process_mask(protos: np.ndarray, masks_in: np.ndarray, bboxes: np.ndarray, shape, upsample: bool = False):
    """protos (c,mh,mw), masks_in (n,c) mask coefficients of the kept detections, bboxes (n,4) xyxy in input-image pixels,
    shape = (ih, iw) of the network input.  Returns (binary masks float32 {0,1}, the pre-threshold values)."""
    c, mh, mw = protos.shape
    ih, iw = shape
    logits = masks_in.astype(np.float32) @ protos.astype(np.float32).reshape(c, -1)
    m = (np.float32(1) / (np.float32(1) + np.exp(-logits, dtype=np.float32))).reshape(-1, mh, mw)
    b = bboxes.astype(np.float32).copy()
    b[:, 0] *= np.float32(mw / iw)
    b[:, 2] *= np.float32(mw / iw)
    b[:, 3] *= np.float32(mh / ih)
    b[:, 1] *= np.float32(mh / ih)
    m = crop_mask(m, b)
    if upsample:
        m = bilinear_resize(m, (ih, iw))
    return (m > np.float32(0.5)).astype(np.float32), m


def process_mask_native(protos: np.ndarray, masks_in: np.ndarray, bboxes: np.ndarray, shape):
    """Up-sample the un-padded window of the prototype-resolution masks to `shape`, THEN crop with the (un-scaled) boxes."""
    c, mh, mw = protos.shape
    logits = masks_in.astype(np.float32) @ protos.astype(np.float32).reshape(c, -1)
    m = (np.float32(1) / (np.float32(1) + np.exp(-logits, dtype=np.float32))).reshape(-1, mh, mw)
    gain = min(mh / shape[0], mw / shape[1])
    pad = (mw - shape[1] * gain) / 2, (mh - shape[0] * gain) / 2
    top, left = int(pad[1]), int(pad[0])
    bottom, right = int(mh - pad[1]), int(mw - pad[0])
    m = bilinear_resize(m[:, top:bottom, left:right], shape)
    m = crop_mask(m, bboxes.astype(np.float32))
    return (m > np.float32(0.5)).astype(np.float32), m


def scale_boxes(img1_shape, boxes: np.ndarray, img0_shape, ratio_pad=None) -> np.ndarray:
    """Map xyxy boxes from the letterboxed network input (img1) back to the original image (img0) and clip.  Returns a
    new array (the reference edits in place)."""
    if ratio_pad is None:
        gain = min(img1_shape[0] / img0_shape[0], img1_shape[1] / img0_shape[1])
        pad = (img1_shape[1] - img0_shape[1] * gain) / 2, (img1_shape[0] - img0_shape[0] * gain) / 2
    else:
        gain, pad = ratio_pad[0][0], ratio_pad[1]
    b = boxes.astype(np.float32).copy()
    b[..., [0, 2]] -= np.float32(pad[0])
    b[..., [1, 3]] -= np.float32(pad[1])
    b[..., :4] /= np.float32(gain)
    b[..., [0, 2]] = b[..., [0, 2]].clip(0, img0_shape[1])
    b[..., [1, 3]] = b[..., [1, 3]].clip(0, img0_shape[0])
    return b


def process_batch(detections: np.ndarray, labels: np.ndarray, iouv: np.ndarray) -> np.ndarray:
    """correct[N, len(iouv)] (bool): detection d counts as a true positive at threshold t if it is matched to a label of
    its class with IoU >= t.  Matching as the reference does it: candidates sorted by IoU descending; each detection keeps
    its best candidate; the survivors are then listed in DETECTION-INDEX order (np.unique sorts) and each label keeps the
    first of them -- i.e. the lowest-index detection among those whose best label it is, not the highest-IoU one.
    detections (N,6) [x1,y1,x2,y2,conf,cls], labels (M,5) [cls,x1,y1,x2,y2]."""
    n, m = detections.shape[0], labels.shape[0]
    correct = np.zeros((n, iouv.shape[0]), dtype=bool)
    if n == 0 or m == 0:
        return correct
    iou = nms_ref.box_iou(labels[:, 1:].astype(np.float32), detections[:, :4].astype(np.float32))  # (M, N)
    same = labels[:, 0:1] == detections[:, 5][None, :]
    for t, thr in enumerate(iouv):
        li, di = np.nonzero((iou >= thr) & same)
        if li.size == 0:
            continue
        v = iou[li, di]
        order = np.argsort(-v, kind="stable")          # IoU descending (ties keep (label, detection) scan order)
        li, di = li[order], di[order]
        _, first = np.unique(di, return_index=True)    # best candidate of every detection, now in detection order
        li, di = li[first], di[first]
        _, first = np.unique(li, return_index=True)    # first of them per label
        correct[di[first], t] = True
    return correct
