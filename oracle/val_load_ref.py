"""ORACLE (test infrastructure, never on the product path): CPU restatement of the validation dataloader's item,
LoadImagesAndLabels[AndMasks].__getitem__ with augment=False + collate_fn, in numpy.

Only tests/ and tools/ may import this.

Reference lines restated (paths relative to the reference tree):
  utils/dataloaders.py:768-790   load_image: resize to ceil(w0 r) x ceil(h0 r), r = img_size / max(h0, w0),
                                 INTER_AREA when r < 1, INTER_LINEAR when r > 1                 -> load_resize
  utils/dataloaders.py:711-736   letterbox(shape, auto=False, scaleup=False), label conversions   -> get_item
  utils/segment/dataloaders.py:144-199  segments, polygons2masks[_overlap], mask dtypes           -> get_item(masks=...)
  utils/dataloaders.py:858-863, utils/segment/dataloaders.py:295-301  collate_fn                  -> get_batch
Third-party arithmetic: OpenCV ``cv2.resize(..., INTER_AREA)`` on uint8 (opencv-python 4.13.0; its source is not
available here).  `resize_area_u8` restates what the installed cv2 computes, pinned by a size sweep against cv2 in
tests/test_val_load_cpu.py:
  * both ratios src / dst integers ("area fast"): the sum over each k_x x k_y cell; at 2 x 2 it is rounded as
    (sum + 2) >> 2, otherwise as round-half-even(float32(sum) * float32(1 / area));
  * otherwise the weighted-area tables: per axis, destination cell [d s, d s + s) with s = 1 / (dst / src) in double,
    partial first / last source pixels weighted (sx1 - f1) / w and min(f2 - sx2, 1) / w (skipped below 1e-3), whole
    ones 1 / w, w = min(s, src - f1); each source row is summed across its x weights in float32 (in table order,
    each product rounded), the rows are summed with their y weights in float32 in order, and the result is rounded
    half to even and saturated.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import pre_ref
from oracle import seg_aug_ref

PAD_VALUE = 114
INTERP_COPY, INTERP_LINEAR, INTERP_AREA = 0, 1, 2  # include/y5b200.h Y5_VAL_*


def _area_tab(src: int, dst: int):
    """Per destination index: the source indices and float32 weights of its area cell, in OpenCV's table order,
    padded with weight 0 (adding 0 * x leaves a float32 sum unchanged)."""
    scale = 1.0 / (dst / src)
    rows = []
    for d in range(dst):
        f1 = d * scale
        f2 = f1 + scale
        cw = min(scale, src - f1)
        s1, s2 = math.ceil(f1), math.floor(f2)
        s2 = min(s2, src - 1)
        s1 = min(s1, s2)
        ent = []
        if s1 - f1 > 1e-3:
            ent.append((s1 - 1, np.float32((s1 - f1) / cw)))
        for s in range(s1, s2):
            ent.append((s, np.float32(1.0 / cw)))
        if f2 - s2 > 1e-3:
            ent.append((s2, np.float32(min(min(f2 - s2, 1.0), cw) / cw)))
        rows.append(ent)
    k = max(len(e) for e in rows)
    idx = np.zeros((dst, k), np.int64)
    wt = np.zeros((dst, k), np.float32)
    for d, ent in enumerate(rows):
        for j, (s, a) in enumerate(ent):
            idx[d, j], wt[d, j] = s, a
    return idx, wt


def area_is_fast(src_hw, dst_hw):
    """OpenCV's is_area_fast: both scales 1 / (dst / src) within DBL_EPSILON of an integer."""
    eps = np.finfo(np.float64).eps
    out = []
    for s, d in zip(src_hw, dst_hw):
        sc = 1.0 / (d / s)
        out.append(abs(sc - round(sc)) < eps)
    return all(out)


def resize_area_u8(img: np.ndarray, dst_wh) -> np.ndarray:
    """cv2.resize(img, dst_wh, interpolation=cv2.INTER_AREA) for uint8 HWC images shrinking in both axes, bit-exact."""
    h, w = img.shape[:2]
    dw, dh = int(dst_wh[0]), int(dst_wh[1])
    if dw > w or dh > h:
        raise ValueError("resize_area_u8 restates the shrinking path only")
    if (dw, dh) == (w, h):
        return img.copy()
    if area_is_fast((h, w), (dh, dw)):
        kx, ky = round(w / dw), round(h / dh)
        s = img[: dh * ky, : dw * kx].astype(np.int64).reshape(dh, ky, dw, kx, -1).sum((1, 3))
        if kx == 2 and ky == 2:
            return ((s + 2) >> 2).astype(np.uint8)
        v = s.astype(np.float32) * np.float32(1.0 / np.float32(kx * ky))
        return np.clip(np.rint(v), 0, 255).astype(np.uint8)
    xi, xw = _area_tab(w, dw)
    yi, yw = _area_tab(h, dh)
    src = img.astype(np.float32)
    buf = np.zeros((h, dw, img.shape[2]), np.float32)
    for k in range(xi.shape[1]):
        buf = buf + src[:, xi[:, k]] * xw[None, :, k, None]
    acc = np.zeros((dh, dw, img.shape[2]), np.float32)
    for k in range(yi.shape[1]):
        acc = acc + yw[:, k, None, None] * buf[yi[:, k]]
    return np.clip(np.rint(acc), 0, 255).astype(np.uint8)


def load_size(hw0, img_size):
    """load_image's target (h, w) and interpolation for an original (h0, w0)."""
    h0, w0 = int(hw0[0]), int(hw0[1])
    r = img_size / max(h0, w0)
    if r == 1:
        return (h0, w0), INTERP_COPY
    return (math.ceil(h0 * r), math.ceil(w0 * r)), (INTERP_LINEAR if r > 1 else INTERP_AREA)


def load_resize(im0: np.ndarray, img_size: int) -> np.ndarray:
    """load_image's resize of an original BGR image (augment=False)."""
    (h, w), interp = load_size(im0.shape[:2], img_size)
    if interp == INTERP_COPY:
        return im0
    if interp == INTERP_LINEAR:
        return pre_ref.resize_linear_u8(im0, (w, h))
    return resize_area_u8(im0, (w, h))


def xywhn2xyxy(x, w, h, padw, padh):
    y = np.copy(x)
    y[..., 0] = w * (x[..., 0] - x[..., 2] / 2) + padw
    y[..., 1] = h * (x[..., 1] - x[..., 3] / 2) + padh
    y[..., 2] = w * (x[..., 0] + x[..., 2] / 2) + padw
    y[..., 3] = h * (x[..., 1] + x[..., 3] / 2) + padh
    return y


def xyxy2xywhn(x, w, h, eps=1e-3):
    """clip=True: clip_boxes to (h - eps, w - eps) in place, then the normalised centre form."""
    x[..., [0, 2]] = x[..., [0, 2]].clip(0, w - eps)
    x[..., [1, 3]] = x[..., [1, 3]].clip(0, h - eps)
    y = np.copy(x)
    y[..., 0] = ((x[..., 0] + x[..., 2]) / 2) / w
    y[..., 1] = ((x[..., 1] + x[..., 3]) / 2) / h
    y[..., 2] = (x[..., 2] - x[..., 0]) / w
    y[..., 3] = (x[..., 3] - x[..., 1]) / h
    return y


def label_rows(labels, ratio, w, h, pad, out_w, out_h):
    """(n, 5) float32 labels -> (n, 5) float32 [cls, xywhn] as __getitem__ converts them: float32 where the scales and
    pads are python floats (weak scalars), float64 before the float32 store where they are np.float64."""
    lab = labels.copy()
    if not lab.size:
        return lab
    lab[:, 1:] = xywhn2xyxy(lab[:, 1:], ratio[0] * w, ratio[1] * h, pad[0], pad[1])
    lab[:, 1:5] = xyxy2xywhn(lab[:, 1:5], out_w, out_h)
    return lab


def get_item(im, hw0, labels, shape, segments=None, overlap=False, ratio_ds=1):
    """One val item from the load_image output `im` -> (CHW RGB uint8, (n, 6) float32 rows, shapes[, masks]).  `shape`:
    the int img_size, or the dataset's batch_shapes row as it is (its numpy integers make letterbox's ratio and pads
    np.float64, which are not weak scalars: the label and segment maths then round like the reference's)."""
    h, w = im.shape[:2]
    h0, w0 = hw0
    out, ratio, pad = pre_ref.letterbox(im, shape, auto=False, scaleup=False)
    shapes = (h0, w0), ((h / h0, w / w0), pad)
    lab = label_rows(labels, ratio, w, h, pad, out.shape[1], out.shape[0])
    rows = np.zeros((len(lab), 6), np.float32)
    rows[:, 1:] = lab
    chw = pre_ref.to_chw_rgb(out)
    if segments is None:
        return chw, rows, shapes
    oh, ow = out.shape[:2]
    segs = [seg_aug_ref.xyn2xy(s, ratio[0] * w, ratio[1] * h, pad[0], pad[1]) for s in segments]
    if len(lab):
        if overlap:
            m, order = seg_aug_ref.polygons2masks_overlap((oh, ow), segs, ratio_ds)
            masks = m[None]
            rows = rows[order]
        else:
            masks = seg_aug_ref.polygons2masks((oh, ow), segs, 1, ratio_ds)
    else:
        masks = np.zeros((1 if overlap else 0, oh // ratio_ds, ow // ratio_ds), np.float32)
    return chw, rows, shapes, masks


def get_batch(items):
    """collate_fn over get_item results."""
    imgs = np.stack([it[0] for it in items])
    rows = [it[1].copy() for it in items]
    for i, r in enumerate(rows):
        r[:, 0] = i
    targets = np.concatenate(rows, 0) if rows else np.zeros((0, 6), np.float32)
    shapes = tuple(it[2] for it in items)
    if len(items[0]) == 3:
        return imgs, targets, shapes
    ms = [it[3] for it in items]
    dt = seg_aug_ref.batch_mask_dtype([m.dtype for m in ms])
    return imgs, targets, shapes, np.concatenate([m.astype(dt) for m in ms], 0)
