"""Metric matching of the validation loop on the device (reference utils/metrics.py:224-265 process_batch, box_iou as used
at :158,:252, and the per-image loops of val.py:282-318 and segment/val.py:263-298): box IoU or mask IoU, class test and the
detection<->label matching rule for the WHOLE batch, with no `.cpu()` round trip per image.  Mask IoU (ultralytics'
mask_iou, imported by the reference into utils.metrics) is a 1-bit GEMM on the tensor cores: every quantity before the one
fp32 division is an integer pixel count, so it is bit-exact.

The last step of validation, ap_per_class (utils/metrics.py:25-126, val.py:328-330), runs on the device too (y5_ap_per_class):
one sort of the predictions, then every class and IoU threshold in float64, equal to the reference's numpy arithmetic bit for
bit under the stable confidence order (see DESIGN.md).  ap_per_class_batch reads the padded per-batch tensors directly.

ConfusionMatrix (utils/metrics.py:129-221) counts on the device (y5_confusion_batch): its updates never wait for the device,
and reading `matrix` syncs once.  `fitness` (utils/metrics.py:19-22) is the host weighting train.py applies to the results."""
from __future__ import annotations

import ctypes as C
import logging
import warnings
from pathlib import Path

import numpy as np
import torch

from .. import _lib


def box_iou(box1: torch.Tensor, box2: torch.Tensor, eps: float = 1e-7) -> torch.Tensor:
    """Pairwise IoU of xyxy boxes: (N,4) x (M,4) -> (N,M) fp32, computed by y5_box_iou on the device."""
    if not (box1.is_cuda and box2.is_cuda):
        raise RuntimeError("y5b200: box_iou runs on CUDA tensors only (no CPU / PyTorch fallback)")
    a = box1.float().contiguous()
    b = box2.float().contiguous()
    out = torch.empty(a.shape[0], b.shape[0], dtype=torch.float32, device=a.device)
    if out.numel():
        with _lib.on(a.device):
            _lib.check(_lib.lib().y5_box_iou(a.data_ptr(), a.shape[0], b.data_ptr(), b.shape[0], float(eps), out.data_ptr(),
                                             C.c_void_p(_lib.stream_ptr(a.device))), "box_iou")
    return out


def match_batch(det_rows: torch.Tensor, count, labels6: torch.Tensor, iouv: torch.Tensor, eps: float = 1e-7) -> torch.Tensor:
    """det_rows (B, max_det, >=6) fp32 [x1,y1,x2,y2,conf,cls,...] in native pixels (what scale_boxes produced), count (B,)
    int32 valid rows per image or None; labels6 (nt,6) [img, cls, x1,y1,x2,y2] native pixels -> correct (B, max_det, niou)
    bool on the device."""
    if not det_rows.is_cuda:
        raise RuntimeError("y5b200: process_batch runs on CUDA tensors only (no CPU / PyTorch fallback)")
    dev = det_rows.device
    assert det_rows.dtype == torch.float32 and det_rows.dim() == 3 and det_rows.stride(2) == 1 and det_rows.shape[2] >= 6
    b, max_det = det_rows.shape[:2]
    iouv = iouv.to(dev, torch.float32).contiguous()
    labels6 = labels6.to(dev, torch.float32).contiguous().view(-1, 6)
    correct = torch.empty(b, max_det, iouv.numel(), dtype=torch.uint8, device=dev)
    if b == 0 or max_det == 0:
        return correct.bool()
    cnt = count.to(dev, torch.int32).contiguous() if count is not None else None
    with _lib.on(dev):
        _lib.check(_lib.lib().y5_match_batch(det_rows.data_ptr(), det_rows.stride(0), det_rows.stride(1), cnt.data_ptr() if cnt is not None else None,
                                             b, max_det, labels6.data_ptr() if labels6.numel() else None, labels6.shape[0], iouv.data_ptr(),
                                             iouv.numel(), float(eps), correct.data_ptr(), C.c_void_p(_lib.stream_ptr(dev))), "match_batch")
    return correct.view(torch.bool)


def process_batch(detections, labels, iouv, pred_masks=None, gt_masks=None, overlap=False, masks=False):
    """Reference signature (utils/metrics.py:224): detections (N,6) [x1,y1,x2,y2,conf,cls], labels (M,5) [cls,x1,y1,x2,y2],
    iouv thresholds -> correct (N, len(iouv)) bool on iouv.device.  masks=True matches by mask IoU (segment/val.py:295):
    pred_masks (N, h, w) 0/1; gt_masks (M, H, W) 0/1, or with `overlap` (1, H, W) holding label k as the value k + 1; gt masks
    of another size are resized as the reference does (bilinear, then > 0.5).  Raises ValueError on 0/1 masks holding other
    values (that one check reads the device, as the reference's own `.cpu()` does)."""
    if masks:
        return _process_batch_masks(detections, labels, iouv, pred_masks, gt_masks, overlap)
    n = detections.shape[0]
    dev = detections.device
    lab6 = torch.cat((torch.zeros(labels.shape[0], 1, device=labels.device, dtype=labels.dtype), labels), 1)
    if n == 0:
        return torch.zeros(0, iouv.numel(), dtype=torch.bool, device=iouv.device)
    det = detections.float().contiguous()[None]
    return match_batch(det, None, lab6, iouv)[0].to(iouv.device)


def labels_to_native(targets: torch.Tensor, meta: torch.Tensor) -> torch.Tensor:
    """val.py:303-306 for all images at once: targets (nt,6) [img, cls, cx, cy, w, h] in network-input pixels, meta (B,5)
    [gain, pad_x, pad_y, w0, h0] -> (nt,6) [img, cls, x1, y1, x2, y2] in native pixels."""
    if not targets.is_cuda:
        raise RuntimeError("y5b200: labels_to_native runs on CUDA tensors only (no CPU / PyTorch fallback)")
    t = targets.float().contiguous().view(-1, 6)
    out = torch.empty_like(t)
    if t.shape[0]:
        m = meta.to(t.device, torch.float32).contiguous()
        with _lib.on(t.device):
            _lib.check(_lib.lib().y5_labels_native(t.data_ptr(), t.shape[0], m.data_ptr(), out.data_ptr(), C.c_void_p(_lib.stream_ptr(t.device))),
                       "labels_native")
    return out


def val_batch_metrics(rows: torch.Tensor, count: torch.Tensor, targets: torch.Tensor, im_shape, shapes, iouv: torch.Tensor, confusion=None):
    """The metric part of val.py:282-318 for a whole batch, on the device: rows/count from nms_device (rows (B,max_det,6+nm)
    in network-input pixels), targets (nt,6) [img, cls, cx, cy, w, h] already in network-input pixels (val.py:274),
    im_shape = (height, width) of the network input, shapes[i] = ((h0, w0), ((ratio_h, ratio_w), (pad_w, pad_h))) as the
    reference dataloader yields, or the (B,5) tensor scale_meta makes of them (already on the device, the loop can then be
    captured in a CUDA graph).  Returns (predn rows in native space, correct (B,max_det,niou) bool); nothing is synced.
    `confusion`, a ConfusionMatrix, is updated from the same native rows and labels as val.py's plots=True loop updates it."""
    from .general import scale_boxes_batch

    meta = _meta(im_shape, shapes, rows.device)
    predn = rows.clone()
    scale_boxes_batch(predn, count, meta)
    labelsn = labels_to_native(targets, meta)
    if confusion is not None:
        confusion.process_batch_padded(predn, count, labelsn)
    return predn, match_batch(predn, count, labelsn, iouv)


_STAGE_BYTES = 256 << 20  # seg_val_batch_metrics stages the uint8 prediction masks of at most this many bytes at a time


def _meta(im_shape, shapes, device):
    if isinstance(shapes, torch.Tensor):
        return shapes.to(device, torch.float32)
    from .general import scale_meta

    return scale_meta(im_shape, [s[0] for s in shapes], [s[1] if len(s) > 1 else None for s in shapes]).to(device)


def _row_words(h: int, w: int) -> int:
    words = int(_lib.lib().y5_mask_row_words(int(h), int(w)))
    if words < 0:
        _lib.check(words, "mask_row_words")
    return words


def _pack(src, src_hw, out_hw, n_rows, nonbinary, overlap=False, targets=None, batch=1, label_index=None):
    """y5_mask_pack: (bits (n_rows, words) int32, popcount (n_rows,) int32) of the masks in `src` (see include/y5b200.h)."""
    if not src.is_cuda:
        raise RuntimeError("y5b200: mask IoU runs on CUDA tensors only (no CPU / PyTorch fallback)")
    m = src.contiguous()
    if m.dtype == torch.bool:
        m = m.view(torch.uint8)
    dev = m.device
    bits = torch.empty(n_rows, _row_words(*out_hw), dtype=torch.int32, device=dev)
    pop = torch.empty(n_rows, dtype=torch.int32, device=dev)
    timg, ts = (targets.data_ptr(), targets.stride(0)) if targets is not None else (None, 0)
    _lib.check(_lib.lib().y5_mask_pack(m.data_ptr() if m.numel() else None, _lib.dtype_code(m.dtype), int(src_hw[0]), int(src_hw[1]),
                                       int(bool(overlap)), timg, ts, batch, n_rows, int(out_hw[0]), int(out_hw[1]),
                                       label_index.data_ptr() if label_index is not None else None, bits.data_ptr(), pop.data_ptr(),
                                       nonbinary.data_ptr(), C.c_void_p(_lib.stream_ptr(dev))), "mask_pack")
    return bits, pop


def _raise_nonbinary(nonbinary: torch.Tensor) -> None:
    bad = int(nonbinary.item())
    if bad:
        raise ValueError(f"y5b200: {bad} mask values are neither 0 nor 1 (mask IoU takes 0/1 masks)")


def mask_iou(mask1, mask2, eps=1e-7):
    """ultralytics.utils.metrics.mask_iou, which the reference imports into utils.metrics: mask1 (N, n), mask2 (M, n) flattened
    0/1 masks -> (N, M) fp32 on the device, inter / (|mask1| + |mask2| - inter + eps).  The intersections are a 1-bit GEMM
    (y5_mask_iou), bit-equal to the fp32 matmul expression.  Raises ValueError when a mask holds a value other than 0 or 1."""
    if mask1.dim() != 2 or mask2.dim() != 2 or mask1.shape[1] != mask2.shape[1]:
        raise ValueError(f"y5b200: mask_iou takes (N, n) and (M, n) masks, got {tuple(mask1.shape)} and {tuple(mask2.shape)}")
    dev = mask1.device
    n, m, px = mask1.shape[0], mask2.shape[0], mask1.shape[1]
    out = torch.zeros(n, m, dtype=torch.float32, device=dev)
    if n == 0 or m == 0 or px == 0:
        return out
    nonbinary = torch.zeros(1, dtype=torch.int32, device=dev)
    with _lib.on(dev):
        g, gp = _pack(mask1, (1, px), (1, px), n, nonbinary)
        p, pp = _pack(mask2, (1, px), (1, px), m, nonbinary)
        _lib.check(_lib.lib().y5_mask_iou(g.data_ptr(), gp.data_ptr(), None, n, p.data_ptr(), pp.data_ptr(), None, 0, 1, m, g.shape[1],
                                          float(eps), out.data_ptr(), C.c_void_p(_lib.stream_ptr(dev))), "mask_iou")
    _raise_nonbinary(nonbinary)
    return out


def _process_batch_masks(detections, labels, iouv, pred_masks, gt_masks, overlap):
    """process_batch(masks=True) (utils/metrics.py:239-252): pack, bit-GEMM IoU and matching for one image."""
    n, nl = detections.shape[0], labels.shape[0]
    if n == 0 or nl == 0:
        return torch.zeros(n, iouv.numel(), dtype=torch.bool, device=iouv.device)
    if not detections.is_cuda:
        raise RuntimeError("y5b200: process_batch runs on CUDA tensors only (no CPU / PyTorch fallback)")
    if pred_masks.dim() != 3 or gt_masks.dim() != 3 or pred_masks.shape[0] != n or (not overlap and gt_masks.shape[0] != nl):
        raise ValueError(f"y5b200: process_batch(masks=True): pred_masks {tuple(pred_masks.shape)}, gt_masks {tuple(gt_masks.shape)} "
                         f"for {n} detections and {nl} labels (overlap={overlap})")
    dev = detections.device
    out_hw = tuple(pred_masks.shape[1:])
    nonbinary = torch.zeros(1, dtype=torch.int32, device=dev)
    iou = torch.empty(nl, n, dtype=torch.float32, device=dev)
    det = detections.float().contiguous()[None]
    lab = labels.to(dev, torch.float32).contiguous()
    iv = iouv.to(dev, torch.float32).contiguous()
    correct = torch.empty(1, n, iv.numel(), dtype=torch.uint8, device=dev)
    lib = _lib.lib()
    with _lib.on(dev):
        g, gp = _pack(gt_masks, gt_masks.shape[1:], out_hw, nl, nonbinary, overlap=overlap)
        p, pp = _pack(pred_masks, out_hw, out_hw, n, nonbinary)
        st = C.c_void_p(_lib.stream_ptr(dev))
        _lib.check(lib.y5_mask_iou(g.data_ptr(), gp.data_ptr(), None, nl, p.data_ptr(), pp.data_ptr(), None, 0, 1, n, g.shape[1], 1e-7,
                                   iou.data_ptr(), st), "mask_iou")
        _lib.check(lib.y5_mask_match_batch(det.data_ptr(), det.stride(0), det.stride(1), None, 1, n, lab.data_ptr(), lab.stride(0), None, nl,
                                           iou.data_ptr(), iv.data_ptr(), iv.numel(), correct.data_ptr(), st), "mask_match_batch")
    _raise_nonbinary(nonbinary)
    return correct[0].view(torch.bool).to(iouv.device)


def seg_val_batch_metrics(rows, count, protos, targets, masks, im_shape, shapes, iouv, overlap, native=False, check=False):
    """The metric part of segment/val.py:263-298 for a whole batch, on the device.  rows/count from nms_device(nm=32) (rows
    (B,max_det,38) in network-input pixels), protos (B,32,mh,mw), targets (nt,6) [img, cls, cx, cy, w, h] in network-input
    pixels, masks as the reference dataloader yields them: (B,H,W) label indices with `overlap`, else (nt,H,W) 0/1 in
    target order; im_shape / shapes as val_batch_metrics takes them.  Prediction masks are process_mask (native=True:
    process_mask_native, --retina-masks) of the network-input boxes, staged as uint8 a chunk of images at a time; gt masks of
    another size are resized as the reference does.  Returns (predn, correct_bboxes, correct_masks), both (B,max_det,niou)
    bool, padding rows False.  Nothing is synced unless `check`, which reads the non-binary counter once and raises
    ValueError when a 0/1 gt mask held another value.  segment/val.py's confusion matrix (box IoU, segment/val.py:297) is
    ConfusionMatrix.process_batch_padded(predn, count, labels_to_native(targets, meta)) on the returned predn."""
    from .segment.general import process_mask_batch

    b, max_det = rows.shape[:2]
    nt = targets.numel() // 6
    if protos.dim() != 4 or protos.shape[0] != b or rows.dim() != 3 or rows.shape[2] < 6 + protos.shape[1]:
        raise ValueError(f"y5b200: seg_val_batch_metrics: rows {tuple(rows.shape)} need 6 + {protos.shape[1] if protos.dim() == 4 else '?'} "
                         f"columns and protos {tuple(protos.shape)} one entry per image")
    if masks.dim() != 3 or masks.shape[0] != (b if overlap else nt):
        raise ValueError(f"y5b200: seg_val_batch_metrics: masks {tuple(masks.shape)} must be ({b if overlap else nt}, H, W) "
                         f"({'one index image per image' if overlap else 'one mask per target'}, overlap={overlap})")
    dev = rows.device
    meta = _meta(im_shape, shapes, dev)
    predn, correct_bboxes = val_batch_metrics(rows, count, targets, im_shape, meta, iouv)
    ih, iw = int(im_shape[0]), int(im_shape[1])
    out_hw = (ih, iw) if native else tuple(protos.shape[-2:])
    t = targets.to(dev, torch.float32).contiguous().view(-1, 6)
    iv = iouv.to(dev, torch.float32).contiguous()
    cnt = count.to(dev, torch.int32).contiguous() if count is not None else None
    nonbinary = torch.zeros(1, dtype=torch.int32, device=dev)
    label_index = torch.empty(b + 1 + 2 * nt, dtype=torch.int32, device=dev)
    iou = torch.empty(nt, max_det, dtype=torch.float32, device=dev)
    correct = torch.empty(b, max_det, iv.numel(), dtype=torch.uint8, device=dev)
    lib = _lib.lib()
    with _lib.on(dev):
        g, gp = _pack(masks, masks.shape[-2:], out_hw, nt, nonbinary, overlap=overlap, targets=t, batch=b, label_index=label_index)
        if nt:
            flat = rows.reshape(b * max_det, rows.shape[2])
            chunk = max(1, min(b, _STAGE_BYTES // (max_det * out_hw[0] * out_hw[1])))
            for b0 in range(0, b, chunk):
                nb = min(chunk, b - b0)
                r = flat[b0 * max_det:(b0 + nb) * max_det]
                img = torch.div(torch.arange(nb * max_det, dtype=torch.int32, device=dev), max_det, rounding_mode="floor")
                pm = process_mask_batch(protos[b0:b0 + nb], r[:, 6:], r[:, :4], img, (ih, iw), out_dtype=torch.uint8, native=native)
                p, pp = _pack(pm, out_hw, out_hw, nb * max_det, nonbinary)
                _lib.check(lib.y5_mask_iou(g.data_ptr(), gp.data_ptr(), label_index.data_ptr(), nt, p.data_ptr(), pp.data_ptr(),
                                           cnt.data_ptr() if cnt is not None else None, b0, nb, max_det, g.shape[1], 1e-7, iou.data_ptr(),
                                           C.c_void_p(_lib.stream_ptr(dev))), "mask_iou")
        _lib.check(lib.y5_mask_match_batch(predn.data_ptr(), predn.stride(0), predn.stride(1), cnt.data_ptr() if cnt is not None else None, b,
                                           max_det, t.data_ptr() + 4 if nt else None, 6, label_index.data_ptr(), nt,
                                           iou.data_ptr() if nt else None, iv.data_ptr(), iv.numel(), correct.data_ptr(),
                                           C.c_void_p(_lib.stream_ptr(dev))), "mask_match_batch")
    if check:
        _raise_nonbinary(nonbinary)
    return predn, correct_bboxes, correct.view(torch.bool)


_AP_GRIDS = {}  # device -> np.linspace(0, 1, 1000) and np.linspace(0, 1, 101), the grids ap_per_class interpolates at
_MAX_CLASSES = 4096


def _ap_grid(dev):
    g = _AP_GRIDS.get(dev)
    if g is None:
        g = _AP_GRIDS[dev] = torch.from_numpy(np.concatenate((np.linspace(0, 1, 1000), np.linspace(0, 1, 101)))).to(dev)
    return g


def _ap_device(*xs):
    for x in xs:
        if isinstance(x, torch.Tensor) and x.is_cuda:
            return x.device
    if not torch.cuda.is_available():
        raise RuntimeError("y5b200: ap_per_class runs on CUDA only (no CPU / numpy fallback)")
    return torch.device("cuda", torch.cuda.current_device())


def _as_f32(x, dev, what):
    """x as a contiguous float32 tensor on dev (numpy input uploaded once); ValueError when float32 cannot hold its values."""
    t = torch.as_tensor(x)
    if t.dtype != torch.float32:
        f = t.to(torch.float32)
        same = f.to(t.dtype) == t
        if t.is_floating_point():
            same |= torch.isnan(t)
        if not bool(same.all()):
            raise ValueError(f"y5b200: {what} ({t.dtype}) holds values float32 cannot represent")
        t = f
    return t.to(dev).contiguous().view(-1)


def _as_tp(x, dev, what):
    t = torch.as_tensor(x)
    if t.dim() != 2:
        raise ValueError(f"y5b200: {what} must be (n, niou), got {tuple(t.shape)}")
    return t.to(dev).bool().contiguous().view(torch.uint8)


def _ap_run(dev, tps, conf_ptr, cls_ptr, img_stride, row_stride, tp_img_stride, count, n_img, rows, niou, target_cls, eps):
    """y5_ap_per_class over rows laid out as include/y5b200.h describes; one result tuple (tp, fp, p, r, f1, ap, classes) per
    tp matrix in `tps`, as numpy arrays."""
    lib = _lib.lib()
    tcls = _as_f32(target_cls, dev, "target_cls")
    nt = tcls.numel()
    nc_cap = min(nt, _MAX_CLASSES)
    sets = len(tps)
    ws_bytes = int(lib.y5_ap_workspace_bytes(n_img, rows, niou, nt, sets))
    if ws_bytes < 0:
        _lib.check(ws_bytes, "ap_workspace_bytes")
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    out = torch.empty(max(sets * nc_cap * (5 + niou), 1), dtype=torch.float64, device=dev)
    meta = torch.empty(_lib.AP_META + nc_cap, dtype=torch.int32, device=dev)
    with _lib.on(dev):
        _lib.check(lib.y5_ap_per_class(tps[0].data_ptr() or None, tps[1].data_ptr() or None if sets == 2 else None, tp_img_stride, niou,
                                       conf_ptr or None, cls_ptr or None, img_stride, row_stride,
                                       count.data_ptr() if count is not None else None, n_img, rows, niou,
                                       tcls.data_ptr() if nt else None, nt, _ap_grid(dev).data_ptr(), float(eps), ws.data_ptr(), ws_bytes,
                                       out.data_ptr(), meta.data_ptr(), C.c_void_p(_lib.stream_ptr(dev))), "ap_per_class")
    meta_h = meta.cpu().numpy()
    if meta_h[2]:
        what = " and ".join(w for bit, w in ((1, "predicted classes"), (2, "target classes")) if meta_h[2] & bit)
        raise ValueError(f"y5b200: ap_per_class takes integral class values in [0, {_MAX_CLASSES}); the {what} hold others")
    nc = int(meta_h[1])
    classes = meta_h[_lib.AP_META:_lib.AP_META + nc].astype(np.int64)
    out_h = out.cpu().numpy()
    results = []
    for s in range(sets):
        o = out_h[s * nc_cap * (5 + niou):(s + 1) * nc_cap * (5 + niou)]
        tp, fp, p, r, f1 = (o[k * nc_cap:k * nc_cap + nc].copy() for k in range(5))
        ap = o[5 * nc_cap:].reshape(nc_cap, niou)[:nc].copy()
        results.append((tp, fp, p, r, f1, ap, classes.copy()))
    return results


def _ap_flat(tps, conf, pred_cls, target_cls, eps):
    dev = _ap_device(*tps, conf, pred_cls, target_cls)
    tps = [_as_tp(t, dev, "tp") for t in tps]
    n, niou = tps[0].shape
    cf, cl = _as_f32(conf, dev, "conf"), _as_f32(pred_cls, dev, "pred_cls")
    if cf.numel() != n or cl.numel() != n or any(t.shape != tps[0].shape for t in tps):
        raise ValueError(f"y5b200: ap_per_class: tp {[tuple(t.shape) for t in tps]}, conf ({cf.numel()},), pred_cls ({cl.numel()},) disagree")
    return _ap_run(dev, tps, cf.data_ptr(), cl.data_ptr(), 0, 1, 0, None, 1, n, niou, target_cls, eps)


def _box_and_mask(res_b, res_m):
    return {k: {"p": r[2], "r": r[3], "ap": r[5], "f1": r[4], "ap_class": r[6]} for k, r in (("boxes", res_b), ("masks", res_m))}


def ap_per_class(tp, conf, pred_cls, target_cls, plot=False, save_dir=".", names=(), eps=1e-16, prefix=""):
    """Reference signature (utils/metrics.py:25): tp (n, niou) bool, conf (n,), pred_cls (n,), target_cls (m,) as numpy arrays
    (uploaded once) or CUDA tensors -> numpy (tp, fp, p, r, f1, ap, unique_classes), float64 and int64, as the reference
    returns them.  Rows are ordered by np.argsort(-conf, kind="stable"); class values must be integers in [0, 4096)
    (ValueError otherwise).  Plots need matplotlib, which the engine does not depend on: plot=True raises."""
    if plot:
        raise NotImplementedError("y5b200: ap_per_class(plot=True): plotting is not ported (validation runs with plots=False)")
    return _ap_flat([tp], conf, pred_cls, target_cls, eps)[0]


def ap_per_class_batch(correct, rows, count, target_cls, eps=1e-16, correct_masks=None):
    """ap_per_class over the padded tensors of a batched val loop, concatenated along dim 0 over batches: correct (I, max_det,
    niou) bool (val_batch_metrics; correct_masks likewise from seg_val_batch_metrics), rows (I, max_det, >=6) float32 with conf
    in column 4 and class in column 5, count (I,) valid rows per image, target_cls (m,) the labels' classes.  Reads rows
    r < count[i] in (image, row) order, the order of val.py's per-image stats.append; padding rows are never read.  Returns
    ap_per_class's tuple, or with correct_masks ap_per_class_box_and_mask's dict (one sort for both)."""
    dev = _ap_device(correct, rows, count, target_cls)
    if rows.dim() != 3 or rows.shape[2] < 6 or rows.dtype != torch.float32:
        raise ValueError(f"y5b200: ap_per_class_batch: rows must be (I, max_det, >=6) float32, got {tuple(rows.shape)} {rows.dtype}")
    n_img, max_det = rows.shape[:2]
    tps = [correct] if correct_masks is None else [correct, correct_masks]
    if any(t.dim() != 3 or tuple(t.shape[:2]) != (n_img, max_det) for t in tps):
        raise ValueError(f"y5b200: ap_per_class_batch: correct {[tuple(t.shape) for t in tps]} must be ({n_img}, {max_det}, niou)")
    if count.numel() != n_img:
        raise ValueError(f"y5b200: ap_per_class_batch: count has {count.numel()} entries for {n_img} images")
    niou = tps[0].shape[2]
    if tps[-1].shape[2] != niou:
        raise ValueError("y5b200: ap_per_class_batch: correct and correct_masks have different thresholds")
    tps = [_as_tp(t.reshape(n_img * max_det, niou), dev, "correct") for t in tps]
    r = rows.to(dev)
    if r.stride(2) != 1:
        r = r.contiguous()
    cnt = count.to(dev, torch.int32).contiguous()
    res = _ap_run(dev, tps, r.data_ptr() + 16, r.data_ptr() + 20, r.stride(0), r.stride(1), max_det * niou, cnt, n_img, max_det, niou,
                  target_cls, eps)
    return res[0] if correct_masks is None else _box_and_mask(*res)


def fitness(x):
    """Reference utils/metrics.py:19: per row of [P, R, mAP@0.5, mAP@0.5:0.95, ...] (numpy, on the host), the model's fitness
    0.1 * mAP@0.5 + 0.9 * mAP@0.5:0.95, summed over the four weighted columns in column order."""
    return np.sum(np.asarray(x)[:, :4] * np.array([0.0, 0.0, 0.1, 0.9]), axis=1)


LOGGER = logging.getLogger("yolov5_b200")


class ConfusionMatrix:
    """Reference utils/metrics.py:129: the detection confusion matrix of val.py's plots, rows = predicted class, columns =
    true class, index nc = background.  The counts accumulate on the device (y5_confusion_batch, one launch per update, no
    host sync); `matrix` folds them into a host float64 array when read (see there).  Equal IoUs are resolved in (label,
    detection) scan order (DESIGN.md, f11); the reference's own order among them depends on numpy's sort and the host."""

    def __init__(self, nc, conf=0.25, iou_thres=0.45):
        self.nc = nc
        self.conf = conf
        self.iou_thres = iou_thres
        self._matrix = np.zeros((nc + 1, nc + 1))
        self._acc = None  # device int64: (nc+1)^2 counts not yet read, then the error word (low 32 bits of the last entry)

    @property
    def matrix(self):
        """The (nc+1, nc+1) float64 host array.  Reading it syncs once: the device counts since the last read are added into
        it and the device accumulator is zeroed on the current stream; the same array is returned every time, so in-place
        edits persist and later updates add on top.  Raises ValueError when an update met a class outside [0, nc) (the
        reference would index out of range); the counts since the last read are dropped with the error."""
        if self._acc is not None:
            acc = self._acc.cpu().numpy()
            self._acc.zero_()
            k = (self.nc + 1) ** 2
            if acc[k]:
                what = " and ".join(w for bit, w in ((1, "a label"), (2, "a detection")) if acc[k] & bit)
                raise ValueError(f"y5b200: ConfusionMatrix: {what} class is outside [0, {self.nc}) (nc={self.nc}); the counts since "
                                 "the last read are dropped")
            self._matrix += acc[:k].reshape(self.nc + 1, self.nc + 1)
        return self._matrix

    @matrix.setter
    def matrix(self, value):
        """Replace the host array; device counts not yet read are dropped, as the reference drops every earlier count."""
        if self._acc is not None:
            self._acc.zero_()
        self._matrix = value

    def _accumulator(self, dev):
        if self._acc is None:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("y5b200: ConfusionMatrix allocates its device counts on the first update; make one update "
                                   "(or read `matrix`) before capturing a CUDA graph")
            self._acc = torch.zeros((self.nc + 1) ** 2 + 1, dtype=torch.int64, device=dev)
        elif self._acc.device != dev:
            raise ValueError(f"y5b200: ConfusionMatrix counts live on {self._acc.device}, got tensors on {dev}")
        return self._acc

    def _launch(self, det, img_stride, row_stride, count, batch, max_det, labels6):
        dev = labels6.device if det is None else det.device
        acc = self._accumulator(dev)
        k = (self.nc + 1) ** 2
        with _lib.on(dev):
            _lib.check(_lib.lib().y5_confusion_batch(det.data_ptr() if det is not None and det.numel() else None, img_stride, row_stride,
                                                     count.data_ptr() if count is not None else None, batch, max_det,
                                                     labels6.data_ptr() if labels6.numel() else None, labels6.shape[0], self.nc,
                                                     float(self.conf), float(self.iou_thres), 1e-7, acc.data_ptr(), acc.data_ptr() + 8 * k,
                                                     C.c_void_p(_lib.stream_ptr(dev))), "confusion_batch")

    def process_batch(self, detections, labels):
        """Reference signature (utils/metrics.py:139): detections (N, >=6) float32 [x1,y1,x2,y2,conf,cls,...] and labels (M,5)
        float32 [cls,x1,y1,x2,y2] in pixels, CUDA tensors; or detections=None and labels (M,) float32 classes, all counted as
        background.  Launches one kernel; nothing is synced.  CPU tensors raise RuntimeError, other dtypes TypeError (the
        reference computes the IoU in the input dtype)."""
        if detections is None:
            cls = _cuda_f32(labels, "labels", 1)
            labels6 = torch.zeros(cls.shape[0], 6, dtype=torch.float32, device=cls.device)
            labels6[:, 1] = cls
            self._launch(None, 0, 6, None, 1, 0, labels6)
            return
        det = _cuda_f32(detections, "detections", 2)
        lab = _cuda_f32(labels, "labels", 2)
        if det.shape[1] < 6 or lab.shape[1] != 5 or det.device != lab.device:
            raise ValueError(f"y5b200: ConfusionMatrix.process_batch takes detections (N, >=6) and labels (M, 5) on one device, got "
                             f"{tuple(det.shape)} on {det.device} and {tuple(lab.shape)} on {lab.device}")
        if det.stride(1) != 1:
            det = det.contiguous()
        labels6 = torch.cat((lab.new_zeros(lab.shape[0], 1), lab), 1)
        self._launch(det, 0, det.stride(0), None, 1, det.shape[0], labels6)

    def process_batch_padded(self, rows, count, labels6):
        """The whole batch in one launch, as val.py's per-image loop with plots=True counts it: rows (B, max_det, >=6) float32
        in native pixels (val_batch_metrics' predn, image b's valid rows r < count[b]; seg rows of 6 + nm columns work as
        they are), count (B,) int32 or None (all rows valid), labels6 (nt, 6) [img, cls, x1,y1,x2,y2] in native pixels
        (labels_to_native).  An image without rows counts its labels as background (val.py's detections=None call), one
        without labels counts nothing.  No sync and no allocation once the first update has run: capturable in a CUDA graph."""
        rows = _cuda_f32(rows, "rows", 3)
        if rows.shape[2] < 6 or rows.stride(2) != 1:
            raise ValueError(f"y5b200: process_batch_padded: rows must be (B, max_det, >=6) with unit column stride, got {tuple(rows.shape)}")
        labels6 = _cuda_f32(labels6, "labels6", 2)
        if labels6.shape[1] != 6:
            raise ValueError(f"y5b200: process_batch_padded: labels6 must be (nt, 6), got {tuple(labels6.shape)}")
        labels6 = labels6.contiguous()
        b, max_det = rows.shape[:2]
        cnt = None
        if count is not None:
            if count.numel() != b:
                raise ValueError(f"y5b200: process_batch_padded: count has {count.numel()} entries for {b} images")
            cnt = count.to(rows.device, torch.int32).contiguous()
        self._launch(rows, rows.stride(0), rows.stride(1), cnt, b, max_det, labels6)

    def plot(self, normalize=True, save_dir="", names=()):
        """Reference utils/metrics.py:185 on the host from `matrix`: seaborn heatmap saved as save_dir/confusion_matrix.png.
        As the reference's TryExcept does, a failure (seaborn or matplotlib missing included) is logged, not raised."""
        try:
            import matplotlib.pyplot as plt
            import seaborn as sn

            m = self.matrix
            array = m / ((m.sum(0).reshape(1, -1) + 1e-9) if normalize else 1)  # each true class (column) sums to 1
            array[array < 0.005] = np.nan  # left blank rather than annotated 0.00
            fig, ax = plt.subplots(1, 1, figsize=(12, 9), tight_layout=True)
            nc, nn = self.nc, len(names)
            sn.set(font_scale=1.0 if nc < 50 else 0.8)
            ticklabels = [*names, "background"] if 0 < nn < 99 and nn == nc else "auto"
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")  # an all-NaN column warns
                sn.heatmap(array, ax=ax, annot=nc < 30, annot_kws={"size": 8}, cmap="Blues", fmt=".2f", square=True, vmin=0.0,
                           xticklabels=ticklabels, yticklabels=ticklabels).set_facecolor((1, 1, 1))
            ax.set_xlabel("True")
            ax.set_ylabel("Predicted")
            ax.set_title("Confusion Matrix")
            fig.savefig(Path(save_dir) / "confusion_matrix.png", dpi=250)
            plt.close(fig)
        except Exception as e:
            LOGGER.warning(f"ConfusionMatrix plot failure: {e}")

    def print(self):
        """Reference utils/metrics.py:218: log each of the nc + 1 rows of `matrix`, values separated by spaces."""
        m = self.matrix
        for i in range(self.nc + 1):
            LOGGER.info(" ".join(map(str, m[i])))


def _cuda_f32(x, what, dim):
    if not isinstance(x, torch.Tensor):
        raise TypeError(f"y5b200: ConfusionMatrix takes torch tensors, got {type(x).__name__} for {what}")
    if not x.is_cuda:
        raise RuntimeError("y5b200: ConfusionMatrix runs on CUDA tensors only (no CPU / PyTorch fallback)")
    if x.dtype != torch.float32:
        raise TypeError(f"y5b200: ConfusionMatrix takes float32 {what}, got {x.dtype}")
    if x.dim() != dim:
        raise ValueError(f"y5b200: ConfusionMatrix: {what} must have {dim} dimension(s), got {tuple(x.shape)}")
    return x
