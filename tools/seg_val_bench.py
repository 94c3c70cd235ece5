"""Segmentation validation metric timing on the GPU: the engine's batched seg_val_batch_metrics (process_mask + box and
mask-IoU matching for the whole batch, csrc/mask_metrics.cu) vs the reference's per-image expressions of
segment/val.py:263-298 on the same GPU (torch process_mask / process_mask_native, scale_boxes, process_batch box and mask
branches with their `.cpu()` round trips), at yolov5s-seg val shapes.

    python tools/seg_val_bench.py [--batch 32] [--size 640] [--max-det 300] [--min-seconds 1.0]

max_det rows per image (conf_thres 0.001 keeps that many on a real model), labels COCO-like (about 7 per image) and a crowded
batch of 100 per image.  Configurations: overlap gt at 640^2 (mask ratio 1, resized to 160^2) and at 160^2 (ratio 4), non-
overlap gt at 160^2, and --retina-masks (process_mask_native, predictions at 640^2, gt 160^2 up-sampled).  Prints one JSON
line: the GPU and its power limit, ms per batch of both arms per configuration.  CUDA-event timing after warm-up, each timed
window at least --min-seconds long.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import mask_val_ref  # noqa: E402
from tests.seg_loss_ref import paint_masks  # noqa: E402
from yolov5_b200.utils import metrics  # noqa: E402
from yolov5_b200.utils.general import scale_meta, xywh2xyxy  # noqa: E402


def timed(fn, min_seconds, warmup=2):
    """mean ms per call over a window of at least `min_seconds` (device events)."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    n = 1
    while True:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        if ms >= 1000 * min_seconds:
            return ms / n, n
        n = max(n * 2, int(n * 1.2 * 1000 * min_seconds / max(ms, 1e-3)))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def crop_mask(masks, boxes):
    n, h, w = masks.shape
    x1, y1, x2, y2 = torch.chunk(boxes[:, :, None], 4, 1)
    r = torch.arange(w, device=masks.device, dtype=x1.dtype)[None, None, :]
    c = torch.arange(h, device=masks.device, dtype=x1.dtype)[None, :, None]
    return masks * ((r >= x1) * (r < x2) * (c >= y1) * (c < y2))


def process_mask_torch(protos, masks_in, bboxes, shape, native):
    """utils/segment/general.py:25-76 in the reference's torch expressions."""
    c, mh, mw = protos.shape
    ih, iw = shape
    masks = (masks_in @ protos.float().view(c, -1)).sigmoid().view(-1, mh, mw)
    if native:
        gain = min(mh / ih, mw / iw)
        pad = (mw - iw * gain) / 2, (mh - ih * gain) / 2
        top, left = int(pad[1]), int(pad[0])
        bottom, right = int(mh - pad[1]), int(mw - pad[0])
        masks = F.interpolate(masks[None, :, top:bottom, left:right], shape, mode="bilinear", align_corners=False)[0]
        return crop_mask(masks, bboxes).gt_(0.5)
    b = bboxes.clone()
    b[:, 0] *= mw / iw
    b[:, 2] *= mw / iw
    b[:, 3] *= mh / ih
    b[:, 1] *= mh / ih
    return crop_mask(masks, b).gt_(0.5)


def make_batch(dev, bs, sz, max_det, per_image, overlap, gt_size, seed):
    rs = np.random.RandomState(seed)
    tg = []
    for b in range(bs):
        k = per_image if per_image > 20 else rs.poisson(per_image)
        for _ in range(k):
            tg.append([b, rs.randint(0, 80), *rs.uniform(0.2, 0.8, 2), *rs.uniform(0.03, 0.4, 2)])
    tg = np.array(tg, np.float32).reshape(-1, 6)
    if overlap:
        masks = np.stack([paint_masks((gt_size, gt_size), tg[tg[:, 0] == b, 2:6], np.arange(1, int((tg[:, 0] == b).sum()) + 1))
                          for b in range(bs)])
    else:
        masks = np.stack([paint_masks((gt_size, gt_size), tg[i:i + 1, 2:6], [1.0]) for i in range(len(tg))])
    px = tg.copy()
    px[:, 2:6] *= sz
    rows = np.zeros((bs, max_det, 38), np.float32)
    for b in range(bs):
        lab = px[px[:, 0] == b]
        pick = lab[rs.randint(len(lab), size=max_det)] if len(lab) else np.tile([[b, 0, sz / 2, sz / 2, 64, 64]], (max_det, 1))
        box = pick[:, 2:6] + rs.normal(0, 4, (max_det, 4))
        rows[b, :, :4] = np.concatenate((box[:, :2] - box[:, 2:] / 2, box[:, :2] + box[:, 2:] / 2), 1)
        rows[b, :, 4] = np.sort(rs.uniform(0.001, 1, max_det))[::-1]
        rows[b, :, 5] = np.where(rs.uniform(size=max_det) < 0.7, pick[:, 1], rs.randint(0, 80, max_det))
        rows[b, :, 6:] = rs.normal(0, 0.5, (max_det, 32))
        rows[b, :, 6] = 1.0
    protos = rs.normal(0, 1, (bs, 32, sz // 4, sz // 4)).astype(np.float32)
    protos[:, 0] = 6.0
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    count = torch.full((bs,), max_det, dtype=torch.int32, device=dev)
    return t(rows), count, t(protos).half(), t(px), t(masks.astype(np.float32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=640)
    ap.add_argument("--max-det", type=int, default=300)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("seg_val_bench: needs a CUDA device")
    dev = torch.device("cuda:0")
    bs, sz, md = args.batch, args.size, args.max_det
    iouv = torch.linspace(0.5, 0.95, 10, device=dev)
    im_shape = (sz, sz)
    shapes = [((sz, sz), ((1.0, 1.0), (0.0, 0.0))) for _ in range(bs)]
    configs = {  # name: (overlap, gt size, retina, labels per image)
        "overlap_gt640": (True, sz, False, 7),
        "overlap_gt160": (True, sz // 4, False, 7),
        "nonoverlap_gt160": (False, sz // 4, False, 7),
        "retina_gt160": (True, sz // 4, True, 7),
        "overlap_gt640_crowded100": (True, sz, False, 100),
    }
    out = dict(gpu=gpu_info(), batch=bs, size=sz, max_det=md, proto_dtype="fp16")
    for name, (overlap, gsz, native, per_image) in configs.items():
        rows, count, protos, tg, masks = make_batch(dev, bs, sz, md, per_image, overlap, gsz, seed=len(name))
        meta = scale_meta(im_shape, [s[0] for s in shapes], [s[1] for s in shapes]).to(dev)

        def engine():
            return metrics.seg_val_batch_metrics(rows, count, protos, tg, masks, im_shape, meta, iouv, overlap, native=native)

        def reference():  # segment/val.py:263-298, one image at a time
            res = []
            for si in range(bs):
                pred = rows[si]
                labels = tg[tg[:, 0] == si, 1:]
                midx = [si] if overlap else tg[:, 0] == si
                gt_masks = masks[midx]
                pred_masks = process_mask_torch(protos[si], pred[:, 6:], pred[:, :4], im_shape, native)
                predn = pred.clone()
                predn[:, [0, 2]] = ((predn[:, [0, 2]] - meta[si, 1]) / meta[si, 0]).clamp(0, sz)
                predn[:, [1, 3]] = ((predn[:, [1, 3]] - meta[si, 2]) / meta[si, 0]).clamp(0, sz)
                tbox = xywh2xyxy(labels[:, 1:5])
                labelsn = torch.cat((labels[:, 0:1], tbox), 1)
                cb = mask_val_ref.process_batch_torch(predn, labelsn, iouv)
                cm = mask_val_ref.process_batch_torch(predn, labelsn, iouv, pred_masks, gt_masks, overlap=overlap, masks=True)
                res.append((cb, cm))
            return res

        _, cb, cm = engine()
        ref = reference()
        agree = all(torch.equal(cm[b], ref[b][1]) for b in range(bs))  # equal-IoU runs may order labels differently
        eng_ms, eng_n = timed(engine, args.min_seconds)
        ref_ms, ref_n = timed(reference, args.min_seconds)
        out[name] = dict(labels=int(tg.shape[0]), engine_ms=round(eng_ms, 3), torch_reference_ms=round(ref_ms, 3), speedup=round(ref_ms / eng_ms, 1),
                         iters=dict(engine=eng_n, torch_reference=ref_n), correct_masks_equal=agree, true_positives=int(cm.sum()))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
