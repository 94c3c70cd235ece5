"""ultralytics.data.utils' polygon2mask / polygons2masks / polygons2masks_overlap, restated from the public package for
the reference's segmentation dataloader (utils/segment/dataloaders.py:10 imports the last two).  Third-party code, parity
unpinned like the other ultralytics helpers of refshim.py; their cv2 calls are the real ones.

`register()` adds them to refshim's stand-in `ultralytics.data.utils` module; call it before refshim.install().  Only
tests/golden/make_seg_aug_golden.py uses this file, where the reference tree and cv2 exist.
"""
from __future__ import annotations

import cv2
import numpy as np

OVERLAP_ORDERS = []  # every order polygons2masks_overlap returned, so the generator can replay the host's own argsort


def polygon2mask(imgsz, polygons, color=1, downsample_ratio=1):
    mask = np.zeros(imgsz, dtype=np.uint8)
    polygons = np.asarray(polygons, dtype=np.int32)
    polygons = polygons.reshape((polygons.shape[0], -1, 2))
    cv2.fillPoly(mask, polygons, color=color)
    nh, nw = (imgsz[0] // downsample_ratio, imgsz[1] // downsample_ratio)
    return cv2.resize(mask, (nw, nh))


def polygons2masks(imgsz, polygons, color, downsample_ratio=1):
    return np.array([polygon2mask(imgsz, [x.reshape(-1)], color, downsample_ratio) for x in polygons])


def polygons2masks_overlap(imgsz, segments, downsample_ratio=1):
    masks = np.zeros((imgsz[0] // downsample_ratio, imgsz[1] // downsample_ratio), dtype=np.int32 if len(segments) > 255 else np.uint8)
    areas = []
    ms = []
    for si in range(len(segments)):
        mask = polygon2mask(imgsz, [segments[si].reshape(-1)], downsample_ratio=downsample_ratio, color=1)
        ms.append(mask.astype(masks.dtype))
        areas.append(mask.sum())
    areas = np.asarray(areas)
    index = np.argsort(-areas)
    OVERLAP_ORDERS.append(index)
    ms = np.array(ms)[index]
    for i in range(len(segments)):
        mask = ms[i] * (i + 1)
        masks = masks + mask
        masks = np.clip(masks, a_min=0, a_max=i + 1)
    return masks, index


def register(refshim):
    refshim._REAL.setdefault("ultralytics.data.utils", {}).update(
        polygon2mask=polygon2mask, polygons2masks=polygons2masks, polygons2masks_overlap=polygons2masks_overlap)
