"""ORACLE (test infrastructure, never on the product path): numpy restatement of the segmentation training dataloader
(`LoadImagesAndLabelsAndMasks`, augment=True, rect=False) -- the segment path of mosaic / random_perspective / mixup, the
label filter and the polygon masks.  The image arithmetic is the detection loader's (oracle/aug_ref.py).

Only tests/ and tools/ may import this.

Reference lines restated (paths relative to the reference tree):
  utils/segment/dataloaders.py:130-233  __getitem__ (draw order: mixup partner random.randint(0, n - 1), masks, flips)
  utils/segment/dataloaders.py:235-292  load_mosaic (tiles not shuffled, xyn2xy per segment, clip of labels and segments
                                        to [0, 2s])
  utils/segment/dataloaders.py:294-301  collate_fn (torch.cat of the per-image masks: dtype promotion)
  utils/segment/augmentations.py:14-23  mixup (segments concatenated)
  utils/segment/augmentations.py:26-91  random_perspective, segment path (resample_segments, xy @ M.T, segment2box,
                                        box_candidates(area_thr=0.01))
  utils/general.py:584-610              xyn2xy, segment2box, resample_segments
Third-party arithmetic, pinned against the installed packages by tests/golden/make_seg_aug_golden.py and
tests/test_seg_augment_cpu.py:
  * ultralytics.data.utils polygon2mask / polygons2masks / polygons2masks_overlap.
  * cv2.fillPoly(mask, [int32 (n, 2)], 1) (shift 0, LINE_8): every edge's 8-connected line (cv2.clipLine to the image,
    then Bresenham left to right with err = dx - 2dy), plus the scan fill: edges in 16.16 fixed point, x = vertex x << 16
    (no half-pixel offset), an edge with an endpoint outside the image starting from its clipped x (and clipped y when
    the clipped line is not horizontal), slope = dx / dy truncated toward zero, active on rows y0 <= y < y1, the
    sorted crossings pair into spans [ceil(x_2k), floor(x_2k+1)].
  * cv2.resize(uint8, INTER_LINEAR) of a 0/1 mask by 1/4: 1 iff at least two of source pixels (4k+1 | 4k+2)^2 are set.
  * numpy's float64 `xy @ M.T` (OpenBLAS) at the 1000-row shapes: x*M00, fma(y, M01, .), + M02 -- the same order as at the
    4-row shapes of the box path; restated here with an exact fma so that the oracle does not depend on the host's BLAS.
  * np.linspace(0, L - 1, 1000) = i * ((L - 1) / 999) with the last point L - 1; np.interp on unit-spaced points:
    (d[j+1] - d[j]) * (x - j) + d[j], two roundings, d[j] itself where x == j.
"""
from __future__ import annotations

import random

import numpy as np

from oracle import aug_ref

N_POINTS = 1000
XY_SHIFT = 16

# ----------------------------------------------------------------------------------------------------------------------
# float64 helpers
# ----------------------------------------------------------------------------------------------------------------------


def _two_prod(a, b):
    """p + e == a * b exactly (Dekker), for finite a, b far from overflow and underflow."""
    p = a * b
    c = 134217729.0 * a
    ah = c - (c - a)
    al = a - ah
    c = 134217729.0 * b
    bh = c - (c - b)
    bl = b - bh
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def fma(a, b, c):
    """Correctly rounded a * b + c for float64 arrays: Boldo & Melquiond's emulation through rounding to odd."""
    a, b, c = (np.asarray(v, np.float64) for v in (a, b, c))
    uh, ul = _two_prod(a, b)
    th, tl = _two_sum(c, uh)
    v, e = _two_sum(tl, ul)
    odd = (v.view(np.int64) & 1) == 1
    v = np.where((e != 0) & ~odd, np.nextafter(v, np.where(e > 0, np.inf, -np.inf)), v)  # round to odd
    return th + v


def affine_points(xy, M):
    """`xy1 @ M.T` for float64 (n, 2) points as OpenBLAS computes it, first two columns."""
    x, y = xy[:, 0], xy[:, 1]
    return np.stack([fma(y, M[r, 1], x * M[r, 0]) + M[r, 2] for r in range(2)], 1)


def resample(seg, n=N_POINTS):
    """resample_segments for one float32 (k, 2) segment -> float64 (n, 2)."""
    s = np.concatenate((seg, seg[0:1, :]), axis=0).astype(np.float64)
    L = len(s)
    x = np.arange(n, dtype=np.float64) * ((L - 1) / (n - 1))
    x[-1] = L - 1
    j = np.minimum(np.floor(x).astype(np.int64), L - 1)
    j1 = np.minimum(j + 1, L - 1)
    out = (s[j1] - s[j]) * (x - j)[:, None] + s[j]
    return np.where(((x == j) | (j >= L - 1))[:, None], s[j], out)


def xyn2xy(x, w, h, padw=0, padh=0):
    """utils/general.py xyn2xy on a float32 array with Python-scalar w, h, pads (NumPy 2: the scalars become float32)."""
    y = np.copy(x)
    y[..., 0] = w * x[..., 0] + padw
    y[..., 1] = h * x[..., 1] + padh
    return y


def segment2box(xy, width, height):
    x, y = xy.T
    inside = (x >= 0) & (y >= 0) & (x <= width) & (y <= height)
    x, y = x[inside], y[inside]
    return np.array([x.min(), y.min(), x.max(), y.max()]) if len(x) else np.zeros((1, 4))


# ----------------------------------------------------------------------------------------------------------------------
# cv2.fillPoly and polygon2mask
# ----------------------------------------------------------------------------------------------------------------------


def clip_lines(w, h, x1, y1, x2, y2):
    """cv2.clipLine for arrays of int64 segments against [0, w) x [0, h): (x1, y1, x2, y2, inside).  The points are
    updated even where the line misses the image, as cv2 does."""
    x1, y1, x2, y2 = (np.array(a, np.int64) for a in (x1, y1, x2, y2))
    right, bottom = w - 1, h - 1

    def code(x, y=None):
        c = (x < 0).astype(np.int64) + (x > right) * 2
        return c if y is None else c + (y < 0) * 4 + (y > bottom) * 8

    def step(num, den):  # (int64)((double)num_a * num_b / den), guarded where inactive
        return np.trunc(num / np.where(den == 0, 1.0, den)).astype(np.int64)

    c1, c2 = code(x1, y1), code(x2, y2)
    act = ((c1 & c2) == 0) & ((c1 | c2) != 0)
    m = act & ((c1 & 12) != 0)
    a = np.where(c1 < 8, 0, bottom)
    x1 = np.where(m, x1 + step((a - y1).astype(np.float64) * (x2 - x1), (y2 - y1).astype(np.float64)), x1)
    y1 = np.where(m, a, y1)
    c1 = np.where(m, code(x1), c1)
    m = act & ((c2 & 12) != 0)
    a = np.where(c2 < 8, 0, bottom)
    x2 = np.where(m, x2 + step((a - y2).astype(np.float64) * (x2 - x1), (y2 - y1).astype(np.float64)), x2)
    y2 = np.where(m, a, y2)
    c2 = np.where(m, code(x2), c2)
    act = act & ((c1 & c2) == 0) & ((c1 | c2) != 0)
    m = act & (c1 != 0)
    a = np.where(c1 == 1, 0, right)
    y1 = np.where(m, y1 + step((a - x1).astype(np.float64) * (y2 - y1), (x2 - x1).astype(np.float64)), y1)
    x1 = np.where(m, a, x1)
    c1 = np.where(m, 0, c1)
    m = act & (c2 != 0)
    a = np.where(c2 == 1, 0, right)
    y2 = np.where(m, y2 + step((a - x2).astype(np.float64) * (y2 - y1), (x2 - x1).astype(np.float64)), y2)
    x2 = np.where(m, a, x2)
    c2 = np.where(m, 0, c2)
    return x1, y1, x2, y2, (c1 | c2) == 0


def line_pixels(w, h, x1, y1, x2, y2):
    """(xs, ys) of every pixel cv2's 8-connected Line draws for the given segments (clipped, drawn left to right;
    after n major steps the minor offset is floor((2 minor n + major - 1) / (2 major)))."""
    x1, y1, x2, y2, ok = clip_lines(w, h, x1, y1, x2, y2)
    x1, y1, x2, y2 = x1[ok], y1[ok], x2[ok], y2[ok]
    sw = x2 < x1
    x1, x2 = np.where(sw, x2, x1), np.where(sw, x1, x2)
    y1, y2 = np.where(sw, y2, y1), np.where(sw, y1, y2)
    dx, dy = x2 - x1, y2 - y1
    sy = np.where(dy < 0, -1, 1)
    ady = np.abs(dy)
    vert = ady > dx
    major, minor = np.maximum(dx, ady), np.minimum(dx, ady)
    cnt = major + 1
    li = np.repeat(np.arange(len(x1)), cnt)
    n = np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    M, m = major[li], minor[li]
    k = np.where(M > 0, (2 * m * n + M - 1) // np.maximum(2 * M, 1), 0)
    v = vert[li]
    return x1[li] + np.where(v, k, n), y1[li] + sy[li] * np.where(v, n, k)


def fill_poly(pts, h, w):
    """cv2.fillPoly(np.zeros((h, w), np.uint8), [pts], 1) for one int32 (n, 2) polygon."""
    pts = np.asarray(pts, np.int64).reshape(-1, 2)
    out = np.zeros((h, w), np.uint8)
    if not len(pts):
        return out
    p0 = np.roll(pts, 1, 0)
    ax, ay, bx, by = p0[:, 0], p0[:, 1], pts[:, 0], pts[:, 1]
    xs, ys = line_pixels(w, h, ax, ay, bx, by)
    out[ys, xs] = 1
    cx1, cy1, cx2, cy2, _ = clip_lines(w, h, ax, ay, bx, by)
    outside = (ax < 0) | (ax >= w) | (bx < 0) | (bx >= w) | (ay < 0) | (ay >= h) | (by < 0) | (by >= h)
    use_y = outside & (cy1 != cy2)
    p0x = np.where(outside, cx1, ax) << XY_SHIFT
    p1x = np.where(outside, cx2, bx) << XY_SHIFT
    p0y, p1y = np.where(use_y, cy1, ay), np.where(use_y, cy2, by)
    e = ay != by
    p0x, p0y, p1x, p1y, ay, by = p0x[e], p0y[e], p1x[e], p1y[e], ay[e], by[e]
    if len(ay) < 2:
        return out
    num, den = p1x - p0x, p1y - p0y
    dxe = np.sign(num) * np.sign(den) * (np.abs(num) // np.abs(den))  # C division: truncation toward zero
    down = ay < by
    ey0 = np.minimum(ay, by)
    ex = np.where(down, p0x, p1x) + (ey0 - np.where(down, p0y, p1y)) * dxe
    lo, hi = np.maximum(ey0, 0), np.minimum(np.maximum(ay, by), h)
    cnt = np.maximum(hi - lo, 0)
    ei = np.repeat(np.arange(len(ey0)), cnt)
    yy = np.repeat(lo, cnt) + np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    x = ex[ei] + (yy - ey0[ei]) * dxe[ei]
    F = x >> XY_SHIFT
    # column c is set iff an odd number of crossings lie left of it, or a crossing is exactly c
    below = np.zeros(h, np.int64)
    np.add.at(below, yy[F < 0], 1)
    hist = np.zeros((h, w), np.int64)
    m = (F >= 0) & (F < w)
    np.add.at(hist, (yy[m], F[m]), 1)
    lt = below[:, None] + np.concatenate([np.zeros((h, 1), np.int64), np.cumsum(hist[:, :-1], 1)], 1)
    exact = np.zeros((h, w), bool)
    m &= (x & ((1 << XY_SHIFT) - 1)) == 0
    exact[yy[m], F[m]] = True
    out[((lt & 1) == 1) | exact] = 1
    return out


def resize_mask(mask, r):
    """cv2.resize(mask, (w // r, h // r)) for a 0/1 uint8 mask, r in {1, 4} (h, w multiples of r)."""
    if r == 1:
        return mask.copy()
    if r != 4:
        raise NotImplementedError(f"downsample_ratio {r}")
    a = mask[1::4, 1::4].astype(np.int64) + mask[1::4, 2::4] + mask[2::4, 1::4] + mask[2::4, 2::4]
    return (a >= 2).astype(np.uint8)


def polygon2mask(imgsz, polygons, color=1, downsample_ratio=1):
    """ultralytics.data.utils.polygon2mask for one polygon (the segmentation loader's only use)."""
    pts = np.asarray(polygons, dtype=np.int32).reshape(-1, 2)
    return resize_mask(fill_poly(pts, imgsz[0], imgsz[1]) * np.uint8(color), downsample_ratio)


def polygons2masks(imgsz, polygons, color, downsample_ratio=1):
    return np.array([polygon2mask(imgsz, [x.reshape(-1)], color, downsample_ratio) for x in polygons])


def overlap_order(areas):
    """np.argsort(-areas) on uint64 areas with ties in label order: zero areas first, then larger areas first."""
    areas = np.asarray(areas, np.uint64)
    return np.argsort(-areas, kind="stable")


def polygons2masks_overlap(imgsz, segments, downsample_ratio=1, order=None):
    """ultralytics.data.utils.polygons2masks_overlap; `order(areas)` picks the sort (default: overlap_order)."""
    masks = np.zeros((imgsz[0] // downsample_ratio, imgsz[1] // downsample_ratio), dtype=np.int32 if len(segments) > 255 else np.uint8)
    ms, areas = [], []
    for si in range(len(segments)):
        mask = polygon2mask(imgsz, [segments[si].reshape(-1)], downsample_ratio=downsample_ratio, color=1)
        ms.append(mask.astype(masks.dtype))
        areas.append(mask.sum())
    areas = np.asarray(areas)
    index = (order or overlap_order)(areas)
    ms = np.array(ms)[index]
    for i in range(len(segments)):
        masks = np.clip(masks + ms[i] * (i + 1), a_min=0, a_max=i + 1)
    return masks, index


# ----------------------------------------------------------------------------------------------------------------------
# the segment path of one item
# ----------------------------------------------------------------------------------------------------------------------


def warp_segments(targets, segments, M, s, width, height):
    """random_perspective's segment path (affine): float32 (n, 5) xyxy labels + n float32 segments -> kept labels and
    their float64 (k, 1000, 2) polygons."""
    n = len(targets)
    if not n:
        return targets, []
    new = np.zeros((n, 4))
    polys = []
    for i, seg in enumerate(segments):
        xy = affine_points(resample(seg), M)
        new[i] = segment2box(xy, width, height)
        polys.append(xy)
    keep = aug_ref.box_candidates(box1=targets[:, 1:5].T * s, box2=new.T, area_thr=0.01)
    targets = targets[keep]
    targets[:, 1:5] = new[keep]
    return targets, np.array(polys)[keep]


def _mosaic_draws(ds, index):
    """load_mosaic's draws: centre and three more indices -- unlike the detection loader's, the tiles are not shuffled."""
    yc, xc = (int(random.uniform(-x, 2 * ds.img_size + x)) for x in ds.mosaic_border)
    indices = [index, *random.choices(ds.indices, k=3)]
    return dict(xc=xc, yc=yc, indices=[int(i) for i in indices], persp=aug_ref.perspective_draws(ds.hyp))


def sample_params(ds, index):
    """Every random draw of LoadImagesAndLabelsAndMasks.__getitem__(index), in the reference's order."""
    hyp = ds.hyp
    p = dict(index=int(ds.indices[index]))
    p["mosaic"] = bool(ds.mosaic and random.random() < hyp["mosaic"])
    if p["mosaic"]:
        p["m"] = [_mosaic_draws(ds, p["index"])]
        if random.random() < hyp["mixup"]:
            p["m"].append(_mosaic_draws(ds, random.randint(0, ds.n - 1)))
            p["r"] = np.random.beta(32.0, 32.0)
    else:
        p["persp"] = aug_ref.perspective_draws(hyp)
    p["hsv"] = aug_ref.hsv_gains(hyp["hsv_h"], hyp["hsv_s"], hyp["hsv_v"])
    p["flipud"] = random.random() < hyp["flipud"]
    p["fliplr"] = random.random() < hyp["fliplr"]
    return p


def mosaic(ds, md):
    """load_mosaic with segments: (warped image, float32 labels, float64 polygons)."""
    s = ds.img_size
    img4 = np.full((s * 2, s * 2, 3), aug_ref.BORDER, np.uint8)
    ims = [ds.load_image(i) for i in md["indices"]]
    labels4, segments4 = [], []
    for (im, _, (h, w)), (x1a, y1a, x2a, y2a, x1b, y1b), idx in zip(ims, aug_ref.placements(md["xc"], md["yc"], s, [x[2] for x in ims]),
                                                                    md["indices"]):
        img4[y1a:y2a, x1a:x2a] = im[y1b:y1b + (y2a - y1a), x1b:x1b + (x2a - x1a)]
        labels, segments = ds.labels[idx].copy(), list(ds.segments[idx])
        if labels.size:
            labels[:, 1:] = aug_ref.xywhn2xyxy(labels[:, 1:], w, h, x1a - x1b, y1a - y1b)
            segments = [xyn2xy(x, w, h, x1a - x1b, y1a - y1b) for x in segments]
        labels4.append(labels)
        segments4.extend(segments)
    labels4 = np.concatenate(labels4, 0)
    for x in (labels4[:, 1:], *segments4):
        np.clip(x, 0, 2 * s, out=x)
    M = aug_ref.affine(md["persp"], img4.shape[:2], ds.mosaic_border)
    img = aug_ref.warp_affine(img4, M[:2], (s, s))
    labels, polys = warp_segments(labels4, segments4, M, md["persp"][3], s, s)
    return img, labels, polys


def letterbox_item(ds, index, persp):
    from oracle import pre_ref

    img, (h0, w0), (h, w) = ds.load_image(index)
    img, ratio, pad = pre_ref.letterbox(img, ds.img_size, auto=False, scaleup=True)
    labels = ds.labels[index].copy()
    segments = [xyn2xy(x, ratio[0] * w, ratio[1] * h, padw=pad[0], padh=pad[1]) for x in ds.segments[index]]
    if labels.size:
        labels[:, 1:] = aug_ref.xywhn2xyxy(labels[:, 1:], ratio[0] * w, ratio[1] * h, padw=pad[0], padh=pad[1])
    M = aug_ref.affine(persp, img.shape[:2], (0, 0))
    if (M != np.eye(3)).any():
        img = aug_ref.warp_affine(img, M[:2], (img.shape[1], img.shape[0]))
    labels, polys = warp_segments(labels, segments, M, persp[3], img.shape[1], img.shape[0])
    return img, labels, polys


def item_from_params(ds, p, overlap, ratio, order=None):
    """(CHW RGB uint8 image, float32 (nl, 6) labels_out, masks) of one item; masks as __getitem__ returns them."""
    if p["mosaic"]:
        img, labels, polys = mosaic(ds, p["m"][0])
        if len(p["m"]) == 2:
            im2, labels2, polys2 = mosaic(ds, p["m"][1])
            r = p["r"]
            img = (img * r + im2 * (1 - r)).astype(np.uint8)
            labels = np.concatenate((labels, labels2), 0)
            polys = [*polys, *polys2]
    else:
        img, labels, polys = letterbox_item(ds, p["index"], p["persp"])
    nl = len(labels)
    h, w = img.shape[:2]
    if nl:
        labels[:, 1:5] = aug_ref.xyxy2xywhn(labels[:, 1:5], w, h)
        if overlap:
            masks, idx = polygons2masks_overlap((h, w), polys, ratio, order)
            masks = masks[None]
            labels = labels[idx]
        else:
            masks = polygons2masks((h, w), polys, 1, ratio)
    else:
        masks = np.zeros((1 if overlap else 0, h // ratio, w // ratio), np.float32)
    if p["hsv"] is not None:
        img = aug_ref.apply_hsv(img, p["hsv"])
    if p["flipud"]:
        img = np.flipud(img)
        if nl:
            labels[:, 2] = 1 - labels[:, 2]
            masks = masks[:, ::-1]
    if p["fliplr"]:
        img = np.fliplr(img)
        if nl:
            labels[:, 1] = 1 - labels[:, 1]
            masks = masks[:, :, ::-1]
    out = np.zeros((nl, 6), np.float32)
    out[:, 1:] = labels
    return np.ascontiguousarray(img.transpose(2, 0, 1)[::-1]), out, np.ascontiguousarray(masks)


def batch_mask_dtype(dtypes):
    """torch.cat's promotion of the per-image mask tensors (uint8, int32, or float32 zeros for an image without labels)."""
    out = np.uint8
    for d in dtypes:
        out = np.promote_types(out, d)
    return {np.dtype(np.uint8): np.uint8, np.dtype(np.int32): np.int32}.get(np.dtype(out), np.float32)


def get_batch(ds, batch_indices, overlap, ratio, order=None):
    """collate_fn over __getitem__: (imgs, targets, masks, params)."""
    params = [sample_params(ds, i) for i in batch_indices]
    items = [item_from_params(ds, p, overlap, ratio, order) for p in params]
    for i, (_, lb, _) in enumerate(items):
        lb[:, 0] = i
    dt = batch_mask_dtype([x[2].dtype for x in items])
    masks = np.concatenate([x[2].astype(dt) for x in items], 0)
    return np.stack([x[0] for x in items]), np.concatenate([x[1] for x in items], 0), masks, params
