"""ORACLE (test infrastructure, never on the product path): numpy restatement of the detection training augmentation
(`augment=True`, `rect=False`) -- mosaic, random_perspective (affine), mixup, HSV and flips -- and its label path.

Only tests/ and tools/ may import this.

Reference lines restated (paths relative to the reference tree):
  utils/dataloaders.py:696-766   LoadImagesAndLabels.__getitem__ (draw order, non-mosaic branch, flips, CHW RGB) -> sample_params, item_from_params
  utils/dataloaders.py:798-855   load_mosaic (centre, tile placement x1a..y2b, label pads, clip to [0, 2s])       -> placements, mosaic
  utils/augmentations.py:69-82   augment_hsv (gains, LUTs in float64, cvtColor both ways)                          -> hsv_gains, apply_hsv
  utils/augmentations.py:118-197 random_perspective (M = T @ S @ R @ P @ C, warpAffine, box warp + filter)          -> affine, warp_labels
  utils/augmentations.py:225-233 mixup (np.random.beta(32, 32), trunc(a*r + b*(1-r)))                              -> item_from_params
  utils/augmentations.py:236-245 box_candidates                                                                    -> box_candidates
Third-party arithmetic, pinned against the installed cv2 by tests/golden/make_aug_golden.py:
  * cv2.warpAffine (uint8, INTER_LINEAR, constant border): OpenCV's fixed-point remap.  M is inverted in double
    (invertAffineTransform), adelta[x] = rint(iM00*x*1024), X0 = rint((iM01*y + iM02)*1024) + 16, X = (X0 + adelta) >> 5
    (a 5-bit fraction), weights (32-fy)(32-fx)*32 etc., result (sum + 2^14) >> 15; taps outside the source read 114.
  * COLOR_BGR2HSV on uint8: the integer formula (hsv_shift 12, sdiv / hdiv tables).
  * COLOR_HSV2BGR on uint8: float32 with 1 - s*h and 1 - s*(1-h) FUSED (one rounding), times 255, truncated -- for
    pixels inside the 32-pixel SIMD blocks of a row.  The last (width % 32) pixels of a row go through the scalar
    tail, which rounds to nearest instead.  Both forms equal cv2 over all 180*256*256 inputs.
  * numpy's float64 `xy @ M.T` (OpenBLAS): x*M00, then fma(y, M01, .), then + M02.
"""
from __future__ import annotations

import math
import random

import numpy as np

BORDER = 114
SIMD_BLOCK = 32  # pixels per SIMD block of the AVX2 HSV2BGR path: the tail of a row rounds instead of truncating

# ----------------------------------------------------------------------------------------------------------------------
# warpAffine
# ----------------------------------------------------------------------------------------------------------------------


def invert_affine(M):
    """cv2.invertAffineTransform for a 2x3 float64 matrix, in the same double operation order."""
    m = [float(v) for v in np.asarray(M, np.float64).reshape(6)]
    D = m[0] * m[4] - m[1] * m[3]
    D = 1.0 / D if D != 0 else 0.0
    A11, A22, A12, A21 = m[4] * D, m[0] * D, -m[1] * D, -m[3] * D
    b1 = -A11 * m[2] - A12 * m[5]
    b2 = -A21 * m[2] - A22 * m[5]
    return np.array([[A11, A12, b1], [A21, A22, b2]], np.float64)


def warp_affine(im, M, dsize, border=BORDER):
    """cv2.warpAffine(im, M, dsize, borderValue=(border,)*3) for uint8 HWC images, bit-exact."""
    W, H = int(dsize[0]), int(dsize[1])
    iM = invert_affine(M)
    h, w = im.shape[:2]
    xs = np.arange(W, dtype=np.float64)
    ys = np.arange(H, dtype=np.float64)
    adelta = np.rint(iM[0, 0] * xs * 1024).astype(np.int64)
    bdelta = np.rint(iM[1, 0] * xs * 1024).astype(np.int64)
    X0 = np.rint((iM[0, 1] * ys + iM[0, 2]) * 1024).astype(np.int64) + 16
    Y0 = np.rint((iM[1, 1] * ys + iM[1, 2]) * 1024).astype(np.int64) + 16
    X = (X0[:, None] + adelta[None, :]) >> 5
    Y = (Y0[:, None] + bdelta[None, :]) >> 5
    sx, sy = np.clip(X >> 5, -32768, 32767), np.clip(Y >> 5, -32768, 32767)
    fx, fy = X & 31, Y & 31
    pad = np.full((h + 2, w + 2, im.shape[2]), border, np.int64)
    pad[1:-1, 1:-1] = im

    def tap(yy, xx):
        return pad[np.clip(yy + 1, 0, h + 1), np.clip(xx + 1, 0, w + 1)]

    wts = [((32 - fy) * (32 - fx) * 32), ((32 - fy) * fx * 32), (fy * (32 - fx) * 32), (fy * fx * 32)]
    v = tap(sy, sx) * wts[0][..., None] + tap(sy, sx + 1) * wts[1][..., None] + tap(sy + 1, sx) * wts[2][..., None] + tap(sy + 1, sx + 1) * wts[3][..., None]
    return np.clip((v + (1 << 14)) >> 15, 0, 255).astype(np.uint8)


# ----------------------------------------------------------------------------------------------------------------------
# HSV
# ----------------------------------------------------------------------------------------------------------------------
_SH = 12
_SDIV = np.array([0] + [int(np.rint((255 << _SH) / (1.0 * i))) for i in range(1, 256)], np.int64)
_HDIV = np.array([0] + [int(np.rint((180 << _SH) / (6.0 * i))) for i in range(1, 256)], np.int64)
_SECTOR = np.array([[1, 3, 0], [1, 0, 2], [3, 0, 1], [0, 2, 1], [0, 1, 3], [2, 1, 0]])


def bgr2hsv(im):
    """cv2.cvtColor(im, COLOR_BGR2HSV) for uint8, bit-exact."""
    b, g, r = (im[..., k].astype(np.int64) for k in range(3))
    v = np.maximum(np.maximum(b, g), r)
    diff = v - np.minimum(np.minimum(b, g), r)
    vr = v == r
    vg = (v == g) & ~vr
    s = (diff * _SDIV[v] + (1 << (_SH - 1))) >> _SH
    h = np.where(vr, g - b, np.where(vg, b - r + 2 * diff, r - g + 4 * diff))
    h = (h * _HDIV[diff] + (1 << (_SH - 1))) >> _SH
    h = np.where(h < 0, h + 180, h)
    return np.stack([h, s, v], -1).astype(np.uint8)


def _fma32(a, b, c):
    """float32 a*b + c with one rounding (the exact product of two floats fits a double, the sum is rounded once more
    only when it is inexact in double, which cannot change the float32 result here: |a*b|, |c| <= 1 at 2^-48 spacing)."""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def hsv2bgr(hsv):
    """cv2.cvtColor(hsv, COLOR_HSV2BGR) for uint8 HWC (or (..., 3)) arrays, bit-exact: columns inside the row's
    32-pixel SIMD blocks truncate, the row's tail (last width % 32 columns) rounds."""
    f32 = np.float32
    one = f32(1)
    h = hsv[..., 0].astype(f32) * f32(6.0 / 180)
    s = hsv[..., 1].astype(f32) * f32(1 / 255)
    v = hsv[..., 2].astype(f32) * f32(1 / 255)
    sec = np.floor(h).astype(np.int64)
    fr = (h - sec.astype(f32)).astype(f32)
    ones = np.ones_like(s)
    tab = np.stack([v, v * (one - s), v * _fma32(-s, fr, ones), v * _fma32(-s, one - fr, ones)], -1).astype(f32)
    out = (np.take_along_axis(tab, _SECTOR[sec % 6], -1) * f32(255)).astype(f32)
    res = np.trunc(out)
    if hsv.ndim >= 2:
        width = hsv.shape[-2]
        tail = width - width % SIMD_BLOCK
        res[..., tail:, :] = np.rint(out[..., tail:, :])
    return np.clip(res, 0, 255).astype(np.uint8)


def hsv_gains(hgain, sgain, vgain):
    """The draw augment_hsv makes (none when every gain is zero): float64 (3,) gains, or None."""
    if hgain or sgain or vgain:
        return np.random.uniform(-1, 1, 3) * [hgain, sgain, vgain] + 1
    return None


def hsv_luts(r):
    """(3, 256) uint8 LUTs built in float64 exactly as augment_hsv builds them."""
    x = np.arange(0, 256, dtype=r.dtype)
    return np.stack([((x * r[0]) % 180).astype(np.uint8), np.clip(x * r[1], 0, 255).astype(np.uint8),
                     np.clip(x * r[2], 0, 255).astype(np.uint8)])


def apply_hsv(im, r):
    """augment_hsv's colour transform for given gains r (not in place)."""
    lut = hsv_luts(r)
    hsv = bgr2hsv(im)
    hsv = np.stack([lut[k][hsv[..., k]] for k in range(3)], -1)
    return hsv2bgr(hsv)


# ----------------------------------------------------------------------------------------------------------------------
# geometry and labels
# ----------------------------------------------------------------------------------------------------------------------


def rotation_matrix(angle, scale):
    """cv2.getRotationMatrix2D(angle=angle, center=(0, 0), scale=scale)."""
    a = angle * (math.pi / 180)
    alpha, beta = math.cos(a) * scale, math.sin(a) * scale
    return np.array([[alpha, beta, (1 - alpha) * 0 - beta * 0], [-beta, alpha, beta * 0 + (1 - alpha) * 0]])


def affine(draws, im_hw, border):
    """random_perspective's M (3x3 float64) from its draws (px, py, a, s, shx, shy, tx, ty) and the input image size."""
    px, py, a, s, shx, shy, tx, ty = draws
    height, width = im_hw[0] + border[0] * 2, im_hw[1] + border[1] * 2
    C = np.eye(3)
    C[0, 2] = -im_hw[1] / 2
    C[1, 2] = -im_hw[0] / 2
    P = np.eye(3)
    P[2, 0], P[2, 1] = px, py
    R = np.eye(3)
    R[:2] = rotation_matrix(a, s)
    S = np.eye(3)
    S[0, 1] = math.tan(shx * math.pi / 180)
    S[1, 0] = math.tan(shy * math.pi / 180)
    T = np.eye(3)
    T[0, 2] = tx * width
    T[1, 2] = ty * height
    return T @ S @ R @ P @ C


def placements(xc, yc, s, hws):
    """load_mosaic's (x1a, y1a, x2a, y2a, x1b, y1b) for the four tiles of (h, w) sizes `hws`, in tile order."""
    out = []
    for i, (h, w) in enumerate(hws):
        if i == 0:
            x1a, y1a, x2a, y2a = max(xc - w, 0), max(yc - h, 0), xc, yc
            x1b, y1b = w - (x2a - x1a), h - (y2a - y1a)
        elif i == 1:
            x1a, y1a, x2a, y2a = xc, max(yc - h, 0), min(xc + w, s * 2), yc
            x1b, y1b = 0, h - (y2a - y1a)
        elif i == 2:
            x1a, y1a, x2a, y2a = max(xc - w, 0), yc, xc, min(s * 2, yc + h)
            x1b, y1b = w - (x2a - x1a), 0
        else:
            x1a, y1a, x2a, y2a = xc, yc, min(xc + w, s * 2), min(s * 2, yc + h)
            x1b, y1b = 0, 0
        out.append((x1a, y1a, x2a, y2a, x1b, y1b))
    return out


def xywhn2xyxy(x, w, h, padw=0, padh=0):
    y = np.copy(x)
    y[..., 0] = w * (x[..., 0] - x[..., 2] / 2) + padw
    y[..., 1] = h * (x[..., 1] - x[..., 3] / 2) + padh
    y[..., 2] = w * (x[..., 0] + x[..., 2] / 2) + padw
    y[..., 3] = h * (x[..., 1] + x[..., 3] / 2) + padh
    return y


def xyxy2xywhn(x, w, h, eps=1e-3):
    """xyxy2xywhn(clip=True): clips `x` in place to (w - eps, h - eps) first, as the reference does."""
    x[..., [0, 2]] = x[..., [0, 2]].clip(0, w - eps)
    x[..., [1, 3]] = x[..., [1, 3]].clip(0, h - eps)
    y = np.copy(x)
    y[..., 0] = ((x[..., 0] + x[..., 2]) / 2) / w
    y[..., 1] = ((x[..., 1] + x[..., 3]) / 2) / h
    y[..., 2] = (x[..., 2] - x[..., 0]) / w
    y[..., 3] = (x[..., 3] - x[..., 1]) / h
    return y


def box_candidates(box1, box2, wh_thr=2, ar_thr=100, area_thr=0.1, eps=1e-16):
    w1, h1 = box1[2] - box1[0], box1[3] - box1[1]
    w2, h2 = box2[2] - box2[0], box2[3] - box2[1]
    ar = np.maximum(w2 / (h2 + eps), h2 / (w2 + eps))
    return (w2 > wh_thr) & (h2 > wh_thr) & (w2 * h2 / (w1 * h1 + eps) > area_thr) & (ar < ar_thr)


def warp_labels(targets, M, s, width, height):
    """random_perspective's box path (affine, no segments): float32 (n, 5) xyxy labels -> kept rows, float32."""
    n = len(targets)
    if not n:
        return targets
    xy = np.ones((n * 4, 3))
    xy[:, :2] = targets[:, [1, 2, 3, 4, 1, 4, 3, 2]].reshape(n * 4, 2)
    xy = (xy @ M.T)[:, :2].reshape(n, 8)
    x, y = xy[:, [0, 2, 4, 6]], xy[:, [1, 3, 5, 7]]
    new = np.concatenate((x.min(1), y.min(1), x.max(1), y.max(1))).reshape(4, n).T
    new[:, [0, 2]] = new[:, [0, 2]].clip(0, width)
    new[:, [1, 3]] = new[:, [1, 3]].clip(0, height)
    i = box_candidates(box1=targets[:, 1:5].T * s, box2=new.T, area_thr=0.10)
    targets = targets[i]
    targets[:, 1:5] = new[i]
    return targets


# ----------------------------------------------------------------------------------------------------------------------
# the draw sequence of __getitem__
# ----------------------------------------------------------------------------------------------------------------------


def perspective_draws(hyp):
    """random_perspective's eight draws, in order (the two perspective draws happen even when perspective == 0)."""
    p, d, sc, sh, t = hyp["perspective"], hyp["degrees"], hyp["scale"], hyp["shear"], hyp["translate"]
    px = random.uniform(-p, p)
    py = random.uniform(-p, p)
    a = random.uniform(-d, d)
    s = random.uniform(1 - sc, 1 + sc)
    shx = random.uniform(-sh, sh)
    shy = random.uniform(-sh, sh)
    tx = random.uniform(0.5 - t, 0.5 + t)
    ty = random.uniform(0.5 - t, 0.5 + t)
    return (px, py, a, s, shx, shy, tx, ty)


def _mosaic_draws(ds, index):
    yc, xc = (int(random.uniform(-x, 2 * ds.img_size + x)) for x in ds.mosaic_border)
    indices = [index, *random.choices(ds.indices, k=3)]
    random.shuffle(indices)
    return dict(xc=xc, yc=yc, indices=[int(i) for i in indices], persp=perspective_draws(ds.hyp))


def sample_params(ds, index):
    """Every random draw __getitem__(index) makes, in the reference's order, from Python's `random` and `np.random`."""
    hyp = ds.hyp
    index = int(ds.indices[index])
    p = dict(index=index)
    p["mosaic"] = bool(ds.mosaic and random.random() < hyp["mosaic"])
    if p["mosaic"]:
        p["m"] = [_mosaic_draws(ds, index)]
        if random.random() < hyp["mixup"]:  # drawn even when mixup == 0
            p["m"].append(_mosaic_draws(ds, int(random.choice(ds.indices))))
            p["r"] = np.random.beta(32.0, 32.0)
    else:
        p["persp"] = perspective_draws(hyp)
    p["hsv"] = hsv_gains(hyp["hsv_h"], hyp["hsv_s"], hyp["hsv_v"])
    p["flipud"] = random.random() < hyp["flipud"]
    p["fliplr"] = random.random() < hyp["fliplr"]
    return p


# ----------------------------------------------------------------------------------------------------------------------
# one item
# ----------------------------------------------------------------------------------------------------------------------


def mosaic(ds, md):
    """load_mosaic from its draws: (warped s x s image, float32 labels)."""
    s = ds.img_size
    img4 = np.full((s * 2, s * 2, 3), BORDER, np.uint8)
    ims = [ds.load_image(i) for i in md["indices"]]
    labels4 = []
    for (im, _, (h, w)), (x1a, y1a, x2a, y2a, x1b, y1b), idx in zip(ims, placements(md["xc"], md["yc"], s, [x[2] for x in ims]), md["indices"]):
        img4[y1a:y2a, x1a:x2a] = im[y1b:y1b + (y2a - y1a), x1b:x1b + (x2a - x1a)]
        labels = ds.labels[idx].copy()
        if labels.size:
            labels[:, 1:] = xywhn2xyxy(labels[:, 1:], w, h, x1a - x1b, y1a - y1b)
        labels4.append(labels)
    labels4 = np.concatenate(labels4, 0)
    np.clip(labels4[:, 1:], 0, 2 * s, out=labels4[:, 1:])
    M = affine(md["persp"], img4.shape[:2], ds.mosaic_border)
    img = warp_affine(img4, M[:2], (s, s))
    return img, warp_labels(labels4, M, md["persp"][3], s, s)


def letterbox_item(ds, index, persp):
    """The non-mosaic branch: letterbox(auto=False, scaleup=True) then random_perspective with border (0, 0)."""
    from oracle import pre_ref

    img, _, (h, w) = ds.load_image(index)
    img, ratio, pad = pre_ref.letterbox(img, ds.img_size, auto=False, scaleup=True)
    labels = ds.labels[index].copy()
    if labels.size:
        labels[:, 1:] = xywhn2xyxy(labels[:, 1:], ratio[0] * w, ratio[1] * h, padw=pad[0], padh=pad[1])
    M = affine(persp, img.shape[:2], (0, 0))
    if (M != np.eye(3)).any():
        img = warp_affine(img, M[:2], (img.shape[1], img.shape[0]))
    return img, warp_labels(labels, M, persp[3], img.shape[1], img.shape[0])


def item_from_params(ds, p):
    """(CHW RGB uint8 image, float32 (nl, 6) labels_out with column 0 zero) for one item's draws."""
    if p["mosaic"]:
        img, labels = mosaic(ds, p["m"][0])
        if len(p["m"]) == 2:
            im2, labels2 = mosaic(ds, p["m"][1])
            r = p["r"]
            img = (img * r + im2 * (1 - r)).astype(np.uint8)
            labels = np.concatenate((labels, labels2), 0)
    else:
        img, labels = letterbox_item(ds, p["index"], p["persp"])
    nl = len(labels)
    if nl:
        labels[:, 1:5] = xyxy2xywhn(labels[:, 1:5], img.shape[1], img.shape[0])
    if p["hsv"] is not None:
        img = apply_hsv(img, p["hsv"])
    if p["flipud"]:
        img = np.flipud(img)
        if nl:
            labels[:, 2] = 1 - labels[:, 2]
    if p["fliplr"]:
        img = np.fliplr(img)
        if nl:
            labels[:, 1] = 1 - labels[:, 1]
    out = np.zeros((nl, 6), np.float32)
    out[:, 1:] = labels
    return np.ascontiguousarray(img.transpose(2, 0, 1)[::-1]), out


def draw_vector(p):
    """One item's draws as a fixed-length float64 row (for the fixture): mosaic flag, per mosaic xc, yc, 4 indices and
    the 8 perspective draws (the non-mosaic branch fills the first mosaic's perspective slots), r, gains, flips."""
    v = np.full(2 + 2 * 14 + 1 + 3 + 2, np.nan)
    v[0], v[1] = p["index"], p["mosaic"]
    for k, m in enumerate(p.get("m", [])):
        v[2 + 14 * k: 2 + 14 * (k + 1)] = [m["xc"], m["yc"], *m["indices"], *m["persp"]]
    if not p["mosaic"]:
        v[8:16] = p["persp"]
    v[30] = p.get("r", np.nan)
    if p["hsv"] is not None:
        v[31:34] = p["hsv"]
    v[34], v[35] = p["flipud"], p["fliplr"]
    return v


def get_batch(ds, batch_indices):
    """collate_fn over __getitem__ for the given dataset indices: (imgs (B,3,s,s) uint8, targets (nt, 6) float32, params)."""
    params = [sample_params(ds, i) for i in batch_indices]
    items = [item_from_params(ds, p) for p in params]
    for i, (_, lb) in enumerate(items):
        lb[:, 0] = i
    return np.stack([x[0] for x in items]), np.concatenate([x[1] for x in items], 0), params
