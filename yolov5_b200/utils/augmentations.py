"""The step right before the hot path, on the device: letterbox resize/pad + BGR->RGB + HWC->CHW + /255
(reference utils/augmentations.py:85-115, utils/dataloaders.py:354-357, detect.py:205-208, models/common.py:924-926),
and the training augmentations random_perspective (affine), augment_hsv and mixup (reference :69-82, :118-197, :225-233).

``letterbox`` keeps the reference's signature and return value ``(image, ratio, (dw, dh))``; the resize itself runs in
liby5b200 (y5_letterbox: OpenCV's fixed-point bilinear kernel restated bit for bit, so the letterboxed bytes equal what
``cv2.resize`` + ``cv2.copyMakeBorder`` produce).  ``letterbox_batch`` is the batched form the engine wants: a list of
device-resident uint8 HWC images of different sizes -> one (B,3,H,W) tensor (uint8, or already scaled to [0,1] in
fp16/bf16/fp32), one launch per 24 images, no host synchronisation.
"""
from __future__ import annotations

import ctypes as C
import math
import random

import numpy as np
import torch

from .. import _lib


def letterbox_geometry(shape_hw, new_shape=(640, 640), auto=True, scaleFill=False, scaleup=True, stride=32):
    """(new_unpad (w, h), ratio (w, h), (dw, dh), (top, bottom, left, right)) as utils/augmentations.py:85-113 derives them."""
    if isinstance(new_shape, int):
        new_shape = (new_shape, new_shape)
    h, w = int(shape_hw[0]), int(shape_hw[1])
    r = min(new_shape[0] / h, new_shape[1] / w)
    if not scaleup:  # only scale down (better val mAP)
        r = min(r, 1.0)
    ratio = r, r
    new_unpad = round(w * r), round(h * r)
    dw, dh = new_shape[1] - new_unpad[0], new_shape[0] - new_unpad[1]
    if auto:  # minimum rectangle
        dw, dh = float(np.mod(dw, stride)), float(np.mod(dh, stride))
    elif scaleFill:  # stretch
        dw, dh = 0.0, 0.0
        new_unpad = (new_shape[1], new_shape[0])
        ratio = new_shape[1] / w, new_shape[0] / h
    dw /= 2
    dh /= 2
    top, bottom = round(dh - 0.1), round(dh + 0.1)
    left, right = round(dw - 0.1), round(dw + 0.1)
    return new_unpad, ratio, (dw, dh), (top, bottom, left, right)


def _as_device_hwc(im, device):
    if isinstance(im, np.ndarray):
        im = torch.from_numpy(np.ascontiguousarray(im))
    if not isinstance(im, torch.Tensor) or im.dtype != torch.uint8 or im.dim() != 3 or im.shape[2] != 3:
        raise TypeError("y5b200: letterbox expects uint8 HWC images with 3 channels")
    if not im.is_cuda:
        if device is None:
            if not torch.cuda.is_available():
                raise RuntimeError("y5b200: letterbox runs in liby5b200 on a CUDA device (no CPU / OpenCV fallback)")
            device = torch.device("cuda", torch.cuda.current_device())
        im = im.to(device, non_blocking=True)
    if im.stride(2) != 1 or im.stride(1) != 3:
        im = im.contiguous()
    return im


def letterbox_batch(images, new_shape=(640, 640), color=(114, 114, 114), auto=False, scaleFill=False, scaleup=True, stride=32,
                    swap_rb=True, dtype=torch.uint8, device=None, out=None, s2d_out=None):
    """images: list of uint8 HWC (BGR unless swap_rb=False) tensors / arrays of any sizes.  All images are letterboxed to
    the SAME canvas: `new_shape` (auto=False), or the minimum-rectangle canvas of the first image (auto=True, as the
    reference does per image: then every image must produce that canvas).  Returns (batch, ratios, pads):
    batch (B,3,H,W) `dtype` (uint8 = the dataloader's bytes; float dtypes are divided by 255), CHW with RGB order when
    swap_rb.  `s2d_out` = (buffer, row_px, x_off) writes the stem's space-to-depth cells instead (engine internal)."""
    if isinstance(new_shape, int):
        new_shape = (new_shape, new_shape)
    if len(set(color)) != 1:
        raise NotImplementedError("y5b200: letterbox border colour must be grey (the reference uses (114, 114, 114))")
    ims = [_as_device_hwc(im, device) for im in images]
    dev = ims[0].device
    geo = [letterbox_geometry(im.shape[:2], new_shape, auto, scaleFill, scaleup, stride) for im in ims]
    canvases = {(g[0][1] + g[3][0] + g[3][1], g[0][0] + g[3][2] + g[3][3]) for g in geo}
    if len(canvases) != 1:
        raise ValueError(f"y5b200: letterbox_batch needs one output shape for the whole batch, got {sorted(canvases)} (use auto=False)")
    out_h, out_w = canvases.pop()
    lib = _lib.lib()
    arr = (_lib.LetterboxImage * len(ims))()
    for d, im, g in zip(arr, ims, geo):
        d.data, d.src_h, d.src_w, d.row_bytes = im.data_ptr(), im.shape[0], im.shape[1], im.stride(0)
        d.new_w, d.new_h = g[0]
        d.top, d.left = g[3][0], g[3][2]
    with _lib.on(dev):
        if s2d_out is not None:
            buf, row_px, x_off = s2d_out
            _lib.check(lib.y5_letterbox(arr, len(ims), out_h, out_w, int(swap_rb), int(color[0]), buf.data_ptr(), _lib.dtype_code(buf.dtype), 1,
                                        row_px, x_off, C.c_void_p(_lib.stream_ptr(dev))), "letterbox")
            res = buf
        else:
            res = out if out is not None else torch.empty(len(ims), 3, out_h, out_w, dtype=dtype, device=dev)
            assert res.shape == (len(ims), 3, out_h, out_w) and res.is_contiguous()
            _lib.check(lib.y5_letterbox(arr, len(ims), out_h, out_w, int(swap_rb), int(color[0]), res.data_ptr(), _lib.dtype_code(res.dtype), 0, 0,
                                        0, C.c_void_p(_lib.stream_ptr(dev))), "letterbox")
    for im in ims:  # the launch reads these buffers asynchronously: tie their lifetime to the stream
        im.record_stream(torch.cuda.current_stream(dev))
    return res, [g[1] for g in geo], [g[2] for g in geo]


def letterbox(im, new_shape=(640, 640), color=(114, 114, 114), auto=True, scaleFill=False, scaleup=True, stride=32):
    """Reference signature (utils/augmentations.py:85): one HWC uint8 image -> (letterboxed HWC image, ratio, (dw, dh)).
    numpy in -> numpy out (the bytes cv2 would produce), CUDA tensor in -> CUDA tensor out."""
    is_np = isinstance(im, np.ndarray)
    batch, ratios, pads = letterbox_batch([im], new_shape, color, auto, scaleFill, scaleup, stride, swap_rb=False)
    hwc = batch[0].permute(1, 2, 0).contiguous()
    return (hwc.cpu().numpy() if is_np else hwc), ratios[0], pads[0]


# ----------------------------------------------------------------------------------------------------------------------
# training augmentation (liby5b200 y5_aug_gather / y5_aug_labels; utils/dataloaders.py batches these per training step)
# ----------------------------------------------------------------------------------------------------------------------
def perspective_draws(degrees, translate, scale, shear, perspective):
    """random_perspective's eight draws (px, py, angle, scale, shear x, shear y, tx, ty), in the reference's order: the two
    perspective draws happen even when perspective == 0."""
    px = random.uniform(-perspective, perspective)
    py = random.uniform(-perspective, perspective)
    a = random.uniform(-degrees, degrees)
    s = random.uniform(1 - scale, 1 + scale)
    shx = random.uniform(-shear, shear)
    shy = random.uniform(-shear, shear)
    tx = random.uniform(0.5 - translate, 0.5 + translate)
    ty = random.uniform(0.5 - translate, 0.5 + translate)
    return px, py, a, s, shx, shy, tx, ty


def affine_matrix(draws, im_hw, border=(0, 0)):
    """random_perspective's M = T @ S @ R @ P @ C (3x3 float64, numpy products as the reference forms them) for an input
    of size im_hw; R is cv2.getRotationMatrix2D(angle, (0, 0), scale) restated."""
    px, py, a, s, shx, shy, tx, ty = draws
    C = np.eye(3)
    C[0, 2] = -im_hw[1] / 2
    C[1, 2] = -im_hw[0] / 2
    P = np.eye(3)
    P[2, 0], P[2, 1] = px, py
    ang = a * (math.pi / 180)
    alpha, beta = math.cos(ang) * s, math.sin(ang) * s
    R = np.eye(3)
    R[:2] = [[alpha, beta, (1 - alpha) * 0 - beta * 0], [-beta, alpha, beta * 0 + (1 - alpha) * 0]]
    S = np.eye(3)
    S[0, 1] = math.tan(shx * math.pi / 180)
    S[1, 0] = math.tan(shy * math.pi / 180)
    T = np.eye(3)
    T[0, 2] = tx * (im_hw[1] + border[1] * 2)
    T[1, 2] = ty * (im_hw[0] + border[0] * 2)
    return T @ S @ R @ P @ C


def invert_affine(M):
    """cv2.invertAffineTransform(M[:2]) in the same double operation order -> 6 floats."""
    m = [float(v) for v in np.asarray(M, np.float64)[:2].reshape(6)]
    D = m[0] * m[4] - m[1] * m[3]
    D = 1.0 / D if D != 0 else 0.0
    A11, A22, A12, A21 = m[4] * D, m[0] * D, -m[1] * D, -m[3] * D
    return [A11, A12, -A11 * m[2] - A12 * m[5], A21, A22, -A21 * m[2] - A22 * m[5]]


def hsv_luts(r):
    """augment_hsv's three uint8 LUTs, built in float64 as the reference builds them."""
    x = np.arange(0, 256, dtype=r.dtype)
    return np.stack([((x * r[0]) % 180).astype(np.uint8), np.clip(x * r[1], 0, 255).astype(np.uint8),
                     np.clip(x * r[2], 0, 255).astype(np.uint8)])


def set_tile(tile, src, x1a, y1a, x2a, y2a, dx, dy):
    """Fill a y5_aug_tile from a device uint8 tensor: HWC (h, w, 3) or CHW planes (3, h, w)."""
    if src.dim() == 3 and src.shape[0] == 3 and src.shape[2] != 3:
        tile.row_bytes, tile.pixel_stride, tile.channel_stride = src.stride(1), src.stride(2), src.stride(0)
    else:
        tile.row_bytes, tile.pixel_stride, tile.channel_stride = src.stride(0), src.stride(1), src.stride(2)
    tile.src = src.data_ptr()
    tile.x1a, tile.y1a, tile.x2a, tile.y2a, tile.dx, tile.dy = x1a, y1a, x2a, y2a, dx, dy


def upload_table(table, dev):
    """A ctypes array of y5_aug_image -> device bytes (one copy from pinned memory)."""
    host = torch.frombuffer(bytearray(bytes(table)), dtype=torch.uint8).pin_memory()
    return host.to(dev, non_blocking=True), host


def aug_gather(table_dev, n, out_h, out_w, swap_rb=True, dtype=torch.uint8, device=None, out=None, s2d_out=None):
    """y5_aug_gather over a device table of n images -> (n, 3, out_h, out_w) `dtype` (or the stem's s2d buffer)."""
    lib = _lib.lib()
    simd_cols = out_w - out_w % 32  # cv2's HSV->BGR: 32-pixel SIMD blocks truncate, the row tail rounds
    with _lib.on(device):
        st = C.c_void_p(_lib.stream_ptr(device))
        if s2d_out is not None:
            buf, row_px, x_off = s2d_out
            _lib.check(lib.y5_aug_gather(table_dev.data_ptr(), n, out_h, out_w, simd_cols, int(swap_rb), buf.data_ptr(), _lib.dtype_code(buf.dtype), 1,
                                         row_px, x_off, st), "aug_gather")
            return buf
        res = out if out is not None else torch.empty(n, 3, out_h, out_w, dtype=dtype, device=device)
        if res.shape != (n, 3, out_h, out_w) or not res.is_contiguous():
            raise ValueError(f"y5b200: augmentation output must be a contiguous ({n}, 3, {out_h}, {out_w}) tensor")
        _lib.check(lib.y5_aug_gather(table_dev.data_ptr(), n, out_h, out_w, simd_cols, int(swap_rb), res.data_ptr(), _lib.dtype_code(res.dtype), 0, 0, 0,
                                     st), "aug_gather")
    return res


def aug_labels(table_dev, n_images, labels_dev, n_labels, out_h, out_w, device=None):
    """y5_aug_labels -> (padded (n_labels, 6) float32 rows, device int32 count of the kept rows)."""
    padded = torch.empty(max(n_labels, 1), 6, dtype=torch.float32, device=device)
    count = torch.empty(1, dtype=torch.int32, device=device)
    with _lib.on(device):
        _lib.check(_lib.lib().y5_aug_labels(table_dev.data_ptr(), n_images, labels_dev.data_ptr() if n_labels else None, n_labels, out_h, out_w,
                                            padded.data_ptr(), count.data_ptr(), C.c_void_p(_lib.stream_ptr(device))), "aug_labels")
    return padded, count


def _single_image_table(srcs, warps=None, r=None, luts=None):
    """A one-entry y5_aug_image whose mosaics are whole device images (HWC, canvas = the image)."""
    table = (_lib.AugImage * 1)()
    e = table[0]
    e.n_mosaic = len(srcs)
    e.canvas_h, e.canvas_w = srcs[0].shape[0], srcs[0].shape[1]
    for m, src in enumerate(srcs):
        e.n_tiles[m] = 1
        set_tile(e.tiles[4 * m], src, 0, 0, src.shape[1], src.shape[0], 0, 0)
        if warps is not None and warps[m] is not None:
            M, s = warps[m]
            e.warp[m] = 1
            e.inv_m[m][:] = invert_affine(M)
            e.m[m][:] = [float(v) for v in M[:2].reshape(6)]
            e.scale[m] = s
    if r is not None:
        e.mix_r = r
    if luts is not None:
        e.hsv = 1
        for k in range(3):
            e.lut[k][:] = luts[k].tolist()
    return table


def _hwc_result(chw, like_numpy):
    hwc = chw[0].permute(1, 2, 0).contiguous()
    return hwc.cpu().numpy() if like_numpy else hwc


def random_perspective(im, targets=(), segments=(), degrees=10, translate=0.1, scale=0.1, shear=10, perspective=0.0, border=(0, 0)):
    """Reference signature (utils/augmentations.py:118): warp a uint8 HWC BGR image with a random affine map and move its
    float32 (n, 5) [cls, x1, y1, x2, y2] pixel targets with it.  numpy in -> numpy out (the bytes cv2.warpAffine gives),
    CUDA tensor in -> CUDA tensor out.  perspective > 0 (warpPerspective) and segments are not implemented."""
    if perspective:
        raise NotImplementedError("y5b200: random_perspective with perspective > 0 (cv2.warpPerspective) is not implemented")
    if any(len(x) for x in segments):
        raise NotImplementedError("y5b200: random_perspective with segments is not implemented")
    is_np = isinstance(im, np.ndarray)
    if len(targets) and (getattr(targets, "dtype", None) not in (np.float32, torch.float32) or targets.ndim != 2 or targets.shape[1] != 5):
        raise ValueError("y5b200: random_perspective targets must be float32 (n, 5) [cls, x1, y1, x2, y2]")
    src = _as_device_hwc(im, None)
    dev = src.device
    draws = perspective_draws(degrees, translate, scale, shear, perspective)
    M = affine_matrix(draws, src.shape[:2], border)
    height, width = src.shape[0] + border[0] * 2, src.shape[1] + border[1] * 2
    if height <= 0 or width <= 0:
        raise ValueError("y5b200: random_perspective border leaves no output image")
    table = _single_image_table([src], [(M, draws[3])])
    table_dev, _ = upload_table(table, dev)
    if border[0] != 0 or border[1] != 0 or (M != np.eye(3)).any():
        im = _hwc_result(aug_gather(table_dev, 1, height, width, swap_rb=False, device=dev), is_np)
    if len(targets):
        t = torch.as_tensor(targets).to(dev, torch.float32)
        rec = torch.zeros(len(t), 12, dtype=torch.float32, device=dev)
        rec[:, :5] = t
        rec.view(torch.int32)[:, 11] = _lib.AUG_IN_XYXY | _lib.AUG_OUT_XYXY
        padded, count = aug_labels(table_dev, 1, rec, len(t), height, width, device=dev)
        out = padded[: int(count.item()), 1:]
        targets = out.cpu().numpy() if isinstance(targets, np.ndarray) else out
    src.record_stream(torch.cuda.current_stream(dev))
    return im, targets


def augment_hsv(im, hgain=0.5, sgain=0.5, vgain=0.5):
    """Reference signature (utils/augmentations.py:69): HSV gains on a uint8 HWC BGR image, IN PLACE (numpy array or CUDA
    tensor), with the bytes cv2's BGR2HSV -> LUT -> HSV2BGR give."""
    if hgain or sgain or vgain:
        r = np.random.uniform(-1, 1, 3) * [hgain, sgain, vgain] + 1
        src = _as_device_hwc(im, None)
        table_dev, _ = upload_table(_single_image_table([src], luts=hsv_luts(r)), src.device)
        res = aug_gather(table_dev, 1, src.shape[0], src.shape[1], swap_rb=False, device=src.device)[0].permute(1, 2, 0)
        if isinstance(im, np.ndarray):
            im[...] = res.cpu().numpy()
        else:
            im.copy_(res)


def mixup(im, labels, im2, labels2):
    """Reference signature (utils/augmentations.py:225): blend two same-size uint8 HWC images with r ~ Beta(32, 32) as
    trunc(im * r + im2 * (1 - r)) and concatenate their labels."""
    if tuple(im.shape) != tuple(im2.shape):
        raise ValueError(f"y5b200: mixup needs images of one shape, got {tuple(im.shape)} and {tuple(im2.shape)}")
    r = np.random.beta(32.0, 32.0)
    is_np = isinstance(im, np.ndarray)
    a, b = _as_device_hwc(im, None), _as_device_hwc(im2, None)
    table_dev, _ = upload_table(_single_image_table([a, b], r=r), a.device)
    out = _hwc_result(aug_gather(table_dev, 1, a.shape[0], a.shape[1], swap_rb=False, device=a.device), is_np)
    labels = np.concatenate((labels, labels2), 0) if isinstance(labels, np.ndarray) else torch.cat((labels, labels2), 0)
    return out, labels
