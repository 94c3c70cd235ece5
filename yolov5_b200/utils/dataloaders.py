"""The detection training dataloader's augmentation on the device (reference utils/dataloaders.py:696-866,
LoadImagesAndLabels.__getitem__ + collate_fn with augment=True, rect=False).

``DeviceAugmentLoader`` iterates like ``create_dataloader``'s loader and yields ``(imgs, targets, paths, shapes)`` as
``collate_fn`` builds them, with ``imgs`` already on the device.  Per batch:
  1. host: every random number, drawn in the reference's order from Python's ``random`` and ``np.random`` (so the same
     seeds give the same batches), and the dataset's ``load_image`` (imread + resize, or its RAM cache);
  2. one host-to-device copy of a pinned staging buffer holding the batch's distinct source images, the per-image
     parameter table and the label rows;
  3. device: ``y5_aug_gather`` writes the finished batch (mosaic, affine warp, mixup, HSV, flips, CHW RGB) reading the
     placed tiles directly -- the 2s x 2s mosaic canvas is never built; images that take the non-mosaic branch are
     letterboxed first (``y5_letterbox``) into a scratch canvas; ``y5_aug_labels`` transforms, filters and compacts the
     labels.  The one host synchronisation is the read of the label count that sizes ``targets``.
With num_workers=0 and the same seeds the batches equal the reference's byte for byte (tests/test_augment_gpu.py).

``DeviceValLoader`` is the validation loader (``create_dataloader(..., augment=False, rect=True, pad=0.5)``, reference
utils/dataloaders.py:696-790): a pool of host threads decodes one batch ahead, and ``y5_val_letterbox`` does
load_image's resize (cv2 INTER_AREA / INTER_LINEAR) and the letterbox in one launch; see its docstring.

``DeviceClassifyLoader`` is ``create_classification_dataloader``'s loader (reference utils/dataloaders.py:949-1009,
without Albumentations): host threads decode one batch ahead, and ``y5_cls_batch`` does classify_transforms' center
crop, resize, ToTensor and Normalize in one launch; see its docstring.

Every loader lays out its host data with ``StagingLayout`` and uploads it with ``stage_upload``, one pinned
host-to-device copy per batch.  The segmentation loaders (utils/segment/dataloaders.py) subclass ``DeviceAugmentLoader``
and ``DeviceValLoader``.
"""
from __future__ import annotations

import ctypes
import math
import os
import random
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from .. import _lib
from .augmentations import (affine_matrix, aug_gather, aug_labels, hsv_luts, invert_affine, letterbox_batch, letterbox_geometry,
                            perspective_draws, set_tile)

_ALIGN = 16


def _aligned(nbytes):
    return (nbytes + _ALIGN - 1) // _ALIGN * _ALIGN


class StagingLayout:
    """Host arrays placed at _ALIGN-byte aligned offsets of one staging buffer: what one ``stage_upload`` copies."""

    def __init__(self):
        self.blocks = []  # (offset, array)
        self.size = 0

    def add(self, a):
        """Place host array `a` after the blocks so far -> its byte offset.  `a` may be a strided view; it is read when
        the layout is uploaded."""
        off = self.size
        self.blocks.append((off, a))
        self.size += _aligned(a.nbytes)
        return off


class _Staging:
    """`count` pinned staging buffers used in turn; a buffer is reused once the copy that last read it has run."""

    def __init__(self, count):
        self.buf = [None] * count
        self.done = [None] * count
        self.turn = 0

    def get(self, nbytes):
        k = self.turn
        self.turn = (k + 1) % len(self.buf)
        if self.done[k] is not None:
            self.done[k].synchronize()
        if self.buf[k] is None or self.buf[k].numel() < nbytes:
            self.buf[k] = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8).pin_memory()
        return k, self.buf[k]

    def mark(self, k, stream):
        self.done[k] = torch.cuda.Event()
        self.done[k].record(stream)


def stage_upload(staging, dev_buf, layout):
    """Write the blocks of `layout` (a StagingLayout) into a pinned buffer of `staging` and copy its first `layout.size`
    bytes to `dev_buf` on the current stream."""
    total = layout.size
    k, pinned = staging.get(total)
    host = pinned.numpy()
    for off, a in layout.blocks:
        np.copyto(host[off: off + a.nbytes].view(a.dtype).reshape(a.shape), a)
    dev_buf[:total].copy_(pinned[:total], non_blocking=True)
    staging.mark(k, torch.cuda.current_stream(dev_buf.device))


def _check_augment(ds, name):
    """The refusals both training loaders share, before any draw or launch."""
    hyp = ds.hyp
    if getattr(ds, "rect", False) or not getattr(ds, "augment", True):
        raise NotImplementedError(f"y5b200: {name} implements augment=True, rect=False only")
    if hyp.get("perspective", 0.0) > 0:
        raise NotImplementedError("y5b200: perspective > 0 (cv2.warpPerspective) is not implemented")
    alb = getattr(ds, "albumentations", None)
    if alb is not None and getattr(alb, "transform", None) is not None:
        raise NotImplementedError("y5b200: an active Albumentations transform is not implemented")


def _mosaic_draws(ds, index, shuffle_tiles=True):
    s = ds.img_size
    yc, xc = (int(random.uniform(-x, 2 * s + x)) for x in ds.mosaic_border)
    indices = [index, *random.choices(ds.indices, k=3)]
    if shuffle_tiles:
        random.shuffle(indices)
    hyp = ds.hyp
    return dict(xc=xc, yc=yc, indices=[int(i) for i in indices],
                persp=perspective_draws(hyp["degrees"], hyp["translate"], hyp["scale"], hyp["shear"], hyp["perspective"]))


def draw_item(ds, i, partner=None, shuffle_tiles=True):
    """Every random draw of __getitem__(i), in the reference's order (utils/dataloaders.py:696-756).  The segmentation
    loader (utils/segment/dataloaders.py:130-142, 235-243) differs in two draws: `partner()` draws the mixup partner's
    index (random.randint(0, n - 1) instead of random.choice(ds.indices)) and its mosaics keep the tile order
    (shuffle_tiles=False)."""
    hyp = ds.hyp
    p = dict(index=int(ds.indices[i]))
    p["mosaic"] = bool(ds.mosaic and random.random() < hyp["mosaic"])
    if p["mosaic"]:
        p["m"] = [_mosaic_draws(ds, p["index"], shuffle_tiles)]
        if random.random() < hyp["mixup"]:  # drawn even when mixup == 0
            p["m"].append(_mosaic_draws(ds, int(partner() if partner else random.choice(ds.indices)), shuffle_tiles))
            p["r"] = np.random.beta(32.0, 32.0)
    else:
        p["persp"] = perspective_draws(hyp["degrees"], hyp["translate"], hyp["scale"], hyp["shear"], hyp["perspective"])
    p["hsv"] = np.random.uniform(-1, 1, 3) * [hyp["hsv_h"], hyp["hsv_s"], hyp["hsv_v"]] + 1 if (hyp["hsv_h"] or hyp["hsv_s"] or hyp["hsv_v"]) else None
    p["flipud"] = random.random() < hyp["flipud"]
    p["fliplr"] = random.random() < hyp["fliplr"]
    return p


def _placements(xc, yc, s, hws):
    """load_mosaic's canvas rectangle and source offset (x1a, y1a, x2a, y2a, x1b, y1b) per tile."""
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


def _label_rows(labels, image, mosaic, tile_w, tile_h, pad_w, pad_h, flags):
    """y5_aug_label records (12 x 4 bytes) for a float32 (n, 5) label array."""
    rec = np.zeros((len(labels), 12), np.float32)
    rec[:, :5] = labels
    rec[:, 5:9] = np.array([tile_w, tile_h, pad_w, pad_h], np.float32)
    rec.view(np.int32)[:, 9:12] = (image, mosaic, flags)
    return rec


class DeviceAugmentLoader:
    """Drop-in for ``create_dataloader``'s loader over a ``LoadImagesAndLabels``-like dataset (duck-typed on
    indices, labels, segments, img_size, mosaic, mosaic_border, hyp, im_files, load_image, albumentations).  Batches are
    cut from ``torch.utils.data.DataLoader(range(len(dataset)), batch_size, shuffle, sampler, generator)`` -- the same
    index stream the reference's DataLoader draws -- and each batch is augmented on ``device``.  A sampler gives the
    per-rank shards under DDP.  ``dtype``: torch.uint8 (what collate_fn yields) or fp16/bf16/fp32 already divided by 255.
    """

    def __init__(self, dataset, batch_size, sampler=None, shuffle=False, device=None, dtype=torch.uint8, generator=None, drop_last=False):
        self._check_dataset(dataset)
        if dtype not in (torch.uint8, torch.float16, torch.bfloat16, torch.float32):
            raise ValueError(f"y5b200: unsupported output dtype {dtype}")
        self.dataset = dataset
        self.batch_size = int(batch_size)
        self.dtype = dtype
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.index_loader = torch.utils.data.DataLoader(range(len(dataset.indices)), batch_size=self.batch_size, shuffle=shuffle and sampler is None,
                                                        sampler=sampler, generator=generator, drop_last=drop_last, collate_fn=list)
        self.sampler = sampler
        self._staging = _Staging(1)  # a batch's upload waits for the previous batch's copy

    def __len__(self):
        return len(self.index_loader)

    def __iter__(self):
        for batch in self.index_loader:
            yield self.collate(batch)

    def _check_dataset(self, ds):
        """Refuse what the device path does not implement, before any draw or launch."""
        _check_augment(ds, "DeviceAugmentLoader")
        if any(len(s) for s in getattr(ds, "segments", ())):
            # segments change random_perspective's box path and make copy_paste active: segmentation datasets
            raise NotImplementedError("y5b200: datasets with segments (copy_paste, segment-derived boxes) are not implemented")
        if int(ds.img_size) <= 0 or int(ds.img_size) > 16384:
            raise ValueError(f"y5b200: img_size {ds.img_size} outside (0, 16384]")

    def _draw(self, i):
        return draw_item(self.dataset, i)

    def _stage_labels(self, lay, labelled, n):
        """Add the batch's label data to the staging layout -> (offset of the y5_aug_label records, their count).
        labelled: (image, dataset index, records) for each labelled tile, in table order; n: the batch size."""
        rec = np.concatenate([r for _, _, r in labelled], 0) if labelled else np.zeros((0, 12), np.float32)
        return lay.add(rec), len(rec)

    def _augment(self, batch):
        """Draw, load and stage dataset items `batch`, then letterbox the non-mosaic items and run y5_aug_gather ->
        (imgs, device image table, device staging buffer, what _stage_labels returned, paths, shapes)."""
        ds, dev, s = self.dataset, self.device, int(self.dataset.img_size)
        params = [self._draw(i) for i in batch]
        need = []
        for p in params:
            for k in ([i for m in p["m"] for i in m["indices"]] if p["mosaic"] else [p["index"]]):
                if k not in need:
                    need.append(k)
        loaded = {}
        for k in need:
            im, hw0, hw = ds.load_image(k)
            if not isinstance(im, np.ndarray) or im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3:
                raise ValueError(f"y5b200: load_image({k}) must return a uint8 HWC BGR image with 3 channels")
            if max(im.shape[:2]) > 2 * s or min(im.shape[:2]) < 1:
                raise ValueError(f"y5b200: load_image({k}) returned {im.shape[:2]}, outside [1, {2 * s}]")
            loaded[k] = (np.ascontiguousarray(im), hw0, hw)
        # staging layout: sources | table | label data
        lay = StagingLayout()
        offs = {k: lay.add(loaded[k][0]) for k in need}
        n = len(params)
        table = (_lib.AugImage * n)()
        labelled, shapes, src_tiles = [], [], []
        lb_items = [b for b, p in enumerate(params) if not p["mosaic"]]
        canvas = torch.empty(len(lb_items), 3, s, s, dtype=torch.uint8, device=dev) if lb_items else None
        for b, p in enumerate(params):
            e = table[b]
            if p["mosaic"]:
                e.n_mosaic = len(p["m"])
                e.canvas_w = e.canvas_h = 2 * s
                e.clip_max = 2 * s
                for m, md in enumerate(p["m"]):
                    srcs = [loaded[k] for k in md["indices"]]
                    M = affine_matrix(md["persp"], (2 * s, 2 * s), ds.mosaic_border)
                    e.warp[m] = 1
                    e.inv_m[m][:] = invert_affine(M)
                    e.m[m][:] = [float(v) for v in M[:2].reshape(6)]
                    e.scale[m] = md["persp"][3]
                    e.n_tiles[m] = 4
                    for t, ((x1a, y1a, x2a, y2a, x1b, y1b), k, (im, _, (h, w))) in enumerate(
                            zip(_placements(md["xc"], md["yc"], s, [x[2] for x in srcs]), md["indices"], srcs)):
                        tile = e.tiles[4 * m + t]
                        src_tiles.append((tile, offs[k]))  # device address patched in once the buffer exists
                        tile.row_bytes, tile.pixel_stride, tile.channel_stride = im.shape[1] * 3, 3, 1
                        tile.x1a, tile.y1a, tile.x2a, tile.y2a, tile.dx, tile.dy = x1a, y1a, x2a, y2a, x1b - x1a, y1b - y1a
                        lab = ds.labels[k]
                        if len(lab):
                            labelled.append((b, k, _label_rows(lab, b, m, w, h, x1a - x1b, y1a - y1b, _lib.AUG_CLIP)))
                if len(p["m"]) == 2:
                    e.mix_r = p["r"]
                shapes.append(None)
            else:
                k = p["index"]
                im, (h0, w0), (h, w) = loaded[k]
                _, ratio, pad, _ = letterbox_geometry(im.shape[:2], s, auto=False, scaleup=True)
                shapes.append(((h0, w0), ((h / h0, w / w0), pad)))
                M = affine_matrix(p["persp"], (s, s), (0, 0))
                e.n_mosaic = 1
                e.canvas_w = e.canvas_h = s
                e.warp[0] = int((M != np.eye(3)).any())
                e.inv_m[0][:] = invert_affine(M)
                e.m[0][:] = [float(v) for v in M[:2].reshape(6)]
                e.scale[0] = p["persp"][3]
                e.n_tiles[0] = 1
                set_tile(e.tiles[0], canvas[lb_items.index(b)], 0, 0, s, s, 0, 0)
                lab = ds.labels[k]
                if len(lab):
                    labelled.append((b, k, _label_rows(lab, b, 0, ratio[0] * w, ratio[1] * h, pad[0], pad[1], 0)))
            if p["hsv"] is not None:
                e.hsv = 1
                luts = hsv_luts(p["hsv"])
                for c in range(3):
                    e.lut[c][:] = luts[c].tolist()
            e.flipud, e.fliplr = int(p["flipud"]), int(p["fliplr"])
        table_off = lay.add(np.frombuffer(table, np.uint8))  # a view: the upload copies the table with the addresses below
        labels = self._stage_labels(lay, labelled, n)
        dev_buf = torch.empty(lay.size, dtype=torch.uint8, device=dev)
        for tile, off in src_tiles:
            tile.src = dev_buf.data_ptr() + off
        with _lib.on(dev):
            stage_upload(self._staging, dev_buf, lay)
            if lb_items:
                views = [dev_buf[offs[k]: offs[k] + loaded[k][0].nbytes].view(loaded[k][0].shape) for k in (params[b]["index"] for b in lb_items)]
                letterbox_batch(views, (s, s), auto=False, scaleup=True, swap_rb=False, device=dev, out=canvas)
            table_dev = dev_buf[table_off: table_off + ctypes.sizeof(table)]
            imgs = aug_gather(table_dev, n, s, s, swap_rb=True, dtype=self.dtype, device=dev)
        return imgs, table_dev, dev_buf, labels, tuple(ds.im_files[p["index"]] for p in params), tuple(shapes)

    def collate(self, batch, sync=True):
        """Augment dataset items `batch` (positions into dataset.indices) -> (imgs, targets, paths, shapes); with
        sync=False targets is (padded (n, 6) rows, device int32 count) and nothing waits for the device."""
        s = int(self.dataset.img_size)
        imgs, table_dev, dev_buf, (off, n_labels), paths, shapes = self._augment(batch)
        rec = dev_buf[off: off + n_labels * ctypes.sizeof(_lib.AugLabel)]
        padded, count = aug_labels(table_dev, len(batch), rec, n_labels, s, s, device=self.device)
        if not sync:
            return imgs, (padded, count), paths, shapes
        nt = int(count.item())
        return imgs, padded[:nt], paths, shapes


# ----------------------------------------------------------------------------------------------------------------------
# validation
# ----------------------------------------------------------------------------------------------------------------------
def load_val_image(ds, i):
    """The validation loader's decode step for dataset image i -> (uint8 HWC BGR image, (h0, w0), cached).  cached: the
    image is the RAM cache's ``ds.ims[i]``, already resized by load_image; otherwise it is the original image, from the
    ``.npy`` disk cache or ``cv2.imread``.  Runs on the loader's worker threads (cv2 and np.load release the GIL)."""
    ims = getattr(ds, "ims", None)
    if ims is not None and ims[i] is not None:
        return ims[i], tuple(int(v) for v in ds.im_hw0[i]), True
    npy = getattr(ds, "npy_files", None)
    if npy is not None and npy[i].exists():
        im = np.load(npy[i])
    else:
        import cv2

        im = cv2.imread(ds.im_files[i])
        if im is None:
            raise FileNotFoundError(f"Image Not Found {ds.im_files[i]}")
    return im, tuple(int(v) for v in im.shape[:2]), False


def check_val_dataset(ds, batch_size, name="DeviceValLoader"):
    """Refuse what the validation path does not implement, before any work."""
    if getattr(ds, "augment", False):
        raise NotImplementedError(f"y5b200: {name} implements augment=False only (use the augment loaders for training batches)")
    if getattr(ds, "image_weights", False):
        raise NotImplementedError(f"y5b200: {name}: image_weights is not implemented")
    s = int(ds.img_size)
    if s <= 0 or s > 16384:
        raise ValueError(f"y5b200: img_size {ds.img_size} outside (0, 16384]")
    if getattr(ds, "rect", False):
        n = len(ds.batch)
        if not np.array_equal(np.asarray(ds.batch), np.arange(n) // int(batch_size)):
            raise ValueError(f"y5b200: batch_size {batch_size} disagrees with the dataset's rect batches (built for another batch size)")


def val_geometry(ds, k, hw0, cached, im_hw):
    """(load_image size (h, w), interp, batch shape (H, W), letterbox geometry) of dataset image k."""
    s = int(ds.img_size)
    if cached:
        (h, w), interp = im_hw, _lib.VAL_COPY
    else:
        h0, w0 = hw0
        r = s / max(h0, w0)
        if r == 1:
            (h, w), interp = (h0, w0), _lib.VAL_COPY
        else:
            (h, w), interp = (math.ceil(h0 * r), math.ceil(w0 * r)), (_lib.VAL_LINEAR if r > 1 else _lib.VAL_AREA)
    # the batch_shapes row as __getitem__ passes it: its numpy integers make letterbox's ratio and pads np.float64, which
    # NumPy does not treat as weak scalars, so the label maths below round as the reference's do
    shape = ds.batch_shapes[ds.batch[k]] if getattr(ds, "rect", False) else s
    new_unpad, ratio, pad, (top, bottom, left, right) = letterbox_geometry((h, w), shape, auto=False, scaleup=False)
    hw = (int(shape[0]), int(shape[1])) if getattr(ds, "rect", False) else (s, s)
    return (h, w), interp, hw, ((int(new_unpad[0]), int(new_unpad[1])), ratio, pad, (int(top), int(bottom), int(left), int(right)))


def val_label_rows(labels, ratio, w, h, pad, out_w, out_h):
    """__getitem__'s label path (augment=False): xywhn2xyxy(ratio * w, ratio * h, pad) then xyxy2xywhn(clip=True,
    eps=1e-3), in float32 as NumPy computes it from the float32 labels -> (n, 5) float32 [cls, xywhn]."""
    lab = np.array(labels, dtype=np.float32, copy=True).reshape(-1, 5)
    if not lab.size:
        return lab
    x = lab[:, 1:]
    y = np.copy(x)
    sw, sh = ratio[0] * w, ratio[1] * h
    y[..., 0] = sw * (x[..., 0] - x[..., 2] / 2) + pad[0]
    y[..., 1] = sh * (x[..., 1] - x[..., 3] / 2) + pad[1]
    y[..., 2] = sw * (x[..., 0] + x[..., 2] / 2) + pad[0]
    y[..., 3] = sh * (x[..., 1] + x[..., 3] / 2) + pad[1]
    lab[:, 1:] = y
    b = lab[:, 1:5]
    b[..., [0, 2]] = b[..., [0, 2]].clip(0, out_w - 1e-3)
    b[..., [1, 3]] = b[..., [1, 3]].clip(0, out_h - 1e-3)
    y = np.copy(b)
    y[..., 0] = ((b[..., 0] + b[..., 2]) / 2) / out_w
    y[..., 1] = ((b[..., 1] + b[..., 3]) / 2) / out_h
    y[..., 2] = (b[..., 2] - b[..., 0]) / out_w
    y[..., 3] = (b[..., 3] - b[..., 1]) / out_h
    lab[:, 1:5] = y
    return lab


def decode_ahead(ds, batches, decode, workers):
    """(batch, decoded items) for each batch of the iterable `batches`, with `workers` threads running decode(ds, i) for
    every i of the next batch while the caller works on the current one."""
    it = iter(batches)
    b = next(it, None)
    if b is None:
        return
    with ThreadPoolExecutor(max_workers=workers) as pool:
        def submit(b):
            return [pool.submit(decode, ds, i) for i in b]

        ahead = submit(b)
        while b is not None:
            loaded = [f.result() for f in ahead]
            nxt = next(it, None)
            if nxt is not None:
                ahead = submit(nxt)
            yield b, loaded
            b = nxt


class ValBatchLayout(StagingLayout):
    """Host side of one validation batch: decoded images, geometry, shapes and label rows, laid out in one staging
    buffer as [sources | blocks added later], plus the device scratch the letterboxes that resize again need."""

    def __init__(self, ds, positions, loaded):
        super().__init__()
        self.keys = [int(ds.indices[p]) for p in positions]
        self.n = len(positions)
        self.items, self.shapes, self.offs = [], [], []
        scratch = 0
        batch_shape = None
        for b, (k, (im, hw0, cached)) in enumerate(zip(self.keys, loaded)):
            if not isinstance(im, np.ndarray) or im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3:
                raise ValueError(f"y5b200: image {k} must be a uint8 HWC BGR image with 3 channels")
            if min(im.shape[:2]) < 1:
                raise ValueError(f"y5b200: image {k} is empty")
            im = np.ascontiguousarray(im)
            (h, w), interp, shape, (new_unpad, ratio, pad, (top, _, left, _)) = val_geometry(ds, k, hw0, cached, im.shape[:2])
            if batch_shape is None:
                batch_shape = shape
            elif shape != batch_shape:
                raise ValueError(f"y5b200: image {k} has batch shape {shape}, the batch {batch_shape}")
            again = tuple(new_unpad) != (w, h)
            self.items.append(dict(im=im, res=(h, w), interp=interp, new=(new_unpad[1], new_unpad[0]), top=top, left=left,
                                   scratch=scratch if again else None, ratio=ratio, pad=pad))
            if again:
                scratch += _aligned(h * w * 3)
            self.shapes.append(((int(hw0[0]), int(hw0[1])), ((h / hw0[0], w / hw0[1]), pad)))
            self.offs.append(self.add(im))
        self.out_hw = batch_shape
        self.scratch_bytes = scratch

    def label_rows(self, ds, b, out_w, out_h):
        it = self.items[b]
        return val_label_rows(ds.labels[self.keys[b]], it["ratio"], it["res"][1], it["res"][0], it["pad"], out_w, out_h)

    def upload(self, staging, dev):
        """One pinned host-to-device copy of the sources and blocks -> the device buffer, the scratch after them."""
        dev_buf = torch.empty(self.size + self.scratch_bytes, dtype=torch.uint8, device=dev)
        stage_upload(staging, dev_buf, self)
        return dev_buf

    def letterbox(self, dev_buf, dtype, dev):
        """y5_val_letterbox over the uploaded sources -> (n, 3, H, W) `dtype`."""
        H, W = self.out_hw
        table = (_lib.ValImage * self.n)()
        base = dev_buf.data_ptr()
        for d, off, it in zip(table, self.offs, self.items):
            im = it["im"]
            d.data, d.src_h, d.src_w, d.row_bytes = base + off, im.shape[0], im.shape[1], im.shape[1] * 3
            d.res_h, d.res_w = it["res"]
            d.interp = it["interp"]
            d.new_h, d.new_w = it["new"]
            d.top, d.left = it["top"], it["left"]
            d.scratch = base + self.size + it["scratch"] if it["scratch"] is not None else None
        imgs = torch.empty(self.n, 3, H, W, dtype=dtype, device=dev)
        _lib.check(_lib.lib().y5_val_letterbox(table, self.n, H, W, imgs.data_ptr(), _lib.dtype_code(dtype),
                                               ctypes.c_void_p(_lib.stream_ptr(dev))), "val_letterbox")
        return imgs


class DeviceValLoader:
    """Drop-in for the validation ``create_dataloader(..., augment=False)`` loader over a ``LoadImagesAndLabels``-like
    dataset (duck-typed on indices, labels, img_size, rect, batch, batch_shapes, im_files, ims, im_hw0, npy_files).
    Yields collate_fn's ``(imgs, targets, paths, shapes)`` in dataset order with ``imgs`` and ``targets`` on ``device``;
    ``dtype``: torch.uint8 (what collate_fn yields) or fp16/bf16/fp32 as ``imgs.to(dtype) / 255`` computes them.
    Per batch:
      1. ``workers`` host threads run ``decode`` (default ``load_val_image``: the RAM cache, the .npy cache or
         cv2.imread) one batch ahead of the consumer;
      2. the host works out load_image's size and interpolation, letterbox's geometry, ``shapes`` and the label rows
         (float32, as the reference computes them), and makes one pinned host-to-device copy of the sources and rows;
      3. ``y5_val_letterbox`` resizes (INTER_AREA when shrinking, INTER_LINEAR when enlarging) and letterboxes every
         image in one launch.
    Nothing waits for the device.  The batches equal the reference's byte for byte (tests/test_val_load_gpu.py)."""

    def __init__(self, dataset, batch_size, device=None, dtype=torch.uint8, workers=8, decode=None):
        check_val_dataset(dataset, batch_size)
        if dtype not in (torch.uint8, torch.float16, torch.bfloat16, torch.float32):
            raise ValueError(f"y5b200: unsupported output dtype {dtype}")
        self.dataset = dataset
        self.batch_size = int(batch_size)
        self.dtype = dtype
        self.workers = max(1, int(workers))
        self.decode = decode or load_val_image
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self._staging = _Staging(2)  # the next batch is staged while the previous copy may still run

    def __len__(self):
        return (len(self.dataset.indices) + self.batch_size - 1) // self.batch_size

    def _batches(self):
        n = len(self.dataset.indices)
        return [list(range(i, min(i + self.batch_size, n))) for i in range(0, n, self.batch_size)]

    def __iter__(self):
        for b, loaded in decode_ahead(self.dataset, self._batches(), lambda ds, p: self.decode(ds, int(ds.indices[p])), self.workers):
            yield self.collate(b, loaded)

    def collate(self, positions, loaded=None):
        """Batch of dataset positions (into dataset.indices) -> (imgs, targets, paths, shapes).  `loaded`: the decode
        results, decoded here when None."""
        ds, dev = self.dataset, self.device
        if loaded is None:
            loaded = [self.decode(ds, int(ds.indices[p])) for p in positions]
        lay = ValBatchLayout(ds, positions, loaded)
        H, W = lay.out_hw
        rows = [lay.label_rows(ds, b, W, H) for b in range(lay.n)]
        nt = sum(len(r) for r in rows)
        tg = np.zeros((nt, 6), np.float32)
        i = 0
        for b, r in enumerate(rows):
            tg[i: i + len(r), 0] = b
            tg[i: i + len(r), 1:] = r
            i += len(r)
        t_off = lay.add(tg)
        with _lib.on(dev):
            dev_buf = lay.upload(self._staging, dev)
            imgs = lay.letterbox(dev_buf, self.dtype, dev)
        targets = dev_buf[t_off: t_off + tg.nbytes].view(torch.float32).view(nt, 6)
        return imgs, targets, tuple(ds.im_files[k] for k in lay.keys), tuple(lay.shapes)


# ----------------------------------------------------------------------------------------------------------------------
# classification
# ----------------------------------------------------------------------------------------------------------------------
IMAGENET_MEAN = 0.485, 0.456, 0.406  # RGB, as utils/augmentations.py defines them
IMAGENET_STD = 0.229, 0.224, 0.225


def load_cls_image(ds, i):
    """The classification loader's decode step for dataset item i -> uint8 HWC BGR image, with
    ClassificationDataset.__getitem__'s caches: the RAM cache keeps cv2.imread's result in ``samples[i][3]``, the disk
    cache writes ``samples[i][2]`` (.npy) on first use and reads it with np.load.  A RAM-cached image is used as it is
    (the reference's __getitem__ reads the file again once its cache is filled; the bytes are the same).  Runs on the
    loader's worker threads."""
    import cv2

    f, _, fn, im = ds.samples[i]
    if ds.cache_ram and im is not None:
        return im
    if ds.cache_disk and fn.exists():
        return np.load(fn)
    im = cv2.imread(str(f))
    if im is None:
        raise FileNotFoundError(f"Image Not Found {f}")
    if ds.cache_ram:
        ds.samples[i][3] = im
    elif ds.cache_disk:  # written under a private name first: a padded DistributedSampler batch can hold an item twice
        tmp = f"{fn.as_posix()}.{os.getpid()}.{threading.get_ident()}.npy"
        np.save(tmp, im)
        os.replace(tmp, fn)
    return im


# Where classify_transforms' CenterCrop and ToTensor may come from: the reference's utils/augmentations.py (also when it is
# imported as part of a package, e.g. yolov5.utils.augmentations), or the call-compatible numpy stand-ins of the test oracle
_CLS_TRANSFORM_MODULES = ("utils.augmentations", "oracle.cls_load_ref")


def _from_module(t, modules):
    m = type(t).__module__
    return any(m == x or m.endswith("." + x) for x in modules)


def check_cls_dataset(ds):
    """Refuse what the classification path does not implement, before any work -> the output size (h, w).
    torch_transforms must be classify_transforms' Compose([CenterCrop, ToTensor(half=False), Normalize(ImageNet)]): the
    reference's CenterCrop and ToTensor classes (checked by class and module) and torchvision's Normalize."""
    if getattr(ds, "album_transforms", None):  # __getitem__ takes this branch whenever the transform is truthy
        raise NotImplementedError("y5b200: DeviceClassifyLoader: an active Albumentations transform is not implemented")
    ts = list(getattr(getattr(ds, "torch_transforms", None), "transforms", None) or ())
    names = [f"{type(t).__module__}.{type(t).__name__}" for t in ts]
    if ([type(t).__name__ for t in ts] != ["CenterCrop", "ToTensor", "Normalize"] or not all(_from_module(t, _CLS_TRANSFORM_MODULES) for t in ts[:2])
            or not _from_module(ts[2], ("torchvision.transforms.transforms",)) or not all(hasattr(ts[0], a) for a in ("h", "w"))):
        raise NotImplementedError(f"y5b200: DeviceClassifyLoader implements classify_transforms (CenterCrop, ToTensor, Normalize) only, got {names}")
    if getattr(ts[1], "half", None) is not False:
        raise NotImplementedError("y5b200: DeviceClassifyLoader implements ToTensor(half=False) only")
    mean, std = (tuple(float(v) for v in getattr(ts[2], a)) for a in ("mean", "std"))
    if mean != IMAGENET_MEAN or std != IMAGENET_STD:
        raise NotImplementedError(f"y5b200: DeviceClassifyLoader implements Normalize(IMAGENET_MEAN, IMAGENET_STD) only, got {mean}, {std}")
    h, w = ts[0].h, ts[0].w
    if not all(isinstance(v, (int, np.integer)) and 0 < v <= 16384 for v in (h, w)):
        raise ValueError(f"y5b200: image size {(h, w)} outside (0, 16384]")
    return int(h), int(w)


class DeviceClassifyLoader:
    """Drop-in for ``create_classification_dataloader``'s loader (reference utils/dataloaders.py:988-1009) over a
    ``ClassificationDataset``-like dataset (duck-typed on samples, root, classes, torch_transforms, album_transforms,
    cache_ram, cache_disk).  Yields ``(images (B, 3, h, w) dtype, labels (B,) int64)``, both on ``device``; ``dtype``
    torch.float32 is what the reference yields, fp16 / bf16 that value rounded once (``images.half()``).

    The batches are the reference's: the same ``min(batch_size, len(dataset))``, the same generator seed
    (6148914691236517205 + RANK), shuffling or a ``DistributedSampler(dataset, shuffle=shuffle)`` when ``rank != -1``, and
    one persistent index stream, as InfiniteDataLoader keeps it: each pass yields the next ``len(self)`` batches of
    the stream, so ``next(iter(loader))`` advances it.  A pass draws its batches as it yields them (plus the one batch
    being decoded ahead), so under DDP an epoch's DistributedSampler permutation is taken after classify/train.py's
    ``set_epoch``.  The reference matches that with num_workers=0; with workers, its InfiniteDataLoader prefetches
    ``prefetch_factor * num_workers`` batches and can take the next epoch's permutation before ``set_epoch`` runs, so its
    later DDP epochs depend on its worker count.  Per batch:
      1. ``workers`` host threads run ``decode`` (default ``load_cls_image``: the caches or cv2.imread) one batch ahead;
      2. the host stages each image's center m x m square (m = min(h, w)), the y5_cls_image table and the labels in one
         pinned buffer and makes one host-to-device copy;
      3. ``y5_cls_batch`` resizes (cv2 INTER_LINEAR), converts and normalises the whole batch in one launch.
    Nothing waits for the device.  The batches equal the reference's bit for bit (tests/test_cls_load_gpu.py)."""

    def __init__(self, dataset, batch_size, rank=-1, shuffle=True, device=None, dtype=torch.float32, workers=8, decode=None):
        self.size = check_cls_dataset(dataset)
        if dtype not in (torch.float16, torch.bfloat16, torch.float32):
            raise ValueError(f"y5b200: unsupported output dtype {dtype}")
        self.dataset = dataset
        n = len(dataset.samples)
        self.batch_size = min(int(batch_size), n)
        self.dtype = dtype
        self.workers = max(1, int(workers))
        self.decode = decode or load_cls_image
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.sampler = None if rank == -1 else torch.utils.data.DistributedSampler(dataset, shuffle=shuffle)
        generator = torch.Generator()
        generator.manual_seed(6148914691236517205 + int(os.getenv("RANK", "-1")))
        index = torch.utils.data.DataLoader(range(n), batch_size=self.batch_size, shuffle=shuffle and self.sampler is None, sampler=self.sampler,
                                            generator=generator, collate_fn=list)
        self._batch_sampler = index.batch_sampler
        object.__setattr__(index, "batch_sampler", _Repeat(index.batch_sampler))  # DataLoader refuses a plain assignment
        self._stream = iter(index)  # created once: the iterator's base seed is drawn from the generator here, as the reference's is
        self._carry = None  # a batch drawn from the stream but not yielded (a pass left early)
        self._staging = _Staging(2)  # the next batch is staged while the previous copy may still run
        self._mean = (ctypes.c_float * 3)(*IMAGENET_MEAN)
        self._std = (ctypes.c_float * 3)(*IMAGENET_STD)

    def __len__(self):
        return len(self._batch_sampler)

    def _draw(self):
        for j in range(len(self)):
            if j > 0 or self._carry is None:
                self._carry = next(self._stream)
            yield self._carry

    def __iter__(self):
        for b, loaded in decode_ahead(self.dataset, self._draw(), self.decode, self.workers):
            if self._carry is b:  # nothing drawn ahead of this batch
                self._carry = None
            yield self.collate(b, loaded)

    def collate(self, items, loaded=None):
        """Dataset items -> (images, labels) on the device.  `loaded`: the decode results, decoded here when None."""
        ds, dev = self.dataset, self.device
        if loaded is None:
            loaded = [self.decode(ds, i) for i in items]
        n = len(items)
        lay = StagingLayout()
        offs, sides = [], []
        for i, im in zip(items, loaded):
            if not isinstance(im, np.ndarray) or im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3:
                raise ValueError(f"y5b200: image {i} must be a uint8 HWC BGR image with 3 channels")
            h, w = im.shape[:2]
            m = min(h, w)
            if m < 1:
                raise ValueError(f"y5b200: image {i} is empty")
            top, left = (h - m) // 2, (w - m) // 2
            offs.append(lay.add(im[top: top + m, left: left + m]))
            sides.append(m)
        table = (_lib.ClsImage * n)()
        table_off = lay.add(np.frombuffer(table, np.uint8))  # a view: the upload copies the table with the addresses below
        labels = np.array([ds.samples[i][1] for i in items], np.int64)
        label_off = lay.add(labels)
        with _lib.on(dev):
            dev_buf = torch.empty(lay.size, dtype=torch.uint8, device=dev)
            base = dev_buf.data_ptr()
            for d, off, m in zip(table, offs, sides):
                d.data, d.side, d.row_bytes = base + off, m, 3 * m
            stage_upload(self._staging, dev_buf, lay)
            h, w = self.size
            images = torch.empty(n, 3, h, w, dtype=self.dtype, device=dev)
            _lib.check(_lib.lib().y5_cls_batch(base + table_off, n, h, w, self._mean, self._std, images.data_ptr(), _lib.dtype_code(self.dtype),
                                               ctypes.c_void_p(_lib.stream_ptr(dev))), "cls_batch")
        return images, dev_buf[label_off: label_off + labels.nbytes].view(torch.int64)


class _Repeat:
    """A batch sampler that starts over whenever it runs out, so one DataLoader iterator is an endless stream."""

    def __init__(self, batch_sampler):
        self.sampler = batch_sampler

    def __iter__(self):
        while True:
            yield from iter(self.sampler)
