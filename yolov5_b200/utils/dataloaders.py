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
"""
from __future__ import annotations

import ctypes
import random

import numpy as np
import torch

from .. import _lib
from .augmentations import (affine_matrix, aug_gather, aug_labels, hsv_luts, invert_affine, letterbox_batch, letterbox_geometry,
                            perspective_draws, set_tile)

_ALIGN = 16


def _check_dataset(ds):
    """Refuse what the device path does not implement, before any draw or launch."""
    hyp = ds.hyp
    if getattr(ds, "rect", False) or not getattr(ds, "augment", True):
        raise NotImplementedError("y5b200: DeviceAugmentLoader implements augment=True, rect=False only")
    if hyp.get("perspective", 0.0) > 0:
        raise NotImplementedError("y5b200: perspective > 0 (cv2.warpPerspective) is not implemented")
    if any(len(s) for s in getattr(ds, "segments", ())):
        # segments change random_perspective's box path and make copy_paste active: segmentation datasets
        raise NotImplementedError("y5b200: datasets with segments (copy_paste, segment-derived boxes) are not implemented")
    alb = getattr(ds, "albumentations", None)
    if alb is not None and getattr(alb, "transform", None) is not None:
        raise NotImplementedError("y5b200: an active Albumentations transform is not implemented")
    if int(ds.img_size) <= 0 or int(ds.img_size) > 16384:
        raise ValueError(f"y5b200: img_size {ds.img_size} outside (0, 16384]")


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
        _check_dataset(dataset)
        if dtype not in (torch.uint8, torch.float16, torch.bfloat16, torch.float32):
            raise ValueError(f"y5b200: unsupported output dtype {dtype}")
        self.dataset = dataset
        self.batch_size = int(batch_size)
        self.dtype = dtype
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.index_loader = torch.utils.data.DataLoader(range(len(dataset.indices)), batch_size=self.batch_size, shuffle=shuffle and sampler is None,
                                                        sampler=sampler, generator=generator, drop_last=drop_last, collate_fn=list)
        self.sampler = sampler
        self._pinned = None
        self._copied = None  # event: the last staging upload has been read

    def __len__(self):
        return len(self.index_loader)

    def __iter__(self):
        for batch in self.index_loader:
            yield self.collate(batch)

    def _staging(self, nbytes):
        if self._copied is not None:
            self._copied.synchronize()  # the previous batch's copy still reads the pinned buffer
        if self._pinned is None or self._pinned.numel() < nbytes:
            self._pinned = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8).pin_memory()
        return self._pinned

    def collate(self, batch, sync=True):
        """Augment dataset items `batch` (positions into dataset.indices) -> (imgs, targets, paths, shapes); with
        sync=False targets is (padded (n, 6) rows, device int32 count) and nothing waits for the device."""
        ds, dev, s = self.dataset, self.device, int(self.dataset.img_size)
        params = [draw_item(ds, i) for i in batch]
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
        # staging layout: sources | table | label rows
        offs, pos = {}, 0
        for k in need:
            offs[k] = pos
            pos += (loaded[k][0].nbytes + _ALIGN - 1) // _ALIGN * _ALIGN
        n = len(params)
        table = (_lib.AugImage * n)()
        table_off = pos
        pos += ctypes.sizeof(table)
        rows, shapes, src_tiles = [], [], []
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
                            rows.append(_label_rows(lab, b, m, w, h, x1a - x1b, y1a - y1b, _lib.AUG_CLIP))
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
                    rows.append(_label_rows(lab, b, 0, ratio[0] * w, ratio[1] * h, pad[0], pad[1], 0))
            if p["hsv"] is not None:
                e.hsv = 1
                luts = hsv_luts(p["hsv"])
                for c in range(3):
                    e.lut[c][:] = luts[c].tolist()
            e.flipud, e.fliplr = int(p["flipud"]), int(p["fliplr"])
        rec = np.concatenate(rows, 0) if rows else np.zeros((0, 12), np.float32)
        n_labels = len(rec)
        total = pos + rec.nbytes
        dev_buf = torch.empty(total, dtype=torch.uint8, device=dev)
        for tile, off in src_tiles:
            tile.src = dev_buf.data_ptr() + off
        pinned = self._staging(total)
        host = pinned.numpy()
        for k in need:
            a = loaded[k][0]
            host[offs[k]: offs[k] + a.nbytes] = a.reshape(-1)
        host[table_off: table_off + ctypes.sizeof(table)] = np.frombuffer(bytes(table), np.uint8)
        host[pos: total] = rec.view(np.uint8).reshape(-1)
        with _lib.on(dev):
            stream = torch.cuda.current_stream(dev)
            dev_buf[:total].copy_(pinned[:total], non_blocking=True)
            self._copied = torch.cuda.Event()
            self._copied.record(stream)
            if lb_items:
                views = [dev_buf[offs[k]: offs[k] + loaded[k][0].nbytes].view(loaded[k][0].shape) for k in (params[b]["index"] for b in lb_items)]
                letterbox_batch(views, (s, s), auto=False, scaleup=True, swap_rb=False, device=dev, out=canvas)
            table_dev = dev_buf[table_off: table_off + ctypes.sizeof(table)]
            imgs = aug_gather(table_dev, n, s, s, swap_rb=True, dtype=self.dtype, device=dev)
            padded, count = aug_labels(table_dev, n, dev_buf[pos: total], n_labels, s, s, device=dev)
        paths = tuple(ds.im_files[p["index"]] for p in params)
        if not sync:
            return imgs, (padded, count), paths, tuple(shapes)
        nt = int(count.item())
        return imgs, padded[:nt], paths, tuple(shapes)

