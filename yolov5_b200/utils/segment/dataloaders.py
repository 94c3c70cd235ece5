"""The segmentation training dataloader's augmentation on the device (reference utils/segment/dataloaders.py:130-301,
LoadImagesAndLabelsAndMasks.__getitem__ + collate_fn with augment=True, rect=False, copy_paste=0).

``DeviceSegAugmentLoader`` is a ``DeviceAugmentLoader`` that yields ``(imgs, targets, paths, shapes, masks)`` as
``collate_fn`` builds them, with ``imgs``, ``targets`` and ``masks`` on the device.  Per batch:
  1. host: every random draw in the reference's order (``draw_item``: the mixup partner is random.randint(0, n - 1)
     and the mosaic tiles keep their order),
     ``load_image``, and one pinned host-to-device copy of the sources, the image table, the label rows, the
     polygons' normalised points and the per-image label ranges;
  2. device: ``y5_aug_gather`` writes the images through the detection loader's code (the segmentation loader's image
     arithmetic is the same when copy_paste == 0); ``y5_seg_warp`` runs each label's segment through xyn2xy, the clip,
     resample_segments, the affine map, segment2box and box_candidates; ``y5_seg_raster`` rasterizes each kept polygon
     as cv2.fillPoly + cv2.resize do; ``y5_seg_order`` compacts the labels (in overlap mode in the order of
     np.argsort(-areas), equal areas in label order); ``y5_seg_compose`` writes the mask tensor.
The one host synchronisation is the read of the kept-label counts, which size ``targets`` and ``masks`` and decide the
masks' dtype (torch.cat's promotion: uint8, int32 for an overlap image with more than 255 labels, float32 as soon as one
image has no labels).  ``polygons2masks`` / ``polygons2masks_overlap`` expose the rasterizer with ultralytics'
signatures.  With num_workers=0 and the same seeds the batches equal the reference's (tests/test_seg_augment_gpu.py).

``DeviceSegValLoader`` is the segmentation validation loader (augment=False, rect batches): ``DeviceValLoader``'s
images and label rows, plus the polygon masks through the same rasterizer, order and compose kernels.
"""
from __future__ import annotations

import ctypes
import random

import numpy as np
import torch

from ... import _lib
from ..dataloaders import DeviceAugmentLoader, DeviceValLoader, ValBatchLayout, _check_augment, check_val_dataset, draw_item

_RATIOS = (1, 4)  # r = 2 is cv2.resize's INTER_AREA special case, not implemented


def _check_segments(ds):
    """One float32 (n >= 1, 2) segment of normalised points per label."""
    for k, (lab, segs) in enumerate(zip(ds.labels, ds.segments)):
        if len(lab) and len(segs) != len(lab):
            raise NotImplementedError(f"y5b200: image {k} has {len(lab)} labels and {len(segs)} segments (one segment per label is implemented)")
        for seg in segs:
            if not isinstance(seg, np.ndarray) or seg.dtype != np.float32 or seg.ndim != 2 or seg.shape[1] != 2 or len(seg) < 1:
                raise ValueError(f"y5b200: image {k}: segments must be float32 (n >= 1, 2) arrays of normalised points")


def _mixup_partner(ds):
    return lambda: random.randint(0, ds.n - 1)


class DeviceSegAugmentLoader(DeviceAugmentLoader):
    """Drop-in for utils/segment/dataloaders.py ``create_dataloader``'s loader over a ``LoadImagesAndLabelsAndMasks``-like
    dataset (duck-typed as ``DeviceAugmentLoader``'s, plus n, segments, overlap, downsample_ratio).  The index stream,
    sampler / DDP behaviour, the images and their output ``dtype`` are ``DeviceAugmentLoader``'s.  ``overlap`` and
    ``downsample_ratio`` default to the dataset's."""

    def __init__(self, dataset, batch_size, sampler=None, shuffle=False, device=None, dtype=torch.uint8, generator=None, drop_last=False,
                 overlap=None, downsample_ratio=None):
        self.overlap = bool(getattr(dataset, "overlap", False) if overlap is None else overlap)
        self.downsample_ratio = int(getattr(dataset, "downsample_ratio", 1) if downsample_ratio is None else downsample_ratio)
        super().__init__(dataset, batch_size, sampler=sampler, shuffle=shuffle, device=device, dtype=dtype, generator=generator, drop_last=drop_last)

    def _check_dataset(self, ds):
        """Refuse what the device path does not implement, before any draw or launch."""
        _check_augment(ds, "DeviceSegAugmentLoader")
        if ds.hyp.get("copy_paste", 0.0) > 0:
            raise NotImplementedError("y5b200: copy_paste > 0 is not implemented")
        r = self.downsample_ratio
        if r not in _RATIOS:
            raise NotImplementedError(f"y5b200: downsample_ratio {r} is not implemented (1 or 4)")
        s = int(ds.img_size)
        if s <= 0 or s > 4096:
            raise ValueError(f"y5b200: img_size {ds.img_size} outside (0, 4096]")
        if s % r:
            raise NotImplementedError(f"y5b200: img_size {s} is not a multiple of downsample_ratio {r}")
        _check_segments(ds)

    def _draw(self, i):
        return draw_item(self.dataset, i, _mixup_partner(self.dataset), shuffle_tiles=False)

    def _stage_labels(self, lay, labelled, n):
        """The label records, then each label's y5_aug_segment (point offset, point count), the segments' normalised points
        and the per-image label ranges -> (their four offsets, label count, longest segment)."""
        rec_off, n_rows = super()._stage_labels(lay, labelled, n)
        polys = [seg for _, k, _ in labelled for seg in self.dataset.segments[k]]
        seg = np.zeros((max(n_rows, 1), 2), np.int32)
        lens = np.array([len(x) for x in polys], np.int64)
        seg[:n_rows, 0] = np.cumsum(lens) - lens
        seg[:n_rows, 1] = lens
        pts = np.concatenate(polys, 0) if polys else np.zeros((1, 2), np.float32)
        image_rows = np.zeros(n + 1, np.int32)
        for b, _, rec in labelled:
            image_rows[b + 1:] += len(rec)
        offs = (rec_off, *(lay.add(a) for a in (seg, pts, image_rows)))
        return offs, n_rows, int(lens.max()) if n_rows else 1

    def collate(self, batch):
        """Augment dataset items `batch` (positions into dataset.indices) -> (imgs, targets, paths, shapes, masks)."""
        dev, s, r, n = self.device, int(self.dataset.img_size), self.downsample_ratio, len(batch)
        imgs, table_dev, dev_buf, (offs, n_rows, max_points), paths, shapes = self._augment(batch)
        lab_p, seg_p, pts_p, rows_p = (dev_buf.data_ptr() + off for off in offs)
        mh, mw = s // r, s // r
        nl = max(n_rows, 1)
        lib = _lib.lib()
        with _lib.on(dev):
            st = ctypes.c_void_p(_lib.stream_ptr(dev))
            verts = torch.empty(nl, _lib.SEG_POINTS, 2, dtype=torch.int32, device=dev)
            label_rows = torch.empty(nl, 6, dtype=torch.float32, device=dev)
            keep = torch.empty(nl, dtype=torch.int32, device=dev)
            raster = torch.empty(nl, mh, mw, dtype=torch.uint8, device=dev)
            areas = torch.empty(nl, dtype=torch.int32, device=dev)
            targets = torch.empty(nl, 6, dtype=torch.float32, device=dev)
            plane = torch.empty(nl, dtype=torch.int32, device=dev)
            counts = torch.empty(n + 1, dtype=torch.int32, device=dev)
            _lib.check(lib.y5_seg_warp(table_dev.data_ptr(), n, lab_p, seg_p, pts_p, max_points, n_rows, s, s, verts.data_ptr(),
                                       label_rows.data_ptr(), keep.data_ptr(), st), "seg_warp")
            _lib.check(lib.y5_seg_raster(verts.data_ptr(), _lib.SEG_POINTS, keep.data_ptr(), n_rows, s, s, r, raster.data_ptr(), areas.data_ptr(),
                                         st), "seg_raster")
            _lib.check(lib.y5_seg_order(rows_p, n, keep.data_ptr(), areas.data_ptr(), label_rows.data_ptr(), int(self.overlap), targets.data_ptr(),
                                        plane.data_ptr(), counts.data_ptr(), st), "seg_order")
            per_image = counts.cpu().tolist()  # the one host synchronisation
            nt = per_image[0]
            mdtype = _mask_dtype(per_image[1:], self.overlap)
            n_out = n if self.overlap else nt
            masks = torch.empty(n_out, mh, mw, dtype=mdtype, device=dev)
            _lib.check(lib.y5_seg_compose(table_dev.data_ptr(), lab_p, counts.data_ptr(), plane.data_ptr(), raster.data_ptr(), n_out, mh, mw,
                                          int(self.overlap), masks.data_ptr(), _MASK_CODE[mdtype], st), "seg_compose")
        return imgs, targets[:nt], paths, shapes, masks


_MASK_CODE = {torch.uint8: _lib.Y5_U8, torch.int32: _lib.SEG_I32, torch.float32: _lib.Y5_F32}


def _mask_dtype(kept_per_image, overlap):
    """torch.cat's dtype over the per-image masks: uint8 planes, an int32 overlap plane past 255 labels, float32 zeros for
    an image without labels."""
    dt = torch.uint8
    for k in kept_per_image:
        dt = torch.promote_types(dt, torch.float32 if k == 0 else (torch.int32 if overlap and k > 255 else torch.uint8))
    return dt


def _pad_polygons(polys):
    """Non-empty int32 (k, 2) polygons -> (max(n, 1), v, 2) int32 vertices for y5_seg_raster, v the longest polygon's
    count: shorter polygons repeat their last vertex (a zero-length edge draws nothing new)."""
    verts = np.zeros((max(len(polys), 1), max([len(p) for p in polys], default=1), 2), np.int32)
    for i, p in enumerate(polys):
        verts[i, :len(p)] = p
        verts[i, len(p):] = p[-1]
    return verts


def _rasterize(imgsz, polygons, downsample_ratio, device):
    """Host polygons -> (uint8 (n, h / r, w / r) masks, int32 areas, device) through y5_seg_raster."""
    h, w = int(imgsz[0]), int(imgsz[1])
    r = int(downsample_ratio)
    if r not in _RATIOS:
        raise NotImplementedError(f"y5b200: downsample_ratio {r} is not implemented (1 or 4)")
    if h % r or w % r:
        raise NotImplementedError(f"y5b200: image size {(h, w)} is not a multiple of downsample_ratio {r}")
    polys = [np.asarray(p, dtype=np.int32).reshape(-1, 2) for p in polygons]  # np.asarray(polygons, dtype=np.int32) as polygon2mask does
    if any(len(p) == 0 for p in polys):
        raise ValueError("y5b200: empty polygon")
    n = len(polys)
    verts = _pad_polygons(polys)
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    v = torch.from_numpy(verts).to(dev)
    keep = torch.ones(max(n, 1), dtype=torch.int32, device=dev)
    masks = torch.zeros(max(n, 1), h // r, w // r, dtype=torch.uint8, device=dev)
    areas = torch.zeros(max(n, 1), dtype=torch.int32, device=dev)
    with _lib.on(dev):
        _lib.check(_lib.lib().y5_seg_raster(v.data_ptr(), verts.shape[1], keep.data_ptr(), n, h, w, r, masks.data_ptr(), areas.data_ptr(),
                                            ctypes.c_void_p(_lib.stream_ptr(dev))), "seg_raster")
    return masks[:n], areas, dev


def polygons2masks(imgsz, polygons, color, downsample_ratio=1, device=None):
    """ultralytics.data.utils.polygons2masks on the device: (n, h / r, w / r) uint8, one plane per polygon, value `color`."""
    if color != 1 and downsample_ratio != 1:
        raise NotImplementedError("y5b200: polygons2masks with color != 1 is implemented at downsample_ratio 1 only")
    masks, _, _ = _rasterize(imgsz, polygons, downsample_ratio, device)
    return masks * np.uint8(color) if color != 1 else masks


def polygons2masks_overlap(imgsz, segments, downsample_ratio=1, device=None):
    """ultralytics.data.utils.polygons2masks_overlap on the device: (one (h / r, w / r) plane, uint8 up to 255 polygons,
    else int32, where polygon index[i] has value i + 1 where it is on top; index as a device int64 tensor).  Equal areas
    keep polygon order (np.argsort's order among them is not defined)."""
    masks, areas, dev = _rasterize(imgsz, segments, downsample_ratio, device)
    n = masks.shape[0]
    mh, mw = masks.shape[1:]
    mdtype = torch.int32 if n > 255 else torch.uint8
    out = torch.empty(1, mh, mw, dtype=mdtype, device=dev)
    table = (_lib.AugImage * 1)()
    host = torch.frombuffer(bytearray(bytes(table)), dtype=torch.uint8)
    table_dev = host.to(dev)
    image_rows = torch.tensor([0, n], dtype=torch.int32, device=dev)
    keep = torch.ones(max(n, 1), dtype=torch.int32, device=dev)
    rows = torch.zeros(max(n, 1), 6, dtype=torch.float32, device=dev)
    targets = torch.empty_like(rows)
    plane = torch.zeros(max(n, 1), dtype=torch.int32, device=dev)
    counts = torch.empty(2, dtype=torch.int32, device=dev)
    lib = _lib.lib()
    with _lib.on(dev):
        st = ctypes.c_void_p(_lib.stream_ptr(dev))
        _lib.check(lib.y5_seg_order(image_rows.data_ptr(), 1, keep.data_ptr(), areas.data_ptr(), rows.data_ptr(), 1, targets.data_ptr(),
                                    plane.data_ptr(), counts.data_ptr(), st), "seg_order")
        _lib.check(lib.y5_seg_compose(table_dev.data_ptr(), None, counts.data_ptr(), plane.data_ptr(), masks.data_ptr(), 1, mh, mw, 1,
                                      out.data_ptr(), _MASK_CODE[mdtype], st), "seg_compose")
    return out[0], plane[:n].long()


# ----------------------------------------------------------------------------------------------------------------------
# validation
# ----------------------------------------------------------------------------------------------------------------------
class DeviceSegValLoader(DeviceValLoader):
    """``DeviceValLoader`` for a ``LoadImagesAndLabelsAndMasks``-like dataset (plus segments, overlap, downsample_ratio):
    yields the segmentation collate_fn's ``(imgs, targets, paths, shapes, masks)`` with ``imgs``, ``targets`` and
    ``masks`` on the device.  Each segment goes through xyn2xy with the letterbox's ratio and pad (float32 on the host)
    and polygon2mask's int32 cast; ``y5_seg_raster`` rasterizes it at the batch shape (cv2.fillPoly + cv2.resize at
    ``downsample_ratio`` 1 or 4), ``y5_seg_order`` orders an overlap image's labels by decreasing area (equal areas in
    label order, as ``DeviceSegAugmentLoader`` does) and ``y5_seg_compose`` writes the masks.  Every label is kept, so
    the counts and the masks' dtype (``_mask_dtype``: uint8, int32 past 255 labels in overlap mode, float32 once an
    image has no labels) are known on the host: nothing waits for the device."""

    def __init__(self, dataset, batch_size, device=None, dtype=torch.uint8, workers=8, decode=None, overlap=None, downsample_ratio=None):
        self.overlap = bool(getattr(dataset, "overlap", False) if overlap is None else overlap)
        self.downsample_ratio = int(getattr(dataset, "downsample_ratio", 1) if downsample_ratio is None else downsample_ratio)
        if self.downsample_ratio not in _RATIOS:
            raise NotImplementedError(f"y5b200: downsample_ratio {self.downsample_ratio} is not implemented (1 or 4)")
        check_val_dataset(dataset, batch_size, "DeviceSegValLoader")
        _check_segments(dataset)
        super().__init__(dataset, batch_size, device=device, dtype=dtype, workers=workers, decode=decode)

    def collate(self, positions, loaded=None):
        """Batch of dataset positions -> (imgs, targets, paths, shapes, masks)."""
        ds, dev, r = self.dataset, self.device, self.downsample_ratio
        if loaded is None:
            loaded = [self.decode(ds, int(ds.indices[p])) for p in positions]
        lay = ValBatchLayout(ds, positions, loaded)
        H, W = lay.out_hw
        if H % r or W % r:
            raise NotImplementedError(f"y5b200: batch shape {(H, W)} is not a multiple of downsample_ratio {r}")
        if H > 4096 or W > 4096:
            raise NotImplementedError(f"y5b200: batch shape {(H, W)}: masks are implemented up to 4096 x 4096")
        rows, polys, image_rows = [], [], [0]
        for b, k in enumerate(lay.keys):
            lab = lay.label_rows(ds, b, W, H)
            if len(lab):
                it = lay.items[b]
                (h, w), ratio, pad = it["res"], it["ratio"], it["pad"]
                for seg in ds.segments[k]:
                    xy = np.copy(seg)  # xyn2xy: float32, the python-float scales and pads are weak scalars
                    xy[..., 0] = ratio[0] * w * seg[..., 0] + pad[0]
                    xy[..., 1] = ratio[1] * h * seg[..., 1] + pad[1]
                    polys.append(np.asarray(xy, dtype=np.int32).reshape(-1, 2))
                r6 = np.zeros((len(lab), 6), np.float32)
                r6[:, 0] = b
                r6[:, 1:] = lab
                rows.append(r6)
            image_rows.append(image_rows[-1] + len(lab))
        nl = image_rows[-1]
        per_image = [image_rows[b + 1] - image_rows[b] for b in range(lay.n)]
        verts = _pad_polygons(polys)
        lab6 = np.concatenate(rows, 0) if rows else np.zeros((1, 6), np.float32)
        rec = np.zeros((max(nl, 1), 12), np.float32)  # y5_aug_label records: y5_seg_compose reads their image index
        rec.view(np.int32)[:nl, 9] = lab6[:nl, 0].astype(np.int32)
        table = np.zeros((lay.n, ctypes.sizeof(_lib.AugImage)), np.uint8)  # no flips
        offs = [lay.add(a) for a in (verts, lab6, rec, table, np.asarray(image_rows, np.int32), np.ones(max(nl, 1), np.int32))]
        mh, mw = H // r, W // r
        mdtype = _mask_dtype(per_image, self.overlap)
        n_out = lay.n if self.overlap else nl
        lib = _lib.lib()
        with _lib.on(dev):
            st = ctypes.c_void_p(_lib.stream_ptr(dev))
            dev_buf = lay.upload(self._staging, dev)
            imgs = lay.letterbox(dev_buf, self.dtype, dev)
            verts_p, rows_p, rec_p, table_p, image_rows_p, keep_p = (dev_buf.data_ptr() + o for o in offs)
            raster = torch.empty(max(nl, 1), mh, mw, dtype=torch.uint8, device=dev)
            areas = torch.empty(max(nl, 1), dtype=torch.int32, device=dev)
            targets = torch.empty(max(nl, 1), 6, dtype=torch.float32, device=dev)
            plane = torch.empty(max(nl, 1), dtype=torch.int32, device=dev)
            counts = torch.empty(lay.n + 1, dtype=torch.int32, device=dev)
            masks = torch.empty(n_out, mh, mw, dtype=mdtype, device=dev)
            _lib.check(lib.y5_seg_raster(verts_p, verts.shape[1], keep_p, nl, H, W, r, raster.data_ptr(), areas.data_ptr(), st), "seg_raster")
            _lib.check(lib.y5_seg_order(image_rows_p, lay.n, keep_p, areas.data_ptr(), rows_p, int(self.overlap), targets.data_ptr(),
                                        plane.data_ptr(), counts.data_ptr(), st), "seg_order")
            _lib.check(lib.y5_seg_compose(table_p, rec_p, counts.data_ptr(), plane.data_ptr(), raster.data_ptr(), n_out, mh, mw,
                                          int(self.overlap), masks.data_ptr(), _MASK_CODE[mdtype], st), "seg_compose")
        return imgs, targets[:nl], tuple(ds.im_files[k] for k in lay.keys), tuple(lay.shapes), masks
