"""The segmentation training dataloader's augmentation on the device (reference utils/segment/dataloaders.py:130-301,
LoadImagesAndLabelsAndMasks.__getitem__ + collate_fn with augment=True, rect=False, copy_paste=0).

``DeviceSegAugmentLoader`` yields ``(imgs, targets, paths, shapes, masks)`` as ``collate_fn`` builds them, with
``imgs``, ``targets`` and ``masks`` on the device.  Per batch:
  1. host: every random draw in the reference's order (``draw_item``: the mixup partner is random.randint(0, n - 1)
     and the mosaic tiles keep their order),
     ``load_image``, and one pinned host-to-device copy of the sources, the image table, the label rows, the
     polygons' normalised points and the per-image label ranges;
  2. device: ``y5_aug_gather`` writes the images exactly as the detection loader does (the segmentation loader's image
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
from ..augmentations import affine_matrix, aug_gather, hsv_luts, invert_affine, letterbox_batch, letterbox_geometry, set_tile
from ..dataloaders import _ALIGN, DeviceValLoader, ValBatchLayout, _label_rows, _placements, check_val_dataset, draw_item

_RATIOS = (1, 4)  # r = 2 is cv2.resize's INTER_AREA special case, not implemented


def _check_dataset(ds, overlap, downsample_ratio):
    """Refuse what the device path does not implement, before any draw or launch."""
    hyp = ds.hyp
    if getattr(ds, "rect", False) or not getattr(ds, "augment", True):
        raise NotImplementedError("y5b200: DeviceSegAugmentLoader implements augment=True, rect=False only")
    if hyp.get("perspective", 0.0) > 0:
        raise NotImplementedError("y5b200: perspective > 0 (cv2.warpPerspective) is not implemented")
    if hyp.get("copy_paste", 0.0) > 0:
        raise NotImplementedError("y5b200: copy_paste > 0 is not implemented")
    alb = getattr(ds, "albumentations", None)
    if alb is not None and getattr(alb, "transform", None) is not None:
        raise NotImplementedError("y5b200: an active Albumentations transform is not implemented")
    if downsample_ratio not in _RATIOS:
        raise NotImplementedError(f"y5b200: downsample_ratio {downsample_ratio} is not implemented (1 or 4)")
    s = int(ds.img_size)
    if s <= 0 or s > 4096:
        raise ValueError(f"y5b200: img_size {ds.img_size} outside (0, 4096]")
    if s % downsample_ratio:
        raise NotImplementedError(f"y5b200: img_size {s} is not a multiple of downsample_ratio {downsample_ratio}")
    for k, (lab, segs) in enumerate(zip(ds.labels, ds.segments)):
        if len(lab) and len(segs) != len(lab):
            raise NotImplementedError(f"y5b200: image {k} has {len(lab)} labels and {len(segs)} segments (one segment per label is implemented)")
        for seg in segs:
            if not isinstance(seg, np.ndarray) or seg.dtype != np.float32 or seg.ndim != 2 or seg.shape[1] != 2 or len(seg) < 1:
                raise ValueError(f"y5b200: image {k}: segments must be float32 (n >= 1, 2) arrays of normalised points")


def _mixup_partner(ds):
    return lambda: random.randint(0, ds.n - 1)


class DeviceSegAugmentLoader:
    """Drop-in for utils/segment/dataloaders.py ``create_dataloader``'s loader over a ``LoadImagesAndLabelsAndMasks``-like
    dataset (duck-typed as ``DeviceAugmentLoader``'s, plus n, segments, overlap, downsample_ratio).  The index stream,
    sampler / DDP behaviour and output ``dtype`` of the images are ``DeviceAugmentLoader``'s.  ``overlap`` and
    ``downsample_ratio`` default to the dataset's."""

    def __init__(self, dataset, batch_size, sampler=None, shuffle=False, device=None, dtype=torch.uint8, generator=None, drop_last=False,
                 overlap=None, downsample_ratio=None):
        self.overlap = bool(getattr(dataset, "overlap", False) if overlap is None else overlap)
        self.downsample_ratio = int(getattr(dataset, "downsample_ratio", 1) if downsample_ratio is None else downsample_ratio)
        _check_dataset(dataset, self.overlap, self.downsample_ratio)
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

    def collate(self, batch):
        """Augment dataset items `batch` (positions into dataset.indices) -> (imgs, targets, paths, shapes, masks)."""
        ds, dev, s, r = self.dataset, self.device, int(self.dataset.img_size), self.downsample_ratio
        partner = _mixup_partner(ds)
        params = [draw_item(ds, i, partner, shuffle_tiles=False) for i in batch]
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
        offs, pos = {}, 0
        for k in need:
            offs[k] = pos
            pos += (loaded[k][0].nbytes + _ALIGN - 1) // _ALIGN * _ALIGN
        n = len(params)
        table = (_lib.AugImage * n)()
        table_off = pos
        pos += ctypes.sizeof(table)
        rows, polys, image_rows, shapes, src_tiles = [], [], [0], [], []
        n_rows = 0

        def add_labels(k, b, m, tw, th, pw, ph, flags):
            nonlocal n_rows
            lab = ds.labels[k]
            if len(lab):
                rows.append(_label_rows(lab, b, m, tw, th, pw, ph, flags))
                polys.extend(ds.segments[k])
                n_rows += len(lab)

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
                        src_tiles.append((tile, offs[k]))
                        tile.row_bytes, tile.pixel_stride, tile.channel_stride = im.shape[1] * 3, 3, 1
                        tile.x1a, tile.y1a, tile.x2a, tile.y2a, tile.dx, tile.dy = x1a, y1a, x2a, y2a, x1b - x1a, y1b - y1a
                        add_labels(k, b, m, w, h, x1a - x1b, y1a - y1b, _lib.AUG_CLIP)
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
                add_labels(k, b, 0, ratio[0] * w, ratio[1] * h, pad[0], pad[1], 0)
            if p["hsv"] is not None:
                e.hsv = 1
                luts = hsv_luts(p["hsv"])
                for c in range(3):
                    e.lut[c][:] = luts[c].tolist()
            e.flipud, e.fliplr = int(p["flipud"]), int(p["fliplr"])
            image_rows.append(n_rows)
        rec = np.concatenate(rows, 0) if rows else np.zeros((0, 12), np.float32)
        seg = np.zeros((max(n_rows, 1), 2), np.int32)
        lens = np.array([len(x) for x in polys], np.int64)
        seg[:n_rows, 0] = np.cumsum(lens) - lens
        seg[:n_rows, 1] = lens
        pts = np.concatenate(polys, 0) if polys else np.zeros((1, 2), np.float32)
        max_points = int(lens.max()) if n_rows else 1
        blocks = [rec.view(np.uint8).reshape(-1), seg.view(np.uint8).reshape(-1), pts.view(np.uint8).reshape(-1),
                  np.asarray(image_rows, np.int32).view(np.uint8)]
        block_off = []
        for a in blocks:
            block_off.append(pos)
            pos += (a.nbytes + _ALIGN - 1) // _ALIGN * _ALIGN
        total = pos
        dev_buf = torch.empty(total, dtype=torch.uint8, device=dev)
        for tile, off in src_tiles:
            tile.src = dev_buf.data_ptr() + off
        pinned = self._staging(total)
        host = pinned.numpy()
        for k in need:
            a = loaded[k][0]
            host[offs[k]: offs[k] + a.nbytes] = a.reshape(-1)
        host[table_off: table_off + ctypes.sizeof(table)] = np.frombuffer(bytes(table), np.uint8)
        for off, a in zip(block_off, blocks):
            host[off: off + a.nbytes] = a
        lab_p, seg_p, pts_p, rows_p = (dev_buf.data_ptr() + off for off in block_off)
        mh, mw = s // r, s // r
        nl = max(n_rows, 1)
        lib = _lib.lib()
        with _lib.on(dev):
            stream = torch.cuda.current_stream(dev)
            st = ctypes.c_void_p(stream.cuda_stream)
            dev_buf[:total].copy_(pinned[:total], non_blocking=True)
            self._copied = torch.cuda.Event()
            self._copied.record(stream)
            if lb_items:
                views = [dev_buf[offs[k]: offs[k] + loaded[k][0].nbytes].view(loaded[k][0].shape) for k in (params[b]["index"] for b in lb_items)]
                letterbox_batch(views, (s, s), auto=False, scaleup=True, swap_rb=False, device=dev, out=canvas)
            table_dev = dev_buf[table_off: table_off + ctypes.sizeof(table)]
            imgs = aug_gather(table_dev, n, s, s, swap_rb=True, dtype=self.dtype, device=dev)
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
        paths = tuple(ds.im_files[p["index"]] for p in params)
        return imgs, targets[:nt], paths, tuple(shapes), masks


_MASK_CODE = {torch.uint8: _lib.Y5_U8, torch.int32: _lib.SEG_I32, torch.float32: _lib.Y5_F32}


def _mask_dtype(kept_per_image, overlap):
    """torch.cat's dtype over the per-image masks: uint8 planes, an int32 overlap plane past 255 labels, float32 zeros for
    an image without labels."""
    dt = torch.uint8
    for k in kept_per_image:
        dt = torch.promote_types(dt, torch.float32 if k == 0 else (torch.int32 if overlap and k > 255 else torch.uint8))
    return dt


def _rasterize(imgsz, polygons, downsample_ratio, device):
    """Host polygons -> (uint8 (n, h / r, w / r) masks, int32 areas, device) through y5_seg_raster."""
    h, w = int(imgsz[0]), int(imgsz[1])
    r = int(downsample_ratio)
    if r not in _RATIOS:
        raise NotImplementedError(f"y5b200: downsample_ratio {r} is not implemented (1 or 4)")
    if h % r or w % r:
        raise NotImplementedError(f"y5b200: image size {(h, w)} is not a multiple of downsample_ratio {r}")
    # np.asarray(polygons, dtype=np.int32) as polygon2mask does; shorter polygons are padded by repeating their last
    # vertex (a zero-length edge draws nothing new), so all share one vertex count
    polys = [np.asarray(p, dtype=np.int32).reshape(-1, 2) for p in polygons]
    if any(len(p) == 0 for p in polys):
        raise ValueError("y5b200: empty polygon")
    n = len(polys)
    nv = max([len(p) for p in polys], default=1)
    verts = np.zeros((max(n, 1), nv, 2), np.int32)
    for i, p in enumerate(polys):
        verts[i, :len(p)] = p
        verts[i, len(p):] = p[-1]
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    v = torch.from_numpy(verts).to(dev)
    keep = torch.ones(max(n, 1), dtype=torch.int32, device=dev)
    masks = torch.zeros(max(n, 1), h // r, w // r, dtype=torch.uint8, device=dev)
    areas = torch.zeros(max(n, 1), dtype=torch.int32, device=dev)
    with _lib.on(dev):
        _lib.check(_lib.lib().y5_seg_raster(v.data_ptr(), nv, keep.data_ptr(), n, h, w, r, masks.data_ptr(), areas.data_ptr(),
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
def _check_val_segments(ds):
    for k, (lab, segs) in enumerate(zip(ds.labels, ds.segments)):
        if len(lab) and len(segs) != len(lab):
            raise NotImplementedError(f"y5b200: image {k} has {len(lab)} labels and {len(segs)} segments (one segment per label is implemented)")
        for seg in segs:
            if not isinstance(seg, np.ndarray) or seg.dtype != np.float32 or seg.ndim != 2 or seg.shape[1] != 2 or len(seg) < 1:
                raise ValueError(f"y5b200: image {k}: segments must be float32 (n >= 1, 2) arrays of normalised points")


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
        _check_val_segments(dataset)
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
        nv = max([len(p) for p in polys], default=1)
        verts = np.zeros((max(nl, 1), nv, 2), np.int32)
        for i, p in enumerate(polys):  # shorter polygons repeat their last vertex (a zero-length edge draws nothing)
            verts[i, :len(p)] = p
            verts[i, len(p):] = p[-1]
        lab6 = np.concatenate(rows, 0) if rows else np.zeros((1, 6), np.float32)
        rec = np.zeros((max(nl, 1), 12), np.float32)  # y5_aug_label records: y5_seg_compose reads their image index
        rec.view(np.int32)[:nl, 9] = lab6[:nl, 0].astype(np.int32)
        table = np.zeros((lay.n, ctypes.sizeof(_lib.AugImage)), np.uint8)  # no flips
        offs = [lay.add_block(a) for a in (verts, lab6, rec, table, np.asarray(image_rows, np.int32), np.ones(max(nl, 1), np.int32))]
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
            _lib.check(lib.y5_seg_raster(verts_p, nv, keep_p, nl, H, W, r, raster.data_ptr(), areas.data_ptr(), st), "seg_raster")
            _lib.check(lib.y5_seg_order(image_rows_p, lay.n, keep_p, areas.data_ptr(), rows_p, int(self.overlap), targets.data_ptr(),
                                        plane.data_ptr(), counts.data_ptr(), st), "seg_order")
            _lib.check(lib.y5_seg_compose(table_p, rec_p, counts.data_ptr(), plane.data_ptr(), raster.data_ptr(), n_out, mh, mw,
                                          int(self.overlap), masks.data_ptr(), _MASK_CODE[mdtype], st), "seg_compose")
        return imgs, targets[:nl], tuple(ds.im_files[k] for k in lay.keys), tuple(lay.shapes), masks
