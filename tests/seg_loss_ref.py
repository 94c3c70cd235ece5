"""ORACLE (test infrastructure, never on the product path): restatement of the segmentation ComputeLoss.

reference utils/segment/loss.py:15-195 and crop_mask (utils/segment/general.py:10-22) with the default
hyper-parameters (fl_gamma 0, label_smoothing 0, autobalance False, gr 1.0).  The box / objectness / class terms are
oracle.loss_ref's; this module adds the target bookkeeping of the mask term (tidx, xywhn) and the mask BCE.
- ``build_targets_seg``: numpy, fp32 arithmetic, int64 results (compared bit-exactly).
- ``compute_seg_loss``: fp32 torch on the CPU (autograd gives the oracle gradients).
- ``compute_seg_loss_torch``: the reference's own expressions (torch build_targets, per-image Python loop with its
  device-to-host sync) on any device: the torch-cuda arm of tools/seg_loss_bench.py.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle import loss_ref


def build_targets_seg(targets: np.ndarray, anchors: np.ndarray, shapes, batch: int, overlap: bool, anchor_t: float = 4.0):
    """loss_ref.build_targets plus, per level, ``tidx`` (n,) int64 and ``xywhn`` (n,4) fp32 in the same match order.

    tidx: the target row, or with `overlap` the value at the row's position in cat([1..n_0, 1..n_1, ...]) (n_i = rows of
    image i) -- the running index inside each image only when targets are sorted by image."""
    targets = np.asarray(targets, np.float32).reshape(-1, 6)
    nt = targets.shape[0]
    if overlap:
        ti = np.concatenate([np.arange(int((targets[:, 0] == i).sum()), dtype=np.float32) + 1 for i in range(batch)] or
                            [np.zeros(0, np.float32)])
    else:
        ti = np.arange(nt, dtype=np.float32)
    # the same selection as loss_ref.build_targets (anchor-major, then offset-major, then target order), tracking rows
    out = loss_ref.build_targets(targets, anchors, shapes, anchor_t)
    na = anchors.shape[1]
    for i, (ny, nx) in enumerate(shapes):
        if nt:
            anc = np.asarray(anchors[i], np.float32)
            gain = np.array([nx, ny, nx, ny], np.float32)
            t = np.repeat(targets[None], na, 0)  # (na, nt, 6)
            rows = np.repeat(np.arange(nt)[None], na, 0)
            tg = t[..., 2:6] * gain
            r = tg[..., 2:4] / anc[:, None]
            keep = np.maximum(r, np.float32(1) / r).max(2) < np.float32(anchor_t)
            tg, rows = tg[keep], rows[keep]
            gxy = tg[:, 0:2]
            gxi = gain[[0, 1]] - gxy
            g = np.float32(0.5)
            jm, km = ((np.fmod(gxy, np.float32(1)) < g) & (gxy > 1)).T
            lm, mm = ((np.fmod(gxi, np.float32(1)) < g) & (gxi > 1)).T
            sel = np.stack((np.ones_like(jm), jm, km, lm, mm))
            tg = np.repeat(tg[None], 5, 0)[sel]
            rows = np.repeat(rows[None], 5, 0)[sel]
            xywhn = (tg / gain).astype(np.float32)
        else:
            rows = np.zeros(0, np.int64)
            xywhn = np.zeros((0, 4), np.float32)
        assert len(rows) == len(out[i]["b"])
        out[i]["tidx"] = ti[rows].astype(np.int64)
        out[i]["xywhn"] = xywhn
    return out


def _downsample(masks, proto):
    mh, mw = proto.shape[2:]
    return F.interpolate(masks[None], (mh, mw), mode="nearest")[0] if tuple(masks.shape[-2:]) != (mh, mw) else masks


def _mask_term(pmask, proto, masks, b, tidx, xywhn, overlap):
    """One level's sum over images of mean_j(crop BCE / (mh*mw) / area_j) (segment/loss.py:89-99,116-120)."""
    bs, nm, mh, mw = proto.shape
    marea = xywhn[:, 2:].prod(1)
    xy = xywhn * torch.tensor([mw, mh, mw, mh], device=xywhn.device, dtype=xywhn.dtype)
    mxyxy = torch.cat((xy[:, :2] - xy[:, 2:] / 2, xy[:, :2] + xy[:, 2:] / 2), 1)
    lseg = torch.zeros(1, device=proto.device, dtype=proto.dtype)  # float64 inputs accumulate in float64
    for bi in b.unique():
        j = b == bi
        if overlap:
            gt = torch.where(masks[bi][None] == tidx[j].view(-1, 1, 1), 1.0, 0.0)
        else:
            gt = masks[tidx][j]
        pred = (pmask[j] @ proto[bi].reshape(nm, -1)).view(-1, mh, mw)
        loss = F.binary_cross_entropy_with_logits(pred, gt.to(pred.dtype), reduction="none")
        x1, y1, x2, y2 = torch.chunk(mxyxy[j][:, :, None], 4, 1)
        r = torch.arange(mw, device=pred.device, dtype=x1.dtype)[None, None, :]
        c = torch.arange(mh, device=pred.device, dtype=x1.dtype)[None, :, None]
        crop = loss * ((r >= x1) * (r < x2) * (c >= y1) * (c < y2))
        lseg = lseg + (crop.mean(dim=(1, 2)) / marea[j]).mean()
    return lseg


def compute_seg_loss(p, proto, targets, masks, anchors, hyp, overlap, balance=(4.0, 1.0, 0.4)):
    """p: list of (B,na,ny,nx,5+nc+nm) fp32 CPU tensors, proto (B,nm,mh,mw), masks (N,H,W) fp32.
    Returns (loss (1,), items (4,) = [lbox, lseg, lobj, lcls])."""
    tg = targets.detach().cpu().numpy() if isinstance(targets, torch.Tensor) else np.asarray(targets, np.float32)
    anc = anchors.detach().cpu().numpy() if isinstance(anchors, torch.Tensor) else np.asarray(anchors)
    bs, nm = proto.shape[:2]
    nc = p[0].shape[-1] - 5 - nm
    det, items = loss_ref.compute_loss([pi[..., : 5 + nc] for pi in p], tg, anc, hyp, balance)
    lbox, lobj, lcls = items.view(3, 1).unbind(0)
    bt = build_targets_seg(tg, anc, [tuple(pi.shape[2:4]) for pi in p], bs, overlap, hyp["anchor_t"])
    masks = _downsample(torch.as_tensor(masks, dtype=torch.float32), proto)
    lseg = torch.zeros(1, dtype=proto.dtype)
    for i, pi in enumerate(p):
        d = bt[i]
        if len(d["b"]):
            b, a, gj, gi = (torch.from_numpy(d[k]) for k in ("b", "a", "gj", "gi"))
            pmask = pi[b, a, gj, gi][:, 5 + nc:]
            lseg = lseg + _mask_term(pmask, proto, masks, b, torch.from_numpy(d["tidx"]), torch.from_numpy(d["xywhn"]), overlap)
    lseg = lseg * (hyp["box"] / bs)
    return det + lseg * bs, torch.cat((lbox, lseg.detach(), lobj, lcls))


def compute_seg_loss_torch(p, proto, targets, masks, anchors, hyp, overlap, balance=(4.0, 1.0, 0.4)):
    """The reference's expressions on the device of `p`, in one pass as segment/loss.py:48-120 runs them: torch
    build_targets (boolean-mask indexing) once per level, one gather of the matched rows, CIoU, objectness / class BCE, and
    the mask term's per-image loop over ``b.unique()``."""
    dev = p[0].device
    targets = targets.to(dev, torch.float32).view(-1, 6)
    anchors = anchors.to(dev, torch.float32)
    bs, nm = proto.shape[:2]
    nc = p[0].shape[-1] - 5 - nm
    na, nt = anchors.shape[1], targets.shape[0]
    cp, cn = 1.0 - 0.5 * hyp.get("label_smoothing", 0.0), 0.5 * hyp.get("label_smoothing", 0.0)
    pw_cls = torch.tensor([hyp["cls_pw"]], device=dev)
    pw_obj = torch.tensor([hyp["obj_pw"]], device=dev)
    if overlap:
        ti = torch.cat([torch.arange(int((targets[:, 0] == i).sum()), device=dev).float().view(1, -1).repeat(na, 1) + 1
                        for i in range(bs)], 1)
    else:
        ti = torch.arange(nt, device=dev).float().view(1, nt).repeat(na, 1)
    ai = torch.arange(na, device=dev).float().view(na, 1).repeat(1, nt)
    t8 = torch.cat((targets.repeat(na, 1, 1), ai[..., None], ti[..., None]), 2)
    off = torch.from_numpy(loss_ref._OFF).to(dev)
    gain = torch.ones(8, device=dev)
    lbox, lobj, lcls, lseg = (torch.zeros(1, device=dev) for _ in range(4))
    masks = _downsample(masks, proto)
    for i, pi in enumerate(p):
        ny, nx = pi.shape[2:4]
        gain[2:6] = torch.tensor([nx, ny, nx, ny], device=dev, dtype=torch.float32)
        t = t8 * gain
        if nt:
            r = t[..., 4:6] / anchors[i][:, None]
            t = t[torch.max(r, 1 / r).max(2)[0] < hyp["anchor_t"]]
            gxy = t[:, 2:4]
            gxi = gain[[2, 3]] - gxy
            j, k = ((gxy % 1 < 0.5) & (gxy > 1)).T
            l, m = ((gxi % 1 < 0.5) & (gxi > 1)).T
            sel = torch.stack((torch.ones_like(j), j, k, l, m))
            t = t.repeat((5, 1, 1))[sel]
            offsets = (torch.zeros_like(gxy)[None] + off[:, None])[sel]
        else:
            t, offsets = t8[0], 0
        b, c, a, tidx = t[:, 0].long(), t[:, 1].long(), t[:, 6].long(), t[:, 7].long()
        gxy, gwh = t[:, 2:4], t[:, 4:6]
        gij = (gxy - offsets).long()
        gi, gj = gij[:, 0].clamp(0, nx - 1), gij[:, 1].clamp(0, ny - 1)
        tobj = torch.zeros(pi.shape[:4], dtype=pi.dtype, device=dev)
        n = b.shape[0]
        if n:
            pxy, pwh, _, pcls, pmask = pi[b, a, gj, gi].split((2, 2, 1, nc, nm), 1)
            pxy = pxy.sigmoid() * 2 - 0.5
            pwh = (pwh.sigmoid() * 2) ** 2 * anchors[i][a]
            iou = loss_ref.bbox_ciou(torch.cat((pxy, pwh), 1), torch.cat((gxy - torch.stack((gi, gj), 1), gwh), 1))
            lbox = lbox + (1.0 - iou).mean()
            tobj[b, a, gj, gi] = iou.detach().clamp(0).type(tobj.dtype)
            if nc > 1:
                tc = torch.full_like(pcls, cn)
                tc[torch.arange(n, device=dev), c] = cp
                lcls = lcls + F.binary_cross_entropy_with_logits(pcls, tc, pos_weight=pw_cls)
            lseg = lseg + _mask_term(pmask, proto, masks, b, tidx, torch.cat((gxy, gwh), 1) / gain[2:6], overlap)
        lobj = lobj + F.binary_cross_entropy_with_logits(pi[..., 4], tobj, pos_weight=pw_obj) * balance[i]
    lbox, lobj, lcls = lbox * hyp["box"], lobj * hyp["obj"], lcls * hyp["cls"]
    lseg = lseg * (hyp["box"] / bs)
    return (lbox + lobj + lcls + lseg) * bs, torch.cat((lbox, lseg, lobj, lcls)).detach()


def paint_masks(shape, boxes, values):
    """(H, W) fp32 map: each xywhn box filled with its value, later boxes on top (synthetic masks for tests / benchmarks)."""
    h, w = shape
    m = np.zeros((h, w), np.float32)
    for (x, y, bw, bh), v in zip(boxes, values):
        x0, x1 = int(max(0, (x - bw / 2) * w)), int(min(w, np.ceil((x + bw / 2) * w)))
        y0, y1 = int(max(0, (y - bh / 2) * h)), int(min(h, np.ceil((y + bh / 2) * h)))
        m[y0:y1, x0:x1] = v
    return m


def overlap_masks(targets: np.ndarray, batch: int, h: int, w: int) -> np.ndarray:
    """(batch, h, w) overlap-style masks: pixel value k marks the image's k-th target row (1-based), drawn from the boxes."""
    masks = np.zeros((batch, h, w), np.float32)
    for b in range(batch):
        rows = np.nonzero(targets[:, 0] == b)[0]
        masks[b] = paint_masks((h, w), targets[rows, 2:6], np.arange(1, len(rows) + 1))
    return masks
