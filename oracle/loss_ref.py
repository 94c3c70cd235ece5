"""ORACLE (test infrastructure, never on the product path): restatement of ComputeLoss / build_targets.

reference utils/loss.py:101-247 (ComputeLoss.__init__/__call__/build_targets) with the default hyper-parameters
(fl_gamma 0 -> plain BCEWithLogits, label_smoothing 0, autobalance False, gr 1.0, sort_obj_iou False).
``build_targets`` is index work and is restated in numpy (fp32 arithmetic, int64 results -- compared bit-exactly);
the loss itself is fp32 torch so tests can also take its autograd gradient.

Third-party pieces (ultralytics >= 8.4.118, requirements.txt:16, source not under /root/reference, parity unpinned):
``bbox_iou(xywh=True, CIoU=True, eps=1e-7)`` and ``smooth_bce`` -- restated from SURVEY.md Appendix C.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

# (dx, dy) neighbour offsets scaled by g=0.5, in the order the reference stacks its masks (utils/loss.py:198-211):
# own cell, x-frac<.5 -> left, y-frac<.5 -> up, inverse-x -> right, inverse-y -> down
_OFF = np.array([[0, 0], [1, 0], [0, 1], [-1, 0], [0, -1]], np.float32) * np.float32(0.5)


def build_targets(targets: np.ndarray, anchors: np.ndarray, shapes, anchor_t: float = 4.0):
    """targets (nt,6) [img, cls, x, y, w, h] normalised; anchors (nl,na,2) grid units; shapes: [(ny,nx)] per level.

    Returns per level: tcls (n,) int64, tbox (n,4) fp32, (b, a, gj, gi) int64 each, anch (n,2) fp32 -- in exactly
    the order the reference produces (offset-major, then anchor-major, then target order)."""
    targets = np.asarray(targets, np.float32).reshape(-1, 6)
    na, nt = anchors.shape[1], targets.shape[0]
    ai = np.repeat(np.arange(na, dtype=np.float32)[:, None], nt, 1)  # (na, nt)
    t7 = np.concatenate((np.repeat(targets[None], na, 0), ai[..., None]), 2)  # (na, nt, 7)
    g = np.float32(0.5)
    out = []
    for i, (ny, nx) in enumerate(shapes):
        anc = np.asarray(anchors[i], np.float32)
        gain = np.ones(7, np.float32)
        gain[2:6] = np.array([nx, ny, nx, ny], np.float32)
        t = t7 * gain
        if nt:
            r = t[..., 4:6] / anc[:, None]
            keep = np.maximum(r, np.float32(1) / r).max(2) < np.float32(anchor_t)
            t = t[keep]  # (n,7) anchor-major then target order
            gxy = t[:, 2:4]
            gxi = gain[[2, 3]] - gxy
            jm, km = ((np.fmod(gxy, np.float32(1)) < g) & (gxy > 1)).T
            lm, mm = ((np.fmod(gxi, np.float32(1)) < g) & (gxi > 1)).T
            sel = np.stack((np.ones_like(jm), jm, km, lm, mm))  # (5, n)
            t = np.repeat(t[None], 5, 0)[sel]
            offsets = (np.zeros_like(gxy)[None] + _OFF[:, None])[sel]
        else:
            t = t7[0]
            offsets = np.zeros((0, 2), np.float32)
        b = t[:, 0].astype(np.int64)
        c = t[:, 1].astype(np.int64)
        gxy, gwh = t[:, 2:4], t[:, 4:6]
        a = t[:, 6].astype(np.int64)
        gij = (gxy - offsets).astype(np.int64)  # trunc toward zero, like .long()
        gi = np.clip(gij[:, 0], 0, nx - 1)
        gj = np.clip(gij[:, 1], 0, ny - 1)
        # NB the reference clamps gj/gi in place *after* gij was used for tbox only through the aliasing of
        # gi, gj = gij.T -> clamp_ modifies gij too, and tbox is built afterwards from the clamped gij (:242-243)
        gij_c = np.stack((gi, gj), 1)
        tbox = np.concatenate((gxy - gij_c.astype(np.float32), gwh), 1).astype(np.float32)
        out.append(dict(tcls=c, tbox=tbox, b=b, a=a, gj=gj, gi=gi, anch=anc[a]))
    return out


def bbox_ciou(p: torch.Tensor, t: torch.Tensor, eps: float = 1e-7) -> torch.Tensor:
    """CIoU of xywh boxes (n,4) vs (n,4) -> (n,)  (SURVEY.md Appendix C)."""
    x1, y1, w1, h1 = p.unbind(1)
    x2, y2, w2, h2 = t.unbind(1)
    b1x1, b1x2, b1y1, b1y2 = x1 - w1 / 2, x1 + w1 / 2, y1 - h1 / 2, y1 + h1 / 2
    b2x1, b2x2, b2y1, b2y2 = x2 - w2 / 2, x2 + w2 / 2, y2 - h2 / 2, y2 + h2 / 2
    inter = (torch.minimum(b1x2, b2x2) - torch.maximum(b1x1, b2x1)).clamp(0) * (
        torch.minimum(b1y2, b2y2) - torch.maximum(b1y1, b2y1)
    ).clamp(0)
    union = w1 * h1 + w2 * h2 - inter + eps
    iou = inter / union
    cw = torch.maximum(b1x2, b2x2) - torch.minimum(b1x1, b2x1)
    ch = torch.maximum(b1y2, b2y2) - torch.minimum(b1y1, b2y1)
    c2 = cw**2 + ch**2 + eps
    rho2 = ((b2x1 + b2x2 - b1x1 - b1x2) ** 2 + (b2y1 + b2y2 - b1y1 - b1y2) ** 2) / 4
    v = (4 / math.pi**2) * (torch.atan(w2 / h2) - torch.atan(w1 / h1)) ** 2
    with torch.no_grad():
        alpha = v / (v - iou + (1 + eps))
    return iou - (rho2 / c2 + v * alpha)


def compute_loss(p, targets, anchors, hyp, balance=(4.0, 1.0, 0.4)):
    """p: list of (B,na,ny,nx,no) fp32 torch tensors (may require grad); targets (nt,6) numpy/torch;
    anchors (nl,na,2) grid units.  Returns (loss (1,), items (3,) = [lbox, lobj, lcls])."""
    tg = targets.detach().cpu().numpy() if isinstance(targets, torch.Tensor) else np.asarray(targets)
    anc = anchors.detach().cpu().numpy() if isinstance(anchors, torch.Tensor) else np.asarray(anchors)
    nc = p[0].shape[-1] - 5
    bt = build_targets(tg, anc, [tuple(pi.shape[2:4]) for pi in p], hyp["anchor_t"])
    dt = p[0].dtype  # fp32 like the reference, or float64 for the tests' float64 cross-checks
    lcls = torch.zeros(1, dtype=dt)
    lbox = torch.zeros(1, dtype=dt)
    lobj = torch.zeros(1, dtype=dt)
    cp, cn = 1.0 - 0.5 * hyp.get("label_smoothing", 0.0), 0.5 * hyp.get("label_smoothing", 0.0)
    pw_cls = torch.tensor([hyp["cls_pw"]], dtype=dt)
    pw_obj = torch.tensor([hyp["obj_pw"]], dtype=dt)
    for i, pi in enumerate(p):
        d = bt[i]
        b, a, gj, gi = (torch.from_numpy(d[k]) for k in ("b", "a", "gj", "gi"))
        tobj = torch.zeros(pi.shape[:4], dtype=pi.dtype)
        n = b.shape[0]
        if n:
            ps = pi[b, a, gj, gi]
            pxy = ps[:, 0:2].sigmoid() * 2 - 0.5
            pwh = (ps[:, 2:4].sigmoid() * 2) ** 2 * torch.from_numpy(d["anch"]).to(dt)
            iou = bbox_ciou(torch.cat((pxy, pwh), 1), torch.from_numpy(d["tbox"]).to(dt))
            lbox = lbox + (1.0 - iou).mean()
            tobj[b, a, gj, gi] = iou.detach().clamp(0).type(tobj.dtype)  # duplicates: last writer wins
            if nc > 1:
                t = torch.full_like(ps[:, 5:], cn)
                t[torch.arange(n), torch.from_numpy(d["tcls"])] = cp
                lcls = lcls + F.binary_cross_entropy_with_logits(ps[:, 5:], t, pos_weight=pw_cls)
        lobj = lobj + F.binary_cross_entropy_with_logits(pi[..., 4], tobj, pos_weight=pw_obj) * balance[i]
    lbox = lbox * hyp["box"]
    lobj = lobj * hyp["obj"]
    lcls = lcls * hyp["cls"]
    bs = p[0].shape[0]
    return (lbox + lobj + lcls) * bs, torch.cat((lbox, lobj, lcls)).detach()


def synth_targets(bs: int, seed: int = 1, nc: int = 80) -> np.ndarray:
    """COCO128-shaped labels (SURVEY.md section 8d): n ~ Poisson(7.3) clipped to [1,40] per image."""
    rs = np.random.RandomState(seed)
    rows = []
    for b in range(bs):
        n = int(np.clip(rs.poisson(7.3), 1, 40))
        cls = rs.randint(0, nc, n)
        xy = rs.uniform(0.1, 0.9, (n, 2))
        wh = np.exp(rs.uniform(-4, -1, (n, 2)))
        rows.append(np.concatenate((np.full((n, 1), b), cls[:, None], xy, wh), 1))
    return np.concatenate(rows, 0).astype(np.float32)


def compute_loss_torch(p, targets, anchors, hyp, balance=(4.0, 1.0, 0.4)):
    """The same loss as `compute_loss`, expressed with torch ops ON THE DEVICE OF `p` the way the reference executes it
    (utils/loss.py:134-247: build_targets with boolean-mask indexing, gather / scatter, BCEWithLogits): the loss half of the
    "reference's own torch-cuda build" arm in bench.py.  Checked against `compute_loss` by tests/test_oracle_golden.py."""
    dev = p[0].device
    targets = targets.to(dev, torch.float32).view(-1, 6)
    anchors = anchors.to(dev, torch.float32)
    na, nt, nc = anchors.shape[1], targets.shape[0], p[0].shape[-1] - 5
    cp, cn = 1.0 - 0.5 * hyp.get("label_smoothing", 0.0), 0.5 * hyp.get("label_smoothing", 0.0)
    pw_cls = torch.tensor([hyp["cls_pw"]], device=dev)
    pw_obj = torch.tensor([hyp["obj_pw"]], device=dev)
    ai = torch.arange(na, device=dev).float().view(na, 1).repeat(1, nt)
    t7 = torch.cat((targets.repeat(na, 1, 1), ai[..., None]), 2)
    off = torch.from_numpy(_OFF).to(dev)
    gain = torch.ones(7, device=dev)
    lcls, lbox, lobj = (torch.zeros(1, device=dev) for _ in range(3))
    for i, pi in enumerate(p):
        ny, nx = pi.shape[2:4]
        gain[2:6] = torch.tensor([nx, ny, nx, ny], device=dev, dtype=torch.float32)
        t = t7 * gain
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
            t, offsets = t7[0], 0
        b, c = t[:, 0].long(), t[:, 1].long()
        gxy, gwh, a = t[:, 2:4], t[:, 4:6], t[:, 6].long()
        gij = (gxy - offsets).long()
        gi, gj = gij[:, 0].clamp(0, nx - 1), gij[:, 1].clamp(0, ny - 1)
        tbox = torch.cat((gxy - torch.stack((gi, gj), 1), gwh), 1)
        tobj = torch.zeros(pi.shape[:4], dtype=pi.dtype, device=dev)
        n = b.shape[0]
        if n:
            ps = pi[b, a, gj, gi]
            pxy = ps[:, 0:2].sigmoid() * 2 - 0.5
            pwh = (ps[:, 2:4].sigmoid() * 2) ** 2 * anchors[i][a]
            iou = bbox_ciou(torch.cat((pxy, pwh), 1), tbox)
            lbox = lbox + (1.0 - iou).mean()
            tobj[b, a, gj, gi] = iou.detach().clamp(0).type(tobj.dtype)
            if nc > 1:
                tc = torch.full_like(ps[:, 5:], cn)
                tc[torch.arange(n, device=dev), c] = cp
                lcls = lcls + F.binary_cross_entropy_with_logits(ps[:, 5:], tc, pos_weight=pw_cls)
        lobj = lobj + F.binary_cross_entropy_with_logits(pi[..., 4], tobj, pos_weight=pw_obj) * balance[i]
    lbox, lobj, lcls = lbox * hyp["box"], lobj * hyp["obj"], lcls * hyp["cls"]
    return (lbox + lobj + lcls) * p[0].shape[0], torch.cat((lbox, lobj, lcls)).detach()
