"""ORACLE (test infrastructure, never on the product path): the detection ComputeLoss in float64, restricted to the
logits the loss reads.

The index work is `oracle.loss_ref.build_targets` (numpy fp32 like the reference, pinned to tests/golden/loss.npz);
float64 starts after it (tbox and the anchors promote exactly).  The loss is the reference's own expressions
(utils/loss.py:134-183, `loss_ref.bbox_ciou`) in torch ops, so ties follow torch's rules (minimum / maximum split the
gradient, clamp(0) passes it at 0).  The autograd leaves are not the whole (B, na, ny, nx, no) maps -- at 16 images of
640 pixels P3 alone would be 0.8 GB in float64 -- but:
- the objectness planes p[..., 4], (B, na, ny, nx);
- the rows of the unique matched cells, (u, no), gathered once per match through a match -> row map, so autograd sums
  the gradients of duplicate matches as the reference's gather backward does.
`tobj` is rounded to the logits dtype (`iou.detach().clamp(0).type(tobj.dtype)`), the last match of a cell wins.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle import loss_ref

BALANCE = (4.0, 1.0, 0.4)


def match_cells(bt, shapes, batch, na):
    """Per level: `lin` (n,) linear cell index ((b*na + a)*ny + gj)*nx + gi of every match, `ucell` (u,) the sorted
    unique cells, `inv` (n,) match -> unique row, `mult` (u,) matches per unique cell.  Adds them to the dicts of `bt`."""
    for d, (ny, nx) in zip(bt, shapes):
        lin = ((torch.from_numpy(d["b"]) * na + torch.from_numpy(d["a"])) * ny + torch.from_numpy(d["gj"])) * nx + torch.from_numpy(d["gi"])
        ucell, inv, mult = torch.unique(lin, sorted=True, return_inverse=True, return_counts=True)
        d.update(lin=lin, ucell=ucell, inv=inv, mult=mult, cells=batch * na * ny * nx)
    return bt


def targets_for(targets, anchors, shapes, batch, anchor_t=4.0):
    """loss_ref.build_targets + match_cells."""
    anc = np.asarray(anchors, np.float32)
    bt = loss_ref.build_targets(np.asarray(targets, np.float32).reshape(-1, 6), anc, shapes, anchor_t)
    return match_cells(bt, shapes, batch, anc.shape[1])


def leaves_from_maps(p, bt):
    """(obj planes, unique rows) in float64 from full head maps (B, na, ny, nx, no) on any device."""
    obj = [t[..., 4].detach().double().cpu() for t in p]
    rows = [t.detach().reshape(-1, t.shape[-1])[d["ucell"].to(t.device)].double().cpu() for t, d in zip(p, bt)]
    return obj, rows


def loss64(obj, rows, bt, hyp, nc, batch, dtype=torch.float64, scale=1.0, balance=BALANCE):
    """obj: per level (B, na, ny, nx) float64 objectness logits; rows: per level (u, no) float64 logits of the unique matched
    cells (the logits already rounded to `dtype`); bt: `targets_for` output.  `nc == 1` means no class term.

    Returns dict: loss (float), items (3,) float64 [lbox, lobj, lcls], and per level gobj (B, na, ny, nx) and grows (u, no),
    the gradients of `loss * scale`; arows (u, no), the sum over the matches of a cell of |per-match contribution|; tobj
    (u,) the objectness target of every unique cell (rounded to `dtype`)."""
    cp, cn = 1.0 - 0.5 * hyp.get("label_smoothing", 0.0), 0.5 * hyp.get("label_smoothing", 0.0)
    pw_cls = torch.tensor([hyp["cls_pw"]], dtype=torch.float64)
    pw_obj = torch.tensor([hyp["obj_pw"]], dtype=torch.float64)
    lbox, lobj, lcls = (torch.zeros(1, dtype=torch.float64) for _ in range(3))
    ol = [o.detach().double().clone().requires_grad_(True) for o in obj]
    rl = [r.detach().double().clone().requires_grad_(True) for r in rows]
    ps_all, tobj_u = [], []
    for i, d in enumerate(bt):
        n = len(d["b"])
        tobj = torch.zeros(ol[i].shape, dtype=torch.float64)
        if n:
            ps = rl[i][d["inv"]]
            ps.retain_grad()
            ps_all.append(ps)
            pxy = ps[:, 0:2].sigmoid() * 2 - 0.5
            pwh = (ps[:, 2:4].sigmoid() * 2) ** 2 * torch.from_numpy(d["anch"]).double()
            iou = loss_ref.bbox_ciou(torch.cat((pxy, pwh), 1), torch.from_numpy(d["tbox"]).double())
            lbox = lbox + (1.0 - iou).mean()
            # last writer wins on a duplicate cell: the value of its highest match index
            last = torch.zeros(len(d["ucell"]), dtype=torch.int64).scatter_reduce(0, d["inv"], torch.arange(n), "amax")
            tv = iou.detach().clamp(0).to(dtype).double()[last]
            tobj.view(-1)[d["ucell"]] = tv
            tobj_u.append(tv)
            if nc > 1:
                t = torch.full_like(ps[:, 5:], cn)
                t[torch.arange(n), torch.from_numpy(d["tcls"])] = cp
                lcls = lcls + F.binary_cross_entropy_with_logits(ps[:, 5:], t, pos_weight=pw_cls)
        else:
            ps_all.append(None)
            tobj_u.append(torch.zeros(0, dtype=torch.float64))
        lobj = lobj + F.binary_cross_entropy_with_logits(ol[i], tobj, pos_weight=pw_obj) * balance[i]
    lbox, lobj, lcls = lbox * hyp["box"], lobj * hyp["obj"], lcls * hyp["cls"]
    loss = (lbox + lobj + lcls) * batch
    (loss * scale).backward()
    out = dict(loss=float(loss.detach()), items=torch.cat((lbox, lobj, lcls)).detach(), gobj=[], grows=[], arows=[], tobj=tobj_u)
    for i, d in enumerate(bt):
        out["gobj"].append(ol[i].grad)
        no = rl[i].shape[1]
        ps = ps_all[i]
        if ps is None:
            out["grows"].append(torch.zeros(0, no, dtype=torch.float64))
            out["arows"].append(torch.zeros(0, no, dtype=torch.float64))
            continue
        g = ps.grad if ps.grad is not None else torch.zeros_like(ps)
        out["grows"].append(rl[i].grad if rl[i].grad is not None else torch.zeros_like(rl[i]))
        out["arows"].append(torch.zeros_like(rl[i]).index_add_(0, d["inv"], g.abs()))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# targets at the edges of build_targets and CIoU.  Positions are given for a 64 x 64 image (P3 8 x 8 cells, anchors in
# grid units as Detect stores them: P3 (1.25, 1.625), (2, 3.75), (4.125, 2.875)), every value exact in fp32.
# ---------------------------------------------------------------------------------------------------------------------
_f = np.float32


def _below(v):
    return np.nextafter(_f(v), _f(0))


def _above(v):
    return np.nextafter(_f(v), _f(2))


def edge_targets():
    """(nt, 6) rows for 2 images on an 8 x 8 P3 grid: fractional positions 0, 0.5 and the float below 0.5, gx == 1 and
    the float above it, gxi <= 1 at the right / bottom border, x == 0 and x == 1 (the clamp), w / h ratios of exactly
    anchor_t and just below, identical rows and different classes in one cell."""
    w, h = 0.15625, 0.203125  # P3 anchor 0 exactly
    rows = [
        [0, 1, 3 / 8, 3 / 8, w, h],                         # gx, gy = 3: fractional part 0
        [0, 2, 3.5 / 8, 4.5 / 8, w, h],                     # fractional part exactly 0.5: no left / up neighbour
        [1, 3, _below(3.5 / 8), _below(4.5 / 8), w, h],     # just below 0.5
        [1, 4, 1 / 8, 1 / 8, w, h],                         # gx == gy == 1: not > 1
        [0, 5, _above(1 / 8), _above(1 / 8), w, h],         # the float above 1
        [1, 6, 7.5 / 8, 7.5 / 8, w, h],                     # gxi = gyi = 0.5
        [0, 7, 7 / 8, 7 / 8, w, h],                         # gxi = gyi = 1
        [1, 8, 1.0, 1.0, w, h],                             # x == y == 1: gij clamped to the last cell
        [1, 9, 0.0, 0.0, w, h],                             # x == y == 0
        [0, 10, 0.3, 0.7, 0.625, h],                        # gw / aw == anchor_t for anchor 0: dropped there
        [1, 11, 0.6, 0.3, _below(0.625), h],                # just below anchor_t: kept
        [0, 12, 0.55, 0.45, 0.0390625, h],                  # aw / gw == anchor_t
        [0, 13, 0.55, 0.45, w, h],
        [0, 13, 0.55, 0.45, w, h],                          # an identical row
        [0, 14, 0.55, 0.45, w, h],                          # another class in the same cell
        [1, 15, 0.2, 0.8, 0.3, 0.05],
    ]
    return np.array(rows, np.float32)


def invalid_rows(batch, nc):
    """Rows the loss ignores: class >= nc, class < 0, image >= batch, image < 0."""
    return np.array([[0, nc, 0.5, 0.5, 0.2, 0.2], [0, -1, 0.4, 0.4, 0.2, 0.2], [batch, 0, 0.5, 0.5, 0.2, 0.2],
                     [-1, 0, 0.3, 0.3, 0.1, 0.1]], np.float32)


def tie_targets():
    """Image-0 rows on an 8 x 8 P3 grid that, with box logits 0 (predicted box (0.5, 0.5, aw, ah) in every cell), tie
    CIoU's min / max / clamp for P3 anchor 0: full overlap, one shared edge, and boxes that touch (intersection width
    exactly 0, through the left-neighbour match)."""
    w, h = 1.25 / 8, 1.625 / 8
    return np.array([
        [0, 1, 2.5 / 8, 3.5 / 8, w, h],          # the predicted box of cell (2, 3)
        [0, 2, 5.75 / 8, 2.5 / 8, 1.75 / 8, h],  # cell (5, 2): tbox x 0.75, w 1.75 -> the left edges coincide
        [0, 3, 3.375 / 8, 5.5 / 8, 0.5 / 8, h],  # left neighbour (2, 5): tbox x 1.375, w 0.5 -> touches at x = 1.125
    ], np.float32)


def crowded_targets(batch, per_image, size, seed=7, nc=80):
    """`per_image` small boxes per image of `size` pixels, 12-30 px wide and high: every P3 anchor (10x13, 16x30, 33x23)
    passes the ratio test, so each target makes up to 9 P3 matches."""
    rs = np.random.RandomState(seed)
    n = batch * per_image
    b = np.repeat(np.arange(batch), per_image)
    wh = rs.uniform(12, 30, (n, 2)) / size
    xy = rs.uniform(0.02, 0.98, (n, 2))
    return np.concatenate((b[:, None], rs.randint(0, nc, (n, 1)), xy, wh), 1).astype(np.float32)


def dense_grad(res, bt, shapes, batch, na, no):
    """The expected gradient of level l as full (B, na, ny, nx, no) float64 maps (small shapes only)."""
    out = []
    for i, (d, (ny, nx)) in enumerate(zip(bt, shapes)):
        g = torch.zeros(batch * na * ny * nx, no, dtype=torch.float64)
        if len(d["ucell"]):
            g[d["ucell"]] = res["grows"][i]
        g[:, 4] = res["gobj"][i].reshape(-1)
        out.append(g.view(batch, na, ny, nx, no))
    return out
