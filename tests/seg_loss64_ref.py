"""ORACLE (test infrastructure, never on the product path): the segmentation ComputeLoss in float64, with the bound sums
the device kernels' error bounds need, on any device.

The index work is `tests/seg_loss_ref.build_targets_seg` (numpy fp32 like the reference): tidx, xywhn, and from them the
crop bounds `mxyxy = xywh2xyxy(xywhn * [mw, mh, mw, mh])` and `marea = w * h`, both in fp32 exactly as the reference
computes them (reference utils/segment/loss.py:88-99).  The masks are downsampled by `F.interpolate(mode="nearest")`
itself.  Float64 starts after that; every one of these values promotes exactly.

- Detection terms: `loss64_ref.loss64` on the unique matched rows, sliced to `[:, :5 + nc]`.
- Mask term, in closed form, one chunk of matches of one image at a time (autograd over dense maps does not fit at
  16 x 160^2 with thousands of matches).  For match j of level l in image b, over the proto pixels p:
      x = coef_j @ proto[b]                          (float64)
      l_j = sum_{p in crop_j} BCE(x_p, gt_jp) / (mh mw) / marea_j
      lseg = box / B * sum_(l, b) mean_{j in (l, b)} l_j
      g_jp = (sigmoid(x_p) - gt_jp) s_j on the crop, 0 elsewhere,   s_j = scale box / n_(l,b) / (mh mw) / marea_j
      dcoef_j = g_j @ proto[b]^T,   dproto[b] = sum_j coef_j^T g_j      (all levels' matches of the image)
  crop_j is `crop_mask`'s half-open [x1, x2) x [y1, y2): the columns ceil(x1) .. ceil(x2) - 1.

Alongside the values it returns the sums the error bounds need (see `ratios`):
- acoef_j = |g_j| @ |proto[b]|^T and aproto[b] = sum_j |coef_j|^T |g_j|;
- ecoef_j = E_j @ |proto[b]|^T and eproto[b] = sum_j |coef_j|^T E_j, with E_jp a bound, in units of the fp32 unit
  roundoff, on the error of an fp32 evaluation of g_jp:
      E = 7 |g| + s (sig (1 - sig) (2 + 1.2 |x| + nm X) + 3 sig),   X = |coef_j| @ |proto[b]|
  (nm X: the nm-term FMA chain of the logit, propagated through sigmoid' <= sig (1 - sig); 2 + 1.2 |x|: __expf's ulp
  error; 3 sig: the rounding of 1 + e^-x and __fdividef's two ulps; 7 |g|: sigmoid - gt, the product with s and the
  five roundings of s itself);
- ncover[b, p], the number of matches whose crop covers pixel p.

`MUTATIONS` are deliberately wrong variants of the mask term; the CPU suite shows `check` rejects each of them.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from tests import loss64_ref as R
from tests import seg_loss_ref
from tests.golden import make_seg_golden as mg

F16, BF16, F32 = torch.float16, torch.bfloat16, torch.float32
U = {F32: 2.0**-24, F16: 2.0**-11, BF16: 2.0**-8}
Z = {F32: 0.0, F16: 2.0**-25, BF16: 0.0}   # half the fp16 subnormal spacing
U32 = U[F32]
F16_OVERFLOW = 65520.0                     # the smallest magnitude that rounds to inf in fp16
TILE, MATCH_THREADS = 16, 256              # seg_proto_kernel's pixel tile, seg_match_kernel's block

MUTATIONS = (
    "edge_inclusive",     # crop keeps r <= x2, c <= y2
    "floor",              # crop bounds floor(x1), floor(x2) instead of ceil
    "swap_hw",            # mh and mw swapped in the crop bounds
    "tidx_own_image",     # overlap tidx = the row's rank inside its image, not the value at its position
    "mean_crop_pixels",   # crop mean over the crop's pixel count instead of mh * mw
    "mean_per_image",     # one mean per image over all levels instead of per (level, image)
    "nearest_round",      # nearest-neighbour source index rounded instead of floored
)


# ---------------------------------------------------------------------------------------------------------------------
# index work (fp32, as the reference)
# ---------------------------------------------------------------------------------------------------------------------
def targets_for(targets, anchors, shapes, batch, overlap, nc, anchor_t=4.0, mutate=()):
    """build_targets_seg + loss64_ref.match_cells.  Rows the device loss ignores (class outside [0, nc), image outside
    [0, batch)) are dropped after the fact, so tidx stays the global row in non-overlap mode."""
    tg = np.asarray(targets, np.float32).reshape(-1, 6)
    anc = np.asarray(anchors, np.float32)
    bt = seg_loss_ref.build_targets_seg(tg, anc, shapes, batch, overlap, anchor_t)
    if "tidx_own_image" in mutate and overlap:
        rows = seg_loss_ref.build_targets_seg(tg, anc, shapes, batch, False, anchor_t)
        own = np.zeros(len(tg), np.int64)
        seen = {}
        for r, b in enumerate(tg[:, 0].astype(np.int64)):
            seen[b] = seen.get(b, 0) + 1
            own[r] = seen[b]
        for d, dr in zip(bt, rows):
            d["tidx"] = own[dr["tidx"]]
    for d in bt:
        keep = (d["b"] >= 0) & (d["b"] < batch) & (d["tcls"] >= 0) & (d["tcls"] < nc)
        if not keep.all():
            for k in ("tcls", "tbox", "b", "a", "gj", "gi", "anch", "tidx", "xywhn"):
                d[k] = d[k][keep]
    return R.match_cells(bt, shapes, batch, anc.shape[1])


def crop_xyxy(xywhn, mh, mw, mutate=()):
    """mxyxy = xywh2xyxy(xywhn * [mw, mh, mw, mh]) in fp32 (n, 4)."""
    g = (mh, mw, mh, mw) if "swap_hw" in mutate else (mw, mh, mw, mh)
    xy = torch.from_numpy(np.asarray(xywhn, np.float32)).reshape(-1, 4) * torch.tensor(g, dtype=torch.float32)
    return torch.cat((xy[:, :2] - xy[:, 2:] / 2, xy[:, :2] + xy[:, 2:] / 2), 1)


def crop_pixels(mxyxy, mh, mw):
    """The integer crop [x0, x1) x [y0, y1) of every box, clipped to the map: (n, 4) int64 x0, x1, y0, y1."""
    c = torch.ceil(mxyxy.double())
    x = c[:, [0, 2]].clamp(0, mw).long()
    y = c[:, [1, 3]].clamp(0, mh).long()
    return torch.stack((x[:, 0], x[:, 1], y[:, 0], y[:, 1]), 1)


def downsample(masks, mh, mw, mutate=()):
    """masks (N, H, W) -> float32 (N, mh, mw), F.interpolate(mode="nearest") as the reference does it."""
    masks = masks.float()
    h, w = masks.shape[-2:]
    if (h, w) == (mh, mw):
        return masks
    if "nearest_round" in mutate:
        iy = torch.round(torch.arange(mh, dtype=torch.float32) * (np.float32(h) / np.float32(mh))).long().clamp(max=h - 1)
        ix = torch.round(torch.arange(mw, dtype=torch.float32) * (np.float32(w) / np.float32(mw))).long().clamp(max=w - 1)
        return masks[:, iy.to(masks.device)][:, :, ix.to(masks.device)]
    return F.interpolate(masks[None], (mh, mw), mode="nearest")[0]


# ---------------------------------------------------------------------------------------------------------------------
# the mask term in closed form
# ---------------------------------------------------------------------------------------------------------------------
def mask64(bt, coef, proto, gt, overlap, box, scale=1.0, mutate=(), chunk=128):
    """bt: `targets_for` output; coef: per level (n_l, nm) float64 mask coefficients of every match; proto (B, nm, mh, mw)
    float64; gt (N, mh, mw) float32 downsampled masks (all on one device).

    Returns dict: lseg (sum over (level, image) of the mean crop loss, before box / B); per level (n_l, ...) dcoef,
    acoef, ecoef, npix, crop; per image gproto, aproto, eproto (B, nm, mh, mw), ncover (B, mh, mw); and nimg (nl, B)."""
    dev = proto.device
    B, nm, mh, mw = proto.shape
    hw = mh * mw
    nl = len(bt)
    lvl = torch.cat([torch.full((len(d["b"]),), i, dtype=torch.int64) for i, d in enumerate(bt)])
    b = torch.cat([torch.from_numpy(d["b"]) for d in bt])
    tidx = torch.cat([torch.from_numpy(d["tidx"]) for d in bt])
    xywhn = np.concatenate([d["xywhn"] for d in bt]) if len(b) else np.zeros((0, 4), np.float32)
    mxyxy = crop_xyxy(xywhn, mh, mw, mutate)
    marea = torch.from_numpy(xywhn[:, 2:]).prod(1)  # fp32, as the reference
    cf = torch.cat([c.to(dev, torch.float64) for c in coef]) if len(b) else torch.zeros(0, nm, dtype=torch.float64, device=dev)
    nimg = torch.zeros(nl, B, dtype=torch.int64)
    nimg.index_put_((lvl, b), torch.ones_like(b), accumulate=True)
    n = nimg.sum(0)[b] if "mean_per_image" in mutate else nimg[lvl, b]
    n_all = len(b)
    dcoef, acoef, ecoef = (torch.zeros(n_all, nm, dtype=torch.float64, device=dev) for _ in range(3))
    npix = torch.zeros(n_all, dtype=torch.int64, device=dev)
    gproto, aproto, eproto = (torch.zeros(B, nm, hw, dtype=torch.float64, device=dev) for _ in range(3))
    ncover = torch.zeros(B, hw, dtype=torch.int64, device=dev)
    r = torch.arange(mw, dtype=torch.float64, device=dev)
    c = torch.arange(mh, dtype=torch.float64, device=dev)
    gtf = gt.reshape(gt.shape[0], hw)
    lseg = 0.0
    for bi in range(B):
        sel = torch.nonzero(b == bi).flatten()
        P = proto[bi].reshape(nm, hw)
        Pa = P.abs()
        for s0 in range(0, len(sel), chunk):
            j = sel[s0:s0 + chunk]
            jd = j.to(dev)
            cj = cf[jd]
            x = cj @ P
            xy = mxyxy[j].to(dev, torch.float64)
            if "floor" in mutate:
                xy = torch.floor(xy)
            x1, y1, x2, y2 = (xy[:, k:k + 1] for k in range(4))
            if "edge_inclusive" in mutate:
                inside = ((r >= x1) & (r <= x2))[:, None, :] & ((c >= y1) & (c <= y2))[:, :, None]
            else:
                inside = ((r >= x1) & (r < x2))[:, None, :] & ((c >= y1) & (c < y2))[:, :, None]
            inside = inside.reshape(len(j), hw)
            if overlap:
                t = (gtf[bi][None] == tidx[j].to(dev, torch.float32)[:, None]).double()
            else:
                t = gtf[tidx[j].to(dev)].double()
            npj = inside.sum(1)
            area = marea[j].to(dev, torch.float64)
            denom = npj.clamp_min(1).double() if "mean_crop_pixels" in mutate else float(hw)
            bce = F.binary_cross_entropy_with_logits(x, t, reduction="none") * inside
            lseg += float((bce.sum(1) / denom / area / n[j].to(dev).double()).sum())
            s = scale * box / n[j].to(dev).double() / denom / area
            sig = torch.sigmoid(x)
            g = (sig - t) * inside * s[:, None]
            X = cj.abs() @ Pa
            E = (7 * g.abs() + s[:, None] * (sig * (1 - sig) * (2 + 1.2 * x.abs() + nm * X) + 3 * sig)) * inside
            dcoef[jd] = g @ P.T
            acoef[jd] = g.abs() @ Pa.T
            ecoef[jd] = E @ Pa.T
            npix[jd] = npj
            gproto[bi] += cj.T @ g
            aproto[bi] += cj.abs().T @ g.abs()
            eproto[bi] += cj.abs().T @ E
            ncover[bi] += inside.sum(0)
    crop = crop_pixels(mxyxy, mh, mw)
    split = [len(d["b"]) for d in bt]
    out = dict(lseg=lseg, nimg=nimg, gproto=gproto.view(B, nm, mh, mw), aproto=aproto.view(B, nm, mh, mw),
               eproto=eproto.view(B, nm, mh, mw), ncover=ncover.view(B, mh, mw))
    for k, v in (("dcoef", dcoef), ("acoef", acoef), ("ecoef", ecoef), ("npix", npix), ("crop", crop)):
        out[k] = list(torch.split(v, split))
    return out


def reference(p, proto, targets, masks, overlap, hyp, dtype=None, scale=1.0, anchors=None, mutate=(), chunk=128):
    """The whole segmentation loss in float64 on the inputs as given (head maps (B, na, ny, nx, 5 + nc + nm) and proto
    already in the logits dtype, on any device; masks (N, H, W) in any dtype).  The mask term runs on proto's device.

    Returns dict: loss, items (4,) [lbox, lseg, lobj, lcls]; per level gobj (B, na, ny, nx), grows / arows (u, no) and
    frows (u, nm) -- the fp32 error bound of the mask channels, u32 * sum_j (k_j acoef_j + ecoef_j); gproto, aproto,
    eproto, ncover; bt and the mask-term details (`mask`)."""
    dtype = dtype or p[0].dtype
    anchors = mg.anchors_grid().numpy() if anchors is None else np.asarray(anchors, np.float32)
    B, nm, mh, mw = proto.shape
    no = p[0].shape[-1]
    nc = no - 5 - nm
    shapes = [tuple(t.shape[2:4]) for t in p]
    tg = targets.detach().cpu().numpy() if isinstance(targets, torch.Tensor) else np.asarray(targets, np.float32)
    bt = targets_for(tg, anchors, shapes, B, overlap, nc, hyp["anchor_t"], mutate)
    obj, rows = R.leaves_from_maps(p, bt)
    det = R.loss64(obj, [q[:, : 5 + nc] for q in rows], bt, hyp, nc, B, dtype=dtype, scale=scale)
    dev = proto.device
    gt = downsample(masks.to(dev), mh, mw, mutate)
    coef = [q[d["inv"]][:, 5 + nc:] for q, d in zip(rows, bt)]
    m = mask64(bt, coef, proto.detach().to(torch.float64), gt, overlap, hyp["box"], scale, mutate, chunk)
    lseg = m["lseg"] * hyp["box"] / B
    lbox, lobj, lcls = (float(v) for v in det["items"])
    res = dict(loss=(lbox + lobj + lcls + lseg) * B, items=torch.tensor([lbox, lseg, lobj, lcls], dtype=torch.float64),
               gobj=det["gobj"], grows=[], arows=[], frows=[], tobj=det["tobj"], bt=bt, mask=m, dtype=dtype, scale=scale,
               hyp=dict(hyp), batch=B, nc=nc, nm=nm, gproto=m["gproto"], aproto=m["aproto"], eproto=m["eproto"],
               ncover=m["ncover"])
    for i, d in enumerate(bt):
        u = len(d["ucell"])
        inv = d["inv"].to(dev)
        k = (torch.ceil(m["npix"][i].double() / MATCH_THREADS) + 5 + 8)[:, None]  # serial per thread, warp tree, 8 warps
        gm = torch.zeros(u, nm, dtype=torch.float64, device=dev).index_add_(0, inv, m["dcoef"][i]).cpu()
        am = torch.zeros(u, nm, dtype=torch.float64, device=dev).index_add_(0, inv, m["dcoef"][i].abs()).cpu()
        fm = torch.zeros(u, nm, dtype=torch.float64, device=dev).index_add_(0, inv, U32 * (k * m["acoef"][i] + m["ecoef"][i])).cpu()
        gd = det["grows"][i] if det["grows"][i].numel() else torch.zeros(u, 5 + nc, dtype=torch.float64)
        ad = det["arows"][i] if det["arows"][i].numel() else torch.zeros(u, 5 + nc, dtype=torch.float64)
        res["grows"].append(torch.cat((gd, gm), 1))
        res["arows"].append(torch.cat((ad, am), 1))
        res["frows"].append(fm)
    return res


# ---------------------------------------------------------------------------------------------------------------------
# the bounds
# ---------------------------------------------------------------------------------------------------------------------
def _ulp(t, dtype):
    return 2 * U[dtype] * torch.exp2(torch.floor(torch.log2(t.clamp_min(torch.finfo(dtype).tiny))))


def _ratio(got, ref, bound, dtype, reach=None):
    """max err / bound; err 0 needs bound 0 or more.  fp16: where the float64 value rounds to inf the kernel must give inf of
    the same sign; an inf is also accepted where the reference plus its bound (or `reach`, the sum of the absolute
    contributions) reaches the overflow threshold."""
    got, ref, bound = got.double(), ref.double().to(got.device), bound.double().to(got.device)
    err = (got - ref).abs()
    if dtype == F16:
        reach = (ref.abs() + bound) if reach is None else torch.maximum(ref.abs() + bound, reach.double().to(got.device))
        ok_inf = torch.isinf(got) & (torch.sign(got) == torch.sign(ref)) & (reach >= F16_OVERFLOW)
        err = torch.where(ok_inf, torch.zeros_like(err), err)
        err = torch.where((ref.abs() >= F16_OVERFLOW) & ~ok_inf, torch.full_like(err, math.inf), err)
    err = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err)
    r = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    return float(r.max()) if r.numel() else 0.0


def ratios(got, ref):
    """[(where, term, worst err / bound)] of a result `got` against the reference `ref` (`reference`'s output).

    got: dict loss (float), items (4,) [lbox, lseg, lobj, lcls], obj per level (B, na, ny, nx), rows per level (u, no) at
    ref's unique matched cells, proto (B, nm, mh, mw), outside (number of nonzero gradient elements outside the objectness
    channel and the matched cells; 0 if not given).

    Bounds (u_D: unit roundoff of the logits dtype, u32: fp32's, S: the largest |ref| of that level and term, z_D: half the
    fp16 subnormal spacing, m: matches of the cell, A: the sum of their absolute contributions):
    - loss and items: 2e-5 |ref| + 1e-7;
    - obj, xy, wh, cls: the detection suite's bounds (u_D |ref| + 1e-5 S + z_D, one dtype ulp of tobj at matched cells;
      m u_D A + 1e-5 S + z_D);
    - mask channels of matched cells: sum_j u32 (k_j acoef_j + ecoef_j) + m u_D A + 1e-5 S + z_D, k_j = ceil(npix_j / 256)
      + 5 + 8 (seg_match's per-thread serial sum over the crop, the warp shuffle tree, the serial sum of the 8 warps);
    - dproto: u_D |ref| + (n_cover + 1) u32 aproto + u32 eproto + z_D where n_cover > 0 (seg_proto's one FMA per covering
      match, then one rounding to the proto dtype), and exactly 0 where no crop of the image covers the pixel;
    - everything else exactly 0."""
    dtype, hyp, B = ref["dtype"], ref["hyp"], ref["batch"]
    u, z = U[dtype], Z[dtype]
    nc = ref["nc"]
    out = []
    g = torch.cat((torch.tensor([float(got["loss"])], dtype=torch.float64), torch.as_tensor(got["items"]).double().cpu()))
    e = torch.cat((torch.tensor([ref["loss"]], dtype=torch.float64), ref["items"]))
    out.append(("all", "loss", _ratio(g, e, 2e-5 * e.abs() + 1e-7, F32)))
    out.append(("all", "outside", math.inf if got.get("outside", 0) else 0.0))
    pwf = max(1.0, hyp["obj_pw"])
    terms = (("xy", slice(0, 2)), ("wh", slice(2, 4)), ("cls", slice(5, 5 + nc)), ("mask", slice(5 + nc, None)))
    for l, d in enumerate(ref["bt"]):
        go, gr = got["obj"][l].double().cpu().reshape(-1), ref["gobj"][l].reshape(-1)
        gs = hyp["obj"] * R.BALANCE[l] * B * ref["scale"] / d["cells"]
        bound = u * gr.abs() + 1e-5 * float(gr.abs().max()) + z
        if len(d["ucell"]):
            bound[d["ucell"]] += pwf * gs * _ulp(ref["tobj"][l], dtype)
        out.append((f"P{l + 3}", "obj", _ratio(go, gr, bound, dtype)))
        grow, erow, arow = got["rows"][l].double().cpu(), ref["grows"][l], ref["arows"][l]
        m = d["mult"].double()[:, None]
        for term, sl in terms:
            ev, av = erow[:, sl], arow[:, sl]
            s = float(ev.abs().max()) if ev.numel() else 0.0
            bound = m * u * av + 1e-5 * s + z
            if term == "mask":
                bound = bound + ref["frows"][l]
            out.append((f"P{l + 3}", term, _ratio(grow[:, sl], ev, bound, dtype, reach=av)))
    gp, rp = got["proto"], ref["gproto"]
    gp = gp.to(rp.device)
    cover = ref["ncover"][:, None].expand_as(rp)
    bound = u * rp.abs() + (cover + 1) * U32 * ref["aproto"] + U32 * ref["eproto"] + z
    bound = torch.where(cover > 0, bound, torch.zeros_like(bound))
    out.append(("proto", "proto", _ratio(gp, rp, bound, dtype)))
    return out


def check(got, ref):
    """The worst err / bound of `ratios`: <= 1 passes."""
    return max(r for _, _, r in ratios(got, ref))


def as_got(res):
    """A reference result in the form `ratios` takes for the kernel's (for checking one reference against another)."""
    return dict(loss=res["loss"], items=res["items"], obj=res["gobj"], rows=res["grows"], proto=res["gproto"], outside=0)


# ---------------------------------------------------------------------------------------------------------------------
# cases: numpy inputs (fp32 head maps and proto, targets, masks) at the shapes segmentation trains with
# ---------------------------------------------------------------------------------------------------------------------
def _case(batch, h, w, tg, masks, overlap, nc=80, nm=32, seed=0, proto_std=0.5, ratio=4):
    rs = np.random.RandomState(seed)
    p = [rs.normal(0, 1.5, (batch, 3, h // s, w // s, 5 + nc + nm)).astype(np.float32) for s in (8, 16, 32)]
    proto = rs.normal(0, proto_std, (batch, nm, h // 4, w // 4)).astype(np.float32)
    return dict(p=p, proto=proto, targets=np.asarray(tg, np.float32), masks=masks, overlap=overlap, nc=nc, nm=nm)


def _holes(masks, rs):
    return (masks * (rs.uniform(size=masks.shape) > 0.2)).astype(np.float32)


def training_case(batch=16, size=640, seed=201, mask_dtype=np.float32):
    """batch x size^2, nc 80, nm 32, synth_targets, overlap masks at size / 4 (train.py's defaults)."""
    from oracle import loss_ref

    tg = loss_ref.synth_targets(batch, seed=seed)
    masks = seg_loss_ref.overlap_masks(tg, batch, size // 4, size // 4).astype(mask_dtype)
    return _case(batch, size, size, tg, masks, True, seed=seed + 1)


def no_overlap_case(batch=16, size=640, seed=211):
    """--no-overlap: one (size / 4)^2 mask per target row, each its box with ~20 % holes."""
    from oracle import loss_ref

    tg = loss_ref.synth_targets(batch, seed=seed)
    rs = np.random.RandomState(seed + 2)
    m = size // 4
    masks = _holes(np.stack([seg_loss_ref.paint_masks((m, m), tg[i:i + 1, 2:6], [1.0]) for i in range(len(tg))]), rs)
    return _case(batch, size, size, tg, masks, False, seed=seed + 1)


def mask_ratio_case(ratio, batch=16, size=640, seed=221):
    """Overlap masks at size / ratio for a size / 4 proto: ratio 1 downsamples by 4, ratio 8 upsamples by 2."""
    from oracle import loss_ref

    tg = loss_ref.synth_targets(batch, seed=seed)
    masks = seg_loss_ref.overlap_masks(tg, batch, size // ratio, size // ratio)
    return _case(batch, size, size, tg, masks, True, seed=seed + 1)


def rect_case(batch, h, w, seed=231):
    """A rectangular batch (val.py / --rect): maps h/8 x w/8 ..., proto and masks h/4 x w/4."""
    from oracle import loss_ref

    tg = loss_ref.synth_targets(batch, seed=seed)
    masks = seg_loss_ref.overlap_masks(tg, batch, h // 4, w // 4)
    return _case(batch, h, w, tg, masks, True, seed=seed + 1)


def crowded_case(batch=4, per_image=300, size=640, seed=241, mask_dtype=np.int32):
    """`per_image` small boxes per image: overlap indices past 255 (the loader's masks are int32 then), tens of matches per
    proto tile and many rounds of seg_match's grid-stride loop."""
    tg = R.crowded_targets(batch, per_image, size, seed=seed)
    masks = seg_loss_ref.overlap_masks(tg, batch, size // 4, size // 4).astype(mask_dtype)
    return _case(batch, size, size, tg, masks, True, seed=seed + 1)


# 640 x 640, proto 160 x 160 (4 image pixels per proto pixel, 8 per P3 cell).  Dyadic positions keep
# (t * nx) / nx == t and the crop bounds exact in fp32.
SMALLEST_P3 = (2.75 / 640, 3.5 / 640)  # just above a quarter of P3 anchor 0 (10 x 13 px): one anchor passes


def edge_targets():
    """Image 0: crops with integer edges on the 160^2 proto (x1 = 60, x2 = 100, ...), boxes over the map border (clipped),
    a box whose crop holds no pixel; image 1: the smallest box P3 matches, alone at P3 and centred in its cell (one
    match: the largest mask-gradient scale there is), plus boxes only P4 / P5 match."""
    sw, sh = SMALLEST_P3
    rows = [
        [0, 1, 0.5, 0.5, 0.25, 0.25],          # crop [60, 100) x [60, 100): integer edges
        [0, 2, 0.375, 0.625, 0.125, 0.0625],   # [50, 70) x [95, 105)
        [0, 3, 0.25, 0.125, 0.09375, 0.15625], # [32.5, 47.5) x [7.5, 32.5)
        [0, 4, 0.015625, 0.5, 0.0625, 0.1],    # x1 = -2.5: over the left border
        [0, 5, 0.984375, 0.9875, 0.0625, 0.05],  # over the right and bottom borders
        [0, 6, 42 / 640, 200 / 640, sw, sh],   # proto x 10.5: [10.16, 10.84) holds no pixel column
        [0, 7, 0.8, 0.2, 0.3, 0.2],
        [1, 8, 0.15625, 0.15625, sw, sh],      # P3 cell (12, 12) centre: one match, proto pixel (25, 25)
        [1, 9, 0.7, 0.7, 0.5, 0.5],            # P5 only
        [1, 10, 0.75, 0.3, 0.25, 0.25],        # P4 and P5
    ]
    return np.array(rows, np.float32)


def edges_case(seed=251):
    tg = edge_targets()
    masks = seg_loss_ref.overlap_masks(tg, 2, 160, 160)
    c = _case(2, 640, 640, tg, masks, True, seed=seed)
    # the smallest box's cell (P3 anchor 0, cell (12, 12) of image 1) and its one proto pixel: logit -16 against gt 1, so
    # g ~ -s, with |proto| 2 in the even channels and |coef| 2 in the odd ones, so that under a GradScaler-sized scale
    # dcoef (g * proto) and dproto (g * coef) both pass the fp16 range
    sign = np.where(c["proto"][1, :, 25, 25] >= 0, 1.0, -1.0).astype(np.float32)
    big = np.arange(c["nm"]) % 2 == 0
    c["proto"][1, :, 25, 25] = sign * np.where(big, 2.0, 0.25)
    c["p"][0][1, 0, 12, 12, 5 + c["nc"]:] = -sign * np.where(big, 0.25, 2.0)
    return c


def batch_layout_case(batch=8, size=320, seed=261, empty=(0, 3, 7), mask_dtype=np.uint8):
    """Images without labels first, in the middle and last; targets shuffled, so an overlap tidx is the value at the row's
    position in cat([1..n_0, 1..n_1, ...]), not its rank in its image."""
    from oracle import loss_ref

    tg = loss_ref.synth_targets(batch, seed=seed)
    tg = tg[~np.isin(tg[:, 0], empty)]
    tg = tg[np.random.RandomState(seed + 2).permutation(len(tg))]
    masks = seg_loss_ref.overlap_masks(tg, batch, size // 4, size // 4).astype(mask_dtype)
    return _case(batch, size, size, tg, masks, True, seed=seed + 1)


def nm_case(nm, nc, batch=4, h=256, w=320, seed=271):
    from oracle import loss_ref

    tg = loss_ref.synth_targets(batch, seed=seed, nc=nc)
    masks = seg_loss_ref.overlap_masks(tg, batch, h // 4, w // 4)
    return _case(batch, h, w, tg, masks, True, nc=nc, nm=nm, seed=seed + 1)


def invalid_rows_case(batch=4, size=320, seed=281, nc=80):
    """Non-overlap, with rows of class >= nc and image >= batch in the middle: the device loss ignores them, but they keep
    their mask slot, so tidx is still the row in the full target list.  `ref_targets` is None: the reference drops the
    rows itself."""
    from oracle import loss_ref

    good = loss_ref.synth_targets(batch, seed=seed, nc=nc)
    bad = np.array([[0, nc, 0.5, 0.5, 0.2, 0.2], [batch, 0, 0.5, 0.5, 0.2, 0.2], [1, nc + 3, 0.3, 0.6, 0.1, 0.3]], np.float32)
    k = len(good) // 2
    tg = np.concatenate((good[:k], bad, good[k:]))
    rs = np.random.RandomState(seed + 2)
    m = size // 4
    masks = _holes(np.stack([seg_loss_ref.paint_masks((m, m), tg[i:i + 1, 2:6], [1.0]) for i in range(len(tg))]), rs)
    return _case(batch, size, size, tg, masks, False, nc=nc, seed=seed + 1)
