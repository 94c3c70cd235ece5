"""Generate tests/golden/seg_loss.npz and seg_signatures.json by running the UNMODIFIED reference's segmentation loss
(reference utils/segment/loss.py) through tests/golden/refshim.py.

Runs only where the reference tree exists:
    python tests/golden/make_seg_golden.py
The inputs of every case are regenerated from the seed and shapes listed in `CASES` below (tests/test_seg_loss_*.py
call `case_inputs`), so seg_loss.npz holds only the reference's outputs.  While generating, the oracle
(tests/seg_loss_ref.py) is checked against the reference (hard assert).
"""
from __future__ import annotations

import inspect
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from oracle import loss_ref  # noqa: E402
from tests import seg_loss_ref  # noqa: E402
from yolov5_b200.cfg import HYP_SCRATCH_LOW  # noqa: E402

NM = 32
STRIDES = (8, 16, 32)
ANCHORS_PX = ((10, 13, 16, 30, 33, 23), (30, 61, 62, 45, 59, 119), (116, 90, 156, 198, 373, 326))
# tag: (bs, img h, img w, mask h, mask w, nc, overlap, order, seed); proto is (bs, 32, h/4, w/4)
CASES = {
    "ov_sorted": (2, 64, 64, 16, 16, 80, True, "sorted", 51),
    "ov_unsorted": (3, 64, 64, 16, 16, 80, True, "shuffled", 52),
    "nonov": (2, 64, 64, 16, 16, 80, False, "sorted", 53),
    "ov_x4": (2, 64, 64, 64, 64, 80, True, "sorted", 54),
    "nonov_frac": (2, 64, 64, 24, 40, 80, False, "shuffled", 55),
    "edges": (2, 64, 64, 16, 16, 80, True, "edges", 56),
    "nc1": (2, 64, 64, 16, 16, 1, False, "sorted", 57),
    "none": (2, 64, 64, 16, 16, 80, True, "none", 58),
    "grid12": (2, 96, 96, 24, 24, 80, True, "sorted", 59),  # grids 12 / 6 / 3: (t * nx) / nx differs from t
}


def anchors_grid():
    """(nl, na, 2) anchors in grid units, as Detect stores them."""
    a = torch.tensor(ANCHORS_PX, dtype=torch.float32).view(3, 3, 2)
    return a / torch.tensor(STRIDES, dtype=torch.float32).view(3, 1, 1)


class _Head(torch.nn.Module):
    def __init__(self, nc):
        super().__init__()
        self.na, self.nc, self.nl, self.nm = 3, nc, 3, NM
        self.register_buffer("anchors", anchors_grid())
        self.stride = torch.tensor(STRIDES, dtype=torch.float32)


class LossModel(torch.nn.Module):
    """The attributes ComputeLoss reads from a model: .hyp, .parameters() and the head model[-1]."""

    def __init__(self, nc):
        super().__init__()
        self.model = torch.nn.ModuleList([_Head(nc)])
        self.w = torch.nn.Parameter(torch.zeros(1))
        self.hyp = dict(HYP_SCRATCH_LOW)


def case_inputs(tag):
    """(p list of fp32 numpy (bs,3,ny,nx,5+nc+32), proto (bs,32,mh,mw), targets (nt,6), masks (N,H,W), overlap, nc)."""
    bs, h, w, gh, gw, nc, overlap, order, seed = CASES[tag]
    rs = np.random.RandomState(seed)
    no = 5 + nc + NM
    p = [rs.normal(0, 1.5, (bs, 3, h // s, w // s, no)).astype(np.float32) for s in STRIDES]
    proto = rs.normal(0, 0.5, (bs, NM, h // 4, w // 4)).astype(np.float32)
    if order == "none":
        tg = np.zeros((0, 6), np.float32)
    else:
        tg = loss_ref.synth_targets(bs, seed, nc)
        big = np.array([[0, 0, 0.5, 0.5, 0.7, 0.6], [bs - 1, 0, 0.45, 0.55, 0.5, 0.8]], np.float32)  # P4 / P5 matches
        tg = np.concatenate((tg, big), 0)
        tg = tg[np.argsort(tg[:, 0], kind="stable")]
        if order == "edges":  # crop edges exactly on integer pixels at 16x16 (x1 = 6, x2 = 10, y1 = 4, y2 = 8)
            extra = np.array([[0, 0, 0.5, 0.375, 0.25, 0.25], [1, 0, 0.25, 0.5, 0.125, 0.5]], np.float32)
            tg = np.concatenate((tg, extra), 0)
            tg = tg[np.argsort(tg[:, 0], kind="stable")]
        if order == "shuffled":
            tg = tg[rs.permutation(len(tg))]
    nt = len(tg)
    if overlap:
        masks = seg_loss_ref.overlap_masks(tg, bs, gh, gw)
    else:
        masks = np.stack([seg_loss_ref.paint_masks((gh, gw), tg[i:i + 1, 2:6], [1.0]) * (rs.uniform(size=(gh, gw)) > 0.2)
                          for i in range(nt)]) if nt else np.zeros((0, gh, gw), np.float32)
        masks = masks.astype(np.float32)
    return p, proto, tg, masks, overlap, nc


def gen_segloss():
    sys.path.insert(0, HERE)
    import refshim

    refshim.install()
    from utils.segment.loss import ComputeLoss

    store = {}
    for tag in CASES:
        p_np, proto_np, tg, masks, overlap, nc = case_inputs(tag)
        bs = p_np[0].shape[0]
        crit = ComputeLoss(LossModel(nc), overlap=overlap)
        p = [torch.from_numpy(a).requires_grad_(True) for a in p_np]
        proto = torch.from_numpy(proto_np).requires_grad_(True)
        loss, items = crit((p, proto), torch.from_numpy(tg), masks=torch.from_numpy(masks))
        loss.backward()
        bt = crit.build_targets(p, torch.from_numpy(tg))
        anchors = anchors_grid().numpy()
        orc = seg_loss_ref.build_targets_seg(tg, anchors, [tuple(a.shape[2:4]) for a in p_np], bs, overlap)
        for i in range(3):
            tcls, tbox, idx, anch, tidx, xywhn = (x[i] for x in bt)
            assert tidx.dtype == torch.int64 and all(t.dtype == torch.int64 for t in idx)
            assert np.array_equal(tidx.numpy(), orc[i]["tidx"]), (tag, i)
            assert np.array_equal(xywhn.numpy(), orc[i]["xywhn"]), (tag, i)
            assert np.array_equal(tbox.numpy(), orc[i]["tbox"]) and np.array_equal(tcls.numpy(), orc[i]["tcls"]), (tag, i)
            for q, k in enumerate(("b", "a", "gj", "gi")):
                assert np.array_equal(idx[q].numpy(), orc[i][k]), (tag, i, k)
            store[f"{tag}.idx{i}"] = np.stack([idx[q].numpy() for q in range(4)] + [tcls.numpy(), tidx.numpy()])
            store[f"{tag}.tbox{i}"] = tbox.numpy()
            store[f"{tag}.anch{i}"] = anch.numpy()
            store[f"{tag}.xywhn{i}"] = xywhn.numpy()
        for fn in (seg_loss_ref.compute_seg_loss, seg_loss_ref.compute_seg_loss_torch):
            p2 = [torch.from_numpy(a).requires_grad_(True) for a in p_np]
            proto2 = torch.from_numpy(proto_np).requires_grad_(True)
            lo, it = fn(p2, proto2, torch.from_numpy(tg), torch.from_numpy(masks), anchors_grid(), HYP_SCRATCH_LOW, overlap)
            lo.backward()
            assert torch.allclose(loss, lo, rtol=1e-5, atol=1e-6), (tag, fn.__name__, loss, lo)
            assert torch.allclose(items, it, rtol=1e-5, atol=1e-6), (tag, fn.__name__, items, it)
            for a, b in zip(p + [proto], p2 + [proto2]):
                for t in (a, b):
                    if t.grad is None:  # no match: the mask term never touches proto
                        t.grad = torch.zeros_like(t)
                assert torch.allclose(a.grad, b.grad, rtol=1e-4, atol=1e-7), (tag, fn.__name__, (a.grad - b.grad).abs().max())
        store[f"{tag}.loss"] = np.concatenate((loss.detach().numpy(), items.numpy()))
        for i, a in enumerate(p):
            store[f"{tag}.grad{i}"] = a.grad.numpy()
        store[f"{tag}.grad_proto"] = proto.grad.numpy()
        print(f"seg loss {tag}: {loss.item():.6f} items {items.tolist()} matches {[len(d['b']) for d in orc]}; oracle == reference")
    np.savez_compressed(f"{HERE}/seg_loss.npz", **store)
    sig = {name: [(n, repr(q.default) if q.default is not inspect._empty else None, str(q.kind))
                  for n, q in inspect.signature(getattr(ComputeLoss, name)).parameters.items()]
           for name in ("__init__", "__call__", "build_targets")}
    with open(f"{HERE}/seg_signatures.json", "w") as f:
        json.dump(sig, f, indent=1, sort_keys=True)
    print("written", f"{HERE}/seg_loss.npz", os.path.getsize(f"{HERE}/seg_loss.npz"), "bytes")


if __name__ == "__main__":
    which = sys.argv[1:] or ["segloss"]
    for w in which:
        {"segloss": gen_segloss}[w]()
