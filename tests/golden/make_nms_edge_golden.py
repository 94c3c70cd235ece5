"""Generate tests/golden/nms_edges.npz by running the UNMODIFIED reference's non_max_suppression (utils/general.py:658-767)
on the regimes tests/golden/nms.npz leaves out, one image per call (as make_golden.py::gen_nms does):

- bf16 in val.py's regime (conf 0.001, multi-label, the max_nms = 30000 cut) and segment/val.py's (the same with nm = 32),
  where the threshold is rounded to bf16 and coarse scores tie at the cut;
- 1280-pixel inputs (100800 rows) in single-label mode, where the cut runs on ~90000 best-class candidates;
- small hand-built inputs with non-finite values: NaN class scores (single- and multi-label), NaN objectness, +inf and
  -inf class scores, inf objectness times a zero class score (a NaN product), NaN / inf box coordinates, and zero or
  negative widths and heights.

Runs only where the reference tree exists:
    python tests/golden/make_nms_edge_golden.py
The synthetic inputs are regenerated from the seeds in `meta` by oracle.nms_ref.synth_predictions; the hand-built inputs are
small and stored as `<tag>.pred`.  While generating, the oracle is checked against the reference (hard assert, see `check`);
the oracle's rows are what the fixture stores, and each case's `pinned` says how closely the reference agreed.
"""
from __future__ import annotations

import contextlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden import canon_ties, run_ref_nms  # noqa: E402  (installs the reference shim)

import torch  # noqa: E402

from oracle import nms_ref  # noqa: E402

SYNTH = [
    dict(tag="val_bf16", bs=2, n=25200, nc=80, nm=0, seed=31, dtype="bf16", img=640.0,
         kw=dict(conf_thres=0.001, iou_thres=0.6, multi_label=True, max_det=300)),
    dict(tag="segval_bf16", bs=2, n=25200, nc=80, nm=32, seed=32, dtype="bf16", img=640.0,
         kw=dict(conf_thres=0.001, iou_thres=0.6, multi_label=True, max_det=300, nm=32)),
    dict(tag="segval_fp16", bs=1, n=25200, nc=80, nm=32, seed=33, dtype="fp16", img=640.0,
         kw=dict(conf_thres=0.001, iou_thres=0.6, multi_label=True, max_det=300, nm=32)),
    dict(tag="p1280_fp32", bs=1, n=100800, nc=80, nm=0, seed=34, dtype="fp32", img=1280.0,
         kw=dict(conf_thres=0.001, iou_thres=0.45, max_det=1000)),
    dict(tag="p1280_fp16", bs=1, n=100800, nc=80, nm=0, seed=35, dtype="fp16", img=1280.0,
         kw=dict(conf_thres=0.001, iou_thres=0.45, max_det=1000)),
    dict(tag="p1280_bf16", bs=1, n=100800, nc=80, nm=0, seed=36, dtype="bf16", img=1280.0,
         kw=dict(conf_thres=0.001, iou_thres=0.45, max_det=1000)),
]


def _base(rs, n, nc):
    """n well-separated boxes on a grid (nothing overlaps), obj in [0.6, 1], one clear best class per row in [0.6, 1]."""
    x = np.zeros((n, 5 + nc), np.float32)
    x[:, 0] = 40.0 + 50.0 * (np.arange(n) % 16)
    x[:, 1] = 40.0 + 50.0 * (np.arange(n) // 16)
    x[:, 2:4] = rs.uniform(10, 30, (n, 2))
    x[:, 4] = rs.uniform(0.6, 1.0, n)
    x[:, 5:] = rs.uniform(0.0, 0.4, (n, nc))
    x[np.arange(n), 5 + rs.randint(0, nc, n)] = rs.uniform(0.6, 1.0, n)
    return x


def hand_cases():
    """(tag, x (n, 5+nc) fp32, [kw, ...]) for the non-finite and degenerate inputs, run in fp32, fp16 and bf16."""
    rs = np.random.RandomState(41)
    out = []
    # NaN class scores at every class position, so each of the 8 lanes of the kernel's best-class search sees one as its
    # first value (j < 8) and as a later value (j >= 8); the row's finite best class is above the threshold
    nc = 20
    x = _base(rs, 96, nc)
    for r in range(0, 96, 2):
        j = (r // 2) % nc
        x[r, 5 + j] = np.nan
    x[1, 5:] = np.nan  # every class NaN
    out.append(("nan_cls", x, [dict(conf_thres=0.25, iou_thres=0.45), dict(conf_thres=0.25, iou_thres=0.45, multi_label=True)]))
    # NaN objectness; inf objectness with some zero class scores (0 * inf = NaN in the product); +inf and -inf class scores
    x = _base(rs, 64, nc)
    x[0:6, 4] = np.nan
    x[6:10, 4] = np.inf
    x[6, 5 + 3] = 0.0
    x[7, 5:] = 0.0
    x[8, 5 + 11] = 0.0
    x[10:14, 5 + 2] = np.inf        # four +inf scores: ties at the top of the order
    x[14, 5:] = -np.inf             # all -inf: never a candidate
    x[15, 5 + 17] = -np.inf
    x[10:14, 0:2] = x[16, 0:2]       # the +inf rows overlap row 16 and each other
    x[16, 5 + 2] = 0.9
    out.append(("inf_obj_cls", x, [dict(conf_thres=0.25, iou_thres=0.45), dict(conf_thres=0.25, iou_thres=0.45, multi_label=True)]))
    # non-finite box coordinates, each overlapping a finite copy of itself in the same class
    x = _base(rs, 48, nc)
    for k, (col, v) in enumerate([(0, np.nan), (1, np.nan), (2, np.nan), (3, np.nan), (0, np.inf), (1, -np.inf),
                                  (2, np.inf), (3, np.inf), (0, -np.inf), (2, -np.inf)]):
        r, twin = 2 * k, 2 * k + 1
        x[twin] = x[r]
        x[twin, 4] = x[r, 4] * 0.8
        x[r, col] = v
    out.append(("nonfinite_box", x, [dict(conf_thres=0.25, iou_thres=0.45), dict(conf_thres=0.25, iou_thres=0.3, agnostic=True)]))
    # zero and negative widths / heights next to ordinary boxes of the same class and place: rows 0-15 rank the degenerate
    # box above its ordinary twin, rows 16-31 below it
    x = _base(rs, 48, nc)
    wh = [(0, 20), (20, 0), (0, 0), (-20, 20), (20, -20), (-20, -20), (-1, 30), (30, -1)]
    for k, (w, h) in enumerate(wh):
        r, twin = 2 * k, 2 * k + 1
        x[twin] = x[r]
        x[twin, 4] = x[r, 4] * 0.8
        x[r, 2:4] = (w, h)
        r, twin = 16 + 2 * k, 17 + 2 * k
        x[twin] = x[r]
        x[twin, 4] = x[r, 4] * 0.8
        x[twin, 2:4] = (w, h)
    out.append(("degenerate_box", x, [dict(conf_thres=0.25, iou_thres=0.45), dict(conf_thres=0.25, iou_thres=0.0)]))
    return out


def same(a, b):
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


@contextlib.contextmanager
def stable_argsort():
    """Tensor.argsort with stable=True: equal scores keep candidate order, the rule the oracle and the kernels define."""
    orig = torch.Tensor.argsort
    torch.Tensor.argsort = lambda self, dim=-1, descending=False: torch.sort(self, dim=dim, descending=descending, stable=True).indices
    try:
        yield
    finally:
        torch.Tensor.argsort = orig


def check(tag, pred, dtype, kw, orc):
    """The reference's argsort(descending=True) (utils/general.py:745) is not stable, so the order inside equal-score runs is
    implementation-defined there.  Equal-score runs are first compared in a canonical order.  Where the order also decides
    which tied boxes survive (one suppresses the other, or max_det cuts the run), the reference is run again with a stable
    argsort and must then agree; its score column must agree either way."""
    ref = run_ref_nms(pred, dtype, **kw)
    if all(same(r, o) for r, o in zip(ref, orc)):
        return "bit-exact"
    if all(same(canon_ties(r), canon_ties(o)) for r, o in zip(ref, orc)):
        return "exact up to the order inside equal-score runs"
    for b, (r, o) in enumerate(zip(ref, orc)):
        assert r.shape == o.shape and np.array_equal(r[:, 4], o[:, 4]), (tag, b)
    with stable_argsort():
        ref = run_ref_nms(pred, dtype, **kw)
    for b, (r, o) in enumerate(zip(ref, orc)):
        assert same(r, o), (tag, b)
    return "exact with the reference's argsort made stable; as it is, the same scores"


def main():
    store, meta = {}, []
    for c in SYNTH:
        pred = nms_ref.synth_predictions(c["bs"], c["n"], c["nc"], c["nm"], c["seed"], c["dtype"], img=c["img"])
        orc = nms_ref.non_max_suppression(pred, dtype=c["dtype"], **c["kw"])
        c = dict(c, pinned=check(c["tag"], pred, c["dtype"], c["kw"], orc))
        for b in range(c["bs"]):
            store[f"{c['tag']}.{b}"] = orc[b]
        meta.append(c)
        print(f"NMS {c['tag']}: oracle == reference {c['pinned']}; dets/img {[o.shape[0] for o in orc]}")
    for tag, x, kws in hand_cases():
        for dtype in ("fp32", "fp16", "bf16"):
            pred = nms_ref.round_to(x[None], dtype)
            for k, kw in enumerate(kws):
                t = f"{tag}_{dtype}_{k}"
                orc = nms_ref.non_max_suppression(pred, dtype=dtype, **kw)
                how = check(t, pred, dtype, kw, orc)
                store[f"{t}.0"] = orc[0]
                meta.append(dict(tag=t, pred=f"{tag}_{dtype}.pred", bs=1, dtype=dtype, kw=kw, pinned=how))
                print(f"NMS {t}: oracle == reference {how}; dets {orc[0].shape[0]}")
            store[f"{tag}_{dtype}.pred"] = pred
    store["meta"] = np.array(json.dumps(meta))
    np.savez_compressed(f"{HERE}/nms_edges.npz", **store)


if __name__ == "__main__":
    main()
