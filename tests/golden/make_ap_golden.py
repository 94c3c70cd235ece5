"""Generate tests/golden/ap.npz by running the UNMODIFIED reference's ap_per_class (utils/metrics.py:25-126) through
tests/golden/refshim.py.  The shim serves ultralytics' `smooth` as an inert stub, so a restatement of its public definition is
set on the shimmed `ultralytics.utils.metrics` before the reference imports it.

Runs only where the reference tree exists:
    python tests/golden/make_ap_golden.py
Every case stores its inputs and the reference's outputs.  Cases with equal confidences are recorded twice: under the
reference's own np.argsort (`.default`, host dependent) and with np.argsort patched to kind="stable" (`.stable`, the order the
engine defines).  While generating, the oracle (oracle/ap_ref.py) is checked against the stable record (hard assert).
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ap_ref  # noqa: E402

KEYS = ("tp", "fp", "p", "r", "f1", "ap", "classes")


def smooth(y, f=0.05):
    """ultralytics.utils.metrics.smooth (public definition): box filter of odd length with edge-value padding."""
    nf = round(len(y) * f * 2) // 2 + 1
    p = np.ones(nf // 2)
    yp = np.concatenate((p * y[0], y, p * y[-1]), 0)
    return np.convolve(yp, np.ones(nf) / nf, mode="valid")


def cases():
    def synth(niou, ties, seed, n_img=24, max_det=60, nc=12):
        tp, conf, pc, tc = ap_ref.concat_stats(ap_ref.synth_stats(n_img, max_det, nc, 5.0, niou, seed, ties))
        # a labelled class without predictions, predictions of a class without labels
        tc = np.concatenate((tc, np.full(3, 40, np.float32)))
        extra = np.random.RandomState(seed + 100).rand(25).astype(np.float32)
        extra = extra.astype(np.float16).astype(np.float32) if ties else extra * np.float32(1e-3) + np.float32(0.25)
        return (np.concatenate((tp, np.zeros((25, niou), bool))), np.concatenate((conf, extra)),
                np.concatenate((pc, np.full(25, 41, np.float32))), tc)

    out = {}
    for niou in (1, 10):
        out[f"tiefree{niou}"] = synth(niou, False, 10 + niou)
        out[f"ties{niou}"] = synth(niou, True, 20 + niou)
    tp, conf, pc, tc = ap_ref.concat_stats(ap_ref.synth_stats(30, 40, 1, 3.0, 10, 5, True))
    out["one_class"] = (tp, conf, pc, tc)
    out["n1"] = (np.ones((1, 10), bool), np.array([0.7], np.float32), np.array([3], np.float32), np.array([3, 3, 5], np.float32))
    out["n0"] = (np.zeros((0, 10), bool), np.zeros(0, np.float32), np.zeros(0, np.float32), np.array([1, 2, 2], np.float32))
    tp, conf, pc, _ = ap_ref.concat_stats(ap_ref.synth_stats(4, 20, 5, 3.0, 10, 6, True))
    out["no_labels"] = (tp, conf, pc, np.zeros(0, np.float32))
    return out


def main():
    sys.path.insert(0, HERE)
    import refshim

    refshim.install()
    import ultralytics.utils.metrics as um

    um.smooth = smooth
    from utils.metrics import ap_per_class

    argsort = np.argsort

    def stable_argsort(a, *args, **kwargs):
        kwargs.setdefault("kind", "stable")
        return argsort(a, *args, **kwargs)

    store, meta = {}, {}
    for tag, (tp, conf, pc, tc) in cases().items():
        for k, v in zip(("in_tp", "in_conf", "in_pred_cls", "in_target_cls"), (tp, conf, pc, tc)):
            store[f"{tag}.{k}"] = v
        ties = len(np.unique(conf)) < len(conf)
        records = {"default": None, "stable": None}
        with np.errstate(all="ignore"):
            records["default"] = ap_per_class(tp, conf, pc, tc, names={})
            np.argsort = stable_argsort
            try:
                records["stable"] = ap_per_class(tp, conf, pc, tc, names={})
            finally:
                np.argsort = argsort
        for name, res in records.items():
            if name == "default" and not ties:
                continue
            for k, v in zip(KEYS, res):
                store[f"{tag}.{name}.{k}"] = v
        ours, idx, gap = ap_ref.ap_per_class(tp, conf, pc, tc, return_index=True)
        for k, a, b in zip(KEYS, ours, records["stable"]):
            assert a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a, b, equal_nan=True), (tag, k, "oracle != reference (stable order)")
        same = all(np.array_equal(a, b, equal_nan=True) for a, b in zip(records["default"], records["stable"]))
        meta[tag] = dict(rows=int(len(conf)), niou=int(tp.shape[1]), ties=bool(ties), default_equals_stable=bool(same), argmax=idx,
                         smooth_gap=gap)
        print(f"ap {tag}: {meta[tag]}")
    store["meta"] = np.array(json.dumps(meta, sort_keys=True))
    np.savez_compressed(f"{HERE}/ap.npz", **store)
    print("written", f"{HERE}/ap.npz", os.path.getsize(f"{HERE}/ap.npz"), "bytes")


if __name__ == "__main__":
    main()
