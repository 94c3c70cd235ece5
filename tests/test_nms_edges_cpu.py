"""CPU: the NMS oracle (oracle/nms_ref.py) against tests/golden/nms_edges.npz, which the unmodified reference generated
(tests/golden/make_nms_edge_golden.py): bf16 in val.py's and segment/val.py's regimes with the max_nms cut, 1280-pixel
single-label inputs with the cut, and NaN / inf / degenerate inputs.  This anchors the oracle's rules for NaN scores, the
bf16 threshold and ties at the cut to the reference, so the GPU tests can compare the kernels with the oracle anywhere."""
import json
import os

import numpy as np
import pytest

from oracle import nms_ref

G = os.path.join(os.path.dirname(__file__), "golden")


def _cases():
    g = np.load(os.path.join(G, "nms_edges.npz"))
    return g, json.loads(str(g["meta"]))


def edge_pred(g, c):
    """The input of fixture case c: regenerated from its seed, or the stored hand-built array."""
    if "pred" in c:
        return g[c["pred"]]
    return nms_ref.synth_predictions(c["bs"], c["n"], c["nc"], c["nm"], c["seed"], c["dtype"], img=c["img"])


@pytest.mark.filterwarnings("ignore:invalid value:RuntimeWarning")
def test_oracle_matches_edge_fixture():
    g, meta = _cases()
    assert len(meta) == 30
    for c in meta:
        out = nms_ref.non_max_suppression(edge_pred(g, c), dtype=c["dtype"], **c["kw"])
        for b in range(c["bs"]):
            ref = g[f"{c['tag']}.{b}"]
            assert out[b].shape == ref.shape and np.array_equal(out[b], ref, equal_nan=True), (c["tag"], b)


def test_fixture_covers_the_cut_and_nonfinite_rows():
    """The regimes the fixture exists for are really in it: the cut runs, NaN rows are dropped, +inf scores are kept."""
    g, meta = _cases()
    by_tag = {c["tag"]: c for c in meta}
    for tag in ("val_bf16", "segval_bf16", "p1280_fp16", "p1280_bf16"):
        c = by_tag[tag]
        pred = edge_pred(g, c)
        thr = nms_ref.round_to(np.float32(c["kw"]["conf_thres"]), c["dtype"])
        x = pred[0][pred[0, :, 4] > thr]
        conf = nms_ref.round_to(x[:, 5 : 5 + c["nc"]] * x[:, 4:5], c["dtype"])
        n = int((conf > thr).sum()) if c["kw"].get("multi_label") else int((conf.max(1) > thr).sum())
        assert n > 30000, (tag, n)
    nan = g["nan_cls_fp32_0.0"]
    assert not np.isnan(nan[:, 4]).any() and len(nan) == 47  # the 48 rows with one NaN class score and the all-NaN row go
    assert np.isinf(g["inf_obj_cls_fp32_0.0"][:, 4]).sum() >= 1


@pytest.mark.filterwarnings("ignore:invalid value:RuntimeWarning")
def test_oracle_max_nms_keyword():
    """max_nms at or above the candidate count changes nothing; below it, only the top max_nms candidates in stable score
    order reach the greedy pass."""
    pred = nms_ref.synth_predictions(1, 2000, 5, 0, 3)
    kw = dict(conf_thres=0.001, iou_thres=0.5, multi_label=True, max_det=4096)
    full, fidx = nms_ref.non_max_suppression(pred, return_index=True, **kw)
    same, sidx = nms_ref.non_max_suppression(pred, return_index=True, max_nms=10**6, **kw)
    assert np.array_equal(fidx[0], sidx[0]) and np.array_equal(full[0], same[0])
    x = pred[0][pred[0, :, 4] > np.float32(0.001)]
    conf = x[:, 5:] * x[:, 4:5]
    top = np.sort(conf[conf > np.float32(0.001)])[::-1]
    assert len(top) > 1000
    for k in (1, 2, 63, 64, 1000):
        out, idx = nms_ref.non_max_suppression(pred, return_index=True, max_nms=k, **kw)
        assert 1 <= len(idx[0]) <= k and out[0][:, 4].min() >= top[k - 1], k
    assert out[0][0, 4] == top[0]
