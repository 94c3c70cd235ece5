"""GPU: ap_per_class / ap_per_class_box_and_mask / ap_per_class_batch on the device against the float64 oracle
(oracle/ap_ref.py) and the reference fixture (tests/golden/ap.npz), np.array_equal on every output."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import ap_ref, post_ref
from yolov5_b200.utils import metrics
from yolov5_b200.utils.segment.metrics import ap_per_class_box_and_mask

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ap.npz")
KEYS = ("tp", "fp", "p", "r", "f1", "ap", "classes")
IOUV = np.linspace(0.5, 0.95, 10).astype(np.float32)


def _assert_equal(got, want, tag, index_free=False):
    """index_free: the two largest smoothed mean-F1 values lie within 1e-12, so either index is accepted and only the
    outputs that do not depend on it (ap, classes) are compared."""
    for k, a, b in zip(KEYS, got, want):
        if index_free and k not in ("ap", "classes"):
            continue
        assert a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a, b, equal_nan=True), (tag, k)


def _oracle(tp, conf, pc, tc):
    want, _, gap = ap_ref.ap_per_class(tp, conf, pc, tc, return_index=True)
    return want, gap < 1e-12 and gap != 0.0


def _stats(rows, niou, seed, ties=True, nc=80):
    st = ap_ref.synth_stats(max(1, rows // 150 + 1), 300, nc, 7.3, niou, seed, ties)
    tp, conf, pc, tc = ap_ref.concat_stats(st)
    assert len(conf) >= rows
    return tp[:rows], conf[:rows], pc[:rows], tc


def test_fixture_cases(cuda):
    g = np.load(GOLDEN)
    for tag in sorted(json.loads(str(g["meta"]))):
        ins = [g[f"{tag}.in_{k}"] for k in ("tp", "conf", "pred_cls", "target_cls")]
        want = [g[f"{tag}.stable.{k}"] for k in KEYS]
        _assert_equal(metrics.ap_per_class(*ins), want, tag)
        _assert_equal(metrics.ap_per_class(*ins), ap_ref.ap_per_class(*ins), tag)


@pytest.mark.parametrize("niou", [1, 10])
@pytest.mark.parametrize("rows", [0, 1, 7, 1000, 300_000, 1_500_000])
def test_random_cases_equal_oracle(cuda, rows, niou):
    tp, conf, pc, tc = _stats(rows, niou, seed=rows % 9973 + niou, ties=niou == 10)
    want, index_free = _oracle(tp, conf, pc, tc)
    _assert_equal(metrics.ap_per_class(tp, conf, pc, tc), want, (rows, niou), index_free)
    if rows >= 1000:
        assert want[5].max() > 0 and len(want[6]) > 10


def test_numpy_and_cuda_inputs_give_the_same_bits(cuda):
    tp, conf, pc, tc = _stats(20_000, 10, seed=4)
    a = metrics.ap_per_class(tp, conf, pc, tc)
    b = metrics.ap_per_class(*(torch.from_numpy(x).to(cuda) for x in (tp, conf, pc, tc)))
    _assert_equal(b, a, "cuda inputs")
    c = metrics.ap_per_class(tp, conf.astype(np.float64), pc.astype(np.int64), tc.astype(np.float64))  # exact in float32
    _assert_equal(c, a, "float64 / int64 inputs")


def test_two_calls_are_bit_identical(cuda):
    tp, conf, pc, tc = _stats(300_000, 10, seed=8)
    _assert_equal(metrics.ap_per_class(tp, conf, pc, tc), metrics.ap_per_class(tp, conf, pc, tc), "repeat")


def test_ties_follow_the_stable_order(cuda):
    """Equal confidences everywhere: the result is the stable order's, not the order of any unstable sort."""
    rs = np.random.RandomState(2)
    n = 5000
    conf = np.round(rs.rand(n) * 4).astype(np.float32) / 4
    conf[::11] = -0.0  # ties with +0
    conf[::7] = np.nan  # NaN rows sort last
    pc = rs.randint(0, 5, n).astype(np.float32)
    tc = rs.randint(0, 6, 3000).astype(np.float32)
    tp = np.zeros((n, 10), bool)
    for c in range(5):
        rows = np.nonzero(pc == c)[0]
        keep = rows[rs.permutation(len(rows))[: (tc == c).sum() // 2]]
        tp[keep, : rs.randint(1, 11)] = True
    tp[np.isnan(conf)] = False
    got = metrics.ap_per_class(tp, conf, pc, tc)
    i = np.argsort(-conf, kind="stable")
    assert np.isnan(conf[i][-int(np.isnan(conf).sum()):]).all()
    want, index_free = _oracle(tp, conf, pc, tc)
    _assert_equal(got, want, "ties", index_free)


def _padded(stats, dev, max_det, rs):
    """val.py-order stats -> the padded (correct, rows, count) a batched loop holds, with garbage in every padding row."""
    n_img, niou = len(stats), stats[0][0].shape[1]
    correct = np.ones((n_img, max_det, niou), bool)
    rows = np.full((n_img, max_det, 6), np.nan, np.float32)
    rows[..., 4] = rs.choice([np.nan, 3e38, -1e30, 0.5], (n_img, max_det))
    rows[..., 5] = rs.choice([np.nan, 1e9, -7, 2.5], (n_img, max_det))
    count = np.zeros(n_img, np.int32)
    for b, (c, conf, pc, _) in enumerate(stats):
        n = len(conf)
        count[b] = n
        correct[b, :n], rows[b, :n, 4], rows[b, :n, 5] = c, conf, pc
    t = lambda a: torch.from_numpy(a).to(dev)  # noqa: E731
    return t(correct), t(rows), t(count)


def test_batch_form_equals_the_concatenation(cuda):
    rs = np.random.RandomState(5)
    parts, flat = [], []
    for seed in range(3):  # three batches of 16 images, concatenated along dim 0
        st = ap_ref.synth_stats(16, 120, 30, 6.0, 10, seed=40 + seed)
        st[3] = (st[3][0][:0], st[3][1][:0], st[3][2][:0], st[3][3])  # an image with no predictions
        parts.append(_padded(st, cuda, 120, rs))
        flat += st
    correct, rows, count = (torch.cat([p[i] for p in parts]) for i in range(3))
    tp, conf, pc, tc = ap_ref.concat_stats(flat)
    want = metrics.ap_per_class(tp, conf, pc, tc)
    _assert_equal(metrics.ap_per_class_batch(correct, rows, count, torch.from_numpy(tc).to(cuda)), want, "batch")
    want_o, index_free = _oracle(tp, conf, pc, tc)
    _assert_equal(want, want_o, "batch oracle", index_free)
    # box and mask: the dict of ap_per_class_box_and_mask, both from one sort
    masks = correct & torch.from_numpy(rs.rand(*correct.shape) < 0.7).to(cuda)
    tp_m = np.concatenate([masks[b, :int(count[b])].cpu().numpy() for b in range(len(count))])
    d = metrics.ap_per_class_batch(correct, rows, count, tc, correct_masks=masks)
    ref = ap_per_class_box_and_mask(tp_m, tp, conf, pc, tc)
    for k in ("boxes", "masks"):
        for f in ("p", "r", "ap", "f1", "ap_class"):
            assert np.array_equal(d[k][f], ref[k][f]), (k, f)


def test_box_and_mask_equals_two_oracle_runs(cuda):
    tp_b, conf, pc, tc = _stats(50_000, 10, seed=12)
    tp_m = tp_b & (np.random.RandomState(1).rand(*tp_b.shape) < 0.6)
    d = ap_per_class_box_and_mask(tp_m, tp_b, conf, pc, tc)
    for key, tp in (("boxes", tp_b), ("masks", tp_m)):
        want, index_free = _oracle(tp, conf, pc, tc)
        got = (None, None, d[key]["p"], d[key]["r"], d[key]["f1"], d[key]["ap"], d[key]["ap_class"])
        for k, a, b in list(zip(KEYS, got, want))[2:]:
            if index_free and k not in ("ap", "classes"):
                continue
            assert np.array_equal(a, b), (key, k)


@pytest.mark.parametrize("bad", ["pred_fraction", "pred_negative", "pred_4096", "pred_nan", "target_fraction"])
def test_invalid_classes_raise(cuda, bad):
    tp, conf, pc, tc = _stats(1000, 10, seed=3)
    pc, tc = pc.copy(), tc.copy()
    if bad.startswith("pred"):
        pc[17] = {"pred_fraction": 2.5, "pred_negative": -1.0, "pred_4096": 4096.0, "pred_nan": np.nan}[bad]
    else:
        tc[3] = 1.5
    with pytest.raises(ValueError, match="class"):
        metrics.ap_per_class(tp, conf, pc, tc)


def test_end_to_end_from_nms(cuda):
    """nms_device -> val_batch_metrics -> ap_per_class_batch equals val.py's per-image stats (process_batch oracle) + oracle."""
    from yolov5_b200.utils.general import nms_device

    rs = np.random.RandomState(7)
    bs, n, nc = 8, 2000, 6
    pred = np.zeros((bs, n, 5 + nc), np.float32)
    pred[..., :2] = rs.uniform(20, 300, (bs, n, 2))
    pred[..., 2:4] = rs.uniform(8, 80, (bs, n, 2))
    pred[..., 4] = rs.rand(bs, n).astype(np.float16)
    pred[..., 5:] = rs.rand(bs, n, nc).astype(np.float16)
    tg = []
    for b in range(bs):
        for _ in range(rs.randint(0, 12)):
            tg.append([b, rs.randint(0, nc), *rs.uniform(40, 280, 2), *rs.uniform(10, 60, 2)])
    tg = np.array(tg, np.float32)
    im_hw = (320, 320)
    shapes = [((320, 320), ((1.0, 1.0), (0.0, 0.0)))] * bs
    rows, _, count = nms_device(torch.from_numpy(pred).to(cuda), 0.001, 0.6, max_det=300)
    iouv = torch.from_numpy(IOUV).to(cuda)
    predn, correct = metrics.val_batch_metrics(rows, count, torch.from_numpy(tg).to(cuda), im_hw, shapes, iouv)
    labelsn = metrics.labels_to_native(torch.from_numpy(tg).to(cuda), metrics._meta(im_hw, shapes, cuda)).cpu().numpy()
    got = metrics.ap_per_class_batch(correct, rows, count, torch.from_numpy(tg[:, 1]).to(cuda))
    stats = []
    for b in range(bs):
        k = int(count[b])
        p = predn[b, :k].cpu().numpy()
        lab = labelsn[labelsn[:, 0] == b][:, 1:]
        c = post_ref.process_batch(p[:, :6], lab, IOUV) if len(lab) and k else np.zeros((k, 10), bool)
        stats.append((c, rows[b, :k, 4].cpu().numpy(), rows[b, :k, 5].cpu().numpy(), lab[:, 0]))
    tp, conf, pc, tc = ap_ref.concat_stats(stats)
    assert tp.any() and len(conf) > 1000
    want, index_free = _oracle(tp, conf, pc, tc)
    _assert_equal(got, want, "nms chain", index_free)
