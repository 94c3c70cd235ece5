"""CPU: the AP oracle (oracle/ap_ref.py) against the reference's ap_per_class outputs in tests/golden/ap.npz, its restated
numpy orders against numpy itself, the argument checks of y5_ap_per_class (no GPU needed), and the public signatures."""
import inspect
import json
import os

import numpy as np
import pytest

from oracle import ap_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ap.npz")
KEYS = ("tp", "fp", "p", "r", "f1", "ap", "classes")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _tags(g):
    return sorted(json.loads(str(g["meta"])))


def test_fixture_covers_the_cases(golden):
    meta = json.loads(str(golden["meta"]))
    assert {m["niou"] for m in meta.values()} == {1, 10}
    assert any(m["ties"] and not m["default_equals_stable"] for m in meta.values())  # the reference's own order differs there
    assert meta["n1"]["rows"] == 1 and meta["n0"]["rows"] == 0
    assert golden["no_labels.stable.ap"].shape == (0, 10)
    assert 40 in golden["tiefree10.stable.classes"] and 41 in golden["tiefree10.in_pred_cls"]


def test_oracle_equals_reference_fixture(golden):
    for tag in _tags(golden):
        ins = [golden[f"{tag}.in_{k}"] for k in ("tp", "conf", "pred_cls", "target_cls")]
        got = ap_ref.ap_per_class(*ins)
        for k, a in zip(KEYS, got):
            b = golden[f"{tag}.stable.{k}"]
            assert a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a, b, equal_nan=True), (tag, k)
        if f"{tag}.default.tp" in golden:  # the reference's own, host-dependent tie order: same classes, AP within 1e-2
            assert np.array_equal(golden[f"{tag}.default.classes"], golden[f"{tag}.stable.classes"])
            assert np.abs(golden[f"{tag}.default.ap"] - golden[f"{tag}.stable.ap"]).max() < 1e-2


def test_interp_restatement_equals_numpy():
    rs = np.random.RandomState(0)
    for trial in range(300):
        n = rs.randint(1, 60)
        xp = np.sort(rs.choice(rs.rand(max(1, n // 3)), n))  # many equal xp values
        if trial % 3 == 0:
            xp = np.sort(np.round(rs.rand(n) * 8) / 8)
        fp = rs.rand(n) if trial % 2 else np.round(rs.rand(n) * 4) / 4
        x = np.concatenate((rs.rand(200) * 1.4 - 0.2, xp, [xp[0], xp[-1]]))
        for left, right in ((None, None), (0.0, None), (1.0, 0.5)):
            assert np.array_equal(ap_ref.interp(x, xp, fp, left, right), np.interp(x, xp, fp, left, right)), trial
    xp = -np.sort(rs.rand(500).astype(np.float16).astype(np.float32))[::-1].astype(np.float64)  # -conf of a class, fp16 ties
    fp = rs.rand(500)
    assert np.array_equal(ap_ref.interp(-ap_ref.PX, xp, fp, left=1), np.interp(-ap_ref.PX, xp, fp, left=1))


def test_trapezoid_and_mean_restatements_equal_numpy():
    rs = np.random.RandomState(1)
    trapezoid = np.trapezoid if hasattr(np, "trapezoid") else np.trapz
    for _ in range(2000):
        y = rs.rand(101) * rs.choice([1e-3, 1, 1e3])
        assert ap_ref.trapezoid(y, ap_ref.X101) == trapezoid(y, ap_ref.X101)
    for n in range(1, 129):
        t = rs.randn(n) * 10 ** rs.uniform(-3, 3, n)
        assert ap_ref.pairwise_sum(t) == np.add.reduce(t), n
    for nc in (1, 2, 3, 7, 80, 200):
        a = rs.rand(nc, 1000) * rs.choice([0, 1], (nc, 1))
        assert np.array_equal(ap_ref.mean0(a), a.mean(0)), nc


def test_synth_stats_nest_and_respect_label_counts():
    for correct, conf, pc, tc in ap_ref.synth_stats(40, 50, 10, 5.0, 10, seed=3):
        assert (correct[:, 1:] <= correct[:, :-1]).all()
        for c in np.unique(pc):
            assert correct[pc == c, 0].sum() <= (tc == c).sum()
        assert conf.dtype == np.float32 and pc.dtype == np.float32


def test_ap_entry_points_reject_bad_arguments_without_gpu(built_lib):
    lib = built_lib
    assert lib.y5_ap_workspace_bytes(1, 1000, 10, 50, 1) > 1000 * 10 * 4
    assert lib.y5_ap_workspace_bytes(1, 1000, 10, 50, 2) > lib.y5_ap_workspace_bytes(1, 1000, 10, 50, 1)
    assert lib.y5_ap_workspace_bytes(1, 1000, 0, 50, 1) == -1
    assert lib.y5_ap_workspace_bytes(1, 1000, 33, 50, 1) == -2 and b"32" in lib.y5_last_error()
    assert lib.y5_ap_workspace_bytes(1 << 16, 1 << 15, 10, 50, 1) == -2  # 2^31 rows
    assert lib.y5_ap_workspace_bytes(-1, 10, 10, 50, 1) == -1 and lib.y5_ap_workspace_bytes(1, 10, 10, 50, 3) == -1
    # y5_ap_per_class(tp, tp2, tp_img_stride, tp_row_stride, conf, pred_cls, img_stride, row_stride, count, n_img, rows_per_image,
    #                 niou, target_cls, nt, grid, eps, workspace, workspace_bytes, out, meta, stream)
    ok = (4096, None, 0, 10, 4096, 4096, 0, 1, None, 1, 100, 10, 4096, 5, 4096, 1e-16, 4096, 1 << 30, 4096, 4096, None)

    def call(**kw):
        names = ["tp", "tp2", "tpis", "tprs", "conf", "cls", "is_", "rs", "count", "n_img", "rows", "niou", "tc", "nt", "grid", "eps", "ws",
                 "wsb", "out", "meta", "stream"]
        args = dict(zip(names, ok))
        args.update(kw)
        return lib.y5_ap_per_class(*[args[n] for n in names])

    assert call(tp=None) == -1
    assert call(tprs=9) == -1  # tp rows narrower than niou
    assert call(niou=0) == -1 and call(niou=33, tprs=33) == -2
    assert call(rows=1 << 16, n_img=1 << 15, is_=1, tpis=1) == -2
    assert call(n_img=2) == -1  # several images need image strides
    assert call(tc=None) == -1 and call(grid=None) == -1 and call(meta=None) == -1 and call(out=None) == -1
    assert call(wsb=100) == -1 and b"workspace" in lib.y5_last_error()
    assert call(nt=-1) == -1


def test_ap_requires_cuda_and_refuses_plots():
    import torch

    from yolov5_b200.utils.metrics import ap_per_class
    from yolov5_b200.utils.segment.metrics import ap_per_class_box_and_mask

    args = (np.ones((2, 10), bool), np.array([0.5, 0.4], np.float32), np.zeros(2, np.float32), np.zeros(1, np.float32))
    with pytest.raises(NotImplementedError):
        ap_per_class(*args, plot=True)
    with pytest.raises(NotImplementedError):
        ap_per_class_box_and_mask(args[0], *args, plot=True)
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="CUDA"):
            ap_per_class(*args)


def test_reference_signatures():
    from yolov5_b200.utils import metrics
    from yolov5_b200.utils.segment import metrics as seg_metrics

    assert str(inspect.signature(metrics.ap_per_class)) == "(tp, conf, pred_cls, target_cls, plot=False, save_dir='.', names=(), eps=1e-16, prefix='')"
    assert str(inspect.signature(seg_metrics.ap_per_class_box_and_mask)) == "(tp_m, tp_b, conf, pred_cls, target_cls, plot=False, save_dir='.', names=())"
    assert list(inspect.signature(metrics.ap_per_class_batch).parameters) == ["correct", "rows", "count", "target_cls", "eps", "correct_masks"]
