"""CPU: the confusion-matrix oracle (oracle/confusion_ref.py) against the reference's matrices in tests/golden/confusion.npz,
fitness / Metric / Metrics against the reference's outputs, y5_confusion_batch's declaration and argument checks (no GPU
needed), the public signatures, and the reference scripts' metric imports under compat.install()."""
import ctypes
import inspect
import json
import os
import re
import sys

import numpy as np
import pytest

from oracle import confusion_ref
from yolov5_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "confusion.npz")
HEADER = os.path.join(os.path.dirname(HERE), "include", "y5b200.h")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _meta(g):
    return json.loads(str(g["meta"]))


def golden_calls(g, tag):
    """(nc, conf, iou_thres, [(detections or None, labels), ...]) of one fixture case."""
    nc, conf, iou = g[f"{tag}.params"]
    calls = []
    for k in range(_meta(g)["cases"][tag]["calls"]):
        det = g[f"{tag}.{k}.det"] if f"{tag}.{k}.det" in g else None
        calls.append((det, g[f"{tag}.{k}.lab"]))
    return int(nc), float(conf), float(iou), calls


def test_fixture_covers_the_cases(golden):
    cases = _meta(golden)["cases"]
    assert {"coco_a", "no_detections", "no_labels", "no_match", "thresholds", "ties", "detections_none", "nc1"} <= set(cases)
    assert any(not c["default_equals_stable"] for c in cases.values())  # equal IoUs: the reference's own order differs there
    nc = cases["no_match"]["nc"]
    m = golden["no_match.stable"]
    assert m[nc].sum() == 2 and m[:, nc].sum() == 0  # labels background, no detection counted without a match
    assert golden["no_labels.stable"].sum() == 0
    t = golden["thresholds.stable"]
    assert t[5, 2] == 1 and t[1, 2] == 1 and t.sum() == 2  # conf == 0.25 and IoU == fp32(0.45) are both dropped
    coco = golden["coco_a.stable"]
    assert coco[80].sum() > 0 and coco[:80, 80].sum() > 0 and np.trace(coco[:80, :80]) > 0


def test_oracle_equals_reference_fixture(golden):
    for tag, c in _meta(golden)["cases"].items():
        nc, conf, iou, calls = golden_calls(golden, tag)
        stable = np.zeros((nc + 1, nc + 1))
        for det, lab in calls:
            confusion_ref.process_batch(stable, det, lab, nc, conf, iou)
        assert np.array_equal(stable, golden[f"{tag}.stable"]), tag
        if c["default_equals_stable"]:
            assert np.array_equal(stable, golden[f"{tag}.reference"]), tag
        else:  # equal IoUs between classes: same totals per true class, the counts move between rows
            assert np.array_equal(golden[f"{tag}.reference"][:, :nc].sum(0), stable[:, :nc].sum(0)), tag


def test_val_loop_matches_per_call_oracle():
    rows, count, lab6 = confusion_ref.synth_batch(6, 50, 10, 4.0, seed=5)
    count[1] = 0
    lab6 = lab6[lab6[:, 0] != 2]
    want = np.zeros((11, 11))
    for si in range(6):
        lab = lab6[lab6[:, 0] == si, 1:]
        if len(lab):
            confusion_ref.process_batch(want, rows[si, :count[si], :6] if count[si] else None, lab if count[si] else lab[:, 0], 10)
    assert np.array_equal(confusion_ref.val_loop(np.zeros((11, 11)), rows, count, lab6, 10), want)


def test_fitness_and_metrics_equal_reference(golden):
    from yolov5_b200.utils import metrics
    from yolov5_b200.utils.segment import metrics as seg

    x = {k[len("metrics.in."):]: golden[k] for k in golden.files if k.startswith("metrics.in.")}
    sys.path.insert(0, os.path.join(HERE, "golden"))
    try:
        import make_confusion_golden as mk
    finally:
        sys.path.pop(0)
    for name, (fit, seg_fit) in {"engine": (metrics.fitness, seg.fitness), "oracle": (confusion_ref.fitness, confusion_ref.seg_fitness)}.items():
        got = mk.metrics_record(fit, seg_fit, seg.Metrics, x)
        for k, v in got.items():
            want = golden[f"metrics.out.{k}"]
            assert v.shape == want.shape and np.array_equal(v, want), (name, k)
    m = seg.Metric()
    assert m.ap50 == [] and m.ap == [] and m.mean_results() == (0.0, 0.0, 0.0, 0.0)
    assert seg.KEYS == _meta(golden)["keys"]


def _header_args(name):
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    decl = re.search(rf"\bint\s+{name}\s*\(([^)]*)\)", src).group(1)
    return [" ".join(a.split()) for a in decl.split(",")]


def test_header_declaration_agrees_with_binding():
    args = _header_args("y5_confusion_batch")
    kinds = {"float*": _lib._P, "int32_t*": _lib._P, "int64_t*": _lib._P, "void*": _lib._P, "int64_t": _lib._I64, "int32_t": _lib._I32,
             "float": _lib._F}
    mapped = []
    for a in args:
        t = a.replace("const ", "").rsplit(" ", 1)[0].replace(" *", "*")
        if "*" in a.rsplit(" ", 1)[-1]:
            t += "*"
        mapped.append(kinds[t])
    restype, argtypes = _lib.SIGNATURES["y5_confusion_batch"]
    assert restype is _lib._I32 and argtypes == mapped, (args, argtypes)
    assert [a.rsplit(" ", 1)[-1].lstrip("*") for a in args] == ["det", "img_stride", "row_stride", "count", "batch", "max_det", "labels", "nt",
                                                                "nc", "conf_thres", "iou_thres", "eps", "matrix", "error", "stream"]


def test_confusion_entry_point_rejects_bad_arguments_without_gpu(built_lib):
    lib = built_lib
    # y5_confusion_batch(det, img_stride, row_stride, count, batch, max_det, labels, nt, nc, conf, iou, eps, matrix, error, stream)
    ok = dict(det=4096, img_stride=1800, row_stride=6, count=None, batch=2, max_det=300, labels=4096, nt=5, nc=80, conf=0.25, iou=0.45,
              eps=1e-7, matrix=4096, error=4096, stream=None)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.y5_confusion_batch(*a.values())

    assert call(batch=0) == 0  # nothing to do, nothing launched
    assert call(matrix=None) == -1 and call(error=None) == -1
    assert call(det=None) == -1 and call(labels=None) == -1
    assert call(nc=0) == -1 and call(row_stride=5) == -1 and call(nt=-1) == -1 and call(batch=-1) == -1
    assert call(max_det=5000) == -2 and b"4096" in lib.y5_last_error()
    assert call(nc=40000) == -2


def test_signatures_match_the_reference(golden):
    import importlib

    bad = []
    for key, theirs in _meta(golden)["signatures"].items():
        mod, qual = key.split(":")
        obj = importlib.import_module("yolov5_b200." + mod)
        for part in qual.split("."):
            obj = getattr(obj, part)
        mine = [[n, repr(p.default) if p.default is not inspect._empty else None, str(p.kind)] for n, p in inspect.signature(obj).parameters.items()]
        if mine != theirs:
            bad.append((key, theirs, mine))
    assert not bad, bad
    from yolov5_b200.utils.metrics import ConfusionMatrix

    assert list(inspect.signature(ConfusionMatrix.process_batch_padded).parameters) == ["self", "rows", "count", "labels6"]
    cm = ConfusionMatrix(3)
    assert (cm.nc, cm.conf, cm.iou_thres) == (3, 0.25, 0.45) and cm.matrix.shape == (4, 4) and cm.matrix.dtype == np.float64


def test_scripts_metric_imports_resolve_under_compat():
    """The import lines of val.py:60, segment/val.py:63,67, train.py:85 and segment/train.py:79."""
    from yolov5_b200 import compat
    from yolov5_b200.utils import metrics
    from yolov5_b200.utils.segment import metrics as seg

    saved = {k: sys.modules.get(k) for k in compat.ALIASES}
    try:
        assert compat.install()
        ns = {}
        exec("from utils.metrics import ConfusionMatrix, ap_per_class, process_batch\n"
             "from utils.metrics import ConfusionMatrix as SegConfusionMatrix\n"
             "from utils.segment.metrics import Metrics, ap_per_class_box_and_mask\n"
             "from utils.metrics import fitness\n"
             "from utils.segment.metrics import KEYS, fitness as seg_fitness\n", ns)
        assert ns["ConfusionMatrix"] is metrics.ConfusionMatrix is ns["SegConfusionMatrix"]
        assert ns["ap_per_class"] is metrics.ap_per_class and ns["process_batch"] is metrics.process_batch
        assert ns["Metrics"] is seg.Metrics and ns["ap_per_class_box_and_mask"] is seg.ap_per_class_box_and_mask
        assert ns["fitness"] is metrics.fitness and ns["seg_fitness"] is seg.fitness and ns["KEYS"] is seg.KEYS
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def test_confusion_refuses_cpu_and_other_dtypes():
    import torch

    from yolov5_b200.utils.metrics import ConfusionMatrix

    cm = ConfusionMatrix(5)
    with pytest.raises(RuntimeError, match="CUDA"):
        cm.process_batch(torch.zeros(2, 6), torch.zeros(1, 5))
    with pytest.raises(RuntimeError, match="CUDA"):
        cm.process_batch(None, torch.zeros(3))
    with pytest.raises(TypeError):
        cm.process_batch(np.zeros((2, 6), np.float32), np.zeros((1, 5), np.float32))


def test_plot_failure_is_logged_not_raised(tmp_path, caplog):
    from yolov5_b200.utils.metrics import ConfusionMatrix

    cm = ConfusionMatrix(2)
    cm.matrix[0, 0] = 3
    cm.plot(save_dir=str(tmp_path), names=("a", "b"))  # without seaborn / matplotlib: a warning, no exception
    cm.print()
    assert cm.matrix[0, 0] == 3


def test_ctypes_word_layout_of_error_slot():
    """The Python layer reads the int32 error word from the low half of the accumulator's last int64 entry."""
    v = ctypes.c_int64(0)
    ctypes.cast(ctypes.addressof(v), ctypes.POINTER(ctypes.c_int32))[0] = 3
    assert v.value == 3
