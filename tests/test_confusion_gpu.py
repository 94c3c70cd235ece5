"""GPU: ConfusionMatrix on the device (y5_confusion_batch) against the reference's matrices (tests/golden/confusion.npz, the
stable tie order) and against val.py's per-image loop run through the oracle (oracle/confusion_ref.py): exact counts."""
import numpy as np
import pytest
import torch

from oracle import confusion_ref
from tests.test_confusion_cpu import GOLDEN, _meta, golden_calls
from yolov5_b200.utils import metrics
from yolov5_b200.utils.general import scale_meta
from yolov5_b200.utils.metrics import ConfusionMatrix

pytestmark = pytest.mark.gpu


def _dev(x, dev):
    return None if x is None else torch.from_numpy(np.ascontiguousarray(x)).to(dev)


def _padded(dev, n_img=32, seed=0, extra_cols=0):
    rows, count, lab6 = confusion_ref.synth_batch(n_img, 300, 80, 7.3, seed=seed, extra_cols=extra_cols)
    count[3] = 0  # an image without rows (val.py: detections=None)
    lab6 = lab6[lab6[:, 0] != 5]  # an image without labels (val.py: no call)
    assert (lab6[:, 0] == 3).any()
    return rows, count, lab6


def test_process_batch_equals_reference_fixture(cuda):
    g = np.load(GOLDEN)
    for tag in _meta(g)["cases"]:
        nc, conf, iou, calls = golden_calls(g, tag)
        cm = ConfusionMatrix(nc=nc, conf=conf, iou_thres=iou)
        for det, lab in calls:
            cm.process_batch(_dev(det, cuda), _dev(lab, cuda))
        assert np.array_equal(cm.matrix, g[f"{tag}.stable"]), tag


@pytest.mark.parametrize("extra_cols", [0, 32])
def test_padded_batch_equals_val_loop(cuda, extra_cols):
    """B = 32, 300 rows: detection rows (6 columns) and segmentation rows (38), padding rows holding garbage."""
    rows, count, lab6 = _padded(cuda, seed=11 + extra_cols, extra_cols=extra_cols)
    want = confusion_ref.val_loop(np.zeros((81, 81)), rows, count, lab6, 80)
    cm = ConfusionMatrix(nc=80)
    r = _dev(rows, cuda)
    assert r.stride(1) == 6 + extra_cols
    cm.process_batch_padded(r, _dev(count, cuda), _dev(lab6, cuda))
    got = cm.matrix
    assert np.array_equal(got, want)
    assert got[80].sum() > 0 and got[:80, 80].sum() > 0 and np.trace(got[:80, :80]) > 0


def test_padded_batch_equals_per_image_process_batch(cuda):
    rows, count, lab6 = _padded(cuda, n_img=8, seed=4)
    a, b = ConfusionMatrix(80), ConfusionMatrix(80)
    a.process_batch_padded(_dev(rows, cuda), _dev(count, cuda), _dev(lab6, cuda))
    for si in range(8):
        lab = _dev(lab6[lab6[:, 0] == si, 1:], cuda)
        if count[si] == 0:
            if len(lab):
                b.process_batch(None, lab[:, 0])
        elif len(lab):
            b.process_batch(_dev(rows[si, :count[si]], cuda), lab)  # (N, 6) rows with garbage beyond count never read
    assert np.array_equal(a.matrix, b.matrix)


def test_accumulates_across_batches(cuda):
    cm = ConfusionMatrix(80)
    want = np.zeros((81, 81))
    for k in range(4):
        rows, count, lab6 = _padded(cuda, n_img=16, seed=30 + k)
        confusion_ref.val_loop(want, rows, count, lab6, 80)
        cm.process_batch_padded(_dev(rows, cuda), _dev(count, cuda), _dev(lab6, cuda))
        if k == 1:
            assert np.array_equal(cm.matrix, want)  # a read in between folds the counts so far
    assert np.array_equal(cm.matrix, want)
    rows, count, lab6 = _padded(cuda, n_img=16, seed=30)
    cm2 = ConfusionMatrix(80)
    for _ in range(3):  # integer atomics: the same input gives the same counts every time
        cm2.process_batch_padded(_dev(rows, cuda), _dev(count, cuda), _dev(lab6, cuda))
    assert np.array_equal(cm2.matrix, 3 * confusion_ref.val_loop(np.zeros((81, 81)), rows, count, lab6, 80))


def test_matrix_read_and_write_semantics(cuda):
    rows, count, lab6 = _padded(cuda, n_img=4, seed=8)
    once = confusion_ref.val_loop(np.zeros((81, 81)), rows, count, lab6, 80)
    args = (_dev(rows, cuda), _dev(count, cuda), _dev(lab6, cuda))
    cm = ConfusionMatrix(80)
    m = cm.matrix
    assert m.shape == (81, 81) and m.dtype == np.float64 and not m.any()
    cm.process_batch_padded(*args)
    assert cm.matrix is m and np.array_equal(m, once)  # the same array, updated in place
    cm.matrix[0, 0] += 7  # in-place edits persist
    cm.process_batch_padded(*args)
    want = 2 * once
    want[0, 0] += 7
    assert np.array_equal(cm.matrix, want)  # later device counts add on top
    cm.process_batch_padded(*args)  # pending, then replaced: the setter drops counts not yet read
    fresh = np.ones((81, 81))
    cm.matrix = fresh
    assert cm.matrix is fresh and np.array_equal(fresh, np.ones((81, 81)))
    cm.process_batch_padded(*args)
    assert np.array_equal(cm.matrix, once + 1)


def test_padded_update_replays_in_a_cuda_graph(cuda):
    """Capture fails on any host synchronisation: the update captures after one eager update, and each replay adds one
    batch's counts."""
    rows, count, lab6 = _padded(cuda, seed=2)
    once = confusion_ref.val_loop(np.zeros((81, 81)), rows, count, lab6, 80)
    args = (_dev(rows, cuda), _dev(count, cuda), _dev(lab6, cuda))
    cm = ConfusionMatrix(80)
    cm.process_batch_padded(*args)
    assert np.array_equal(cm.matrix, once)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cm.process_batch_padded(*args)
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(cm.matrix, 4 * once)


@pytest.mark.parametrize("where", ["label", "detection", "negative"])
def test_out_of_range_class_raises_on_read(cuda, where):
    box = [10.0, 10.0, 60.0, 60.0]
    det = torch.tensor([box + [0.9, 2.0]], device=cuda)
    lab = torch.tensor([[1.0] + box], device=cuda)
    if where == "label":
        lab[0, 0] = 5.0
    elif where == "detection":
        det[0, 5] = 7.0
    else:
        det[0, 5] = -1.0
    cm = ConfusionMatrix(5)
    cm.process_batch(det, lab)
    with pytest.raises(ValueError, match="outside"):
        cm.matrix
    assert not cm.matrix.any()  # the error and its batch's counts are dropped together
    det[0, 5] = -0.5  # .int() truncates toward zero: class 0
    lab[0, 0] = 4.9
    cm.process_batch(det, lab)
    assert cm.matrix[0, 4] == 1 and cm.matrix.sum() == 1


def test_process_batch_argument_checks(cuda):
    cm = ConfusionMatrix(5)
    with pytest.raises(TypeError):
        cm.process_batch(torch.zeros(2, 6, device=cuda, dtype=torch.float16), torch.zeros(1, 5, device=cuda))
    with pytest.raises(TypeError):
        cm.process_batch(torch.zeros(2, 6, device=cuda), torch.zeros(1, 5, device=cuda, dtype=torch.float64))
    with pytest.raises(ValueError):
        cm.process_batch(torch.zeros(2, 6, device=cuda), torch.zeros(1, 6, device=cuda))
    with pytest.raises(RuntimeError, match="CUDA"):
        cm.process_batch(torch.zeros(2, 6), torch.zeros(1, 5))
    assert not cm.matrix.any()


def _net_batch(dev, seed, extra_cols=0):
    """A padded batch in network-input pixels with val.py-style targets: rows (B,300,6+extra), count, targets (nt,6)
    [img, cls, cx, cy, w, h], the network input's (h, w) and the (B,5) scale meta."""
    rows, count, lab6 = _padded(dev, n_img=12, seed=seed, extra_cols=extra_cols)
    im_hw = (640, 640)
    shapes = [((480, 640), ((1.0, 1.0), (0.0, 80.0)))] * rows.shape[0]
    tg = lab6.copy()
    tg[:, 2:4] = (lab6[:, 2:4] + lab6[:, 4:6]) / 2
    tg[:, 4:6] = lab6[:, 4:6] - lab6[:, 2:4]
    meta = scale_meta(im_hw, [s[0] for s in shapes], [s[1] for s in shapes]).to(dev)
    return _dev(rows, dev), _dev(count, dev), _dev(tg, dev), im_hw, shapes, meta


def test_val_batch_metrics_confusion_keyword(cuda):
    rows, count, tg, im_hw, shapes, meta = _net_batch(cuda, 50)
    iouv = torch.linspace(0.5, 0.95, 10, device=cuda)
    cm = ConfusionMatrix(80)
    predn, correct = metrics.val_batch_metrics(rows, count, tg, im_hw, shapes, iouv, confusion=cm)
    predn0, correct0 = metrics.val_batch_metrics(rows, count, tg, im_hw, shapes, iouv)
    assert torch.equal(predn, predn0) and torch.equal(correct, correct0)
    labelsn = metrics.labels_to_native(tg, meta)
    separate = ConfusionMatrix(80)
    separate.process_batch_padded(predn0, count, labelsn)
    got = cm.matrix
    assert np.array_equal(got, separate.matrix) and got.sum() > 0
    want = confusion_ref.val_loop(np.zeros((81, 81)), predn0.cpu().numpy(), count.cpu().numpy(), labelsn.cpu().numpy(), 80)
    assert np.array_equal(got, want)


def test_seg_val_batch_metrics_rows_count_as_segment_val(cuda):
    """segment/val.py counts the confusion matrix on the box IoU: process_batch_padded on seg_val_batch_metrics' 38-column
    native rows equals its per-image loop."""
    rows, count, tg, im_hw, shapes, meta = _net_batch(cuda, 51, extra_cols=32)
    protos = torch.randn(rows.shape[0], 32, 160, 160, device=cuda)
    masks = torch.zeros(rows.shape[0], 640, 640, device=cuda)  # overlap index images; mask IoU is not what is checked here
    iouv = torch.linspace(0.5, 0.95, 10, device=cuda)
    predn, _, _ = metrics.seg_val_batch_metrics(rows, count, protos, tg, masks, im_hw, meta, iouv, True)
    labelsn = metrics.labels_to_native(tg, meta)
    cm = ConfusionMatrix(80)
    cm.process_batch_padded(predn, count, labelsn)
    want = confusion_ref.val_loop(np.zeros((81, 81)), predn.cpu().numpy(), count.cpu().numpy(), labelsn.cpu().numpy(), 80)
    assert predn.shape[2] == 38 and np.array_equal(cm.matrix, want) and want.sum() > 0
