"""CPU: the mask-IoU oracle (tests/mask_val_ref.py) against the reference's process_batch(masks=True) outputs in
tests/golden/mask_val.npz, the argument checks of the mask-IoU entry points (no GPU needed), and the public signatures."""
import ctypes
import inspect
import itertools
import json
import os

import numpy as np
import pytest
import torch

from tests import mask_val_ref
from yolov5_b200 import _lib

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mask_val.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.mark.parametrize("tag", list(mask_val_ref.CASES))
def test_oracle_equals_reference_fixture(golden, tag):
    det, labels, pred, gt, overlap = mask_val_ref.case_inputs(tag)
    correct, iou, _, _ = mask_val_ref.process_batch_masks(det, labels, mask_val_ref.IOUV, pred, gt, overlap)
    assert np.array_equal(iou, golden[f"{tag}.iou"])
    assert np.array_equal(correct, golden[f"{tag}.correct"])
    meta = json.loads(str(golden["meta"]))[tag]
    if meta["pinned"] == "exact":
        assert np.array_equal(correct, golden[f"{tag}.correct_reference"])
    else:  # the reference's order inside equal-IoU runs comes from numpy's unstable sort on the generating host
        assert meta["equal_iou_runs"]
        _assert_differs_only_in_equal_iou_choice(iou, labels[:, 0], det[:, 5], correct, golden[f"{tag}.correct_reference"])


def _outcomes_over_tie_choices(iou, label_cls, det_cls, thr):
    """Every `correct` column process_batch can produce at threshold `thr` when each detection may keep ANY of its
    highest-IoU same-class labels (the freedom an unstable sort leaves), then each label keeps its lowest detection."""
    cand = (iou >= thr) & (label_cls[:, None] == det_cls[None, :])
    best = np.where(cand, iou, -1.0).max(0)
    options = [np.nonzero(cand[:, d] & (iou[:, d] == best[d]))[0] if cand[:, d].any() else np.array([], int) for d in range(iou.shape[1])]
    tied = [d for d, o in enumerate(options) if len(o) > 1]
    assert len(tied) <= 16, "too many equal-IoU choices to enumerate"
    outs = set()
    for pick in itertools.product(*(options[d] for d in tied)):
        chosen = {d: (o[0] if len(o) else -1) for d, o in enumerate(options)}
        chosen.update(zip(tied, pick))
        col = np.zeros(iou.shape[1], bool)
        claimed = set()
        for d in range(iou.shape[1]):
            if chosen[d] >= 0 and chosen[d] not in claimed:
                claimed.add(chosen[d])
                col[d] = True
        outs.add(col.tobytes())
    return outs


def _assert_differs_only_in_equal_iou_choice(iou, label_cls, det_cls, ours, ref):
    """Both results come from the same IoU matrix and the same rule up to which equal-IoU label a detection keeps: each
    column of each is one of the outcomes of some choice among equal IoUs."""
    for t, thr in enumerate(mask_val_ref.IOUV):
        outs = _outcomes_over_tie_choices(iou, label_cls, det_cls, thr)
        assert ours[:, t].tobytes() in outs and ref[:, t].tobytes() in outs, t


def test_fixture_covers_exact_half_pixels_and_equal_iou(golden):
    meta = json.loads(str(golden["meta"]))
    assert meta["down640"]["exact_half_pixels"] > 100 and meta["rect"]["exact_half_pixels"] > 100
    assert meta["dup"]["equal_iou_runs"]
    assert all(m["true_positives"] > 0 for m in meta.values())


def test_pack_bits_layout():
    m = np.zeros((2, 3, 100), np.uint8)
    m[0, 0, 0] = m[0, 0, 33] = m[1, 2, 99] = 1
    w = mask_val_ref.pack_bits(m)
    assert w.shape == (2, 16)  # 300 pixels -> 512 bits
    assert w[0, 0] == 1 and w[0, 1] == 2 and (w[0, 2:] == 0).all()
    assert w[1, 299 // 32] == 1 << (299 % 32)


def test_mask_entry_points_reject_bad_arguments_without_gpu(built_lib):
    lib = built_lib
    assert lib.y5_mask_row_words(160, 160) == 800 and lib.y5_mask_row_words(1, 1) == 8 and lib.y5_mask_row_words(1280, 1280) == 51200
    assert lib.y5_mask_row_words(0, 160) == -1
    assert lib.y5_mask_row_words(4096, 4096) == -2 and b"2^23" in lib.y5_last_error()
    u8, f32 = _lib.Y5_U8, _lib.Y5_F32
    # y5_mask_pack(src, dtype, sh, sw, overlap, target_img, target_stride, batch, n_rows, oh, ow, label_index, bits, pop, nonbinary, stream)
    assert lib.y5_mask_pack(None, u8, 160, 160, 0, None, 0, 1, 4, 160, 160, None, None, None, None, None) == -1
    assert lib.y5_mask_pack(4096, u8, 160, 160, 0, None, 0, 1, 4, 160, 160, None, 4096, 4096, None, None) == -1  # no counter
    assert lib.y5_mask_pack(4096, u8, 640, 640, 0, None, 0, 1, 4, 4096, 4096, None, 4096, 4096, 4096, None) == -2
    assert lib.y5_mask_pack(4096, 9, 160, 160, 0, None, 0, 1, 4, 160, 160, None, 4096, 4096, 4096, None) == -2  # dtype
    assert lib.y5_mask_pack(4096, f32, 160, 160, 1, 4096, 6, 2, 4, 160, 160, None, 4096, 4096, 4096, None) == -1  # no label_index
    assert lib.y5_mask_pack(None, f32, 160, 160, 0, None, 0, 1, 0, 160, 160, None, None, None, None, None) == 0  # nothing to do
    assert lib.y5_mask_pack(4096, f32, 160, 160, 0, None, 6, 2, 4, 160, 160, 4096, 4096, 4096, 4096, None) == -1  # rows need targets
    assert lib.y5_mask_pack(None, f32, 160, 160, 1, None, 6, 0, 0, 160, 160, 4096, None, None, None, None) == -1  # label_index, no images
    # y5_mask_iou(gt, gt_pop, label_index, n_gt, pred, pred_pop, count, img0, n_img, rows_per_image, words, eps, iou, stream)
    assert lib.y5_mask_iou(None, None, None, 3, None, None, None, 0, 1, 5, 800, 1e-7, None, None) == -1
    assert lib.y5_mask_iou(4096, 4096, None, 3, 4096, 4096, None, 0, 1, 5, 801, 1e-7, 4096, None) == -1  # not whole K tiles
    assert lib.y5_mask_iou(4096, 4096, None, 3, 4096, 4096, None, 0, 1, 5, (1 << 23) // 32 + 8, 1e-7, 4096, None) == -2
    assert lib.y5_mask_iou(4096, 4096, None, 3, 4096, 4096, None, 0, 2, 5, 800, 1e-7, 4096, None) == -1  # batch needs label_index
    # y5_mask_match_batch(det, img_stride, row_stride, count, batch, max_det, label_cls, cls_stride, label_index, nt, iou, iouv, niou,
    #                     correct, stream)
    assert lib.y5_mask_match_batch(None, 1800, 6, None, 1, 300, 4096, 5, None, 3, 4096, 4096, 10, 4096, None) == -1
    assert lib.y5_mask_match_batch(4096, 1800, 6, None, 1, 300, None, 5, None, 3, 4096, 4096, 10, 4096, None) == -1
    assert lib.y5_mask_match_batch(4096, 30000, 6, None, 1, 5000, 4096, 5, None, 3, 4096, 4096, 10, 4096, None) == -2
    assert lib.y5_mask_match_batch(4096, 1800, 6, None, 2, 300, 4096, 6, None, 3, 4096, 4096, 10, 4096, None) == -1
    assert ctypes.c_int32(lib.y5_mask_match_batch(4096, 1800, 6, None, 0, 300, None, 6, None, 0, None, None, 10, None, None)).value == 0


def test_seg_val_batch_metrics_rejects_mismatched_shapes():
    """Checked before anything reaches the device: the kernels index one mask plane per image (overlap) or per target."""
    from yolov5_b200.utils.metrics import seg_val_batch_metrics

    b, md = 3, 10
    rows, count, protos = torch.zeros(b, md, 38), torch.full((b,), md, dtype=torch.int32), torch.zeros(b, 32, 16, 16)
    tg = torch.tensor([[0, 1, 32, 32, 10, 10], [1, 2, 20, 20, 8, 8], [1, 0, 40, 40, 8, 8], [2, 0, 30, 30, 6, 6]], dtype=torch.float32)
    iouv = torch.linspace(0.5, 0.95, 10)
    args = (rows, count, protos, tg)
    with pytest.raises(ValueError, match="one mask per target"):
        seg_val_batch_metrics(*args, torch.zeros(b, 64, 64), (64, 64), [((64, 64),)] * b, iouv, False)
    with pytest.raises(ValueError, match="one index image per image"):
        seg_val_batch_metrics(*args, torch.zeros(len(tg), 64, 64), (64, 64), [((64, 64),)] * b, iouv, True)
    with pytest.raises(ValueError, match="columns"):
        seg_val_batch_metrics(rows[..., :37], count, protos, tg, torch.zeros(b, 64, 64), (64, 64), [((64, 64),)] * b, iouv, True)
    with pytest.raises(ValueError, match="columns"):
        seg_val_batch_metrics(rows, count, protos[:2], tg, torch.zeros(b, 64, 64), (64, 64), [((64, 64),)] * b, iouv, True)


def test_public_signatures():
    from yolov5_b200.utils import metrics

    assert str(inspect.signature(metrics.mask_iou)) == "(mask1, mask2, eps=1e-07)"
    assert str(inspect.signature(metrics.process_batch)) == "(detections, labels, iouv, pred_masks=None, gt_masks=None, overlap=False, masks=False)"
    params = list(inspect.signature(metrics.seg_val_batch_metrics).parameters)
    assert params == ["rows", "count", "protos", "targets", "masks", "im_shape", "shapes", "iouv", "overlap", "native", "check"]
