"""Generate tests/golden/mask_val.npz by running the UNMODIFIED reference's process_batch(masks=True) (utils/metrics.py:224-265)
through tests/golden/refshim.py, with ultralytics' mask_iou restated from its public definition and injected into the shimmed
`ultralytics.utils.metrics` before the reference imports it.

Runs only where the reference tree exists:
    python tests/golden/make_mask_val_golden.py
The inputs of every case are regenerated from the seeds in tests/mask_val_ref.py `CASES`, so mask_val.npz holds only outputs.
While generating, the oracle (tests/mask_val_ref.py) is checked against the reference (hard assert):
- replaying the reference's own sort, it must agree exactly on every case;
- with the engine's rule (first label in target order on equal IoU) it must agree on every case without equal-IoU runs; cases
  where the two differ are recorded in `meta` as pinned "up to the label order inside equal-IoU runs".
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from tests import mask_val_ref  # noqa: E402


def mask_iou(mask1, mask2, eps=1e-7):
    """ultralytics.utils.metrics.mask_iou (public definition): (N, n) x (M, n) -> (N, M)."""
    intersection = torch.matmul(mask1, mask2.T).clamp_(0)
    union = (mask1.sum(1)[:, None] + mask2.sum(1)[None]) - intersection
    return intersection / (union + eps)


def main():
    sys.path.insert(0, HERE)
    import refshim

    refshim.install()
    import ultralytics.utils.metrics as um

    um.mask_iou = mask_iou
    from utils.metrics import process_batch

    store, meta = {}, {}
    iouv = torch.from_numpy(mask_val_ref.IOUV)
    for tag in mask_val_ref.CASES:
        det, labels, pred, gt, overlap = mask_val_ref.case_inputs(tag)
        ref = process_batch(torch.from_numpy(det), torch.from_numpy(labels), iouv, torch.from_numpy(pred), torch.from_numpy(gt),
                            overlap=overlap, masks=True).numpy()
        replay, iou, _, vals = mask_val_ref.process_batch_masks(det, labels, mask_val_ref.IOUV, pred, gt, overlap, replay_reference_sort=True)
        assert np.array_equal(ref, replay), (tag, "oracle (reference sort) != reference")
        ours = mask_val_ref.process_batch_masks(det, labels, mask_val_ref.IOUV, pred, gt, overlap)[0]
        ties = any(len(np.unique(col[col > 0])) < int((col > 0).sum()) for col in iou.T)
        if not np.array_equal(ours, ref):
            assert ties, (tag, "oracle differs from the reference without equal IoUs")
        half = int((vals == 0.5).sum()) if vals is not None else 0
        meta[tag] = dict(pinned="exact" if np.array_equal(ours, ref) else "exact up to the label order inside equal-IoU runs",
                         equal_iou_runs=bool(ties), exact_half_pixels=half, true_positives=int(ours.sum()))
        store[f"{tag}.correct"] = ours
        store[f"{tag}.correct_reference"] = ref
        store[f"{tag}.iou"] = iou
        print(f"mask val {tag}: {meta[tag]}")
    store["meta"] = np.array(json.dumps(meta, sort_keys=True))
    np.savez_compressed(f"{HERE}/mask_val.npz", **store)
    print("written", f"{HERE}/mask_val.npz", os.path.getsize(f"{HERE}/mask_val.npz"), "bytes")


if __name__ == "__main__":
    main()
