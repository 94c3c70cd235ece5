"""GPU: ComputeLoss (y5_loss_fwd_bwd_scaled) vs the oracle: build_targets bit-exact (int64 indices, order, fp32 tbox);
loss / items / gradients within fp32 tolerance (rtol 1e-4) for fp32 logits, 2e-3 for fp16 logits."""
import os

import numpy as np
import pytest
import torch

from oracle import loss_ref, model_ref
from yolov5_b200.cfg import HYP_SCRATCH_LOW, model_cfg
from yolov5_b200.models.yolo import DetectionModel
from yolov5_b200.utils.loss import ComputeLoss

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")


def _setup(dev):
    m = DetectionModel("yolov5n")
    m.load_state_dict(model_ref.synth_state_dict(model_cfg("yolov5n"), seed=30))
    m.hyp = dict(HYP_SCRATCH_LOW)
    return m.to(dev), ComputeLoss(m.to(dev))


@pytest.mark.parametrize("tag", ["a", "b", "none"])
def test_loss_and_targets_vs_golden_fp32(cuda, tag):
    g = np.load(os.path.join(G, "loss.npz"))
    m, crit = _setup(cuda)
    anchors = m.model[-1].anchors.detach().cpu().numpy()
    bs, h, w, seed = (int(v) for v in g[f"{tag}.meta"])
    rs = np.random.RandomState(seed)
    pn = [rs.normal(0, 1.5, (bs, 3, h // s, w // s, 85)).astype(np.float32) for s in (8, 16, 32)]
    tg = loss_ref.synth_targets(bs, seed) if tag != "none" else np.zeros((0, 6), np.float32)
    p = [torch.from_numpy(a).to(cuda).requires_grad_(True) for a in pn]
    tcls, tbox, indices, anch = crit.build_targets(p, torch.from_numpy(tg).to(cuda))
    for i in range(3):
        ref = g[f"{tag}.idx{i}"]
        got = np.stack([indices[i][q].cpu().numpy() for q in range(4)] + [tcls[i].cpu().numpy()])
        assert got.dtype == np.int64 and np.array_equal(got, ref), (tag, i)
        assert np.array_equal(tbox[i].cpu().numpy(), g[f"{tag}.tbox{i}"]), (tag, i)
    loss, items = crit(p, torch.from_numpy(tg).to(cuda))
    loss.backward()
    ref = g[f"{tag}.loss"]
    np.testing.assert_allclose(np.concatenate((loss.detach().cpu().numpy(), items.cpu().numpy())), ref, rtol=1e-4, atol=1e-6)
    p2 = [torch.from_numpy(a).requires_grad_(True) for a in pn]
    lo, _ = loss_ref.compute_loss(p2, tg, anchors, HYP_SCRATCH_LOW)
    lo.backward()
    for a, b in zip(p, p2):
        ga, gb = a.grad.cpu(), b.grad
        assert float((ga - gb).abs().max()) <= 1e-4 * float(gb.abs().max()) + 1e-9, tag


def test_loss_fp16_logits_and_upstream_scale(cuda):
    m, crit = _setup(cuda)
    anchors = m.model[-1].anchors.detach().cpu().numpy()
    rs = np.random.RandomState(40)
    pn = [rs.normal(0, 1.5, (8, 3, 64 // s, 96 // s, 85)).astype(np.float32) for s in (8, 16, 32)]
    tg = loss_ref.synth_targets(8, 41)
    ph = [torch.from_numpy(a).to(cuda).half().requires_grad_(True) for a in pn]
    loss, items = crit(ph, torch.from_numpy(tg).to(cuda))
    (loss * 8.0).backward()  # e.g. WORLD_SIZE scaling at train.py:405
    p2 = [torch.from_numpy(a).half().float().requires_grad_(True) for a in pn]
    lo, it = loss_ref.compute_loss(p2, tg, anchors, HYP_SCRATCH_LOW)
    (lo * 8.0).backward()
    assert abs(loss.item() - lo.item()) <= 2e-3 * abs(lo.item())
    np.testing.assert_allclose(items.cpu().numpy(), it.numpy(), rtol=2e-3, atol=1e-5)
    for a, b in zip(ph, p2):
        assert float((a.grad.float().cpu() - b.grad).abs().max()) <= 3e-3 * float(b.grad.abs().max())
