"""CPU: the float64 detection-loss reference (tests/loss64_ref.py) against the fixture the real reference produced
(tests/golden/loss.npz) and against full float64 autograd through oracle.loss_ref.compute_loss; the host-side shape
checks ComputeLoss runs before any launch."""
import os

import numpy as np
import pytest
import torch

from oracle import loss_ref
from tests import loss64_ref as R
from tests.golden import make_seg_golden as mg
from yolov5_b200.cfg import HYP_SCRATCH_LOW
from yolov5_b200.utils.loss import ComputeLoss

G = os.path.join(os.path.dirname(__file__), "golden")
TERMS = {"xy": slice(0, 2), "wh": slice(2, 4), "obj": slice(4, 5), "cls": slice(5, None)}


def _maps(bs, h, w, no, seed, scale=1.5):
    rs = np.random.RandomState(seed)
    return [rs.normal(0, scale, (bs, 3, h // s, w // s, no)).astype(np.float32) for s in (8, 16, 32)]


def _ref(pn, tg, hyp, nc, dtype=torch.float64, scale=1.0):
    bs = pn[0].shape[0]
    shapes = [tuple(a.shape[2:4]) for a in pn]
    bt = R.targets_for(tg, mg.anchors_grid().numpy(), shapes, bs, hyp["anchor_t"])
    obj, rows = R.leaves_from_maps([torch.from_numpy(a) for a in pn], bt)
    res = R.loss64(obj, rows, bt, hyp, nc, bs, dtype=dtype, scale=scale)
    return res, R.dense_grad(res, bt, shapes, bs, 3, pn[0].shape[-1]), bt


@pytest.mark.parametrize("tag", ["a", "b", "none"])
def test_reproduces_reference_fixture(tag):
    """Loss and items equal the real reference's (fp32) to rtol 2e-5; the gradients equal loss_ref's fp32 autograd per level
    and per term within fp32 rounding of that term's largest gradient."""
    g = np.load(os.path.join(G, "loss.npz"))
    bs, h, w, seed = (int(v) for v in g[f"{tag}.meta"])
    rs = np.random.RandomState(seed)
    pn = [rs.normal(0, 1.5, (bs, 3, h // s, w // s, 85)).astype(np.float32) for s in (8, 16, 32)]
    tg = loss_ref.synth_targets(bs, seed) if tag != "none" else np.zeros((0, 6), np.float32)
    res, dense, bt = _ref(pn, tg, HYP_SCRATCH_LOW, 80)
    for i, d in enumerate(bt):
        got = np.stack([d["b"], d["a"], d["gj"], d["gi"], d["tcls"]])
        assert np.array_equal(got, g[f"{tag}.idx{i}"]) and np.array_equal(d["tbox"], g[f"{tag}.tbox{i}"]), (tag, i)
    np.testing.assert_allclose(np.concatenate(([res["loss"]], res["items"].numpy())), g[f"{tag}.loss"], rtol=2e-5, atol=1e-7)
    p32 = [torch.from_numpy(a).requires_grad_(True) for a in pn]
    lo, _ = loss_ref.compute_loss(p32, tg, mg.anchors_grid(), HYP_SCRATCH_LOW)
    lo.backward()
    for i, (a, e) in enumerate(zip(p32, dense)):
        for term, sl in TERMS.items():
            got, ref = a.grad[..., sl].double(), e[..., sl]
            s = float(ref.abs().max())
            assert float((got - ref).abs().max()) <= 1e-5 * s + 1e-12, (tag, i, term)


def _dup_targets(bs):
    """synth targets plus rows that share cells: identical rows and other classes at one position."""
    tg = loss_ref.synth_targets(bs, 11, nc=80)
    extra = np.array([[0, 3, 0.41, 0.52, 0.2, 0.3], [0, 3, 0.41, 0.52, 0.2, 0.3], [0, 9, 0.41, 0.52, 0.2, 0.3],
                      [1, 0, 0.41, 0.52, 0.21, 0.29]], np.float32)
    return np.concatenate((tg, extra), 0)


SMALL = {
    # tag: (nc, hyp overrides, targets, box logits zeroed in image 0)
    "dup": (80, {}, lambda: _dup_targets(2), False),
    "nc1": (1, {}, lambda: loss_ref.synth_targets(2, 12, nc=1), False),
    "smooth_pw": (3, {"label_smoothing": 0.1, "cls_pw": 1.3, "obj_pw": 1.3}, lambda: loss_ref.synth_targets(2, 13, nc=3), False),
    "edges": (80, {}, R.edge_targets, False),
    "ties": (80, {}, lambda: np.concatenate((R.tie_targets(), R.tie_targets()[:1], loss_ref.synth_targets(2, 14)[-5:])), True),
}


@pytest.mark.parametrize("tag", list(SMALL))
def test_restricted_leaves_equal_full_autograd(tag):
    """The (obj planes, unique rows) bookkeeping gives the gradient of full float64 autograd through loss_ref.compute_loss:
    duplicates summed, last-writer tobj, no class term at nc 1, label smoothing and pos weights, and ties."""
    nc, over, make, zero_box = SMALL[tag]
    hyp = dict(HYP_SCRATCH_LOW, **over)
    pn = _maps(2, 64, 64, 5 + nc, seed=5)
    if zero_box:
        pn[0][0, ..., 0:4] = 0
    tg = make()
    res, dense, bt = _ref(pn, tg, hyp, nc)
    assert sum(int((d["mult"] > 1).sum()) for d in bt) > 0 or tag in ("nc1", "smooth_pw")
    p64 = [torch.from_numpy(a).double().requires_grad_(True) for a in pn]
    lo, it = loss_ref.compute_loss(p64, tg, mg.anchors_grid(), hyp)
    lo.backward()
    assert abs(res["loss"] - lo.item()) <= 1e-12 * abs(lo.item())
    assert torch.allclose(res["items"], it.double(), rtol=1e-12, atol=1e-15)
    for i, (a, e) in enumerate(zip(p64, dense)):
        assert float((a.grad - e).abs().max()) <= 1e-12 * float(e.abs().max()) + 1e-18, (tag, i)
    if nc == 1:
        assert float(res["items"][2]) == 0.0 and all(not g[:, 5].any() for g in res["grows"])


def test_upstream_scale_and_rounded_tobj():
    """`scale` multiplies every gradient; `dtype` rounds only the objectness target."""
    pn = _maps(2, 64, 64, 85, seed=6)
    tg = loss_ref.synth_targets(2, 15)
    a, _, _ = _ref(pn, tg, HYP_SCRATCH_LOW, 80)
    b, _, _ = _ref(pn, tg, HYP_SCRATCH_LOW, 80, scale=8.0)
    c, _, _ = _ref(pn, tg, HYP_SCRATCH_LOW, 80, dtype=torch.bfloat16)
    for i in range(3):
        assert torch.equal(a["grows"][i] * 8, b["grows"][i]) and torch.equal(a["gobj"][i] * 8, b["gobj"][i])
        assert torch.equal(c["tobj"][i], a["tobj"][i].to(torch.bfloat16).double())
        assert torch.equal(c["grows"][i], a["grows"][i])


def test_tie_gradient_follows_torch():
    """Logits 0 on a target equal to the predicted box: the IoU is at its maximum, so torch's w / h gradient is ~0 (the
    first-operand rule for min / max would give about -1 per unit of box gain)."""
    pn = _maps(2, 64, 64, 85, seed=8)
    pn[0][0, ..., 0:4] = 0
    tg = R.tie_targets()[:1]
    res, _, bt = _ref(pn, tg, HYP_SCRATCH_LOW, 80)
    d = bt[0]
    k = int(np.nonzero((d["a"] == 0) & (d["gi"] == 2) & (d["gj"] == 3))[0][0])
    g = res["grows"][0][d["inv"][k]]
    gbox = HYP_SCRATCH_LOW["box"] * 2 / len(d["b"])  # d loss / d (1 - iou) of one match
    assert float(g[2:4].abs().max()) < 1e-6 * gbox and float(g[0:2].abs().max()) == 0.0


# -------------------------------------------------------------------------------------------------------------------
# host-side shape checks: they run before the CUDA-only check, so CPU tensors reach them
# -------------------------------------------------------------------------------------------------------------------
def _inputs(bs=2, nc=80, dtype=torch.float32):
    p = [torch.zeros(bs, 3, 64 // s, 64 // s, 5 + nc, dtype=dtype) for s in (8, 16, 32)]
    return p, torch.tensor([[0, 1, 0.5, 0.5, 0.2, 0.2], [1, 2, 0.4, 0.4, 0.3, 0.1]])


def test_cpu_tensors_raise():
    p, tg = _inputs()
    with pytest.raises(RuntimeError, match="CUDA"):
        ComputeLoss(mg.LossModel(80))(p, tg)


@pytest.mark.parametrize("mutate,match", [
    (lambda p, t: (p[:2], t), "head maps"),
    (lambda p, t: (p + p[:1], t), "head maps"),
    (lambda p, t: ([p[0], p[1][:1], p[2]], t), "head map"),                      # another batch
    (lambda p, t: ([p[0], p[1][:, :2], p[2]], t), "head map"),                   # na 2
    (lambda p, t: ([p[0], p[1], p[2][..., :-1]], t), "head map"),                # no 84
    (lambda p, t: ([q[..., :-1] for q in p], t), "head map"),                    # no 84 everywhere
    (lambda p, t: ([p[0], p[1][0], p[2]], t), "head map"),                       # 4-D
    (lambda p, t: ([p[0].half(), p[1].half(), p[2]], t), "dtype"),               # one fp32 level among fp16
    (lambda p, t: (p, torch.zeros(6, 7)), "targets"),                            # 42 elements: divisible by 6
    (lambda p, t: (p, t.reshape(-1)), "targets"),
    (lambda p, t: (p, t[None]), "targets"),
])
def test_malformed_inputs_raise_value_error(mutate, match):
    p, tg = _inputs()
    p, tg = mutate(p, tg)
    with pytest.raises(ValueError, match=match):
        ComputeLoss(mg.LossModel(80))(p, tg)
    with pytest.raises(ValueError, match=match):
        ComputeLoss(mg.LossModel(80)).build_targets(p, tg)


def test_nc1_head_maps_have_six_channels():
    p, tg = _inputs(nc=1)
    with pytest.raises(RuntimeError, match="CUDA"):
        ComputeLoss(mg.LossModel(1))(p, tg)
    with pytest.raises(ValueError, match="head map"):
        ComputeLoss(mg.LossModel(1))(_inputs(nc=80)[0], tg)
