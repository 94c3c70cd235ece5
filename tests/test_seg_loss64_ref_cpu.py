"""CPU: the float64 segmentation-loss reference (tests/seg_loss64_ref.py) against the fixture the real reference produced
(tests/golden/seg_loss.npz), against full float64 autograd through tests/seg_loss_ref.py's expressions, and the
sensitivity of its bound check: every deliberately wrong variant of the mask term in `MUTATIONS` is rejected at the
shapes the GPU suite runs."""
import os

import numpy as np
import pytest
import torch

from tests import loss64_ref as R
from tests import seg_loss64_ref as S
from tests import seg_loss_ref
from tests.golden import make_seg_golden as mg
from yolov5_b200.cfg import HYP_SCRATCH_LOW

G = os.path.join(os.path.dirname(__file__), "golden")


def _terms(nc):
    return {"xy": slice(0, 2), "wh": slice(2, 4), "obj": slice(4, 5), "cls": slice(5, 5 + nc), "mask": slice(5 + nc, None)}


def _ref(case, dtype=torch.float32, scale=1.0, mutate=()):
    p = [torch.from_numpy(a).to(dtype) for a in case["p"]]
    proto = torch.from_numpy(case["proto"]).to(dtype)
    return S.reference(p, proto, case["targets"], torch.from_numpy(case["masks"]), case["overlap"], HYP_SCRATCH_LOW,
                       dtype=dtype, scale=scale, mutate=mutate)


def _dense(res, case):
    shapes = [tuple(a.shape[2:4]) for a in case["p"]]
    return R.dense_grad(res, res["bt"], shapes, res["batch"], 3, case["p"][0].shape[-1])


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(G, "seg_loss.npz"))


@pytest.mark.parametrize("tag", list(mg.CASES))
def test_reproduces_reference_fixture(golden, tag):
    """Loss and items equal the real reference's (fp32) to rtol 2e-5; the gradients equal its fp32 autograd per level and
    per term within 1e-5 of that term's largest value, and dproto within 1e-5 of its largest value."""
    p_np, proto_np, tg, masks, overlap, nc = mg.case_inputs(tag)
    case = dict(p=p_np, proto=proto_np, targets=tg, masks=masks, overlap=overlap, nc=nc)
    res = _ref(case)
    for i, d in enumerate(res["bt"]):
        got = np.stack([d["b"], d["a"], d["gj"], d["gi"], d["tcls"], d["tidx"]])
        assert np.array_equal(got, golden[f"{tag}.idx{i}"]) and np.array_equal(d["xywhn"], golden[f"{tag}.xywhn{i}"]), (tag, i)
    got = np.concatenate(([res["loss"]], res["items"].numpy()))
    np.testing.assert_allclose(got, golden[f"{tag}.loss"], rtol=2e-5, atol=1e-7)
    for i, e in enumerate(_dense(res, case)):
        r = torch.from_numpy(golden[f"{tag}.grad{i}"]).double()
        for term, sl in _terms(nc).items():
            s = float(r[..., sl].abs().max()) if r[..., sl].numel() else 0.0
            assert float((e[..., sl] - r[..., sl]).abs().max()) <= 1e-5 * s + 1e-12, (tag, i, term)
    r = torch.from_numpy(golden[f"{tag}.grad_proto"]).double()
    assert float((res["gproto"] - r).abs().max()) <= 1e-5 * float(r.abs().max()) + 1e-12, tag


SMALL = {
    # tag: (bs, img h, img w, nm, nc, overlap, order)
    "ov-nm32": (2, 64, 96, 32, 80, True, "shuffled"),
    "ov-nm16-nc3": (2, 96, 64, 16, 3, True, "sorted"),
    "nonov-nm1-nc1": (2, 64, 96, 1, 1, False, "shuffled"),
    "nonov-nm16": (3, 64, 64, 16, 80, False, "sorted"),
}


def _small(tag, seed=5):
    bs, h, w, nm, nc, overlap, order = SMALL[tag]
    from oracle import loss_ref

    tg = loss_ref.synth_targets(bs, seed, nc)
    tg = np.concatenate((tg, np.array([[0, 0, 0.5, 0.5, 0.7, 0.6], [bs - 1, 0, 0.45, 0.55, 0.5, 0.8]], np.float32)))
    rs = np.random.RandomState(seed)
    if order == "shuffled":
        tg = tg[rs.permutation(len(tg))]
    if overlap:
        masks = seg_loss_ref.overlap_masks(tg, bs, h // 4, w // 4)
    else:
        masks = S._holes(np.stack([seg_loss_ref.paint_masks((h // 4, w // 4), tg[i:i + 1, 2:6], [1.0]) for i in range(len(tg))]), rs)
    return S._case(bs, h, w, tg, masks, overlap, nc=nc, nm=nm, seed=seed + 1)


@pytest.mark.parametrize("tag", list(SMALL))
def test_closed_form_equals_float64_autograd(tag):
    """The closed-form mask term (and the restricted detection leaves) give the loss and every gradient of float64 autograd
    through seg_loss_ref.compute_seg_loss: nm 1 / 16 / 32, nc 1 / 3 / 80, non-square protos, overlap and not."""
    case = _small(tag)
    res = _ref(case, torch.float64, scale=3.0)
    p64 = [torch.from_numpy(a).double().requires_grad_(True) for a in case["p"]]
    proto64 = torch.from_numpy(case["proto"]).double().requires_grad_(True)
    lo, it = seg_loss_ref.compute_seg_loss(p64, proto64, case["targets"], case["masks"], mg.anchors_grid(), HYP_SCRATCH_LOW,
                                           case["overlap"])
    (lo * 3.0).backward()
    assert lo.dtype == torch.float64 and abs(res["loss"] - lo.item()) <= 1e-12 * abs(lo.item())
    assert torch.allclose(res["items"], it.double(), rtol=1e-12, atol=1e-15)
    assert float(res["items"][1]) > 0
    for i, (a, e) in enumerate(zip(p64, _dense(res, case))):
        assert float((a.grad - e).abs().max()) <= 1e-12 * float(e.abs().max()) + 1e-18, (tag, i)
    assert float((proto64.grad - res["gproto"]).abs().max()) <= 1e-12 * float(res["gproto"].abs().max()), tag
    # dproto is zero exactly where no crop covers the pixel
    assert not bool(res["gproto"][res["ncover"][:, None].expand_as(res["gproto"]) == 0].any())


# ---------------------------------------------------------------------------------------------------------------------
# sensitivity: each mutation at a GPU case that reaches it, in that case's loosest dtype and scale
# ---------------------------------------------------------------------------------------------------------------------
SENS = {
    "edge_inclusive": (S.edges_case, torch.bfloat16, 8.0),
    "floor": (S.batch_layout_case, torch.float32, 1.0),
    "swap_hw": (lambda: S.rect_case(8, 320, 256), torch.float16, 65536.0 * 8),
    "tidx_own_image": (S.batch_layout_case, torch.float32, 1.0),
    "mean_crop_pixels": (S.batch_layout_case, torch.float32, 1.0),
    "mean_per_image": (S.batch_layout_case, torch.float32, 1.0),
    "nearest_round": (lambda: S.mask_ratio_case(8), torch.float16, 65536.0 * 8),
}


def test_every_mutation_has_a_case():
    assert set(SENS) == set(S.MUTATIONS)


@pytest.mark.parametrize("mutation", list(SENS))
def test_bounds_reject_each_mutation(mutation):
    make, dtype, scale = SENS[mutation]
    case = make()
    ref = _ref(case, dtype, scale)
    assert S.check(S.as_got(ref), ref) == 0.0
    bad = _ref(case, dtype, scale, mutate=(mutation,))
    worst = S.check(S.as_got(bad), ref)
    print(f"\nsensitivity {mutation:<18} worst err/bound {worst:.3g}")
    assert worst > 1.0, mutation
