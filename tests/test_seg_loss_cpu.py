"""CPU: the segmentation-loss oracle vs the reference fixture (tests/golden/seg_loss.npz), the drop-in interface
(signatures, the utils.segment.loss alias) and the host-side shape checks that run before any kernel launch."""
import inspect
import json
import os
import sys

import numpy as np
import pytest
import torch

from tests import seg_loss_ref
from tests.golden import make_seg_golden as mg
from yolov5_b200.cfg import HYP_SCRATCH_LOW
from yolov5_b200.utils.segment.loss import ComputeLoss

G = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(G, "seg_loss.npz"))


@pytest.mark.parametrize("tag", list(mg.CASES))
def test_oracle_matches_reference_fixture(golden, tag):
    p_np, proto_np, tg, masks, overlap, nc = mg.case_inputs(tag)
    anchors = mg.anchors_grid()
    bt = seg_loss_ref.build_targets_seg(tg, anchors.numpy(), [tuple(a.shape[2:4]) for a in p_np], p_np[0].shape[0], overlap)
    for i in range(3):
        d = bt[i]
        got = np.stack([d["b"], d["a"], d["gj"], d["gi"], d["tcls"], d["tidx"]])
        assert got.dtype == np.int64 and np.array_equal(got, golden[f"{tag}.idx{i}"]), (tag, i)
        assert np.array_equal(d["tbox"], golden[f"{tag}.tbox{i}"]) and np.array_equal(d["xywhn"], golden[f"{tag}.xywhn{i}"])
        assert np.array_equal(d["anch"], golden[f"{tag}.anch{i}"])
    p = [torch.from_numpy(a).requires_grad_(True) for a in p_np]
    proto = torch.from_numpy(proto_np).requires_grad_(True)
    loss, items = seg_loss_ref.compute_seg_loss(p, proto, tg, masks, anchors, HYP_SCRATCH_LOW, overlap)
    loss.backward()
    np.testing.assert_allclose(np.concatenate((loss.detach().numpy(), items.numpy())), golden[f"{tag}.loss"], rtol=1e-5, atol=1e-6)
    for i, a in enumerate(p):
        np.testing.assert_allclose(a.grad.numpy(), golden[f"{tag}.grad{i}"], rtol=1e-4, atol=1e-7)
    gp = proto.grad.numpy() if proto.grad is not None else np.zeros_like(proto_np)
    np.testing.assert_allclose(gp, golden[f"{tag}.grad_proto"], rtol=1e-4, atol=1e-7)


def test_signatures_match_the_reference():
    with open(os.path.join(G, "seg_signatures.json")) as f:
        ref = json.load(f)
    for name, theirs in ref.items():
        mine = [(n, repr(q.default) if q.default is not inspect._empty else None, str(q.kind))
                for n, q in inspect.signature(getattr(ComputeLoss, name)).parameters.items()]
        assert mine == [tuple(x) for x in theirs], name


def test_compat_alias_serves_the_engine_loss():
    from yolov5_b200 import compat

    saved = {k: sys.modules.get(k) for k in compat.ALIASES}
    try:
        assert compat.install()
        from utils.segment.loss import ComputeLoss as Aliased

        assert Aliased is ComputeLoss
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def _crit(overlap, nc=80):
    return ComputeLoss(mg.LossModel(nc), overlap=overlap)


def _inputs(bs=2, nm=32, nc=80, mh=16, mw=16):
    p = [torch.zeros(bs, 3, 64 // s, 64 // s, 5 + nc + nm) for s in (8, 16, 32)]
    tg = torch.tensor([[0, 1, 0.5, 0.5, 0.2, 0.2], [1, 2, 0.4, 0.4, 0.3, 0.1], [1, 3, 0.6, 0.6, 0.1, 0.3]])
    return p, torch.zeros(bs, nm, mh, mw), tg


def test_cpu_tensors_raise():
    p, proto, tg = _inputs()
    with pytest.raises(RuntimeError, match="CUDA"):
        _crit(True)((p, proto), tg, torch.zeros(2, 16, 16))


@pytest.mark.parametrize("overlap,masks_shape,proto_shape,match", [
    (True, (3, 16, 16), None, "per image"),           # overlap: one map per image
    (False, (2, 16, 16), None, "masks for 3 targets"),  # non-overlap: one mask per target row
    (True, (2, 16), None, "N, H, W"),
    (True, (1, 2, 16, 16), None, "N, H, W"),
    (True, (2, 16, 16), (2, 16, 16, 16), "proto"),    # wrong nm
    (True, (2, 16, 16), (3, 32, 16, 16), "proto"),    # wrong batch
    (True, (2, 16, 16), (2, 32, 16), "proto"),
])
def test_malformed_shapes_raise_value_error(overlap, masks_shape, proto_shape, match):
    p, proto, tg = _inputs()
    if proto_shape is not None:
        proto = torch.zeros(*proto_shape)
    with pytest.raises(ValueError, match=match):
        _crit(overlap)((p, proto), tg, torch.zeros(*masks_shape))


def test_malformed_head_maps_raise_value_error():
    p, proto, tg = _inputs()
    with pytest.raises(ValueError, match="head map"):
        _crit(True)(([q[..., :-1] for q in p], proto), tg, torch.zeros(2, 16, 16))
    with pytest.raises(ValueError, match="head maps"):
        _crit(True)((p[:2], proto), tg, torch.zeros(2, 16, 16))


def test_unsupported_options_raise():
    with pytest.raises(NotImplementedError):
        ComputeLoss(mg.LossModel(80), autobalance=True)
    m = mg.LossModel(80)
    m.hyp["fl_gamma"] = 1.5
    with pytest.raises(NotImplementedError):
        ComputeLoss(m)
    c = _crit(True)
    assert (c.overlap, c.nm, c.na, c.nc, c.nl, c.sort_obj_iou, c.gr) == (True, 32, 3, 80, 3, False, 1.0)
    assert c.balance == [4.0, 1.0, 0.4] and c.hyp is not None and tuple(c.anchors.shape) == (3, 3, 2)
