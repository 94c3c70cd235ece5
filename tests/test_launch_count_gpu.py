"""GPU: y5_launch_count() per call of the entry points that launch more than one kernel or a shape-dependent number of
kernels.  bench.py reports the counter (gpu_launches, launches_per_forward), so each number here is the count of kernels
the entry point launches on that path: one more or one fewer kernel changes it."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import loss_ref, model_ref, pre_ref
from tests.golden import make_seg_golden as mg
from yolov5_b200 import _lib
from yolov5_b200.cfg import HYP_SCRATCH_LOW, model_cfg

pytestmark = pytest.mark.gpu


def _launches(fn):
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    fn()
    torch.cuda.synchronize()
    return _lib.launch_count() - n0


def _st(dev):
    return C.c_void_p(_lib.stream_ptr(dev))


@pytest.mark.parametrize("max_nms,want", [(30000, 5), (10, 11)])
def test_nms_batched(cuda, max_nms, want):
    """Without the max_nms cut: pass, scan, pass, sort, greedy.  With it: six more (two pick rounds and a rescan)."""
    lib = _lib.lib()
    pred = torch.from_numpy(np.random.RandomState(0).uniform(0, 1, (2, 200, 85)).astype(np.float32)).to(cuda, torch.float16)
    p = _lib.NmsParams()
    p.batch, p.n_rows, p.no, p.nc, p.nm = 2, 200, 85, 80, 0
    p.dtype = _lib.dtype_code(pred.dtype)
    p.conf_thres, p.iou_thres, p.max_det, p.max_nms, p.max_wh = 0.25, 0.45, 300, max_nms, 7680.0
    need = lib.y5_nms_workspace_bytes(C.byref(p))
    ws = torch.empty(need + 256, dtype=torch.uint8, device=cuda)
    rows = torch.empty(2, 300, 6, device=cuda)
    idx = torch.empty(2, 300, dtype=torch.int64, device=cuda)
    count = torch.empty(2, dtype=torch.int32, device=cuda)
    run = lambda: _lib.check(lib.y5_nms_batched(C.byref(p), pred.data_ptr(), rows.data_ptr(), idx.data_ptr(), count.data_ptr(),  # noqa: E731
                                                (ws.data_ptr() + 255) & ~255, need, _st(cuda)), "nms_batched")
    assert _launches(run) == want


def test_loss_fwd_bwd_scaled(cuda):
    from yolov5_b200.models.yolo import DetectionModel
    from yolov5_b200.utils.loss import ComputeLoss

    m = DetectionModel("yolov5n")
    m.load_state_dict(model_ref.synth_state_dict(model_cfg("yolov5n"), seed=30))
    m.hyp = dict(HYP_SCRATCH_LOW)
    crit = ComputeLoss(m.to(cuda))
    g = torch.Generator().manual_seed(1)
    p = [torch.randn(2, 3, s, s, 85, generator=g).to(cuda) for s in (8, 4, 2)]
    tgt = torch.from_numpy(loss_ref.synth_targets(2, seed=2)).float().to(cuda)
    assert _launches(lambda: crit._run(p, tgt, want_grad=True)) == 6


@pytest.mark.parametrize("want_grad,want", [(True, 11), (False, 10)])
def test_seg_loss_fwd_bwd_scaled(cuda, want_grad, want):
    """The detection loss's 6, then prep, bucket, match, finalize, and the proto-gradient kernel when grad_proto is given."""
    from yolov5_b200.utils.segment.loss import ComputeLoss

    p_np, proto_np, tg, masks, overlap, nc = mg.case_inputs("ov_sorted")
    crit = ComputeLoss(mg.LossModel(nc).to(cuda), overlap=overlap)
    p = [torch.from_numpy(a).to(cuda) for a in p_np]
    proto, tg, masks = torch.from_numpy(proto_np).to(cuda), torch.from_numpy(tg).to(cuda), torch.from_numpy(masks).to(cuda)
    assert _launches(lambda: crit._run(p, proto, tg, masks, want_grad=want_grad)) == want


@pytest.mark.parametrize("rows,sets,want", [(50, 1, 23), (50, 2, 25), (0, 1, 3)])
def test_ap_per_class(cuda, rows, sets, want):
    """setup, gather, 6 radix passes of 3 kernels, permute, then class + tail per set; with no rows only setup and the sets."""
    from yolov5_b200.utils.metrics import _ap_flat

    rs = np.random.RandomState(3)
    tps = [torch.from_numpy(rs.rand(rows, 10) < 0.5).to(cuda) for _ in range(sets)]
    conf = torch.from_numpy(rs.rand(rows).astype(np.float32)).to(cuda)
    pred_cls = torch.from_numpy(rs.randint(0, 5, rows).astype(np.float32)).to(cuda)
    target_cls = torch.from_numpy(rs.randint(0, 5, 20).astype(np.float32)).to(cuda)
    assert _launches(lambda: _ap_flat(tps, conf, pred_cls, target_cls, 1e-16)) == want


@pytest.mark.parametrize("entry,want", [("y5_sppf_pool_bwd", 5), ("y5_spp_pool_bwd", 2)])
def test_pool_bwd(cuda, entry, want):
    b, h, w, c = 2, 8, 8, 16
    lib = _lib.lib()
    cat = torch.randn(b, h, w, 4 * c, device=cuda).half()
    dcat = torch.randn(b, h, w, 4 * c, device=cuda).half()
    da = torch.empty(b, h, w, c, dtype=torch.float16, device=cuda)
    ws = torch.empty(3 * b * h * w * c, dtype=torch.float32, device=cuda)
    fn = getattr(lib, entry)
    run = lambda: _lib.check(fn(cat.data_ptr(), 4 * c, dcat.data_ptr(), 4 * c, da.data_ptr(), c, b, h, w, c, 5, _lib.Y5_F16, ws.data_ptr(),  # noqa: E731
                                _st(cuda)), entry)
    assert _launches(run) == want


@pytest.mark.parametrize("entry", ["y5_bn_act_bwd", "y5_bn_act_bwd_reduce", "y5_col_sum"])
def test_bn_two_kernel_passes(cuda, entry):
    """bn_act_bwd: reduce + apply; bn_act_bwd_reduce: reduce + affine gradient; col_sum: column stats + finalize."""
    lib = _lib.lib()
    rows, ch = 256, 32
    y, dz, dy = (torch.randn(rows, ch, device=cuda).half() for _ in range(3))
    mean, invstd, gamma, beta, dg, db = (torch.rand(ch, device=cuda) + 0.5 for _ in range(6))
    ws = torch.zeros(2 * ch + 1, dtype=torch.float64, device=cuda)
    if entry == "y5_col_sum":
        run = lambda: _lib.check(lib.y5_col_sum(y.data_ptr(), ch, rows, ch, _lib.Y5_F16, dg.data_ptr(), ws.data_ptr(), _st(cuda)), entry)  # noqa: E731
    else:
        fn = getattr(lib, entry)
        run = lambda: _lib.check(fn(y.data_ptr(), ch, dz.data_ptr(), ch, dy.data_ptr(), ch, rows, ch, _lib.Y5_F16, mean.data_ptr(),  # noqa: E731
                                    invstd.data_ptr(), gamma.data_ptr(), beta.data_ptr(), 1, 0.0, dg.data_ptr(), db.data_ptr(),
                                    ws.data_ptr(), _st(cuda)), entry)
    assert _launches(run) == 2


@pytest.mark.parametrize("upsample,native,want", [(False, False, 1), (True, False, 2), (False, True, 2)])
def test_process_mask(cuda, upsample, native, want):
    """Mode 0 (mask resolution): one kernel.  Modes 1 (up-sampled) and 2 (native): low-resolution masks, then the up-sampling kernel."""
    from yolov5_b200.utils.segment.general import process_mask_batch

    rs = np.random.RandomState(4)
    protos = torch.from_numpy(rs.randn(1, 32, 16, 16).astype(np.float32)).to(cuda)
    coef = torch.from_numpy(rs.randn(3, 32).astype(np.float32)).to(cuda)
    boxes = torch.tensor([[4, 4, 40, 30], [0, 0, 64, 64], [10, 20, 50, 60]], dtype=torch.float32, device=cuda)
    assert _launches(lambda: process_mask_batch(protos, coef, boxes, None, (64, 64), upsample=upsample, native=native)) == want


def test_letterbox_chunks(cuda):
    """One launch per chunk of y5_letterbox_max_images() images."""
    from yolov5_b200.utils.augmentations import letterbox_batch

    per = _lib.lib().y5_letterbox_max_images()
    ims = [torch.from_numpy(pre_ref.synth_image(40, 50, i)).to(cuda) for i in range(per + 1)]
    assert _launches(lambda: letterbox_batch(ims, (64, 64), auto=False)) == 2
