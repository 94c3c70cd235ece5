"""GPU: the validation loaders (y5_val_letterbox through DeviceValLoader / DeviceSegValLoader) against the reference's
batches (tests/golden/val_load.npz) and the kernel alone against the oracle (oracle/val_load_ref.py) over a size sweep."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import pre_ref
from oracle import val_load_ref as V
from tests import val_load_fixture as F

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None
_BITS = {torch.float16: torch.int16, torch.bfloat16: torch.int16, torch.float32: torch.int32}


@pytest.fixture(scope="module")
def z():
    return F.load()


def _loader(ds, dtype=torch.uint8, workers=4):
    from yolov5_b200.utils.dataloaders import DeviceValLoader
    from yolov5_b200.utils.segment.dataloaders import DeviceSegValLoader

    cls = DeviceSegValLoader if ds.run.startswith("seg.") else DeviceValLoader
    return cls(ds, ds.batch_size, device=DEV, dtype=dtype, workers=workers, decode=F.decode)


@pytest.mark.parametrize("cache", [False, True])
@pytest.mark.parametrize("run", ["det.rect", "det.square", "det.again", "seg.o1.r1", "seg.o1.r4", "seg.o0.r1", "seg.o0.r4"])
def test_loader_reproduces_fixture(z, run, cache):
    ds = F.ValDataset(z, run, cache=cache)
    loader = _loader(ds)
    assert len(loader) == ds.n_batches
    n = 0
    for bi, batch in enumerate(loader):
        imgs, targets, shapes, masks = F.expected(z, run, bi)
        gi, gt, paths, gs = batch[:4]
        assert gi.device == DEV and gt.device == DEV and gi.dtype == torch.uint8
        assert np.array_equal(gi.cpu().numpy(), imgs), (run, bi)
        gt = gt.cpu().numpy()
        assert gt.dtype == np.float32 and gt.shape == targets.shape and np.array_equal(gt.view(np.uint32), targets.view(np.uint32)), (run, bi)
        assert F.as_json(gs) == shapes, (run, bi)
        assert list(paths) == ds.im_files[bi * ds.batch_size: bi * ds.batch_size + len(paths)]
        if masks is not None:
            gm = batch[4]
            assert gm.device == DEV
            gm = gm.cpu().numpy()
            assert gm.dtype == masks.dtype and gm.shape == masks.shape and np.array_equal(gm, masks), (run, bi, gm.dtype, masks.dtype)
        n += 1
    assert n == ds.n_batches


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
@pytest.mark.parametrize("run", ["det.rect", "det.again"])
def test_float_outputs_equal_torch_division(z, run, dtype):
    ds = F.ValDataset(z, run)
    for (u8, *_), (fl, *_) in zip(_loader(ds), _loader(ds, dtype)):
        assert fl.dtype == dtype
        want = u8.to(dtype) / 255
        assert torch.equal(fl.view(_BITS[dtype]), want.view(_BITS[dtype])), (run, dtype)


def _sweep(img_size):
    rs = np.random.RandomState(4)
    sizes = [(1280, 960), (1080, 1920), (1440, 1920), (1920, 2560), (750, 1000), (768, 1366), (1, 1000), (1000, 1), (7, 3), (480, 640),
             (640, 640), (300, 200), (427, 640)]
    sizes += [(2 * img_size, 4), (3 * img_size, 3), (4 * img_size, 8)]  # "area fast": 2 x 2, 3 x 3, 4 x 4 cells
    sizes += [(int(rs.randint(1, 1500)), int(rs.randint(1, 1500))) for _ in range(27)]
    return sizes


@pytest.mark.parametrize("img_size", [640, 1280, 333])
def test_kernel_equals_oracle_over_a_size_sweep(img_size):
    """Mixed sizes in one launch: every interpolation, the area-fast and weighted paths, and (canvas one row / column
    short of some images) letterbox's second resize through the scratch."""
    from yolov5_b200 import _lib

    rs = np.random.RandomState(img_size)
    srcs = [pre_ref.synth_image(h, w, h + 3 * w) if rs.rand() < 0.7 else rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in _sweep(img_size)]
    H, W = img_size, img_size - 1  # images whose load size is img_size wide are letterboxed again
    offs, pos = [], 0
    for s in srcs:
        offs.append(pos)
        pos += (s.nbytes + 15) // 16 * 16
    loads = [V.load_size(s.shape[:2], img_size) for s in srcs]
    scratch_offs, spos = [], pos
    for (h, w), _ in loads:
        scratch_offs.append(spos)
        spos += (h * w * 3 + 15) // 16 * 16
    host = np.zeros(spos, np.uint8)
    for o, s in zip(offs, srcs):
        host[o: o + s.nbytes] = s.reshape(-1)
    buf = torch.from_numpy(host).to(DEV)
    table = (_lib.ValImage * len(srcs))()
    want, again = [], 0
    for d, s, o, so, ((h, w), interp) in zip(table, srcs, offs, scratch_offs, loads):
        new_unpad, _, _, (top, _, left, _) = pre_ref.letterbox_geometry((h, w), (H, W), auto=False, scaleup=False)
        d.data, d.src_h, d.src_w, d.row_bytes = buf.data_ptr() + o, s.shape[0], s.shape[1], s.shape[1] * 3
        d.res_h, d.res_w, d.interp = h, w, interp
        d.new_h, d.new_w, d.top, d.left = new_unpad[1], new_unpad[0], top, left
        d.scratch = buf.data_ptr() + so
        again += tuple(new_unpad) != (w, h)
        im = V.load_resize(s, img_size)
        want.append(pre_ref.to_chw_rgb(pre_ref.letterbox(im, (H, W), auto=False, scaleup=False)[0]))
    assert again > 0
    for dtype in (torch.uint8, torch.float16, torch.float32):
        out = torch.empty(len(srcs), 3, H, W, dtype=dtype, device=DEV)
        _lib.check(_lib.lib().y5_val_letterbox(table, len(srcs), H, W, out.data_ptr(), _lib.dtype_code(dtype),
                                               ctypes.c_void_p(_lib.stream_ptr(DEV))), "val_letterbox")
        if dtype == torch.uint8:
            got = out.cpu().numpy()
            for i, w_ in enumerate(want):
                assert np.array_equal(got[i], w_), (img_size, srcs[i].shape, loads[i])
            u8 = out
        else:
            ref = u8.to(dtype) / 255
            assert torch.equal(out.view(_BITS[dtype]), ref.view(_BITS[dtype])), dtype
    assert [V.area_is_fast(s.shape[:2], ld[0]) for s, ld in zip(srcs, loads) if ld[1] == V.INTERP_AREA].count(True) >= 3


def test_val_step_end_to_end(z):
    """loader -> yolov5n engine forward -> NMS -> val_batch_metrics gives the same `correct` as the reference loader's batch."""
    from oracle import model_ref
    from yolov5_b200.cfg import model_cfg
    from yolov5_b200.models.yolo import DetectionModel
    from yolov5_b200.utils import metrics
    from yolov5_b200.utils.general import nms_device

    m = DetectionModel("yolov5n")
    m.load_state_dict(model_ref.synth_state_dict(model_cfg("yolov5n"), seed=5))
    m = m.to(DEV).half().eval()
    iouv = torch.linspace(0.5, 0.95, 10, device=DEV)
    ds = F.ValDataset(z, "det.rect")

    def step(imgs, targets, shapes):
        h, w = imgs.shape[2:]
        x = imgs.half() / 255 if imgs.dtype == torch.uint8 else imgs
        rows, _, count = nms_device(m(x)[0], 0.001, 0.6, max_det=300)
        tg = targets.clone()
        tg[:, 2:] *= torch.tensor((w, h, w, h), device=DEV)
        return metrics.val_batch_metrics(rows, count, tg, (h, w), shapes, iouv)[1], count

    for bi, (imgs, targets, _, shapes) in enumerate(_loader(ds, torch.float16)):
        ri, rt, rs, _ = F.expected(z, "det.rect", bi)
        got, gc = step(imgs, targets, shapes)
        want, wc = step(torch.from_numpy(ri).to(DEV), torch.from_numpy(rt).to(DEV), [((a[0], a[1]), (tuple(b[0]), tuple(b[1]))) for a, b in rs])
        assert torch.equal(gc, wc) and torch.equal(got, want), bi
