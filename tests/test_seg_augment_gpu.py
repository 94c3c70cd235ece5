"""GPU: segmentation training augmentation (y5_seg_warp / y5_seg_raster / y5_seg_order / y5_seg_compose through
DeviceSegAugmentLoader and polygons2masks[_overlap]) against the reference's batches (tests/golden/seg_aug.npz) and the
oracle (oracle/seg_aug_ref.py) at 640."""
import random

import numpy as np
import pytest
import torch

from oracle import pre_ref
from oracle import seg_aug_ref as S
from tests import seg_aug_fixture as F

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None


@pytest.fixture(scope="module")
def z():
    return F.load()


def _seed(s):
    random.seed(s)
    np.random.seed(s)


def _check(batch, imgs, targets, masks, where):
    gi, gt, _, _, gm = batch
    assert gi.device == DEV and gt.device == DEV and gm.device == DEV
    assert np.array_equal(gi.cpu().numpy(), imgs), where
    gt = gt.cpu().numpy()
    assert gt.dtype == np.float32 and gt.shape == targets.shape and np.array_equal(gt.view(np.uint32), targets.view(np.uint32)), where
    gm = gm.cpu().numpy()
    assert gm.dtype == masks.dtype and gm.shape == masks.shape, (where, gm.dtype, masks.dtype, gm.shape, masks.shape)
    assert np.array_equal(gm, masks), (where, np.argwhere(gm != masks)[:5])


@pytest.mark.parametrize("run", [f"{t}.o{o}.r{r}" for t in ("low", "med", "mixed") for o in (1, 0) for r in (1, 4)])
def test_loader_reproduces_fixture(z, run):
    from yolov5_b200.utils.segment.dataloaders import DeviceSegAugmentLoader

    tag, overlap, ratio = F.run_options(run)
    ds = F.SegDataset(z, F.hyps(z)[tag], overlap, ratio)
    loader = DeviceSegAugmentLoader(ds, F.BATCH, shuffle=False, device=DEV)
    assert loader.overlap == overlap and loader.downsample_ratio == ratio
    _seed(int(z[f"{run}.seed"]))
    n = 0
    for bi, batch in enumerate(loader):
        _check(batch, z[f"{tag}.imgs{bi}"], z[f"{run}.targets{bi}"], z[f"{run}.masks{bi}"], (run, bi))
        n += 1
    assert n == 2


def _polygon(rs, c, r):
    n = int(rs.randint(3, 24))
    t = np.sort(rs.uniform(0, 2 * np.pi, n))
    rad = r * rs.uniform(0.3, 1.0, n)
    return (c + np.stack([np.cos(t), np.sin(t)], 1) * rad[:, None]).astype(np.float32)


def _labels_for(segs, rs):
    boxes = []
    for s in segs:
        x, y = np.clip(s, 0, 1).T
        boxes.append([(x.min() + x.max()) / 2, (y.min() + y.max()) / 2, x.max() - x.min(), y.max() - y.min()])
    return np.concatenate((rs.randint(0, 80, (len(segs), 1)), np.array(boxes).reshape(-1, 4)), 1).astype(np.float32)


def _dataset_640(hyp, overlap, ratio, seed=3):
    """COCO-like: 12 images of mixed shapes, Poisson(7.3) polygons each (concave, some crossing the border); image 4
    has none."""
    rs = np.random.RandomState(seed)
    shapes = [(480, 640), (640, 427), (640, 640), (360, 640), (640, 480), (512, 384), (200, 640), (640, 300), (427, 640),
              (640, 512), (300, 300), (640, 360)]
    srcs, labels, segments = [], [], []
    for k, (h, w) in enumerate(shapes):
        srcs.append(pre_ref.synth_image(h, w, 300 + k))
        n = 0 if k == 4 else max(1, rs.poisson(7.3))
        segs = [_polygon(rs, rs.uniform(0.0, 1.0, 2), rs.uniform(0.03, 0.4)) for _ in range(n)]
        segments.append(segs)
        labels.append(_labels_for(segs, rs) if n else np.zeros((0, 5), np.float32))
    return F.SegDataset(None, hyp, overlap, ratio, sources=srcs, labels=labels, segments=segments, img_size=640)


def _oracle_batch(ds, idx, overlap, ratio, seed):
    _seed(seed)
    imgs, targets, masks, _ = S.get_batch(ds, idx, overlap, ratio)
    return imgs, targets, masks


@pytest.mark.parametrize("overlap,ratio", [(True, 4), (False, 4), (True, 1)])
def test_loader_equals_oracle_640(z, overlap, ratio):
    from yolov5_b200.utils.segment.dataloaders import DeviceSegAugmentLoader

    hyp = dict(F.hyps(z)["med"], mixup=0.5, degrees=20.0, shear=5.0, flipud=0.5, mosaic=0.8)
    ds = _dataset_640(hyp, overlap, ratio)
    idx = [i % ds.n for i in range(16)]
    ref = _oracle_batch(ds, idx, overlap, ratio, 7)
    loader = DeviceSegAugmentLoader(ds, 16, device=DEV)
    _seed(7)
    _check(loader.collate(idx), *ref, (overlap, ratio))


def _crowd_dataset(hyp, overlap, ratio):
    """Non-mosaic, identity warp: image 0 has 300 small polygons (an int32 overlap plane), image 1 has 200 polygons that
    all cover the centre (the uint8 sum wraps past label ~128), image 2 has none."""
    rs = np.random.RandomState(11)
    srcs = [pre_ref.synth_image(640, 640, 400 + k) for k in range(3)]
    grid = [_polygon(rs, np.array([(i % 20 + 0.5) / 20, (i // 20 + 0.5) / 15]), 0.02) for i in range(300)]
    centre = [_polygon(rs, 0.5 + rs.uniform(-0.05, 0.05, 2), rs.uniform(0.1, 0.45)) for _ in range(200)]
    segments = [grid, centre, []]
    labels = [_labels_for(grid, rs), _labels_for(centre, rs), np.zeros((0, 5), np.float32)]
    return F.SegDataset(None, hyp, overlap, ratio, sources=srcs, labels=labels, segments=segments, img_size=640)


@pytest.mark.parametrize("idx,dtype", [([0, 1], np.int32), ([1, 2], np.float32), ([1, 1], np.uint8)])
def test_crowded_images_and_mask_dtypes(z, idx, dtype):
    from yolov5_b200.utils.segment.dataloaders import DeviceSegAugmentLoader

    hyp = dict(F.hyps(z)["low"], mosaic=0.0, scale=0.0, translate=0.0, fliplr=0.5)
    ds = _crowd_dataset(hyp, True, 4)
    ref = _oracle_batch(ds, idx, True, 4, 5)
    assert ref[2].dtype == dtype
    loader = DeviceSegAugmentLoader(ds, len(idx), device=DEV)
    _seed(5)
    _check(loader.collate(idx), *ref, idx)
    if idx == [1, 1]:  # image 1 reaches the uint8 wrap: its plane differs from the same sums in int64
        _, _, polys = S.letterbox_item(ds, 1, (0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.5, 0.5))
        assert len(polys) == 200
        ms = [S.polygon2mask((640, 640), [p.reshape(-1)], 1, 4) for p in polys]
        v8, v64 = np.zeros((160, 160), np.uint8), np.zeros((160, 160), np.int64)
        for i, j in enumerate(S.overlap_order([m.sum() for m in ms])):
            v8 = np.clip(v8 + ms[j] * (i + 1), 0, i + 1)
            v64 = np.clip(v64 + ms[j].astype(np.int64) * (i + 1), 0, i + 1)
        assert (v8 != v64).any()


def test_polygons2masks_entry_points():
    from yolov5_b200.utils.segment.dataloaders import polygons2masks, polygons2masks_overlap

    rs = np.random.RandomState(2)
    polys = [(_polygon(rs, rs.uniform(-0.2, 1.2, 2), rs.uniform(0.05, 0.6)) * 160).astype(np.float64) for _ in range(40)]
    polys += [np.array([[10.7, 10.2]]), np.array([[5.0, 5.0], [150.0, 5.0]])]  # a point and a horizontal line
    for r in (1, 4):
        got = polygons2masks((160, 160), polys, 1, r, device=DEV)
        ref = S.polygons2masks((160, 160), polys, 1, r)
        assert got.dtype == torch.uint8 and np.array_equal(got.cpu().numpy(), ref), r
        gm, gi = polygons2masks_overlap((160, 160), polys, r, device=DEV)
        rm, ri = S.polygons2masks_overlap((160, 160), polys, r)
        assert gm.dtype == torch.uint8 and np.array_equal(gm.cpu().numpy(), rm) and np.array_equal(gi.cpu().numpy(), ri), r


def test_training_step_from_loader_output(z):
    from tests.test_seg_loss_gpu import _seg_model
    from yolov5_b200.utils.segment.dataloaders import DeviceSegAugmentLoader
    from yolov5_b200.utils.segment.loss import ComputeLoss
    from yolov5_b200.utils.torch_utils import FusedSGD

    hyp = dict(F.hyps(z)["low"])
    ds = _dataset_640(hyp, True, 4)
    _seed(9)
    imgs, targets, _, _, masks = DeviceSegAugmentLoader(ds, 8, device=DEV).collate(list(range(8)))
    _, _, m = _seg_model(DEV, seed=52)
    m.train()
    crit = ComputeLoss(m, overlap=True)
    opt = FusedSGD([q for q in m.parameters() if q.requires_grad], lr=0.01, momentum=0.9)
    opt.zero_grad(set_to_none=True)
    with torch.autocast("cuda", dtype=torch.float16):
        pred = m(imgs)
    loss, items = crit(pred, targets, masks.float())
    loss.backward()
    opt.fused_step()
    assert torch.isfinite(loss).all() and float(items[1]) > 0
    assert all(torch.isfinite(q).all() for q in m.parameters())
