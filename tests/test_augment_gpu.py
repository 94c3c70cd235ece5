"""Training augmentation on the device (y5_aug_gather / y5_aug_labels through DeviceAugmentLoader and the public
augmentation functions), byte-exact against the reference's batches (tests/golden/aug.npz) and the oracle."""
import random

import numpy as np
import pytest
import torch

from oracle import aug_ref, pre_ref
from tests import aug_fixture

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None


@pytest.fixture(scope="module")
def z():
    return aug_fixture.load()


def _seed(s):
    random.seed(s)
    np.random.seed(s)


def _same_targets(a, b):
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else a
    return a.dtype == np.float32 and a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("tag", ["low", "high", "mixed"])
def test_loader_reproduces_fixture(z, tag):
    from yolov5_b200.utils.dataloaders import DeviceAugmentLoader

    ds = aug_fixture.FixtureDataset(z, aug_fixture.hyps(z)[tag])
    loader = DeviceAugmentLoader(ds, aug_fixture.BATCH, shuffle=False, device=DEV)
    _seed(int(z[f"{tag}.seed"]))
    n = 0
    for bi, (imgs, targets, paths, shapes) in enumerate(loader):
        assert imgs.device == DEV and imgs.dtype == torch.uint8
        assert np.array_equal(imgs.cpu().numpy(), z[f"{tag}.imgs{bi}"]), (tag, bi)
        assert _same_targets(targets, z[f"{tag}.targets{bi}"]), (tag, bi)
        assert len(paths) == imgs.shape[0] and len(shapes) == imgs.shape[0]
        n += 1
    assert n == 2


def _odd_dataset(hyp, seed, s=64, empty_all=False):
    """Sources narrower than a tile, 1-px wide / tall, non-square; tiny boxes when empty_all (all filtered out)."""
    rs = np.random.RandomState(seed)
    shapes = [(64, 48), (1, 40), (50, 1), (7, 64), (64, 3), (33, 17), (20, 64), (64, 64)]
    srcs = [pre_ref.synth_image(h, w, seed * 10 + k) for k, (h, w) in enumerate(shapes)]
    labels = []
    for k in range(len(shapes)):
        n = 0 if k == 3 else 1 + k % 3
        xy, wh = rs.uniform(0.1, 0.9, (n, 2)), rs.uniform(0.001, 0.01, (n, 2)) if empty_all else rs.uniform(0.05, 0.9, (n, 2))
        labels.append(np.concatenate((rs.randint(0, 80, (n, 1)), xy, wh), 1).astype(np.float32))
    return aug_fixture.FixtureDataset(None, hyp, sources=srcs, labels=labels, img_size=s)


def _compare_with_oracle(ds, seed, batch=4, dtype=torch.uint8):
    from yolov5_b200.utils.dataloaders import DeviceAugmentLoader

    loader = DeviceAugmentLoader(ds, batch, device=DEV, dtype=dtype)
    for b0 in range(0, ds.n, batch):
        idx = list(range(b0, min(b0 + batch, ds.n)))
        _seed(seed + b0)
        imgs, targets, _, _ = loader.collate(idx)
        _seed(seed + b0)
        ri, rt, params = aug_ref.get_batch(ds, idx)
        assert np.array_equal(imgs.cpu().numpy(), ri), (seed, b0, np.argwhere(imgs.cpu().numpy() != ri)[:4])
        assert _same_targets(targets, rt), (seed, b0)
    return params


@pytest.mark.parametrize("seed", range(6))
def test_warp_geometries_against_oracle(z, seed):
    """Rotations up to +-180 with shear, scale 0.1-1.9, tiny and 1-px sources: every tap of the virtual canvas, the
    seams between tiles and the canvas edge, against the oracle's materialised canvas + warpAffine."""
    hyp = dict(aug_fixture.hyps(z)["low"], degrees=180.0, shear=15.0, scale=0.9, mixup=0.5, flipud=0.5)
    _compare_with_oracle(_odd_dataset(hyp, seed), 100 + seed)


def test_warp_scale_extremes(z):
    from yolov5_b200.utils.augmentations import random_perspective

    rng = np.random.default_rng(5)
    for k, (h, w, sc, border) in enumerate([(64, 48, 0.9, (-16, -16)), (40, 1, 0.9, (0, 0)), (1, 50, 0.5, (0, 0)), (90, 120, 0.9, (-30, -30))]):
        im = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        for seed in range(4):
            _seed(1000 * k + seed)
            got, _ = random_perspective(im, degrees=180, translate=0.2, scale=sc, shear=20, border=border)
            _seed(1000 * k + seed)
            d = aug_ref.perspective_draws(dict(perspective=0.0, degrees=180, scale=sc, shear=20, translate=0.2))
            M = aug_ref.affine(d, (h, w), border)
            ref = aug_ref.warp_affine(im, M[:2], (w + 2 * border[1], h + 2 * border[0]))
            assert np.array_equal(got, ref), (k, seed)


def test_mosaic_centre_extremes(z, monkeypatch):
    """Mosaic centres at both ends of uniform(s/2, 3s/2)."""
    hyp = dict(aug_fixture.hyps(z)["low"], degrees=10.0)
    for end in (0.0, 1.0 - 1e-12):
        real = random.uniform
        calls = {"n": 0}

        def uniform(a, b):
            calls["n"] += 1
            return a + (b - a) * end if a == 32 and b == 96 else real(a, b)

        monkeypatch.setattr(random, "uniform", uniform)
        _compare_with_oracle(_odd_dataset(hyp, 7), 55)
        monkeypatch.undo()
        assert calls["n"] > 0


def test_hsv_all_inputs():
    """BGR -> HSV -> LUT -> HSV -> BGR over all 2^24 BGR inputs, as 32-pixel SIMD rows and as a row tail."""
    from yolov5_b200.utils.augmentations import augment_hsv

    B, G, R = np.meshgrid(np.arange(256), np.arange(256), np.arange(256), indexing="ij")
    im = np.stack([B, G, R], -1).astype(np.uint8).reshape(4096, 4096, 3)
    for seed, gains in ((1, (0.015, 0.7, 0.4)), (2, (0.5, 0.9, 0.9))):
        _seed(seed)
        got = im.copy()
        augment_hsv(got, *gains)
        _seed(seed)
        ref = aug_ref.apply_hsv(im, aug_ref.hsv_gains(*gains))
        assert np.array_equal(got, ref), seed
    # rows of 37 pixels: the last 5 of every row take the scalar tail (rounding); images of at most 16384 rows
    rows = (4096 * 4096) // 37
    flat = im.reshape(-1, 3)
    for r0 in range(0, rows, 16384):
        n = min(16384, rows - r0)
        tail = flat[r0 * 37: (r0 + n) * 37].reshape(n, 37, 3).copy()
        _seed(3)
        got = torch.from_numpy(tail).to(DEV)
        augment_hsv(got, 0.3, 0.7, 0.4)
        _seed(3)
        assert np.array_equal(got.cpu().numpy(), aug_ref.apply_hsv(tail, aug_ref.hsv_gains(0.3, 0.7, 0.4))), r0


@pytest.mark.parametrize("r", [0.5, 0.49999999999999994, 0.5000000000000001, 0.25, 0.75, 0.4375])
def test_mixup_blend(r):
    from yolov5_b200.utils.augmentations import _single_image_table, aug_gather, mixup, upload_table

    rng = np.random.default_rng(int(r * 1e6))
    a = rng.integers(0, 256, (64, 96, 3), dtype=np.uint8)
    b = a.copy() if r == 0.5 else rng.integers(0, 256, (64, 96, 3), dtype=np.uint8)
    b[:8] = a[:8]  # a*r + a*(1-r) lands on (or next to) an integer
    ta, tb = torch.from_numpy(a).to(DEV), torch.from_numpy(b).to(DEV)
    tdev, _ = upload_table(_single_image_table([ta, tb], r=r), DEV)
    got = aug_gather(tdev, 1, 64, 96, swap_rb=False, device=DEV)[0].permute(1, 2, 0).cpu().numpy()
    assert np.array_equal(got, (a * r + b * (1 - r)).astype(np.uint8))
    _seed(4)
    got2, lab = mixup(a, np.zeros((1, 5), np.float32), b, np.ones((2, 5), np.float32))
    _seed(4)
    rr = np.random.beta(32.0, 32.0)
    assert np.array_equal(got2, (a * rr + b * (1 - rr)).astype(np.uint8)) and lab.shape == (3, 5)


def test_output_modes_agree(z):
    from yolov5_b200.utils.dataloaders import DeviceAugmentLoader

    ds = aug_fixture.FixtureDataset(z, aug_fixture.hyps(z)["high"])
    outs = {}
    for dt in (torch.uint8, torch.float16, torch.bfloat16, torch.float32):
        _seed(9)
        outs[dt] = DeviceAugmentLoader(ds, 4, device=DEV, dtype=dt).collate([0, 1, 2, 3])[0]
    # true division by 255 in fp32, as the letterbox kernel and the oracle (pre_ref.to_chw_rgb) divide
    ref = torch.from_numpy(outs[torch.uint8].cpu().numpy().astype(np.float32) / np.float32(255)).to(DEV)
    assert torch.equal(outs[torch.float32], ref)
    assert torch.equal(outs[torch.float16], ref.half()) and torch.equal(outs[torch.bfloat16], ref.bfloat16())
    # the stem's space-to-depth cells: channel (dy*2+dx)*3 + c of cell (y/2, x/2), 4 zero channels
    from yolov5_b200.utils.augmentations import _single_image_table, affine_matrix, aug_gather, hsv_luts, upload_table

    src = torch.from_numpy(pre_ref.synth_image(90, 120, 4)).to(DEV)
    M = affine_matrix((0.0, 0.0, 30.0, 0.8, 5.0, -5.0, 0.45, 0.55), (90, 120), (0, 0))
    tdev, _ = upload_table(_single_image_table([src], [(M, 0.8)], luts=hsv_luts(np.array([1.01, 0.7, 1.2]))), DEV)
    h, w = 96, 128
    u8 = aug_gather(tdev, 1, h, w, device=DEV)
    for dt in (torch.float16, torch.bfloat16):
        buf = torch.zeros(1 * (h // 2) * (w // 2) * 16, dtype=dt, device=DEV)
        aug_gather(tdev, 1, h, w, device=DEV, s2d_out=(buf, 0, 0))
        cells = buf.view(1, h // 2, w // 2, 16)
        expect = torch.zeros_like(cells)
        for dy in range(2):
            for dx in range(2):
                for c in range(3):
                    q = torch.from_numpy(u8[:, c, dy::2, dx::2].cpu().numpy().astype(np.float32) / np.float32(255))
                    expect[..., (dy * 2 + dx) * 3 + c] = q.to(DEV).to(dt)
        assert torch.equal(cells, expect), dt


@pytest.mark.parametrize("case", ["letterbox", "identity", "no_labels", "all_filtered"])
def test_other_cases(z, case):
    base = dict(aug_fixture.hyps(z)["low"])
    if case == "letterbox":
        hyp = dict(base, mosaic=0.0, degrees=20.0, shear=5.0)
    elif case == "identity":  # M == I: random_perspective skips the warp
        hyp = dict(base, mosaic=0.0, degrees=0.0, translate=0.0, scale=0.0, shear=0.0)
    else:
        hyp = dict(base, mixup=0.5)
    ds = _odd_dataset(hyp, 21, empty_all=case == "all_filtered")
    if case == "no_labels":
        ds.labels = [np.zeros((0, 5), np.float32) for _ in ds.labels]
    params = _compare_with_oracle(ds, 300)
    if case in ("letterbox", "identity"):
        assert not any(p["mosaic"] for p in params)
    if case in ("no_labels", "all_filtered"):
        from yolov5_b200.utils.dataloaders import DeviceAugmentLoader

        _seed(300)
        imgs, (padded, count), _, _ = DeviceAugmentLoader(ds, 4, device=DEV).collate([0, 1, 2, 3], sync=False)
        assert int(count.item()) == 0


def test_training_step_on_loader_output(z):
    """A yolov5n FusedSGD training step runs on the loader's output."""
    from oracle import model_ref
    from yolov5_b200.cfg import HYP_SCRATCH_LOW, model_cfg
    from yolov5_b200.models.yolo import DetectionModel
    from yolov5_b200.utils.dataloaders import DeviceAugmentLoader
    from yolov5_b200.utils.loss import ComputeLoss
    from yolov5_b200.utils.torch_utils import FusedSGD

    ds = aug_fixture.FixtureDataset(z, aug_fixture.hyps(z)["low"])
    _seed(0)
    imgs, targets, _, _ = next(iter(DeviceAugmentLoader(ds, 4, device=DEV)))
    m = DetectionModel("yolov5n")
    m.load_state_dict(model_ref.synth_state_dict(model_cfg("yolov5n"), seed=3))
    m = m.to(DEV).train()
    m.hyp = dict(HYP_SCRATCH_LOW)
    opt = FusedSGD(m.parameters(), lr=0.01, momentum=0.937, nesterov=True)
    before = [p.detach().clone() for p in m.parameters()]
    with torch.autocast("cuda", dtype=torch.float16):
        p = m(imgs.float() / 255)
    loss, _ = ComputeLoss(m)(p, targets)
    loss.backward()
    opt.fused_step()
    assert torch.isfinite(loss).all() and targets.shape[0] > 0
    assert any(not torch.equal(a, b) for a, b in zip(before, m.parameters()))
