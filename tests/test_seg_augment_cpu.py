"""CPU: the segmentation augmentation oracle (oracle/seg_aug_ref.py) against cv2 / numpy and against the reference's
batches (tests/golden/seg_aug.npz); the loader's draws, refusals and ABI structs."""
import ctypes
import random
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from oracle import seg_aug_ref as S
from tests import seg_aug_fixture as F


@pytest.fixture(scope="module")
def z():
    return F.load()


def _random_polygon(rng, t, h, w):
    n = int(rng.integers(1, 40))
    kind = t % 6
    if kind == 0:  # inside and just outside
        return rng.integers(-10, max(h, w) + 10, (n, 2))
    if kind == 1:  # far outside on every side
        return rng.integers(-300, 300, (n, 2))
    if kind == 2:  # resampled: many horizontal and zero-length edges after the int32 cast
        return S.resample(rng.uniform(-20, max(h, w) + 20, (n, 2)).astype(np.float32))
    if kind == 3:  # vertices far outside
        return rng.integers(-5000, 5000, (n, 2))
    if kind == 4:  # self-intersecting cloud around the centre
        return rng.normal(h / 2, h / 4, (n, 2))
    return rng.integers(0, max(min(h, w), 1), (n, 2))  # inside


@pytest.mark.parametrize("ratio", [1, 4])
def test_rasterizer_equals_cv2(ratio):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(100 + ratio)
    for t in range(1500):
        h, w = int(rng.integers(1, 40)) * 4, int(rng.integers(1, 40)) * 4
        pts = np.asarray(_random_polygon(rng, t, h, w), np.int32)
        ref = cv2.resize(cv2.fillPoly(np.zeros((h, w), np.uint8), [pts.reshape(-1, 1, 2)], 1), (w // ratio, h // ratio))
        assert np.array_equal(ref, S.polygon2mask((h, w), [pts.reshape(-1)], 1, ratio)), (t, h, w)


def test_clip_and_lines_equal_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(3)
    for t in range(2000):
        w, h = int(rng.integers(1, 50)), int(rng.integers(1, 50))
        p = rng.integers(-60, 110, 4)
        ok, a, b = cv2.clipLine((0, 0, w, h), (int(p[0]), int(p[1])), (int(p[2]), int(p[3])))
        x1, y1, x2, y2, ok2 = S.clip_lines(w, h, p[0:1], p[1:2], p[2:3], p[3:4])
        assert (bool(ok), tuple(a), tuple(b)) == (bool(ok2[0]), (int(x1[0]), int(y1[0])), (int(x2[0]), int(y2[0]))), t
        ref = cv2.line(np.zeros((h, w), np.uint8), (int(p[0]), int(p[1])), (int(p[2]), int(p[3])), 1, thickness=1, lineType=cv2.LINE_8)
        got = np.zeros((h, w), np.uint8)
        xs, ys = S.line_pixels(w, h, p[0:1], p[1:2], p[2:3], p[3:4])
        got[ys, xs] = 1
        assert np.array_equal(ref, got), t


def test_resample_and_transform_equal_numpy():
    rng = np.random.default_rng(5)
    for k in range(200):
        seg = rng.uniform(-50, 1300, (int(rng.integers(1, 300)), 2)).astype(np.float32)
        s = np.concatenate((seg, seg[0:1, :]), axis=0)
        x = np.linspace(0, len(s) - 1, 1000)
        ref = np.concatenate([np.interp(x, np.arange(len(s)), s[:, i]) for i in range(2)]).reshape(2, -1).T
        assert np.array_equal(ref, S.resample(seg)), k
    for k in range(30):  # 1000-row shapes, as random_perspective's segment path multiplies them
        M = rng.normal(size=(3, 3)) * 3
        M[2] = [0, 0, 1]
        xy = S.resample(rng.uniform(-50, 1300, (int(rng.integers(3, 80)), 2)).astype(np.float32))
        xy1 = np.ones((len(xy), 3))
        xy1[:, :2] = xy
        assert np.array_equal((xy1 @ M.T)[:, :2], S.affine_points(xy, M)), k


def test_fma_is_correctly_rounded():
    rng = np.random.default_rng(6)
    a, b, c = rng.uniform(-2e3, 2e3, (3, 5000))
    ref = np.array([float(Fraction(x) * Fraction(y) + Fraction(v)) for x, y, v in zip(a, b, c)])
    assert np.array_equal(S.fma(a, b, c), ref)


def test_overlap_order_is_zero_first_then_descending_stable():
    areas = np.array([5, 0, 7, 5, 0, 9], np.uint64)
    assert S.overlap_order(areas).tolist() == [1, 4, 5, 2, 0, 3]


@pytest.mark.parametrize("run", [f"{t}.o{o}.r{r}" for t in ("low", "med", "mixed") for o in (1, 0) for r in (1, 4)])
def test_oracle_equals_fixture(z, run):
    tag, overlap, ratio = F.run_options(run)
    ds = F.SegDataset(z, F.hyps(z)[tag], overlap, ratio)
    random.seed(int(z[f"{run}.seed"]))
    np.random.seed(int(z[f"{run}.seed"]))
    for bi in range(2):
        idx = list(range(bi * F.BATCH, min((bi + 1) * F.BATCH, ds.n)))
        imgs, targets, masks, _ = S.get_batch(ds, idx, overlap, ratio)
        assert np.array_equal(imgs, z[f"{tag}.imgs{bi}"]), (run, bi)
        assert np.array_equal(targets.view(np.uint32), z[f"{run}.targets{bi}"].view(np.uint32)), (run, bi)
        ref = z[f"{run}.masks{bi}"]
        assert masks.dtype == ref.dtype and masks.shape == ref.shape and np.array_equal(masks, ref), (run, bi)


def test_fixture_covers_branches(z):
    """Mosaic and letterboxed items, mixup, and overlap images where the label order decides equal areas."""
    assert any(not z[k].all() for k in z.files if ".mosaic" in k)
    assert any(z[k].any() for k in z.files if ".mixup" in k)
    assert "order_differs" in str(z["meta"])


def test_loader_draws_match_oracle(z):
    from yolov5_b200.utils.dataloaders import draw_item
    from yolov5_b200.utils.segment.dataloaders import _mixup_partner

    for tag in ("med", "mixed"):
        ds = F.SegDataset(z, F.hyps(z)[tag], True, 4)
        for seed in range(20):
            random.seed(seed)
            np.random.seed(seed)
            a = [S.sample_params(ds, i) for i in range(ds.n)]
            random.seed(seed)
            np.random.seed(seed)
            b = [draw_item(ds, i, _mixup_partner(ds), shuffle_tiles=False) for i in range(ds.n)]
            assert repr(a) == repr(b), (tag, seed)


def test_mask_dtype_matches_torch_cat():
    import torch

    from yolov5_b200.utils.segment.dataloaders import _mask_dtype

    def cat(kept, overlap):
        parts = []
        for k in kept:
            if k == 0:
                parts.append(torch.zeros(1 if overlap else 0, 4, 4))
            elif overlap:
                parts.append(torch.zeros(1, 4, 4, dtype=torch.int32 if k > 255 else torch.uint8))
            else:
                parts.append(torch.zeros(k, 4, 4, dtype=torch.uint8))
        return torch.cat(parts, 0).dtype

    for kept in ([3, 5], [0, 5], [300, 2], [300, 0], [0, 0], [256]):
        for overlap in (True, False):
            assert _mask_dtype(kept, overlap) == cat(kept, overlap), (kept, overlap)


def _hyp(z, **kw):
    return dict(F.hyps(z)["low"], **kw)


@pytest.mark.parametrize("what", ["copy_paste", "perspective", "albumentations", "rect", "augment", "segments", "ratio2", "ratio8"])
def test_refused_options(z, what):
    from yolov5_b200.utils.segment.dataloaders import DeviceSegAugmentLoader

    ds = F.SegDataset(z, _hyp(z), True, 4)
    ratio = None
    if what == "copy_paste":
        ds.hyp = _hyp(z, copy_paste=0.1)
    elif what == "perspective":
        ds.hyp = _hyp(z, perspective=0.0005)
    elif what == "albumentations":
        ds.albumentations = type("A", (), {"transform": object()})()
    elif what == "rect":
        ds.rect = True
    elif what == "augment":
        ds.augment = False
    elif what == "segments":
        ds.segments[0] = ds.segments[0][:-1]
    else:
        ratio = int(what[5:])
    state = random.getstate()
    with pytest.raises(NotImplementedError):
        DeviceSegAugmentLoader(ds, 4, device="cpu", downsample_ratio=ratio)
    assert random.getstate() == state  # nothing drawn


def test_bad_segments_raise(z):
    from yolov5_b200.utils.segment.dataloaders import DeviceSegAugmentLoader

    ds = F.SegDataset(z, _hyp(z), True, 4)
    ds.segments[0][0] = ds.segments[0][0].astype(np.float64)
    with pytest.raises(ValueError):
        DeviceSegAugmentLoader(ds, 4, device="cpu")


def test_detection_loader_still_refuses_segments(z):
    from yolov5_b200.utils.dataloaders import DeviceAugmentLoader

    with pytest.raises(NotImplementedError):
        DeviceAugmentLoader(F.SegDataset(z, _hyp(z), True, 4), 4, device="cpu")


def test_seg_struct_matches_the_c_layout(tmp_path):
    from yolov5_b200 import _lib

    hdr = __import__("os").path.join(__import__("os").path.dirname(__file__), "..", "include", "y5b200.h")
    src = f'#include <stdio.h>\n#include <stddef.h>\n#include "{hdr}"\nint main(void) {{\n'
    src += '  printf("%zu %zu %zu %d %d\\n", sizeof(y5_aug_segment), offsetof(y5_aug_segment, point_offset), '
    src += "offsetof(y5_aug_segment, n_points), Y5_SEG_POINTS, Y5_SEG_I32);\n  return 0;\n}\n"
    (tmp_path / "seg.c").write_text(src)
    subprocess.run(["gcc", "-o", str(tmp_path / "seg"), str(tmp_path / "seg.c")], check=True)
    out = subprocess.run([str(tmp_path / "seg")], capture_output=True, text=True, check=True).stdout.split()
    A = _lib.AugSegment
    assert [int(v) for v in out] == [ctypes.sizeof(A), A.point_offset.offset, A.n_points.offset, _lib.SEG_POINTS, _lib.SEG_I32]


def test_seg_argument_validation_without_gpu():
    """Null pointers give -1, an unsupported ratio or dtype -2, before any launch."""
    from yolov5_b200 import _lib

    lib = _lib.lib()
    assert lib.y5_seg_warp(None, 1, None, None, None, 1, 1, 64, 64, None, None, None, None) == -1
    assert lib.y5_seg_raster(None, 1000, None, 1, 64, 64, 4, None, None, None) == -1
    assert lib.y5_seg_raster(ctypes.c_void_p(16), 1000, ctypes.c_void_p(16), 1, 64, 64, 2, ctypes.c_void_p(16), ctypes.c_void_p(16), None) == -2
    assert lib.y5_seg_raster(ctypes.c_void_p(16), 1000, ctypes.c_void_p(16), 1, 66, 66, 4, ctypes.c_void_p(16), ctypes.c_void_p(16), None) == -2
    assert lib.y5_seg_order(None, 1, None, None, None, 1, None, None, None, None) == -1
    p = ctypes.c_void_p(16)
    assert lib.y5_seg_compose(p, p, p, p, p, 1, 8, 8, 1, p, 1, None) == -2
    assert lib.y5_seg_compose(p, None, p, p, p, 1, 8, 8, 0, p, 3, None) == -1
