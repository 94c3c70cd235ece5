"""CPU: the validation loaders' host side and oracle -- oracle/val_load_ref.py against tests/golden/val_load.npz (the
reference's own batches) and against cv2.resize over a size sweep; the loaders' geometry, shapes and label rows; their
refusals; the y5_val_image ABI."""
import ctypes
import random
import subprocess

import numpy as np
import pytest
import torch

from oracle import pre_ref
from oracle import val_load_ref as V
from tests import val_load_fixture as F
from yolov5_b200 import _lib
from yolov5_b200.utils.dataloaders import DeviceValLoader, ValBatchLayout, load_val_image
from yolov5_b200.utils.segment.dataloaders import DeviceSegValLoader

CPU_DEV = "cuda:0"  # a device name only: nothing below reaches the device


@pytest.fixture(scope="module")
def z():
    return F.load()


def _positions(ds, bi):
    return list(range(bi * ds.batch_size, min((bi + 1) * ds.batch_size, ds.n)))


def _oracle(ds, bi, seg):
    items = []
    for i in _positions(ds, bi):
        im = V.load_resize(ds.src[i], F.IMG_SIZE)
        shape = ds.batch_shapes[ds.batch[i]] if ds.rect else F.IMG_SIZE
        if seg:
            items.append(V.get_item(im, ds.src[i].shape[:2], ds.labels[i], shape, ds.segments[i], ds.overlap, ds.downsample_ratio))
        else:
            items.append(V.get_item(im, ds.src[i].shape[:2], ds.labels[i], shape))
    return V.get_batch(items)


def test_oracle_equals_fixture(z):
    for run in F.runs(z):
        seg = run.startswith("seg.")
        ds = F.ValDataset(z, run)
        for bi in range(ds.n_batches):
            imgs, targets, shapes, masks = F.expected(z, run, bi)
            got = _oracle(ds, bi, seg)
            assert np.array_equal(got[0], imgs), (run, bi)
            assert got[1].shape == targets.shape and np.array_equal(got[1].view(np.uint32), targets.view(np.uint32)), (run, bi)
            assert F.as_json(got[2]) == shapes, (run, bi)
            if seg:
                assert got[3].dtype == masks.dtype and got[3].shape == masks.shape and np.array_equal(got[3], masks), (run, bi)


def test_fixture_covers_every_path(z):
    interps, again, dtypes = set(), False, set()
    for run in F.runs(z):
        ds = F.ValDataset(z, run)
        for i in range(ds.n):
            (h, w), interp = V.load_size(ds.src[i].shape[:2], F.IMG_SIZE)
            interps.add(interp)
            if interp == V.INTERP_AREA:
                interps.add(("fast", V.area_is_fast(ds.src[i].shape[:2], (h, w))))
            shape = ds.batch_shapes[ds.batch[i]] if ds.rect else F.IMG_SIZE
            new_unpad = pre_ref.letterbox_geometry((h, w), shape, auto=False, scaleup=False)[0]
            again |= tuple(new_unpad) != (w, h)
        for bi in range(ds.n_batches):
            m = F.expected(z, run, bi)[3]
            if m is not None:
                dtypes.add(m.dtype)
    assert interps >= {V.INTERP_COPY, V.INTERP_LINEAR, V.INTERP_AREA, ("fast", True), ("fast", False)}
    assert again and dtypes == {np.dtype(np.uint8), np.dtype(np.int32), np.dtype(np.float32)}


def _cv2():
    return pytest.importorskip("cv2", reason="the INTER_AREA / INTER_LINEAR restatements are pinned against the installed cv2")


def _sweep_sizes():
    rs = np.random.RandomState(0)
    sizes = [(1280, 960, 640), (1920, 1080, 640), (1920, 1440, 640), (2560, 1920, 640), (1000, 750, 640), (768, 1366, 640),
             (1080, 1920, 1280), (1, 1000, 640), (1000, 1, 640), (7, 3, 2), (2000, 3, 640), (641, 640, 640), (427, 1000, 640), (480, 640, 640)]
    for _ in range(150):
        h, w = int(rs.randint(1, 1400)), int(rs.randint(1, 1400))
        sizes.append((h, w, int(rs.randint(1, 1500))))
    return sizes


def test_load_resize_equals_cv2_over_a_size_sweep():
    cv2 = _cv2()
    rs = np.random.RandomState(1)
    seen = set()
    for h, w, s in _sweep_sizes():
        im = pre_ref.synth_image(h, w, h * 7 + w) if rs.rand() < 0.7 else rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
        (nh, nw), interp = V.load_size((h, w), s)
        seen.add(interp)
        if interp == V.INTERP_COPY:
            continue
        want = cv2.resize(im, (nw, nh), interpolation=cv2.INTER_AREA if interp == V.INTERP_AREA else cv2.INTER_LINEAR)
        assert np.array_equal(V.load_resize(im, s), want), (h, w, s, interp)
    assert seen == {V.INTERP_COPY, V.INTERP_LINEAR, V.INTERP_AREA}


def test_area_fast_rounding_differs_from_the_weighted_form():
    """2 x 2 cells round half up ((sum + 2) >> 2) where cvRound(sum / 4) would round half to even."""
    cv2 = _cv2()
    im = np.zeros((2, 4, 3), np.uint8)
    im[0, 0] = 1
    im[0, 1] = 1  # cell sum 2: 0.5
    im[:, 2:] = 3  # cell sum 12: 3
    got = V.resize_area_u8(im, (2, 1))
    assert np.array_equal(got, cv2.resize(im, (2, 1), interpolation=cv2.INTER_AREA))
    assert got[0, 0, 0] == 1 and got[0, 1, 0] == 3


def test_host_geometry_shapes_and_rows(z):
    """ValBatchLayout's load sizes, batch shapes, shapes and the label rows equal the fixture, with and without the RAM cache."""
    for run in ("det.rect", "det.square", "det.again"):
        for cache in (False, True):
            ds = F.ValDataset(z, run, cache=cache)
            for bi in range(ds.n_batches):
                pos = _positions(ds, bi)
                lay = ValBatchLayout(ds, pos, [F.decode(ds, p) for p in pos])
                imgs, targets, shapes, _ = F.expected(z, run, bi)
                assert lay.out_hw == imgs.shape[2:], (run, bi)
                assert F.as_json(lay.shapes) == shapes, (run, bi, cache)
                rows = [lay.label_rows(ds, b, lay.out_hw[1], lay.out_hw[0]) for b in range(lay.n)]
                got = np.concatenate([np.concatenate((np.full((len(r), 1), b, np.float32), r), 1) for b, r in enumerate(rows)], 0)
                assert np.array_equal(got.view(np.uint32), targets.view(np.uint32)), (run, bi, cache)
                for it, p in zip(lay.items, pos):
                    want = V.load_size(ds.src[p].shape[:2], F.IMG_SIZE)
                    assert it["res"] == want[0] and it["interp"] == (_lib.VAL_COPY if cache else want[1])
                    assert (it["scratch"] is not None) == (it["new"] != it["res"])
                if run != "det.again":  # with pad 0.5 letterbox only pads
                    assert all(it["scratch"] is None for it in lay.items)


class _Plain:
    """A minimal val dataset: one 20 x 30 image, no labels."""

    def __init__(self, **kw):
        self.img_size, self.augment, self.image_weights, self.rect = 32, False, False, False
        self.indices, self.batch = np.arange(2), np.array([0, 0])
        self.labels, self.segments = [np.zeros((0, 5), np.float32)] * 2, [[], []]
        self.im_files = ["a.png", "b.png"]
        self.ims = [None, None]
        self.overlap, self.downsample_ratio = False, 1
        self.__dict__.update(kw)


def _state():
    return random.getstate(), np.random.get_state()[1].copy(), torch.random.get_rng_state()


def _same_state(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and torch.equal(a[2], b[2])


@pytest.mark.parametrize("cls,kw,exc,match", [
    (DeviceValLoader, dict(augment=True), NotImplementedError, "augment"),
    (DeviceSegValLoader, dict(augment=True), NotImplementedError, "augment"),
    (DeviceValLoader, dict(image_weights=True), NotImplementedError, "image_weights"),
    (DeviceSegValLoader, dict(image_weights=True), NotImplementedError, "image_weights"),
    (DeviceSegValLoader, dict(downsample_ratio=2), NotImplementedError, "downsample_ratio"),
    (DeviceSegValLoader, dict(downsample_ratio=8), NotImplementedError, "downsample_ratio"),
    (DeviceValLoader, dict(rect=True, batch=np.array([0, 1]), batch_shapes=np.array([[32, 32], [32, 32]])), ValueError, "batch_size"),
])
def test_refusals_raise_before_any_work(cls, kw, exc, match):
    ds = _Plain(**kw)
    before = _state()
    calls = []
    with pytest.raises(exc, match=match):
        cls(ds, 2, device=CPU_DEV, decode=lambda d, i: calls.append(i))
    assert _same_state(before, _state()) and not calls


@pytest.mark.parametrize("cls", [DeviceValLoader, DeviceSegValLoader])
@pytest.mark.parametrize("bad", [np.zeros((20, 30, 3), np.float32), np.zeros((20, 30), np.uint8), np.zeros((20, 30, 4), np.uint8),
                                 np.zeros((0, 30, 3), np.uint8)])
def test_images_that_are_not_uint8_bgr_raise(cls, bad):
    ds = _Plain()
    loader = cls(ds, 2, device=CPU_DEV, decode=lambda d, i: (bad, bad.shape[:2], False))
    with pytest.raises(ValueError, match="uint8 HWC|empty"):
        loader.collate([0, 1])


def test_segment_datasets_are_checked():
    with pytest.raises(NotImplementedError, match="segments"):
        DeviceSegValLoader(_Plain(labels=[np.zeros((2, 5), np.float32)] * 2, segments=[[np.zeros((3, 2), np.float32)]] * 2), 2, device=CPU_DEV)
    with pytest.raises(ValueError, match="float32"):
        DeviceSegValLoader(_Plain(labels=[np.zeros((1, 5), np.float32)] * 2, segments=[[np.zeros((3, 2), np.float64)]] * 2), 2, device=CPU_DEV)


def test_default_decode_reads_the_ram_cache_npy_and_image_files(tmp_path):
    cv2 = _cv2()
    from pathlib import Path

    im = pre_ref.synth_image(20, 30, 3)
    f = tmp_path / "a.png"
    cv2.imwrite(str(f), im)
    ds = _Plain(im_files=[str(f), str(f)], npy_files=[Path(tmp_path / "a.npy"), Path(tmp_path / "b.npy")], im_hw0=[(40, 60), None],
                ims=[im[:10], None])
    got, hw0, cached = load_val_image(ds, 0)
    assert cached and hw0 == (40, 60) and got is ds.ims[0]
    got, hw0, cached = load_val_image(ds, 1)
    assert not cached and hw0 == (20, 30) and np.array_equal(got, im)
    np.save(tmp_path / "b.npy", im[::-1])
    got, _, _ = load_val_image(ds, 1)
    assert np.array_equal(got, im[::-1])


def test_val_image_struct_matches_the_c_layout(tmp_path):
    import os

    header = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "y5b200.h")
    fields = [f for f, _ in _lib.ValImage._fields_]
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{header}"', "int main(void) {",
             '  printf("%zu", sizeof(y5_val_image));']
    lines += [f'  printf(" %zu", offsetof(y5_val_image, {f}));' for f in fields]
    lines += ['  printf(" %d %d %d\\n", Y5_VAL_COPY, Y5_VAL_LINEAR, Y5_VAL_AREA);', "  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-o", str(exe), str(src)], check=True)
    size, *rest = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert int(size) == ctypes.sizeof(_lib.ValImage)
    assert [int(v) for v in rest[: len(fields)]] == [getattr(_lib.ValImage, f).offset for f in fields]
    assert [int(v) for v in rest[len(fields):]] == [_lib.VAL_COPY, _lib.VAL_LINEAR, _lib.VAL_AREA]


def test_val_letterbox_argument_validation_without_gpu(built_lib):
    lib = built_lib
    assert lib.y5_val_letterbox(None, 1, 64, 64, 4096, _lib.Y5_U8, None) == -1
    im = _lib.ValImage()
    im.data, im.src_h, im.src_w, im.row_bytes = 4096, 100, 80, 240
    im.res_h, im.res_w, im.new_h, im.new_w, im.interp = 64, 52, 64, 52, _lib.VAL_AREA
    assert lib.y5_val_letterbox(ctypes.byref(im), 1, 64, 64, 4096, 7, None) == -2  # output dtype
    im.top = 1
    assert lib.y5_val_letterbox(ctypes.byref(im), 1, 64, 64, 4096, _lib.Y5_U8, None) == -1 and b"does not fit" in lib.y5_last_error()
    im.top, im.new_h, im.new_w = 0, 60, 48
    assert lib.y5_val_letterbox(ctypes.byref(im), 1, 64, 64, 4096, _lib.Y5_U8, None) == -1 and b"no scratch" in lib.y5_last_error()
    im.new_h, im.new_w, im.res_h, im.res_w = 64, 100, 64, 100
    assert lib.y5_val_letterbox(ctypes.byref(im), 1, 64, 128, 4096, _lib.Y5_U8, None) == -2  # INTER_AREA cannot enlarge
    im.interp, im.res_w, im.new_w = _lib.VAL_COPY, 52, 52
    assert lib.y5_val_letterbox(ctypes.byref(im), 1, 64, 64, 4096, _lib.Y5_U8, None) == -2  # a copy keeps the size
