"""Training augmentation, host side: the oracle (oracle/aug_ref.py) against the reference's batches in
tests/golden/aug.npz, its draw sequence, the public signatures, refused options and argument checks."""
import hashlib
import inspect
import json
import os
import random

import numpy as np
import pytest
import torch

from oracle import aug_ref
from tests import aug_fixture

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def z():
    return aug_fixture.load()


@pytest.mark.parametrize("tag", ["low", "high", "mixed"])
def test_oracle_equals_fixture(z, tag):
    ds = aug_fixture.FixtureDataset(z, aug_fixture.hyps(z)[tag])
    seed = int(z[f"{tag}.seed"])
    random.seed(seed)
    np.random.seed(seed)
    for bi in range(2):
        idx = list(range(bi * aug_fixture.BATCH, min((bi + 1) * aug_fixture.BATCH, ds.n)))
        imgs, targets, params = aug_ref.get_batch(ds, idx)
        assert np.array_equal(imgs, z[f"{tag}.imgs{bi}"])
        assert targets.dtype == np.float32 and np.array_equal(targets.view(np.uint32), z[f"{tag}.targets{bi}"].view(np.uint32))
        draws = np.array([aug_ref.draw_vector(p) for p in params])
        assert np.array_equal(draws, z[f"{tag}.draws{bi}"], equal_nan=True)


def test_fixture_covers_branches(z):
    """The fixture has mosaic and non-mosaic items, mixup, an image without labels and both flips."""
    assert any(z[k].all() == False for k in z.files if k.endswith(("mosaic0", "mosaic1")))  # noqa: E712
    assert any(z[k].any() for k in z.files if ".mixup" in k)
    assert any(len(z[k]) == 0 for k in z.files if k.startswith("labels"))


def test_hsv_tables_digest():
    with open(os.path.join(HERE, "golden", "aug_signatures.json")) as f:
        dig = json.load(f)["hsv_digest"]
    B, G, R = np.meshgrid(np.arange(256), np.arange(256), np.arange(256), indexing="ij")
    bgr = np.stack([B, G, R], -1).astype(np.uint8).reshape(-1, 32, 3)
    assert hashlib.sha256(aug_ref.bgr2hsv(bgr).tobytes()).hexdigest() == dig["bgr2hsv"]
    H, S, V = np.meshgrid(np.arange(180), np.arange(256), np.arange(256), indexing="ij")
    hsv = np.stack([H, S, V], -1).astype(np.uint8)
    assert hashlib.sha256(aug_ref.hsv2bgr(hsv.reshape(-1, 32, 3)).tobytes()).hexdigest() == dig["hsv2bgr_simd"]
    assert hashlib.sha256(aug_ref.hsv2bgr(hsv.reshape(-1, 1, 3)).tobytes()).hexdigest() == dig["hsv2bgr_tail"]


def test_signatures_match_reference():
    from yolov5_b200.utils import augmentations

    with open(os.path.join(HERE, "golden", "aug_signatures.json")) as f:
        ref = json.load(f)
    for name in ("random_perspective", "augment_hsv", "mixup"):
        got = [[n, repr(q.default) if q.default is not inspect._empty else None, str(q.kind)]
               for n, q in inspect.signature(getattr(augmentations, name)).parameters.items()]
        assert got == ref[name], name


def test_loader_draws_match_oracle(z):
    """The loader's draw sequence (yolov5_b200.utils.dataloaders.draw_item) equals the oracle's."""
    from yolov5_b200.utils.dataloaders import draw_item

    for tag, hyp in aug_fixture.hyps(z).items():
        ds = aug_fixture.FixtureDataset(z, hyp)
        for seed in range(3):
            random.seed(seed)
            np.random.seed(seed)
            a = [aug_ref.draw_vector(draw_item(ds, i)) for i in range(ds.n)]
            random.seed(seed)
            np.random.seed(seed)
            b = [aug_ref.draw_vector(aug_ref.sample_params(ds, i)) for i in range(ds.n)]
            assert np.array_equal(np.array(a), np.array(b), equal_nan=True)


def test_affine_matrix_matches_oracle():
    from yolov5_b200.utils.augmentations import affine_matrix, invert_affine

    rng = np.random.default_rng(3)
    for _ in range(200):
        d = (0.0, 0.0, *rng.uniform(-180, 180, 1), *rng.uniform(0.1, 1.9, 1), *rng.uniform(-20, 20, 2), *rng.uniform(0.3, 0.7, 2))
        M = affine_matrix(d, (256, 256), (-64, -64))
        assert np.array_equal(M, aug_ref.affine(d, (256, 256), (-64, -64)))
        assert np.array_equal(np.array(invert_affine(M)).reshape(2, 3), aug_ref.invert_affine(M[:2]))


@pytest.mark.parametrize("key,value", [("perspective", 0.001), ("rect", True), ("segments", True), ("albumentations", True), ("augment", False)])
def test_refused_options(z, key, value):
    from yolov5_b200.utils.augmentations import random_perspective
    from yolov5_b200.utils.dataloaders import DeviceAugmentLoader

    hyp = dict(aug_fixture.hyps(z)["low"])
    ds = aug_fixture.FixtureDataset(z, hyp)
    if key == "perspective":
        hyp["perspective"] = value
        with pytest.raises(NotImplementedError):
            random_perspective(np.zeros((8, 8, 3), np.uint8), perspective=value)
    elif key == "segments":
        ds.segments[1] = [np.zeros((3, 2), np.float32)]
        with pytest.raises(NotImplementedError):
            random_perspective(np.zeros((8, 8, 3), np.uint8), segments=[np.ones((3, 2))])
    elif key == "albumentations":
        ds.albumentations = type("A", (), {"transform": object()})()
    else:
        setattr(ds, key, value)
    with pytest.raises(NotImplementedError):
        DeviceAugmentLoader(ds, 4, device="cpu")


def test_bad_arguments(z):
    from yolov5_b200.utils.augmentations import mixup, random_perspective
    from yolov5_b200.utils.dataloaders import DeviceAugmentLoader

    ds = aug_fixture.FixtureDataset(z, aug_fixture.hyps(z)["low"])
    with pytest.raises(ValueError):
        DeviceAugmentLoader(ds, 4, device="cpu", dtype=torch.int32)
    ds.img_size = 0
    with pytest.raises(ValueError):
        DeviceAugmentLoader(ds, 4, device="cpu")
    with pytest.raises(ValueError):
        random_perspective(np.zeros((8, 8, 3), np.uint8), targets=np.zeros((2, 5), np.float64))
    ds = aug_fixture.FixtureDataset(z, aug_fixture.hyps(z)["low"])
    ds.ims[0] = np.zeros((10, 10), np.uint8)
    loader = DeviceAugmentLoader(ds, 4, device="cpu")
    random.seed(0)
    with pytest.raises(ValueError):
        loader.collate([0, 1, 2, 3])
    with pytest.raises((ValueError, TypeError)):
        mixup(np.zeros((8, 8, 3), np.uint8), np.zeros((0, 5), np.float32), np.zeros((9, 8, 3), np.uint8), np.zeros((0, 5), np.float32))


def test_aug_structs_match_the_c_layout(tmp_path):
    """sizeof / offsetof of y5_aug_tile, y5_aug_image and y5_aug_label (compiled by gcc) == the ctypes mirrors."""
    import ctypes
    import subprocess

    from yolov5_b200 import _lib

    header = os.path.join(os.path.dirname(HERE), "include", "y5b200.h")
    mirrors = {"y5_aug_tile": _lib.AugTile, "y5_aug_image": _lib.AugImage, "y5_aug_label": _lib.AugLabel}
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{header}"', "int main(void) {"]
    for s, cls in mirrors.items():
        lines.append(f'  printf("{s} %zu", sizeof({s}));')
        for f, _ in cls._fields_:
            lines.append(f'  printf(" %zu", offsetof({s}, {f}));')
        lines.append('  printf("\\n");')
    lines += ["  return 0;", "}"]
    (tmp_path / "layout.c").write_text("\n".join(lines))
    subprocess.run(["gcc", "-o", str(tmp_path / "layout"), str(tmp_path / "layout.c")], check=True)
    out = subprocess.run([str(tmp_path / "layout")], capture_output=True, text=True, check=True).stdout.split("\n")
    for line in filter(None, out):
        name, size, *offs = line.split()
        cls = mirrors[name]
        assert int(size) == ctypes.sizeof(cls), name
        assert [int(o) for o in offs] == [getattr(cls, f).offset for f, _ in cls._fields_], name


def test_aug_argument_validation_without_gpu():
    """Null pointers and inconsistent sizes give -1, unsupported dtypes / sizes -2, before any launch."""
    from yolov5_b200 import _lib

    lib = _lib.lib()
    fake = 0x1000
    assert lib.y5_aug_gather(None, 1, 64, 64, 64, 1, fake, _lib.Y5_U8, 0, 0, 0, None) == -1
    assert lib.y5_aug_gather(fake, 1, 64, 64, 65, 1, fake, _lib.Y5_U8, 0, 0, 0, None) == -1
    assert lib.y5_aug_gather(fake, 1, 63, 64, 64, 1, fake, _lib.Y5_F16, 1, 0, 0, None) == -1
    assert lib.y5_aug_gather(fake, 1, 64, 64, 64, 1, fake, 7, 0, 0, 0, None) == -2
    assert lib.y5_aug_gather(fake, 1, 64, 64, 64, 1, fake, _lib.Y5_U8, 1, 0, 0, None) == -2
    assert lib.y5_aug_gather(fake, 1, 40000, 64, 64, 1, fake, _lib.Y5_U8, 0, 0, 0, None) == -2
    assert lib.y5_aug_labels(fake, 1, None, 3, 64, 64, fake, fake, None) == -1
    assert lib.y5_aug_labels(fake, 1, fake, -1, 64, 64, fake, fake, None) == -1
    assert lib.y5_aug_labels(fake, 1, fake, 3, 64, 64, fake, None, None) == -1
