"""CPU: the classification loader's host side and oracle -- oracle/cls_load_ref.py against tests/golden/cls_load.npz (the
reference's own batches) and against cv2 + torchvision over a size sweep; the loader's index stream against the recorded
one; the refusals; the default decode's caches; the y5_cls_image ABI."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import cls_load_ref as R
from oracle import pre_ref
from tests import cls_load_fixture as F
from yolov5_b200 import _lib
from yolov5_b200.utils.dataloaders import DeviceClassifyLoader, load_cls_image

CPU_DEV = "cuda:0"  # a device name only: nothing below reaches the device


@pytest.fixture(scope="module")
def z():
    return F.load()


def test_oracle_equals_fixture(z):
    ds = F.ClsDataset(z)
    for i, src in enumerate(ds.src):
        want = z[f"img{i}"]
        assert np.array_equal(R.transform(src, F.IMG_SIZE).view(np.uint32), want.view(np.uint32)), (i, src.shape)
        assert np.array_equal(ds.torch_transforms(src).numpy().view(np.uint32), want.view(np.uint32)), i


def test_fixture_covers_every_crop_path(z):
    s = F.IMG_SIZE
    sides = {min(src.shape[:2]) for src in F.ClsDataset(z).src}
    shapes = [src.shape[:2] for src in F.ClsDataset(z).src]
    assert {s, 2 * s, 3 * s, 1} <= sides and any(m < s for m in sides) and any(s < m < 2 * s for m in sides)
    assert any(h > w for h, w in shapes) and any(h < w for h, w in shapes) and any(h == w for h, w in shapes)
    assert any((h - w) % 2 for h, w in shapes if h > w) and any((w - h) % 2 for h, w in shapes if w > h)


def _sweep():
    rs = np.random.RandomState(11)
    cases = [(375, 500, 224), (500, 375, 224), (448, 600, 224), (224, 300, 224), (672, 672, 224), (1, 50, 224), (50, 1, 224), (3000, 4000, 224),
             (100, 37, 37), (1, 1, 5)]
    for _ in range(300):
        cases.append((int(rs.randint(1, 800)), int(rs.randint(1, 800)), int(rs.choice([224, 225, 97, 33, 1, 383]))))
    return cases


def test_oracle_equals_cv2_and_torchvision_over_a_size_sweep():
    cv2 = pytest.importorskip("cv2", reason="the crop's resize is pinned against the installed cv2")
    T = pytest.importorskip("torchvision.transforms")
    norm = T.Normalize(R.IMAGENET_MEAN, R.IMAGENET_STD)
    rs = np.random.RandomState(12)
    for h, w, s in _sweep():
        im = pre_ref.synth_image(h, w, h * 5 + w) if rs.rand() < 0.5 else rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
        m = min(h, w)
        top, left = (h - m) // 2, (w - m) // 2
        crop = cv2.resize(im[top: top + m, left: left + m], (s, s), interpolation=cv2.INTER_LINEAR)
        x = torch.from_numpy(np.ascontiguousarray(crop.transpose(2, 0, 1)[::-1])).float()
        x /= 255.0
        want = norm(x).numpy()
        assert np.array_equal(R.transform(im, s).view(np.uint32), want.view(np.uint32)), (h, w, s)


def test_true_division_is_not_the_reciprocal_product():
    """ToTensor's `/= 255` on a CPU float32 tensor differs from x * float32(1 / 255) for many byte values."""
    x = torch.arange(256, dtype=torch.float32)
    y = x.clone()
    y /= 255.0
    assert torch.equal(y, torch.from_numpy(np.arange(256, dtype=np.float32) / np.float32(255)))
    assert int((y != x * torch.tensor(1 / 255, dtype=torch.float32)).sum()) > 50


def _index_loader(ds, batch, **kw):
    loader = DeviceClassifyLoader(ds, batch, device=CPU_DEV, decode=lambda d, i: i, **kw)
    loader.collate = lambda items, loaded: (list(items), loaded)
    return loader


def test_index_stream_equals_the_reference(z):
    """next(iter(loader)), then three passes: the items and their order the reference's InfiniteDataLoader drew."""
    m = F.meta(z)
    ds = F.ClsDataset(z)
    loader = _index_loader(ds, m["batch"], workers=2)
    assert len(loader) == len(m["stream"]["passes"][0])
    items, loaded = next(iter(loader))
    assert items == m["stream"]["first"] and loaded == items
    for p in m["stream"]["passes"]:
        assert [b for b, _ in loader] == p
    for run in m["runs"].values():
        assert run == m["stream"]


def test_batch_size_is_capped_and_a_pass_left_early_keeps_its_drawn_batch(z):
    ds = F.ClsDataset(z)
    assert len(_index_loader(ds, 1000)) == 1 and _index_loader(ds, 1000).batch_size == len(ds)
    a, b = _index_loader(ds, 3, workers=3), _index_loader(ds, 3, workers=1)
    want = [x for _ in range(4) for x, _ in b]
    got = []
    for k in range(4):  # leave passes after k + 1 batches: the batch drawn ahead comes first in the next pass
        for j, (x, _) in enumerate(a):
            got.append(x)
            if j == k:
                break
    assert got == want[: len(got)]


def test_rank_env_seeds_the_generator(z, monkeypatch):
    ds = F.ClsDataset(z)
    base = [x for x, _ in _index_loader(ds, 4)]
    monkeypatch.setenv("RANK", "-1")
    assert [x for x, _ in _index_loader(ds, 4)] == base
    g = torch.Generator()
    g.manual_seed(6148914691236517205 + 3)
    monkeypatch.setenv("RANK", "3")
    assert [x for x, _ in _index_loader(ds, 4)] == [list(b) for b in torch.utils.data.DataLoader(range(len(ds)), 4, shuffle=True, generator=g,
                                                                                             collate_fn=list)]
    assert [x for x, _ in _index_loader(ds, 4, shuffle=False)] == [list(range(i, min(i + 4, len(ds)))) for i in range(0, len(ds), 4)]


def test_distributed_sampler_and_set_epoch(z, tmp_path):
    import torch.distributed as dist

    ds = F.ClsDataset(z)
    dist.init_process_group("gloo", init_method=f"file://{tmp_path / 'store'}", rank=0, world_size=1)
    try:
        loader = _index_loader(ds, 4, rank=0)
        assert isinstance(loader.sampler, torch.utils.data.DistributedSampler) and loader.sampler.shuffle
        e0 = [x for x, _ in loader]
        loader.sampler.set_epoch(1)
        e1 = [x for x, _ in loader]
        s = torch.utils.data.DistributedSampler(ds, shuffle=True)
        want0 = list(s)
        s.set_epoch(1)
        want1 = list(s)
        assert sum(e0, []) == want0 and sum(e1, []) == want1 and want0 != want1
    finally:
        dist.destroy_process_group()


class _Bad:
    def __init__(self, **kw):
        z = F.load()
        self.__dict__.update(F.ClsDataset(z).__dict__)
        self.__dict__.update(kw)

    def __len__(self):
        return len(self.samples)


def _transforms(*ts):
    import torchvision.transforms as T

    return T.Compose(list(ts))


class CenterCrop(R.CenterCrop):
    """A user class with the reference's name and attributes, from another module."""


class ToTensor(R.ToTensor):
    pass


def _refusals():
    import torchvision.transforms as T

    norm = T.Normalize(R.IMAGENET_MEAN, R.IMAGENET_STD)
    return [
        (dict(album_transforms=_transforms(T.RandomHorizontalFlip())), NotImplementedError, "Albumentations"),
        (dict(torch_transforms=_transforms(T.CenterCrop(32), R.ToTensor(), norm)), NotImplementedError, "classify_transforms"),
        (dict(torch_transforms=_transforms(R.CenterCrop(32), R.ToTensor(half=True), norm)), NotImplementedError, "half"),
        (dict(torch_transforms=_transforms(R.CenterCrop(32), T.ToTensor(), norm)), NotImplementedError, "classify_transforms"),
        (dict(torch_transforms=_transforms(R.CenterCrop(32), R.ToTensor(), T.Normalize((0.5,) * 3, (0.5,) * 3))), NotImplementedError, "IMAGENET"),
        (dict(torch_transforms=_transforms(R.CenterCrop(32), R.ToTensor())), NotImplementedError, "classify_transforms"),
        (dict(torch_transforms=None), NotImplementedError, "classify_transforms"),
        (dict(torch_transforms=_transforms(CenterCrop(32), R.ToTensor(), norm)), NotImplementedError, "classify_transforms"),
        (dict(torch_transforms=_transforms(R.CenterCrop(32), ToTensor(), norm)), NotImplementedError, "classify_transforms"),
        (dict(torch_transforms=R.classify_transforms(0)), ValueError, "outside"),
        (dict(torch_transforms=R.classify_transforms(16385)), ValueError, "outside"),
        (dict(torch_transforms=R.classify_transforms((32, 0))), ValueError, "outside"),
    ]


@pytest.mark.parametrize("case", range(12))
def test_refusals_raise_before_any_work(case):
    kw, exc, match = _refusals()[case]
    calls = []
    state = torch.random.get_rng_state()
    with pytest.raises(exc, match=match):
        DeviceClassifyLoader(_Bad(**kw), 4, device=CPU_DEV, decode=lambda d, i: calls.append(i))
    assert not calls and torch.equal(state, torch.random.get_rng_state())


def test_accepts_the_largest_size_and_float_dtypes_only(z):
    DeviceClassifyLoader(_Bad(torch_transforms=R.classify_transforms(16384)), 4, device=CPU_DEV)
    with pytest.raises(ValueError, match="dtype"):
        DeviceClassifyLoader(F.ClsDataset(z), 4, device=CPU_DEV, dtype=torch.uint8)


@pytest.mark.parametrize("bad", [np.zeros((20, 30, 3), np.float32), np.zeros((20, 30), np.uint8), np.zeros((20, 30, 4), np.uint8),
                                 np.zeros((0, 30, 3), np.uint8)])
def test_images_that_are_not_uint8_bgr_raise(z, bad):
    loader = DeviceClassifyLoader(F.ClsDataset(z), 4, device=CPU_DEV, decode=lambda d, i: bad)
    with pytest.raises(ValueError, match="uint8 HWC|empty"):
        loader.collate([0, 1])


def test_default_decode_reads_the_caches_and_image_files(tmp_path):
    cv2 = pytest.importorskip("cv2")
    from pathlib import Path

    im = pre_ref.synth_image(20, 30, 3)
    f = tmp_path / "a.png"
    cv2.imwrite(str(f), im)
    ds = _Bad(samples=[[str(f), 0, Path(tmp_path / "a.npy"), None], [str(tmp_path / "missing.png"), 1, Path(tmp_path / "m.npy"), None]])
    assert np.array_equal(load_cls_image(ds, 0), im) and ds.samples[0][3] is None
    ds.cache_ram = True
    got = load_cls_image(ds, 0)
    assert np.array_equal(got, im) and ds.samples[0][3] is got and load_cls_image(ds, 0) is got
    ds.cache_ram, ds.cache_disk = False, True
    assert np.array_equal(load_cls_image(ds, 0), im) and np.array_equal(np.load(tmp_path / "a.npy"), im)
    np.save(tmp_path / "a.npy", im[::-1])
    assert np.array_equal(load_cls_image(ds, 0), im[::-1])  # the .npy, once written, is what the disk cache reads
    assert sorted(os.listdir(tmp_path)) == ["a.npy", "a.png"]
    with pytest.raises(FileNotFoundError, match="missing.png"):
        load_cls_image(ds, 1)


def test_cls_image_struct_matches_the_c_layout(tmp_path):
    header = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "y5b200.h")
    fields = [f for f, _ in _lib.ClsImage._fields_]
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{header}"', "int main(void) {",
             '  printf("%zu", sizeof(y5_cls_image));']
    lines += [f'  printf(" %zu", offsetof(y5_cls_image, {f}));' for f in fields]
    lines += ['  printf("\\n");', "  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-o", str(exe), str(src)], check=True)
    size, *rest = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert int(size) == ctypes.sizeof(_lib.ClsImage)
    assert [int(v) for v in rest] == [getattr(_lib.ClsImage, f).offset for f in fields]


def test_cls_batch_argument_validation_without_gpu(built_lib):
    lib = built_lib
    mean, std = (ctypes.c_float * 3)(*R.IMAGENET_MEAN), (ctypes.c_float * 3)(*R.IMAGENET_STD)
    assert lib.y5_cls_batch(None, 1, 224, 224, mean, std, 4096, _lib.Y5_F32, None) == -1
    assert lib.y5_cls_batch(4096, 0, 224, 224, mean, std, 4096, _lib.Y5_F32, None) == -1
    assert lib.y5_cls_batch(4096, 1, 224, 224, mean, std, 4096, _lib.Y5_U8, None) == -2  # no uint8 output
    assert lib.y5_cls_batch(4096, 1, 16385, 224, mean, std, 4096, _lib.Y5_F32, None) == -2
    assert lib.y5_cls_batch(4096, 65536, 224, 224, mean, std, 4096, _lib.Y5_F32, None) == -2
    zero = (ctypes.c_float * 3)(0.229, 0.0, 0.225)
    assert lib.y5_cls_batch(4096, 1, 224, 224, mean, zero, 4096, _lib.Y5_F32, None) == -1 and b"std" in lib.y5_last_error()
