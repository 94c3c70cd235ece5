"""GPU: the classification loader (y5_cls_batch through DeviceClassifyLoader) against the reference's batches
(tests/golden/cls_load.npz), the kernel against the oracle (oracle/cls_load_ref.py) over a size sweep at 224, and
classify/val.py's loop body on the loader's batches."""
import numpy as np
import pytest
import torch

from oracle import cls_load_ref as R
from oracle import pre_ref
from tests import cls_load_fixture as F

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0") if torch.cuda.is_available() else None
_BITS = {torch.float16: torch.int16, torch.bfloat16: torch.int16, torch.float32: torch.int32}


@pytest.fixture(scope="module")
def z():
    return F.load()


def _loader(ds, batch, dtype=torch.float32, workers=4, decode=F.decode):
    from yolov5_b200.utils.dataloaders import DeviceClassifyLoader

    return DeviceClassifyLoader(ds, batch, device=DEV, dtype=dtype, workers=workers, decode=decode)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_loader_reproduces_fixture(z, dtype):
    """next(iter(loader)) and three passes: fp32 bit for bit, fp16 / bf16 the reference batch rounded once."""
    m = F.meta(z)
    loader = _loader(F.ClsDataset(z), m["batch"], dtype)
    batches = [next(iter(loader))] + [b for _ in range(3) for b in loader]
    items = [m["stream"]["first"]] + [b for p in m["stream"]["passes"] for b in p]
    assert len(batches) == len(items)
    for (images, labels), it in zip(batches, items):
        want, want_labels = F.expected(z, it)
        assert images.device == DEV and labels.device == DEV and images.dtype == dtype and labels.dtype == torch.int64
        assert images.shape == (len(it), 3, F.IMG_SIZE, F.IMG_SIZE) and labels.shape == (len(it),)
        ref = torch.from_numpy(want).to(DEV).to(dtype)
        assert torch.equal(images.view(_BITS[dtype]), ref.view(_BITS[dtype])), (dtype, it)
        assert torch.equal(labels.cpu(), torch.from_numpy(want_labels)), it


def _sweep():
    s = 224
    rs = np.random.RandomState(21)
    shapes = [(1, 300), (300, 1), (1, 1), (2 * s, 2 * s), (2 * s, 600), (700, 2 * s), (s, s), (s, 400), (3 * s, 3 * s + 1), (4000, 3000), (375, 500),
              (500, 375), (100, 101), (37, 5000)]
    shapes += [(int(rs.randint(1, 900)), int(rs.randint(1, 900))) for _ in range(200)]
    return [pre_ref.synth_image(h, w, h * 3 + w) if rs.rand() < 0.5 else rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]


class _Images:
    """A dataset of in-memory images (the decode hook returns them) with classify_transforms(size)."""

    def __init__(self, ims, size):
        self.ims = ims
        self.samples = [[f"im{i}.jpg", i % 7, None, None] for i in range(len(ims))]
        self.torch_transforms = R.classify_transforms(size)
        self.album_transforms = None
        self.cache_ram = self.cache_disk = False

    def __len__(self):
        return len(self.samples)


def test_kernel_equals_oracle_at_224_over_a_size_sweep():
    """214 images in one launch: 1 x N, N x 1, m = size (a copy), m = 2 size (the 2x average), m = 3 size, 4000 x 3000."""
    from yolov5_b200 import _lib

    ims = _sweep()
    ds = _Images(ims, 224)
    loader = _loader(ds, len(ims), decode=lambda d, i: d.ims[i])
    n0 = _lib.launch_count()
    images, labels = loader.collate(list(range(len(ims))))
    assert _lib.launch_count() - n0 == 1
    got = images.cpu().numpy()
    for i, im in enumerate(ims):
        assert np.array_equal(got[i].view(np.uint32), R.transform(im, 224).view(np.uint32)), im.shape
    assert labels.tolist() == [i % 7 for i in range(len(ims))]
    # m == size: cv2 copies; m == 2 size: (p00 + p01 + p10 + p11 + 2) >> 2
    for k in (6, 3):
        sq = R.center_square(ims[k]).astype(np.int32)
        u8 = sq if sq.shape[0] == 224 else (sq[0::2, 0::2] + sq[0::2, 1::2] + sq[1::2, 0::2] + sq[1::2, 1::2] + 2) >> 2
        want = R.normalize(R.to_float(u8.astype(np.uint8)))
        assert np.array_equal(got[k].view(np.uint32), want.view(np.uint32)), ims[k].shape


def test_130_image_batch_is_one_launch_in_dataset_order(z):
    from yolov5_b200 import _lib

    ds = F.ClsDataset(z)
    n = len(ds.samples)
    ds.samples = [list(ds.samples[i % n]) for i in range(130)]
    ds.src = [ds.src[i % n] for i in range(130)]
    loader = _loader(ds, 130, torch.float16)
    assert len(loader) == 1
    n0 = _lib.launch_count()
    images, labels = loader.collate(list(range(130)))
    assert _lib.launch_count() - n0 == 1
    want, want_labels = F.expected(z, [i % n for i in range(130)])
    assert torch.equal(images.view(torch.int16), torch.from_numpy(want).to(DEV).half().view(torch.int16))
    assert labels.dtype == torch.int64 and labels.device == DEV and torch.equal(labels.cpu(), torch.from_numpy(want_labels))


def test_classify_val_loop_body(z):
    """classify/val.py:110-126 runs unchanged on the loader's output (device, dtype, shapes, int64 labels) with the
    reference-pickled ClassificationModel.  The batches equal the oracle's bit for bit, so the predictions and top-1 /
    top-5 then equal those of the oracle's batches by construction; that comparison only confirms the loop completed."""
    import os

    from yolov5_b200.models.experimental import attempt_load

    model = attempt_load(os.path.join(os.path.dirname(__file__), "golden", "ref_cls_tiny.pt"), device=DEV).half().eval()
    ds = F.ClsDataset(z, size=64)
    loader = _loader(ds, 6)

    def run(batches):
        pred, targets = [], []
        with torch.autocast("cuda"):
            for images, labels in batches:
                images, labels = images.to(DEV, non_blocking=True), labels.to(DEV)
                y = model(images)
                pred.append(y.argsort(1, descending=True)[:, :5])
                targets.append(labels)
        pred, targets = torch.cat(pred), torch.cat(targets)
        correct = (targets[:, None] == pred).float()
        acc = torch.stack((correct[:, 0], correct.max(1).values), dim=1)
        return pred, acc.mean(0).tolist()

    got = list(loader)
    probe = _loader(ds, 6)  # the same index stream: its first pass names the items of `got`
    probe.collate = lambda it, loaded: it
    items = list(probe)
    ref = [(torch.from_numpy(R.batch([ds.src[i] for i in it], 64)).to(DEV), torch.tensor([ds.samples[i][1] for i in it], device=DEV)) for it in items]
    for (a, _), (b, _) in zip(got, ref):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    p_got, acc_got = run(got)
    p_ref, acc_ref = run(ref)
    assert torch.equal(p_got, p_ref) and acc_got == acc_ref
