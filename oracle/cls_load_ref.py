"""ORACLE (test infrastructure, never on the product path): CPU restatement of the classification dataloader's per-item
transform -- classify_transforms(size) = Compose([CenterCrop(size), ToTensor(), Normalize(IMAGENET_MEAN, IMAGENET_STD)])
-- and of ClassificationDataset.__getitem__'s image read.  numpy arithmetic.

Reference lines restated (paths relative to the reference tree):
  utils/augmentations.py:297-341  classify_transforms, CenterCrop, ToTensor            -> center_square, transform
  utils/augmentations.py:15-16    IMAGENET_MEAN, IMAGENET_STD                          -> IMAGENET_MEAN, IMAGENET_STD
  utils/dataloaders.py:968-985    ClassificationDataset.__getitem__ (album_transforms None)
Third-party arithmetic: cv2.resize INTER_LINEAR (oracle/pre_ref.resize_linear_u8, pinned against the installed cv2) and
torchvision's Normalize, which computes (x - mean) / std on float32 tensors of the Python constants.  ToTensor's `/= 255`
runs on a CPU float32 tensor, where torch divides (it multiplies by the reciprocal only for half and bfloat16), so the
restatement divides too.  Pinned by tests/golden/cls_load.npz, written by tests/golden/make_cls_load_golden.py from the
unmodified reference.

`CenterCrop`, `ToTensor` and `classify_transforms` are call-compatible stand-ins for the reference's classes (same names
and attributes), so a test dataset can carry them as its `torch_transforms`.
"""
from __future__ import annotations

import numpy as np
import torch

from .pre_ref import resize_linear_u8

IMAGENET_MEAN = 0.485, 0.456, 0.406  # RGB
IMAGENET_STD = 0.229, 0.224, 0.225


def center_square(im: np.ndarray) -> np.ndarray:
    """The m x m square CenterCrop resizes, m = min(h, w), floored offsets (a view)."""
    h, w = im.shape[:2]
    m = min(h, w)
    top, left = (h - m) // 2, (w - m) // 2
    return im[top: top + m, left: left + m]


def to_float(im_hwc_bgr: np.ndarray) -> np.ndarray:
    """ToTensor: HWC BGR uint8 -> CHW RGB float32 / 255 (a true division)."""
    x = np.ascontiguousarray(im_hwc_bgr.transpose(2, 0, 1)[::-1]).astype(np.float32)
    return x / np.float32(255)


def normalize(x: np.ndarray, mean=IMAGENET_MEAN, std=IMAGENET_STD) -> np.ndarray:
    m = np.asarray(mean, np.float32)[:, None, None]
    s = np.asarray(std, np.float32)[:, None, None]
    return (x - m) / s


def transform(im: np.ndarray, size) -> np.ndarray:
    """classify_transforms(size)(im) -> (3, h, w) float32."""
    h, w = (size, size) if isinstance(size, int) else size
    return normalize(to_float(resize_linear_u8(center_square(im), (w, h))))


def batch(ims, size) -> np.ndarray:
    return np.stack([transform(im, size) for im in ims], 0)


class CenterCrop:
    def __init__(self, size=640):
        self.h, self.w = (size, size) if isinstance(size, int) else size

    def __call__(self, im):
        return resize_linear_u8(center_square(im), (self.w, self.h))


class ToTensor:
    def __init__(self, half=False):
        self.half = half

    def __call__(self, im):
        if self.half:
            raise NotImplementedError("the oracle restates ToTensor(half=False) only")
        return torch.from_numpy(to_float(im))


def classify_transforms(size=224):
    import torchvision.transforms as T

    return T.Compose([CenterCrop(size), ToTensor(), T.Normalize(IMAGENET_MEAN, IMAGENET_STD)])
