"""The dataset behind tests/golden/seg_aug.npz, duck-typed on the attributes the reference's LoadImagesAndLabelsAndMasks
exposes; `load_image` returns the stored outputs of the reference's own load_image, so neither cv2 nor the reference
tree is needed to replay the fixture."""
import json
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "seg_aug.npz")
IMG_SIZE = 128
BATCH = 4


def load():
    return np.load(GOLDEN)


def runs(z):
    return json.loads(str(z["meta"]))["runs"]


def run_options(run):
    """'low.o1.r4' -> ('low', True, 4)"""
    tag, o, r = run.split(".")
    return tag, o == "o1", int(r[1:])


class SegDataset:
    def __init__(self, z, hyp, overlap, ratio, sources=None, labels=None, segments=None, img_size=IMG_SIZE):
        if sources is None:
            n = sum(1 for k in z.files if k.startswith("src"))
            sources = [z[f"src{k}"] for k in range(n)]
            self.hw0 = [tuple(int(v) for v in z[f"hw0_{k}"]) for k in range(n)]
            labels = [z[f"labels{k}"] for k in range(n)]
            segments = [[z[f"seg{k}_{j}"] for j in range(len(labels[k]))] for k in range(n)]
        else:
            self.hw0 = [s.shape[:2] for s in sources]
        n = len(sources)
        self.ims, self.labels, self.segments = sources, labels, segments
        self.img_size = img_size
        self.augment, self.rect, self.mosaic = True, False, True
        self.mosaic_border = [-img_size // 2, -img_size // 2]
        self.hyp = hyp
        self.indices = np.arange(n)
        self.n = n
        self.im_files = [f"im{k}.png" for k in range(n)]
        self.albumentations = None
        self.overlap, self.downsample_ratio = overlap, ratio

    def __len__(self):
        return self.n

    def load_image(self, i):
        return self.ims[i], self.hw0[i], self.ims[i].shape[:2]


def hyps(z):
    return json.loads(str(z["hyps"]))
