"""The dataset behind tests/golden/aug.npz, duck-typed on the attributes the reference's LoadImagesAndLabels exposes:
`load_image` returns the stored outputs of the reference's own load_image (imread + cv2.resize), so neither cv2 nor the
reference tree is needed to replay the fixture."""
import json
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "aug.npz")
IMG_SIZE = 128
BATCH = 4


def load():
    return np.load(GOLDEN)


class FixtureDataset:
    def __init__(self, z, hyp, sources=None, labels=None, img_size=IMG_SIZE):
        n = sum(1 for k in z.files if k.startswith("src")) if sources is None else len(sources)
        self.ims = [z[f"src{k}"] for k in range(n)] if sources is None else sources
        self.hw0 = [tuple(int(v) for v in z[f"hw0_{k}"]) for k in range(n)] if sources is None else [s.shape[:2] for s in sources]
        self.labels = [z[f"labels{k}"] for k in range(n)] if labels is None else labels
        self.segments = [[] for _ in range(n)]
        self.img_size = img_size
        self.augment, self.rect, self.mosaic = True, False, True
        self.mosaic_border = [-img_size // 2, -img_size // 2]
        self.hyp = hyp
        self.indices = np.arange(n)
        self.n = n
        self.im_files = [f"im{k}.png" for k in range(n)]
        self.albumentations = None

    def __len__(self):
        return self.n

    def load_image(self, i):
        return self.ims[i], self.hw0[i], self.ims[i].shape[:2]


def hyps(z):
    return json.loads(str(z["hyps"]))
