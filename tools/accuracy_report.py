"""Prints max-abs error / max|oracle| of the engine and of torch's low-precision evaluation of the reference, per
model output (z, raw levels, proto), on an H100.   python tools/accuracy_report.py"""
import os, sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests.test_model_gpu import _check_model


def main():
    dev = torch.device("cuda:0")
    cases = [("yolov5s", (2, 3, 640, 640), torch.float16), ("yolov5s", (2, 3, 640, 640), torch.bfloat16),
             ("yolov5l", (2, 3, 320, 320), torch.float16), ("yolov5x-seg", (1, 3, 128, 128), torch.float16),
             ("yolov5n", (1, 3, 640, 640), torch.float16)]
    for name, shape, dt in cases:
        try:
            rep, _, _ = _check_model(name, shape, 3, 103, dt, dev)
            print(name, shape, dt, " ".join(f"{k}:eng={a:.2e}/low={b:.2e}" for k, (a, b) in rep.items()), flush=True)
        except AssertionError as e:
            print(name, shape, dt, "FAIL", e, flush=True)


if __name__ == "__main__":
    main()
