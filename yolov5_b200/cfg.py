"""Architecture tables for the YOLOv5 v6.0 family (n/s/m/l/x and the -seg variants).

The reference keeps these as YAML files (``models/yolov5{n,s,m,l,x}.yaml``,
``models/segment/yolov5*-seg.yaml``); all ten share one topology and differ only in the two
scaling multiples.  Here the topology is data in code so the engine needs no file on disk, and
``model_cfg`` returns a dict with exactly the keys ``yaml.safe_load`` yields for the reference
files (pinned by tests/test_cfg_golden.py against a digest taken from the reference YAMLs).
A user-supplied ``*.yaml`` path is still accepted by ``DetectionModel`` (see models/yolo.py).

``yolov5s-transformer`` (reference models/hub/yolov5s-transformer.yaml) is yolov5s with a C3TR in place of the backbone's last
C3 (layer 8); it is a built-in name too, pinned by tests/test_transformer_cpu.py against a digest of that YAML.
``yolov5s-ghost`` (reference models/hub/yolov5s-ghost.yaml) is yolov5s built from GhostConv and C3Ghost; ``model_cfg`` accepts
it, pinned by tests/test_ghost_cpu.py, but it is not one of ``model_names()``.
"""
from __future__ import annotations

import copy
from pathlib import Path

# (depth_multiple, width_multiple) -- reference models/yolov5{n,s,m,l,x}.yaml:10-11
_SCALES = {"n": (0.33, 0.25), "s": (0.33, 0.50), "m": (0.67, 0.75), "l": (1.0, 1.0), "x": (1.33, 1.25)}

# reference models/yolov5s.yaml:12-15 (pixels, P3/P4/P5)
_ANCHORS = [[10, 13, 16, 30, 33, 23], [30, 61, 62, 45, 59, 119], [116, 90, 156, 198, 373, 326]]


def _topology(head_module: str, head_args: list) -> tuple[list, list]:
    """[from, repeats, module, args] rows; reference models/yolov5s.yaml:18-54."""
    down = lambda c: [-1, 1, "Conv", [c, 3, 2]]  # noqa: E731  stride-2 3x3
    csp = lambda c, n, *a: [-1, n, "C3", [c, *a]]  # noqa: E731
    backbone = [
        [-1, 1, "Conv", [64, 6, 2, 2]],  # 0  P1/2
        down(128),  # 1  P2/4
        csp(128, 3),
        down(256),  # 3  P3/8
        csp(256, 6),
        down(512),  # 5  P4/16
        csp(512, 9),
        down(1024),  # 7  P5/32
        csp(1024, 3),
        [-1, 1, "SPPF", [1024, 5]],  # 9
    ]
    up = [-1, 1, "nn.Upsample", ["None", 2, "nearest"]]  # YAML loads the bare word None as a string
    head = [
        [-1, 1, "Conv", [512, 1, 1]],  # 10
        copy.deepcopy(up),
        [[-1, 6], 1, "Concat", [1]],
        csp(512, 3, False),  # 13
        [-1, 1, "Conv", [256, 1, 1]],  # 14
        copy.deepcopy(up),
        [[-1, 4], 1, "Concat", [1]],
        csp(256, 3, False),  # 17 P3 out
        [-1, 1, "Conv", [256, 3, 2]],
        [[-1, 14], 1, "Concat", [1]],
        csp(512, 3, False),  # 20 P4 out
        [-1, 1, "Conv", [512, 3, 2]],
        [[-1, 10], 1, "Concat", [1]],
        csp(1024, 3, False),  # 23 P5 out
        [[17, 20, 23], 1, head_module, head_args],
    ]
    return backbone, head


_YOLOV3 = ("yolov3", "yolov3-spp", "yolov3-tiny")


def _yolov3(name: str) -> dict:
    """Reference models/hub/yolov3.yaml, yolov3-spp.yaml and yolov3-tiny.yaml as yaml.safe_load returns them."""
    conv = lambda c, k=1, s=1: [-1, 1, "Conv", [c, k, s]]  # noqa: E731
    up = [-1, 1, "nn.Upsample", ["None", 2, "nearest"]]
    if name == "yolov3-tiny":
        pool = [-1, 1, "nn.MaxPool2d", [2, 2, 0]]
        backbone = []
        for c in (16, 32, 64, 128, 256):
            backbone += [conv(c, 3, 1), copy.deepcopy(pool)]
        backbone += [conv(512, 3, 1), [-1, 1, "nn.ZeroPad2d", [[0, 1, 0, 1]]], [-1, 1, "nn.MaxPool2d", [2, 1, 0]]]
        head = [conv(1024, 3, 1), conv(256, 1, 1), conv(512, 3, 1), [-2, 1, "Conv", [128, 1, 1]], copy.deepcopy(up),
                [[-1, 8], 1, "Concat", [1]], conv(256, 3, 1), [[19, 15], 1, "Detect", ["nc", "anchors"]]]
        anchors = [[10, 14, 23, 27, 37, 58], [81, 82, 135, 169, 344, 319]]
    else:
        backbone = [conv(32, 3, 1), conv(64, 3, 2), [-1, 1, "Bottleneck", [64]]]
        for c, n in ((128, 2), (256, 8), (512, 8), (1024, 4)):
            backbone += [conv(c, 3, 2), [-1, n, "Bottleneck", [c]]]
        p5 = [-1, 1, "SPP", [512, [5, 9, 13]]] if name == "yolov3-spp" else conv(512, 1, 1)
        head = [[-1, 1, "Bottleneck", [1024, False]], p5, conv(1024, 3, 1), conv(512, 1, 1), conv(1024, 3, 1),
                [-2, 1, "Conv", [256, 1, 1]], copy.deepcopy(up), [[-1, 8], 1, "Concat", [1]], [-1, 1, "Bottleneck", [512, False]],
                [-1, 1, "Bottleneck", [512, False]], conv(256, 1, 1), conv(512, 3, 1), [-2, 1, "Conv", [128, 1, 1]], copy.deepcopy(up),
                [[-1, 6], 1, "Concat", [1]], [-1, 1, "Bottleneck", [256, False]], [-1, 2, "Bottleneck", [256, False]],
                [[27, 22, 15], 1, "Detect", ["nc", "anchors"]]]
        anchors = copy.deepcopy(_ANCHORS)
    return {"nc": 80, "depth_multiple": 1.0, "width_multiple": 1.0, "anchors": anchors, "backbone": backbone, "head": head}


def _ghost() -> dict:
    """Reference models/hub/yolov5s-ghost.yaml as yaml.safe_load returns it: yolov5s with every stride-2 Conv and the head's 1x1
    Convs as GhostConv, and every C3 as C3Ghost."""
    cfg = model_cfg("yolov5s")
    for row in cfg["backbone"] + cfg["head"]:
        if row[2] == "C3":
            row[2] = "C3Ghost"
        elif row[2] == "Conv" and row[3] != [64, 6, 2, 2]:  # all but the stem
            row[2] = "GhostConv"
    return cfg


def model_names() -> list[str]:
    return [f"yolov5{k}" for k in _SCALES] + [f"yolov5{k}-seg" for k in _SCALES]


def model_cfg(name: str) -> dict:
    """Return the model dict for ``yolov5s`` / ``yolov5l.yaml`` / ``models/segment/yolov5x-seg.yaml`` /
    ``models/hub/yolov5s-transformer.yaml`` ..."""
    stem = Path(str(name)).name
    if stem.endswith(".yaml"):
        stem = stem[: -len(".yaml")]
    if stem == "yolov5s-transformer":
        cfg = model_cfg("yolov5s")
        cfg["backbone"][8][2] = "C3TR"  # [-1, 3, C3TR, [1024]]: layer 8, the backbone's last C3
        return cfg
    if stem in _YOLOV3:
        return _yolov3(stem)
    if stem == "yolov5s-ghost":
        return _ghost()
    seg = stem.endswith("-seg")
    key = stem[: -len("-seg")] if seg else stem
    if not (key.startswith("yolov5") and key[6:] in _SCALES):
        raise KeyError(f"unknown YOLOv5 model '{name}' (known: {model_names()})")
    gd, gw = _SCALES[key[6:]]
    if seg:
        backbone, head = _topology("Segment", ["nc", "anchors", 32, 256])
    else:
        backbone, head = _topology("Detect", ["nc", "anchors"])
    return {
        "nc": 80,
        "depth_multiple": gd,
        "width_multiple": gw,
        "anchors": copy.deepcopy(_ANCHORS),
        "backbone": backbone,
        "head": head,
    }


# reference data/hyps/hyp.scratch-low.yaml -- only the keys the loss path reads
# (utils/loss.py:107-132 and train.py:326-328).
HYP_SCRATCH_LOW = {
    "lr0": 0.01,
    "lrf": 0.01,
    "momentum": 0.937,
    "weight_decay": 0.0005,
    "warmup_epochs": 3.0,
    "warmup_momentum": 0.8,
    "warmup_bias_lr": 0.1,
    "box": 0.05,
    "cls": 0.5,
    "cls_pw": 1.0,
    "obj": 1.0,
    "obj_pw": 1.0,
    "iou_t": 0.20,
    "anchor_t": 4.0,
    "fl_gamma": 0.0,
    "label_smoothing": 0.0,
}
