"""Import-path compatibility with the reference: ``install()`` registers this package's modules under the names the
reference's scripts and pickled checkpoints use (``models.common``, ``models.yolo``, ``models.experimental``,
``utils.general``, ``utils.loss``, ``utils.metrics``, ``utils.torch_utils``, ``utils.augmentations``,
``utils.segment.general``, ``utils.segment.loss``, ``utils.segment.metrics``), so

    from models.yolo import DetectionModel          # reference val.py:39 / train.py:49 style imports
    torch.load("reference_checkpoint.pt")           # pickles naming models.yolo.DetectionModel, models.common.Conv ...

resolve to the engine's classes.  Nothing is registered when a *different* package already owns one of those names (for
example the reference itself on sys.path) unless ``force=True``.
"""
from __future__ import annotations

import importlib
import sys

ALIASES = {
    "models": "yolov5_b200.models",
    "models.common": "yolov5_b200.models.common",
    "models.yolo": "yolov5_b200.models.yolo",
    "models.experimental": "yolov5_b200.models.experimental",
    "utils": "yolov5_b200.utils",
    "utils.general": "yolov5_b200.utils.general",
    "utils.loss": "yolov5_b200.utils.loss",
    "utils.metrics": "yolov5_b200.utils.metrics",
    "utils.torch_utils": "yolov5_b200.utils.torch_utils",
    "utils.augmentations": "yolov5_b200.utils.augmentations",
    "utils.segment": "yolov5_b200.utils.segment",
    "utils.segment.general": "yolov5_b200.utils.segment.general",
    "utils.segment.loss": "yolov5_b200.utils.segment.loss",
    "utils.segment.metrics": "yolov5_b200.utils.segment.metrics",
}


def install(force: bool = False) -> bool:
    """Register the aliases; returns True when they are (already) in place."""
    owned = [n for n in ALIASES if n in sys.modules and not getattr(sys.modules[n], "__name__", "").startswith("yolov5_b200")]
    if owned and not force:
        return False
    for alias, real in ALIASES.items():
        sys.modules[alias] = importlib.import_module(real)
    return True


def uninstall() -> None:
    for alias in ALIASES:
        m = sys.modules.get(alias)
        if m is not None and getattr(m, "__name__", "").startswith("yolov5_b200"):
            del sys.modules[alias]
