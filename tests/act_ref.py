"""The oracle (oracle/model_ref.py, oracle/cls_ref.py) evaluated with a Conv activation other than SiLU.

Both oracle modules apply the Conv activation as `F.silu(...)` through their module-level `F` (torch.nn.functional).
`conv_activation(act)` swaps that name, for the duration of a `with` block, for a namespace whose `silu` is `act` and whose every
other attribute is torch.nn.functional's, so the oracle's own expressions run unchanged with the activation the reference's
Conv.default_act would hold (models/yolo.py:383-388)."""
from __future__ import annotations

import contextlib

import torch
import torch.nn.functional as F

from oracle import cls_ref, model_ref


def activation_of(cfg: dict):
    """The Conv activation of a model dict: its `activation:` expression evaluated as the reference does, else SiLU."""
    expr = cfg.get("activation")
    return eval(expr, {"nn": torch.nn, "torch": torch}) if expr else F.silu


class _Functional:
    def __init__(self, act):
        self.silu = act

    def __getattr__(self, name):
        return getattr(F, name)


@contextlib.contextmanager
def conv_activation(act):
    saved = model_ref.F, cls_ref.F
    model_ref.F = cls_ref.F = _Functional(act)
    try:
        yield
    finally:
        model_ref.F, cls_ref.F = saved


def forward(cfg: dict, sd: dict, x: torch.Tensor, **kw):
    """model_ref.forward with the model dict's activation."""
    with conv_activation(activation_of(cfg)):
        return model_ref.forward(cfg, sd, x, **kw)


def cls_forward(cfg: dict, sd: dict, x: torch.Tensor, **kw):
    """cls_ref.forward with the model dict's activation."""
    with conv_activation(activation_of(cfg)):
        return cls_ref.forward(cfg, sd, x, **kw)
