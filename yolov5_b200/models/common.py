"""Layer zoo of the hot path with the reference's class names, constructor signatures, attribute names and
state_dict keys (reference models/common.py:62-92,164-181,230-246,318-340,443-453,1104-1140), so checkpoints and
state_dicts move between the two unchanged.  The modules only *hold* parameters: executing one (``forward``) lowers it
to liby5b200 kernels through yolov5_b200.engine.Program (eval) or yolov5_b200.train_ops (training: batch-statistics
BatchNorm, autograd) -- there is no torch.nn convolution behind them and CPU tensors are rejected.
"""
from __future__ import annotations

import torch
from torch import nn


def autopad(k, p=None, d=1):
    """'same' padding for kernel k (dilation d); reference models/common.py:62-71."""
    if d > 1:
        k = d * (k - 1) + 1 if isinstance(k, int) else [d * (x - 1) + 1 for x in k]
    if p is None:
        p = k // 2 if isinstance(k, int) else [x // 2 for x in k]
    return p


class _EngineLayer(nn.Module):
    """Runs a single layer through a cached single-layer Program (keyed by input shape / dtype / training flag)."""

    def _engine_forward(self, x: torch.Tensor) -> torch.Tensor:
        from ..engine import Program

        if not (isinstance(x, torch.Tensor) and x.is_cuda):
            raise RuntimeError(
                f"y5b200: {type(self).__name__} executes only on CUDA tensors through liby5b200 (no CPU/PyTorch fallback)"
            )
        if self.training:  # batch-statistics BatchNorm + autograd: yolov5_b200/train_ops.py
            from ..train_ops import _run, train_dtype

            dt = train_dtype(self)
            with torch.autocast("cuda", enabled=False):
                return _run(self, x.to(dt), dt)
        key = (tuple(x.shape), x.dtype, x.device.index, _param_version(self))
        b, c, h, w = x.shape
        with _lib_on(x.device):
            return _cached_program(self, key, lambda: Program(self, b, h, w, x.dtype, x.device, in_channels=c)).run_layer(x)

    def forward(self, x):
        return self._engine_forward(x)

    def __getstate__(self):  # programs hold raw pointers: never pickle them (checkpoints pickle whole modules)
        d = self.__dict__.copy()
        d.pop("_y5_programs", None)
        d.pop("_y5_tensors", None)
        d.pop("_y5_pack_plans", None)  # persistent packed-weight buffers of the training path (train_ops.PackPlan)
        return d

    def _apply(self, fn, *a, **k):
        _drop_engine_cache(self)
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        _drop_engine_cache(self)
        return super().load_state_dict(*a, **k)


def _lib_on(device):
    from .. import _lib

    return _lib.on(device)


def _param_version(m: nn.Module) -> int:
    """In-place edits of parameters / buffers (optimizer steps, BN statistics, manual surgery) invalidate the packed weights
    of a cached Program.  The tensor list is gathered once per module (walking ~350 sub-modules per forward cost more than the
    yolov5n forward itself); `_apply` / `load_state_dict` / `fuse` drop it together with the programs."""
    ts = m.__dict__.get("_y5_tensors")
    if ts is None:
        ts = m.__dict__["_y5_tensors"] = list(m.parameters()) + list(m.buffers())
    v = 0
    for t in ts:
        v += t._version
    return v


def _drop_engine_cache(m: nn.Module) -> None:
    m.__dict__.pop("_y5_programs", None)
    m.__dict__.pop("_y5_tensors", None)


PROGRAM_CACHE = 8  # cached Programs per module (least recently used one is dropped)


def _cached_program(m: nn.Module, key, build):
    from collections import OrderedDict

    cache = m.__dict__.get("_y5_programs")
    if cache is None:
        cache = m.__dict__["_y5_programs"] = OrderedDict()
    prog = cache.get(key)
    if prog is None:
        # programs of an older parameter version can never be hit again: drop them first
        for k in [k for k in cache if k[-1] != key[-1]]:
            del cache[k]
        while len(cache) >= PROGRAM_CACHE:
            cache.popitem(last=False)
        prog = cache[key] = build()
    else:
        cache.move_to_end(key)
    return prog


class Conv(_EngineLayer):
    """conv(bias=False) -> BatchNorm2d -> SiLU, executed as one fused kernel."""

    default_act = nn.SiLU()

    def __init__(self, c1, c2, k=1, s=1, p=None, g=1, d=1, act=True):
        super().__init__()
        self.conv = nn.Conv2d(c1, c2, k, s, autopad(k, p, d), groups=g, dilation=d, bias=False)
        self.bn = nn.BatchNorm2d(c2)
        self.act = self.default_act if act is True else act if isinstance(act, nn.Module) else nn.Identity()

    def forward_fuse(self, x):
        return self._engine_forward(x)


class Bottleneck(_EngineLayer):
    def __init__(self, c1, c2, shortcut=True, g=1, e=0.5):
        super().__init__()
        c_ = int(c2 * e)
        self.cv1 = Conv(c1, c_, 1, 1)
        self.cv2 = Conv(c_, c2, 3, 1, g=g)
        self.add = shortcut and c1 == c2


class C3(_EngineLayer):
    def __init__(self, c1, c2, n=1, shortcut=True, g=1, e=0.5):
        super().__init__()
        c_ = int(c2 * e)
        self.cv1 = Conv(c1, c_, 1, 1)
        self.cv2 = Conv(c1, c_, 1, 1)
        self.cv3 = Conv(2 * c_, c2, 1)
        self.m = nn.Sequential(*(Bottleneck(c_, c_, shortcut, g, e=1.0) for _ in range(n)))


class SPPF(_EngineLayer):
    def __init__(self, c1, c2, k=5):
        super().__init__()
        c_ = c1 // 2
        self.cv1 = Conv(c1, c_, 1, 1)
        self.cv2 = Conv(c_ * 4, c2, 1, 1)
        self.m = nn.MaxPool2d(kernel_size=k, stride=1, padding=k // 2)


class Concat(nn.Module):
    """Channel concatenation.  Inside a model it costs nothing (producers write into slices of one buffer); called on
    its own it has no arithmetic to offload and simply concatenates."""

    def __init__(self, dimension=1):
        super().__init__()
        self.d = dimension

    def forward(self, x):
        return torch.cat(x, self.d)


class Proto(_EngineLayer):
    """Segmentation prototype branch: Conv3x3 -> 2x nearest upsample -> Conv3x3 -> Conv1x1."""

    def __init__(self, c1, c_=256, c2=32):
        super().__init__()
        self.cv1 = Conv(c1, c_, k=3)
        self.upsample = nn.Upsample(scale_factor=2, mode="nearest")
        self.cv2 = Conv(c_, c_, k=3)
        self.cv3 = Conv(c_, c2)


class Classify(nn.Module):
    """Classification head (reference models/common.py:1120-1140): Conv(c1, 1280) -> global average pool -> Dropout ->
    Linear(1280, c2).  Inside ClassificationModel.forward it runs as conv_gemm + y5_global_avg_pool + conv_gemm (the Linear
    as a 1x1 conv with bias); Dropout is the identity in eval, and p > 0 is refused in training."""

    def __init__(self, c1, c2, k=1, s=1, p=None, g=1, dropout_p=0.0):
        super().__init__()
        c_ = 1280  # efficientnet_b0 size
        self.conv = Conv(c1, c_, k, s, autopad(k, p), g)
        self.pool = nn.AdaptiveAvgPool2d(1)
        self.drop = nn.Dropout(p=dropout_p, inplace=True)
        self.linear = nn.Linear(c_, c2)

    def forward(self, x):
        raise RuntimeError("y5b200: Classify runs inside ClassificationModel.forward (conv, pool and linear as liby5b200 kernels)")
