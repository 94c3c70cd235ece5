"""Model assembly with the reference's API surface (reference models/yolo.py:71-150,160-195,215-261,314-372,375-458):
``DetectionModel(cfg, ch, nc, anchors)``, ``.forward(x)``, ``.fuse()``, attributes ``yaml names stride model save nc
inplace``, ``Detect`` / ``Segment`` with ``nc no nl na anchors m stride``, ``ClassificationModel(cfg, model, nc, cutoff)``,
and identical ``state_dict`` keys.

Differences that follow from being an engine rather than a torch.nn graph:
  * strides are derived from the layer table instead of a 256x256 probe forward (models/yolo.py:250-256);
  * ``forward`` accepts CUDA tensors only and runs a cached engine Program per (batch, H, W, dtype); in training mode
    (``model.train()``) it runs yolov5_b200.train_ops.forward_train instead (batch-statistics BN, autograd);
  * eval forward returns ``(z, [raw_i])`` / Segment ``(z, proto, [raw_i])`` exactly like models/yolo.py:115,150.
"""
from __future__ import annotations

import math
from copy import deepcopy
from pathlib import Path

import torch
from torch import nn

from ..cfg import model_cfg
from .common import (C3, C3TR, SPP, SPPF, Bottleneck, C3Ghost, Classify, Concat, Conv, GhostBottleneck, GhostConv, Proto,  # noqa: F401
                     _cached_program, _drop_engine_cache, _lib_on, _param_version)


def make_divisible(x, divisor):
    return math.ceil(x / divisor) * divisor


class Detect(nn.Module):
    stride = None
    dynamic = False
    export = False

    def __init__(self, nc=80, anchors=(), ch=(), inplace=True):
        super().__init__()
        self.nc = nc
        self.no = nc + 5
        self.nl = len(anchors)
        self.na = len(anchors[0]) // 2
        self.grid = [torch.empty(0) for _ in range(self.nl)]
        self.anchor_grid = [torch.empty(0) for _ in range(self.nl)]
        self.register_buffer("anchors", torch.tensor(anchors).float().view(self.nl, -1, 2))
        self.m = nn.ModuleList(nn.Conv2d(x, self.no * self.na, 1) for x in ch)
        self.inplace = inplace

    def forward(self, x):
        raise RuntimeError("y5b200: Detect runs as the epilogue of the head GEMM inside DetectionModel.forward")


class Segment(Detect):
    def __init__(self, nc=80, anchors=(), nm=32, npr=256, ch=(), inplace=True):
        super().__init__(nc, anchors, ch, inplace)
        self.nm = nm
        self.npr = npr
        self.no = 5 + nc + self.nm
        self.m = nn.ModuleList(nn.Conv2d(x, self.no * self.na, 1) for x in ch)
        self.proto = Proto(ch[0], self.npr, self.nm)


_MODULES = {"Conv": Conv, "C3": C3, "C3TR": C3TR, "SPP": SPP, "SPPF": SPPF, "Bottleneck": Bottleneck, "Concat": Concat,
            "nn.Upsample": nn.Upsample, "nn.MaxPool2d": nn.MaxPool2d, "nn.ZeroPad2d": nn.ZeroPad2d, "Detect": Detect, "Segment": Segment,
            "GhostConv": GhostConv, "GhostBottleneck": GhostBottleneck, "C3Ghost": C3Ghost}


def parse_model(d, ch):
    """Model dict -> (nn.Sequential, save list); same scaling rules as reference models/yolo.py:375-458."""
    anchors, nc, gd, gw = d["anchors"], d["nc"], d["depth_multiple"], d["width_multiple"]
    ch_mul = d.get("channel_multiple") or 8
    act = d.get("activation")
    if act:  # e.g. "nn.LeakyReLU(0.1)" (models/hub/yolov5s-LeakyReLU.yaml): every Conv built from here on uses it
        Conv.default_act = eval(act, {"nn": nn, "torch": torch})
    na = (len(anchors[0]) // 2) if isinstance(anchors, list) else anchors
    no = na * (nc + 5)
    layers, save, c2 = [], [], ch[-1]
    names = {"nc": nc, "anchors": anchors, "None": None, "False": False, "True": True}
    for i, (f, n, m, args) in enumerate(d["backbone"] + d["head"]):
        if isinstance(m, str):
            if m not in _MODULES:
                raise NotImplementedError(f"y5b200: module '{m}' is outside the engine's hot path (models n/s/m/l/x[-seg], n6-x6, "
                                          "yolov3[-spp|-tiny], yolov5s-ghost)")
            m = _MODULES[m]
        args = [names.get(a, a) if isinstance(a, str) else a for a in args]
        n = n_ = max(round(n * gd), 1) if n > 1 else n
        if m in (Conv, Bottleneck, SPP, SPPF, C3, C3TR, GhostConv, GhostBottleneck, C3Ghost):
            c1, c2 = ch[f], args[0]
            if c2 != no:
                c2 = make_divisible(c2 * gw, ch_mul)
            args = [c1, c2, *args[1:]]
            if m in (C3, C3TR, C3Ghost):
                args.insert(2, n)
                n = 1
        elif m is Concat:
            c2 = sum(ch[x] for x in f)
        elif m in (Detect, Segment):
            args.append([ch[x] for x in f])
            if isinstance(args[1], int):
                args[1] = [list(range(args[1] * 2))] * len(f)
            if m is Segment:
                args[3] = make_divisible(args[3] * gw, ch_mul)
        else:
            c2 = ch[f]
        m_ = nn.Sequential(*(m(*args) for _ in range(n))) if n > 1 else m(*args)
        m_.i, m_.f, m_.type = i, f, m.__name__
        m_.np = sum(x.numel() for x in m_.parameters())
        save.extend(x % i for x in ([f] if isinstance(f, int) else f) if x != -1)
        layers.append(m_)
        if i == 0:
            ch = []
        ch.append(c2)
    return nn.Sequential(*layers), sorted(save)


def initialize_weights(model):
    """BatchNorm eps / momentum and in-place activations as ultralytics.initialize_weights sets them
    (called at reference models/yolo.py:259)."""
    for m in model.modules():
        if type(m) is nn.BatchNorm2d:
            m.eps = 1e-3
            m.momentum = 0.03
        elif type(m) in (nn.SiLU, nn.ReLU, nn.LeakyReLU, nn.Hardswish, nn.ReLU6):
            m.inplace = True


def _layer_strides(model: nn.Sequential) -> list[float]:
    red = []
    for m in model:
        f = m.f
        if isinstance(m, Detect):
            return [float(red[j]) for j in f]
        r = red[f if isinstance(f, int) else f[0]] if red else 1
        if isinstance(m, Conv):
            r = r * m.conv.stride[0]
        elif isinstance(m, GhostConv):  # its stride sits in cv1 (yolov5s-ghost downsamples with GhostConv(c, 3, 2))
            r = r * m.cv1.conv.stride[0]
        elif isinstance(m, nn.Upsample):
            r = r / float(m.scale_factor)
        elif isinstance(m, nn.MaxPool2d):
            s = m.stride if m.stride is not None else m.kernel_size
            r = r * (s if isinstance(s, int) else s[0])
        red.append(r)
    return []


def scale_img(img, ratio=1.0, same_shape=False, gs=32):
    """(B,C,H,W) image batch resized by `ratio` (bilinear) and padded right/bottom with the ImageNet grey 0.447 up to a
    multiple of `gs` -- ultralytics.utils.torch_utils.scale_img as used by the TTA path (reference models/yolo.py:276)."""
    if ratio == 1.0:
        return img
    h, w = img.shape[2:]
    s = (int(h * ratio), int(w * ratio))
    img = torch.nn.functional.interpolate(img, size=s, mode="bilinear", align_corners=False)
    if not same_shape:
        h, w = (math.ceil(x * ratio / gs) * gs for x in (h, w))
    return torch.nn.functional.pad(img, [0, w - s[1], 0, h - s[0]], value=0.447)


class BaseModel(nn.Module):
    def forward(self, x, profile=False, visualize=False):
        return self._forward_once(x, profile, visualize)

    def _program(self, x):
        from ..engine import Program

        key = (tuple(x.shape), x.dtype, x.device.index, _param_version(self))
        b, c, h, w = x.shape

        def build():
            dt = x.dtype if x.dtype in (torch.float16, torch.bfloat16) else next(self.parameters()).dtype
            return Program(self, b, h, w, dt, x.device)

        return _cached_program(self, key, build)

    def _forward_once(self, x, profile=False, visualize=False):
        if not (isinstance(x, torch.Tensor) and x.is_cuda):
            raise RuntimeError("y5b200: the engine executes on CUDA tensors only (no CPU / PyTorch fallback); "
                               "move the model and the input to an H100")
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"y5b200: expected a (B,3,H,W) image batch, got {tuple(x.shape)}")
        head = self.model[-1]
        gs = int(max(self.stride)) if getattr(self, "stride", None) is not None else 32
        if x.shape[2] % gs or x.shape[3] % gs:
            raise ValueError(f"y5b200: image size {tuple(x.shape[2:])} must be a multiple of the max stride {gs}")
        if self.training:  # list of raw (B,na,ny,nx,no) maps with an autograd graph, as models/yolo.py:98 returns
            from ..train_ops import forward_train

            with _lib_on(x.device):
                return forward_train(self, x)
        with _lib_on(x.device):
            prog = self._program(x)
            if isinstance(head, Classify):  # (B, nc) logits, as models/yolo.py:160-170 returns for a ClassificationModel
                return prog.run_classify(x)
            z, raws, proto = prog.run_model(x)
        if isinstance(head, Segment):
            return (z, proto) if head.export else (z, proto, raws)
        return (z,) if head.export else (z, raws)

    def fuse(self):
        """Fold BatchNorm into the conv weights in place, as reference models/yolo.py:186-195 does (the engine folds
        on the fly either way; this keeps `.fuse()`-d checkpoints and state_dicts interchangeable)."""
        from ..utils.torch_utils import fuse_conv_and_bn

        for m in self.model.modules():
            if isinstance(m, Conv) and hasattr(m, "bn"):
                m.conv = fuse_conv_and_bn(m.conv, m.bn)
                delattr(m, "bn")
        _drop_engine_cache(self)
        return self

    def info(self, verbose=False, img_size=640):
        n_p = sum(p.numel() for p in self.parameters())
        return f"{type(self).__name__}: {len(list(self.modules()))} modules, {n_p} parameters"

    def _apply(self, fn):
        self = super()._apply(fn)
        m = self.model[-1]
        if isinstance(m, Detect) and m.stride is not None:
            m.stride = fn(m.stride)
        _drop_engine_cache(self)
        return self

    def load_state_dict(self, *a, **k):
        _drop_engine_cache(self)
        return super().load_state_dict(*a, **k)

    def __getstate__(self):
        d = self.__dict__.copy()
        d.pop("_y5_programs", None)
        d.pop("_y5_tensors", None)
        d.pop("_y5_pack_plans", None)  # persistent packed-weight buffers of the training path (train_ops.PackPlan)
        return d


class DetectionModel(BaseModel):
    def __init__(self, cfg="yolov5s.yaml", ch=3, nc=None, anchors=None):
        super().__init__()
        if isinstance(cfg, dict):
            self.yaml = cfg
        else:
            self.yaml_file = Path(cfg).name
            if Path(cfg).is_file():
                import yaml

                with open(cfg, encoding="ascii", errors="ignore") as f:
                    self.yaml = yaml.safe_load(f)
            else:
                self.yaml = model_cfg(cfg)  # built-in table for yolov5{n,s,m,l,x}[-seg]
        ch = self.yaml["ch"] = self.yaml.get("ch", ch)
        if nc and nc != self.yaml["nc"]:
            self.yaml["nc"] = nc
        if anchors:
            self.yaml["anchors"] = round(anchors)
        self.model, self.save = parse_model(deepcopy(self.yaml), ch=[ch])
        self.names = [str(i) for i in range(self.yaml["nc"])]
        self.inplace = self.yaml.get("inplace", True)
        m = self.model[-1]
        if isinstance(m, Detect):
            m.inplace = self.inplace
            m.stride = torch.tensor(_layer_strides(self.model))
            if (m.anchors.prod(-1).mean(-1).view(-1)[-1] - m.anchors.prod(-1).mean(-1).view(-1)[0]).sign() != (
                m.stride[-1] - m.stride[0]
            ).sign():  # check_anchor_order (utils/autoanchor.py): anchors must grow with stride
                m.anchors[:] = m.anchors.flip(0)
            m.anchors /= m.stride.view(-1, 1, 1)
            self.stride = m.stride
            self._initialize_biases()
        initialize_weights(self)

    def forward(self, x, augment=False, profile=False, visualize=False):
        """Same call signature as reference models/yolo.py:263: single-scale inference / training forward, or test-time
        augmentation over three scales and a left-right flip (`augment=True`)."""
        if augment:
            return self._forward_augment(x)
        return self._forward_once(x, profile, visualize)

    def _forward_augment(self, x):
        """TTA (reference models/yolo.py:269-283): the engine runs each scaled / flipped copy (one cached Program per
        shape); de-scaling, de-flipping and the tail clipping are host-side tensor edits on the decoded predictions."""
        if self.training:
            raise RuntimeError("y5b200: augment=True is an inference-time option (model.eval())")
        img_size = x.shape[-2:]
        gs = int(self.stride.max())
        if x.dtype == torch.uint8:
            x = x.to(next(self.parameters()).dtype) / 255
        ys = []
        for scale, flip in zip((1, 0.83, 0.67), (None, 3, None)):
            xi = scale_img(x.flip(flip) if flip else x, scale, gs=gs)
            yi = self._forward_once(xi)[0]
            yi[..., :4] /= scale
            if flip == 3:
                yi[..., 0] = img_size[1] - yi[..., 0]
            ys.append(yi)
        # drop the largest-stride rows of the full-scale copy and the smallest-stride rows of the smallest copy
        nl = self.model[-1].nl
        g = sum(4 ** k for k in range(nl))
        ys[0] = ys[0][:, : ys[0].shape[1] - ys[0].shape[1] // g]
        ys[-1] = ys[-1][:, (ys[-1].shape[1] // g) * 4 ** (nl - 1) :]
        return torch.cat(ys, 1), None

    def _initialize_biases(self, cf=None):
        """Detect bias prior (reference models/yolo.py:314-327)."""
        m = self.model[-1]
        for mi, s in zip(m.m, m.stride):
            b = mi.bias.view(m.na, -1)
            b.data[:, 4] += math.log(8 / (640 / s) ** 2)
            b.data[:, 5 : 5 + m.nc] += math.log(0.6 / (m.nc - 0.99999)) if cf is None else torch.log(cf / cf.sum())
            mi.bias = torch.nn.Parameter(b.view(-1), requires_grad=True)


Model = DetectionModel


class SegmentationModel(DetectionModel):
    def __init__(self, cfg="yolov5s-seg.yaml", ch=3, nc=None, anchors=None):
        super().__init__(cfg, ch, nc, anchors)


class ClassificationModel(BaseModel):
    """Reference models/yolo.py:343-372: a DetectionModel's backbone cut at `cutoff` with a Classify head in place of its last
    layer.  ``forward(x)`` returns the (B, nc) logits -- in eval through a cached engine Program, in training mode through
    yolov5_b200.train_ops (batch-statistics BN, autograd)."""

    def __init__(self, cfg=None, model=None, nc=1000, cutoff=10):
        super().__init__()
        self._from_detection_model(model, nc, cutoff) if model is not None else self._from_yaml(cfg)

    def _from_detection_model(self, model, nc=1000, cutoff=10):
        model.model = model.model[:cutoff]  # backbone
        m = model.model[-1]  # last layer
        ch = m.conv.in_channels if hasattr(m, "conv") else m.cv1.conv.in_channels  # ch into module
        c = Classify(ch, nc)
        c.i, c.f, c.type = m.i, m.f, "models.common.Classify"
        model.model[-1] = c
        _drop_engine_cache(model)
        self.model = model.model
        self.stride = model.stride
        self.save = []
        self.nc = nc

    def _from_yaml(self, cfg):
        self.model = None  # the reference does not build classification models from a *.yaml either

    def _program(self, x):
        """As BaseModel._program, except that an fp32 model called under autocast computes in the autocast dtype:
        classify/train.py validates its fp32 EMA model that way (classify/val.py:110)."""
        from ..engine import Program

        dt = x.dtype if x.dtype in (torch.float16, torch.bfloat16) else next(self.parameters()).dtype
        if dt == torch.float32 and torch.is_autocast_enabled("cuda"):
            dt = torch.get_autocast_dtype("cuda")
        key = (tuple(x.shape), x.dtype, dt, x.device.index, _param_version(self))
        b, _, h, w = x.shape
        return _cached_program(self, key, lambda: Program(self, b, h, w, dt, x.device))
