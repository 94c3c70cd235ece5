"""Oracle for models built from GhostConv / GhostBottleneck / C3Ghost (reference models/common.py GhostConv, GhostBottleneck,
C3Ghost; models/hub/yolov5s-ghost.yaml).

  GhostConv(c1, c2, k, s, act)   y = Conv(c1, c2 // 2, k, s, act)(x);  cat(y, Conv(c2 // 2, c2 // 2, 5, 1, groups=c2 // 2, act)(y))
  GhostBottleneck(c, c)          GhostConv(c, c // 2) -> GhostConv(c // 2, c, act=False), + x
  C3Ghost(c1, c2, n)             C3 with m = n GhostBottlenecks; it adds the identity whatever `shortcut` says

Every other layer is oracle/model_ref.py's own function.  model_ref parses only Conv / C3 / SPPF / Upsample / Concat / Detect, so
the model dict is parsed with GhostConv read as Conv and C3Ghost as C3 (the same channel, stride and repeat rules); the ghost rows
then run here.  The depthwise conv is F.conv2d with groups = channels.  Runs in the dtype and on the device of its inputs."""
from __future__ import annotations

import copy
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import model_ref


def _as_plain(cfg: dict) -> tuple[dict, dict]:
    """(cfg with GhostConv rows read as Conv and C3Ghost rows as C3, {row index: original module name})"""
    c = copy.deepcopy(cfg)
    rows = c["backbone"] + c["head"]
    ghost = {i: r[2] for i, r in enumerate(rows) if r[2] in ("GhostConv", "C3Ghost")}
    for i, kind in ghost.items():
        rows[i][2] = "Conv" if kind == "GhostConv" else "C3"
    return c, ghost


def dw_block(sd, p, x, fused=False, act=True):
    """Conv(c, c, 5, 1, None, c): depthwise 5x5 conv -> BN -> SiLU, as model_ref.conv_block with groups = channels."""
    w = sd[f"{p}.conv.weight"]
    c = w.shape[0]
    if f"{p}.bn.weight" in sd:
        g, b, m, v = (sd[f"{p}.bn.{q}"] for q in ("weight", "bias", "running_mean", "running_var"))
        if fused:
            w2, b2 = model_ref.fold_bn(w, g, b, m, v)
            y = F.conv2d(x, w2, b2, padding=2, groups=c)
        else:
            y = F.conv2d(x, w, None, padding=2, groups=c)
            if model_ref._BN_BATCH_STATS:
                y = F.batch_norm(y, None, None, g, b, training=True, eps=model_ref.BN_EPS)
            else:
                y = F.batch_norm(y, m, v, g, b, training=False, eps=model_ref.BN_EPS)
    else:
        y = F.conv2d(x, w, sd[f"{p}.conv.bias"], padding=2, groups=c)
    return F.silu(y) if act else y


def ghost_conv(sd, p, x, k=1, s=1, fused=False, act=True):
    y = model_ref.conv_block(sd, f"{p}.cv1", x, k, s, None, fused, act)
    return torch.cat((y, dw_block(sd, f"{p}.cv2", y, fused, act)), 1)


def ghost_bottleneck(sd, p, x, fused=False):
    return ghost_conv(sd, f"{p}.conv.2", ghost_conv(sd, f"{p}.conv.0", x, fused=fused), fused=fused, act=False) + x


def c3ghost(sd, p, x, n, fused=False):
    a = model_ref.conv_block(sd, f"{p}.cv1", x, fused=fused)
    for j in range(n):
        a = ghost_bottleneck(sd, f"{p}.m.{j}", a, fused)
    b = model_ref.conv_block(sd, f"{p}.cv2", x, fused=fused)
    return model_ref.conv_block(sd, f"{p}.cv3", torch.cat((a, b), 1), fused=fused)


def forward(cfg: dict, sd: dict, x: torch.Tensor, training: bool = False, fused: bool = False, ch: int = 3, bn_batch_stats: bool = False):
    """model_ref.forward for a Detect model dict that may hold GhostConv / C3Ghost rows; same outputs."""
    plain, ghost = _as_plain(cfg)
    layers, save = model_ref.parse_layers(plain, ch)
    strides = model_ref.model_strides(plain)
    prev, model_ref._BN_BATCH_STATS = model_ref._BN_BATCH_STATS, bool(bn_batch_stats)
    try:
        ys = []
        for L in layers:
            f, i, kind = L["f"], L["i"], L["kind"]
            if f != -1:
                x = ys[f] if isinstance(f, int) else [x if j == -1 else ys[j] for j in f]
            p, a = f"model.{i}", L.get("args", [])
            if ghost.get(i) == "GhostConv":
                x = ghost_conv(sd, p, x, a[0] if a else 1, a[1] if len(a) > 1 else 1, fused)
            elif ghost.get(i) == "C3Ghost":
                x = c3ghost(sd, p, x, L["n"], fused)
            elif kind == "Conv":
                x = model_ref.conv_block(sd, p, x, a[0] if a else 1, a[1] if len(a) > 1 else 1, a[2] if len(a) > 2 else None, fused)
            elif kind == "C3":
                x = model_ref.c3(sd, p, x, L["n"], a[0] if a else True, fused)
            elif kind == "SPPF":
                x = model_ref.sppf(sd, p, x, a[0] if a else 5, fused)
            elif kind == "nn.Upsample":
                x = F.interpolate(x, scale_factor=L["scale"], mode="nearest")
            elif kind == "Concat":
                x = torch.cat(x, 1)
            elif kind == "Detect":
                x = model_ref.detect(sd, p, list(x), L["nc"], 0, strides, training)
            else:
                raise NotImplementedError(kind)
            ys.append(x if i in save else None)
        return x
    finally:
        model_ref._BN_BATCH_STATS = prev


def param_shapes(cfg: dict, ch: int = 3) -> dict:
    """state_dict key -> shape of the unfused model, in the reference's key order: model_ref's keys with each GhostConv row's
    cv1 / cv2 (depthwise, (c, 1, 5, 5)) and each C3Ghost's GhostBottlenecks in place of the plain Conv / Bottleneck keys."""
    plain, ghost = _as_plain(cfg)
    layers, _ = model_ref.parse_layers(plain, ch)
    base = model_ref.param_shapes(plain, ch)
    out: dict = {}

    def conv(p, c1, c2, k, groups=1):
        out[f"{p}.conv.weight"] = (c2, c1 // groups, k, k)
        for q in ("weight", "bias", "running_mean", "running_var"):
            out[f"{p}.bn.{q}"] = (c2,)
        out[f"{p}.bn.num_batches_tracked"] = ()

    def gconv(p, c1, c2, k):
        c_ = c2 // 2
        conv(f"{p}.cv1", c1, c_, k)
        conv(f"{p}.cv2", c_, c_, 5, groups=c_)

    for L in layers:
        p = f"model.{L['i']}"
        own = {k: v for k, v in base.items() if k.startswith(p + ".")}
        kind = ghost.get(L["i"])
        if kind == "GhostConv":
            gconv(p, L["c1"], L["c2"], L["args"][0] if L["args"] else 1)
        elif kind == "C3Ghost":
            c_ = int(L["c2"] * 0.5)
            out.update({k: v for k, v in own.items() if not k.startswith(f"{p}.m.")})
            for j in range(L["n"]):
                gconv(f"{p}.m.{j}.conv.0", c_, c_ // 2, 1)
                gconv(f"{p}.m.{j}.conv.2", c_ // 2, c_, 1)
        else:
            out.update(own)
    return out


def synth_state_dict(cfg: dict, seed: int = 0, ch: int = 3, head_bias: str = "init") -> dict:
    """model_ref.synth_state_dict for the keys model_ref also has (same values), plus seeded Ghost parameters drawn by the same
    rules: conv W ~ U(-a, a), a = 1/sqrt(fan_in) (fan_in = 25 for a depthwise filter); BN gamma ~ U(.5, 1.5), beta ~ N(0, .1),
    mean ~ N(0, .1), var ~ U(.5, 1.5)."""
    plain, _ = _as_plain(cfg)
    sd = model_ref.synth_state_dict(plain, seed, ch, head_bias)
    rs = np.random.RandomState(seed + 5555)
    out = {}
    for k, shp in param_shapes(cfg, ch).items():
        if k in sd and tuple(sd[k].shape) == tuple(shp):
            out[k] = sd[k]
        elif k.endswith("num_batches_tracked"):
            out[k] = torch.tensor(0, dtype=torch.int64)
        elif k.endswith("conv.weight"):
            out[k] = torch.from_numpy((rs.uniform(-1, 1, shp) / math.sqrt(int(np.prod(shp[1:])))).astype(np.float32))
        elif k.endswith("bn.weight") or k.endswith("running_var"):
            out[k] = torch.from_numpy(rs.uniform(0.5, 1.5, shp).astype(np.float32))
        else:  # bn.bias, running_mean
            out[k] = torch.from_numpy((rs.randn(*shp) * 0.1).astype(np.float32))
    return out
