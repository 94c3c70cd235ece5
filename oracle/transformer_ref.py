"""Oracle for models with a C3TR (reference models/common.py:115-161, 261-270; models/hub/yolov5s-transformer.yaml).

The transformer layers are restated with explicit matmul / softmax / matmul expressions (no nn.MultiheadAttention); every other
layer is oracle/model_ref.py's own function.  model_ref parses only Conv / C3 / SPPF / Upsample / Concat / Detect, so the model
dict is parsed with each C3TR read as a C3 (same channel and repeat rules, models/yolo.py:427) and the C3TR rows are then run
with `c3tr` here.  Runs in the dtype and on the device of its inputs (float64 on the CPU for the fixtures)."""
from __future__ import annotations

import copy
import math

import numpy as np
import torch

from oracle import model_ref

HEADS = 4  # C3TR builds TransformerBlock(c_, c_, 4, n)


def _as_c3(cfg: dict) -> tuple[dict, set]:
    """(cfg with every C3TR row read as C3, indices of those rows)"""
    c = copy.deepcopy(cfg)
    rows = c["backbone"] + c["head"]
    tr = {i for i, r in enumerate(rows) if r[2] == "C3TR"}
    for i in tr:
        rows[i][2] = "C3"
    return c, tr


def transformer_block(sd: dict, p: str, x: torch.Tensor, n: int, heads: int = HEADS) -> torch.Tensor:
    """TransformerBlock(c, c, heads, n).forward: tokens (B, L = H*W, c) in row-major pixel order."""
    b, c, h, w = x.shape
    dh = c // heads
    t = x.flatten(2).transpose(1, 2)
    t = t + t @ sd[f"{p}.linear.weight"].T + sd[f"{p}.linear.bias"]
    for j in range(n):
        q = f"{p}.tr.{j}"
        wi, bi = sd[f"{q}.ma.in_proj_weight"], sd[f"{q}.ma.in_proj_bias"]
        qs, ks, vs = (t @ sd[f"{q}.{s}.weight"].T @ wi[i * c : (i + 1) * c].T + bi[i * c : (i + 1) * c] for i, s in enumerate("qkv"))
        qs, ks, vs = (u.reshape(b, h * w, heads, dh).transpose(1, 2) for u in (qs, ks, vs))
        a = torch.softmax(qs @ ks.transpose(-1, -2) / math.sqrt(dh), -1) @ vs
        a = a.transpose(1, 2).reshape(b, h * w, c)
        t = a @ sd[f"{q}.ma.out_proj.weight"].T + sd[f"{q}.ma.out_proj.bias"] + t
        t = t @ sd[f"{q}.fc1.weight"].T @ sd[f"{q}.fc2.weight"].T + t
    return t.transpose(1, 2).reshape(b, c, h, w)


def c3tr(sd: dict, p: str, x: torch.Tensor, n: int, fused: bool) -> torch.Tensor:
    a = transformer_block(sd, f"{p}.m", model_ref.conv_block(sd, f"{p}.cv1", x, fused=fused), n)
    b = model_ref.conv_block(sd, f"{p}.cv2", x, fused=fused)
    return model_ref.conv_block(sd, f"{p}.cv3", torch.cat((a, b), 1), fused=fused)


def forward(cfg: dict, sd: dict, x: torch.Tensor, training: bool = False, fused: bool = False, ch: int = 3, bn_batch_stats: bool = False):
    """model_ref.forward for a Detect model dict that may hold C3TR rows; same outputs."""
    c3cfg, tr = _as_c3(cfg)
    layers, save = model_ref.parse_layers(c3cfg, ch)
    strides = model_ref.model_strides(c3cfg)
    prev, model_ref._BN_BATCH_STATS = model_ref._BN_BATCH_STATS, bool(bn_batch_stats)
    try:
        ys = []
        for L in layers:
            f, i, kind = L["f"], L["i"], L["kind"]
            if f != -1:
                x = ys[f] if isinstance(f, int) else [x if j == -1 else ys[j] for j in f]
            p = f"model.{i}"
            if i in tr:
                x = c3tr(sd, p, x, L["n"], fused)
            elif kind == "Conv":
                a = L["args"]
                x = model_ref.conv_block(sd, p, x, a[0] if a else 1, a[1] if len(a) > 1 else 1, a[2] if len(a) > 2 else None, fused)
            elif kind == "C3":
                x = model_ref.c3(sd, p, x, L["n"], L["args"][0] if L["args"] else True, fused)
            elif kind == "SPPF":
                x = model_ref.sppf(sd, p, x, L["args"][0] if L["args"] else 5, fused)
            elif kind == "nn.Upsample":
                x = torch.nn.functional.interpolate(x, scale_factor=L["scale"], mode="nearest")
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
    """state_dict key -> shape of the unfused model: model_ref's keys with each C3TR's Bottlenecks replaced by its
    TransformerBlock (linear, then per layer q, k, v, ma.in_proj_*, ma.out_proj.*, fc1, fc2), in the reference's order."""
    c3cfg, tr = _as_c3(cfg)
    layers, _ = model_ref.parse_layers(c3cfg, ch)
    base = model_ref.param_shapes(c3cfg, ch)
    out = {}
    for i, L in enumerate(layers):
        p = f"model.{i}"
        own = {k: v for k, v in base.items() if k.startswith(p + ".")}
        if i not in tr:
            out.update(own)
            continue
        c = int(L["c2"] * 0.5)
        out.update({k: v for k, v in own.items() if not k.startswith(f"{p}.m.")})
        out[f"{p}.m.linear.weight"], out[f"{p}.m.linear.bias"] = (c, c), (c,)
        for j in range(L["n"]):
            q = f"{p}.m.tr.{j}"
            for s in "qkv":
                out[f"{q}.{s}.weight"] = (c, c)
            out[f"{q}.ma.in_proj_weight"], out[f"{q}.ma.in_proj_bias"] = (3 * c, c), (3 * c,)
            out[f"{q}.ma.out_proj.weight"], out[f"{q}.ma.out_proj.bias"] = (c, c), (c,)
            out[f"{q}.fc1.weight"], out[f"{q}.fc2.weight"] = (c, c), (c, c)
    return out


def synth_state_dict(cfg: dict, seed: int = 0, ch: int = 3, head_bias: str = "init") -> dict:
    """model_ref.synth_state_dict for the layers model_ref knows, plus seeded C3TR parameters: every matrix ~ U(-a, a) with
    a = 1/sqrt(fan_in) (what nn.Linear draws), biases ~ U(-0.1, 0.1) (nn.MultiheadAttention starts its biases at zero; random ones
    exercise the bias paths)."""
    c3cfg, _ = _as_c3(cfg)
    sd = model_ref.synth_state_dict(c3cfg, seed, ch, head_bias)
    shapes = param_shapes(cfg, ch)
    rs = np.random.RandomState(seed + 7777)
    out = {}
    for k, shp in shapes.items():
        if k in sd:
            out[k] = sd[k]
        elif len(shp) == 2:
            out[k] = torch.from_numpy((rs.uniform(-1, 1, shp) / math.sqrt(shp[1])).astype(np.float32))
        else:
            out[k] = torch.from_numpy(rs.uniform(-0.1, 0.1, shp).astype(np.float32))
    return out
