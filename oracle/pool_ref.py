"""Float64-capable restatement of the YOLOv3 pooling layers and their backward tie rule, written from the documented semantics of
nn.MaxPool2d / nn.ZeroPad2d (no reference code).

  maxpool(x, k, s, pad, zero_pad_hi)    max over k x k windows at stride s.  `pad` cells of -inf on every side (MaxPool2d's
                                        padding), then `zero_pad_hi` cells of 0 right and below (nn.ZeroPad2d((0, z, 0, z)) in
                                        front of the pool).  Returns the maxima and, per output, the flat index (row-major over
                                        the unpadded input) of the cell the gradient goes to, or -1 for a zero-pad cell.
  maxpool_backward(idx, dy, shape)      routes every window's gradient to its chosen cell, summed in float64.
  spp(a, ks) / spp_backward(a, dcat, ks)  SPP's cat(a, mp_k0(a), mp_k1(a), ...) with stride-1 'same' pools, and its gradient.

Tie rule: scanning a window in row-major order, a cell takes the window when its value is larger than the running maximum or NaN,
so the first maximum wins and a NaN takes over from any earlier cell.
"""
from __future__ import annotations

import numpy as np
import torch


def maxpool(x: torch.Tensor, k: int, s: int, pad: int = 0, zero_pad_hi: int = 0) -> tuple[torch.Tensor, torch.Tensor]:
    """x (B,C,H,W) -> (values (B,C,Ho,Wo), indices (B,C,Ho,Wo) int64)."""
    b, c, h, w = x.shape
    hp, wp = h + 2 * pad + zero_pad_hi, w + 2 * pad + zero_pad_hi
    ho, wo = (hp - k) // s + 1, (wp - k) // s + 1
    xs = x.detach().cpu().double().numpy()
    best = np.full((b, c, ho, wo), -np.inf)
    arg = np.full((b, c, ho, wo), -2, dtype=np.int64)  # -2: nothing taken yet
    for dy in range(k):
        for dx in range(k):
            yy = np.arange(ho) * s + dy - pad  # input row of this window cell, per output row
            xx = np.arange(wo) * s + dx - pad
            vy, vx = (yy >= 0) & (yy < h + zero_pad_hi), (xx >= 0) & (xx < w + zero_pad_hi)
            real = (yy[:, None] < h) & (xx[None, :] < w) & vy[:, None] & vx[None, :]
            inside = vy[:, None] & vx[None, :]  # -inf padding cells are never part of the scan
            v = np.zeros((b, c, ho, wo))
            yc, xc = np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)
            v[...] = np.where(real, xs[:, :, yc][:, :, :, xc], 0.0)
            take = inside & ((arg == -2) | (v > best) | np.isnan(v))
            best = np.where(take, v, best)
            flat = np.where(real, yc[:, None] * w + xc[None, :], -1)
            arg = np.where(take, np.broadcast_to(flat, arg.shape), arg)
    return torch.from_numpy(best), torch.from_numpy(arg)


def maxpool_backward(idx: torch.Tensor, dy: torch.Tensor, shape) -> torch.Tensor:
    """dx (float64) of a maxpool whose forward chose `idx`: each window's dy added at its index (-1: dropped)."""
    b, c, h, w = shape
    dx = torch.zeros(b, c, h * w + 1, dtype=torch.float64)
    i = idx.reshape(b, c, -1).clone()
    i[i < 0] = h * w
    dx.scatter_add_(2, i, dy.detach().cpu().double().reshape(b, c, -1))
    return dx[:, :, : h * w].reshape(b, c, h, w)


def spp(a: torch.Tensor, ks=(5, 9, 13)) -> torch.Tensor:
    return torch.cat([a.detach().cpu().double()] + [maxpool(a, k, 1, k // 2)[0] for k in ks], 1)


def spp_backward(a: torch.Tensor, dcat: torch.Tensor, ks=(5, 9, 13)) -> torch.Tensor:
    c = a.shape[1]
    dcat = dcat.detach().cpu().double()
    da = dcat[:, :c].clone()
    for j, k in enumerate(ks):
        da += maxpool_backward(maxpool(a, k, 1, k // 2)[1], dcat[:, (j + 1) * c : (j + 2) * c], a.shape)
    return da
