"""Helpers shared by the -m gpu parity tests: drive liby5b200 through its C ABI on NHWC buffers."""
import ctypes as C

import numpy as np
import torch
import torch.nn.functional as F

from yolov5_b200 import _lib
from yolov5_b200.engine import pack_weight


def conv_case(dev, dtype, B, H, W, cin, cout, k, s, p, act=True, residual=False, in_extra=0, out_extra=0, seed=0, direct=False,
              block_n=0, a_mode=0, mt2=False, cluster=1, cg2=False, direct_store=False, narrow_patch=False, wide_patch=False,
              staged=False, expect=None):
    """Runs y5_conv_bn_silu_fwd (or the direct cross-check kernel) on seeded data; returns (got NCHW fp32, oracle fp32).
    `expect` ({y5_plan_info field: value}, "wide": bool for the wide patch) asserts the plan the case claims to run.
    `in_extra` / `out_extra` put the views inside wider buffers (channel offset 8, pitch + extra) to exercise slices.
    Stores: the library's default (direct from the registers) unless `staged` asks for the shared-memory staged epilogue;
    `direct_store` forces the direct stores."""
    lib = _lib.lib()
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(B, cin, H, W, generator=g) * 2 - 1)
    w = (torch.rand(cout, cin, k, k, generator=g) * 2 - 1) / (cin * k * k) ** 0.5 * 2
    b = torch.rand(cout, generator=g) - 0.5
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    r = torch.rand(B, cout, Ho, Wo, generator=g) - 0.5 if residual else None
    xq, wq = x.to(dtype).float(), w.to(dtype).float()
    y = F.conv2d(xq, wq, b, stride=s, padding=p)
    if act:
        y = F.silu(y)
    if residual:
        y = y + r.to(dtype).float()
    in_off, out_off = (8, 8) if (in_extra or out_extra) else (0, 0)
    ibuf = torch.full((B, H, W, cin + in_extra + in_off), 7.0, dtype=dtype, device=dev)
    ibuf[..., in_off : in_off + cin] = x.permute(0, 2, 3, 1).to(dev, dtype)
    obuf = torch.full((B, Ho, Wo, cout + out_extra + out_off), -3.0, dtype=dtype, device=dev)
    bk, bn = C.c_int32(), C.c_int32()
    _lib.check(lib.y5_conv_pick(cin, cout, B * Ho * Wo, C.byref(bk), C.byref(bn)))
    wp = pack_weight(w, bk.value, dtype).to(dev)
    bias = b.to(dev)
    rbuf = r.permute(0, 2, 3, 1).contiguous().to(dev, dtype) if residual else None
    d = _lib.ConvDesc()
    es = ibuf.element_size()
    d.inp, d.in_pitch = ibuf.data_ptr() + in_off * es, ibuf.shape[3]
    d.batch, d.in_h, d.in_w, d.in_c = B, H, W, cin
    d.weight, d.bias = wp.data_ptr(), bias.data_ptr()
    d.out, d.out_pitch, d.out_c = obuf.data_ptr() + out_off * es, obuf.shape[3], cout
    d.residual, d.res_pitch = (rbuf.data_ptr(), cout) if residual else (None, 0)
    d.ksize, d.stride, d.pad = k, s, p
    d.act, d.dtype, d.block_k, d.block_n = int(act), _lib.dtype_code(dtype), bk.value, block_n
    d.a_mode = a_mode  # 0 auto, 1 TMA-im2col, 2 shifted patches
    d.reserved = (2 if mt2 else 0) | (4 if cg2 else 0) | (16 if direct_store else 0) | (8 if staged else 0) | (32 if narrow_patch else 0) | (128 if wide_patch else 0) | (cluster << 8 if cluster > 1 else 0)  # forced block_n: 256-row tiles / CTA pairs / multicast cluster
    if expect:
        assert_plan(d, expect)
    fn = lib.y5_conv_direct_fwd if direct else lib.y5_conv_bn_silu_fwd
    _lib.check(fn(C.byref(d), C.c_void_p(_lib.stream_ptr(dev))), "conv")
    torch.cuda.synchronize()
    got = obuf[..., out_off : out_off + cout].float().cpu().permute(0, 3, 1, 2)
    untouched = True
    if out_off:
        untouched = bool((obuf[..., :out_off] == -3.0).all() and (obuf[..., out_off + cout :] == -3.0).all())
    return got, y, untouched


def plan_info(desc) -> dict:
    """y5_conv_plan_info of the plan y5_conv_plan_create makes for `desc`, plus "wide" (the wide patch fetch)."""
    lib = _lib.lib()
    plan = C.c_void_p()
    _lib.check(lib.y5_conv_plan_create(C.byref(desc), C.byref(plan)), "conv_plan_create")
    try:
        info = _lib.PlanInfo()
        _lib.check(lib.y5_conv_plan_info(plan, C.byref(info)), "conv_plan_info")
    finally:
        lib.y5_conv_plan_destroy(plan)
    out = info.as_dict()
    out["wide"] = out["patch_pw"] > 0
    return out


def assert_plan(desc, expect: dict):
    info = plan_info(desc)
    assert {k: info[k] for k in expect} == expect, ("plan differs from the path the case names", info)


def rel_err(got, ref):
    return float((got - ref).abs().max() / ref.abs().max().clamp_min(1e-6))
