"""Program planner: turns a DetectionModel (or a single layer) into a fixed sequence of liby5b200 kernel launches.

What the reference does layer by layer through torch.nn (models/yolo.py:160-170 `_forward_once`) becomes, for one
(batch, height, width, dtype):

  * every activation is a channel-slice VIEW of a pre-allocated NHWC buffer; a Concat's inputs are allocated inside
    the Concat's buffer, so torch.cat (models/common.py:246,340,453) disappears;
  * GhostConv's cv1 writes the first half of its output and the depthwise 5x5 conv (y5_dwconv_fwd) reads it and writes the
    second half; a GhostBottleneck's residual rides the depthwise kernel, which writes both halves of the C3's slice in place;
  * C3's cv1 and cv2 (same input, models/common.py:246) run as ONE GEMM with stacked output channels that lands
    directly in the C3's concat buffer; each Bottleneck's residual add (models/common.py:181) is the epilogue of its
    3x3 conv, in place; SPPF's three pools are one kernel; Upsample writes into its Concat slice;
  * Conv = conv + folded BN + SiLU / (Leaky)ReLU in one wgmma implicit-GEMM kernel (weights are folded/packed once, here);
  * the Detect/Segment head levels run the GEMM with the decode epilogue and write fresh output tensors each call;
  * the whole fixed part is captured in a CUDA graph and replayed.

PyTorch is used for device memory and streams only; all arithmetic is in liby5b200.so.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from collections import namedtuple

import torch

from . import _lib
from ._lib import ConvDesc, DetectDesc, WgradDesc
from .models.common import (C3Ghost, TransformerBlock, check_grouped_convs, ghost_bottleneck_convs, ghost_dw_channels, pool_modes, spp_kernel,
                            transformer_spec)

BN_EPS_DEFAULT = 1e-3
# Detect head GEMM (conv_gemm.cu): an anchor's no = 5 + nc + nm outputs are ceil(no / HEAD_N) N tiles of HEAD_N columns
HEAD_N = 128
HEAD_MAX_NO = 8192  # kHeadMaxNo
HEAD_MAX_NC = 4096  # kHeadMaxNc: the NMS / AP class limit


class View:
    """Channel slice [coff, coff+c) of an NHWC buffer (B, H, W, pitch)."""

    __slots__ = ("buf", "coff", "c", "h", "w")

    def __init__(self, buf: torch.Tensor, coff: int, c: int):
        self.buf, self.coff, self.c = buf, coff, c
        self.h, self.w = buf.shape[1], buf.shape[2]

    @property
    def pitch(self) -> int:
        return self.buf.shape[3]

    @property
    def ptr(self) -> int:
        return self.buf.data_ptr() + self.coff * self.buf.element_size()

    def slice(self, coff: int, c: int) -> "View":
        assert 0 <= coff and coff + c <= self.c
        return View(self.buf, self.coff + coff, c)

    def dense_nhwc(self) -> torch.Tensor:
        return self.buf[..., self.coff : self.coff + self.c]


def _pad8(c: int) -> int:
    return (c + 7) // 8 * 8


def fold_conv_bn(conv: torch.nn.Conv2d, bn) -> tuple[torch.Tensor, torch.Tensor]:
    """fp32 (W', b') of conv followed by eval-mode BN; same algebra as utils/torch_utils.py:245-252."""
    w = conv.weight.detach().float()
    if bn is None:
        b = conv.bias.detach().float() if conv.bias is not None else torch.zeros(w.shape[0], device=w.device)
        return w, b
    scale = bn.weight.detach().float() / torch.sqrt(bn.running_var.detach().float() + bn.eps)
    w2 = w * scale.view(-1, 1, 1, 1)
    b0 = conv.bias.detach().float() if conv.bias is not None else torch.zeros_like(scale)
    b2 = bn.bias.detach().float() + (b0 - bn.running_mean.detach().float()) * scale
    return w2, b2


def pack_weight(w: torch.Tensor, block_k: int, dtype: torch.dtype) -> torch.Tensor:
    """OIHW fp32 -> [O][kh][kw][cin_pad] (K-major) in the activation dtype, channel dim zero padded to block_k."""
    o, i, kh, kw = w.shape
    cin_pad = (i + block_k - 1) // block_k * block_k
    out = torch.zeros(o, kh, kw, cin_pad, dtype=dtype, device=w.device)
    out[..., :i] = w.permute(0, 2, 3, 1).to(dtype)
    return out.contiguous()


def stem_weight_s2d(w: torch.Tensor) -> torch.Tensor:
    """(O,3,6,6) stride-2 pad-2 filter -> equivalent (O,16,3,3) stride-1 pad-1 filter over the 2x2 space-to-depth
    input (channel = (dy*2+dx)*3 + c, see y5_stem_s2d); 4 of the 16 channels stay zero."""
    o = w.shape[0]
    out = torch.zeros(o, 16, 3, 3, dtype=w.dtype, device=w.device)
    for dy in range(2):
        for dx in range(2):
            for c in range(3):
                out[:, (dy * 2 + dx) * 3 + c] = w[:, c, dy::2, dx::2]
    return out


def stem_weight_wide(w3: torch.Tensor) -> torch.Tensor:
    """(O,16,3,3) space-to-depth stem filter -> the (O,48,3,1) filter of its wide-pixel form: [o][s*16+c][r][0] = w3[o][c][r][s]."""
    return w3.permute(0, 3, 1, 2).reshape(w3.shape[0], 48, 3, 1)


def stem_weight_narrow(wv: torch.Tensor) -> torch.Tensor:
    """Inverse of stem_weight_wide: (O,48,3,1) -> (O,16,3,3), a view."""
    return wv.view(wv.shape[0], 3, 16, 3).permute(0, 2, 3, 1)


def stem_buffer(b: int, h: int, w: int, dtype: torch.dtype, device) -> torch.Tensor:
    """Zeroed [B][H/2][W/2 + 2][16] buffer for the space-to-depth cells of a (B,3,H,W) image, with one zero cell at each end
    of a row (stem_geom reads them as padding); stem_s2d writes the inner cells only."""
    return torch.zeros(b, h // 2, w // 2 + 2, 16, dtype=dtype, device=device)


def stem_s2d(img: torch.Tensor, out: torch.Tensor) -> None:
    """y5_stem_s2d of a (B,3,H,W) image into `out`, NHWC [B][H/2][row][16]: a stem_buffer (row W/2 + 2, cells from x = 1) or a
    dense one (row W/2)."""
    b, _, h, w = img.shape
    row = out.shape[2]
    img = img.contiguous()
    _lib.check(_lib.lib().y5_stem_s2d(img.data_ptr(), _lib.dtype_code(img.dtype), out.data_ptr(), _lib.dtype_code(out.dtype), b, h, w, row,
                                      (row - w // 2) // 2, C.c_void_p(_lib.stream_ptr(out.device))), "stem_s2d")


IMAGE_C = 16  # channels of the NHWC image buffer of a plain first layer (3 used), a count the conv GEMM takes, as the stem's cells


def image_nhwc(img: torch.Tensor, out: torch.Tensor) -> None:
    """y5_image_nhwc of a (B,3,H,W) image into `out`, a dense NHWC [B][H][W][c] buffer: channels 0..2 the image, the rest zero."""
    b, _, h, w = img.shape
    img = img.contiguous()
    _lib.check(_lib.lib().y5_image_nhwc(img.data_ptr(), _lib.dtype_code(img.dtype), out.data_ptr(), _lib.dtype_code(out.dtype), b, h, w,
                                        out.shape[3], C.c_void_p(_lib.stream_ptr(out.device))), "image_nhwc")


def pad_image_weight(w: torch.Tensor) -> torch.Tensor:
    """(O,3,k,k) filter of a plain first layer -> (O,IMAGE_C,k,k), zero for the image buffer's padding channels."""
    return torch.nn.functional.pad(w, (0, 0, 0, 0, 0, IMAGE_C - w.shape[1]))


_block_k_cache: dict = {}


def block_k(cin: int, cout: int, m_rows: int) -> int:
    """y5_conv_pick's K block for a cin -> cout conv over m_rows output pixels (weights are packed to it)."""
    key = (cin, cout, m_rows)
    v = _block_k_cache.get(key)
    if v is None:  # a pure function of the shape: one library call per distinct layer shape
        bk = C.c_int32()
        _lib.check(_lib.lib().y5_conv_pick(cin, cout, m_rows, C.byref(bk), None), "conv_pick")
        v = _block_k_cache[key] = bk.value
    return v


def is_v6_stem(m) -> bool:
    """The YOLOv5 v6 stem Conv(3, c, 6, 2, 2), which runs as a 3x3 conv over the image's 2x2 space-to-depth cells."""
    c = m.conv
    return c.kernel_size[0] == 6 and c.stride[0] == 2 and c.padding[0] == 2 and c.in_channels == 3


def act_spec(act: torch.nn.Module) -> tuple[int, float]:
    """(Y5_ACT_* code, negative slope) of a Conv's activation module: SiLU, Identity, ReLU (LeakyReLU with slope 0) or LeakyReLU
    with a finite slope.  Any other activation raises NotImplementedError with its name."""
    if isinstance(act, torch.nn.SiLU):
        return _lib.ACT_SILU, 0.0
    if isinstance(act, torch.nn.Identity):
        return _lib.ACT_NONE, 0.0
    if isinstance(act, torch.nn.ReLU):
        return _lib.ACT_LEAKY, 0.0
    if isinstance(act, torch.nn.LeakyReLU) and math.isfinite(act.negative_slope):
        return _lib.ACT_LEAKY, float(act.negative_slope)
    raise NotImplementedError(f"y5b200: activation {act!r} (SiLU, ReLU, LeakyReLU and Identity are built)")


# The input-view fields of y5_conv_desc and y5_wgrad_desc (include/y5b200.h): an NHWC view of in_c channels at element pointer
# `inp`, in_pitch elements per pixel.  The optional ones (0: the plain case) describe the strided views of stem_geom.
ConvInput = namedtuple("ConvInput", "inp in_pitch batch in_h in_w in_c kw pad_w in_x_stride in_y_stride in_n_stride", defaults=(0,) * 5)


def stem_geom(buf: torch.Tensor, wide: bool) -> ConvInput:
    """The stem conv's input over a stem_buffer: a 3x3/s1/p1 conv of the 16-channel cells.  Three horizontally adjacent cells are
    contiguous, so the wide form reads overlapping 48-channel "wide pixels" (x stride 16) from the left padding cell on with a
    3x1 filter and no horizontal padding: 3 taps of K=48 instead of 9 of K=16.  The narrow form is the 3x3x16 view of the cells."""
    b, h2, row, _ = buf.shape
    geom = dict(in_pitch=16, batch=b, in_h=h2, in_w=row - 2, in_x_stride=16, in_y_stride=row * 16, in_n_stride=h2 * row * 16)
    if wide:
        return ConvInput(inp=buf.data_ptr(), in_c=48, kw=1, pad_w=0, **geom)
    return ConvInput(inp=buf.data_ptr() + 16 * buf.element_size(), in_c=16, kw=3, pad_w=1, **geom)


def conv_desc(x: ConvInput, wp: torch.Tensor, bias: torch.Tensor, bk: int, out: int, out_pitch: int, k: int, s: int, p: int,
              act: bool | tuple[int, float], dtype: torch.dtype, residual: int | None = None, res_pitch: int = 0) -> ConvDesc:
    """y5_conv_desc of out = act(conv(x, w) + bias [+ residual]).  wp: w packed [cout][k][kw][cin_pad] for K block bk (pack_weight,
    fold_pack); bias: fp32 [cout]; out / residual: element pointers of NHWC views with their pitches; act: an act_spec pair, or a
    bool for SiLU / none."""
    d = ConvDesc()
    d.inp, d.in_pitch, d.batch, d.in_h, d.in_w, d.in_c, d.kw, d.pad_w, d.in_x_stride, d.in_y_stride, d.in_n_stride = x
    d.weight, d.bias = wp.data_ptr(), bias.data_ptr()
    d.out, d.out_pitch, d.out_c = out, out_pitch, wp.shape[0]
    d.residual, d.res_pitch = residual, res_pitch
    d.ksize, d.stride, d.pad = k, s, p
    d.act, d.act_slope = act if isinstance(act, tuple) else (_lib.ACT_SILU if act else _lib.ACT_NONE, 0.0)
    d.dtype, d.block_k = _lib.dtype_code(dtype), bk
    return d


def wgrad_desc(x: ConvInput, dy: int, dy_pitch: int, dw: torch.Tensor, k: int, s: int, p: int, dtype: torch.dtype) -> WgradDesc:
    """y5_wgrad_desc of the fp32 weight gradient dw ([cout][k][kw][cin], KRSC) of a conv over x, from dy (element pointer, pitch)."""
    d = WgradDesc()
    d.inp, d.in_pitch, d.batch, d.in_h, d.in_w, d.in_c, d.kw, d.pad_w, d.in_x_stride, d.in_y_stride, d.in_n_stride = x
    d.dout, d.dout_pitch, d.out_c = dy, dy_pitch, dw.shape[0]
    d.dweight = dw.data_ptr()
    d.ksize, d.stride, d.pad = k, s, p
    d.dtype = _lib.dtype_code(dtype)
    return d


class _Op:
    """One launch: (function, ctypes args...) bound at plan time; run(stream) issues it."""

    __slots__ = ("fn", "args", "name", "keep")

    def __init__(self, name, fn, args, keep=()):
        self.name, self.fn, self.args, self.keep = name, fn, args, keep

    def run(self, stream: int):
        _lib.check(self.fn(*self.args, C.c_void_p(stream)), self.name)


class Program:
    """Kernel sequence for one module (a whole DetectionModel or a single layer) at a fixed input shape."""

    def __init__(self, module, batch: int, height: int, width: int, dtype: torch.dtype, device, in_channels=None):
        if dtype not in (torch.float16, torch.bfloat16):
            raise TypeError(f"y5b200 engine computes in fp16 or bf16, got {dtype} (call model.half() / .bfloat16())")
        self.lib = _lib.lib()
        self.module = module
        self.B, self.H, self.W = batch, height, width
        self.dtype, self.device = dtype, torch.device(device)
        self.dt_code = _lib.dtype_code(dtype)
        self.ops: list[_Op] = []          # graph-capturable fixed part
        self.head_ops: list = []          # detect levels (fresh outputs per call)
        self._plans: list = []            # (destroy_fn, handle)
        self._keep: list = []             # packed weights / biases / buffers
        self.graph = None
        self.flops = 0                    # 2*MAC of every conv in the program (per batch)
        self.act_bytes = 0                # algorithmic activation bytes: each conv reads its input once, writes its output once
        self.weight_bytes = 0
        self.in_channels = in_channels
        self._build()

    # ------------------------------------------------------------------ allocation helpers
    def new_buf(self, h: int, w: int, c: int) -> torch.Tensor:
        t = torch.zeros(self.B, h, w, _pad8(c), dtype=self.dtype, device=self.device)
        self._keep.append(t)
        return t

    def new_view(self, h: int, w: int, c: int) -> View:
        return View(self.new_buf(h, w, c), 0, c)

    # ------------------------------------------------------------------ op emitters
    def fold_pack(self, parts, m_rows: int):
        """Folded + packed weights of one GEMM from module parameters, one y5_fold_pack launch per part (no ATen arithmetic).
        parts: list of (weight (O,I,kh,kw) tensor, conv bias | None, bn | None); several parts stack along the output channels
        (C3's cv1 | cv2).  Returns (packed [sum O][kh][kw][I_pad] in the activation dtype, fp32 bias [sum O], block_k)."""
        cin, kh, kw = parts[0][0].shape[1:]
        cout = sum(w.shape[0] for w, _, _ in parts)
        bk = block_k(cin, cout, m_rows)
        ipad = (cin + bk - 1) // bk * bk
        wp = torch.empty(cout, kh, kw, ipad, dtype=self.dtype, device=self.device)
        bias = torch.empty(cout, dtype=torch.float32, device=self.device)
        self.fold_pack_into(parts, wp, bias, 0, ipad)
        return wp, bias, bk

    def fold_pack_into(self, parts, wp, bias, row0: int, ipad: int, pad_rows_to: int | None = None):
        st = C.c_void_p(_lib.stream_ptr(self.device))
        es = wp.element_size()
        for w, cb, bn in parts:
            w = w.detach()
            if not w.is_contiguous():
                w = w.contiguous()
            if w.device != self.device:
                raise RuntimeError("y5b200: module parameters and the input must live on the same CUDA device")
            o, i, kh, kw = w.shape
            rows = pad_rows_to or o
            keep = [w]
            if cb is not None:
                cb = cb.detach().to(w.dtype).contiguous()
                keep.append(cb)
            g = b_ = mu = var = None
            bn_code, eps = _lib.Y5_F32, 0.0
            if bn is not None:
                g, b_, mu, var = (t.detach().contiguous() for t in (bn.weight, bn.bias, bn.running_mean, bn.running_var))
                if not (g.dtype == b_.dtype == mu.dtype == var.dtype):
                    g, b_, mu, var = g.float(), b_.float(), mu.float(), var.float()
                bn_code, eps = _lib.dtype_code(g.dtype), float(bn.eps)
                keep += [g, b_, mu, var]
            _lib.check(self.lib.y5_fold_pack(w.data_ptr(), _lib.dtype_code(w.dtype), o, i, kh, kw, cb.data_ptr() if cb is not None else None,
                                             g.data_ptr() if g is not None else None, b_.data_ptr() if b_ is not None else None,
                                             mu.data_ptr() if mu is not None else None, var.data_ptr() if var is not None else None, bn_code, eps,
                                             wp.data_ptr() + row0 * kh * kw * ipad * es, ipad, rows, bias.data_ptr() + row0 * 4, self.dt_code, st),
                       "fold_pack")
            self._keep += keep  # the launch is asynchronous: temporaries must outlive it
            row0 += rows

    def emit_conv(self, d: ConvDesc, name: str, keep):
        """Plan the conv of descriptor d and append its launch; `keep` (its weights and bias) lives as long as the program."""
        self._keep += keep
        d.block_n = int(os.environ.get("Y5_FORCE_BLOCK_N", "0"))  # 0: the library's tile cost model decides (block_n, MT)
        d.a_mode = int(os.environ.get("Y5_FORCE_A_MODE", "0"))
        if d.a_mode == 2 and d.stride != 1:
            d.a_mode = 0
        plan = C.c_void_p()
        _lib.check(self.lib.y5_conv_plan_create(C.byref(d), C.byref(plan)), f"conv_plan_create[{name}]")
        self._plans.append((self.lib.y5_conv_plan_destroy, plan))
        self.ops.append(_Op(name, self.lib.y5_conv_plan_run, (plan,)))

    def conv(self, x: View, out: View, packed, k: int, s: int, p: int, act, residual: View | None = None, name: str = "conv"):
        """Emit one fused conv of view x into view out; packed = (wp, bias, block_k) as fold_pack returns them; act as conv_desc
        takes it."""
        wp, bias, bk = packed
        ho, wo = (x.h + 2 * p - k) // s + 1, (x.w + 2 * p - k) // s + 1
        cout, cin = out.c, x.c
        assert (ho, wo) == (out.h, out.w) and wp.shape == (cout, k, k, -(-cin // bk) * bk), (name, ho, wo, out.h, out.w, wp.shape, cin)
        res = (residual.ptr, residual.pitch) if residual is not None else (None, 0)
        d = conv_desc(ConvInput(x.ptr, x.pitch, self.B, x.h, x.w, cin), wp, bias, bk, out.ptr, out.pitch, k, s, p, act, self.dtype, *res)
        self.emit_conv(d, name, (wp, bias))
        m_rows = self.B * ho * wo
        self.flops += 2 * m_rows * cout * cin * k * k
        self.act_bytes += 2 * (self.B * x.h * x.w * cin + m_rows * cout)
        self.weight_bytes += 2 * cout * cin * k * k

    def conv_module(self, m, x: View, out: View, residual: View | None = None, name="conv"):
        """m: models.common.Conv (conv + bn + act) in its fused or unfused state."""
        k, s, p = m.conv.kernel_size[0], m.conv.stride[0], m.conv.padding[0]
        act = act_spec(m.act)
        if m.conv.groups != 1 or m.conv.dilation[0] != 1:
            raise NotImplementedError("y5b200: grouped / dilated convolutions are outside the YOLOv5 n..x hot path")
        ho, wo = (x.h + 2 * p - k) // s + 1, (x.w + 2 * p - k) // s + 1
        packed = self.fold_pack([(m.conv.weight, m.conv.bias, getattr(m, "bn", None))], self.B * ho * wo)
        self.conv(x, out, packed, k, s, p, act, residual, name)

    def out_hw(self, m, x: View):
        k, s, p = m.conv.kernel_size[0], m.conv.stride[0], m.conv.padding[0]
        return (x.h + 2 * p - k) // s + 1, (x.w + 2 * p - k) // s + 1

    # ------------------------------------------------------------------ module lowering
    def lower_conv(self, m, x, out: View | None, name):
        from .models.common import Conv  # noqa: F401

        k, s, p, cin = m.conv.kernel_size[0], m.conv.stride[0], m.conv.padding[0], m.conv.in_channels
        if isinstance(x, torch.Tensor) and not is_v6_stem(m):  # network input, plain Conv(3, c, k, s): over the NHWC image buffer
            if cin != 3 or m.conv.groups != 1 or m.conv.dilation[0] != 1:
                raise NotImplementedError(f"y5b200: the first layer must be a plain Conv(3, c, k, s) or the v6 stem, got {m.conv!r}")
            self.image_in = torch.zeros(self.B, self.H, self.W, IMAGE_C, dtype=self.dtype, device=self.device)
            x = View(self.image_in, 0, IMAGE_C)
            ho, wo = self.out_hw(m, x)
            out = out or self.new_view(ho, wo, m.conv.out_channels)
            packed = self.fold_pack([(pad_image_weight(m.conv.weight.detach()), m.conv.bias, getattr(m, "bn", None))], self.B * ho * wo)
            self.conv(x, out, packed, k, s, p, act_spec(m.act), None, name)
            return out
        if isinstance(x, torch.Tensor):  # network input (B,3,H,W) NCHW: v6 stem path
            if self.H % 2 or self.W % 2:
                raise ValueError("y5b200: image height and width must be even")
            h2, w2 = self.H // 2, self.W // 2
            self.stem_in = stem_buffer(self.B, self.H, self.W, self.dtype, self.device)
            w, b = fold_conv_bn(m.conv, getattr(m, "bn", None))
            out = out or self.new_view(h2, w2, m.conv.out_channels)
            w3 = stem_weight_s2d(w)  # (O,16,3,3): 3x3/s1/p1 over the 16-channel cells
            act = act_spec(m.act)

            def stem_conv(wide: bool, form: str):
                wv = stem_weight_wide(w3) if wide else w3
                bk = block_k(wv.shape[1], wv.shape[0], self.B * h2 * w2)
                wp = pack_weight(wv, bk, self.dtype)
                d = conv_desc(stem_geom(self.stem_in, wide), wp, b, bk, out.ptr, out.pitch, 3, 1, 1, act, self.dtype)
                self.emit_conv(d, f"{name}(s2d {form})", (wp, b))

            try:
                stem_conv(True, "3x1x48")
            except RuntimeError:  # driver refused the overlapping-stride tensor map: plain 3x3 over the padded buffer's cells
                stem_conv(False, "3x3x16")
            cout = m.conv.out_channels
            self.flops += 2 * self.B * h2 * w2 * cout * 3 * 36
            self.act_bytes += 2 * (self.B * self.H * self.W * 3 + self.B * h2 * w2 * cout)
            self.weight_bytes += 2 * cout * 3 * 36
            return out
        ho, wo = self.out_hw(m, x)
        out = out or self.new_view(ho, wo, m.conv.out_channels)
        self.conv_module(m, x, out, None, name)
        return out

    def lower_c3(self, m, x: View, out: View | None, name):
        c_ = m.cv1.conv.out_channels
        cat = self.new_view(x.h, x.w, 2 * c_)
        act = act_spec(m.cv1.act)
        if act == act_spec(m.cv2.act):
            # cv1 | cv2 stacked along the output channels: one GEMM, result is already the concat layout
            packed = self.fold_pack([(m.cv1.conv.weight, m.cv1.conv.bias, getattr(m.cv1, "bn", None)),
                                     (m.cv2.conv.weight, m.cv2.conv.bias, getattr(m.cv2, "bn", None))], self.B * x.h * x.w)
            self.conv(x, cat, packed, 1, 1, 0, act, None, f"{name}.cv1|cv2")
        else:  # different activations: one GEMM each, into the two halves of the concat
            self.conv_module(m.cv1, x, cat.slice(0, c_), None, f"{name}.cv1")
            self.conv_module(m.cv2, x, cat.slice(c_, c_), None, f"{name}.cv2")
        a = cat.slice(0, c_)
        if isinstance(m.m, TransformerBlock):  # C3TR
            self.lower_transformer(m.m, a, f"{name}.m")
        elif isinstance(m, C3Ghost):
            scratch = None
            for j, bt in enumerate(m.m):
                scratch = self.lower_ghost_bottleneck(bt, a, a, f"{name}.m{j}", scratch)
        else:
            if len(m.m):
                tmp = self.new_view(x.h, x.w, c_)
            for j, bt in enumerate(m.m):
                self.conv_module(bt.cv1, a, tmp, None, f"{name}.m{j}.cv1")
                self.conv_module(bt.cv2, tmp, a, a if bt.add else None, f"{name}.m{j}.cv2")  # in-place residual add
        out = out or self.new_view(x.h, x.w, m.cv3.conv.out_channels)
        self.conv_module(m.cv3, cat, out, None, f"{name}.cv3")
        return out

    def dwconv(self, m, x: View, out: View, residual: View | None = None, x_out: View | None = None, x_res: View | None = None,
               name: str = "dwconv"):
        """GhostConv.cv2 (depthwise 5x5 conv + folded BN + act) of view x into view out on y5_dwconv_fwd, + residual; x_out
        (optional) receives x + x_res in the same launch.  The weights are y5_fold_pack's [c][5][5][1] packing."""
        c = x.c
        wp = torch.empty(c, 5, 5, 1, dtype=self.dtype, device=self.device)
        bias = torch.empty(c, dtype=torch.float32, device=self.device)
        self.fold_pack_into([(m.conv.weight, m.conv.bias, getattr(m, "bn", None))], wp, bias, 0, 1)
        self._keep += [wp, bias]
        code, slope = act_spec(m.act)

        def view(v):
            return (v.ptr, v.pitch) if v is not None else (None, 0)

        self.ops.append(_Op(name, self.lib.y5_dwconv_fwd, (x.ptr, x.pitch, wp.data_ptr(), bias.data_ptr(), out.ptr, out.pitch, *view(residual),
                                                           *view(x_res), *view(x_out), self.B, x.h, x.w, c, 5, 1, code, slope, 0, self.dt_code)))
        pix = self.B * x.h * x.w
        self.flops += 2 * 25 * pix * c
        self.act_bytes += 2 * pix * c * (2 + (residual is not None) + (x_out is not None) + (x_res is not None))
        self.weight_bytes += 2 * 25 * c

    def lower_ghost(self, m, x: View, out: View | None, name):
        """GhostConv: cv1 on the conv GEMM straight into out[:, :c_], the depthwise conv from that slice into out[:, c_:]."""
        c_ = ghost_dw_channels(m)
        ho, wo = self.out_hw(m.cv1, x)
        out = out or self.new_view(ho, wo, 2 * c_)
        y = out.slice(0, c_)
        self.conv_module(m.cv1, x, y, None, f"{name}.cv1")
        self.dwconv(m.cv2, y, out.slice(c_, c_), name=f"{name}.cv2")
        return out

    def lower_ghost_bottleneck(self, m, x: View, out: View | None, name, scratch=None):
        """GhostBottleneck (s=1): out = cat(u, dw(u)) + x with u = g2.cv1(g1(x)).  g1 writes a scratch view t, g2.cv1 writes u to
        a second one, and one y5_dwconv_fwd launch writes both halves of out: u + x[:, :c] and dw(u) + b + x[:, c:].  out may be x
        itself (C3Ghost's concat slice, in place).  Returns the scratch views (t, u) for the next bottleneck of the chain."""
        g1, g2 = ghost_bottleneck_convs(m)
        c1_, c2_ = ghost_dw_channels(g1), ghost_dw_channels(g2)
        if 2 * c2_ != x.c:
            raise NotImplementedError(f"y5b200: GhostBottleneck {x.c} -> {2 * c2_} channels (its identity shortcut needs c1 == c2)")
        t, u = scratch or (self.new_view(x.h, x.w, 2 * c1_), self.new_view(x.h, x.w, c2_))
        self.lower_ghost(g1, x, t, f"{name}.conv.0")
        self.conv_module(g2.cv1, t, u, None, f"{name}.conv.2.cv1")
        out = out or self.new_view(x.h, x.w, x.c)
        self.dwconv(g2.cv2, u, out.slice(c2_, c2_), residual=x.slice(c2_, c2_), x_out=out.slice(0, c2_), x_res=x.slice(0, c2_),
                    name=f"{name}.conv.2.cv2")
        return t, u

    def lower_transformer(self, tb, a: View, name):
        """C3TR's TransformerBlock (reference models/common.py:115-161) over the H*W tokens of view `a`, in place: its result
        lands in `a` (the C3's concat slice).  Per layer, with the projections folded in fp32 here, as BatchNorm is:
          qkv = x [in_q q | in_k k | in_v v]^T + in_proj_bias      one GEMM with 3c outputs
          o   = y5_attention_fwd(qkv)                              per image and head, softmax(q k^T / sqrt(dh)) v
          x   = o out_proj^T + out_proj.bias + x                   the residual rides the GEMM epilogue
          x   = x (fc2 fc1)^T + x                                  fc2 . fc1 folded into one GEMM
        after the position embedding x = a linear^T + linear.bias + a."""
        heads, dh = transformer_spec(tb, training=False)
        c, m_rows, es = a.c, self.B * a.h * a.w, self.dtype.itemsize

        def packed(w, b):
            return self.fold_pack([(w.reshape(w.shape[0], w.shape[1], 1, 1), b, None)], m_rows)

        x = self.new_view(a.h, a.w, c)
        qkv, o, y = self.new_view(a.h, a.w, 3 * c), self.new_view(a.h, a.w, c), self.new_view(a.h, a.w, c)
        self.conv(a, x, packed(tb.linear.weight, tb.linear.bias), 1, 1, 0, False, a, f"{name}.linear")
        seq = a.h * a.w
        for j, layer in enumerate(tb.tr):
            ma, nm = layer.ma, f"{name}.tr{j}"
            wi = ma.in_proj_weight.detach().float()
            w_qkv = torch.cat([wi[i * c : (i + 1) * c] @ lin.weight.detach().float() for i, lin in enumerate((layer.q, layer.k, layer.v))])
            self.conv(x, qkv, packed(w_qkv, ma.in_proj_bias.detach().float()), 1, 1, 0, False, None, f"{nm}.qkv")
            self.ops.append(_Op(f"{nm}.attn", self.lib.y5_attention_fwd, (qkv.ptr, qkv.ptr + c * es, qkv.ptr + 2 * c * es, qkv.pitch, o.ptr,
                                                                         o.pitch, None, self.B, seq, heads, dh, dh ** -0.5, self.dt_code)))
            self.flops += 4 * self.B * heads * seq * seq * dh
            self.act_bytes += 2 * self.B * seq * 4 * c
            self.conv(o, y, packed(ma.out_proj.weight, ma.out_proj.bias), 1, 1, 0, False, x, f"{nm}.out_proj")
            w_fc = layer.fc2.weight.detach().float() @ layer.fc1.weight.detach().float()
            self.conv(y, a if j == len(tb.tr) - 1 else x, packed(w_fc, None), 1, 1, 0, False, y, f"{nm}.fc2.fc1")
        if not len(tb.tr):
            self.copy_into(x, a, f"{name}.copy")

    def lower_sppf(self, m, x: View, out: View | None, name, k: int | None = None):
        """SPPF, or SPP with pools (k, 2k-1, 3k-2) (k given): both are cv2(cat(a, mp_k(a), mp_k^2(a), mp_k^3(a))), a = cv1(x)."""
        c_ = m.cv1.conv.out_channels
        if k is None:
            k = m.m.kernel_size if isinstance(m.m.kernel_size, int) else m.m.kernel_size[0]
        cat = self.new_view(x.h, x.w, 4 * c_)
        s0, s1, s2, s3 = (cat.slice(i * c_, c_) for i in range(4))
        self.conv_module(m.cv1, x, s0, None, f"{name}.cv1")
        self.ops.append(_Op(f"{name}.pool", self.lib.y5_sppf_pool,
                            (s0.ptr, s0.pitch, s1.ptr, s2.ptr, s3.ptr, cat.pitch, self.B, x.h, x.w, c_, k, self.dt_code)))
        out = out or self.new_view(x.h, x.w, m.cv2.conv.out_channels)
        self.conv_module(m.cv2, cat, out, None, f"{name}.cv2")
        return out

    def lower_pool(self, x: View, out: View | None, mode: int, name):
        """nn.MaxPool2d(2, 2, 0), or the nn.ZeroPad2d((0, 1, 0, 1)) + nn.MaxPool2d(2, 1, 0) pair, as one y5_maxpool2d launch."""
        ho, wo = (x.h // 2, x.w // 2) if mode == _lib.POOL_K2S2 else (x.h, x.w)
        out = out or self.new_view(ho, wo, x.c)
        assert (out.h, out.w, out.c) == (ho, wo, x.c), name
        self.ops.append(_Op(name, self.lib.y5_maxpool2d, (x.ptr, x.pitch, out.ptr, out.pitch, self.B, x.h, x.w, x.c, mode, self.dt_code)))
        self.act_bytes += 2 * self.B * (x.h * x.w + ho * wo) * x.c
        return out

    def lower_upsample(self, m, x: View, out: View | None, name):
        sf = m.scale_factor
        if float(sf) != 2.0 or m.mode != "nearest":
            raise NotImplementedError("y5b200: only nn.Upsample(scale_factor=2, mode='nearest')")
        out = out or self.new_view(2 * x.h, 2 * x.w, x.c)
        self.ops.append(_Op(name, self.lib.y5_upsample2x, (x.ptr, x.pitch, out.ptr, out.pitch, self.B, x.h, x.w, x.c, self.dt_code)))
        return out

    def copy_into(self, x: View, out: View, name):
        self.ops.append(_Op(name, self.lib.y5_copy_view, (x.ptr, x.pitch, out.ptr, out.pitch, self.B * x.h * x.w, x.c, self.dt_code)))

    def lower_proto(self, m, x: View, name):
        a = self.lower_conv(m.cv1, x, None, f"{name}.cv1")
        u = self.lower_upsample(m.upsample, a, None, f"{name}.up")
        b = self.lower_conv(m.cv2, u, None, f"{name}.cv2")
        return self.lower_conv(m.cv3, b, None, f"{name}.cv3")

    def lower_detect(self, m, xs: list[View], name):
        na, no, nc = m.na, m.no, m.nc
        if no > HEAD_MAX_NO or nc > HEAD_MAX_NC:
            raise NotImplementedError(f"y5b200: Detect with no={no} nc={nc}: the head takes no <= {HEAD_MAX_NO} outputs per anchor "
                                      f"and nc <= {HEAD_MAX_NC} classes")
        npad = -(-no // HEAD_N) * HEAD_N  # rows per anchor in the packed weights: ceil(no / 128) N tiles
        self.z_rows = sum(na * v.h * v.w for v in xs)
        self.det_shapes = [(self.B, na, v.h, v.w, no) for v in xs]
        row0 = 0
        for i, v in enumerate(xs):
            conv = m.m[i]
            # every anchor's `no` rows padded to npad: one fold_pack launch per anchor (weights + bias, no BatchNorm)
            bk = block_k(v.c, na * no, self.B * v.h * v.w)
            ipad = (v.c + bk - 1) // bk * bk
            wp = torch.empty(na * npad, 1, 1, ipad, dtype=self.dtype, device=self.device)
            bias = torch.empty(na * npad, dtype=torch.float32, device=self.device)
            w4 = conv.weight.detach().contiguous().view(na, no, v.c, 1, 1)
            b2 = conv.bias.detach().contiguous().view(na, no)
            for a_i in range(na):
                self.fold_pack_into([(w4[a_i], b2[a_i], None)], wp, bias, a_i * npad, ipad, pad_rows_to=npad)
            self._keep += [wp, bias, w4, b2]
            d = DetectDesc()
            d.inp, d.in_pitch = v.ptr, v.pitch
            d.batch, d.ny, d.nx, d.in_c = self.B, v.h, v.w, v.c
            d.weight, d.bias = wp.data_ptr(), bias.data_ptr()
            dummy = torch.empty(8, dtype=self.dtype, device=self.device)  # real outputs are bound per call
            self._keep.append(dummy)
            d.raw, d.z = dummy.data_ptr(), dummy.data_ptr()
            d.z_rows, d.z_row0 = self.z_rows, row0
            d.na, d.no, d.nc = na, no, nc
            stride = float(m.stride[i])
            d.stride = stride
            anc = (m.anchors[i].detach().float().cpu() * stride).reshape(-1).tolist()
            for q in range(8):
                d.anchor_wh[q] = anc[q] if q < len(anc) else 0.0
            d.dtype, d.block_k = self.dt_code, bk
            plan = C.c_void_p()
            _lib.check(self.lib.y5_detect_plan_create(C.byref(d), C.byref(plan)), f"detect_plan_create[{name}.{i}]")
            self._plans.append((self.lib.y5_detect_plan_destroy, plan))
            self.head_ops.append(plan)
            m_rows = self.B * v.h * v.w
            self.flops += 2 * m_rows * na * no * v.c
            self.act_bytes += 2 * (m_rows * v.c + m_rows * na * no)
            self.weight_bytes += 2 * na * no * v.c
            row0 += na * v.h * v.w

    def lower_classify(self, m, x, name):
        """Classify (models/common.py:1138-1140): conv + folded BN + SiLU, global average pool into a (B,1,1,1280) buffer, then
        the Linear as a 1x1 conv with bias and no activation on that view (nc padded with zero rows to a multiple of 8).
        Dropout is the identity in eval.  The logits stay in the (B,1,1,ncpad) buffer; run_classify exports them."""
        if isinstance(x, list):
            raise NotImplementedError("y5b200: Classify behind a Concat (list input) is outside the engine's hot path")
        a = self.lower_conv(m.conv, x, None, f"{name}.conv")
        pooled = self.new_view(1, 1, a.c)
        self.ops.append(_Op(f"{name}.pool", self.lib.y5_global_avg_pool,
                            (a.ptr, a.pitch, pooled.ptr, pooled.pitch, self.B, a.h, a.w, a.c, self.dt_code)))
        lin = m.linear
        nc, cin = lin.weight.shape
        ncpad = _pad8(nc)
        bk = block_k(cin, ncpad, self.B)
        ipad = (cin + bk - 1) // bk * bk
        wp = torch.empty(ncpad, 1, 1, ipad, dtype=self.dtype, device=self.device)
        bias = torch.empty(ncpad, dtype=torch.float32, device=self.device)
        self.fold_pack_into([(lin.weight.view(nc, cin, 1, 1), lin.bias, None)], wp, bias, 0, ipad, pad_rows_to=ncpad)
        out = self.new_view(1, 1, ncpad)
        self.conv(pooled, out, (wp, bias, bk), 1, 1, 0, False, None, f"{name}.linear")
        self.cls_view = View(out.buf, 0, nc)

    # ------------------------------------------------------------------ builders
    def _build(self):
        from .models import common as mc
        from .models import yolo as my

        mod = self.module
        check_grouped_convs(mod)  # every refusal of a grouped conv before the first launch
        self.stem_in = None
        self.image_in = None
        self.proto_view = None
        self.cls_view = None
        self.single_out = None
        if isinstance(mod, my.BaseModel):
            self._build_model(mod)
        else:
            cin = self.in_channels
            x = self.new_view(self.H, self.W, cin)
            self.layer_in = x
            self.single_out = self._lower(mod, x, None, type(mod).__name__)

    def _lower(self, m, x, out, name):
        from .models import common as mc

        if isinstance(m, mc.Conv):
            return self.lower_conv(m, x, out, name)
        if isinstance(m, mc.C3):
            return self.lower_c3(m, x, out, name)
        if isinstance(m, mc.SPPF):
            return self.lower_sppf(m, x, out, name)
        if isinstance(m, mc.SPP):
            return self.lower_sppf(m, x, out, name, k=spp_kernel(m))
        if isinstance(m, mc.GhostConv):
            return self.lower_ghost(m, x, out, name)
        if isinstance(m, mc.GhostBottleneck):
            out = out or self.new_view(x.h, x.w, x.c)
            self.lower_ghost_bottleneck(m, x, out, name)
            return out
        if isinstance(m, mc.Bottleneck):
            tmp = self.new_view(x.h, x.w, m.cv1.conv.out_channels)
            self.conv_module(m.cv1, x, tmp, None, f"{name}.cv1")
            out = out or self.new_view(x.h, x.w, m.cv2.conv.out_channels)
            self.conv_module(m.cv2, tmp, out, x if m.add else None, f"{name}.cv2")
            return out
        if isinstance(m, torch.nn.Upsample):
            return self.lower_upsample(m, x, out, name)
        if isinstance(m, mc.Proto):
            return self.lower_proto(m, x, name)
        if isinstance(m, torch.nn.Sequential):
            for j, sub in enumerate(m):
                x = self._lower(sub, x, out if j == len(m) - 1 else None, f"{name}.{j}")
            return x
        raise NotImplementedError(f"y5b200: module {type(m).__name__} is outside the engine's hot path")

    def _build_model(self, model):
        from .models import common as mc
        from .models import yolo as my

        layers = list(model.model)
        n = len(layers)
        pools = pool_modes(layers, model.save)
        # pass 1: symbolic (c, h, w) of every layer output
        shp = []
        for i, m in enumerate(layers):
            f = m.f
            src = ((3, self.H, self.W) if i == 0 else shp[i - 1]) if f == -1 else (
                shp[f] if isinstance(f, int) else [shp[i - 1] if j == -1 else shp[j] for j in f])
            shp.append(self._shape_of(m, src))
        # pass 2: pre-assign concat members to slices of the concat's buffer
        assigned: dict[int, View] = {}
        concat_buf: dict[int, View] = {}
        for i, m in enumerate(layers):
            if isinstance(m, mc.Concat):
                if m.d != 1:
                    raise NotImplementedError("y5b200: Concat along a dimension other than channels")
                c, h, w = shp[i]
                cat = self.new_view(h, w, c)
                concat_buf[i] = cat
                off = 0
                for j in m.f:
                    src = i - 1 if j == -1 else j
                    cj = shp[src][0]
                    if src not in assigned and cj % 8 == 0 and off % 8 == 0:
                        assigned[src] = cat.slice(off, cj)
                    off += cj
        # pass 3: emit
        outs: list = [None] * n
        x = None
        for i, m in enumerate(layers):
            f = m.f
            name = f"model.{i}"
            if isinstance(m, (my.Detect,)):
                xs = [outs[j] for j in f]
                if isinstance(m, my.Segment):
                    self.proto_view = self.lower_proto(m.proto, xs[0], f"{name}.proto")
                self.lower_detect(m, xs, name)
                continue
            if isinstance(m, mc.Classify):
                self.lower_classify(m, outs[i - 1] if f == -1 else (outs[f] if isinstance(f, int) else [outs[j] for j in f]), name)
                continue
            if isinstance(m, mc.Concat):
                cat = concat_buf[i]
                off = 0
                for j in f:
                    src = i - 1 if j == -1 else j
                    v = outs[src]
                    want = cat.slice(off, v.c)
                    if not (v.buf is cat.buf and v.coff == want.coff):
                        self.copy_into(v, want, f"{name}.copy{src}")
                    off += v.c
                outs[i] = cat
                continue
            xin = (torch.empty(0) if i == 0 else outs[i - 1]) if f == -1 else outs[f % i]  # f < 0 counts back from layer i
            if isinstance(m, torch.nn.ZeroPad2d):  # runs inside the max-pool after it (pool_modes checked the pair)
                outs[i] = xin
            elif isinstance(m, torch.nn.MaxPool2d):
                outs[i] = self.lower_pool(xin, assigned.get(i), pools[i], name)
            else:
                outs[i] = self._lower(m, xin, assigned.get(i), name)
        self.outs = outs

    def _shape_of(self, m, src):
        from .models import common as mc
        from .models import yolo as my

        if isinstance(m, mc.Conv):
            c, h, w = src
            k, s, p = m.conv.kernel_size[0], m.conv.stride[0], m.conv.padding[0]
            return (m.conv.out_channels, (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1)
        if isinstance(m, mc.C3):
            return (m.cv3.conv.out_channels, src[1], src[2])
        if isinstance(m, (mc.SPPF, mc.SPP, mc.Bottleneck)):
            return (m.cv2.conv.out_channels, src[1], src[2])
        if isinstance(m, mc.GhostConv):
            c, h, w = src
            k, s, p = m.cv1.conv.kernel_size[0], m.cv1.conv.stride[0], m.cv1.conv.padding[0]
            return (2 * m.cv1.conv.out_channels, (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1)
        if isinstance(m, mc.GhostBottleneck):  # the stride-1 form (check_grouped_convs refused the other)
            return (2 * m.conv[2].cv1.conv.out_channels, src[1], src[2])
        if isinstance(m, torch.nn.Sequential):
            for sub in m:
                src = self._shape_of(sub, src)
            return src
        if isinstance(m, torch.nn.ZeroPad2d):
            left, right, top, bottom = m.padding
            return (src[0], src[1] + top + bottom, src[2] + left + right)
        if isinstance(m, torch.nn.MaxPool2d):  # a form pool_modes accepted: (2, 2, 0) or (2, 1, 0)
            s = m.stride if isinstance(m.stride, int) else m.stride[0]
            return (src[0], (src[1] - 2) // s + 1, (src[2] - 2) // s + 1)
        if isinstance(m, torch.nn.Upsample):
            return (src[0], src[1] * 2, src[2] * 2)
        if isinstance(m, mc.Concat):
            return (sum(s[0] for s in src), src[0][1], src[0][2])
        if isinstance(m, (my.Detect, mc.Classify)):
            return None
        raise NotImplementedError(f"y5b200: module {type(m).__name__} is outside the engine's hot path")

    # ------------------------------------------------------------------ execution
    def _run_fixed(self, stream: int):
        for op in self.ops:
            op.run(stream)

    def capture(self):
        """Capture the fixed part into a CUDA graph (input pointer independent: starts after the stem s2d)."""
        s = torch.cuda.Stream(device=self.device)
        s.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(s):
            self._run_fixed(s.cuda_stream)  # warm-up outside capture (lazy module loading, attribute setup)
        torch.cuda.current_stream(self.device).wait_stream(s)
        torch.cuda.synchronize(self.device)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            self._run_fixed(torch.cuda.current_stream(self.device).cuda_stream)
        self.graph = g

    def _run_body(self, img: torch.Tensor, use_graph: bool) -> int:
        """stem space-to-depth of `img`, then the fixed part (graph replay); returns the stream pointer."""
        assert img.is_cuda and img.shape == (self.B, 3, self.H, self.W), (img.shape, (self.B, 3, self.H, self.W))
        if self.image_in is not None:
            image_nhwc(img, self.image_in)
        else:
            stem_s2d(img, self.stem_in)
        st = _lib.stream_ptr(self.device)
        if use_graph and os.environ.get("Y5_NO_GRAPH") != "1":
            if self.graph is None:
                self.capture()
            self.graph.replay()
        else:
            self._run_fixed(st)
        return st

    def run_classify(self, img: torch.Tensor, use_graph: bool = True) -> torch.Tensor:
        """ClassificationModel: img (B,3,H,W) as run_model takes it -> a fresh (B, nc) logits tensor every call."""
        st = self._run_body(img, use_graph)
        v = self.cls_view
        y = torch.empty(self.B, v.c, dtype=self.dtype, device=self.device)
        _lib.check(self.lib.y5_nhwc_to_nchw(v.ptr, v.pitch, y.data_ptr(), self.B, 1, 1, v.c, self.dt_code, C.c_void_p(st)), "nhwc_to_nchw")
        return y

    def run_model(self, img: torch.Tensor, use_graph: bool = True):
        """img: (B,3,H,W) NCHW uint8 (scaled by 1/255 on the fly) or fp16/bf16/fp32 in [0,1]."""
        st = self._run_body(img, use_graph)
        # head: fresh output tensors every call, like the reference
        no = self.det_shapes[0][-1]
        z = torch.empty(self.B, self.z_rows, no, dtype=self.dtype, device=self.device)
        raws = [torch.empty(s, dtype=self.dtype, device=self.device) for s in self.det_shapes]
        for plan, raw in zip(self.head_ops, raws):
            _lib.check(self.lib.y5_detect_plan_run_to(plan, raw.data_ptr(), z.data_ptr(), C.c_void_p(st)), "detect")
        proto = None
        if self.proto_view is not None:
            pv = self.proto_view
            proto = torch.empty(self.B, pv.c, pv.h, pv.w, dtype=self.dtype, device=self.device)
            _lib.check(self.lib.y5_nhwc_to_nchw(pv.ptr, pv.pitch, proto.data_ptr(), self.B, pv.h, pv.w, pv.c, self.dt_code,
                                                C.c_void_p(st)), "nhwc_to_nchw")
        return z, raws, proto

    def run_layer(self, x: torch.Tensor) -> torch.Tensor:
        """Single-layer program: x (B,C,H,W) NCHW -> (B,C2,H2,W2) NCHW.  The NCHW->NHWC staging of the input is a
        torch copy (plumbing); the layer itself and the NHWC->NCHW export run in liby5b200."""
        v = self.layer_in
        v.buf[..., : v.c].copy_(x.permute(0, 2, 3, 1))
        st = _lib.stream_ptr(self.device)
        self._run_fixed(st)
        o = self.single_out
        y = torch.empty(self.B, o.c, o.h, o.w, dtype=self.dtype, device=self.device)
        _lib.check(self.lib.y5_nhwc_to_nchw(o.ptr, o.pitch, y.data_ptr(), self.B, o.h, o.w, o.c, self.dt_code, C.c_void_p(st)),
                   "nhwc_to_nchw")
        return y

    def launches_per_forward(self) -> int:
        n = len(self.ops) + len(self.head_ops) + (1 if self.stem_in is not None or self.image_in is not None else 0)
        n += 1 if self.proto_view is not None else 0
        return n + (1 if self.cls_view is not None else 0)

    def __del__(self):
        try:
            for fn, h in self._plans:
                fn(h)
        except Exception:
            pass
