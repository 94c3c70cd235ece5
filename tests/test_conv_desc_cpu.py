"""CPU: the conv / weight-gradient descriptors the engine and the training path build (engine.conv_desc, engine.wgrad_desc) and
the stem's two views of its padded space-to-depth buffer (engine.stem_geom), field by field, plus the wide-pixel filter view
against a torch conv."""
import pytest
import torch
import torch.nn.functional as F

from yolov5_b200 import _lib
from yolov5_b200.engine import (ConvInput, conv_desc, pack_weight, stem_buffer, stem_geom, stem_weight_narrow, stem_weight_wide,
                                wgrad_desc)

B, H, W, O = 2, 64, 96, 24


@pytest.mark.parametrize("wide", [True, False])
def test_stem_views(wide):
    buf = stem_buffer(B, H, W, torch.float16, "cpu")
    assert buf.shape == (B, H // 2, W // 2 + 2, 16) and not buf.any()
    row = W // 2 + 2
    w3 = torch.randn(O, 16, 3, 3)
    wv = stem_weight_wide(w3) if wide else w3
    wp = pack_weight(wv, 16, torch.float16)
    bias = torch.zeros(O)
    out = torch.empty(B, H // 2, W // 2, O, dtype=torch.float16)
    d = conv_desc(stem_geom(buf, wide), wp, bias, 16, out.data_ptr(), O, 3, 1, 1, True, torch.float16)
    dw = torch.empty(O, 3, 1 if wide else 3, 48 if wide else 16)
    g = wgrad_desc(stem_geom(buf, wide), out.data_ptr(), O, dw, 3, 1, 1, torch.float16)
    for e in (d, g):
        assert e.inp == buf.data_ptr() + (0 if wide else 16 * buf.element_size())
        assert (e.in_pitch, e.batch, e.in_h, e.in_w, e.in_c) == (16, B, H // 2, W // 2, 48 if wide else 16)
        assert (e.in_x_stride, e.in_y_stride, e.in_n_stride) == (16, row * 16, (H // 2) * row * 16)
        assert (e.kw, e.pad_w) == ((1, 0) if wide else (3, 1))
        assert (e.ksize, e.stride, e.pad, e.dtype) == (3, 1, 1, _lib.Y5_F16)
    assert (d.weight, d.bias, d.out, d.out_pitch, d.out_c) == (wp.data_ptr(), bias.data_ptr(), out.data_ptr(), O, O)
    assert (d.residual, d.res_pitch, d.act, d.block_k, d.block_n, d.a_mode, d.reserved) == (None, 0, _lib.ACT_SILU, 16, 0, 0, 0)
    assert (g.dout, g.dout_pitch, g.out_c, g.dweight, g.accumulate, g.reserved) == (out.data_ptr(), O, O, dw.data_ptr(), 0, 0)


def test_plain_conv_desc():
    x = torch.empty(B, 40, 40, 80, dtype=torch.bfloat16)  # the view: channels [8, 72) of a pitch-80 buffer
    wp = pack_weight(torch.randn(32, 64, 3, 3), 32, torch.bfloat16)
    bias = torch.zeros(32)
    y = torch.empty(B, 20, 20, 48, dtype=torch.bfloat16)
    xv = ConvInput(x.data_ptr() + 8 * x.element_size(), 80, B, 40, 40, 64)
    d = conv_desc(xv, wp, bias, 32, y.data_ptr(), 48, 3, 2, 1, False, torch.bfloat16, y.data_ptr(), 48)
    assert (d.inp, d.in_pitch, d.batch, d.in_h, d.in_w, d.in_c) == (x.data_ptr() + 16, 80, B, 40, 40, 64)
    assert (d.kw, d.pad_w, d.in_x_stride, d.in_y_stride, d.in_n_stride) == (0, 0, 0, 0, 0)
    assert (d.weight, d.bias, d.out, d.out_pitch, d.out_c, d.residual, d.res_pitch) == (wp.data_ptr(), bias.data_ptr(), y.data_ptr(), 48,
                                                                                          32, y.data_ptr(), 48)
    assert (d.ksize, d.stride, d.pad, d.act, d.dtype, d.block_k) == (3, 2, 1, _lib.ACT_NONE, _lib.Y5_BF16, 32)
    dw = torch.empty(32, 3, 3, 64)
    g = wgrad_desc(xv, y.data_ptr(), 48, dw, 3, 2, 1, torch.bfloat16)
    assert (g.inp, g.in_pitch, g.in_c, g.kw, g.in_x_stride, g.dout_pitch, g.out_c, g.ksize, g.stride) == (x.data_ptr() + 16, 80, 64, 0, 0,
                                                                                                         48, 32, 3, 2)


def test_stem_weight_wide_is_the_3x3x16_conv():
    """A 3x1 conv of the (O,48,3,1) filter over the overlapping 48-channel pixels of the padded buffer (what stem_geom's wide
    view reads) equals the 3x3/s1/p1 conv of the (O,16,3,3) filter over the cells; stem_weight_narrow undoes the view."""
    g = torch.Generator().manual_seed(0)
    cells = torch.randn(B, 16, H // 2, W // 2, generator=g, dtype=torch.float64)
    w3 = torch.randn(O, 16, 3, 3, generator=g, dtype=torch.float64)
    buf = stem_buffer(B, H, W, torch.float64, "cpu")
    buf[:, :, 1:-1] = cells.permute(0, 2, 3, 1)
    wide = torch.cat([buf[:, :, s : s + W // 2] for s in range(3)], dim=3).permute(0, 3, 1, 2)
    ref = F.conv2d(cells, w3, padding=1)
    assert torch.allclose(F.conv2d(wide, stem_weight_wide(w3), padding=(1, 0)), ref, rtol=0, atol=1e-12)
    assert torch.equal(stem_weight_narrow(stem_weight_wide(w3)), w3)
