"""GPU: the conv epilogue's residual add with the residual in place (residual == out, the engine's Bottleneck lowering) and in a
separate buffer, both as channel slices of wider buffers.  The epilogue loads a batch of residual words before storing any of
them, so the in-place case checks that each thread still reads every element before it overwrites it, also across the two
load batches of 256-wide tiles.  Both placements must give the same bytes (the arithmetic is the same), match the fp32 oracle
SiLU(conv2d(x, W') + b') + r, and leave the bytes outside the slice untouched; the staged store path (reserved bit 8) must give
the same bytes again."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from yolov5_b200 import _lib
from yolov5_b200.engine import pack_weight

from .gpu_util import rel_err

pytestmark = pytest.mark.gpu
TOL = {torch.float16: 2e-3, torch.bfloat16: 1.6e-2}
SENTINEL = -3.0


def run_residual(dev, dtype, B, H, W, cin, cout, k, s, p, act=True, in_place=False, block_n=0, mt2=False, a_mode=0, staged=False,
                 seed=0):
    """Runs one conv with a residual; out and residual are channels [8, 8 + cout) of [B, Ho, Wo, cout + 24] buffers.
    Returns (whole output buffer, oracle NCHW fp32)."""
    lib = _lib.lib()
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(B, cin, H, W, generator=g) * 2 - 1
    w = (torch.rand(cout, cin, k, k, generator=g) * 2 - 1) / (cin * k * k) ** 0.5 * 2
    b = torch.rand(cout, generator=g) - 0.5
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    r = torch.rand(B, cout, Ho, Wo, generator=g) - 0.5
    y = F.conv2d(x.to(dtype).float(), w.to(dtype).float(), b, stride=s, padding=p)
    if act:
        y = F.silu(y)
    y = y + r.to(dtype).float()
    off, pitch = 8, cout + 24
    xin = x.permute(0, 2, 3, 1).contiguous().to(dev, dtype)
    obuf = torch.full((B, Ho, Wo, pitch), SENTINEL, dtype=dtype, device=dev)
    rbuf = obuf if in_place else torch.full((B, Ho, Wo, pitch), 5.0, dtype=dtype, device=dev)
    rbuf[..., off : off + cout] = r.permute(0, 2, 3, 1).to(dev, dtype)
    bk, bn = C.c_int32(), C.c_int32()
    _lib.check(lib.y5_conv_pick(cin, cout, B * Ho * Wo, C.byref(bk), C.byref(bn)))
    wp = pack_weight(w, bk.value, dtype).to(dev)
    bias = b.to(dev)
    es = obuf.element_size()
    d = _lib.ConvDesc()
    d.inp, d.in_pitch = xin.data_ptr(), cin
    d.batch, d.in_h, d.in_w, d.in_c = B, H, W, cin
    d.weight, d.bias = wp.data_ptr(), bias.data_ptr()
    d.out, d.out_pitch, d.out_c = obuf.data_ptr() + off * es, pitch, cout
    d.residual, d.res_pitch = rbuf.data_ptr() + off * es, pitch
    d.ksize, d.stride, d.pad = k, s, p
    d.act, d.dtype, d.block_k, d.block_n = int(act), _lib.dtype_code(dtype), bk.value, block_n
    d.a_mode = a_mode
    d.reserved = (2 if mt2 else 0) | (8 if staged else 0)
    _lib.check(lib.y5_conv_bn_silu_fwd(C.byref(d), C.c_void_p(_lib.stream_ptr(dev))), "conv")
    torch.cuda.synchronize()
    return obuf, y


def check(dev, dtype, case, **kw):
    sep, ref = run_residual(dev, dtype, *case, **kw)
    inp, _ = run_residual(dev, dtype, *case, in_place=True, **kw)
    cout = case[4]
    assert bool((sep[..., :8] == SENTINEL).all() and (sep[..., 8 + cout :] == SENTINEL).all()), "wrote outside the slice"
    got = sep[..., 8 : 8 + cout].float().cpu().permute(0, 3, 1, 2)
    assert rel_err(got, ref) < TOL[dtype], (case, kw, rel_err(got, ref))
    assert torch.equal(inp.view(torch.int16), sep.view(torch.int16)), (case, kw, "in-place residual differs from a separate one")
    stg, _ = run_residual(dev, dtype, *case, in_place=True, staged=True, **kw)
    assert torch.equal(stg.view(torch.int16), sep.view(torch.int16)), (case, kw, "staged stores differ from direct ones")


# every (block_n, MT) instantiation of the plain epilogue, forced; layer shapes with M tails and N tails
TILES = [(32, False), (64, False), (128, False), (128, True), (256, False)]
CASES = [
    # B, H, W, cin, cout, k, s, p, a_mode
    (2, 20, 20, 64, 64, 1, 1, 0, 0),     # LINEAR, M = 800: a 128-row tail
    (2, 20, 20, 64, 64, 3, 1, 1, 1),     # IM2COL
    (3, 13, 27, 32, 64, 3, 1, 1, 2),     # PATCH, tiles overhanging Ho and Wo
    (2, 9, 130, 64, 32, 3, 1, 1, 2),     # PATCH, wide map: overhang in x
    (1, 16, 24, 64, 384, 1, 1, 0, 0),    # N tail: 384 = 1.5 256-wide tiles
    (2, 16, 24, 32, 72, 3, 2, 1, 0),     # stride 2 (IM2COL), N tail inside a 32-column group
    (2, 20, 20, 64, 256, 3, 1, 1, 2),    # PATCH, 256 channels: every tile width runs, 256 with two load batches
    (2, 20, 20, 64, 256, 3, 1, 1, 1),    # the same through IM2COL
    (2, 9, 130, 64, 128, 3, 1, 1, 2),    # PATCH overhang in x with 128 channels (bn 64 / 128 / 128x2)
]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("tile", TILES, ids=[f"bn{b}{'x2' if m else ''}" for b, m in TILES])
@pytest.mark.parametrize("case", CASES, ids=lambda c: "x".join(map(str, c)))
def test_residual_in_place_every_tile(cuda, dtype, tile, case):
    if tile[0] >= 2 * case[4]:
        pytest.skip("N tile more than twice the layer width")
    check(cuda, dtype, case[:8], block_n=tile[0], mt2=tile[1], a_mode=case[8])


@pytest.mark.parametrize("act", [True, False])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("case", [(4, 160, 160, 64, 64, 3, 1, 1), (8, 40, 40, 256, 256, 3, 1, 1), (3, 13, 27, 32, 72, 3, 1, 1)],
                         ids=["yolov5l-160", "yolov5l-40", "odd"])
def test_residual_default_plan(cuda, dtype, case, act):
    """The planner's own tile choice at Bottleneck shapes, several tiles per CTA, with and without SiLU."""
    check(cuda, dtype, case, act=act)


def test_residual_many_tiles_per_cta(cuda):
    """1600 tiles of 512 x 32 over at most 132 CTAs: a dozen tiles per CTA, in place."""
    check(cuda, torch.float16, (16, 160, 160, 64, 64, 3, 1, 1), block_n=32)
