"""GPU: the conv mainloop keeps one wgmma batch in flight and hands a batch's shared-memory stages back to the producer only
after the next batch has been issued and this one has completed.  Every place where that deferred release can go wrong is run
here against the fp32 oracle of test_conv_gpu.py (same criterion, both dtypes): one K block per tile (the only release is the
one at the tile's end), long K loops through 2 A stages, grouped weight stages (kh members per stage), the wide patch (kh*kw
members per A stage), 2- and 4-CTA clusters (remote releases of multicast stages), forced 16- and 32-channel K blocks (1 and 2
k16 steps per batch), far more tiles than CTAs (ring phases wrap many times), and the Detect-head epilogue with M not a
multiple of 128."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from yolov5_b200 import _lib
from yolov5_b200.engine import pack_weight

from .gpu_util import conv_case, rel_err

pytestmark = pytest.mark.gpu
TOL = {torch.float16: 2e-3, torch.bfloat16: 1.6e-2}
DTYPES = [torch.float16, torch.bfloat16]


def _check(dev, dtype, case, **kw):
    got, ref, untouched = conv_case(dev, dtype, *case, **kw)
    assert rel_err(got, ref) < TOL[dtype], (case, kw, rel_err(got, ref))
    assert untouched, "epilogue wrote outside its channel slice"


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", [
    (2, 16, 16, 64, 64, 1, 1, 0),    # 4 tiles, one K block each
    (64, 40, 40, 64, 64, 1, 1, 0),   # 400 tiles of one K block: the tile-end release is the only one, hundreds of times per CTA
    (3, 13, 11, 48, 256, 1, 1, 0),   # one K block, 256-wide tiles, M tail
])
def test_single_k_block_per_tile(cuda, dtype, case):
    _check(cuda, dtype, case, residual=True)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", [
    # 7x7 stride-1 patches, 64-wide N tiles with 2 sub-tiles: a 22 x 8-pixel patch per sub-tile (45 KB a stage) and grouped weight
    # stages of 7 tiles (56 KB) leave room for 2 A and 2 B stages only; 49 / 98 K blocks per tile
    (2, 32, 32, 64, 64, 7, 1, 3),
    (4, 32, 32, 128, 64, 7, 1, 3),
])
def test_many_k_blocks_two_a_stages(cuda, dtype, case):
    _check(cuda, dtype, case, a_mode=2, residual=True)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("bn", [32, 64, 128])
@pytest.mark.parametrize("case", [(2, 40, 40, 128, 128, 3, 1, 1), (3, 13, 27, 64, 128, 3, 1, 1), (2, 24, 24, 192, 128, 5, 1, 2)])
def test_grouped_weight_stages(cuda, dtype, bn, case):
    """3x3 / 5x5 patches with block_n <= 128: one weight stage holds the kh tiles of a (chunk, horizontal tap) group and is released
    after its last member; 5x5 at 128 wide gets only 2 weight stages."""
    _check(cuda, dtype, case, a_mode=2, block_n=bn, residual=True, in_extra=8, out_extra=24)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case,kw", [
    ((2, 32, 32, 64, 64, 3, 1, 1), dict()),                         # two sub-tiles in one patch, 9 taps per A stage
    ((1, 48, 80, 128, 128, 3, 1, 1), dict()),                       # two channel chunks
    ((2, 24, 24, 192, 128, 5, 1, 2), dict()),                       # 25 taps per A stage
    ((8, 40, 40, 256, 256, 3, 1, 1), dict(block_n=256)),            # 256-wide weight tiles, 36 K blocks, several tiles per CTA
    ((4, 32, 32, 64, 64, 3, 1, 1), dict(block_n=64, cg2=True)),     # wide patch inside a CTA pair
])
def test_wide_patch(cuda, dtype, case, kw):
    _check(cuda, dtype, case, a_mode=2, wide_patch=True, residual=True, in_extra=8, out_extra=24, expect=dict(wide=True), **kw)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("cluster", [2, 4])
@pytest.mark.parametrize("case,kw", [
    ((4, 40, 40, 64, 256, 3, 1, 1), dict(block_n=256, a_mode=2)),             # patch, 256-wide multicast stages
    ((4, 32, 32, 128, 128, 3, 1, 1), dict(block_n=128, a_mode=2, mt2=True)),  # grouped multicast stages, two sub-tiles
    ((5, 24, 24, 128, 512, 1, 1, 0), dict(block_n=128)),                      # linear, 2 K blocks, super-tile count not a multiple
    ((3, 40, 40, 128, 384, 3, 2, 1), dict(block_n=256)),                      # im2col stride 2, N tail
    ((16, 80, 80, 64, 256, 3, 1, 1), dict(block_n=256)),                      # many tiles per cluster: phases wrap
])
def test_clusters(cuda, dtype, cluster, case, kw):
    _check(cuda, dtype, case, cluster=cluster, residual=True, expect=dict(cluster=cluster), **kw)


# ------------------------------------------------------------------------------------------------------------------------------
# forced K-block widths: conv_case takes the planner's block_k, so this helper packs and plans with the width asked for
def _conv_block_k(dev, dtype, B, H, W, cin, cout, k, s, p, block_k, a_mode=0, block_n=0, seed=1):
    lib = _lib.lib()
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(B, cin, H, W, generator=g) * 2 - 1
    w = (torch.rand(cout, cin, k, k, generator=g) * 2 - 1) / (cin * k * k) ** 0.5 * 2
    b = torch.rand(cout, generator=g) - 0.5
    ref = F.silu(F.conv2d(x.to(dtype).float(), w.to(dtype).float(), b, stride=s, padding=p))
    Ho, Wo = ref.shape[2], ref.shape[3]
    xin = x.permute(0, 2, 3, 1).contiguous().to(dev, dtype)
    out = torch.empty(B, Ho, Wo, cout, dtype=dtype, device=dev)
    wp = pack_weight(w, block_k, dtype).to(dev)
    bias = b.to(dev)
    d = _lib.ConvDesc()
    d.inp, d.in_pitch = xin.data_ptr(), cin
    d.batch, d.in_h, d.in_w, d.in_c = B, H, W, cin
    d.weight, d.bias = wp.data_ptr(), bias.data_ptr()
    d.out, d.out_pitch, d.out_c = out.data_ptr(), cout, cout
    d.residual, d.res_pitch = None, 0
    d.ksize, d.stride, d.pad = k, s, p
    d.act, d.dtype, d.block_k, d.block_n, d.a_mode = 1, _lib.dtype_code(dtype), block_k, block_n, a_mode
    _lib.check(lib.y5_conv_bn_silu_fwd(C.byref(d), C.c_void_p(_lib.stream_ptr(dev))), "conv")
    torch.cuda.synchronize()
    return out.float().cpu().permute(0, 3, 1, 2), ref


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("block_k", [16, 32])
@pytest.mark.parametrize("case,kw", [
    ((2, 16, 16, 64, 64, 1, 1, 0), dict()),                     # linear
    ((2, 20, 20, 64, 128, 3, 1, 1), dict(a_mode=1)),            # im2col
    ((2, 40, 40, 64, 128, 3, 1, 1), dict(a_mode=2)),            # patch, grouped weight stages
    ((2, 20, 20, 96, 256, 3, 1, 1), dict(a_mode=2, block_n=256)),
    ((2, 16, 24, 48, 64, 3, 2, 1), dict()),                     # stride 2, channel count not a multiple of the block
    ((16, 80, 80, 32, 64, 3, 1, 1), dict()),                    # many tiles per CTA
])
def test_forced_block_k(cuda, dtype, block_k, case, kw):
    got, ref = _conv_block_k(cuda, dtype, *case, block_k=block_k, **kw)
    assert rel_err(got, ref) < TOL[dtype], (case, block_k, kw, rel_err(got, ref))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", [(16, 80, 80, 64, 128, 3, 1, 1), (32, 40, 40, 128, 256, 3, 1, 1), (64, 20, 20, 256, 512, 3, 2, 1)])
def test_many_tiles_per_cta(cuda, dtype, case):
    """Hundreds of tiles over 132 persistent CTAs: the A and B rings wrap their phases many times, with a release pending at every
    tile boundary."""
    _check(cuda, dtype, case)


# ------------------------------------------------------------------------------------------------------------------------------
# Detect head: the same mainloop with the head epilogue (raw logits + decoded boxes staged in shared memory)
def _detect_case(dev, dtype, B, ny, nx, cin, na=3, nc=80, stride=16.0, seed=2):
    HEAD_N = 128
    no = nc + 5
    lib = _lib.lib()
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(B, ny, nx, cin, generator=g) * 2 - 1
    w = (torch.rand(na * no, cin, generator=g) * 2 - 1) / cin ** 0.5 * 2
    b = torch.rand(na * no, generator=g) - 0.5
    anchors = torch.tensor([[10.0, 13.0], [16.0, 30.0], [33.0, 23.0]])[:na]
    # oracle (models/yolo.py Detect): raw (B, na, ny, nx, no); decoded xy, wh in pixels, sigmoid scores
    raw = (x.to(dtype).float().reshape(-1, cin) @ w.to(dtype).float().t() + b).reshape(B, ny, nx, na, no).permute(0, 3, 1, 2, 4)
    sg = raw.sigmoid()
    yv, xv = torch.meshgrid(torch.arange(ny, dtype=torch.float32), torch.arange(nx, dtype=torch.float32), indexing="ij")
    grid = torch.stack((xv, yv), 2).view(1, 1, ny, nx, 2) - 0.5
    xy = (sg[..., :2] * 2 + grid) * stride
    wh = (sg[..., 2:4] * 2) ** 2 * anchors.view(1, na, 1, 1, 2)
    z_ref = torch.cat((xy, wh, sg[..., 4:]), -1).reshape(B, -1, no)

    bk = C.c_int32()
    _lib.check(lib.y5_conv_pick(cin, na * no, B * ny * nx, C.byref(bk), None))
    ipad = (cin + bk.value - 1) // bk.value * bk.value
    wp = torch.zeros(na * HEAD_N, ipad, dtype=dtype)
    bias = torch.zeros(na * HEAD_N, dtype=torch.float32)
    for a in range(na):
        wp[a * HEAD_N : a * HEAD_N + no, :cin] = w[a * no : (a + 1) * no].to(dtype)
        bias[a * HEAD_N : a * HEAD_N + no] = b[a * no : (a + 1) * no]
    wp, bias = wp.to(dev), bias.to(dev)
    xin = x.to(dev, dtype)
    raw_out = torch.full((B, na, ny, nx, no), -5.0, dtype=dtype, device=dev)
    z_out = torch.full((B, na * ny * nx, no), -5.0, dtype=dtype, device=dev)
    d = _lib.DetectDesc()
    d.inp, d.in_pitch = xin.data_ptr(), cin
    d.batch, d.ny, d.nx, d.in_c = B, ny, nx, cin
    d.weight, d.bias = wp.data_ptr(), bias.data_ptr()
    d.z_rows, d.z_row0 = na * ny * nx, 0
    d.na, d.no, d.nc = na, no, nc
    d.stride = stride
    for q, v in enumerate(anchors.reshape(-1).tolist()):
        d.anchor_wh[q] = v
    d.dtype, d.block_k = _lib.dtype_code(dtype), bk.value
    plan = C.c_void_p()
    _lib.check(lib.y5_detect_plan_create(C.byref(d), C.byref(plan)), "detect_plan_create")
    try:
        _lib.check(lib.y5_detect_plan_run_to(plan, C.c_void_p(raw_out.data_ptr()), C.c_void_p(z_out.data_ptr()),
                                             C.c_void_p(_lib.stream_ptr(dev))), "detect")
        torch.cuda.synchronize()
    finally:
        lib.y5_detect_plan_destroy(plan)
    return raw_out.float().cpu(), raw, z_out.float().cpu(), z_ref


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", [
    (3, 10, 10, 128),   # M = 300: last tile of 44 rows, tiles straddle images
    (64, 13, 13, 256),  # M = 10816 (84.5 tiles) x 3 anchors: several tiles per CTA, 4 K blocks each
    (5, 7, 9, 64),      # M = 315, one K block per tile
])
def test_detect_head_run_to(cuda, dtype, case):
    raw, raw_ref, z, z_ref = _detect_case(cuda, dtype, *case)
    assert rel_err(raw, raw_ref) < TOL[dtype], (case, "raw", rel_err(raw, raw_ref))
    assert rel_err(z, z_ref) < TOL[dtype], (case, "z", rel_err(z, z_ref))
