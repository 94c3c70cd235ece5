"""GPU: the wgmma implicit-GEMM conv (through the C ABI) against the fp32 oracle expression
SiLU(conv2d(x, W') + b') [+ residual]  (reference models/common.py:86-92,181) on fp16/bf16-rounded operands.
Tolerance: output is rounded once to fp16 (rel 2^-11) / bf16 (2^-8) after fp32 accumulation -> 2e-3 / 1.6e-2 of max|y|."""
import pytest
import torch

from .gpu_util import conv_case, rel_err

pytestmark = pytest.mark.gpu
TOL = {torch.float16: 2e-3, torch.bfloat16: 1.6e-2}

CASES = [
    # B, H, W, cin, cout, k, s, p
    (2, 16, 16, 64, 64, 1, 1, 0),      # plain GEMM, one K block
    (1, 20, 20, 128, 256, 1, 1, 0),    # M tail (400 rows), N=256
    (3, 8, 12, 32, 32, 1, 1, 0),       # block_k 32 (SW64), M < 128*? tail
    (2, 16, 16, 16, 32, 3, 1, 1),      # im2col, block_k 16 (SW32)  -- the stem's shape class
    (2, 20, 20, 64, 64, 3, 1, 1),      # im2col across rows and images
    (2, 16, 24, 32, 64, 3, 2, 1),      # stride 2
    (1, 40, 40, 128, 128, 3, 1, 1),    # 2 K chunks per tap
    (2, 10, 10, 256, 512, 3, 2, 1),    # deep K (36 blocks), N tiles
    (2, 12, 12, 24, 48, 1, 1, 0),      # channel count not a multiple of 16 (yolov5m widths): TMA zero-fills K
    (1, 12, 12, 48, 96, 3, 1, 1),
    (5, 7, 9, 64, 40, 1, 1, 0),        # odd spatial, N tail inside a tile
]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("case", CASES)
def test_conv_vs_oracle(cuda, dtype, case):
    got, ref, _ = conv_case(cuda, dtype, *case)
    assert rel_err(got, ref) < TOL[dtype], (case, rel_err(got, ref))
    got, ref, _ = conv_case(cuda, dtype, *case, staged=True, expect=dict(staged=1))
    assert rel_err(got, ref) < TOL[dtype], (case, "staged stores", rel_err(got, ref))


@pytest.mark.parametrize("direct_store", [False, True])
@pytest.mark.parametrize("case", [(2, 20, 20, 64, 64, 3, 1, 1), (2, 16, 16, 64, 128, 1, 1, 0), (5, 7, 9, 64, 40, 1, 1, 0), (3, 13, 27, 32, 72, 3, 1, 1)])
def test_conv_residual_and_slices(cuda, case, direct_store):
    """Both epilogue store paths (per-warpgroup staging + 16-byte row-segment stores, and the direct register stores) into a
    channel slice of a wider buffer: N tails inside a 32-channel chunk (40, 72 channels), partial spatial tiles, M tails."""
    got, ref, untouched = conv_case(cuda, torch.float16, *case, residual=True, in_extra=24, out_extra=40, direct_store=direct_store,
                                    staged=not direct_store, expect=dict(staged=int(not direct_store)))
    assert rel_err(got, ref) < 2e-3
    assert untouched, "epilogue wrote outside its channel slice"


@pytest.mark.parametrize("a_mode", [1, 2])
@pytest.mark.parametrize("case", [(2, 20, 20, 64, 64, 3, 1, 1), (2, 16, 16, 16, 32, 3, 1, 1), (1, 40, 40, 128, 128, 3, 1, 1),
                                  (3, 13, 27, 32, 64, 3, 1, 1), (1, 80, 80, 64, 64, 3, 1, 1), (2, 9, 130, 64, 32, 3, 1, 1)])
def test_conv_3x3_both_fetch_modes(cuda, case, a_mode):
    """stride-1 3x3: TMA-im2col (one copy per tap) and shifted-patch (one copy per horizontal tap) must agree with the oracle,
    including partial spatial tiles (13x27, 9x130) and residual + channel-slice views."""
    got, ref, untouched = conv_case(cuda, torch.float16, *case, a_mode=a_mode, residual=True, in_extra=8, out_extra=24)
    assert rel_err(got, ref) < 2e-3, (case, a_mode, rel_err(got, ref))
    assert untouched


# wide-patch requests the planner turns down: two sub-tiles need an even number of 8-pixel tiles per row, four sub-tiles (block_n
# 32) never share a patch, and 9 x 130 tiles with fewer wasted pixels 32 wide than 8 wide
WIDE_FALLS_BACK = {(2, 40, 40, 64, 64, 3, 1, 1), (2, 13, 27, 64, 32, 3, 1, 1), (1, 9, 130, 64, 96, 3, 1, 1), (2, 24, 24, 192, 64, 5, 1, 2),
                   (3, 40, 40, 128, 64, 3, 1, 1)}


@pytest.mark.parametrize("narrow", [False, True])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("case,kw", [
    ((2, 32, 32, 64, 64, 3, 1, 1), dict()),                          # 64 -> 64: two sub-tiles side by side in one 24-pixel-wide patch
    ((2, 40, 40, 64, 64, 3, 1, 1), dict()),                          # odd number of 8-pixel tiles per row: sub-tiles cannot share a patch
    ((1, 48, 80, 128, 128, 3, 1, 1), dict()),                        # two channel chunks, 128-wide N tile
    ((2, 13, 27, 64, 32, 3, 1, 1), dict()),                          # partial tiles in x and y
    ((1, 9, 130, 64, 96, 3, 1, 1), dict()),                          # wide and flat
    ((2, 24, 24, 192, 64, 5, 1, 2), dict()),                         # 5x5, three channel chunks (odd tiles per row -> narrow mode)
    ((4, 40, 40, 64, 256, 3, 1, 1), dict(block_n=256, cg2=True)),    # CTA pairs
    ((4, 32, 32, 128, 128, 3, 1, 1), dict(block_n=128, cg2=True, mt2=True)),  # CTA pairs, two sub-tiles per CTA
    ((4, 32, 32, 64, 64, 3, 1, 1), dict(block_n=64, cg2=True)),      # 64-wide CTA pairs (256 x 64 MMAs), shared 24-pixel patch
    ((3, 40, 40, 128, 64, 3, 1, 1), dict(block_n=64, cg2=True)),     # same, odd tile count per row (separate patches), M tail pair
    ((2, 24, 24, 192, 128, 5, 1, 2), dict()),                        # 5x5 in wide mode (single sub-tile)
])
def test_conv_wide_patch(cuda, case, kw, dtype, narrow):
    """Stride-1 k x k convs with 64-channel chunks fetch ONE (16+k-1) x PW patch per chunk and read all k*k taps from it through
    descriptor offsets (`narrow=False`); the one-copy-per-horizontal-tap mode (`narrow=True`, reserved bit
    32) must give the same answer.  Residual + channel-slice views on both sides."""
    got, ref, untouched = conv_case(cuda, dtype, *case, a_mode=2, residual=True, in_extra=8, out_extra=24, narrow_patch=narrow, wide_patch=not narrow,
                                     expect=dict(wide=not narrow and case not in WIDE_FALLS_BACK), **kw)
    assert rel_err(got, ref) < TOL[dtype], (case, kw, narrow, rel_err(got, ref))
    assert untouched


def test_conv_no_activation(cuda):
    got, ref, _ = conv_case(cuda, torch.float16, 2, 16, 16, 64, 64, 1, 1, 0, act=False)
    assert rel_err(got, ref) < 2e-3


@pytest.mark.parametrize("bn", [32, 64, 128, 256])
def test_conv_every_tile_width(cuda, bn):
    got, ref, _ = conv_case(cuda, torch.float16, 2, 20, 20, 64, 256, 3, 1, 1, block_n=bn)
    assert rel_err(got, ref) < 2e-3


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("case,a_mode", [((2, 20, 20, 64, 256, 3, 1, 1), 1), ((2, 20, 20, 64, 256, 3, 1, 1), 2),
                                         ((3, 16, 16, 128, 256, 1, 1, 0), 0), ((1, 40, 40, 128, 384, 3, 2, 1), 0)])
def test_conv_256_row_tiles(cuda, bn, case, a_mode):
    """MT = 2: two 128-row sub-tiles share every B tile (256x128 tiles; 256-wide weight tiles keep one sub-tile, 128 register columns
    per thread being the limit)."""
    got, ref, _ = conv_case(cuda, torch.float16, *case, block_n=bn, mt2=True, a_mode=a_mode, residual=True)
    assert rel_err(got, ref) < 2e-3, (bn, case, a_mode, rel_err(got, ref))


@pytest.mark.parametrize("bn,mt2", [(128, False), (128, True), (256, False), (256, True)])
@pytest.mark.parametrize("case,a_mode", [((4, 40, 40, 64, 256, 3, 1, 1), 2), ((4, 40, 40, 64, 256, 3, 1, 1), 1), ((5, 24, 24, 128, 512, 1, 1, 0), 0),
                                         ((3, 40, 40, 128, 384, 3, 2, 1), 0)])
def test_conv_cluster_multicast(cuda, bn, mt2, case, a_mode):
    """2-CTA clusters: each CTA fetches half of every weight tile and TMA-multicasts it to its peer; odd super-tile
    counts leave one CTA of the last cluster without work (it must still take part in the multicast protocol).  With block_n 256
    the planner keeps one sub-tile (the accumulators of 256 x 256 do not fit the registers), so (256, True) repeats (256, False)."""
    got, ref, _ = conv_case(cuda, torch.float16, *case, block_n=bn, mt2=mt2, cluster=2, a_mode=a_mode, residual=True, expect=dict(cluster=2))
    assert rel_err(got, ref) < 2e-3, (bn, mt2, case, a_mode, rel_err(got, ref))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("bn,mt2", [(128, False), (128, True), (256, False), (256, True)])
@pytest.mark.parametrize("case,a_mode", [((4, 40, 40, 64, 256, 3, 1, 1), 2), ((4, 40, 40, 64, 256, 3, 1, 1), 1), ((5, 24, 24, 128, 512, 1, 1, 0), 0),
                                         ((3, 40, 40, 128, 384, 3, 2, 1), 0), ((2, 80, 80, 128, 128, 3, 1, 1), 2), ((1, 20, 20, 512, 512, 3, 1, 1), 0)])
def test_conv_cta_pairs(cuda, dtype, bn, mt2, case, a_mode):
    """CTA pairs: the two CTAs of a cluster work on two M super-tiles of the same N tile, each fetching half of every weight tile
    and multicasting it to both; a weight stage is refilled only after the consumers of both CTAs released it.  Odd super-tile
    counts (the second CTA of the last pair has no rows), N tails (384 = 1.5 tiles of 256), every fetch mode, residual operand.
    On Hopper this is the 2-CTA multicast cluster of test_conv_cluster_multicast, checked here in both dtypes and on two more
    shapes; with block_n 256 the planner keeps one sub-tile, so the mt2=True cases of that width repeat mt2=False."""
    if case[4] % bn and bn == 256 and case[4] < 256:
        pytest.skip("N tile wider than the layer")
    got, ref, _ = conv_case(cuda, dtype, *case, block_n=bn, mt2=mt2, cg2=True, a_mode=a_mode, residual=True, expect=dict(cluster=2))
    assert rel_err(got, ref) < TOL[dtype], (bn, mt2, case, a_mode, rel_err(got, ref))


def test_conv_cta_pairs_many_tiles(cuda):
    """Every pair loops over several tiles (barrier phase wrap-around across the pair protocol)."""
    got, ref, _ = conv_case(cuda, torch.float16, 16, 80, 80, 64, 256, 3, 1, 1, block_n=256, cg2=True,  # 800 M tiles -> 400 pair tiles
                            expect=dict(cluster=2))
    assert rel_err(got, ref) < 2e-3


def test_tensor_core_path_agrees_with_direct_kernel(cuda):
    """Two independent device implementations of the same op (wgmma GEMM vs CUDA-core direct conv)."""
    a, ref, _ = conv_case(cuda, torch.float16, 2, 20, 20, 64, 64, 3, 1, 1, seed=5)
    b, _, _ = conv_case(cuda, torch.float16, 2, 20, 20, 64, 64, 3, 1, 1, seed=5, direct=True)
    assert rel_err(a, b) < 2e-3 and rel_err(b, ref) < 2e-3


def test_large_m_many_tiles_per_cta(cuda):
    """More tiles than SMs so every persistent CTA loops, exercising barrier phase wrap-around."""
    got, ref, _ = conv_case(cuda, torch.float16, 8, 80, 80, 64, 64, 3, 1, 1)  # 400 M tiles
    assert rel_err(got, ref) < 2e-3
