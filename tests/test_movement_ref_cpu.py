"""CPU: the data-movement references of tests/movement_ref.py against torch and against naive loops, the identity the
direct SPPF kernel relies on (chained k-pools = one clipped (2k-1) / (3k-2) window, NaN included), and the argument
checks of the forward-path ABI (16-byte aligned views, pitch >= channels) with fake pointers."""

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import movement_ref as mr
from yolov5_b200 import _lib


def _naive_window_max(x: np.ndarray, r: int) -> np.ndarray:
    """max over the clipped (2r+1)^2 window, NaN if any element of the window is NaN"""
    b, c, h, w = x.shape
    out = np.empty_like(x)
    for i in range(h):
        for j in range(w):
            win = x[:, :, max(0, i - r) : i + r + 1, max(0, j - r) : j + r + 1].reshape(b, c, -1)
            out[:, :, i, j] = np.where(np.isnan(win).any(-1), np.nan, np.nanmax(np.where(np.isnan(win), -np.inf, win), -1))
    return out


def _naive_sppf_bwd(a: np.ndarray, dcat: np.ndarray, k: int) -> np.ndarray:
    """The engine's documented backward: last stage first, every output position adds its gradient to the arg-max of its
    window over the stage input (row-major scan, strict '>', a NaN always replaces the running maximum)."""
    b, c, h, w = a.shape
    r = k // 2
    ys = [a]
    for _ in range(3):
        ys.append(_naive_window_max(ys[-1], r))
    acc = [dcat[:, i * c : (i + 1) * c].astype(np.float64).copy() for i in range(4)]
    for stage in (3, 2, 1):  # acc[stage] (gradient of y_stage) -> acc[stage - 1] through the windows of ys[stage - 1]
        src = ys[stage - 1]
        for n in range(b):
            for ch in range(c):
                for i in range(h):
                    for j in range(w):
                        best, arg = -np.inf, None
                        for yy in range(max(0, i - r), min(h, i + r + 1)):
                            for xx in range(max(0, j - r), min(w, j + r + 1)):
                                v = src[n, ch, yy, xx]
                                if arg is None or v > best or np.isnan(v):
                                    best, arg = v, (yy, xx)
                        acc[stage - 1][n, ch][arg] += acc[stage][n, ch, i, j]
    return acc[0]


def test_bit_patterns_hold_every_16_bit_pattern():
    for dtype in (torch.float16, torch.bfloat16):
        x = mr.bit_patterns((2, 8, 64, 128), dtype, seed=3)  # 2 * 65536 elements
        assert x.dtype == dtype and x.shape == (2, 8, 64, 128)
        bits = x.view(torch.int16).flatten().to(torch.int32)
        for half in bits.view(2, 65536):
            assert torch.equal(half.sort().values, torch.arange(-32768, 32768, dtype=torch.int32))
        f = x.float()
        assert bool(f.isnan().any()) and bool(f.isposinf().any()) and bool(f.isneginf().any())
        assert bool(((f == 0) & torch.signbit(f)).any())


@pytest.mark.parametrize("shape", [(1, 2, 1, 1), (1, 2, 2, 2), (2, 3, 3, 5), (1, 2, 7, 9), (1, 1, 1, 17)])
@pytest.mark.parametrize("k", [3, 5, 7])
def test_sppf_fwd_matches_naive_windows_with_nan(shape, k):
    g = torch.Generator().manual_seed(sum(shape) + k)
    x = torch.randint(0, 4, shape, generator=g).double()  # ties everywhere
    x[torch.rand(shape, generator=g) < 0.05] = float("nan")
    x.view(-1)[0] = -float("inf")
    y1, y2, y3 = mr.sppf_fwd(x, k)
    r = k // 2
    n1 = _naive_window_max(x.numpy(), r)
    n2 = _naive_window_max(n1, r)
    n3 = _naive_window_max(n2, r)
    for got, ref in ((y1, n1), (y2, n2), (y3, n3)):
        np.testing.assert_array_equal(got.numpy(), ref)  # NaN positions compared as equal


def test_one_nan_spreads_like_torch_max_pool2d():
    """One NaN in a 7x9 plane: torch's max_pool2d (CPU) spreads it to 25 / 63 / 63 positions of y1 / y2 / y3."""
    x = torch.rand(1, 1, 7, 9, dtype=torch.float64)
    x[0, 0, 3, 4] = float("nan")
    counts = [int(y.isnan().sum()) for y in mr.sppf_fwd(x, 5)]
    assert counts == [25, 63, 63]
    assert [int(y.isnan().sum()) for y in mr.sppf_fwd(x.float(), 5)] == counts  # float32 torch agrees


@pytest.mark.parametrize("shape", [(1, 3, 1, 1), (2, 4, 2, 2), (1, 4, 3, 5), (2, 5, 11, 13), (1, 2, 1, 40), (1, 2, 30, 17)])
@pytest.mark.parametrize("k", [3, 5, 7])
@pytest.mark.parametrize("nan", [False, True])
def test_chained_pools_equal_one_wide_window(shape, k, nan):
    """The direct kernel's identity: y2 is the clipped (2k-1)-window max of x and y3 the (3k-2)-window max."""
    g = torch.Generator().manual_seed(hash((shape, k, nan)) % 1000)
    x = torch.randn(shape, generator=g, dtype=torch.float64)
    x[torch.rand(shape, generator=g) < 0.3] = 0.5  # ties
    if nan:
        x[torch.rand(shape, generator=g) < 0.03] = float("nan")
        x.view(-1)[-1] = float("nan")
    y1, y2, y3 = mr.sppf_fwd(x, k)
    torch.testing.assert_close(y1, mr.windowed_max(x, k), rtol=0, atol=0, equal_nan=True)
    torch.testing.assert_close(y2, mr.windowed_max(x, 2 * k - 1), rtol=0, atol=0, equal_nan=True)
    torch.testing.assert_close(y3, mr.windowed_max(x, 3 * k - 2), rtol=0, atol=0, equal_nan=True)


@pytest.mark.parametrize("shape,k", [((1, 2, 1, 1), 5), ((1, 2, 2, 3), 5), ((2, 2, 5, 6), 5), ((1, 3, 6, 4), 3), ((1, 2, 7, 8), 7)])
@pytest.mark.parametrize("nan", [False, True])
def test_sppf_bwd_routes_like_the_documented_rule(shape, k, nan):
    """float64 autograd through NCHW max_pool2d == the engine's rule (first maximum, last NaN) run as a naive loop,
    exactly, on few-level data (ties everywhere) and small-integer gradients."""
    b, c, h, w = shape
    g = torch.Generator().manual_seed(b * 100 + h * 10 + w + k + nan)
    a = torch.randint(0, 3, shape, generator=g).double()
    if nan:
        a[torch.rand(shape, generator=g) < 0.1] = float("nan")
        a[0, 0, 0, 0] = float("nan")
    dcat = torch.randint(-3, 4, (b, 4 * c, h, w), generator=g).double()
    got = mr.sppf_bwd(a, dcat, k)
    ref = _naive_sppf_bwd(a.numpy(), dcat.numpy(), k)
    np.testing.assert_array_equal(got.numpy(), ref)
    assert float(got.sum()) == float(dcat.sum())  # every gradient lands somewhere


def test_upsample_references_against_torch():
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 8, 5, 7, generator=g).half()
    assert torch.equal(mr.upsample2x(x).float(), F.interpolate(x.float(), scale_factor=2.0, mode="nearest"))
    # integer gradients: every order of the float32 sum is exact, so the emulation equals torch's autograd
    dy = torch.randint(-500, 500, (2, 8, 10, 14), generator=g).float()
    xr = x.float().requires_grad_(True)
    F.interpolate(xr, scale_factor=2.0, mode="nearest").backward(dy)
    assert torch.equal(mr.upsample2x_bwd_f32(dy, torch.float32), xr.grad)
    assert torch.equal(mr.upsample2x_bwd64(dy), xr.grad.double())
    # random gradients: the float32 order is within one float32 rounding per addition of the float64 sum
    dy = torch.randn(2, 8, 10, 14, generator=g)
    e = mr.upsample2x_bwd_f32(dy, torch.float32).double()
    r = mr.upsample2x_bwd64(dy)
    bound = 3 * 2.0 ** -24 * mr.upsample2x_bwd64(dy.abs())
    assert bool(((e - r).abs() <= bound).all())


def test_upsample_bwd_order_is_the_documented_one():
    """(a + b) + c + d in float32, not another order: 1 + 2^-24 + 2^-24 + 0 rounds to 1, 2^-24 + 2^-24 + 1 would not"""
    dy = torch.zeros(1, 1, 2, 2)
    dy[0, 0, 0, 0], dy[0, 0, 0, 1], dy[0, 0, 1, 0] = 1.0, 2.0 ** -24, 2.0 ** -24
    assert float(mr.upsample2x_bwd_f32(dy, torch.float32)) == 1.0
    dy = torch.zeros(1, 1, 2, 2)
    dy[0, 0, 0, 0], dy[0, 0, 0, 1], dy[0, 0, 1, 1] = 2.0 ** -24, 2.0 ** -24, 1.0
    assert float(mr.upsample2x_bwd_f32(dy, torch.float32)) == 1.0 + 2.0 ** -23
    big = torch.full((1, 1, 2, 2), 65504.0)  # fp16's largest finite value: the 2x2 sum overflows to inf
    assert float(mr.upsample2x_bwd_f32(big, torch.float16)) == float("inf")


def test_zero_stuff_matches_a_strided_transposed_conv():
    g = torch.Generator().manual_seed(6)
    x = torch.randn(2, 4, 3, 5, generator=g, dtype=torch.float64)
    ref = F.conv_transpose2d(x, torch.ones(4, 1, 1, 1, dtype=torch.float64), stride=2, output_padding=1, groups=4)
    assert torch.equal(mr.zero_stuff2x(x), ref)
    z = mr.zero_stuff2x(x.half())
    assert z.dtype == torch.float16 and not torch.signbit(z[:, :, 1::2]).any()  # the stuffed zeros are +0


def test_stem_s2d_matches_pixel_unshuffle():
    g = torch.Generator().manual_seed(7)
    img = torch.randint(0, 256, (2, 3, 6, 10), generator=g, dtype=torch.uint8)
    for dtype in (torch.float16, torch.bfloat16):
        got = mr.stem_s2d(img, dtype)
        assert got.shape == (2, 3, 5, 16)
        # pixel_unshuffle puts (c, dy, dx) at channel c*4 + dy*2 + dx; the stem layout is (dy*2 + dx)*3 + c
        pu = F.pixel_unshuffle(img.float() / 255, 2).to(dtype).permute(0, 2, 3, 1)
        for c in range(3):
            for d in range(4):
                assert torch.equal(got[..., d * 3 + c], pu[..., c * 4 + d])
        assert torch.equal(got[..., 12:], torch.zeros_like(got[..., 12:]))
    f = torch.randn(1, 3, 4, 4, generator=g) * 1e5
    assert torch.equal(mr.stem_s2d(f, torch.float16)[0, 0, 0, :12:3], f[0, 0, :2, :2].flatten().half())


def test_nhwc_to_nchw_is_the_index_map():
    x = torch.randn(2, 3, 5, 7)
    y = mr.nhwc_to_nchw(x)
    assert y.shape == (2, 7, 3, 5) and y.is_contiguous()
    for n, c, i, j in ((0, 0, 0, 0), (1, 6, 2, 4), (1, 3, 1, 0)):
        assert float(y[n, c, i, j]) == float(x[n, i, j, c])


# ---- argument checks of the forward-path ABI: views the kernels access as 16-byte vectors ----
# Fake device addresses: the checks must refuse these before any launch.  Skipped on a machine with a GPU, so that a
# regressed check can never turn into a misaligned launch there.
_A, _MIS = 1 << 20, (1 << 20) + 2  # 16-byte aligned / 2-byte aligned fake pointers
_no_gpu = pytest.mark.skipif(torch.cuda.is_available(), reason="fake-pointer refusals run only without a GPU")


def _refused(rc, lib, what=b"aligned"):
    return rc == -1 and what in lib.y5_last_error()  # Y5_E_INVALID


@_no_gpu
def test_sppf_pool_refuses_misaligned_or_narrow_views(built_lib):
    lib, f16 = built_lib, _lib.Y5_F16
    ok = (_A, 16, _A, _A, _A, 64, 1, 4, 4, 16, 5, f16, None)
    for i in (0, 2, 3, 4):  # x, y1, y2, y3
        args = list(ok)
        args[i] = _MIS
        assert _refused(lib.y5_sppf_pool(*args), lib), i
    assert _refused(lib.y5_sppf_pool(_A, 8, _A, _A, _A, 64, 1, 4, 4, 16, 5, f16, None), lib, b"pitch")  # x pitch < c
    assert _refused(lib.y5_sppf_pool(_A, 16, _A, _A, _A, 8, 1, 4, 4, 16, 5, f16, None), lib, b"pitch")  # y pitch < c


@_no_gpu
def test_upsample2x_and_copy_view_refuse_misaligned_or_narrow_views(built_lib):
    lib, f16 = built_lib, _lib.Y5_BF16
    assert _refused(lib.y5_upsample2x(_MIS, 16, _A, 16, 1, 4, 4, 16, f16, None), lib)
    assert _refused(lib.y5_upsample2x(_A, 16, _MIS, 16, 1, 4, 4, 16, f16, None), lib)
    assert _refused(lib.y5_upsample2x(_A, 8, _A, 16, 1, 4, 4, 16, f16, None), lib, b"pitch")
    assert _refused(lib.y5_upsample2x(_A, 16, _A, 8, 1, 4, 4, 16, f16, None), lib, b"pitch")
    assert _refused(lib.y5_copy_view(_MIS, 16, _A, 16, 16, 16, f16, None), lib)
    assert _refused(lib.y5_copy_view(_A, 16, _MIS, 16, 16, 16, f16, None), lib)
    assert _refused(lib.y5_copy_view(_A, 8, _A, 16, 16, 16, f16, None), lib, b"pitch")
    assert _refused(lib.y5_copy_view(_A, 16, _A, 8, 16, 16, f16, None), lib, b"pitch")


@_no_gpu
def test_stem_s2d_refuses_a_misaligned_output(built_lib):
    lib = built_lib
    for img_dt in (_lib.Y5_U8, _lib.Y5_F16, _lib.Y5_F32):
        assert _refused(lib.y5_stem_s2d(_A, img_dt, _MIS, _lib.Y5_F16, 1, 4, 4, 4, 1, None), lib)
        assert _refused(lib.y5_stem_s2d(_A, img_dt, _A + 8, _lib.Y5_BF16, 1, 4, 4, 0, 0, None), lib)
