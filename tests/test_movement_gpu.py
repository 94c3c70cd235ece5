"""-m gpu: the data-movement kernels bit for bit against tests/movement_ref.py at the shapes YOLOv5 runs and at the edges
of each launch rule: SPPF pooling (both kernels) and its backward, 2x upsample and its backward, strided view copy, zero
stuffing, stem space-to-depth and the NHWC -> NCHW export, then the autograd wrappers and one engine SPPF layer.

Every view sits in a buffer pre-filled with a sentinel bit pattern, at channel offset 8 with its pitch wider than its
channels where the case says so, and with guard elements after the buffer's end: whatever a kernel must not write must
still hold the sentinel afterwards.  Pure moves take every 16-bit pattern as input and are compared as int16, so NaN
payloads, subnormals and -0 must survive.  All of these operations are exact (copies, max, one rounding of a short fp32
sum), so nothing here has a tolerance except the random-data SPPF backward, whose bound is derived below."""
import ctypes as C
import math

import pytest
import torch

from oracle import model_ref
from tests import movement_ref as mr
from tests.conv_exact_ref import ulp
from yolov5_b200 import _lib, train_ops

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
SENT = 0x5A5A  # sentinel bit pattern of every byte a kernel must leave alone
GUARD = 4096  # sentinel elements after the end of every buffer
U = 2.0 ** -24  # fp32 unit roundoff


class Buf:
    """A (B, H, W, c) NHWC view at channel `off` of rows `off + c + extra` wide, in a sentinel-filled int16 buffer followed
    by GUARD sentinel elements.  `off` and `extra` are multiples of 8, so the view stays 16-byte aligned."""

    def __init__(self, dev, B, H, W, c, off=0, extra=0):
        self.shape, self.off, self.c, self.pitch = (B, H, W, c), off, c, off + c + extra
        self.n = B * H * W * self.pitch
        self.raw = torch.full((self.n + GUARD,), SENT, dtype=torch.int16, device=dev)
        self.rows = self.raw[: self.n].view(B, H, W, self.pitch)
        self.ptr = self.raw.data_ptr() + 2 * off

    @classmethod
    def pitched(cls, dev, B, H, W, c, pitched):
        return cls(dev, B, H, W, c, 8, 8) if pitched else cls(dev, B, H, W, c)

    def bits(self, c0=0, c1=None):
        """int16 (B, H, W, c1 - c0) of view channels [c0, c1)"""
        return self.rows[..., self.off + c0 : self.off + (self.c if c1 is None else c1)]

    def nchw(self, dtype, c0=0, c1=None):
        return self.bits(c0, c1).view(dtype).permute(0, 3, 1, 2)

    def fill(self, x_nchw, c0=0):
        self.bits(c0, c0 + x_nchw.shape[1]).copy_(x_nchw.permute(0, 2, 3, 1).contiguous().view(torch.int16))

    def intact_outside(self, c0=0, c1=None):
        """the sentinel survives everywhere except view channels [c0, c1)"""
        r = self.raw.clone()
        r[: self.n].view(self.rows.shape)[..., self.off + c0 : self.off + (self.c if c1 is None else c1)] = SENT
        return bool((r == SENT).all())


def _st(dev):
    return C.c_void_p(_lib.stream_ptr(dev))


def _code(dtype):
    return _lib.dtype_code(dtype)


def _same_values(got, ref):
    """value equality with NaN positions compared (payloads not).  -0 == +0 here: the engine's max ranks +0 above -0,
    torch keeps the first zero of a window, and only the sign of a zero maximum may differ."""
    got, ref = got.double(), ref.double()
    return torch.equal(got.isnan(), ref.isnan()) and bool(((got == ref) | ref.isnan()).all())


def _levels(shape, levels, seed, dtype):
    g = torch.Generator().manual_seed(seed)
    return ((torch.randint(0, levels, shape, generator=g).float() - levels / 2) / 4).to(dtype)


def _plant_nan(x, frac, seed):
    g = torch.Generator().manual_seed(seed)
    x = x.clone()
    x[torch.rand(x.shape, generator=g) < frac] = float("nan")
    x.view(-1)[0] = float("nan")
    return x


def _full_range(shape, dtype, seed):
    """every non-NaN 16-bit pattern (both infinities, -0, subnormals); NaN patterns replaced by -inf / -0 / +inf"""
    x = mr.bit_patterns(shape, dtype, seed)
    nan = x.isnan()
    fill = torch.tensor([-float("inf"), -0.0, float("inf")], dtype=dtype)[torch.arange(x.numel()).view(shape) % 3]
    return torch.where(nan, fill, x)


# ---------------------------------------------------------------------------------------------------------------------
# launch rules (aux_kernels.cu / train_kernels.cu) and the case lists they are checked against
# ---------------------------------------------------------------------------------------------------------------------
def sppf_path(H, W):
    """y5_sppf_pool: the shared-memory kernel when both planes of one 8-channel vector fit in 96 KB, else the direct one"""
    return "smem" if 2 * H * W * 16 <= 96 * 1024 else "direct"


def grid_passes(items, threads, sm):
    """passes of a grid-stride loop whose grid is capped at sm_count * 16 blocks"""
    blocks = min(-(-items // threads), sm * 16)
    return -(-items // (blocks * threads))


# (B, c, H, W, k, pitched input, pitched output)
SPPF_FWD = [
    (32, 256, 20, 20, 5, False, True),  # config2
    (64, 512, 20, 20, 5, True, True),  # config3
    (16, 384, 20, 20, 5, False, True),  # yolov5m training
    (2, 640, 40, 40, 5, True, False),  # config5
    (2, 16, 1, 1, 5, True, True), (2, 16, 2, 2, 5, False, True), (3, 16, 3, 5, 5, True, True),
    (1, 16, 1, 3073, 5, True, True),  # one pixel past the shared-memory limit: direct kernel
    (1, 16, 48, 64, 5, True, True),  # 3072 pixels: the largest shared-memory plane
    (2, 32, 56, 56, 5, False, True), (2, 64, 60, 60, 5, True, True),  # direct kernel
    (4, 32, 15, 20, 5, True, True),  # rect batch
    (2, 16, 11, 13, 3, True, True), (2, 16, 11, 13, 7, True, True),  # k = 3 / 7, shared-memory kernel
    (1, 16, 60, 60, 3, True, True), (1, 16, 60, 60, 7, True, True),  # k = 3 / 7, direct kernel
    (2, 512, 60, 60, 5, True, True),  # direct kernel, more than one grid-stride pass
]
# (B, c, H, W, k) with cat, dcat and da pitched
SPPF_BWD = [(16, 384, 20, 20, 5), (32, 256, 20, 20, 5), (2, 16, 1, 1, 5), (3, 16, 3, 5, 5), (4, 32, 15, 20, 5), (1, 32, 60, 60, 5),
            (2, 16, 11, 13, 3), (2, 16, 11, 13, 7)]
# (B, c, H, W) input, pitched input, output at slice 0 of a concat twice as wide
UPSAMPLE = [(2, 256, 20, 20, False, True), (2, 128, 40, 40, True, True), (16, 384, 20, 20, False, True), (4, 192, 40, 40, True, True),
            (2, 512, 20, 20, True, False), (2, 256, 40, 40, False, True), (2, 320, 160, 160, False, False), (1, 8, 1, 1, True, True),
            (3, 16, 3, 5, True, True)]
# (B, c, H, W) of dx, dy pitched, dx pitched
UPSAMPLE_BWD = [(2, 256, 20, 20, True, False), (4, 128, 40, 40, False, False), (16, 384, 20, 20, True, False), (16, 192, 40, 40, False, True),
                (2, 512, 20, 20, True, True), (2, 256, 40, 40, False, False), (1, 8, 1, 1, True, True), (3, 16, 3, 5, True, True)]
# (pixels, c, x (off, extra), y (off, extra))
COPY_VIEW = [(16 * 40 * 40, 384, (0, 0), (0, 384)), (16 * 40 * 40, 384, (192, 8), (384, 0)), (2 * 20 * 20, 256, (8, 8), (256, 512)),
             (7, 8, (8, 8), (8, 8)), (1, 16, (0, 0), (0, 0))]
# (B, c, h, w) of dy (yolov5m at 640, batch 16), dy as (off, extra) inside the concat gradient, z pitched
ZERO_STUFF = [(16, 96, 160, 160, (0, 0), False), (16, 192, 80, 80, (0, 0), True), (16, 384, 40, 40, (0, 0), False),
              (16, 768, 20, 20, (0, 0), False), (16, 192, 40, 40, (0, 192), False), (16, 384, 20, 20, (0, 384), True),
              (2, 8, 1, 1, (8, 8), True), (3, 16, 3, 5, (8, 8), False)]
# (B, C, H, W), input pitched
NHWC_TO_NCHW = [(2, 8, 7, 9, True), (2, 40, 7, 9, False), (1, 255, 7, 9, True), (2, 8, 20, 20, False), (2, 40, 20, 20, True),
                (2, 255, 20, 20, True), (2, 32, 320, 320, False)]
# (B, H, W) image; the output rows are W/2 + 2 cells with the image at x_off = 1 unless `dense`
STEM = [(2, 6, 10, False), (1, 384, 640, False), (8, 640, 640, False), (2, 64, 96, True)]


# ---------------------------------------------------------------------------------------------------------------------
# pure moves
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,c,H,W,pin,pout", UPSAMPLE)
@pytest.mark.parametrize("dtype", DTYPES)
def test_upsample2x_moves_every_bit(cuda, B, c, H, W, pin, pout, dtype):
    x = mr.bit_patterns((B, c, H, W), dtype, seed=B + c + H)
    xb = Buf.pitched(cuda, B, H, W, c, pin)
    xb.fill(x.to(cuda))
    yb = Buf(cuda, B, 2 * H, 2 * W, 2 * c, 0, 0) if pout else Buf(cuda, B, 2 * H, 2 * W, c)
    _lib.check(_lib.lib().y5_upsample2x(xb.ptr, xb.pitch, yb.ptr, yb.pitch, B, H, W, c, _code(dtype), _st(cuda)), "upsample2x")
    torch.cuda.synchronize()
    assert torch.equal(yb.bits(0, c), mr.upsample2x(x.view(torch.int16).to(cuda)).permute(0, 2, 3, 1))
    assert yb.intact_outside(0, c) and xb.intact_outside()  # the concat's other slice, the guard and the input


@pytest.mark.parametrize("pixels,c,xo,yo", COPY_VIEW)
@pytest.mark.parametrize("dtype", DTYPES)
def test_copy_view_moves_every_bit(cuda, pixels, c, xo, yo, dtype):
    x = mr.bit_patterns((1, c, 1, pixels), dtype, seed=pixels + c)
    xb, yb = Buf(cuda, 1, 1, pixels, c, *xo), Buf(cuda, 1, 1, pixels, c, *yo)
    xb.fill(x.to(cuda))
    _lib.check(_lib.lib().y5_copy_view(xb.ptr, xb.pitch, yb.ptr, yb.pitch, pixels, c, _code(dtype), _st(cuda)), "copy_view")
    torch.cuda.synchronize()
    assert torch.equal(yb.bits(), xb.bits())
    assert yb.intact_outside() and xb.intact_outside()


@pytest.mark.parametrize("B,c,h,w,dyv,pout", ZERO_STUFF)
@pytest.mark.parametrize("dtype", DTYPES)
def test_zero_stuff2x_moves_every_bit(cuda, B, c, h, w, dyv, pout, dtype):
    x = mr.bit_patterns((B, c, h, w), dtype, seed=c + h)
    xb = Buf(cuda, B, h, w, c, *dyv)
    xb.fill(x.to(cuda))
    zb = Buf.pitched(cuda, B, 2 * h, 2 * w, c, pout)
    _lib.check(_lib.lib().y5_zero_stuff2x(xb.ptr, xb.pitch, zb.ptr, zb.pitch, B, h, w, c, _code(dtype), _st(cuda)), "zero_stuff2x")
    torch.cuda.synchronize()
    assert torch.equal(zb.bits(), mr.zero_stuff2x(x.view(torch.int16).to(cuda)).permute(0, 2, 3, 1))
    assert zb.intact_outside() and xb.intact_outside()


@pytest.mark.parametrize("B,c,H,W,pin", NHWC_TO_NCHW)
@pytest.mark.parametrize("dtype", DTYPES)
def test_nhwc_to_nchw_moves_every_bit(cuda, B, c, H, W, pin, dtype):
    x = mr.bit_patterns((B, c, H, W), dtype, seed=c + H)
    xb = Buf.pitched(cuda, B, H, W, c, pin)
    xb.fill(x.to(cuda))
    n = B * c * H * W
    out = torch.full((n + GUARD,), SENT, dtype=torch.int16, device=cuda)
    _lib.check(_lib.lib().y5_nhwc_to_nchw(xb.ptr, xb.pitch, out.data_ptr(), B, H, W, c, _code(dtype), _st(cuda)), "nhwc_to_nchw")
    torch.cuda.synchronize()
    assert torch.equal(out[:n].view(B, c, H, W), mr.nhwc_to_nchw(xb.bits()))
    assert bool((out[n:] == SENT).all()) and xb.intact_outside()


def _stem_input(B, H, W, img_dtype, seed):
    g = torch.Generator().manual_seed(seed)
    if img_dtype == torch.uint8:
        return torch.randint(0, 256, (B, 3, H, W), generator=g, dtype=torch.uint8)
    if img_dtype == torch.float32:  # half every float32 bit pattern (NaN, inf, subnormals), half values spread over the 16-bit range
        bits = torch.randint(-2 ** 31, 2 ** 31, (B, 3, H, W), generator=g, dtype=torch.int64).to(torch.int32).view(torch.float32)
        spread = torch.randn(B, 3, H, W, generator=g) * torch.exp2(torch.randint(-30, 30, (B, 3, H, W), generator=g).float())
        return torch.where(torch.rand(B, 3, H, W, generator=g) < 0.5, bits, spread)
    return mr.bit_patterns((B, 3, H, W), img_dtype, seed)


@pytest.mark.parametrize("B,H,W,dense", STEM)
@pytest.mark.parametrize("img_dtype", [torch.uint8, torch.float16, torch.bfloat16, torch.float32])
@pytest.mark.parametrize("dtype", DTYPES)
def test_stem_s2d_rounds_like_the_reference(cuda, B, H, W, dense, img_dtype, dtype):
    img = _stem_input(B, H, W, img_dtype, seed=H + W + B)
    img_d = img.to(cuda)
    row, x_off = (W // 2, 0) if dense else (W // 2 + 2, 1)  # the engine's rows: one zero cell at each end
    ob = Buf(cuda, B, H // 2, row, 16)
    _lib.check(_lib.lib().y5_stem_s2d(img_d.data_ptr(), _code(img_dtype), ob.ptr, _code(dtype), B, H, W, row, x_off, _st(cuda)), "stem_s2d")
    torch.cuda.synchronize()
    ref = mr.stem_s2d(img_d, dtype)
    got = ob.rows[:, :, x_off : x_off + W // 2]
    nan = ref.isnan()
    assert torch.equal(got.view(dtype).isnan(), nan)  # NaN positions; payloads may differ
    assert torch.equal(torch.where(nan, 0, got), torch.where(nan, 0, ref.view(torch.int16)))
    border = ob.raw.clone()
    border[: ob.n].view(ob.rows.shape)[:, :, x_off : x_off + W // 2] = SENT
    assert bool((border == SENT).all())  # border cells and the guard untouched


# ---------------------------------------------------------------------------------------------------------------------
# SPPF forward through the ABI: y1..y3 into slices 1..3 of a concat buffer whose slice 0 must stay untouched
# ---------------------------------------------------------------------------------------------------------------------
def _sppf_input(kind, shape, dtype, seed):
    if kind == "levels":  # 4 levels: ties in every window
        return _levels(shape, 4, seed, dtype)
    if kind == "full":
        return _full_range(shape, dtype, seed)
    return _plant_nan(_levels(shape, 8, seed, dtype), 2e-3, seed)  # "nan": sparse NaNs on few-level data


def _run_sppf_fwd(dev, x, k, pin, pout, dtype):
    B, c, H, W = x.shape
    xb = Buf.pitched(dev, B, H, W, c, pin)
    xb.fill(x.to(dev))
    cb = Buf(dev, B, H, W, 4 * c, 8, 8) if pout else Buf(dev, B, H, W, 4 * c)
    _lib.check(_lib.lib().y5_sppf_pool(xb.ptr, xb.pitch, cb.ptr + 2 * c, cb.ptr + 4 * c, cb.ptr + 6 * c, cb.pitch, B, H, W, c, k, _code(dtype),
                                       _st(dev)), "sppf_pool")
    torch.cuda.synchronize()
    return xb, cb


@pytest.mark.parametrize("B,c,H,W,k,pin,pout", SPPF_FWD)
@pytest.mark.parametrize("kind", ["levels", "full", "nan"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_sppf_pool_matches_max_pool2d(cuda, B, c, H, W, k, pin, pout, kind, dtype):
    x = _sppf_input(kind, (B, c, H, W), dtype, seed=c + H + W + k)
    xb, cb = _run_sppf_fwd(cuda, x, k, pin, pout, dtype)
    refs = mr.sppf_fwd(x.to(cuda), k)
    for i, ref in enumerate(refs):
        assert _same_values(cb.nchw(dtype, (i + 1) * c, (i + 2) * c), ref), (f"y{i + 1}", sppf_path(H, W))
    if kind == "nan":
        assert bool(refs[2].isnan().any()) and not bool(refs[2].isnan().all())
    assert cb.intact_outside(c, 4 * c) and xb.intact_outside()  # slice 0 (the copy of x) is not the pool's to write


# ---------------------------------------------------------------------------------------------------------------------
# SPPF backward through the ABI
# ---------------------------------------------------------------------------------------------------------------------
# Bound for random dcat.  da = round(acc0), where in fp32
#   acc2 = dcat2 + (dcat3 routed through y2's windows),  acc1 = dcat1 + (acc2 routed through y1's),  acc0 = dcat0 + (acc1 routed through a's)
# Each position is the arg-max of at most k*k windows, so each accumulator is a sum of at most 1 + k*k terms added in any
# order by atomics: at most k*k additions.  A leaf of the float64 reference reaches acc0 through at most 3*k*k additions, so
#   |acc0 - ref| <= gamma(3k^2) * sum|leaves| <= (3k^2 + 1) * 2^-24 * ref_abs     (gamma(n) = n u / (1 - n u) < (n + 1) u here)
# with ref_abs the same routing applied to |dcat| (routing is linear with nonnegative weights), and the final rounding adds
# half an ulp of the result.
def _bwd_bound_k(k):
    return 3 * k * k + 1


def _run_sppf_bwd(dev, a, dcat, k, dtype):
    B, c, H, W = a.shape
    ab = Buf(dev, B, H, W, c, 8, 8)
    ab.fill(a.to(dev))
    cb = Buf(dev, B, H, W, 4 * c, 8, 16)  # cat and dcat pitches above 4c
    cb.fill(a.to(dev))  # slice 0 of the concat holds a, as the SPPF layer's copy puts it there
    _lib.check(_lib.lib().y5_sppf_pool(ab.ptr, ab.pitch, cb.ptr + 2 * c, cb.ptr + 4 * c, cb.ptr + 6 * c, cb.pitch, B, H, W, c, k, _code(dtype),
                                       _st(dev)), "sppf_pool")
    gb = Buf(dev, B, H, W, 4 * c, 8, 8)
    gb.fill(dcat.to(dev))
    db = Buf(dev, B, H, W, c, 8, 8)  # da as a channel slice
    ws = torch.empty(_lib.lib().y5_sppf_bwd_workspace_bytes(B, H, W, c) // 4, dtype=torch.float32, device=dev)
    _lib.check(_lib.lib().y5_sppf_pool_bwd(cb.ptr, cb.pitch, gb.ptr, gb.pitch, db.ptr, db.pitch, B, H, W, c, k, _code(dtype), ws.data_ptr(),
                                           _st(dev)), "sppf_pool_bwd")
    torch.cuda.synchronize()
    assert db.intact_outside() and gb.intact_outside() and cb.intact_outside()
    return db.nchw(dtype).double()


@pytest.mark.parametrize("B,c,H,W,k", SPPF_BWD)
@pytest.mark.parametrize("kind", ["int", "nan", "rand"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_sppf_pool_bwd_matches_float64_autograd(cuda, B, c, H, W, k, kind, dtype):
    seed = c + H + W + k
    g = torch.Generator().manual_seed(seed)
    if kind == "rand":
        a = (torch.rand(B, c, H, W, generator=g) * 2 - 1).to(dtype)
        dcat = (torch.rand(B, 4 * c, H, W, generator=g) * 2 - 1).to(dtype)
    else:  # few-level input (ties everywhere), small-integer gradients: every fp32 partial sum and the result are exact
        a = _levels((B, c, H, W), 4, seed, dtype)
        if kind == "nan":
            a = _plant_nan(a, 5e-3, seed)
        m = 8 if dtype == torch.float16 else 2
        dcat = torch.randint(-m, m + 1, (B, 4 * c, H, W), generator=g).to(dtype)
    got = _run_sppf_bwd(cuda, a, dcat, k, dtype)
    ref = mr.sppf_bwd(a.to(cuda), dcat.to(cuda), k)
    if kind == "rand":
        ref_abs = mr.sppf_bwd(a.to(cuda), dcat.to(cuda).abs(), k)
        bound = 0.5 * ulp(got, dtype) + _bwd_bound_k(k) * U * ref_abs
        assert bool(((got - ref).abs() <= bound).all()), float(((got - ref).abs() - bound).max())
    else:
        exact = 2048 if dtype == torch.float16 else 256  # largest integer range the dtype holds exactly
        assert float(ref.abs().max()) <= exact
        assert torch.equal(got, ref)


# ---------------------------------------------------------------------------------------------------------------------
# upsample backward
# ---------------------------------------------------------------------------------------------------------------------
def _run_upsample_bwd(dev, dy, pin, pout, dtype):
    B, c, H2, W2 = dy.shape
    gb = Buf(dev, B, H2, W2, 2 * c, 8, 8) if pin else Buf(dev, B, H2, W2, c)  # dy as a slice of a concat gradient
    gb.fill(dy.to(dev))
    db = Buf.pitched(dev, B, H2 // 2, W2 // 2, c, pout)
    _lib.check(_lib.lib().y5_upsample2x_bwd(gb.ptr, gb.pitch, db.ptr, db.pitch, B, H2 // 2, W2 // 2, c, _code(dtype), _st(dev)),
               "upsample2x_bwd")
    torch.cuda.synchronize()
    assert db.intact_outside() and gb.intact_outside()
    return db.nchw(dtype)


@pytest.mark.parametrize("B,c,H,W,pin,pout", UPSAMPLE_BWD)
@pytest.mark.parametrize("dtype", DTYPES)
def test_upsample2x_bwd_is_one_rounding_of_the_fp32_sum(cuda, B, c, H, W, pin, pout, dtype):
    g = torch.Generator().manual_seed(B + c + H)
    shape = (B, c, 2 * H, 2 * W)
    span = 8 if dtype == torch.float16 else 60  # magnitudes 2^-span .. 2^span: the sums cancel and carry across binades
    dy = (torch.randn(shape, generator=g) * torch.exp2(torch.randint(-span, span, shape, generator=g).float())).to(dtype)
    got = _run_upsample_bwd(cuda, dy, pin, pout, dtype)
    assert torch.equal(got.contiguous().view(torch.int16).cpu(), mr.upsample2x_bwd_f32(dy, dtype).view(torch.int16))
    # within 1 ulp of the rounded float64 sum, plus the error of the three fp32 additions (at most 3u * sum|dy|, zero when
    # the four terms fit in fp32's 24 bits; these magnitudes are spread wider than that, so the sums cancel inexactly)
    r64 = mr.upsample2x_bwd64(dy.to(cuda))
    bound = ulp(torch.maximum(got.double().abs(), r64.abs()), dtype) + 3 * U * mr.upsample2x_bwd64(dy.to(cuda).abs())
    assert bool(((got.double() - r64.to(dtype).double()).abs() <= bound).all())


def test_upsample2x_bwd_overflows_to_inf_like_torch(cuda):
    dtype = torch.float16
    g = torch.Generator().manual_seed(9)
    shape = (2, 16, 6, 10)
    mag = 60000 + torch.rand(shape, generator=g) * 5504  # near 65504: a 2x2 sum of four overflows unless signs cancel
    sign = torch.where(torch.rand(shape, generator=g) < 0.2, -1.0, 1.0)
    dy = (mag * sign).to(dtype)
    got = _run_upsample_bwd(cuda, dy, True, False, dtype)
    emu = mr.upsample2x_bwd_f32(dy, dtype)
    assert torch.equal(got.contiguous().view(torch.int16).cpu(), emu.view(torch.int16))
    x = torch.zeros(2, 16, 3, 5, dtype=dtype, device=cuda, requires_grad=True)
    torch.nn.functional.interpolate(x, scale_factor=2.0, mode="nearest").backward(dy.to(cuda))
    assert bool(got.isinf().any()) and bool(torch.isfinite(got).any())
    assert torch.equal(got.isinf(), x.grad.isinf()) and torch.equal(got[got.isinf()], x.grad[got.isinf()])


# ---------------------------------------------------------------------------------------------------------------------
# autograd wrappers: the upstream gradient as a channel slice of a wider channels_last buffer (what _Concat.backward hands
# out, read in place) and as a dense NCHW tensor (copied to channels_last first)
# ---------------------------------------------------------------------------------------------------------------------
def _as_grad(g, form):
    if form == "dense":
        return g.contiguous()
    b, c, h, w = g.shape
    wide = torch.zeros(b, c + 16, h, w, dtype=g.dtype, device=g.device).contiguous(memory_format=torch.channels_last)
    wide[:, 8 : 8 + c] = g
    return wide[:, 8 : 8 + c]


@pytest.mark.parametrize("form", ["slice", "dense"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_sppf_pool_cat_autograd(cuda, form, dtype):
    B, c, H, W, k = 2, 32, 20, 20, 5
    seed = 21
    a0 = _plant_nan(_levels((B, c, H, W), 4, seed, dtype), 5e-3, seed)
    a = a0.to(cuda).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    cat = train_ops._SppfPoolCat.apply(a, k)
    assert torch.equal(cat[:, :c].contiguous().view(torch.int16), a0.to(cuda).view(torch.int16))  # slice 0: a bit copy
    for i, ref in enumerate(mr.sppf_fwd(a0.to(cuda), k)):
        assert _same_values(cat[:, (i + 1) * c : (i + 2) * c], ref), f"y{i + 1}"
    g = torch.Generator().manual_seed(seed)
    m = 8 if dtype == torch.float16 else 2  # |da| stays exactly representable (see test_sppf_pool_bwd_matches_float64_autograd)
    dcat = torch.randint(-m, m + 1, (B, 4 * c, H, W), generator=g).to(dtype).to(cuda)
    (da,) = torch.autograd.grad(cat, a, _as_grad(dcat, form))
    assert torch.equal(da.double(), mr.sppf_bwd(a0.to(cuda), dcat, k))


@pytest.mark.parametrize("form", ["slice", "dense"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_upsample2x_autograd(cuda, form, dtype):
    x0 = mr.bit_patterns((2, 32, 6, 10), dtype, seed=11)
    x = x0.to(cuda).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    y = train_ops._Upsample2x.apply(x)
    assert torch.equal(y.contiguous().view(torch.int16), mr.upsample2x(x0.view(torch.int16)).to(cuda))
    g = torch.Generator().manual_seed(12)
    dy = (torch.randn(2, 32, 12, 20, generator=g) * 4).to(dtype)
    (dx,) = torch.autograd.grad(y, x, _as_grad(dy.to(cuda), form))
    assert torch.equal(dx.contiguous().view(torch.int16).cpu(), mr.upsample2x_bwd_f32(dy, dtype).view(torch.int16))


@pytest.mark.parametrize("dtype", DTYPES)
def test_concat_autograd(cuda, dtype):
    a0, b0 = mr.bit_patterns((2, 16, 5, 7), dtype, seed=13), mr.bit_patterns((2, 40, 5, 7), dtype, seed=14)
    a = _as_grad(a0.to(cuda), "slice").detach().requires_grad_(True)  # a channel-slice input
    b = b0.to(cuda).requires_grad_(True)  # a dense NCHW input
    c = train_ops._Concat.apply(a, b)
    assert torch.equal(c.contiguous().view(torch.int16), torch.cat((a0, b0), 1).view(torch.int16).to(cuda))
    gc = mr.bit_patterns(tuple(c.shape), dtype, seed=15).to(cuda)
    da, db = torch.autograd.grad(c, (a, b), gc)
    assert torch.equal(da.contiguous().view(torch.int16), gc[:, :16].contiguous().view(torch.int16))
    assert torch.equal(db.contiguous().view(torch.int16), gc[:, 16:].contiguous().view(torch.int16))


# ---------------------------------------------------------------------------------------------------------------------
# engine: an eval SPPF layer whose input holds NaNs gives NaN wherever the reference does
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [20, 60])  # shared-memory kernel / direct kernel
@pytest.mark.parametrize("dtype", DTYPES)
def test_engine_sppf_layer_propagates_nan(cuda, H, dtype):
    from yolov5_b200.models.common import SPPF

    assert sppf_path(H, H) == ("smem" if H == 20 else "direct")
    torch.manual_seed(0)
    layer = SPPF(64, 64, 5).eval()
    sd = {f"model.0.{k}": v.detach().float() for k, v in layer.state_dict().items()}
    x = (torch.rand(2, 64, H, H) * 2 - 1).to(dtype)
    x[0, 5, 3, 4] = x[1, 17, H - 2, H // 2] = float("nan")  # one NaN per image: the reference's NaN covers a 13x13 patch
    with torch.no_grad():
        ref = model_ref.sppf(sd, "model.0", x.float(), 5, False)
    got = layer.to(cuda, dtype)(x.to(cuda)).float().cpu()
    assert torch.equal(got.isnan(), ref.isnan()), (int(got.isnan().sum()), int(ref.isnan().sum()))
    fin = ~ref.isnan()
    tol = 3e-3 if dtype == torch.float16 else 2.5e-2  # test_single_layers_vs_oracle's tolerance
    assert float((got[fin] - ref[fin]).abs().max() / ref[fin].abs().max()) < tol


# ---------------------------------------------------------------------------------------------------------------------
def test_case_list_covers_every_path(cuda):
    """Both SPPF kernels run, every grid-stride kernel makes more than one pass in at least one case, and every ABI sees at
    least one pitched input and one pitched output."""
    sm = torch.cuda.get_device_properties(cuda).multi_processor_count
    paths = {sppf_path(H, W) for _, _, H, W, *_ in SPPF_FWD}
    assert paths == {"smem", "direct"}
    for kern in ("smem", "direct"):
        assert {k for _, _, H, W, k, _, _ in SPPF_FWD if sppf_path(H, W) == kern} >= {3, 7}, kern
    passes = {
        "sppf_pool (direct)": max(grid_passes(B * H * W * c // 8, 128, sm) for B, c, H, W, *_ in SPPF_FWD if sppf_path(H, W) == "direct"),
        "sppf_pool_bwd": max(grid_passes(B * H * W * c, 256, sm) for B, c, H, W, _ in SPPF_BWD),
        "upsample2x": max(grid_passes(B * 4 * H * W * c // 8, 256, sm) for B, c, H, W, *_ in UPSAMPLE),
        "upsample2x_bwd": max(grid_passes(B * H * W * c // 8, 256, sm) for B, c, H, W, *_ in UPSAMPLE_BWD),
        "copy_view": max(grid_passes(p * c // 8, 256, sm) for p, c, *_ in COPY_VIEW),
        "zero_stuff2x": max(grid_passes(B * 4 * h * w * c // 8, 256, sm) for B, c, h, w, *_ in ZERO_STUFF),
        "stem_s2d": max(grid_passes(B * (H // 2) * (W // 2), 256, sm) for B, H, W, _ in STEM),
    }
    assert all(p > 1 for p in passes.values()), passes
    pitched = {
        "sppf_pool": (any(c[5] for c in SPPF_FWD), any(c[6] for c in SPPF_FWD)),
        "sppf_pool_bwd": (True, True),  # _run_sppf_bwd: cat and dcat pitch 4c + 24 / 4c + 16, da a channel slice
        "upsample2x": (any(c[4] for c in UPSAMPLE), any(c[5] for c in UPSAMPLE)),
        "upsample2x_bwd": (any(c[4] for c in UPSAMPLE_BWD), any(c[5] for c in UPSAMPLE_BWD)),
        "copy_view": (any(sum(c[2]) for c in COPY_VIEW), any(sum(c[3]) for c in COPY_VIEW)),
        "zero_stuff2x": (any(sum(c[4]) for c in ZERO_STUFF), any(c[5] for c in ZERO_STUFF)),
        "nhwc_to_nchw": (any(c[4] for c in NHWC_TO_NCHW), True),  # its output is dense NCHW by definition
        "stem_s2d": (True, any(not c[3] for c in STEM)),  # its input is a dense image; the output rows are W/2 + 2 wide
    }
    assert all(i and o for i, o in pitched.values()), pitched
    assert any(math.prod(c[:4]) >= 65536 for c in NHWC_TO_NCHW)  # every 16-bit pattern goes through the export
