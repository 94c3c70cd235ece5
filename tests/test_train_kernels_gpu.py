"""-m gpu kernel-level tests of the training path at the shapes YOLOv5 trains with: weight gradient, data gradient, the
space-to-depth stem, weight packing, the BatchNorm / SiLU passes, the Detect head's 1x1 conv and the side-stream weight
gradients.

Exact arithmetic: the GEMM-like kernels are fed integer-valued operands in {-2..2} with every partial sum below 2^24, so
every fp32 accumulation is exact in any order.  The fp32 weight gradient must then equal the float64 reference bit for
bit, and a convolution or data gradient (one rounding of an exact sum) must equal `ref.float().to(dtype)` bit for bit.  A
relative tolerance could not see one missing 64-pixel block among a million pixels; exact data can.  One random-data case
per kernel keeps the rounding behaviour covered with the usual tolerances.

References are plain float64 torch on the GPU."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from yolov5_b200 import _lib, train_ops
from yolov5_b200.models.common import Conv

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]


# ---------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------
def _ints(shape, seed, dev, lo=-2, hi=2):
    """integer-valued fp32 tensor with entries in [lo, hi] (exact in fp16 and bf16)"""
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randint(lo, hi + 1, shape, generator=g, device=dev, dtype=torch.float32)


def _cl(t, dtype):
    return t.to(dtype).contiguous(memory_format=torch.channels_last)


def _st(dev):
    return C.c_void_p(_lib.stream_ptr(dev))


def _integral(ref, what):
    """the float64 reference of integer data is integral; round away whatever the reference algorithm left behind"""
    r = ref.round()
    assert float((ref - r).abs().max()) < 1e-3, (what, "float64 reference is not integral")
    return r


def _assert_exact(got, ref, what, names=None):
    """bit-exact comparison; on failure report how many elements differ and where (index tuples named by `names`)"""
    got, ref = got.double(), ref.double()
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    bad = got != ref
    n = int(bad.sum())
    if n:
        idx = bad.nonzero()[:6].tolist()
        detail = [(dict(zip(names, i)) if names else i, float(got[tuple(i)]), float(ref[tuple(i)])) for i in idx]
        pytest.fail(f"{what}: {n} of {got.numel()} elements differ, first {detail}")


def _rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _sms(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def _wgrad_plan(cin, cout, taps, m, sms):
    """the work split of y5_conv_wgrad (host code of csrc/conv_wgrad.cu), to state which paths a case reaches"""
    blocks = -(-cin // 64)
    nb = min(blocks, 4)
    ci_tiles = -(-blocks // nb)
    nb = -(-blocks // ci_tiles)
    gmax = max(1, 4 // nb)
    tap_groups = -(-taps // gmax)
    group = -(-taps // tap_groups)
    pix = 128 if (2 + group * nb) * 128 * 128 <= 56 * 1024 else 64
    kblocks = -(-m // pix)
    items = -(-cout // 128) * tap_groups * ci_tiles
    want = min(max(1, -(-sms // items)), kblocks)
    kbps = -(-kblocks // want)
    return dict(n_blocks=nb, ci_tiles=ci_tiles, group=group, tap_groups=tap_groups, pix=pix, kblocks=kblocks, kb_per_split=kbps,
                splits=-(-kblocks // kbps))


# ---------------------------------------------------------------------------------------------------------------------
# A. weight gradient
# ---------------------------------------------------------------------------------------------------------------------
# (B, H, W, cin, cout, k, s, p, expected plan: n_blocks, ci_tiles, group, tap_groups, pix)
WGRAD_CASES = [
    (2, 10, 12, 16, 24, 1, 1, 0, (1, 1, 1, 1, 128)),      # 128 pixels per stage, M = 240 not a multiple of it
    (1, 20, 20, 48, 80, 1, 1, 0, (1, 1, 1, 1, 128)),      # K tail in the 64-channel block, 16-channel tail in the upper dY box
    (2, 12, 10, 320, 192, 1, 1, 0, (3, 2, 1, 1, 64)),     # ci tiles 3 + 2, last co tile = one dY box
    (1, 10, 10, 640, 96, 1, 1, 0, (4, 3, 1, 1, 64)),      # ci tiles 4 + 4 + 2
    (1, 8, 10, 1280, 40, 1, 1, 0, (4, 5, 1, 1, 64)),      # ci tiles 4 x 5, Cout 40 < one dY box
    (2, 9, 11, 768, 384, 1, 1, 0, (4, 3, 1, 1, 64)),      # three co tiles
    (2, 11, 13, 40, 48, 3, 1, 1, (1, 1, 3, 3, 64)),       # tap groups 3 + 3 + 3
    (4, 5, 7, 48, 96, 3, 1, 1, (1, 1, 3, 3, 64)),         # 35-pixel images: every 64-pixel stage spans images
    (1, 14, 10, 96, 80, 3, 1, 1, (2, 1, 2, 5, 64)),       # tap groups 2 + 2 + 2 + 2 + 1
    (2, 18, 14, 192, 96, 3, 2, 1, (3, 1, 1, 9, 64)),      # stride 2, tap groups 1 x 9
    (1, 16, 20, 384, 192, 3, 2, 1, (3, 2, 1, 9, 64)),     # stride 2, ci tiles 3 + 3
    (1, 7, 9, 768, 64, 3, 1, 1, (4, 3, 1, 9, 64)),        # n_blocks 4 with 9 taps
    (1, 20, 24, 24, 16, 3, 2, 1, (1, 1, 3, 3, 64)),       # narrowest widths
]


@pytest.mark.parametrize("B,H,W,cin,cout,k,s,p,plan", WGRAD_CASES)
@pytest.mark.parametrize("dtype", DTYPES)
def test_wgrad_exact(cuda, B, H, W, cin, cout, k, s, p, plan, dtype):
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    pl = _wgrad_plan(cin, cout, k * k, B * Ho * Wo, _sms(cuda))
    assert (pl["n_blocks"], pl["ci_tiles"], pl["group"], pl["tap_groups"], pl["pix"]) == plan, pl
    x = _ints((B, cin, H, W), 1, cuda)
    dy = _ints((B, cout, Ho, Wo), 2, cuda)
    got = train_ops.conv_wgrad(_cl(x, dtype), _cl(dy, dtype), k, s, p)
    ref = _integral(torch.nn.grad.conv2d_weight(x.double(), (cout, cin, k, k), dy.double(), stride=s, padding=p), "wgrad")
    _assert_exact(got, ref, f"wgrad {pl}", ("co", "ci", "r", "s"))


@pytest.mark.parametrize("B,H,W,cin,cout,k,s,p", [
    (16, 320, 320, 48, 96, 3, 2, 1),   # yolov5m layer 1 at batch 16 / 640^2: 409 600 output pixels
    (16, 320, 320, 64, 64, 1, 1, 0),   # 1.64 M pixels
])
def test_wgrad_exact_production_size(cuda, B, H, W, cin, cout, k, s, p):
    """Pixel ranges split over about one CTA per SM; the last range is shorter (kb_per_split does not divide kblocks), so a
    dropped or doubled range changes integer results."""
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    m = B * Ho * Wo
    assert m * 4 < 2 ** 24
    pl = _wgrad_plan(cin, cout, k * k, m, _sms(cuda))
    assert pl["splits"] > 1 and pl["kblocks"] % pl["kb_per_split"] != 0, pl
    x = _ints((B, cin, H, W), 3, cuda)
    dy = _ints((B, cout, Ho, Wo), 4, cuda)
    got = train_ops.conv_wgrad(_cl(x, torch.float16), _cl(dy, torch.float16), k, s, p)
    ref = _integral(torch.nn.grad.conv2d_weight(x.double(), (cout, cin, k, k), dy.double(), stride=s, padding=p), "wgrad")
    _assert_exact(got, ref, f"wgrad {pl}", ("co", "ci", "r", "s"))


def _wgrad_raw(x, dy, kh, kw, s, ph, pw, dtype, in_extra=0, out_extra=0, dw_init=None):
    """y5_conv_wgrad on views inside wider NHWC buffers (channel offset 8 and pitch + extra when extra > 0).  Returns the
    [co][r][s][ci] fp32 gradient; `dw_init` pre-fills it and asks for accumulate = 1."""
    lib = _lib.lib()
    dev = x.device
    b, cin, h, w = x.shape
    cout, ho, wo = dy.shape[1:]
    xo, do = (8 if in_extra else 0), (8 if out_extra else 0)
    xb = torch.full((b, h, w, cin + in_extra + xo), 5.0, dtype=dtype, device=dev)
    xb[..., xo : xo + cin] = x.permute(0, 2, 3, 1).to(dtype)
    db = torch.full((b, ho, wo, cout + out_extra + do), -5.0, dtype=dtype, device=dev)
    db[..., do : do + cout] = dy.permute(0, 2, 3, 1).to(dtype)
    dw = dw_init.clone() if dw_init is not None else torch.full((cout, kh, kw, cin), float("nan"), device=dev)
    d = _lib.WgradDesc()
    es = xb.element_size()
    d.inp, d.in_pitch = xb.data_ptr() + xo * es, xb.shape[3]
    d.batch, d.in_h, d.in_w, d.in_c = b, h, w, cin
    d.dout, d.dout_pitch, d.out_c = db.data_ptr() + do * es, db.shape[3], cout
    d.dweight = dw.data_ptr()
    d.ksize, d.kw, d.stride, d.pad, d.pad_w = kh, kw, s, ph, pw
    d.dtype, d.accumulate = _lib.dtype_code(dtype), int(dw_init is not None)
    _lib.check(lib.y5_conv_wgrad(C.byref(d), _st(dev)), "conv_wgrad")
    return dw


@pytest.mark.parametrize("B,H,W,cin,cout,kh,kw,s,ph,pw,in_extra,out_extra,acc", [
    (2, 12, 10, 40, 48, 3, 3, 1, 1, 1, 24, 16, 0),     # both operands are channel slices of wider buffers
    (3, 9, 7, 96, 80, 3, 3, 2, 1, 1, 8, 40, 1),        # slices + accumulate into a pre-filled gradient
    (2, 10, 14, 64, 64, 1, 1, 1, 0, 0, 64, 8, 1),      # plain 2-D tiles on a slice, accumulate
    (2, 11, 9, 48, 96, 3, 1, 1, 1, 0, 0, 0, 0),        # non-square filter 3x1 (kw / pad_w)
    (2, 8, 12, 80, 40, 1, 3, 1, 0, 1, 16, 0, 1),       # 1x3 on a slice, accumulate
    (1, 16, 10, 48, 64, 3, 1, 2, 1, 0, 0, 24, 0),      # 3x1 stride 2
])
@pytest.mark.parametrize("dtype", DTYPES)
def test_wgrad_raw_abi_views_accumulate_nonsquare(cuda, B, H, W, cin, cout, kh, kw, s, ph, pw, in_extra, out_extra, acc, dtype):
    Ho, Wo = (H + 2 * ph - kh) // s + 1, (W + 2 * pw - kw) // s + 1
    x = _ints((B, cin, H, W), 5, cuda)
    dy = _ints((B, cout, Ho, Wo), 6, cuda)
    init = _ints((cout, kh, kw, cin), 7, cuda, -1000, 1000) if acc else None
    got = _wgrad_raw(x, dy, kh, kw, s, ph, pw, dtype, in_extra, out_extra, init)
    ref = _integral(torch.nn.grad.conv2d_weight(x.double(), (cout, cin, kh, kw), dy.double(), stride=s, padding=(ph, pw)), "wgrad")
    ref = ref.permute(0, 2, 3, 1)
    if acc:
        ref = ref + init.double()
    _assert_exact(got, ref, "raw wgrad", ("co", "r", "s", "ci"))


@pytest.mark.parametrize("dtype", DTYPES)
def test_wgrad_random_rounding(cuda, dtype):
    """random data: exact products, fp32 accumulation in an unfixed order"""
    g = torch.Generator(device=cuda).manual_seed(8)
    x = (torch.rand(2, 320, 20, 16, generator=g, device=cuda) * 2 - 1).to(dtype)
    dy = (torch.rand(2, 192, 10, 8, generator=g, device=cuda) * 2 - 1).to(dtype)
    got = train_ops.conv_wgrad(_cl(x, dtype), _cl(dy, dtype), 3, 2, 1)
    ref = torch.nn.grad.conv2d_weight(x.double(), (192, 320, 3, 3), dy.double(), stride=2, padding=1)
    assert float((got.double() - ref).abs().max() / ref.abs().max()) < 2e-5


# ---------------------------------------------------------------------------------------------------------------------
# B. data gradient (and the forward conv it is built from)
# ---------------------------------------------------------------------------------------------------------------------
# (B, H, W, cin, cout, k, s, p): dx has cin channels (the GEMM's N), the reduction runs over k*k*cout (its K)
DGRAD_CASES = [
    (2, 10, 12, 80, 40, 1, 1, 0),       # K = 40: block_k zero fill
    (2, 9, 11, 40, 48, 3, 1, 1),        # K tail 48, N = 40
    (2, 128, 160, 48, 96, 3, 2, 1),     # stride 2, non-square image: zero-stuffing with h != w
    (1, 96, 64, 320, 192, 3, 2, 1),     # stride 2, taller than wide
    (2, 20, 12, 96, 24, 3, 2, 1),       # K = 24
    (1, 12, 10, 1280, 640, 3, 1, 1),    # yolov5x widths
    (1, 8, 8, 384, 1280, 1, 1, 0),      # K = 1280
    (2, 14, 18, 16, 80, 3, 1, 1),       # N = 16
]


@pytest.mark.parametrize("B,H,W,cin,cout,k,s,p", DGRAD_CASES)
@pytest.mark.parametrize("form", ["oihw", "packed", "packed_slice"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_dgrad_exact(cuda, B, H, W, cin, cout, k, s, p, form, dtype):
    """Both call forms: OIHW weights, and the data-gradient packing with block_k exactly as _ConvBnAct hands them over; the
    slice form reads dy in place from a wider concat gradient, as _Concat.backward hands it out."""
    Ho, Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
    w = _ints((cout, cin, k, k), 9, cuda)
    dy = _ints((B, cout, Ho, Wo), 10, cuda)
    if form == "packed_slice":
        wide = _cl(_ints((B, cout + 48, Ho, Wo), 11, cuda), dtype)
        wide[:, 16 : 16 + cout] = dy.to(dtype)
        dyv = wide[:, 16 : 16 + cout]
        assert train_ops._nhwc(dyv)[1] == cout + 48  # read in place through its pitch, not copied
    else:
        dyv = _cl(dy, dtype)
    if form == "oihw":
        got = train_ops.conv_dgrad(dyv, w, k, s, p, (H, W))
    else:
        _, wp_dg, _, bk_d = train_ops.pack_weights(w, dtype, B * Ho * Wo, True, True)
        got = train_ops.conv_dgrad(dyv, None, k, s, p, (H, W), wp_dgrad=wp_dg, cin=cin, block_k=bk_d)
    ref = _integral(torch.nn.grad.conv2d_input((B, cin, H, W), w.double(), dy.double(), stride=s, padding=p), "dgrad")
    _assert_exact(got, ref.float().to(dtype), "dgrad", ("n", "c", "y", "x"))


@pytest.mark.parametrize("B,H,W,cin,cout,k,s,p", DGRAD_CASES)
@pytest.mark.parametrize("dtype", DTYPES)
def test_forward_conv_exact(cuda, B, H, W, cin, cout, k, s, p, dtype):
    x = _ints((B, cin, H, W), 12, cuda)
    w = _ints((cout, cin, k, k), 13, cuda)
    got = train_ops.conv_raw(_cl(x, dtype), w, None, k, s, p)
    ref = _integral(F.conv2d(x.double(), w.double(), stride=s, padding=p), "conv")
    _assert_exact(got, ref.float().to(dtype), "conv", ("n", "c", "y", "x"))


def test_dgrad_stride2_odd_input_is_refused(cuda):
    w = _ints((32, 16, 3, 3), 15, cuda)
    for h, w_ in ((17, 16), (16, 17), (15, 15)):
        dy = _cl(_ints((1, 32, (h - 1) // 2 + 1, (w_ - 1) // 2 + 1), 14, cuda), torch.float16)
        with pytest.raises(NotImplementedError):
            train_ops.conv_dgrad(dy, w, 3, 2, 1, (h, w_))


@pytest.mark.parametrize("dtype", DTYPES)
def test_dgrad_random_rounding(cuda, dtype):
    g = torch.Generator(device=cuda).manual_seed(16)
    w = torch.rand(96, 48, 3, 3, generator=g, device=cuda) - 0.5
    dy = (torch.rand(2, 96, 24, 20, generator=g, device=cuda) * 2 - 1).to(dtype)
    got = train_ops.conv_dgrad(_cl(dy, dtype), w, 3, 2, 1, (48, 40))
    ref = torch.nn.grad.conv2d_input((2, 48, 48, 40), w.to(dtype).double(), dy.double(), stride=2, padding=1)
    tol = 2e-3 if dtype == torch.float16 else 1.6e-2  # one rounding of the result
    assert float((got.double() - ref).abs().max() / ref.abs().max()) < tol


# ---------------------------------------------------------------------------------------------------------------------
# C. the training stem: Conv(3, c, 6, 2, 2) over the space-to-depth image
# ---------------------------------------------------------------------------------------------------------------------
def _s2d(img):
    """(B,3,H,W) -> (B,16,H/2,W/2): channel (dy*2+dx)*3 + c holds pixel (2i+dy, 2j+dx) of colour c, 4 zero channels"""
    b, _, h, w = img.shape
    t = img.reshape(b, 3, h // 2, 2, w // 2, 2).permute(0, 3, 5, 1, 2, 4).reshape(b, 12, h // 2, w // 2)
    return torch.cat((t, t.new_zeros(b, 4, h // 2, w // 2)), 1)


@pytest.mark.parametrize("B,H,W,O,dtype", [
    (2, 64, 96, 32, torch.float16), (2, 64, 96, 32, torch.bfloat16), (1, 40, 40, 48, torch.float16), (1, 40, 40, 48, torch.bfloat16),
    (16, 640, 640, 16, torch.float16),  # 1.64 M output pixels
])
def test_stem_wide_kernels_exact(cuda, monkeypatch, B, H, W, O, dtype):
    """stem_conv_wide / stem_wgrad_wide on integer images: the forward against the 6x6/s2/p2 conv, the gradient in its
    (O,16,3,3) form and, through _stem_index, in the (O,3,6,6) form of the parameter."""
    monkeypatch.setenv("Y5_TRAIN_STEM_WIDE", "1")
    img = _ints((B, 3, H, W), 17, cuda)
    w6 = _ints((O, 3, 6, 6), 18, cuda)
    buf = train_ops.stem_input(img, dtype)
    s2d = _s2d(img)
    assert torch.equal(buf[:, :, 1:-1].permute(0, 3, 1, 2).float(), s2d)  # float images are not scaled
    assert not buf[:, :, 0].any() and not buf[:, :, -1].any()
    fwd_idx, inv_idx = train_ops._stem_index(cuda)
    w3 = torch.cat((w6.flatten(1), w6.new_zeros(O, 1)), 1)[:, fwd_idx].view(O, 16, 3, 3)
    y = train_ops.stem_conv_wide(buf, w3)
    ref = _integral(F.conv2d(img.double(), w6.double(), stride=2, padding=2), "stem conv")
    _assert_exact(y, ref.float().to(dtype), "stem conv", ("n", "c", "y", "x"))
    dy = _ints((B, O, H // 2, W // 2), 19, cuda)
    g3 = train_ops.stem_wgrad_wide(buf, _cl(dy, dtype))
    ref3 = _integral(torch.nn.grad.conv2d_weight(s2d.double(), (O, 16, 3, 3), dy.double(), padding=1), "stem wgrad")
    _assert_exact(g3, ref3, "stem wgrad (O,16,3,3)", ("o", "c", "r", "s"))
    g6 = g3.reshape(O, -1)[:, inv_idx].view(O, 3, 6, 6)
    ref6 = _integral(torch.nn.grad.conv2d_weight(img.double(), (O, 3, 6, 6), dy.double(), stride=2, padding=2), "stem wgrad")
    _assert_exact(g6, ref6, "stem wgrad (O,3,6,6)", ("o", "c", "ky", "kx"))


@pytest.mark.parametrize("c,B,H,W,kind", [
    (16, 2, 64, 64, "uint8"),
    (32, 2, 48, 80, "int"),
    (48, 1, 96, 64, "uint8"),
    (64, 2, 32, 32, "int"),
    (80, 1, 64, 96, "uint8"),
])
@pytest.mark.parametrize("wide", [True, False])
@pytest.mark.parametrize("dtype", DTYPES)
def test_stem_layer_train(cuda, monkeypatch, c, B, H, W, kind, wide, dtype):
    """The stem layer in training (both stem forms): output, the (O,3,6,6) weight gradient, dgamma and dbeta against float64
    autograd of silu(batch_norm(conv2d(img, w, stride=2, padding=2)))."""
    monkeypatch.setenv("Y5_TRAIN_STEM_WIDE", "1" if wide else "0")
    torch.manual_seed(c)
    m = Conv(3, c, 6, 2, 2).to(cuda)
    m.bn.eps, m.bn.momentum = 1e-3, 0.03
    with torch.no_grad():
        m.bn.weight.uniform_(0.5, 1.5)
        m.bn.bias.uniform_(-0.5, 0.5)
    m.train()
    if kind == "uint8":
        img = _ints((B, 3, H, W), 20, cuda, 0, 255).to(torch.uint8)
        xr = (img.float() / 255).to(dtype).double()
    else:
        img = _ints((B, 3, H, W), 20, cuda, 0, 3)
        xr = img.to(dtype).double()
    with torch.autocast("cuda", enabled=False):
        z = train_ops.conv_module(m, train_ops.stem_input(img, dtype), stem=2 if wide else 1)
    dz = _cl(torch.rand(B, c, H // 2, W // 2, generator=torch.Generator(device=cuda).manual_seed(21), device=cuda) * 2 - 1, dtype)
    z.backward(dz)
    w = m.conv.weight.detach().to(dtype).double().requires_grad_(True)
    g, b = m.bn.weight.detach().double().requires_grad_(True), m.bn.bias.detach().double().requires_grad_(True)
    zr = F.silu(F.batch_norm(F.conv2d(xr, w, stride=2, padding=2), None, None, g, b, training=True, eps=1e-3))
    zr.backward(dz.double())
    tol = 8e-3 if dtype == torch.float16 else 6e-2
    for name, a, r in (("z", z, zr), ("dw", m.conv.weight.grad, w.grad), ("dgamma", m.bn.weight.grad, g.grad), ("dbeta", m.bn.bias.grad, b.grad)):
        e, sc = float((a.detach().double() - r.detach()).abs().max()), float(r.detach().abs().max())
        assert e <= tol * sc, (name, e, sc)


# ---------------------------------------------------------------------------------------------------------------------
# D. weight packing
# ---------------------------------------------------------------------------------------------------------------------
def _pack_ref(w, dtype, ipad, opad):
    """the two K-major packings as torch expressions: fwd[co][r][s][ci], dgrad[ci][r][s][co] = w[co][ci][k-1-r][k-1-s]"""
    o, i, k, _ = w.shape
    fwd = torch.zeros(o, k, k, ipad, dtype=dtype, device=w.device)
    fwd[..., :i] = w.permute(0, 2, 3, 1).to(dtype)
    dg = None
    if opad:
        dg = torch.zeros(i, k, k, opad, dtype=dtype, device=w.device)
        dg[..., :o] = w.flip(2, 3).permute(1, 2, 3, 0).to(dtype)
    return fwd, dg


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int16), b.view(torch.int16))


def _master(o, i, k, wdtype, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    w = torch.randn(o, i, k, k, generator=g, device=dev) * 0.3
    flat = w.view(-1)
    # rounding ties and edges of both target formats: 1 + 2^-11 (fp16 tie), 1 + 2^-8 (bf16 tie), subnormals, large values
    special = torch.tensor([1 + 2 ** -11, -(1 + 3 * 2 ** -11), 1 + 2 ** -8, -(1 + 3 * 2 ** -8), 3e-6, -7e-8, 1e-40, 60000.0, -2.5e5],
                           device=dev)
    n = min(flat.numel(), special.numel())
    flat[:n] = special[:n]
    return w.to(wdtype)


@pytest.mark.parametrize("o,i,k", [(16, 16, 3), (40, 48, 1), (80, 40, 3), (96, 320, 1), (24, 1280, 1), (192, 96, 3), (1280, 640, 3)])
@pytest.mark.parametrize("wdtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("dtype", DTYPES)
def test_weight_pack_matches_torch(cuda, o, i, k, wdtype, dtype):
    w = _master(o, i, k, wdtype, o * 7 + i, cuda)
    fwd, dg, bk_f, bk_d = train_ops.pack_weights(w, dtype, 4096, True, True)
    assert fwd.shape[3] == -(-i // bk_f) * bk_f and dg.shape[3] == -(-o // bk_d) * bk_d
    rf, rd = _pack_ref(w, dtype, fwd.shape[3], dg.shape[3])
    assert _bits_equal(fwd, rf), "forward packing"
    assert _bits_equal(dg, rd), "data-gradient packing"
    only_dg = train_ops.pack_weights(w, dtype, 4096, False, True)[1]
    assert _bits_equal(only_dg, rd)


@pytest.mark.parametrize("dtype", DTYPES)
def test_weight_pack_multi_matches_single(cuda, dtype):
    """A table of filters in one launch: item sizes below, at and across the chunk size, items without a data-gradient
    packing; every buffer must equal its y5_weight_pack result (and the torch expression)."""
    lib = _lib.lib()
    chunk = int(lib.y5_weight_pack_chunk_elems())
    shapes = [(16, 16, 3, True), (32, 16, 1, False), (128, 64, 1, False), (64, 64, 1, True), (40, 48, 3, True), (48, 40, 1, True),
              (96, 48, 3, True), (80, 80, 3, False), (192, 96, 1, True), (96, 192, 3, True), (320, 160, 1, True), (24, 1280, 1, True),
              (1280, 640, 1, False), (256, 256, 3, True), (8, 8, 1, True), (48, 96, 3, False), (384, 384, 1, True), (16, 24, 3, True),
              (640, 1280, 3, True), (72, 56, 3, True)]
    wdtypes = [torch.float32, torch.float16, torch.bfloat16]
    ents, totals = [], []
    arr = (_lib.PackItem * len(shapes))()
    ci, cx = [], []
    for t, (o, i, k, want_dg) in enumerate(shapes):
        w = _master(o, i, k, wdtypes[t % 3], 100 + t, cuda).contiguous()
        bk_f, bk_d = train_ops._block_k(i, o, 4096), train_ops._block_k(o, i, 4096)
        ipad, opad = -(-i // bk_f) * bk_f, (-(-o // bk_d) * bk_d if want_dg else 0)
        fwd = torch.full((o, k, k, ipad), float("nan"), dtype=dtype, device=cuda)
        dg = torch.full((i, k, k, opad), float("nan"), dtype=dtype, device=cuda) if want_dg else None
        it = arr[t]
        it.w, it.fwd, it.dgrad = w.data_ptr(), fwd.data_ptr(), (dg.data_ptr() if dg is not None else None)
        it.w_dtype, it.out_c, it.in_c, it.ksize, it.in_c_pad, it.out_c_pad = _lib.dtype_code(w.dtype), o, i, k, ipad, opad
        total = o * k * k * ipad + (i * k * k * opad if want_dg else 0)
        n = -(-total // chunk)
        ci += [t] * n
        cx += list(range(n))
        ents.append((w, fwd, dg, ipad, opad))
        totals.append(total)
    assert any(t < chunk for t in totals) and any(t == chunk for t in totals)
    assert any(t > chunk and t % chunk for t in totals) and sum(n for n in (-(-t // chunk) for t in totals)) > 2 * len(totals)
    items = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(cuda)
    cit, cxt = torch.tensor(ci, dtype=torch.int32, device=cuda), torch.tensor(cx, dtype=torch.int32, device=cuda)
    _lib.check(lib.y5_weight_pack_multi(items.data_ptr(), cit.data_ptr(), cxt.data_ptr(), len(ci), _lib.dtype_code(dtype), _st(cuda)))
    torch.cuda.synchronize()
    for t, (w, fwd, dg, ipad, opad) in enumerate(ents):
        sf = torch.empty_like(fwd)
        sd = torch.empty_like(dg) if dg is not None else None
        o, i, k, _ = w.shape
        _lib.check(lib.y5_weight_pack(w.data_ptr(), _lib.dtype_code(w.dtype), o, i, k, sf.data_ptr(), ipad, sd.data_ptr() if sd is not None else None,
                                      opad, _lib.dtype_code(dtype), _st(cuda)))
        rf, rd = _pack_ref(w, dtype, ipad, opad)
        assert _bits_equal(fwd, sf) and _bits_equal(fwd, rf), ("forward packing", t, shapes[t], totals[t])
        if dg is not None:
            assert _bits_equal(dg, sd) and _bits_equal(dg, rd), ("data-gradient packing", t, shapes[t], totals[t])


def _yolov5n(dev, seed):
    from oracle import model_ref
    from yolov5_b200.cfg import model_cfg
    from yolov5_b200.models.yolo import DetectionModel

    m = DetectionModel("yolov5n")
    m.load_state_dict(model_ref.synth_state_dict(model_cfg("yolov5n"), seed=seed))
    return m.to(dev).train()


def _step_inputs(dev, B=2, S=128):
    g = torch.Generator(device=dev).manual_seed(31)
    img = torch.randint(0, 256, (B, 3, S, S), generator=g, device=dev, dtype=torch.uint8)
    return img, g


def _grads(m, img, dzs, dtype=torch.float16, keep=False):
    """one training forward / backward with fixed gradients of the head maps; returns {name: grad clone}"""
    if not keep:
        for q in m.parameters():
            q.grad = None
    with torch.autocast("cuda", dtype=dtype):
        p = m(img)
    sum((q.float() * d).sum() for q, d in zip(p, dzs)).backward()
    torch.cuda.synchronize()
    return {k: q.grad.detach().clone() for k, q in m.named_parameters()}


def _head_grads(m, img, gen):
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        p = m(img)
    return [torch.randn(q.shape, generator=gen, device=q.device) * 1e-2 for q in p]


def _noise(ga, gb):
    """per-tensor run-to-run relative L2 difference of the default configuration (fp32 / fp64 atomics)"""
    return {k: _rel_l2(gb[k], ga[k]) for k in ga}


def _assert_within_noise(gc, ga, noise, what):
    worst = max(((_rel_l2(gc[k], ga[k]) - 2 * noise[k]), k) for k in ga)
    bad = [(k, _rel_l2(gc[k], ga[k]), noise[k]) for k in ga if _rel_l2(gc[k], ga[k]) > 2 * noise[k] + 1e-6]
    print(f"{what}: max run-to-run noise {max(noise.values()):.3e}, worst excess over 2x noise {worst}")
    assert not bad, (what, bad[:5])


def test_pack_plan_follows_the_master_weights(cuda):
    """PackPlan: after an optimizer step, and after `.data =` replacements, the forward packs the CURRENT master weights
    into every registered buffer."""
    m = _yolov5n(cuda, 71)
    img, gen = _step_inputs(cuda)
    dzs = _head_grads(m, img, gen)
    opt = torch.optim.SGD(m.parameters(), lr=1.0)
    plan = None

    def check(stage, all_multi):
        nonlocal plan
        plan = m.__dict__["_y5_pack_plans"][(str(cuda), torch.float16)]
        assert len(plan.entries) > 50, stage
        for e in plan.entries.values():
            assert e.wptr == e.weight.data_ptr(), stage
            if all_multi:
                assert e.epoch == plan.epoch, (stage, "not packed by this forward's multi-filter launch")
            rf, rd = _pack_ref(e.weight.detach(), torch.float16, e.ipad, e.opad)
            assert _bits_equal(e.fwd, rf), (stage, "forward packing is stale", tuple(e.weight.shape))
            if e.dg is not None:
                assert _bits_equal(e.dg, rd), (stage, "data-gradient packing is stale", tuple(e.weight.shape))

    _grads(m, img, dzs)   # first forward: layers pack for themselves and register
    check("registration", False)
    before = {id(e.weight): e.fwd.clone() for e in plan.entries.values()}
    gen_w = torch.Generator(device=cuda).manual_seed(74)
    for q in m.parameters():  # a step large enough to move every fp16 weight
        q.grad = torch.randn(q.shape, generator=gen_w, device=cuda) * 0.02
    opt.step()            # in place: same storage, new values
    _grads(m, img, dzs)
    check("after an optimizer step", True)
    assert sum(not torch.equal(before[id(e.weight)], e.fwd) for e in plan.entries.values()) > 50
    convs = [q for k, q in m.named_parameters() if k.endswith("conv.weight")][1:]
    for q in convs[::5]:  # new storage: the plan re-registers these and rebuilds its table on the next forward
        q.data = q.data * 0.5 + 0.01
    _grads(m, img, dzs)
    check("after .data replacement", False)
    with torch.no_grad():
        for q in convs[::3]:
            q.mul_(-1.5)
    _grads(m, img, dzs)
    check("after the table rebuild", True)


def test_pack_plan_off_matches_on(cuda, monkeypatch):
    m = _yolov5n(cuda, 72)
    img, gen = _step_inputs(cuda)
    dzs = _head_grads(m, img, gen)
    _grads(m, img, dzs)  # registration forward
    ga, gb = _grads(m, img, dzs), _grads(m, img, dzs)
    noise = _noise(ga, gb)
    monkeypatch.setenv("Y5_TRAIN_PACK_PLAN", "0")
    _assert_within_noise(_grads(m, img, dzs), ga, noise, "pack plan off vs on")


# ---------------------------------------------------------------------------------------------------------------------
# E. BatchNorm / SiLU training kernels (raw ABI) on channel-slice views
# ---------------------------------------------------------------------------------------------------------------------
def _slice_buf(rows, c, extra, fill, dtype, dev):
    """(buffer [rows][c + extra + 8], view pointer at channel offset 8, pitch)"""
    buf = torch.full((rows, c + extra + 8), fill, dtype=dtype, device=dev)
    return buf, buf.data_ptr() + 8 * buf.element_size(), buf.shape[1]


def _untouched(buf, c, fill):
    return bool((buf[:, :8] == fill).all() and (buf[:, 8 + c :] == fill).all())


@pytest.mark.parametrize("ch,rows,residual", [
    (8, 7, False), (40, 7, True), (1280, 7, False),        # fewer rows than one block's thread rows
    (48, 4099, True), (80, 10007, False), (1280, 3001, True),  # not a multiple of the row block
    (40, 1_600_003, True),                                 # many row blocks
])
@pytest.mark.parametrize("act", [0, 1])
@pytest.mark.parametrize("dtype", DTYPES)
def test_bn_act_passes_on_views(cuda, ch, rows, residual, act, dtype):
    lib = _lib.lib()
    code, st = _lib.dtype_code(dtype), _st(cuda)
    gen = torch.Generator(device=cuda).manual_seed(ch + rows)
    yv = ((torch.rand(rows, ch, generator=gen, device=cuda) * 4 - 2) * torch.linspace(0.5, 2, ch, device=cuda) + 0.3).to(dtype)
    ybuf, yp, ypitch = _slice_buf(rows, ch, 24, 9.0, dtype, cuda)
    ybuf[:, 8 : 8 + ch] = yv
    gamma = torch.rand(ch, generator=gen, device=cuda) + 0.5
    beta = torch.rand(ch, generator=gen, device=cuda) - 0.5
    rm0, rv0 = torch.rand(ch, generator=gen, device=cuda), torch.rand(ch, generator=gen, device=cuda) + 0.5
    rm, rv = rm0.clone(), rv0.clone()
    mean, invstd = torch.empty(ch, device=cuda), torch.empty(ch, device=cuda)
    ws = torch.zeros(2 * ch, dtype=torch.float64, device=cuda)
    zbuf, zp, zpitch = _slice_buf(rows, ch, 16, -7.0, dtype, cuda)
    rbuf, rp, rpitch = (None, None, 0)
    if residual:
        rbuf, rp, rpitch = _slice_buf(rows, ch, 40, 3.0, dtype, cuda)
        rbuf[:, 8 : 8 + ch] = (torch.rand(rows, ch, generator=gen, device=cuda) * 2 - 1).to(dtype)
    _lib.check(lib.y5_bn_stats(yp, ypitch, rows, ch, code, ws.data_ptr(), None, st))
    _lib.check(lib.y5_bn_act_fwd(yp, ypitch, zp, zpitch, rows, ch, code, mean.data_ptr(), invstd.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                                 act, 0.0, ws.data_ptr(), None, 1e-3, 0.03, rm.data_ptr(), rv.data_ptr(), rp, rpitch, st))
    yd = yv.double()
    m_ref, v_ref = yd.mean(0), yd.var(0, unbiased=False)
    assert torch.allclose(mean.double(), m_ref, rtol=1e-5, atol=1e-6)
    assert torch.allclose(invstd.double(), 1 / torch.sqrt(v_ref + 1e-3), rtol=1e-5)
    assert torch.allclose(rm.double(), 0.97 * rm0.double() + 0.03 * m_ref, rtol=1e-5, atol=1e-7)
    assert torch.allclose(rv.double(), 0.97 * rv0.double() + 0.03 * yd.var(0, unbiased=True), rtol=1e-5)
    # forward: the autocast rounding points (BN result rounded, SiLU of it rounded, then the shortcut add rounded)
    t = ((yv.float() - mean) * (invstd * gamma) + beta).to(dtype)
    zr = (F.silu(t.float()).to(dtype) if act else t).float()
    if residual:
        zr = (zr + rbuf[:, 8 : 8 + ch].float()).to(dtype).float()
    ulp = 2.0 ** -10 if dtype == torch.float16 else 2.0 ** -7
    z = zbuf[:, 8 : 8 + ch].float()
    assert float((z - zr).abs().max()) <= 2 * ulp * float(zr.abs().max())
    assert _untouched(zbuf, ch, -7.0) and _untouched(ybuf, ch, 9.0)
    # backward, dz a channel slice with its own pitch
    dzv = (torch.rand(rows, ch, generator=gen, device=cuda) * 2 - 1).to(dtype)
    dzbuf, dzp, dzpitch = _slice_buf(rows, ch, 8, 11.0, dtype, cuda)
    dzbuf[:, 8 : 8 + ch] = dzv
    dybuf, dyp, dypitch = _slice_buf(rows, ch, 32, -13.0, dtype, cuda)
    dg, db = torch.empty(ch, device=cuda), torch.empty(ch, device=cuda)
    ws.zero_()
    _lib.check(lib.y5_bn_act_bwd(yp, ypitch, dzp, dzpitch, dyp, dypitch, rows, ch, code, mean.data_ptr(), invstd.data_ptr(), gamma.data_ptr(),
                                 beta.data_ptr(), act, 0.0, dg.data_ptr(), db.data_ptr(), ws.data_ptr(), st))
    yr = yd.clone().requires_grad_(True)
    gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    out = F.batch_norm(yr, None, None, gr, br, training=True, eps=1e-3)
    (F.silu(out) if act else out).backward(dzv.double())
    tol = 6e-3 if dtype == torch.float16 else 4e-2
    for name, a, b in (("dy", dybuf[:, 8 : 8 + ch], yr.grad), ("dgamma", dg, gr.grad), ("dbeta", db, br.grad)):
        e, sc = float((a.double() - b).abs().max()), float(b.abs().max())
        assert e <= tol * sc, (name, e, sc)
    assert _untouched(dybuf, ch, -13.0) and _untouched(dzbuf, ch, 11.0)


def test_bn_stats_pass_conditioning(cuda):
    """|mean| / std = 16 over 1.6 M rows of fp16: fp32 per-thread partial sums, fp32 block combine, fp64 totals must keep
    invstd within 1e-4 of the float64 value."""
    lib = _lib.lib()
    rows, ch = 1_600_000, 64
    gen = torch.Generator(device=cuda).manual_seed(41)
    std = torch.linspace(0.25, 4, ch, device=cuda, dtype=torch.float64)
    sign = torch.where(torch.arange(ch, device=cuda) % 2 == 0, 1.0, -1.0).double()
    y = (torch.randn(rows, ch, generator=gen, device=cuda, dtype=torch.float64) * std + 16 * std * sign).half()
    yd = y.double()
    m_ref, v_ref = yd.mean(0), yd.var(0, unbiased=False)
    ratio = float((m_ref.abs() / v_ref.sqrt()).min())
    assert ratio > 15, ratio
    ws = torch.zeros(2 * ch, dtype=torch.float64, device=cuda)
    mean, invstd = torch.empty(ch, device=cuda), torch.empty(ch, device=cuda)
    rm, rv = torch.zeros(ch, device=cuda), torch.ones(ch, device=cuda)
    one, zero = torch.ones(ch, device=cuda), torch.zeros(ch, device=cuda)
    z = torch.empty_like(y)
    _lib.check(lib.y5_bn_stats(y.data_ptr(), ch, rows, ch, _lib.Y5_F16, ws.data_ptr(), None, _st(cuda)))
    _lib.check(lib.y5_bn_act_fwd(y.data_ptr(), ch, z.data_ptr(), ch, rows, ch, _lib.Y5_F16, mean.data_ptr(), invstd.data_ptr(), one.data_ptr(),
                                 zero.data_ptr(), 0, 0.0, ws.data_ptr(), None, 1e-3, 0.03, rm.data_ptr(), rv.data_ptr(), None, 0, _st(cuda)))
    is_ref = 1 / torch.sqrt(v_ref + 1e-3)
    err_is = float(((invstd.double() - is_ref) / is_ref).abs().max())
    err_m = float(((mean.double() - m_ref) / m_ref).abs().max())
    print(f"bn conditioning |mean|/std >= {ratio:.1f}, {rows} rows: invstd max rel err {err_is:.3e}, mean max rel err {err_m:.3e}")
    assert err_is <= 1e-4, err_is
    assert err_m <= 1e-5, err_m
    assert torch.allclose(rm.double(), 0.03 * m_ref, rtol=1e-5)
    assert torch.allclose(rv.double(), 0.97 + 0.03 * yd.var(0, unbiased=True), rtol=2e-4)


@pytest.mark.parametrize("dtype", DTYPES)
def test_col_sum_exact_million_rows(cuda, dtype):
    lib = _lib.lib()
    rows, ch = 1_048_583, 40
    buf, p, pitch = _slice_buf(rows, ch, 16, 5.0, dtype, cuda)
    v = _ints((rows, ch), 42, cuda)
    buf[:, 8 : 8 + ch] = v.to(dtype)
    out = torch.empty(ch, device=cuda)
    ws = torch.empty(ch, dtype=torch.float64, device=cuda)
    _lib.check(lib.y5_col_sum(p, pitch, rows, ch, _lib.dtype_code(dtype), out.data_ptr(), ws.data_ptr(), _st(cuda)))
    _assert_exact(out, v.double().sum(0), "col_sum", ("c",))


# ---------------------------------------------------------------------------------------------------------------------
# F. the Detect head's 1x1 conv with bias, and weight gradients on the side stream
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cout,cin,B,H,W", [(255, 64, 2, 16, 20), (18, 128, 2, 8, 10), (351, 256, 1, 4, 6)])
@pytest.mark.parametrize("dtype", DTYPES)
def test_conv_bias_head_exact(cuda, cout, cin, B, H, W, dtype):
    """_ConvBias pads the output channels to a multiple of 8 (256 / 24 / 352): output, dx, dW and the column-sum bias
    gradient on integer data, bit for bit."""
    cpad = -(-cout // 8) * 8
    x = _ints((B, cin, H, W), 43, cuda)
    w = _ints((cout, cin, 1, 1), 44, cuda).requires_grad_(True)
    b = _ints((cout,), 45, cuda, -8, 8).requires_grad_(True)
    xv = _cl(x, dtype).requires_grad_(True)
    y = train_ops._ConvBias.apply(xv, w, b)
    assert tuple(y.shape) == (B, H, W, cpad)
    ref = _integral(F.conv2d(x.double(), w.detach().double(), b.detach().double()), "head conv").permute(0, 2, 3, 1)
    _assert_exact(y[..., :cout], ref.float().to(dtype), "head conv", ("n", "y", "x", "c"))
    assert not y[..., cout:].any()
    dy = _ints((B, H, W, cpad), 46, cuda).to(dtype)
    y.backward(dy)
    g = dy[..., :cout].permute(0, 3, 1, 2).double()
    rdx = _integral(torch.nn.grad.conv2d_input((B, cin, H, W), w.detach().double(), g), "head dx")
    rdw = _integral(torch.nn.grad.conv2d_weight(x.double(), (cout, cin, 1, 1), g), "head dw")
    _assert_exact(xv.grad, rdx.float().to(dtype), "head dx", ("n", "c", "y", "x"))
    _assert_exact(w.grad, rdw, "head dW", ("co", "ci", "r", "s"))
    _assert_exact(b.grad, g.sum((0, 2, 3)), "head bias gradient", ("c",))


def test_async_wgrad_matches_sync_and_accumulates(cuda):
    """Weight gradients on the side stream give the synchronous gradients; with a .grad already present the layer falls back
    to the synchronous path and autograd accumulates (two identical backwards = twice the gradient)."""
    m = _yolov5n(cuda, 73)
    img, gen = _step_inputs(cuda)
    dzs = _head_grads(m, img, gen)
    _grads(m, img, dzs)
    ga, gb = _grads(m, img, dzs), _grads(m, img, dzs)
    noise = _noise(ga, gb)
    old = train_ops.set_async_wgrad(True)
    try:
        gc = _grads(m, img, dzs)
        _assert_within_noise(gc, ga, noise, "async weight gradients")
        gacc = _grads(m, img, dzs, keep=True)  # .grad present: synchronous fallback, accumulated by autograd
        _assert_within_noise({k: v / 2 for k, v in gacc.items()}, ga, noise, "accumulated async + sync weight gradients")
    finally:
        train_ops.set_async_wgrad(old)
        train_ops.finish_async(cuda)
