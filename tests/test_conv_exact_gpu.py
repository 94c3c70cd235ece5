"""GPU: the inference conv (y5_conv_bn_silu_fwd's plans) and the Detect head checked element by element, on every kernel path.

Exact parity.  With x and W integers in [-2, 2], an integer bias and an integer residual in [-8, 8] and no activation, every fp32
partial sum of the GEMM is an integer below 2^24, so the epilogue rounds exactly once (acc + b + r -> fp16/bf16) and the output
must equal the float64 convolution (+ b + r) rounded to the dtype, value for value (+0 == -0).  Input and output are channel
slices of wider NHWC buffers; the output buffer carries sentinel pixels before the first and after the last pixel, and every
half-word outside the view must keep its sentinel; the residual runs from a separate buffer and in place.  Each case names the
plan it must get (fetch form, run_plan instantiation key, cluster size) and asserts it through y5_conv_plan_info, and
test_case_list_covers_every_path checks that the list as a whole reaches every path.

SiLU.  The same cases with the activation on, and an identity 1x1 conv whose input holds every finite fp16 value (every normal
bf16 value) through every conv instantiation: |got - silu64(x)| <= 1 ulp of the dtype at silu64(x) (faithful rounding; the
subnormal step below the smallest normal), plus ulp(ref) when a residual is added.

Detect head.  Unit-vector weights copy one input channel per output column, so raw must reproduce every fp16 / normal bf16 value
at its (b, a, y, x, o) position and z must be the float64 decode of it within ulp(z) + 2^-20 (|grid| + 2) stride; mask columns
pass through.  Integer weights cover na 1/3/4, no 6/85/117/128, M tails, both copy-out branches, block_k 16/32/64, an input view
wider than in_c, and three levels written into one z buffer through y5_detect_plan_run_to."""
import ctypes as C
from dataclasses import dataclass

import pytest
import torch
import torch.nn.functional as F

from yolov5_b200 import _lib
from yolov5_b200.engine import pack_weight

from .conv_exact_ref import all_values, decode64, decode_bound, silu64, ulp

pytestmark = pytest.mark.gpu
DTYPES = [torch.float16, torch.bfloat16]
DT_IDS = ["f16", "bf16"]
SENTINEL = 0x5A5A  # half-word of every byte outside the views
GUARD = 3          # sentinel pixels before the first and after the last output pixel

FORMS = ("LINEAR", "IM2COL", "PATCH_G", "PATCH_U", "WIDE")  # PATCH with / without grouped weight stages, wide patch
KEYS = (324, 642, 1281, 1282, 2561)                           # run_plan's conv instantiations (block_n * 10 + mt); OPT adds 100000


@dataclass(frozen=True)
class Case:
    id: str
    B: int
    H: int
    W: int
    cin: int
    cout: int
    k: int                 # filter height (and width unless kw)
    s: int = 1
    p: int = 0
    kw: int = 0            # non-square filter width (0: square; then pad_w is p)
    pad_w: int = 0
    block_k: int = 0       # 0: y5_conv_pick's choice
    block_n: int = 0
    a_mode: int = 0
    mt2: bool = False
    cluster: int = 1
    cg2: bool = False
    staged: bool = False
    wide: bool = False
    stem: str = ""         # "3x1x48" | "3x3x16": the inference stem's virtual views, built as engine.lower_conv builds them
    form: str = ""         # expected plan
    key: int = 0
    csize: int = 1


CASES = [
    Case("linear_n40_m_tail", 3, 13, 11, 64, 40, 1, block_n=32, form="LINEAR", key=324),
    Case("linear_classify_m1", 1, 1, 1, 1280, 1000, 1, form="LINEAR", key=1281),              # Classify's Linear at batch 1
    Case("linear_m7_n72_staged", 7, 1, 1, 64, 72, 1, block_n=64, staged=True, form="LINEAR", key=100642),
    Case("linear_k8", 2, 10, 10, 8, 64, 1, form="LINEAR", key=642),                           # narrowest K, block_k 16
    Case("linear_n384_staged", 1, 16, 24, 64, 384, 1, block_n=256, staged=True, form="LINEAR", key=102561),
    Case("linear_cluster4_mt2", 5, 24, 24, 128, 512, 1, block_n=128, mt2=True, cluster=4, form="LINEAR", key=101282, csize=4),
    Case("im2col_s2_n72_bk32", 2, 16, 24, 32, 72, 3, 2, 1, block_k=32, block_n=128, form="IM2COL", key=1281),
    Case("im2col_s2_n384_cluster2", 3, 40, 40, 128, 384, 3, 2, 1, block_n=256, cluster=2, form="IM2COL", key=102561, csize=2),
    Case("im2col_7x7_s2_p3", 2, 23, 29, 24, 64, 7, 2, 3, form="IM2COL", key=642),
    Case("im2col_1x1_s2", 2, 15, 17, 64, 96, 1, 2, 0, block_n=32, form="IM2COL", key=324),
    Case("im2col_deep_3x3x1280_staged", 1, 10, 10, 1280, 256, 3, 1, 1, block_n=128, a_mode=1, staged=True, form="IM2COL", key=101281),
    Case("im2col_3x1_pad_w_cta_pair", 2, 14, 9, 32, 40, 3, 1, 1, kw=1, pad_w=1, block_n=64, a_mode=1, cg2=True, form="IM2COL",
         key=100642, csize=2),
    Case("patch_13x27_bk32", 3, 13, 27, 32, 64, 3, 1, 1, block_k=32, block_n=64, a_mode=2, form="PATCH_G", key=642),
    Case("patch_9x130_cta_pair", 2, 9, 130, 64, 128, 3, 1, 1, block_n=128, mt2=True, cg2=True, a_mode=2, form="PATCH_G", key=101282,
         csize=2),
    Case("patch_bn256", 2, 20, 20, 64, 256, 3, 1, 1, block_n=256, a_mode=2, form="PATCH_U", key=2561),
    Case("patch_5x5_p2_staged", 2, 24, 24, 48, 64, 5, 1, 2, block_n=64, a_mode=2, staged=True, form="PATCH_G", key=100642),
    Case("patch_3x3_p0_mt2", 2, 18, 20, 64, 64, 3, 1, 0, block_n=128, mt2=True, a_mode=2, form="PATCH_G", key=1282),
    Case("patch_1x3_pad_w_staged", 2, 12, 20, 64, 64, 1, 1, 0, kw=3, pad_w=1, block_n=64, a_mode=2, staged=True, form="PATCH_U",
         key=100642),
    Case("patch_many_tiles_bn32_staged", 16, 80, 80, 32, 32, 3, 1, 1, block_k=32, staged=True, form="PATCH_G", key=100324),
    Case("patch_many_tiles_cta_pair", 16, 80, 80, 64, 256, 3, 1, 1, block_n=256, cg2=True, form="PATCH_U", key=102561, csize=2),
    Case("wide_mt2", 2, 32, 32, 64, 64, 3, 1, 1, block_n=64, a_mode=2, wide=True, form="WIDE", key=100642),
    # an odd number of 8-pixel tiles per row cannot hold two sub-tiles side by side: the planner falls back to the grouped patch
    Case("wide_fallback_odd_tiles", 2, 40, 40, 64, 64, 3, 1, 1, block_n=64, a_mode=2, wide=True, form="PATCH_G", key=642),
    Case("wide_5x5_cluster4", 4, 24, 24, 192, 128, 5, 1, 2, block_n=128, a_mode=2, wide=True, cluster=4, form="WIDE", key=101281,
         csize=4),
    Case("stem_3x1x48", 2, 24, 40, 48, 32, 3, 1, 1, kw=1, pad_w=0, stem="3x1x48", form="PATCH_G", key=324),
    Case("stem_3x3x16", 2, 24, 40, 16, 32, 3, 1, 1, kw=3, pad_w=1, stem="3x3x16", form="PATCH_G", key=324),
]


def form_of(info: dict) -> str:
    if info["patch_pw"]:
        return "WIDE"
    if info["a_mode"] == 2:
        return "PATCH_G" if info["b_grouped"] else "PATCH_U"
    return ("LINEAR", "IM2COL")[info["a_mode"]]


def key_of(info: dict) -> int:
    return info["opt"] * 100000 + info["epi"] * 10000 + info["block_n"] * 10 + info["mt"]


def _rint(g, lo, hi, *shape):
    return torch.randint(lo, hi + 1, shape, generator=g).double()


def _sentinel(n, dev):
    return torch.full((n,), SENTINEL, dtype=torch.int16, device=dev)


class Operands:
    """Seeded integer operands of a case, its buffers and descriptor.  x (NCHW float64, the tensor the conv reads), w (OIHW
    float64, (kh, kw) filter), bias, residual (M x cout float64)."""

    def __init__(self, c: Case, dtype, dev, seed=0):
        g = torch.Generator().manual_seed(seed)
        self.c, self.dtype, self.dev = c, dtype, dev
        kh, kw = c.k, (c.kw or c.k)
        pad_w = c.pad_w if c.kw else c.p
        d = _lib.ConvDesc()
        if c.stem:
            # [B][h2][w2 + 2][16] space-to-depth cells with one cell left and right of every row (non-zero here: the 3x3x16 view
            # must not read them, the 3x1x48 view reads them as the outer thirds of its edge pixels)
            h2, w2 = c.H, c.W
            buf = _rint(g, -2, 2, c.B, h2, w2 + 2, 16)
            self.ibuf = buf.to(dev, dtype)
            ys, ns = (w2 + 2) * 16, h2 * (w2 + 2) * 16
            if c.stem == "3x1x48":
                x = torch.cat([buf[:, :, s : s + w2, :] for s in range(3)], dim=3)
                d.inp, d.in_pitch = self.ibuf.data_ptr(), 16
            else:
                x = buf[:, :, 1 : w2 + 1, :]
                d.inp, d.in_pitch = self.ibuf.data_ptr() + 16 * self.ibuf.element_size(), 16
            d.in_x_stride, d.in_y_stride, d.in_n_stride = 16, ys, ns
            self.x = x.permute(0, 3, 1, 2).contiguous()
        else:
            x = _rint(g, -2, 2, c.B, c.H, c.W, c.cin)
            in_off, in_pitch = 8, c.cin + 16
            self.ibuf = torch.full((c.B, c.H, c.W, in_pitch), 3.0, dtype=dtype, device=dev)  # non-zero outside the view
            self.ibuf[..., in_off : in_off + c.cin] = x.to(dev, dtype)
            d.inp, d.in_pitch = self.ibuf.data_ptr() + in_off * self.ibuf.element_size(), in_pitch
            self.x = x.permute(0, 3, 1, 2).contiguous()
        self.x = self.x.to(dev)
        self.w = _rint(g, -2, 2, c.cout, c.cin, kh, kw).to(dev)
        self.bias = _rint(g, -8, 8, c.cout).float().to(dev)
        self.Ho = (c.H + 2 * c.p - kh) // c.s + 1
        self.Wo = (c.W + 2 * pad_w - kw) // c.s + 1
        self.M = c.B * self.Ho * self.Wo
        self.res = _rint(g, -8, 8, self.M, c.cout).to(dev)
        self.kh, self.kw, self.pad_w = kh, kw, pad_w
        bk = C.c_int32()
        _lib.check(_lib.lib().y5_conv_pick(c.cin, c.cout, self.M, C.byref(bk), None))
        self.block_k = c.block_k or bk.value
        self.wp = pack_weight(self.w.float(), self.block_k, dtype).to(dev)
        d.batch, d.in_h, d.in_w, d.in_c = c.B, c.H, c.W, c.cin
        d.weight, d.bias = self.wp.data_ptr(), self.bias.data_ptr()
        d.out_c = c.cout
        d.ksize, d.stride, d.pad = c.k, c.s, c.p
        if c.kw:
            d.kw, d.pad_w = c.kw, c.pad_w
        d.dtype, d.block_k, d.block_n, d.a_mode = _lib.dtype_code(dtype), self.block_k, c.block_n, c.a_mode
        d.reserved = ((2 if c.mt2 else 0) | (4 if c.cg2 else 0) | (8 if c.staged else 0) | (128 if c.wide else 0)
                      | (c.cluster << 8 if c.cluster > 1 else 0))
        self.desc = d
        # output: channels [8, 8 + cout) of pitch cout + 24, GUARD sentinel pixels before and after
        self.opitch = c.cout + 24
        self.obuf = _sentinel((GUARD + self.M + GUARD) * self.opitch, dev)
        self.view = self.obuf.view(-1, self.opitch)[GUARD : GUARD + self.M, 8 : 8 + c.cout]
        d.out, d.out_pitch = self.obuf.data_ptr() + (GUARD * self.opitch + 8) * 2, self.opitch

    def plan(self):
        plan = C.c_void_p()
        _lib.check(_lib.lib().y5_conv_plan_create(C.byref(self.desc), C.byref(plan)), f"conv_plan_create[{self.c.id}]")
        return plan

    def info(self) -> dict:
        plan = self.plan()
        try:
            info = _lib.PlanInfo()
            _lib.check(_lib.lib().y5_conv_plan_info(plan, C.byref(info)), "conv_plan_info")
            return info.as_dict()
        finally:
            _lib.lib().y5_conv_plan_destroy(plan)

    def run(self, act: bool, in_place: bool):
        """Runs the conv into a fresh sentinel-filled output; returns (view as float64, separate residual buffer or None)."""
        d = self.desc
        self.obuf.fill_(SENTINEL)
        resv = self.res.to(self.dtype).view(torch.int16)
        if in_place:
            self.view.copy_(resv)
            d.residual, d.res_pitch, rbuf = d.out, self.opitch, None
        else:
            rpitch = self.c.cout + 8
            rbuf = _sentinel(self.M * rpitch, self.dev)
            rbuf.view(-1, rpitch)[:, : self.c.cout].copy_(resv)
            d.residual, d.res_pitch = rbuf.data_ptr(), rpitch
        d.act = int(act)
        plan = self.plan()
        try:
            _lib.check(_lib.lib().y5_conv_plan_run(plan, C.c_void_p(_lib.stream_ptr(self.dev))), f"conv[{self.c.id}]")
            torch.cuda.synchronize()
        finally:
            _lib.lib().y5_conv_plan_destroy(plan)
        outside = torch.ones_like(self.obuf, dtype=torch.bool)
        outside.view(-1, self.opitch)[GUARD : GUARD + self.M, 8 : 8 + self.c.cout] = False
        bad = int((self.obuf[outside] != SENTINEL).sum())
        assert bad == 0, f"{self.c.id}: {bad} half-words outside the output view overwritten"
        if rbuf is not None:
            r = rbuf.view(-1, self.c.cout + 8)
            assert torch.equal(r[:, : self.c.cout], resv) and bool((r[:, self.c.cout :] == SENTINEL).all()), "residual buffer written"
        return self.view.contiguous().view(self.dtype).double()

    def conv64(self):
        """float64 conv (+ bias) as M x cout rows in (b, y, x) order."""
        y = F.conv2d(self.x, self.w, stride=self.c.s, padding=(self.c.p, self.pad_w))
        return y.permute(0, 2, 3, 1).reshape(self.M, self.c.cout) + self.bias.double()


def _first_bad(bad, got, ref):
    i = int(bad.flatten().nonzero()[0])
    m, n = divmod(i, got.shape[1])
    return f"{int(bad.sum())} elements, first at pixel {m} channel {n}: got {float(got[m, n])!r} want {float(ref[m, n])!r}"


def test_case_list_covers_every_path(cuda):
    """Every instantiation key (plain and OPT), fetch form, cluster size, store path and K block width, in both dtypes, as
    y5_conv_plan_info reports them for the case list; and each case gets the plan it names."""
    reached = set()
    for dtype in DTYPES:
        for c in CASES:
            info = Operands(c, dtype, cuda).info()
            assert (form_of(info), key_of(info), info["cluster"]) == (c.form, c.key, c.csize), (c.id, info)
            reached |= {("key", key_of(info), dtype), ("form", form_of(info), dtype), ("cluster", info["cluster"], dtype),
                        ("staged", info["staged"], dtype), ("block_k", info["block_k"], dtype)}
    for dtype in DTYPES:
        want = ({("key", k, dtype) for k in KEYS} | {("key", 100000 + k, dtype) for k in KEYS} | {("form", f, dtype) for f in FORMS}
                | {("cluster", n, dtype) for n in (1, 2, 4)} | {("staged", s, dtype) for s in (0, 1)}
                | {("block_k", b, dtype) for b in (16, 32, 64)})
        assert want <= reached, sorted(want - reached, key=str)
    assert any(c.cg2 for c in CASES)  # CTA pairs (reserved bit 2) as well as explicit cluster sizes


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_conv_exact(cuda, case, dtype):
    """act = 0: bit-exact against the float64 conv + b + r, residual separate and in place; act = 1: SiLU within
    ulp(ref) + ulp(silu64) per element."""
    op = Operands(case, dtype, cuda)
    info = op.info()
    assert (form_of(info), key_of(info), info["cluster"], info["staged"], info["block_k"]) == (
        case.form, case.key, case.csize, int(case.staged), op.block_k), (case.id, info)
    pre = op.conv64()
    ref = (pre + op.res).float().to(dtype).double()
    for in_place in (False, True):
        got = op.run(act=False, in_place=in_place)
        bad = got != ref
        assert not bad.any(), f"{case.id} {'in place' if in_place else 'separate'}: " + _first_bad(bad, got, ref)
    s = silu64(pre)
    ref = s + op.res
    got = op.run(act=True, in_place=False)
    bad = (got - ref).abs() > ulp(ref, dtype) + ulp(s, dtype)
    assert not bad.any(), f"{case.id} SiLU: " + _first_bad(bad, got, ref)


# ------------------------------------------------------------------------------------------------------------------------------
# SiLU on every input value: a 1x1 identity conv 256 -> 256 (bias 0), so the pre-activation is x itself
TILES = [(32, False), (64, False), (128, False), (128, True), (256, False)]


def _identity_conv(dev, dtype, x, bias, block_n, mt2, staged):
    n = 256
    rows = (x.numel() + n - 1) // n
    xin = torch.zeros(rows * n, dtype=dtype, device=dev)
    xin[: x.numel()] = x.to(dev)
    out = torch.empty(rows, n, dtype=dtype, device=dev)
    wp = pack_weight(torch.eye(n).view(n, n, 1, 1), 64, dtype).to(dev)
    d = _lib.ConvDesc()
    d.inp, d.in_pitch = xin.data_ptr(), n
    d.batch, d.in_h, d.in_w, d.in_c = 1, rows, 1, n
    d.weight, d.bias = wp.data_ptr(), bias.data_ptr()
    d.out, d.out_pitch, d.out_c = out.data_ptr(), n, n
    d.ksize, d.stride, d.pad = 1, 1, 0
    d.act, d.dtype, d.block_k, d.block_n = 1, _lib.dtype_code(dtype), 64, block_n
    d.reserved = (2 if mt2 else 0) | (8 if staged else 0)
    lib = _lib.lib()
    plan = C.c_void_p()
    _lib.check(lib.y5_conv_plan_create(C.byref(d), C.byref(plan)), "conv_plan_create")
    try:
        info = _lib.PlanInfo()
        _lib.check(lib.y5_conv_plan_info(plan, C.byref(info)))
        _lib.check(lib.y5_conv_plan_run(plan, C.c_void_p(_lib.stream_ptr(dev))), "conv")
        torch.cuda.synchronize()
    finally:
        lib.y5_conv_plan_destroy(plan)
    return xin, out, info.as_dict()


@pytest.mark.parametrize("random_bias", [False, True], ids=["bias0", "bias_rand"])
@pytest.mark.parametrize("staged", [False, True], ids=["direct", "staged"])
@pytest.mark.parametrize("tile", TILES, ids=[f"bn{b}{'x2' if m else ''}" for b, m in TILES])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_silu_every_value(cuda, dtype, tile, staged, random_bias):
    """Every finite fp16 / normal bf16 value through every conv instantiation's SiLU: within 1 ulp of silu64 (faithful).  With a
    random fp32 bias the reference pre-activation is fp32(x + b)."""
    g = torch.Generator().manual_seed(3)
    bias = (torch.rand(256, generator=g) * 16 - 8 if random_bias else torch.zeros(256)).to(cuda)  # fp16 65504 + b stays finite
    xin, out, info = _identity_conv(cuda, dtype, all_values(dtype), bias, tile[0], tile[1], staged)
    mt = tile[1] + 1 if tile[0] >= 128 else 128 // tile[0]
    assert (info["a_mode"], key_of(info), info["staged"]) == (0, (100000 if staged else 0) + tile[0] * 10 + mt, int(staged)), info
    pre = (xin.view(-1, 256).float() + bias).double()  # fp32 rounding of acc + b, as the epilogue forms it
    ref = silu64(pre)
    got = out.double()
    bad = (got - ref).abs() > ulp(ref, dtype)
    assert not bad.any(), f"{int(bad.sum())} values, first x = {float(pre[bad][0])!r}: got {float(got[bad][0])!r} want {float(ref[bad][0])!r}"


# ------------------------------------------------------------------------------------------------------------------------------
# Detect head
HEAD_N = 128  # rows per anchor in the packed head weight (kHeadN)
ANCHORS = torch.tensor([[10.0, 13.0], [16.0, 30.0], [33.0, 23.0], [62.0, 45.0]])


def _pack_head(w, bias, na, no, block_k, dtype):
    """(na*no, cin) weight and (na*no,) bias -> [na*HEAD_N][cin_pad] / [na*HEAD_N], anchor a in rows [HEAD_N a, HEAD_N a + no)."""
    cin = w.shape[1]
    ipad = (cin + block_k - 1) // block_k * block_k
    wp = torch.zeros(na * HEAD_N, ipad, dtype=dtype)
    bp = torch.zeros(na * HEAD_N, dtype=torch.float32)
    for a in range(na):
        wp[a * HEAD_N : a * HEAD_N + no, :cin] = w[a * no : (a + 1) * no].to(dtype)
        bp[a * HEAD_N : a * HEAD_N + no] = bias[a * no : (a + 1) * no]
    return wp, bp


class Head:
    """One Detect level: input view (channels [8, 8 + cin) of pitch cin + 16, or a plain tensor), packed weights, plan."""

    def __init__(self, dev, dtype, x, w, bias, na, nc, stride, block_k, z_rows=0, z_row0=0, in_extra=True):
        B, ny, nx, cin = x.shape
        self.na, self.no, self.nc, self.stride = na, w.shape[0] // na, nc, stride
        self.B, self.ny, self.nx = B, ny, nx
        self.z_rows, self.z_row0 = z_rows or na * ny * nx, z_row0
        self.dev, self.dtype = dev, dtype
        self.x, self.w, self.bias = x, w, bias
        pitch = (cin + 7) // 8 * 8
        off, pitch = (8, pitch + 16) if in_extra else (0, pitch)
        self.ibuf = torch.full((B, ny, nx, pitch), 3.0, dtype=dtype, device=dev)
        self.ibuf[..., off : off + cin] = x.to(dev, dtype)
        wp, bp = _pack_head(w, bias, na, self.no, block_k, dtype)
        self.wp, self.bp = wp.to(dev), bp.to(dev)
        self.anchors = ANCHORS[:na] * stride / 8
        d = _lib.DetectDesc()
        d.inp, d.in_pitch = self.ibuf.data_ptr() + off * self.ibuf.element_size(), pitch
        d.batch, d.ny, d.nx, d.in_c = B, ny, nx, cin
        d.weight, d.bias = self.wp.data_ptr(), self.bp.data_ptr()
        d.z_rows, d.z_row0 = self.z_rows, z_row0
        d.na, d.no, d.nc = na, self.no, nc
        d.stride = stride
        for q, v in enumerate(self.anchors.reshape(-1).tolist()):
            d.anchor_wh[q] = v
        d.dtype, d.block_k = _lib.dtype_code(dtype), block_k
        self.plan = C.c_void_p()
        _lib.check(_lib.lib().y5_detect_plan_create(C.byref(d), C.byref(self.plan)), "detect_plan_create")

    def close(self):
        _lib.lib().y5_detect_plan_destroy(self.plan)

    def run_to(self, raw_ptr, z_ptr):
        _lib.check(_lib.lib().y5_detect_plan_run_to(self.plan, C.c_void_p(raw_ptr), C.c_void_p(z_ptr), C.c_void_p(_lib.stream_ptr(self.dev))),
                   "detect")
        torch.cuda.synchronize()

    def reference(self):
        """raw (B, na, ny, nx, no) float64, z, per-element bound on z."""
        x = self.x.double().to(self.dev).reshape(-1, self.x.shape[-1])
        raw = (x @ self.w.double().to(self.dev).t() + self.bias.double().to(self.dev))
        raw = raw.reshape(self.B, self.ny, self.nx, self.na, self.no).permute(0, 3, 1, 2, 4).contiguous()
        z, grid = decode64(raw, self.nc, self.stride, self.anchors)
        return raw, z, decode_bound(z, grid, self.stride, self.dtype)


def _check_level(h: Head, raw_got, z_got, what):
    raw, z, bound = h.reference()
    raw_ref = raw.float().to(h.dtype).double()
    bad = raw_got != raw_ref
    assert not bad.any(), f"{what} raw: {int(bad.sum())} elements, first at {bad.nonzero()[0].tolist()}"
    z_got = z_got.reshape(z.shape)
    bad = (z_got - z).abs() > bound
    assert not bad.any(), (f"{what} z: {int(bad.sum())} elements, first at {bad.nonzero()[0].tolist()}: "
                           f"got {float(z_got[bad][0])!r} want {float(z[bad][0])!r} (raw {float(raw[bad][0])!r})")
    m = z_got[..., 5 + h.nc :]
    assert bool((m == raw_ref[..., 5 + h.nc :]).all()), f"{what}: mask columns changed"


def _guarded(n, dev, guard=64):
    """n-element output with `guard` sentinel half-words before and after (16-byte aligned); returns (buffer, view)."""
    buf = _sentinel(guard + n + guard, dev)
    return buf, buf[guard : guard + n]


def _guards_intact(buf, guard=64):
    return bool((buf[:guard] == SENTINEL).all() and (buf[-guard:] == SENTINEL).all())


def _run_single(h: Head, what):
    n_raw = h.B * h.na * h.ny * h.nx * h.no
    rbuf, raw = _guarded(n_raw, h.dev)
    zbuf, z = _guarded(h.B * h.z_rows * h.no, h.dev)
    h.run_to(raw.data_ptr(), z.data_ptr())
    assert _guards_intact(rbuf) and _guards_intact(zbuf), f"{what}: wrote outside raw / z"
    raw_got = raw.view(h.dtype).double().view(h.B, h.na, h.ny, h.nx, h.no)
    _check_level(h, raw_got, z.view(h.dtype).double(), what)


@pytest.mark.parametrize("layout", [(3, 85, 80), (3, 117, 80)], ids=["no85", "no117_masks"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_detect_every_value(cuda, dtype, layout):
    """Unit-vector head weights: output column (a, o) copies input channel a*no + o, so raw reproduces every fp16 (normal bf16)
    value bit for bit (-0 comes out as +0: acc = -0 + 0) and z is its float64 decode within the bound; mask columns pass."""
    na, no, nc = layout
    cin = na * no
    B, ny, nx = 2, 10, 13
    vals = all_values(dtype)
    assert vals.numel() <= B * ny * nx * cin
    x = torch.zeros(B * ny * nx * cin, dtype=dtype)
    x[: vals.numel()] = vals
    x = x.view(B, ny, nx, cin)
    w = torch.eye(cin)
    h = Head(cuda, dtype, x, w, torch.zeros(cin), na, nc, 8.0, 64)
    try:
        _run_single(h, f"every value na {na} no {no}")
    finally:
        h.close()


DET_CASES = [
    # id, B, ny, nx, cin, na, nc, nm, block_k
    ("na1_no6_bk16", 3, 10, 10, 16, 1, 1, 0, 16),        # M = 300: a 44-row tail, tiles straddling images; 6 * rows: both copies
    ("na3_no85_scalar_copy", 2, 7, 9, 64, 3, 80, 0, 32),  # no and ny*nx odd: every copy-out takes the scalar path
    ("na4_no117_masks", 3, 11, 13, 128, 4, 80, 32, 64),   # 4 anchors, 32 mask columns
    ("na3_no128_vector_copy", 2, 16, 16, 96, 3, 91, 32, 64),  # no = 128: every copy-out is 16-byte vectors
]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("case", DET_CASES, ids=[c[0] for c in DET_CASES])
def test_detect_integer(cuda, dtype, case):
    """Integer weights / inputs / bias: raw exact, z within the bound; input view wider than in_c."""
    name, B, ny, nx, cin, na, nc, nm, bk = case
    no = 5 + nc + nm
    g = torch.Generator().manual_seed(5)
    x, w, b = _rint(g, -2, 2, B, ny, nx, cin), _rint(g, -2, 2, na * no, cin), _rint(g, -8, 8, na * no)
    h = Head(cuda, dtype, x, w, b.float(), na, nc, 16.0, bk)
    try:
        _run_single(h, name)
    finally:
        h.close()


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_detect_three_levels_one_z(cuda, dtype):
    """Three levels into one z buffer with z_rows / z_row0 as engine.lower_detect sets them, through y5_detect_plan_run_to into
    outputs allocated after the plans: after each level its rows are right, the rows of the levels still to run keep their
    sentinels, and nothing around the buffers is written."""
    B, na, nc = 2, 3, 80
    no = 5 + nc
    levels = [(12, 16, 64, 8.0, 64), (6, 8, 128, 16.0, 32), (3, 4, 256, 32.0, 16)]  # ny, nx, cin, stride, block_k
    z_rows = sum(na * ny * nx for ny, nx, *_ in levels)
    g = torch.Generator().manual_seed(7)
    heads, row0 = [], 0
    try:
        for ny, nx, cin, stride, bk in levels:
            x, w, b = _rint(g, -2, 2, B, ny, nx, cin), _rint(g, -2, 2, na * no, cin), _rint(g, -8, 8, na * no)
            heads.append(Head(cuda, dtype, x, w, b.float(), na, nc, stride, bk, z_rows=z_rows, z_row0=row0))
            row0 += na * ny * nx
        zbuf, z = _guarded(B * z_rows * no, cuda)
        z3 = z.view(B, z_rows, no)
        for i, h in enumerate(heads):
            rbuf, raw = _guarded(B * na * h.ny * h.nx * no, cuda)
            h.run_to(raw.data_ptr(), z.data_ptr())
            assert _guards_intact(rbuf) and _guards_intact(zbuf), f"level {i}: wrote outside raw / z"
            lo, hi = h.z_row0, h.z_row0 + na * h.ny * h.nx
            assert bool((z3[:, hi:] == SENTINEL).all()), f"level {i} wrote rows of a later level"
            _check_level(h, raw.view(dtype).double().view(B, na, h.ny, h.nx, no), z3[:, lo:hi].view(dtype).double(), f"level {i}")
    finally:
        for h in heads:
            h.close()
