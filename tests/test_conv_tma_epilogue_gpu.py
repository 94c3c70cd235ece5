"""GPU: the conv's TMA epilogue (the default for EPI 0 outside the optional modes).  The tile is staged in shared memory, its
residual is TMA-loaded there by the producer warp, and the tile leaves by TMA bulk stores.  Its bytes must equal the direct
register stores (reserved bit 16) and match the fp32 oracle SiLU(conv2d(x, W') + b') + r.  The cases cover every (block_n, MT)
instantiation, the LINEAR, IM2COL and PATCH fetches (tw 8 and 128), M tails, PATCH overhang, N tails, channel-slice outputs
with canary bytes around them, residuals in place and in a separate buffer, and enough tiles per CTA to cycle the staging block.
A chain of dependent launches under programmatic dependent launch reads each layer's output right after it is stored."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from yolov5_b200 import _lib
from yolov5_b200.engine import pack_weight

from .gpu_util import plan_info, rel_err

pytestmark = pytest.mark.gpu
TOL = {torch.float16: 2e-3, torch.bfloat16: 1.6e-2}
CANARY = -3.0
DIRECT = 16  # reserved bit 4: direct stores from the registers


class Layer:
    """One conv on NHWC device buffers; the output (and a separate residual) is channels [8, 8 + cout) of a buffer 24 channels
    wider, so every store outside the slice shows up in the canary bytes."""

    def __init__(self, dev, dtype, B, H, W, cin, cout, k, s, p, act=True, residual=None, block_n=0, mt2=False, a_mode=0, seed=0):
        g = torch.Generator().manual_seed(seed)
        self.dev, self.dtype, self.cout = dev, dtype, cout
        self.x = torch.rand(B, cin, H, W, generator=g) * 2 - 1
        self.w = (torch.rand(cout, cin, k, k, generator=g) * 2 - 1) / (cin * k * k) ** 0.5 * 2
        self.b = torch.rand(cout, generator=g) - 0.5
        self.Ho, self.Wo = (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1
        self.r = torch.rand(B, cout, self.Ho, self.Wo, generator=g) - 0.5 if residual else None
        self.shape = (B, H, W, cin, cout, k, s, p)
        self.act, self.residual, self.block_n, self.mt2, self.a_mode = act, residual, block_n, mt2, a_mode
        bk, bn = C.c_int32(), C.c_int32()
        _lib.check(_lib.lib().y5_conv_pick(cin, cout, B * self.Ho * self.Wo, C.byref(bk), C.byref(bn)))
        self.bk = bk.value
        self.wp = pack_weight(self.w, self.bk, dtype).to(dev)
        self.bias = self.b.to(dev)

    def oracle(self):
        y = F.conv2d(self.x.to(self.dtype).float(), self.w.to(self.dtype).float(), self.b, stride=self.shape[6], padding=self.shape[7])
        if self.act:
            y = F.silu(y)
        return y + self.r.to(self.dtype).float() if self.r is not None else y

    def buffers(self):
        B, cout = self.shape[0], self.cout
        xin = self.x.permute(0, 2, 3, 1).contiguous().to(self.dev, self.dtype)
        obuf = torch.full((B, self.Ho, self.Wo, cout + 24), CANARY, dtype=self.dtype, device=self.dev)
        rbuf = None
        if self.residual == "in_place":
            rbuf = obuf
        elif self.residual == "separate":
            rbuf = torch.full_like(obuf, 5.0)
        if rbuf is not None:
            rbuf[..., 8 : 8 + cout] = self.r.permute(0, 2, 3, 1).to(self.dev, self.dtype)
        return xin, obuf, rbuf

    def desc(self, xin, obuf, rbuf, reserved=0):
        B, H, W, cin, cout, k, s, p = self.shape
        es = obuf.element_size()
        d = _lib.ConvDesc()
        d.inp, d.in_pitch = xin.data_ptr(), xin.shape[3]
        d.batch, d.in_h, d.in_w, d.in_c = B, H, W, cin
        d.weight, d.bias = self.wp.data_ptr(), self.bias.data_ptr()
        d.out, d.out_pitch, d.out_c = obuf.data_ptr() + 8 * es, obuf.shape[3], cout
        d.residual, d.res_pitch = (rbuf.data_ptr() + 8 * es, rbuf.shape[3]) if rbuf is not None else (None, 0)
        d.ksize, d.stride, d.pad = k, s, p
        d.act, d.dtype, d.block_k, d.block_n = int(self.act), _lib.dtype_code(self.dtype), self.bk, self.block_n
        d.a_mode = self.a_mode
        d.reserved = (2 if self.mt2 else 0) | reserved
        return d

    def run(self, reserved=0, expect=None):
        """Returns (whole output buffer, plan info)."""
        xin, obuf, rbuf = self.buffers()
        d = self.desc(xin, obuf, rbuf, reserved)
        info = plan_info(d)
        if expect:
            assert {k: info[k] for k in expect} == expect, ("plan differs from the path the case names", info)
        _lib.check(_lib.lib().y5_conv_bn_silu_fwd(C.byref(d), C.c_void_p(_lib.stream_ptr(self.dev))), "conv")
        torch.cuda.synchronize()
        return obuf, info


def check(layer, expect=None, tma_fits=True):
    """TMA epilogue == direct stores byte for byte (including the canaries), within the oracle's tolerance.  `tma_fits`: the
    plan takes the TMA epilogue (else its 64 KB staging block does not fit next to two pipeline stages and it keeps direct stores);
    None: whichever the planner picks."""
    tma, info = layer.run(expect=dict(expect or {}, **({} if tma_fits is None else {"tma_epi": int(tma_fits)})))
    direct, dinfo = layer.run(reserved=DIRECT)
    assert dinfo["tma_epi"] == 0
    cout = layer.cout
    assert bool((tma[..., :8] == CANARY).all() and (tma[..., 8 + cout :] == CANARY).all()), "wrote outside the channel slice"
    assert torch.equal(tma.view(torch.int16), direct.view(torch.int16)), (layer.shape, info, "TMA epilogue differs from direct stores")
    got = tma[..., 8 : 8 + cout].float().cpu().permute(0, 3, 1, 2)
    err = rel_err(got, layer.oracle())
    assert err < TOL[layer.dtype], (layer.shape, info, err)
    return info


TILES = [(32, False), (64, False), (128, False), (128, True), (256, False)]
CASES = [
    # B, H, W, cin, cout, k, s, p, a_mode, expected plan fields
    ((2, 20, 20, 64, 64, 1, 1, 0), 0, {"a_mode": 0}),              # LINEAR, M = 800: a 128-row tail
    ((2, 20, 20, 64, 64, 3, 1, 1), 1, {"a_mode": 1}),              # IM2COL
    ((2, 16, 24, 32, 72, 3, 2, 1), 0, {"a_mode": 1}),              # stride 2, N tail inside a 64-column box
    ((3, 13, 27, 32, 64, 3, 1, 1), 2, {"a_mode": 2, "tw": 8}),     # PATCH tw 8, tiles overhanging Ho and Wo
    ((2, 32, 8, 64, 128, 3, 1, 1), 2, {"a_mode": 2, "tw": 8}),     # PATCH tw 8, exact fit
    ((2, 1, 200, 16, 64, 3, 1, 1), 2, {"a_mode": 2, "tw": 128}),   # PATCH tw 128 (one row of 128 pixels), overhang in x
    ((1, 16, 24, 64, 384, 1, 1, 0), 0, {"a_mode": 0}),             # N tail: 384 = 1.5 256-wide tiles
    ((2, 20, 20, 64, 256, 3, 1, 1), 2, {"a_mode": 2}),             # PATCH, 256 channels
]


@pytest.mark.parametrize("residual", [None, "separate", "in_place"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("tile", TILES, ids=[f"bn{b}{'x2' if m else ''}" for b, m in TILES])
@pytest.mark.parametrize("case", CASES, ids=lambda c: "x".join(map(str, c[0])))
def test_tma_epilogue_every_tile(cuda, case, tile, dtype, residual):
    shape, a_mode, expect = case
    if tile[0] >= 2 * shape[4]:
        pytest.skip("N tile more than twice the layer width")
    layer = Layer(cuda, dtype, *shape, residual=residual, block_n=tile[0], mt2=tile[1], a_mode=a_mode)
    # PATCH tiles of a 3 x 3 conv over 64-channel chunks may leave no room for the staging block next to two pipeline stages
    tma_fits = None if a_mode == 2 and shape[3] > 16 else True
    check(layer, dict(expect, block_n=tile[0], mt=2 if tile[1] else max(1, 128 // tile[0])), tma_fits)


@pytest.mark.parametrize("act", [True, False])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("case", [(4, 160, 160, 64, 64, 3, 1, 1), (8, 80, 80, 128, 128, 3, 1, 1), (8, 40, 40, 256, 256, 3, 1, 1),
                                  (8, 20, 20, 512, 512, 3, 1, 1), (8, 80, 80, 256, 128, 1, 1, 0)],
                         ids=["yolov5l-160", "yolov5l-80", "yolov5l-40", "yolov5l-20", "1x1-80"])
def test_tma_epilogue_default_plan(cuda, case, dtype, act):
    """The planner's own tile choice at yolov5l layer shapes, in place (the Bottleneck lowering), with and without SiLU."""
    check(Layer(cuda, dtype, *case, act=act, residual="in_place"), tma_fits=None)


@pytest.mark.parametrize("residual", [None, "in_place"])
def test_tma_epilogue_many_tiles_per_cta(cuda, residual):
    """1600 tiles of 512 x 32 over at most 132 CTAs: a dozen tiles per CTA, so the staging block and its barriers cycle."""
    info = check(Layer(cuda, torch.float16, 16, 160, 160, 64, 64, 3, 1, 1, residual=residual, block_n=32))
    assert info["grid"] * 8 < 1600


def test_tma_epilogue_dependent_launches(cuda):
    """Layers launched back to back under programmatic dependent launch, each reading the previous one's output as its input and
    as its in-place residual: the next grid starts as the previous one retires, so every bulk store of a CTA must be complete when
    it exits.  The chain through TMA stores must give the bytes of the chain through direct stores."""
    dev, dtype = cuda, torch.bfloat16
    B, H, W, c = 8, 40, 40, 128
    layers = [Layer(dev, dtype, B, H, W, c, c, 3, 1, 1, residual="in_place", seed=i) for i in range(4)]
    lib = _lib.lib()
    st = C.c_void_p(_lib.stream_ptr(dev))

    def chain(reserved):
        x0 = layers[0].x.permute(0, 2, 3, 1).contiguous().to(dev, dtype)
        bufs = [torch.full((B, H, W, c + 24), CANARY, dtype=dtype, device=dev) for _ in layers]
        r = layers[0].r.permute(0, 2, 3, 1).to(dev, dtype)
        plans = []
        for i, (L, ob) in enumerate(zip(layers, bufs)):
            ob[..., 8 : 8 + c] = r  # the residual of layer i, overwritten in place by its output
            xin = x0 if i == 0 else bufs[i - 1][..., 8 : 8 + c]
            d = L.desc(xin, ob, ob, reserved)
            if i:  # the previous layer's output slice is this layer's input view
                d.inp, d.in_pitch = bufs[i - 1].data_ptr() + 8 * ob.element_size(), c + 24
            plan = C.c_void_p()
            _lib.check(lib.y5_conv_plan_create(C.byref(d), C.byref(plan)), "conv_plan_create")
            plans.append(plan)
        torch.cuda.synchronize()
        try:
            for _ in range(3):
                for plan in plans:
                    _lib.check(lib.y5_conv_plan_run(plan, st), "conv")
            torch.cuda.synchronize()
        finally:
            for plan in plans:
                lib.y5_conv_plan_destroy(plan)
        return bufs

    tma, direct = chain(0), chain(DIRECT)
    for i, (a, b) in enumerate(zip(tma, direct)):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)), f"layer {i}: TMA chain differs from the direct chain"
    assert bool(torch.isfinite(tma[-1][..., 8 : 8 + c].float()).all())
