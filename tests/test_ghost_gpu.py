"""GPU: yolov5s-ghost (reference models/hub/yolov5s-ghost.yaml).

Kernels.  y5_dwconv_fwd and y5_dwconv_wgrad against float64 torch on the device, in fp16 and bf16: integer-valued data small
enough that every product, sum, LeakyReLU(0.25) and rounding is exact, so the forward, the two-output GhostBottleneck form, the
in-place residual and the rotated-tap data gradient with its accumulated residual are bit-exact; SiLU within one unit in the last
place; the weight gradient exact on integer data and, on Gaussian data, within the fp32 summation bound over B*H*W terms.  Every
view is a channel slice of a wider buffer whose other channels must survive.  Channels 8 to 512, batch 1 and 3, maps 1x1 to
160x160.

Models.  Full-size yolov5s-ghost with seeded weights against oracle/ghost_ref.py (square, rect and augment=True input);
GhostConv and GhostBottleneck run as single layers; the reference-scaled-down model against the reference's stored fp32
forward; the reference-pickled checkpoint through attempt_load and NMS; one AMP training step against the reference's fp32
gradients; GraphedTrainStep against the eager step."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import ghost_ref
from yolov5_b200 import _lib

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
DTYPES = [torch.float16, torch.bfloat16]
SENT = 77.0  # channels next to a view hold this before a launch and must hold it after
# (batch, h, w, c): channels 8..512, batch 1 and 3, the maps the model and its edge cases produce
CASES = [(1, 1, 1, 8), (3, 2, 2, 16), (1, 5, 5, 24), (3, 13, 7, 40), (1, 20, 20, 512), (3, 20, 20, 256), (1, 80, 80, 128), (3, 80, 80, 64),
         (1, 160, 160, 8), (3, 160, 160, 32)]
IDS = [f"b{b}_{h}x{w}_c{c}" for b, h, w, c in CASES]


def _fixture():
    return np.load(os.path.join(G, "ghost_golden.npz"))


def _ints(shape, seed, lo, hi, dev, dtype):
    return torch.from_numpy(np.random.RandomState(seed).randint(lo, hi + 1, shape)).to(dev, dtype)


class _Slice:
    """A (B,C,H,W) tensor held at channels [off, off+C) of an NHWC buffer whose other channels hold SENT."""

    def __init__(self, t, off=8, extra=8):
        b, c, h, w = t.shape
        self.buf = torch.full((b, h, w, c + off + extra), SENT, dtype=t.dtype, device=t.device)
        self.buf[..., off : off + c] = t.permute(0, 2, 3, 1)
        self.off, self.c = off, c
        self.ptr, self.pitch = self.buf.data_ptr() + off * self.buf.element_size(), self.buf.shape[3]

    def sub(self, coff, c):
        """the channels [coff, coff+c) of this view, as a view of the same buffer"""
        v = _Slice.__new__(_Slice)
        v.buf, v.off, v.c, v.pitch = self.buf, self.off + coff, c, self.pitch
        v.ptr = self.ptr + coff * self.buf.element_size()
        return v

    def nchw(self):
        return self.buf[..., self.off : self.off + self.c].permute(0, 3, 1, 2)

    def untouched(self):
        return bool((self.buf[..., : self.off] == SENT).all()) and bool((self.buf[..., self.off + self.c :] == SENT).all())


def _dw(x, w, bias=None, flip=False):
    """float64 depthwise 5x5 / pad 2 conv (flip: with the taps rotated 180 degrees = the data gradient)"""
    w = w.double().view(-1, 1, 5, 5)
    return F.conv2d(x.double(), w.flip(2, 3) if flip else w, None if bias is None else bias.double(), padding=2, groups=w.shape[0])


def _fwd(x, wt, bias, y, res=None, x_out=None, x_res=None, act=_lib.ACT_NONE, slope=0.0, flip=0):
    b, c, h, w = x.nchw().shape
    v = lambda s: (s.ptr, s.pitch) if s is not None else (None, 0)  # noqa: E731
    rc = _lib.lib().y5_dwconv_fwd(x.ptr, x.pitch, wt.data_ptr(), bias.data_ptr() if bias is not None else None, y.ptr, y.pitch, *v(res),
                                  *v(x_res), *v(x_out), b, h, w, c, 5, 1, act, slope, flip, _lib.dtype_code(x.buf.dtype),
                                  _lib.stream_ptr(x.buf.device))
    assert rc == 0, _lib.lib().y5_last_error()


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_dwconv_forward_forms_bit_exact(cuda, dtype, case):
    """act(dw(x) + b) + res with LeakyReLU(0.25) and none; the two-output GhostBottleneck form writing in place over its residuals;
    SiLU within one unit in the last place."""
    b, h, w, c = case
    x = _Slice(_ints((b, c, h, w), 1, -2, 2, cuda, dtype))
    wt = _ints((c, 25), 2, -1, 1, cuda, dtype)
    bias = _ints((c,), 3, -2, 2, cuda, torch.float32)
    r = _ints((b, c, h, w), 4, -3, 3, cuda, dtype)
    ref = _dw(x.nchw(), wt, bias)
    y = _Slice(torch.zeros(b, c, h, w, dtype=dtype, device=cuda), off=16)
    _fwd(x, wt, bias, y)
    assert torch.equal(y.nchw().double(), ref) and y.untouched() and x.untouched()
    res = _Slice(r.clone(), off=24, extra=0)
    _fwd(x, wt, bias, res, res=res, act=_lib.ACT_LEAKY, slope=0.25)  # in place: y aliases the residual
    assert torch.equal(res.nchw().double(), torch.where(ref > 0, ref, 0.25 * ref) + r.double()) and res.untouched()
    # GhostBottleneck: out[:, :c] = x + res[:, :c] and out[:, c:] = dw(x) + b + res[:, c:], in place over one 2c-channel slice
    r2 = _ints((b, 2 * c, h, w), 5, -3, 3, cuda, dtype)
    out = _Slice(r2.clone())
    first, second = out.sub(0, c), out.sub(c, c)
    _fwd(x, wt, bias, second, res=second, x_out=first, x_res=first)
    want = torch.cat((x.nchw().double(), ref), 1) + r2.double()
    assert torch.equal(out.nchw().double(), want) and out.untouched()
    # SiLU: fp32(acc + b) then x * sigmoid(x), rounded once; the exact value is an integer sum, so 1 ulp of the result's dtype
    ys = _Slice(torch.zeros(b, c, h, w, dtype=dtype, device=cuda))
    _fwd(x, wt, bias, ys, act=_lib.ACT_SILU)
    exact = F.silu(ref)
    ulp = torch.finfo(dtype).eps * torch.maximum(exact.abs(), torch.full_like(exact, torch.finfo(dtype).tiny))
    assert bool(((ys.nchw().double() - exact).abs() <= ulp).all())


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_dwconv_data_gradient_bit_exact(cuda, dtype, case):
    """dx = dw^T(dy) + g: the forward kernel with the taps rotated, adding the gradient that reaches x through the concat."""
    b, h, w, c = case
    dy = _Slice(_ints((b, c, h, w), 6, -2, 2, cuda, dtype))
    wt = _ints((c, 25), 7, -1, 1, cuda, dtype)
    g = _Slice(_ints((b, c, h, w), 8, -3, 3, cuda, dtype), off=0, extra=16)
    dx = _Slice(torch.zeros(b, c, h, w, dtype=dtype, device=cuda), off=16, extra=0)
    _fwd(dy, wt, None, dx, res=g, flip=1)
    xr = torch.zeros(b, c, h, w, dtype=torch.float64, device=cuda, requires_grad=True)
    _dw(xr, wt).backward(dy.nchw().double())  # autograd's dx of the depthwise conv
    assert torch.equal(_dw(dy.nchw(), wt, flip=True), xr.grad)
    assert torch.equal(dx.nchw().double(), xr.grad + g.nchw().double()) and dx.untouched() and g.untouched()


def _wgrad(x, dy):
    b, c, h, w = x.nchw().shape
    dw = torch.full((c, 1, 5, 5), 123.0, device=x.buf.device)  # overwritten
    rc = _lib.lib().y5_dwconv_wgrad(x.ptr, x.pitch, dy.ptr, dy.pitch, dw.data_ptr(), b, h, w, c, 5, 1, _lib.dtype_code(x.buf.dtype),
                                    _lib.stream_ptr(x.buf.device))
    assert rc == 0, _lib.lib().y5_last_error()
    return dw


def _wgrad_ref(x, dy):
    c = x.shape[1]
    return torch.nn.grad.conv2d_weight(x.double(), (c, 1, 5, 5), dy.double(), padding=2, groups=c)


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_dwconv_weight_gradient(cuda, dtype, case):
    """Exact on integer data (every partial sum of at most 4*B*H*W is an integer below 2^24, so any summation order gives the same
    fp32 value); on Gaussian data within the summation bound 2 n 2^-24 sum |x * dy| with n = B*H*W, whatever order the atomics take."""
    b, h, w, c = case
    x, dy = _Slice(_ints((b, c, h, w), 9, -2, 2, cuda, dtype)), _Slice(_ints((b, c, h, w), 10, -2, 2, cuda, dtype), off=0)
    assert torch.equal(_wgrad(x, dy).double(), _wgrad_ref(x.nchw(), dy.nchw()))
    gen = torch.Generator(device=cuda).manual_seed(11)
    xg = _Slice(torch.randn(b, c, h, w, device=cuda, generator=gen).to(dtype))
    dg = _Slice(torch.randn(b, c, h, w, device=cuda, generator=gen).to(dtype))
    got, ref = _wgrad(xg, dg).double(), _wgrad_ref(xg.nchw(), dg.nchw())
    # products of two fp16 / bf16 values are exact in fp32; summing n of them in any order errs by at most
    # gamma_(n-1) = (n-1)u / (1 - (n-1)u) <= 2 n u times the sum of their magnitudes (u = 2^-24, (n-1)u <= 1/2)
    bound = 2 * (b * h * w) * 2.0**-24 * _wgrad_ref(xg.nchw().abs(), dg.nchw().abs())
    assert bool(((got - ref).abs() <= bound + 1e-30).all()), float(((got - ref).abs() / (bound + 1e-30)).max())
    assert x.untouched() and dy.untouched()


def _image(shape, seed):
    return torch.from_numpy(np.random.RandomState(seed).uniform(0, 1, shape).astype(np.float32))


def _full_model(dev, dtype, seed=20):
    from yolov5_b200.cfg import model_cfg
    from yolov5_b200.models.yolo import DetectionModel

    sd = ghost_ref.synth_state_dict(model_cfg("yolov5s-ghost"), seed=seed, head_bias="hot")
    m = DetectionModel("yolov5s-ghost")
    m.load_state_dict(sd)
    return m.to(dev, dtype).eval(), sd


@pytest.mark.parametrize("dtype,hw", [(torch.float16, (256, 256)), (torch.float16, (192, 320)), (torch.bfloat16, (256, 192))], ids=str)
def test_full_model_vs_oracle(cuda, dtype, hw):
    from yolov5_b200.cfg import model_cfg

    m, sd = _full_model(cuda, dtype)
    x = _image((2, 3, *hw), 21)
    with torch.no_grad():
        z, raws = m(x.to(cuda, dtype))
        zr, _ = ghost_ref.forward(model_cfg("yolov5s-ghost"), sd, x.to(dtype).float(), fused=True)
    err = float((z.float().cpu() - zr).abs().max() / zr.abs().max())
    assert err < (2e-2 if dtype == torch.float16 else 6e-2), err


def test_full_model_augment(cuda):
    m, _ = _full_model(cuda, torch.float16)
    x = _image((1, 3, 256, 320), 22).to(cuda, torch.float16)
    z, _ = m(x)
    za, _ = m(x, augment=True)
    n0 = z.shape[1] - z.shape[1] // 21  # the full-scale copy without its stride-32 rows (1/21 of the rows)
    assert torch.isfinite(za).all() and torch.equal(za[:, :n0], z[:, :n0])


def test_single_layers_vs_oracle(cuda):
    """GhostConv (stride 2, 3x3 cv1) and GhostBottleneck as single-layer programs."""
    from yolov5_b200.models import common as mc

    torch.manual_seed(0)
    for mod, cin, fn in ((mc.GhostConv(32, 64, 3, 2), 32, lambda sd, x: ghost_ref.ghost_conv(sd, "l", x, 3, 2)),
                         (mc.GhostBottleneck(64, 64), 64, lambda sd, x: ghost_ref.ghost_bottleneck(sd, "l", x))):
        for bn in (q for q in mod.modules() if isinstance(q, torch.nn.BatchNorm2d)):
            bn.eps = 1e-3
            bn.weight.data.uniform_(0.5, 1.5)
            bn.running_mean.normal_(0, 0.1)
            bn.running_var.uniform_(0.5, 1.5)
        sd = {f"l.{k}": v.double() if v.is_floating_point() else v for k, v in mod.state_dict().items()}
        x = _image((2, cin, 40, 24), 23)
        m = mod.to(cuda).half().eval()
        with torch.no_grad():
            y = m(x.to(cuda).half())
        ref = fn(sd, x.half().double())
        assert y.shape == ref.shape
        assert float((y.double().cpu() - ref).abs().max()) <= 2e-2 * float(ref.abs().max())


def _small_model(dev, dtype):
    from yolov5_b200 import compat
    from yolov5_b200.models.yolo import DetectionModel

    compat.install()
    ck = torch.load(os.path.join(G, "ref_ghost_tiny.pt"), map_location="cpu", weights_only=False)
    m = DetectionModel(json.loads(str(_fixture()["small_cfg"])))
    m.load_state_dict({k: v.float() if v.is_floating_point() else v for k, v in ck["model"].state_dict().items()})
    return m.to(dev, dtype).eval() if dtype is not None else m.to(dev)


def test_forward_vs_reference_golden(cuda):
    f = _fixture()
    x = _image(tuple(f["x_shape"]), int(f["x_seed"]))
    zg = f["z"]
    sc = np.abs(zg).max()
    for mdt, xdt, tol in ((torch.float16, torch.float32, 2e-2), (torch.float16, torch.float16, 2e-2), (torch.bfloat16, torch.bfloat16, 6e-2)):
        m = _small_model(cuda, mdt)
        with torch.no_grad():
            z, raws = m(x.to(cuda, xdt))
        assert z.dtype == mdt and z.shape == zg.shape
        e = np.abs(z.float().cpu().numpy() - zg).max()
        assert e <= tol * sc, (mdt, xdt, e / sc)
        for i, r in enumerate(raws):
            rg = f[f"raw{i}"]
            assert np.abs(r.float().cpu().numpy() - rg).max() <= tol * np.abs(rg).max(), (mdt, i)


def test_reference_checkpoint_attempt_load_and_nms(cuda):
    from yolov5_b200.models.experimental import attempt_load
    from yolov5_b200.utils.general import non_max_suppression

    m = attempt_load(os.path.join(G, "ref_ghost_tiny.pt"), device=cuda)
    f = _fixture()
    x = _image(tuple(f["x_shape"]), int(f["x_seed"]))
    z = m.half()(x.to(cuda).half())[0]
    assert np.abs(z.float().cpu().numpy() - f["z"]).max() <= 2e-2 * np.abs(f["z"]).max()
    out = non_max_suppression(z.float(), conf_thres=0.0, iou_thres=0.45, max_det=50)
    assert len(out) == 1 and out[0].shape[1] == 6 and 0 < out[0].shape[0] <= 50


def _train_model(dev):
    from yolov5_b200.cfg import HYP_SCRATCH_LOW

    m = _small_model(dev, None).train()
    m.hyp = dict(HYP_SCRATCH_LOW)
    return m


def _grad_errors(grads, f):
    """(total relative L2 error, sorted [(per-tensor relative error, key)]) of {key: gradient} against the fixture's gradients"""
    errs, num, den = [], 0.0, 0.0
    for k, got in grads.items():
        gr = torch.from_numpy(f[f"grad:{k}"].astype(np.float64))
        n, d = float(gr.norm()), float((got.detach().double().cpu() - gr).norm())
        num, den = num + d * d, den + n * n
        if n > 0:
            errs.append((d / n, k))
    return (num / den) ** 0.5, sorted(errs)


def test_amp_training_step_vs_reference(cuda):
    """One fp16-autocast step on the device against the reference's fp32 step on the CPU: loss items, and every parameter's
    gradient (relative L2 error per tensor and over the whole model).

    This network's gradients are ill-conditioned in low precision: a GhostBottleneck's second BatchNorm has no activation and
    feeds a batch-statistics BatchNorm, so its bias gradient cancels to nearly zero (the fp32 reference moves it by >100 % between
    two summation orders), and the error of every fp16 rounding grows through 30 such blocks.  The same step restated in pure
    fp16 torch on the CPU errs by 0.118 in total against the fixture.  Measured on an H100 80GB HBM3 (700 W), the engine's step
    errs by 0.118 in total, 0.10 for the median tensor and 0.146 for the worst depthwise weight; the bounds below leave room
    above those numbers.  test_ghost_layer_training_vs_float64 checks the Ghost layers' training path to 3 %."""
    from oracle.loss_ref import synth_targets
    from yolov5_b200.utils.loss import ComputeLoss

    f = _fixture()
    shape, (s_img, s_tgt) = tuple(f["train_shape"]), f["train_seeds"].tolist()
    img = torch.from_numpy(np.random.RandomState(s_img).randint(0, 256, shape).astype(np.uint8)).to(cuda)
    targets = torch.from_numpy(synth_targets(shape[0], seed=s_tgt, nc=3)).float().to(cuda)
    m = _train_model(cuda)
    with torch.autocast("cuda", dtype=torch.float16):
        p = m(img)
    loss, items = ComputeLoss(m)(p, targets)
    loss.backward()
    assert np.allclose(items.cpu().numpy(), f["items"], rtol=2e-2, atol=1e-4), (items, f["items"])
    total, errs = _grad_errors({k: q.grad for k, q in m.named_parameters()}, f)
    dw = [e for e, k in errs if k.endswith("cv2.conv.weight") and m.get_parameter(k).shape[1] == 1]
    print(f"engine AMP: total {total:.4f}, median {errs[len(errs) // 2]}, worst {errs[-1]}, depthwise worst {max(dw):.4f}")
    assert len(dw) == 30  # every depthwise weight of the small model has a gradient in the report
    assert total <= 0.18 and errs[len(errs) // 2][0] <= 0.15 and max(dw) <= 0.25, (total, errs[len(errs) // 2], max(dw))


@pytest.mark.parametrize("layer", ["GhostConv", "GhostBottleneck"])
def test_ghost_layer_training_vs_float64(cuda, layer):
    """A GhostConv (3x3 stride-2 cv1) or GhostBottleneck in training mode under fp16 autocast -- batch-statistics BatchNorm, the
    depthwise forward, its data and weight gradients, the residual -- against float64 autograd of oracle/ghost_ref.py: every
    parameter's gradient and the input's within 3 % relative L2 (fp16 activations), the output within 1 %."""
    from yolov5_b200.models import common as mc

    torch.manual_seed(1)
    mod, cin = (mc.GhostConv(32, 64, 3, 2), 32) if layer == "GhostConv" else (mc.GhostBottleneck(64, 64), 64)
    for bn in (q for q in mod.modules() if isinstance(q, torch.nn.BatchNorm2d)):
        bn.eps = 1e-3
        bn.weight.data.uniform_(0.5, 1.5)
        bn.bias.data.normal_(0, 0.1)
    x = _image((4, cin, 48, 40), 24).to(cuda)
    gen = torch.Generator(device=cuda).manual_seed(25)
    sd = {f"l.{k}": v.detach().double().to(cuda).requires_grad_(v.is_floating_point() and "running" not in k)
          for k, v in mod.state_dict().items()}
    mod = mod.to(cuda).train()
    xe = x.clone().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.float16):
        y = mod(xe)
    dy = torch.randn(y.shape, device=cuda, generator=gen)
    (y.float() * dy).sum().backward()
    xr = x.double().requires_grad_(True)
    from oracle import model_ref

    prev, model_ref._BN_BATCH_STATS = model_ref._BN_BATCH_STATS, True
    try:
        yr = ghost_ref.ghost_conv(sd, "l", xr, 3, 2) if layer == "GhostConv" else ghost_ref.ghost_bottleneck(sd, "l", xr)
    finally:
        model_ref._BN_BATCH_STATS = prev
    (yr * dy.double()).sum().backward()
    assert float((y.detach().double() - yr.detach()).norm() / yr.detach().norm()) <= 1e-2
    pairs = [("x", xe.grad, xr.grad)] + [(k, q.grad, sd[f"l.{k}"].grad) for k, q in mod.named_parameters()]
    for k, got, ref in pairs:
        e = float((got.double() - ref).norm() / ref.norm())
        assert e <= 3e-2, (layer, k, e)


def test_graphed_train_step_matches_eager(cuda):
    """GraphedTrainStep captures yolov5s-ghost's small model: its steps give the eager loop's loss items and weights."""
    from oracle import loss_ref
    from yolov5_b200.utils.loss import ComputeLoss
    from yolov5_b200.utils.torch_utils import GraphedTrainStep, smart_optimizer

    ma, mb = _train_model(cuda), _train_model(cuda)
    imgs = [torch.from_numpy(np.random.RandomState(70 + i).randint(0, 256, (2, 3, 128, 128)).astype(np.uint8)).to(cuda) for i in range(3)]
    tgts = [torch.from_numpy(loss_ref.synth_targets(2, seed=80 + i, nc=3)).float().to(cuda) for i in range(3)]
    oa = smart_optimizer(ma, "SGD", lr=0.01, momentum=0.937, decay=5e-4)
    ob = smart_optimizer(mb, "SGD", lr=0.01, momentum=0.937, decay=5e-4)
    step = GraphedTrainStep(ma, ComputeLoss(ma), oa, batch=2, size=128)
    lb, sb = ComputeLoss(mb), torch.amp.GradScaler("cuda")
    w0 = torch.cat([v.detach().flatten() for v in ma.parameters()]).clone()
    for i in range(3):
        items_a = step(imgs[i], tgts[i]).clone()
        with torch.autocast("cuda", dtype=torch.float16):
            pb = mb(imgs[i])
        loss_b, items_b = lb(pb, tgts[i])
        sb.scale(loss_b).backward()
        ob.fused_step(scaler=sb, max_norm=10.0, model=mb)
        ob.zero_grad()
        torch.cuda.synchronize()
        assert torch.allclose(items_a, items_b, rtol=3e-2, atol=1e-4), (i, items_a, items_b)
        if i == 0:
            wa = torch.cat([v.detach().flatten() for v in ma.parameters()])
            wb = torch.cat([v.detach().flatten() for v in mb.parameters()])
            moved = float((wb - w0).norm())
            assert moved > 0 and float((wa - wb).norm()) <= 0.05 * moved, (float((wa - wb).norm()), moved)
    assert all(bool(torch.isfinite(v).all()) for v in ma.parameters())
