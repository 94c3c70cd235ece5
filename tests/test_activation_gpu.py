"""GPU: ReLU / LeakyReLU Conv activations (Y5_ACT_LEAKY) through every layer that carries an activation.

conv_gemm, exact.  The integer operands of tests/test_conv_exact_gpu.py (every fp32 partial sum an exact integer) with the activation
v > 0 ? v : slope * v on v = fp32(acc + bias) (its own kernel instantiation, epi 2): the output must equal fp32(leaky32(v) + residual) rounded once to the dtype, value for
value, for ReLU (slope 0) and LeakyReLU(0.1), (0.01), on every case of that file's list (LINEAR, IM2COL, patch fetches, both stem
views, the staged epilogue, residual separate and in place), each with the default TMA epilogue and with direct register stores
(reserved bit 16); the plan query asserts the path.  The CUDA-core cross-check kernel gives the same values.

BN + activation passes, exact.  y5_bn_act_fwd in training mode equals the host formula applied to the kernel's own BN output t
(its ACT_NONE result): z = round(t > 0 ? t : fp32(slope * t)), and with a residual round(round(...) + r).  Backward: y5_bn_act_bwd
with LeakyReLU equals, bit for bit (dy, dgamma, dbeta), the linear backward fed du = round(t > 0 ? dz : fp32(dz * slope)) computed on
the host -- the same apply pass on the parked du; the SyncBN forms (a row count, the split backward; no all-reduce: one rank) equal the plain ones.

Models.  yolov5n from the reference's yolov5s-LeakyReLU.yaml (scaled to n) against the oracle and the reference's stored forward,
yolov5n-seg and a classifier with LeakyReLU against the oracle, under test_model_gpu.py's tolerance rule; a LeakyReLU yolov5n
training step under test_train_gpu.py's gradient criteria, and the same step under GraphedTrainStep; a model mixing SiLU and
LeakyReLU layers (C3 cv1 / cv2 with different activations run as two GEMMs)."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch
from torch import nn

from oracle import cls_ref, loss_ref, model_ref
from yolov5_b200 import _lib
from yolov5_b200.cfg import HYP_SCRATCH_LOW, model_cfg
from yolov5_b200.models.common import Conv

from .act_ref import cls_forward, conv_activation
from .act_ref import forward as oracle_forward
from .test_conv_exact_gpu import CASES, DT_IDS, DTYPES, Operands, _first_bad, form_of, key_of

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
SLOPES = [0.0, 0.1, 0.01]


@pytest.fixture
def restore_act():
    yield
    Conv.default_act = nn.SiLU()


def _leaky32(v: torch.Tensor, slope: float) -> torch.Tensor:
    v = v.float()
    return torch.where(v > 0, v, v * torch.tensor(slope, dtype=torch.float32, device=v.device))


# ------------------------------------------------------------------------------------------------------------------------------
# conv_gemm epilogue and the CUDA-core cross-check
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_conv_leaky_exact(cuda, case, dtype):
    op = Operands(case, dtype, cuda)
    pre = op.conv64()
    res32 = op.res.float()
    for direct in ((False, True) if not case.staged else (False,)):
        if direct:
            op.desc.reserved |= 16
        op.desc.act = _lib.ACT_LEAKY
        info = op.info()
        # the LeakyReLU epilogue is an instantiation of its own (epi 2) with the tile of the case's SiLU / linear plan
        assert info["epi"] == 2 and (form_of(info), key_of(info) - 20000, info["cluster"], info["staged"]) == (
            case.form, case.key, case.csize, int(case.staged)), info
        assert not (direct and info["tma_epi"]), info  # reserved bit 16: direct register stores
        for slope in SLOPES:
            op.desc.act_slope = slope
            ref = (_leaky32(pre, slope) + res32).to(dtype).double()
            for in_place in (False, True):
                got = op.run(act=_lib.ACT_LEAKY, in_place=in_place)
                bad = got != ref
                assert not bad.any(), f"{case.id} slope {slope} {'direct' if direct else 'default'} {'in place' if in_place else ''}: " + \
                    _first_bad(bad, got, ref)


def test_conv_leaky_paths_cover_tma_and_direct(cuda):
    seen = set()
    for c in CASES:
        op = Operands(c, torch.float16, cuda)
        op.desc.act, op.desc.act_slope = _lib.ACT_LEAKY, 0.1
        info = op.info()
        seen.add((info["tma_epi"], info["staged"], info["opt"]))
    assert {(1, 0, 0), (0, 1, 1), (0, 0, 0), (0, 0, 1)} <= seen, seen  # TMA, staged, direct (plain and OPT) epilogues


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_conv_direct_kernel_leaky(cuda, dtype):
    """y5_conv_direct_fwd (fp32 CUDA-core accumulation) with the same activation gives the same values."""
    for case in (CASES[0], CASES[6], CASES[-2]):
        op = Operands(case, dtype, cuda)
        pre = op.conv64()
        for slope in SLOPES:
            d = op.desc
            out = torch.zeros(op.M, case.cout, dtype=dtype, device=cuda)
            d.out, d.out_pitch, d.residual, d.res_pitch = out.data_ptr(), case.cout, None, 0
            d.act, d.act_slope = _lib.ACT_LEAKY, slope
            _lib.check(_lib.lib().y5_conv_direct_fwd(C.byref(d), C.c_void_p(_lib.stream_ptr(cuda))), "conv_direct")
            torch.cuda.synchronize()
            ref = _leaky32(pre, slope).to(dtype)
            assert torch.equal(out, ref), (case.id, slope)


# ------------------------------------------------------------------------------------------------------------------------------
# BatchNorm + activation passes
def _p(t):
    return t.data_ptr() if t is not None else None


class BnCase:
    """Integer-valued y, dz and residual (NHWC rows x channels) with gamma / beta in a training BN layer."""

    def __init__(self, dev, dtype, rows=3000, c=72, seed=0):
        g = torch.Generator().manual_seed(seed)
        self.dev, self.dtype, self.rows, self.c = dev, dtype, rows, c
        self.code = _lib.dtype_code(dtype)
        self.y = torch.randint(-8, 9, (rows, c), generator=g).to(dev, dtype)
        self.dz = torch.randint(-4, 5, (rows, c), generator=g).to(dev, dtype)
        self.res = torch.randint(-4, 5, (rows, c), generator=g).to(dev, dtype)
        self.gamma = (torch.rand(c, generator=g) + 0.5).to(dev)
        self.beta = (torch.randn(c, generator=g) * 0.5).to(dev)
        self.st = C.c_void_p(_lib.stream_ptr(dev))

    def forward(self, act, slope, residual=None, sync=False):
        lib, c = _lib.lib(), self.c
        ws = torch.zeros(2 * c + 1, dtype=torch.float64, device=self.dev)
        mean, invstd = torch.empty(c, device=self.dev), torch.empty(c, device=self.dev)
        rm, rv = torch.zeros(c, device=self.dev), torch.ones(c, device=self.dev)
        z = torch.empty_like(self.y)
        count = _p(ws[2 * c :]) if sync else None
        _lib.check(lib.y5_bn_stats(_p(self.y), c, self.rows, c, self.code, _p(ws), count, self.st), "bn_stats")
        _lib.check(lib.y5_bn_act_fwd(_p(self.y), c, _p(z), c, self.rows, c, self.code, _p(mean), _p(invstd), _p(self.gamma), _p(self.beta), act,
                                     slope, _p(ws), count, 1e-3, 0.03, _p(rm), _p(rv), _p(residual), c if residual is not None else 0, self.st),
                   "bn_act_fwd")
        torch.cuda.synchronize()
        return z, mean, invstd

    def backward(self, dz, mean, invstd, act, slope, split=False):
        lib, c = _lib.lib(), self.c
        ws = torch.zeros(2 * c + 1, dtype=torch.float64, device=self.dev)
        dy = torch.empty_like(self.y)
        dg, db = torch.empty(c, device=self.dev), torch.empty(c, device=self.dev)
        common = (_p(self.y), c, _p(dz), c, _p(dy), c, self.rows, c, self.code, _p(mean), _p(invstd), _p(self.gamma))
        if split:
            _lib.check(lib.y5_bn_act_bwd_reduce(*common, _p(self.beta), act, slope, _p(dg), _p(db), _p(ws), self.st), "reduce")
            ws[2 * c] = float(self.rows)  # what the forward's y5_bn_stats counted (one rank)
            _lib.check(lib.y5_bn_act_bwd_apply(*common, act, _p(ws), _p(ws[2 * c :]), self.st), "apply")
        else:
            _lib.check(lib.y5_bn_act_bwd(*common, _p(self.beta), act, slope, _p(dg), _p(db), _p(ws), self.st), "bn_act_bwd")
        torch.cuda.synchronize()
        return dy, dg, db


@pytest.mark.parametrize("slope", SLOPES)
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_bn_pass_leaky_forward_exact(cuda, dtype, slope):
    b = BnCase(cuda, dtype)
    t, mean, invstd = b.forward(_lib.ACT_NONE, 0.0)  # the kernel's BN output, rounded to the dtype
    for residual in (None, b.res):
        ref = _leaky32(t, slope).to(dtype)
        if residual is not None:
            ref = (ref.float() + residual.float()).to(dtype)
        for sync in (False, True):
            z, m2, s2 = b.forward(_lib.ACT_LEAKY, slope, residual, sync)
            assert torch.equal(m2, mean) and torch.equal(s2, invstd)
            bad = z.view(torch.int16) != ref.view(torch.int16)
            assert not bad.any(), (slope, residual is not None, sync, int(bad.sum()))


@pytest.mark.parametrize("slope", SLOPES)
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_bn_pass_leaky_backward_exact(cuda, dtype, slope):
    b = BnCase(cuda, dtype, seed=1)
    t, mean, invstd = b.forward(_lib.ACT_NONE, 0.0)
    s32 = torch.tensor(slope, dtype=torch.float32, device=cuda)
    dzf = b.dz.float()
    du = torch.where(t.float() > 0, dzf, dzf * s32).to(dtype)  # torch's leaky_relu_backward in fp32, rounded to the dtype
    ref = b.backward(du, mean, invstd, _lib.ACT_NONE, 0.0)
    if slope == 0.0:  # ReLU: du is integer valued, so every partial sum is exact and dbeta is the float64 column sum
        assert torch.equal(ref[2], du.double().sum(0).float())
    for split in (False, True):  # split: the SyncBN reduce pass (this rank's dgamma / dbeta) + the apply pass over one rank
        got = b.backward(b.dz, mean, invstd, _lib.ACT_LEAKY, slope, split)
        assert torch.equal(got[0].view(torch.int16), ref[0].view(torch.int16)), (slope, split)
        assert torch.equal(got[1], ref[1]) and torch.equal(got[2], ref[2]), (slope, split)


# ------------------------------------------------------------------------------------------------------------------------------
# models
def _image(shape, seed):
    return torch.from_numpy(np.random.RandomState(seed).uniform(0, 1, shape).astype(np.float32))


def _check(cfg, sd, x, dtype, dev, model):
    """test_model_gpu.py's rule: err(engine) <= 1e-3 max|oracle| + 1.5 err(torch's own fp16 evaluation of the reference)."""
    seg = "Segment" in json.dumps(cfg["head"])
    with torch.no_grad():
        ref = oracle_forward(cfg, sd, x.to(dtype).float(), fused=True)
        sd_d = {k: (v.to(dev, dtype) if v.is_floating_point() else v.to(dev)) for k, v in sd.items()}
        low = oracle_forward(cfg, sd_d, x.to(dev, dtype), fused=True)
    out = model(x.to(dev, dtype))
    pairs = [("z", out[0], ref[0], low[0])]
    raws, rraws, lraws = (out[2], ref[2], low[2]) if seg else (out[1], ref[1], low[1])
    pairs += [(f"raw{l}", a, r, lo) for l, (a, r, lo) in enumerate(zip(raws, rraws, lraws))]
    if seg:
        pairs.append(("proto", out[1], ref[1], low[1]))
    for tag, got, r, lo in pairs:
        got, lo = got.float().cpu(), lo.float().cpu()
        scale = float(r.abs().max())
        e, el = float((got - r).abs().max()), float((lo - r).abs().max())
        assert got.shape == r.shape and e <= 1e-3 * scale + 1.5 * el, (tag, e / scale, el / scale)
    return out


def test_leaky_yolov5n_vs_oracle_and_reference_golden(cuda, restore_act):
    from yolov5_b200.models.yolo import DetectionModel

    g = np.load(os.path.join(G, "leaky_forward.npz"))
    cfg = json.loads(str(g["cfg"]))
    sd = model_ref.synth_state_dict(cfg, seed=int(g["seed"][0]))
    m = DetectionModel(cfg)
    m.load_state_dict(sd)
    m = m.to(cuda, torch.float16).eval()
    out = _check(cfg, sd, _image(tuple(g["shape"]), int(g["seed"][1])), torch.float16, cuda, m)
    z = out[0].float().cpu().numpy()
    assert np.abs(z - g["z"]).max() <= 2e-2 * np.abs(g["z"]).max()


def test_leaky_segment_and_relu_bf16(cuda, restore_act):
    from yolov5_b200.models.yolo import DetectionModel, SegmentationModel

    for name, act, dtype, cls in (("yolov5n-seg", "nn.LeakyReLU(0.1)", torch.float16, SegmentationModel),
                                  ("yolov5n", "nn.ReLU()", torch.bfloat16, DetectionModel)):
        cfg = model_cfg(name)
        cfg["activation"] = act
        sd = model_ref.synth_state_dict(cfg, seed=12)
        m = cls(cfg)
        Conv.default_act = nn.SiLU()
        m.load_state_dict(sd)
        _check(cfg, sd, _image((1, 3, 64, 96), 112), dtype, cuda, m.to(cuda, dtype).eval())


def test_leaky_classifier_vs_oracle(cuda, restore_act):
    from yolov5_b200.models.yolo import ClassificationModel, DetectionModel

    cfg = model_cfg("yolov5n")
    cfg["activation"] = "nn.LeakyReLU(0.01)"
    m = ClassificationModel(model=DetectionModel(cfg), nc=10, cutoff=10)
    Conv.default_act = nn.SiLU()
    assert {type(c.act) for c in m.modules() if isinstance(c, Conv)} == {nn.LeakyReLU}
    sd = cls_ref.synth_state_dict(cfg, 10, seed=3)
    m.load_state_dict(sd)
    x = _image((4, 3, 64, 64), 4)
    with torch.no_grad():
        ref = cls_forward(cfg, sd, x.half().float())  # the activation comes from the model dict
        sd_d = {k: (v.to(cuda).half() if v.is_floating_point() else v.to(cuda)) for k, v in sd.items()}
        low = cls_forward(cfg, sd_d, x.to(cuda).half(), fused=True).float().cpu()
    got = m.to(cuda).half().eval()(x.to(cuda).half()).float().cpu()
    scale = float(ref.abs().max())
    e, el = float((got - ref).abs().max()), float((low - ref).abs().max())
    assert e <= 1e-3 * scale + 1.5 * el, (e / scale, el / scale)


def test_mixed_silu_and_leaky_layers_run(cuda):
    from yolov5_b200.models.yolo import DetectionModel

    cfg = model_cfg("yolov5n")
    sd = model_ref.synth_state_dict(cfg, seed=5)
    m = DetectionModel("yolov5n")
    m.load_state_dict(sd)
    leaky = {"model.0", "model.2.cv2", "model.4.m.0.cv1", "model.9.cv1", "model.13.cv3", "model.17.cv1"}
    for name, mod in m.named_modules():
        if isinstance(mod, Conv) and name in leaky:
            mod.act = nn.LeakyReLU(0.1)
    acts = {name: mod.act for name, mod in m.named_modules() if isinstance(mod, Conv)}
    assert sum(isinstance(a, nn.LeakyReLU) for a in acts.values()) == len(leaky)

    def mixed(y, p):  # the oracle's Conv activation chosen per module prefix
        return nn.functional.leaky_relu(y, 0.1) if p in leaky else nn.functional.silu(y)

    x = _image((2, 3, 96, 128), 6)
    orig = model_ref.conv_block

    def conv_block(sd_, p, x_, k=1, s=1, pad=None, fused=False, act=True):
        y = orig(sd_, p, x_, k, s, pad, fused, act=False)
        return mixed(y, p) if act else y

    model_ref.conv_block = conv_block
    try:
        with torch.no_grad():
            ref = model_ref.forward(cfg, sd, x.half().float(), fused=True)
            sd_d = {k: (v.to(cuda).half() if v.is_floating_point() else v.to(cuda)) for k, v in sd.items()}
            low = model_ref.forward(cfg, sd_d, x.to(cuda).half(), fused=True)
    finally:
        model_ref.conv_block = orig
    out = m.to(cuda).half().eval()(x.to(cuda).half())
    for got, r, lo in zip([out[0], *out[1]], [ref[0], *ref[1]], [low[0], *low[1]]):
        got, lo = got.float().cpu(), lo.float().cpu()
        scale = float(r.abs().max())
        e, el = float((got - r).abs().max()), float((lo - r).abs().max())
        assert e <= 1e-3 * scale + 1.5 * el, (e / scale, el / scale)
    # and one training step: every parameter gets a finite gradient
    mt = DetectionModel("yolov5n")
    mt.load_state_dict(sd)
    for name, mod in mt.named_modules():
        if isinstance(mod, Conv) and name in leaky:
            mod.act = nn.LeakyReLU(0.1)
    mt = mt.to(cuda).train()
    mt.hyp = dict(HYP_SCRATCH_LOW)
    from yolov5_b200.utils.loss import ComputeLoss

    img = (torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(7)) * 255).to(torch.uint8).to(cuda)
    with torch.autocast("cuda", dtype=torch.float16):
        p = mt(img)
    loss, _ = ComputeLoss(mt)(p, torch.from_numpy(loss_ref.synth_targets(2, seed=8)).float().to(cuda))
    loss.backward()
    assert all(q.grad is not None and bool(torch.isfinite(q.grad).all()) for q in mt.parameters())


def _leaky_train_model(dev, sd, cfg):
    from yolov5_b200.models.yolo import DetectionModel

    m = DetectionModel(cfg)
    Conv.default_act = nn.SiLU()
    m.load_state_dict(sd)
    m = m.to(dev).train()
    m.hyp = dict(HYP_SCRATCH_LOW)
    return m


def test_leaky_training_step_vs_oracle(cuda, restore_act):
    """test_train_gpu.py's criteria for one yolov5n step with LeakyReLU(0.1): raw maps and per-tensor gradient errors judged
    against torch-AMP's own error on the fp32 oracle."""
    from yolov5_b200.utils.loss import ComputeLoss

    from .test_train_gpu import _ref_train_step

    cfg = model_cfg("yolov5n")
    cfg["activation"] = "nn.LeakyReLU(0.1)"
    sd = model_ref.synth_state_dict(cfg, seed=21)
    shape, dtype = (4, 3, 128, 128), torch.float16
    img = (torch.rand(*shape, generator=torch.Generator().manual_seed(22)) * 255).to(torch.uint8)
    targets = torch.from_numpy(loss_ref.synth_targets(shape[0], seed=23)).float()
    with conv_activation(nn.LeakyReLU(0.1)):
        p32, _, g32 = _ref_train_step(cfg, sd, img, targets, cuda, None)
        pamp, _, gamp = _ref_train_step(cfg, sd, img, targets, cuda, dtype)
    m = _leaky_train_model(cuda, sd, cfg)
    with torch.autocast("cuda", dtype=dtype):
        p = m(img.to(cuda))
    for l, (a, r, lo) in enumerate(zip(p, p32, pamp)):
        sc = float(r.abs().max())
        e, el = float((a.detach().float() - r).abs().max()), float((lo.float() - r).abs().max())
        assert e <= 1e-3 * sc + 1.5 * el, ("raw", l, e / sc, el / sc)
    loss, _ = ComputeLoss(m)(p, targets.to(cuda))
    loss.backward()
    named = dict(m.named_parameters())
    ratios, mine_sq, amp_sq, ref_sq, worst = [], 0.0, 0.0, 0.0, (0.0, None)
    for k, gr in g32.items():
        got = named[k].grad
        assert got is not None, k
        n = float(gr.norm())
        if n == 0:
            continue
        e, el = float((got.float() - gr).norm()) / n, float((gamp[k].float() - gr).norm()) / n
        mine_sq, amp_sq, ref_sq = mine_sq + (e * n) ** 2, amp_sq + (el * n) ** 2, ref_sq + n * n
        r = e / (1e-3 + el)
        ratios.append(r)
        worst = max(worst, (r, k, e, el), key=lambda w: w[0])
    ratios.sort()
    summary = dict(n=len(ratios), median=ratios[len(ratios) // 2], worst=worst, total_mine=(mine_sq / ref_sq) ** 0.5,
                   total_amp=(amp_sq / ref_sq) ** 0.5)
    print("leaky train-step gradient report", summary)
    assert len(ratios) > 150, summary
    assert worst[0] <= 2.5 and summary["median"] <= 1.25, summary
    assert summary["total_mine"] <= 1e-3 + 1.5 * summary["total_amp"], summary


def test_leaky_graphed_train_step_matches_eager(cuda, restore_act):
    """GraphedTrainStep captures a LeakyReLU model: its steps give the eager fused loop's loss items and weights."""
    from yolov5_b200.utils.loss import ComputeLoss
    from yolov5_b200.utils.torch_utils import GraphedTrainStep, smart_optimizer

    cfg = model_cfg("yolov5n")
    cfg["activation"] = "nn.LeakyReLU(0.1)"
    sd = model_ref.synth_state_dict(cfg, seed=0)
    ma, mb = _leaky_train_model(cuda, sd, cfg), _leaky_train_model(cuda, sd, cfg)
    assert all(type(c.act) is nn.LeakyReLU for c in ma.modules() if isinstance(c, Conv))
    imgs = [torch.from_numpy(np.random.RandomState(10 + i).randint(0, 256, (2, 3, 128, 128)).astype(np.uint8)).to(cuda) for i in range(3)]
    tgts = [torch.from_numpy(loss_ref.synth_targets(2, seed=20 + i)).float().to(cuda) for i in range(3)]
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
