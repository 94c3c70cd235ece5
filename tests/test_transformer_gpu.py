"""GPU: C3TR transformer layers (reference models/common.py:115-160, 261-270).

Kernels.  y5_attention_fwd / y5_attention_bwd against float64 autograd of softmax(scale * Q K^T) V, for every built head dim,
L in {1, 7, 64, 65, 240, 400, 1600} (tails of every tile size, the P5 map at 640^2 and 1280^2), B in {1, 3}, fp16 and bf16,
near-uniform and sharp logits.  Q, K, V and O are channel slices of wider buffers whose other channels hold a sentinel that must
survive.  Criterion: err <= 1e-3 * max|ref| + 1.5 * err(torch evaluating the same expressions in the same dtype on the GPU).

Models.  yolov5s-transformer (C3TR at layer 8) against the float64 oracle (oracle/transformer_ref.py) and the reference's stored
forward, at widths 0.25 and 0.5 and one image at 0.75, 1.0 and 1.25 (head dims 96, 128, 160), square and rect, augment=True; the
reference-pickled checkpoint through attempt_load; an AMP training step against the oracle with every C3TR gradient in the
report; GraphedTrainStep against eager over three steps."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from yolov5_b200 import _lib

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")

DHS = [32, 64, 96, 128, 160]
LS = [1, 7, 64, 65, 240, 400, 1600]
DTYPES = [torch.float16, torch.bfloat16]
SENT = 3.0  # neighbouring channels hold this value before the launch and must hold it after


def _err(a, b):
    return float((a.detach().double() - b.detach().double()).abs().max())


class _Case:
    """Q, K, V at channel offsets 8, 8 + hd, 8 + 2 hd of a (B*L, 3 hd + 16) buffer; O at channel 8 of a (B*L, hd + 16) buffer."""

    def __init__(self, dev, B, L, heads, dh, dtype, sharp, seed):
        g = torch.Generator(device="cpu").manual_seed(seed)
        hd = heads * dh
        sig = 12.0 ** 0.5 if sharp else 0.3  # sharp: scaled logits with std ~12, a spread well over 30 in every long row
        self.q, self.k, self.v = ((torch.randn(B, L, hd, generator=g) * (sig if i < 2 else 1.0)).to(dtype) for i in range(3))
        self.do = torch.randn(B, L, hd, generator=g).to(dtype)
        self.B, self.L, self.heads, self.dh, self.hd, self.dtype, self.dev = B, L, heads, dh, hd, dtype, dev
        self.scale = dh ** -0.5
        self.qkv = torch.full((B * L, 3 * hd + 16), SENT, dtype=dtype, device=dev)
        for i, t in enumerate((self.q, self.k, self.v)):
            self.qkv[:, 8 + i * hd : 8 + (i + 1) * hd] = t.reshape(B * L, hd).to(dev)
        self.o = torch.full((B * L, hd + 16), SENT, dtype=dtype, device=dev)

    def ptr(self, t, coff):
        return t.data_ptr() + coff * t.element_size()

    def fwd(self, lse=None):
        hd = self.hd
        _lib.check(_lib.lib().y5_attention_fwd(self.ptr(self.qkv, 8), self.ptr(self.qkv, 8 + hd), self.ptr(self.qkv, 8 + 2 * hd), self.qkv.shape[1],
                                               self.ptr(self.o, 8), self.o.shape[1], lse.data_ptr() if lse is not None else None, self.B, self.L,
                                               self.heads, self.dh, self.scale, _lib.dtype_code(self.dtype),
                                               C.c_void_p(_lib.stream_ptr(self.dev))), "attention_fwd")

    def bwd(self, lse):
        hd, B, L = self.hd, self.B, self.L
        dob = torch.full((B * L, hd + 16), SENT, dtype=self.dtype, device=self.dev)
        dob[:, 8 : 8 + hd] = self.do.reshape(B * L, hd).to(self.dev)
        dqkv = torch.full((B * L, 3 * hd + 16), SENT, dtype=self.dtype, device=self.dev)
        delta = torch.empty(B * self.heads * L, dtype=torch.float32, device=self.dev)
        _lib.check(_lib.lib().y5_attention_bwd(self.ptr(self.qkv, 8), self.ptr(self.qkv, 8 + hd), self.ptr(self.qkv, 8 + 2 * hd), self.qkv.shape[1],
                                               self.ptr(self.o, 8), self.o.shape[1], self.ptr(dob, 8), dob.shape[1], lse.data_ptr(),
                                               delta.data_ptr(), self.ptr(dqkv, 8), self.ptr(dqkv, 8 + hd), self.ptr(dqkv, 8 + 2 * hd),
                                               dqkv.shape[1], B, L, self.heads, self.dh, self.scale, _lib.dtype_code(self.dtype),
                                               C.c_void_p(_lib.stream_ptr(self.dev))), "attention_bwd")
        return dqkv

    def heads_view(self, t):  # (B, L, hd) -> (B, heads, L, dh)
        return t.reshape(self.B, self.L, self.heads, self.dh).transpose(1, 2)

    def expr(self, dt, with_grad):
        """softmax(scale * q k^T) v and its gradients evaluated by torch in dtype dt on the GPU"""
        q, k, v = (self.heads_view(t.to(self.dev, dt)).requires_grad_(with_grad) for t in (self.q, self.k, self.v))
        o = torch.softmax((q @ k.transpose(-1, -2)) * self.scale, -1) @ v
        lse = torch.logsumexp((q.double() @ k.double().transpose(-1, -2)) * self.scale, -1) if dt == torch.float64 else None
        grads = None
        if with_grad:
            grads = torch.autograd.grad(o, (q, k, v), self.heads_view(self.do.to(self.dev, dt)))
        return o.detach(), lse, grads


def _bound(ref, yard):
    return 1e-3 * float(ref.abs().max()) + 1.5 * yard


@pytest.mark.parametrize("sharp", [False, True], ids=["uniform", "sharp"])
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("L", LS)
@pytest.mark.parametrize("dh", DHS)
def test_attention_kernels(cuda, dh, L, B, dtype, sharp):
    cs = _Case(cuda, B, L, 2, dh, dtype, sharp, seed=dh * 7919 + L * 31 + B * 7 + sharp)
    lse = torch.empty(B * 2 * L, dtype=torch.float32, device=cuda)
    cs.fwd(lse)
    cs.fwd(None)  # the logsumexp is optional and does not change O
    o_ref, lse_ref, g_ref = cs.expr(torch.float64, True)
    o_t, _, g_t = cs.expr(dtype, True)
    hd = cs.hd
    o = cs.heads_view(cs.o[:, 8 : 8 + hd].reshape(B, L, hd))
    assert bool((cs.o[:, :8] == SENT).all()) and bool((cs.o[:, 8 + hd :] == SENT).all()), "attention_fwd wrote outside its channels"
    eo = _err(o, o_ref)
    assert eo <= _bound(o_ref, _err(o_t, o_ref)), (eo, _err(o_t, o_ref))
    assert _err(lse.view(B, 2, L), lse_ref) <= 1e-3 * (1 + float(lse_ref.abs().max()))
    dqkv = cs.bwd(lse)
    assert bool((dqkv[:, :8] == SENT).all()) and bool((dqkv[:, 8 + 3 * hd :] == SENT).all()), "attention_bwd wrote outside its channels"
    gmax = max(float(g.abs().max()) for g in g_ref)  # dq and dk vanish exactly at L = 1: their scale is the largest gradient's
    for i, name in enumerate("qkv"):
        got = cs.heads_view(dqkv[:, 8 + i * hd : 8 + (i + 1) * hd].reshape(B, L, hd))
        e, yard = _err(got, g_ref[i]), _err(g_t[i], g_ref[i])
        assert e <= 1e-3 * gmax + 1.5 * yard, (name, e, yard, float(g_ref[i].abs().max()))


# ------------------------------------------------------------------------------------------------------------------------------
# models
def _image(shape, seed):
    return torch.from_numpy(np.random.RandomState(seed).uniform(0, 1, shape).astype(np.float32))


def _cfg(width):
    from yolov5_b200.cfg import model_cfg

    cfg = model_cfg("yolov5s-transformer")
    cfg["width_multiple"] = width
    return cfg


def _model(cfg, sd, dev, dtype):
    from yolov5_b200.models.yolo import DetectionModel

    m = DetectionModel(cfg)
    m.load_state_dict(sd)
    return m.to(dev, dtype).eval()


def _check(cfg, sd, x, dtype, dev, model):
    """test_model_gpu.py's rule: err(engine) <= 1e-3 max|oracle| + 1.5 err(torch's own evaluation of the oracle in `dtype`)."""
    from oracle import transformer_ref

    with torch.no_grad():
        ref = transformer_ref.forward(cfg, {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}, x.to(dtype).double(), fused=True)
        sd_d = {k: (v.to(dev, dtype) if v.is_floating_point() else v.to(dev)) for k, v in sd.items()}
        low = transformer_ref.forward(cfg, sd_d, x.to(dev, dtype), fused=True)
    out = model(x.to(dev, dtype))
    for tag, got, r, lo in [("z", out[0], ref[0], low[0])] + [(f"raw{l}", a, r, lo) for l, (a, r, lo) in enumerate(zip(out[1], ref[1], low[1]))]:
        got, lo = got.double().cpu(), lo.double().cpu()
        scale = float(r.abs().max())
        e, el = float((got - r).abs().max()), float((lo - r).abs().max())
        assert got.shape == r.shape and e <= 1e-3 * scale + 1.5 * el, (tag, e / scale, el / scale)
    return out


@pytest.mark.parametrize("width", [0.5, 0.25])
def test_transformer_model_vs_oracle_and_reference_golden(cuda, width):
    from oracle import transformer_ref

    g = np.load(os.path.join(G, f"transformer_forward_w{int(width * 100)}.npz"))
    cfg = _cfg(width)
    sd = transformer_ref.synth_state_dict(cfg, seed=int(g["seed"][0]))
    m = _model(cfg, sd, cuda, torch.float16)
    out = _check(cfg, sd, _image(tuple(g["shape"]), int(g["seed"][1])), torch.float16, cuda, m)
    zg = g["z"]
    assert np.abs(out[0].float().cpu().numpy() - zg).max() <= 2e-2 * np.abs(zg).max()
    # square and rect batches of other shapes through the same model, and bf16
    _check(cfg, sd, _image((2, 3, 128, 128), 5), torch.float16, cuda, m)
    _check(cfg, sd, _image((1, 3, 320, 192), 6), torch.float16, cuda, m)
    _check(cfg, sd, _image((2, 3, 96, 160), 7), torch.bfloat16, cuda, _model(cfg, sd, cuda, torch.bfloat16))


@pytest.mark.parametrize("width", [0.75, 1.0, 1.25], ids=["dh96", "dh128", "dh160"])
def test_transformer_model_wide_head_dims(cuda, width):
    from oracle import transformer_ref

    cfg = _cfg(width)
    sd = transformer_ref.synth_state_dict(cfg, seed=8)
    _check(cfg, sd, _image((1, 3, 128, 96), 9), torch.float16, cuda, _model(cfg, sd, cuda, torch.float16))


def test_transformer_augment(cuda):
    """augment=True runs the three TTA scales (P5 maps 3x4, 2x3 and 2x3 at 96x128 after padding): its full-scale rows are the
    plain forward's rows."""
    from oracle import transformer_ref

    cfg = _cfg(0.25)
    sd = transformer_ref.synth_state_dict(cfg, seed=12)
    m = _model(cfg, sd, cuda, torch.float16)
    x = _image((2, 3, 96, 128), 13).to(cuda, torch.float16)
    za, _ = m(x, augment=True)
    z = m(x)[0]
    n0 = z.shape[1] - z.shape[1] // 21
    assert torch.isfinite(za).all() and torch.equal(za[:, :n0], z[:, :n0])
    # each scaled copy is itself the engine's forward of that image
    from yolov5_b200.models.yolo import scale_img

    xs = scale_img(x.flip(3), 0.83, gs=32)
    _check(cfg, sd, xs.float().cpu(), torch.float16, cuda, m)


def test_transformer_reference_checkpoint_attempt_load(cuda):
    from yolov5_b200.models.experimental import attempt_load

    m = attempt_load(os.path.join(G, "ref_transformer_tiny.pt"), device=cuda)
    assert type(m.model[8]).__name__ == "C3TR" and type(m.model[8]).__module__ == "yolov5_b200.models.common"
    f = np.load(os.path.join(G, "ref_transformer_tiny_forward.npz"))
    x = _image((1, 3, 64, 96), 11)
    z = m.half()(x.to(cuda).half())[0].float().cpu().numpy()
    assert np.abs(z - f["z"]).max() <= 2e-2 * np.abs(f["z"]).max()


def _train_model(dev, sd, cfg):
    from yolov5_b200.cfg import HYP_SCRATCH_LOW
    from yolov5_b200.models.yolo import DetectionModel

    m = DetectionModel(cfg)
    m.load_state_dict(sd)
    m = m.to(dev).train()
    m.hyp = dict(HYP_SCRATCH_LOW)
    return m


def test_transformer_training_step_vs_oracle(cuda, monkeypatch):
    """test_train_gpu.py's criteria for one width-0.25 step: raw maps and per-tensor gradient errors judged against torch-AMP's
    own error on the fp32 oracle; every C3TR tensor is in the report."""
    from oracle import loss_ref, model_ref, transformer_ref
    from yolov5_b200.utils.loss import ComputeLoss

    from .test_train_gpu import _ref_train_step

    cfg = _cfg(0.25)
    sd = transformer_ref.synth_state_dict(cfg, seed=21)
    shape, dtype = (4, 3, 128, 128), torch.float16
    img = (torch.rand(*shape, generator=torch.Generator().manual_seed(22)) * 255).to(torch.uint8)
    targets = torch.from_numpy(loss_ref.synth_targets(shape[0], seed=23)).float()
    monkeypatch.setattr(model_ref, "forward", transformer_ref.forward)  # _ref_train_step's oracle, with the C3TR rows
    p32, _, g32 = _ref_train_step(cfg, sd, img, targets, cuda, None)
    pamp, _, gamp = _ref_train_step(cfg, sd, img, targets, cuda, dtype)
    m = _train_model(cuda, sd, cfg)
    with torch.autocast("cuda", dtype=dtype):
        p = m(img.to(cuda))
    for l, (a, r, lo) in enumerate(zip(p, p32, pamp)):
        sc = float(r.abs().max())
        e, el = float((a.detach().float() - r).abs().max()), float((lo.float() - r).abs().max())
        assert e <= 1e-3 * sc + 1.5 * el, ("raw", l, e / sc, el / sc)
    loss, _ = ComputeLoss(m)(p, targets.to(cuda))
    loss.backward()
    named = dict(m.named_parameters())
    ratios, mine_sq, amp_sq, ref_sq, worst, seen = [], 0.0, 0.0, 0.0, (0.0, None), set()
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
        seen.add(k)
        worst = max(worst, (r, k, e, el), key=lambda w: w[0])
    tr_keys = {k for k in named if k.startswith("model.8.m.")}
    assert len(tr_keys) == 11 and tr_keys <= seen, tr_keys - seen
    ratios.sort()
    summary = dict(n=len(ratios), median=ratios[len(ratios) // 2], worst=worst, total_mine=(mine_sq / ref_sq) ** 0.5,
                   total_amp=(amp_sq / ref_sq) ** 0.5)
    print("transformer train-step gradient report", summary)
    assert worst[0] <= 2.5 and summary["median"] <= 1.25, summary
    assert summary["total_mine"] <= 1e-3 + 1.5 * summary["total_amp"], summary


def test_transformer_graphed_train_step_matches_eager(cuda):
    """GraphedTrainStep captures the attention kernels: its steps give the eager fused loop's loss items and weights."""
    from oracle import loss_ref, transformer_ref
    from yolov5_b200.utils.loss import ComputeLoss
    from yolov5_b200.utils.torch_utils import GraphedTrainStep, smart_optimizer

    cfg = _cfg(0.25)
    sd = transformer_ref.synth_state_dict(cfg, seed=0)
    ma, mb = _train_model(cuda, sd, cfg), _train_model(cuda, sd, cfg)
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
