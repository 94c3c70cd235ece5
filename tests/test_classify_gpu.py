"""GPU: classification on the engine -- the global-average-pool and cross-entropy kernels against float64, ClassificationModel
eval and training against the fp32 oracle (oracle/cls_ref.py, pinned to the reference by tests/golden/cls.npz) judged by the
criteria of test_model_gpu.py / test_train_gpu.py, the reference-pickled checkpoint, and classify/train.py's loop body."""
import contextlib
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import cls_ref
from yolov5_b200 import _lib
from yolov5_b200.cfg import model_cfg

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
MANT = {torch.float16: 10, torch.bfloat16: 7, torch.float32: 23}


@contextlib.contextmanager
def _exact_fp32():
    """fp32 references on the GPU: no TF32 in cuDNN convolutions or cuBLAS matmuls."""
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _ulp(ref: torch.Tensor, dtype) -> torch.Tensor:
    """one unit in the last place of `dtype` at |ref| (float64), subnormal spacing included"""
    fi = torch.finfo(dtype)
    e = torch.floor(torch.log2(ref.abs().clamp_min(fi.tiny)))
    return torch.exp2(e - MANT[dtype]).clamp_min(fi.tiny * 2.0 ** -MANT[dtype])


def _st(dev):
    return C.c_void_p(_lib.stream_ptr(dev))


# ---------------------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("c", [8, 1280])
@pytest.mark.parametrize("hw", [(1, 1), (2, 2), (7, 7), (20, 20)])
def test_global_avg_pool_forward_backward_vs_float64(cuda, dtype, c, hw):
    lib = _lib.lib()
    h, w = hw
    b, off, xp, yp = 3, 8, c + 24, c + 16  # channel-slice views: offset 8 inside wider buffers
    g = torch.Generator().manual_seed(c + h)
    x = (torch.randn(b, h, w, c, generator=g) * 2 + 0.5).to(dtype)
    xbuf = torch.full((b, h, w, xp), 9.0, dtype=dtype, device=cuda)
    xbuf[..., off : off + c] = x.to(cuda)
    ybuf = torch.full((b, yp), -7.0, dtype=dtype, device=cuda)
    es = xbuf.element_size()
    _lib.check(lib.y5_global_avg_pool(xbuf.data_ptr() + off * es, xp, ybuf.data_ptr() + off * es, yp, b, h, w, c, _lib.dtype_code(dtype), _st(cuda)))
    ref = x.double().mean((1, 2))
    got = ybuf[:, off : off + c].double().cpu()
    assert ((got - ref).abs() <= _ulp(ref, dtype)).all(), float((got - ref).abs().max())
    assert bool((ybuf[:, :off] == -7.0).all() and (ybuf[:, off + c :] == -7.0).all())  # nothing outside the view is written
    # backward: dx = dy / (h w) at every pixel of a channel slice
    dy = (torch.randn(b, c, generator=g) * 3).to(dtype)
    dybuf = torch.zeros(b, yp, dtype=dtype, device=cuda)
    dybuf[:, off : off + c] = dy.to(cuda)
    dxbuf = torch.full((b, h, w, xp), 5.0, dtype=dtype, device=cuda)
    _lib.check(lib.y5_global_avg_pool_bwd(dybuf.data_ptr() + off * es, yp, dxbuf.data_ptr() + off * es, xp, b, h, w, c, _lib.dtype_code(dtype),
                                          _st(cuda)))
    ref = (dy.double() / (h * w)).view(b, 1, 1, c).expand(b, h, w, c)
    got = dxbuf[..., off : off + c].double().cpu()
    assert ((got - ref).abs() <= _ulp(ref, dtype)).all(), float((got - ref).abs().max())
    assert bool((dxbuf[..., :off] == 5.0).all() and (dxbuf[..., off + c :] == 5.0).all())
    # repeatable bit for bit
    y2 = torch.empty_like(ybuf)
    _lib.check(lib.y5_global_avg_pool(xbuf.data_ptr() + off * es, xp, y2.data_ptr() + off * es, yp, b, h, w, c, _lib.dtype_code(dtype), _st(cuda)))
    assert torch.equal(y2[:, off : off + c], ybuf[:, off : off + c])


def _ce(logits, labels, eps, scale=None):
    from yolov5_b200.utils.loss import _cross_entropy

    return _cross_entropy(logits, labels, eps, grad_scale=scale)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
@pytest.mark.parametrize("nc", [2, 10, 1000, 1001])
def test_cross_entropy_vs_float64(cuda, dtype, nc):
    for b in (1, 64, 257):
        for eps in (0.0, 0.1):
            g = torch.Generator().manual_seed(b * 7 + nc)
            z = (torch.randn(b, nc, generator=g) * 1.5).to(dtype)
            lab = torch.randint(0, nc, (b,), generator=g)
            z64 = z.double()
            lref = float(cls_ref.cross_entropy(z64, lab, eps))
            gref = cls_ref.cross_entropy_grad(z64, lab, eps)
            zd, ld = z.to(cuda), lab.to(cuda)
            loss, _ = _ce(zd, ld, eps)
            assert abs(float(loss) - lref) <= 2e-6 * abs(lref) + 1e-6, (b, eps, float(loss), lref)
            loss2, _ = _ce(zd, ld, eps)
            assert loss.view(1).view(torch.int32).item() == loss2.view(1).view(torch.int32).item()  # bitwise repeatable
            for scale in (1.0, 65536.0):
                s = torch.tensor([scale], dtype=torch.float32, device=cuda)
                loss3, d = _ce(zd, ld, eps, s)
                assert d.dtype == dtype and d.shape == (b, nc) and torch.equal(loss3, loss)
                ref = gref * scale
                d = d.double().cpu()
                # finite wherever the exact value is representable; IEEE round-to-nearest overflows beyond fp16's 65520 (B = 1,
                # scale 65536: g (p_y - 1) of a confident miss), as torch-autocast's fp32 -> fp16 cast does -- GradScaler's skip
                big = torch.finfo(dtype).max + _ulp(torch.tensor(torch.finfo(dtype).max, dtype=torch.float64), dtype) / 2
                over = ref.abs() > big * (1 + 1e-5)
                fine = ref.abs() < big * (1 - 1e-5)
                assert bool(torch.isfinite(d[fine]).all()) and bool((d[over] == ref[over].sign() * float("inf")).all()), (b, eps, scale)
                # the kernel's fp32 value, rounded once: within one ulp of the dtype (plus the fp32 softmax's own error)
                tol = _ulp(ref, dtype) + 4e-6 * scale / b
                err = (d[fine] - ref[fine]).abs()
                assert (err <= tol[fine]).all(), (b, eps, scale, float((err / tol[fine]).max()))


def test_cross_entropy_strided_logits_and_bad_labels(cuda):
    g = torch.Generator().manual_seed(5)
    wide = torch.randn(16, 1008, generator=g).half().to(cuda)
    z = wide[:, :1000]  # row stride 1008 (the engine's padded Linear output)
    lab = torch.randint(0, 1000, (16,), generator=g).to(cuda)
    loss, d = _ce(z, lab, 0.1, torch.ones(1, device=cuda))
    loss_c, d_c = _ce(z.contiguous(), lab, 0.1, torch.ones(1, device=cuda))
    assert torch.equal(loss, loss_c) and torch.equal(d, d_c)
    for bad in (1000, -1, -100):
        lb = lab.clone()
        lb[3] = bad
        loss, d = _ce(z, lb, 0.1, torch.ones(1, device=cuda))
        assert bool(torch.isnan(loss)) and bool(torch.isnan(d[3]).all())
        assert bool(torch.isfinite(d[torch.arange(16, device=cuda) != 3]).all())


def test_cross_entropy_module_autograd_and_dtypes(cuda):
    from yolov5_b200.utils.torch_utils import smartCrossEntropyLoss

    crit = smartCrossEntropyLoss(label_smoothing=0.1)
    g = torch.Generator().manual_seed(6)
    z = torch.randn(32, 10, generator=g).to(cuda)
    lab = torch.randint(0, 10, (32,), generator=g).to(cuda)
    for dt in (torch.float32, torch.float16, torch.bfloat16):
        zz = z.to(dt).clone().requires_grad_(True)
        loss = crit(zz, lab)
        zt = z.to(dt).clone().requires_grad_(True)
        lt = torch.nn.CrossEntropyLoss(label_smoothing=0.1)(zt, lab)
        assert loss.dtype == lt.dtype == dt
        (loss * 3).backward()
        (lt * 3).backward()
        tol = 1e-6 if dt == torch.float32 else (2e-3 if dt == torch.float16 else 1.6e-2)
        assert abs(float(loss.detach()) - float(lt.detach())) <= tol * float(lt.detach())
        assert torch.allclose(zz.grad.float(), zt.grad.float(), rtol=tol, atol=tol * float(zt.grad.float().abs().max()))
    with torch.autocast("cuda", dtype=torch.float16):  # classify/val.py: criterion(y, labels) on fp16 logits under autocast
        with torch.no_grad():
            lv = crit(z.half(), lab)
    assert lv.dtype == torch.float32 and abs(float(lv) - float(cls_ref.cross_entropy(z.half().double().cpu(), lab.cpu(), 0.1))) < 1e-5


# ---------------------------------------------------------------------------------------------------------------------------
# models
# ---------------------------------------------------------------------------------------------------------------------------
def _cls_model(name, nc, sd, dev, dtype=None):
    from yolov5_b200.models.yolo import ClassificationModel, DetectionModel

    m = ClassificationModel(model=DetectionModel(name), nc=nc)
    m.load_state_dict(sd)
    return m.to(dev, dtype) if dtype is not None else m.to(dev)


def _image(shape, seed):
    return torch.from_numpy(np.random.RandomState(seed).uniform(0, 1, shape).astype(np.float32))


@pytest.mark.parametrize("shape,dtype", [((64, 3, 224, 224), torch.float16), ((64, 3, 224, 224), torch.bfloat16), ((1, 3, 224, 224), torch.float16)])
def test_yolov5s_cls_eval_vs_oracle(cuda, shape, dtype):
    cfg = model_cfg("yolov5s")
    sd = cls_ref.synth_state_dict(cfg, 1000, seed=50)
    x = _image(shape, 51)
    sd_d = {k: v.to(cuda) for k, v in sd.items()}
    with torch.no_grad(), _exact_fp32():
        ref = cls_ref.forward(cfg, sd_d, x.to(dtype).float().to(cuda)).double().cpu()
        low = cls_ref.forward(cfg, {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in sd_d.items()}, x.to(cuda, dtype), fused=True)
    m = _cls_model("yolov5s", 1000, sd, cuda, dtype).eval()
    y = m(x.to(cuda, dtype))
    assert y.shape == (shape[0], 1000) and y.dtype == dtype
    scale = float(ref.abs().max())
    e_eng, e_low = float((y.double().cpu() - ref).abs().max()), float((low.double().cpu() - ref).abs().max())
    print("yolov5s-cls eval", shape, dtype, dict(engine=e_eng / scale, torch_lowp=e_low / scale))
    assert e_eng <= 1e-3 * scale + 1.5 * e_low, (e_eng / scale, e_low / scale)


def test_fresh_outputs_graph_replay_and_val_py_call(cuda):
    cfg = model_cfg("yolov5n")
    sd = cls_ref.synth_state_dict(cfg, 10, seed=52)
    m = _cls_model("yolov5n", 10, sd, cuda).half().eval()
    x = _image((8, 3, 224, 224), 53).to(cuda)
    xn = (x - torch.tensor([0.485, 0.456, 0.406], device=cuda).view(1, 3, 1, 1)) / torch.tensor([0.229, 0.224, 0.225], device=cuda).view(1, 3, 1, 1)
    y1 = m(xn.half())
    y2 = m(xn.half())
    assert y1.data_ptr() != y2.data_ptr() and torch.equal(y1, y2)
    with torch.autocast("cuda"):  # classify/val.py:110-116: fp32 normalised images into model.half() under autocast
        y3 = m(xn)
    assert y3.dtype == torch.float16 and torch.equal(y3, y1)
    prog = m._program(xn.half())
    assert prog.graph is not None and prog.cls_view.c == 10
    # classify/train.py validates the fp32 EMA model under autocast: it computes in the autocast dtype
    mf = _cls_model("yolov5n", 10, sd, cuda).eval()
    with torch.autocast("cuda"):
        y4 = mf(xn)
    assert y4.dtype == torch.float16 and float((y4.float() - y1.float()).abs().max()) <= 2e-2 * float(y1.float().abs().max())
    with pytest.raises(TypeError):
        mf(xn)  # fp32 without autocast: the engine computes in fp16 / bf16 only


def test_reference_pickled_checkpoint_forward_matches_golden(cuda):
    from tests.golden import make_cls_golden as mk
    from yolov5_b200.models.experimental import attempt_load

    g = np.load(os.path.join(G, "cls.npz"))
    m = attempt_load(os.path.join(G, "ref_cls_tiny.pt"), device=cuda).half()
    y = m(mk.image(mk.CKPT["shape"], mk.CKPT["x_seed"]).to(cuda).half()).float().cpu().numpy()
    ref = g["ckpt.logits"]
    assert np.abs(y - ref).max() <= 2e-2 * np.abs(ref).max(), np.abs(y - ref).max() / np.abs(ref).max()
    assert (y.argmax(1) == ref.argmax(1)).all()


def _oracle_step(cfg, sd, x, lab, eps, dev, amp_dtype):
    params = {k: v.to(dev).clone().requires_grad_(v.is_floating_point() and "running" not in k) for k, v in sd.items()}
    ctx = torch.autocast("cuda", dtype=amp_dtype) if amp_dtype is not None else contextlib.nullcontext()
    with _exact_fp32(), ctx:
        y = cls_ref.forward(cfg, params, x.to(dev), bn_batch_stats=True)
        loss = cls_ref.cross_entropy(y.float(), lab.to(dev), eps)
    with _exact_fp32():
        loss.backward()
    return y.detach(), loss.detach(), {k: v.grad for k, v in params.items() if v.grad is not None}


@pytest.mark.parametrize("name,dtype", [("yolov5n", torch.float16), ("yolov5n", torch.bfloat16), ("yolov5s", torch.float16), ("yolov5s", torch.bfloat16)])
def test_training_vs_oracle_amp_yardstick(cuda, name, dtype):
    from yolov5_b200.utils.torch_utils import smartCrossEntropyLoss

    cfg = model_cfg(name)
    sd = cls_ref.synth_state_dict(cfg, 1000, seed=60)
    x = _image((16, 3, 224, 224), 61)
    lab = torch.from_numpy(np.random.RandomState(62).randint(0, 1000, 16))
    y32, l32, g32 = _oracle_step(cfg, sd, x, lab, 0.1, cuda, None)
    yamp, lamp, gamp = _oracle_step(cfg, sd, x, lab, 0.1, cuda, dtype)
    m = _cls_model(name, 1000, sd, cuda).train()
    with torch.autocast("cuda", dtype=dtype):
        y = m(x.to(cuda))
        loss = smartCrossEntropyLoss(label_smoothing=0.1)(y, lab.to(cuda))
    loss.backward()
    assert y.shape == (16, 1000) and loss.dtype == torch.float32
    sc = float(y32.abs().max())
    e, el = float((y.detach().float() - y32).abs().max()), float((yamp.float() - y32).abs().max())
    assert e <= 1e-3 * sc + 1.5 * el, ("logits", e / sc, el / sc)
    le, lel = abs(float(loss.detach()) - float(l32)), abs(float(lamp) - float(l32))
    assert le <= 1e-3 * abs(float(l32)) + 1.5 * lel, ("loss", float(loss), float(l32), float(lamp))
    named = dict(m.named_parameters())
    ratios, mine_sq, amp_sq, ref_sq, worst = [], 0.0, 0.0, 0.0, (0.0, None)
    for k, gr in g32.items():
        got = named[k].grad
        assert got is not None and got.shape == named[k].shape and got.is_contiguous(), k
        n = float(gr.norm())
        if n == 0:
            continue
        e, el = float((got.float() - gr).norm()) / n, float((gamp[k].float() - gr).norm()) / n
        mine_sq, amp_sq, ref_sq = mine_sq + (e * n) ** 2, amp_sq + (el * n) ** 2, ref_sq + n * n
        r = e / (1e-3 + el)
        ratios.append(r)
        if r > worst[0]:
            worst = (r, k, e, el)
    assert len(named) == len(g32)
    ratios.sort()
    summary = dict(n=len(ratios), median=ratios[len(ratios) // 2], worst=worst, total_mine=(mine_sq / ref_sq) ** 0.5, total_amp=(amp_sq / ref_sq) ** 0.5)
    print("classification train-step gradient report", name, dtype, summary)
    assert worst[0] <= 2.5 and summary["median"] <= 1.25, summary
    assert summary["total_mine"] <= 1e-3 + 1.5 * summary["total_amp"], summary


def test_classify_train_py_loop_body_learns_a_fixed_batch(cuda):
    """classify/train.py:221-236 on one fixed batch: autocast forward, CE(0.1), scaled backward, unscale_, clip_grad_norm_,
    scaler.step / update, zero_grad, ModelEMA.update -- with smart_optimizer(model, 'Adam', 1e-3, 0.9, 5e-5)."""
    from yolov5_b200.models.yolo import ClassificationModel, DetectionModel
    from yolov5_b200.utils.torch_utils import ModelEMA, smart_optimizer, smartCrossEntropyLoss

    torch.manual_seed(70)
    model = ClassificationModel(model=DetectionModel("yolov5n"), nc=10).to(cuda).train()
    opt = smart_optimizer(model, "Adam", 1e-3, 0.9, 5e-5)
    ema = ModelEMA(model)
    scaler = torch.amp.GradScaler("cuda")
    criterion = smartCrossEntropyLoss(label_smoothing=0.1)
    images = _image((16, 3, 224, 224), 71).to(cuda)
    labels = torch.from_numpy(np.random.RandomState(72).randint(0, 10, 16)).to(cuda)
    losses = []
    for _ in range(30):
        with torch.autocast("cuda"):
            loss = criterion(model(images), labels)
        scaler.scale(loss).backward()
        scaler.unscale_(opt)
        torch.nn.utils.clip_grad_norm_(model.parameters(), max_norm=10.0)
        scaler.step(opt)
        scaler.update()
        opt.zero_grad()
        ema.update(model)
        losses.append(float(loss))
    print("classify/train.py loop losses", [round(v, 4) for v in losses])
    assert all(np.isfinite(losses)), losses
    assert losses[-1] < 0.5 * losses[0], losses
    ema.ema.half()
    with torch.no_grad():
        assert bool(torch.isfinite(ema.ema(images.half())).all())
