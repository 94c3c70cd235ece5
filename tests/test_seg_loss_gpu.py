"""GPU: the segmentation ComputeLoss (y5_seg_loss_fwd_bwd_scaled) vs the reference fixture and the oracle.

build_targets bit-exact (six lists, in order); loss / items / gradients of every head level and of proto within fp32
tolerance for fp32 inputs and within the rounding of fp16 / bf16 inputs; NCHW, channels_last and non-dense proto views; run-to-run
determinism; CUDA-graph capture; the validation call form; a yolov5n-seg training step against torch-AMP's own error;
a few optimizer steps lowering the loss."""
import os

import numpy as np
import pytest
import torch

from oracle import loss_ref, model_ref
from tests import seg_loss_ref
from tests.golden import make_seg_golden as mg
from yolov5_b200.cfg import HYP_SCRATCH_LOW, model_cfg
from yolov5_b200.utils.segment.loss import ComputeLoss

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
CASES = list(mg.CASES)


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(G, "seg_loss.npz"))


def _case(tag, dev, dtype=torch.float32, channels_last=False):
    p_np, proto_np, tg, masks, overlap, nc = mg.case_inputs(tag)
    crit = ComputeLoss(mg.LossModel(nc).to(dev), overlap=overlap)
    p = [torch.from_numpy(a).to(dev, dtype).requires_grad_(True) for a in p_np]
    proto = torch.from_numpy(proto_np).to(dev, dtype)
    if channels_last:
        proto = proto.contiguous(memory_format=torch.channels_last)
    proto.requires_grad_(True)
    return crit, p, proto, torch.from_numpy(tg).to(dev), torch.from_numpy(masks).to(dev), (p_np, proto_np, tg, masks, overlap)


def _oracle(p_np, proto_np, tg, masks, overlap, scale=1.0, dtype=torch.float32):
    """oracle loss / items / gradients on the inputs rounded to `dtype`."""
    p = [torch.from_numpy(a).to(dtype).float().requires_grad_(True) for a in p_np]
    proto = torch.from_numpy(proto_np).to(dtype).float().requires_grad_(True)
    lo, it = seg_loss_ref.compute_seg_loss(p, proto, tg, masks, mg.anchors_grid(), HYP_SCRATCH_LOW, overlap)
    (lo * scale).backward()
    gp = proto.grad if proto.grad is not None else torch.zeros_like(proto)
    return lo.detach(), it, [a.grad for a in p] + [gp]


@pytest.mark.parametrize("tag", CASES)
def test_build_targets_bit_exact(cuda, golden, tag):
    crit, p, _, tg, _, _ = _case(tag, cuda)
    bt = crit.build_targets(p, tg)
    assert len(bt) == 6
    tcls, tbox, indices, anch, tidxs, xywhn = bt
    for i in range(3):
        got = torch.stack(list(indices[i]) + [tcls[i], tidxs[i]]).cpu().numpy()
        assert got.dtype == np.int64 and np.array_equal(got, golden[f"{tag}.idx{i}"]), (tag, i)
        assert tbox[i].dtype == torch.float32 and xywhn[i].dtype == torch.float32
        assert np.array_equal(tbox[i].cpu().numpy(), golden[f"{tag}.tbox{i}"]), (tag, i)
        assert np.array_equal(xywhn[i].cpu().numpy(), golden[f"{tag}.xywhn{i}"]), (tag, i)
        assert np.array_equal(anch[i].cpu().numpy(), golden[f"{tag}.anch{i}"]), (tag, i)


@pytest.mark.parametrize("tag", CASES)
def test_loss_and_gradients_fp32(cuda, golden, tag):
    crit, p, proto, tg, masks, raw = _case(tag, cuda)
    loss, items = crit((p, proto), tg, masks)
    loss.backward()
    got = np.concatenate((loss.detach().cpu().numpy(), items.cpu().numpy()))
    np.testing.assert_allclose(got, golden[f"{tag}.loss"], rtol=1e-4, atol=1e-6)
    refs = [golden[f"{tag}.grad{i}"] for i in range(3)] + [golden[f"{tag}.grad_proto"]]
    for k, (a, r) in enumerate(zip(p + [proto], refs)):
        err = float(np.abs(a.grad.cpu().numpy() - r).max())
        assert err <= 1e-4 * float(np.abs(r).max()) + 1e-9, (tag, k, err)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("scale", [8.0, 65536.0 * 8])
@pytest.mark.parametrize("tag", ["ov_unsorted", "nonov_frac"])
def test_low_precision_and_upstream_scale(cuda, tag, dtype, scale):
    crit, p, proto, tg, masks, raw = _case(tag, cuda, dtype)
    loss, items = crit((p, proto), tg, masks)
    (loss * scale).backward()
    lo, it, refs = _oracle(*raw, scale=scale, dtype=dtype)
    assert abs(loss.item() - lo.item()) <= 2e-3 * abs(lo.item())
    np.testing.assert_allclose(items.cpu().numpy(), it.numpy(), rtol=2e-3, atol=1e-5)
    # 3e-3 x max, plus the half-ulp of the gradient's own dtype at max: the final rounding to bf16 alone can reach 3.9e-3
    half_ulp = torch.finfo(dtype).eps / 2
    for k, (a, r) in enumerate(zip(p + [proto], refs)):
        g = a.grad.float().cpu()
        assert a.grad.dtype == dtype and bool(torch.isfinite(g).all()), k
        err, top = float((g / scale - r / scale).abs().max()), float((r / scale).abs().max())
        assert err <= (3e-3 + half_ulp) * top, (k, dtype, scale, err / top)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_proto_memory_format_and_determinism(cuda, dtype):
    outs = []
    for cl in (False, True, True):
        crit, p, proto, tg, masks, _ = _case("ov_x4", cuda, dtype, channels_last=cl)
        loss, items = crit((p, proto), tg, masks)
        (loss * 1024.0).backward()
        assert proto.grad.is_contiguous(memory_format=torch.channels_last) == cl
        assert proto.grad.stride() == proto.stride()
        outs.append([loss.detach(), items] + [a.grad.contiguous() for a in p] + [proto.grad.contiguous()])
    for o in outs[1:]:
        assert torch.equal(o[0], outs[0][0]) and torch.equal(o[1], outs[0][1])
        assert torch.equal(o[-1], outs[0][-1])  # dproto: no atomics
        # head maps: only the arrival order of the atomic adds on cells matched more than once may differ
        tol = 1e-6 if dtype == torch.float32 else 2 * torch.finfo(dtype).eps
        for a, b in zip(o[2:-1], outs[0][2:-1]):
            assert float((a.float() - b.float()).abs().max()) <= tol * float(b.float().abs().max())


@pytest.mark.parametrize("view", ["channel_slice", "crop", "batch_step", "channels_last_slice"])
def test_proto_views_that_are_not_dense(cuda, golden, view):
    """proto as a view of a larger tensor (a channel slice of a wider map, a spatial crop, every other image, a channel slice
    of a channels_last map): the loss and dproto still match the fixture, and the gradient of the larger tensor is zero
    outside the view."""
    tag = "ov_unsorted"
    crit, p, proto, tg, masks, _ = _case(tag, cuda)
    B, nm, mh, mw = proto.shape
    base = torch.full((2 * B, nm + 16, mh + 5, mw + 3), 7.0, device=cuda)
    if view == "channels_last_slice":
        base = base.contiguous(memory_format=torch.channels_last)
    idx = {"channel_slice": (slice(0, B), slice(8, 8 + nm), slice(0, mh), slice(0, mw)),
           "crop": (slice(0, B), slice(0, nm), slice(3, 3 + mh), slice(2, 2 + mw)),
           "batch_step": (slice(0, 2 * B, 2), slice(0, nm), slice(0, mh), slice(0, mw)),
           "channels_last_slice": (slice(B, 2 * B), slice(4, 4 + nm), slice(1, 1 + mh), slice(0, mw))}[view]
    with torch.no_grad():
        base[idx] = proto
    base.requires_grad_(True)
    pv = base[idx]
    assert not (pv.is_contiguous() or pv.is_contiguous(memory_format=torch.channels_last))
    loss, items = crit((p, pv), tg, masks)
    loss.backward()
    got = np.concatenate((loss.detach().cpu().numpy(), items.cpu().numpy()))
    np.testing.assert_allclose(got, golden[f"{tag}.loss"], rtol=1e-4, atol=1e-6)
    r = golden[f"{tag}.grad_proto"]
    g = base.grad[idx].cpu().numpy()
    assert float(np.abs(g - r).max()) <= 1e-4 * float(np.abs(r).max()), view
    outside = base.grad.clone()
    outside[idx] = 0
    assert float(outside.abs().max()) == 0.0
    for i, a in enumerate(p):
        r = golden[f"{tag}.grad{i}"]
        assert float(np.abs(a.grad.cpu().numpy() - r).max()) <= 1e-4 * float(np.abs(r).max()) + 1e-9


def test_cuda_graph_capture_replays_eager(cuda):
    crit, p, proto, tg, masks, _ = _case("ov_unsorted", cuda)
    loss, items = crit((p, proto), tg, masks)
    loss.backward()
    ref = [loss.detach().clone(), items.clone()] + [a.grad.clone() for a in p] + [proto.grad.clone()]
    sp = [a.detach().clone().requires_grad_(True) for a in p]
    sproto = proto.detach().clone().requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):  # warm-up on the capture stream: the scratch is allocated per stream
        for _ in range(2):
            for a in sp + [sproto]:
                a.grad = None
            lw, _ = crit((sp, sproto), tg, masks)
            lw.backward()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    for a in sp + [sproto]:
        a.grad = None
    with torch.cuda.graph(graph, stream=s):
        gl, gi = crit((sp, sproto), tg, masks)
        gl.backward()
    with torch.no_grad():
        for a, b in zip(sp + [sproto], p + [proto]):
            a.copy_(b)
    graph.replay()
    torch.cuda.synchronize()
    got = [gl.detach(), gi] + [a.grad for a in sp] + [sproto.grad]
    for a, b in zip(got, ref):
        assert torch.equal(a, b) or torch.allclose(a, b, rtol=0, atol=float(b.abs().max()) * 1e-6)


def _seg_batch(bs, h, w, seed):
    tg = loss_ref.synth_targets(bs, seed)
    return torch.from_numpy(tg), torch.from_numpy(seg_loss_ref.overlap_masks(tg, bs, h, w))


def _seg_model(dev, seed=41):
    from yolov5_b200.models.yolo import SegmentationModel

    cfg = model_cfg("yolov5n-seg")
    sd = model_ref.synth_state_dict(cfg, seed=seed)
    m = SegmentationModel("yolov5n-seg")
    m.load_state_dict(sd)
    m.hyp = dict(HYP_SCRATCH_LOW)
    return cfg, sd, m.to(dev)


def test_validation_call_form(cuda):
    cfg, sd, m = _seg_model(cuda)
    g = torch.Generator().manual_seed(43)
    img = (torch.rand(2, 3, 128, 128, generator=g) * 255).to(torch.uint8).to(cuda)
    tg, masks = _seg_batch(2, 128, 128, 44)
    crit = ComputeLoss(m, overlap=True)
    m.half().eval()  # eval forward runs in the engine's fp16 path; (z, proto, raws) like Segment in eval (models/yolo.py:147-150)
    with torch.no_grad():
        z, proto, raws = m(img)
        items = crit((raws, proto), tg.to(cuda), masks.to(cuda))[1]
    assert items.shape == (4,) and bool(torch.isfinite(items).all())
    lo, it = seg_loss_ref.compute_seg_loss([r.float().cpu() for r in raws], proto.float().cpu(), tg, masks,
                                           sd["model.24.anchors"], HYP_SCRATCH_LOW, True)
    np.testing.assert_allclose(items.cpu().numpy(), it.numpy(), rtol=2e-3, atol=1e-5)


def _ref_step(cfg, sd, img, tg, masks, dev, amp):
    params = {k: v.to(dev).clone().requires_grad_(v.is_floating_point() and "running" not in k and "anchors" not in k)
              for k, v in sd.items()}
    x = img.to(dev).float() / 255
    ctx = torch.autocast("cuda", dtype=torch.float16) if amp else torch.autocast("cuda", enabled=False)
    with ctx:
        outs, proto = model_ref.forward(cfg, params, x, training=True, bn_batch_stats=True)
    loss, _ = seg_loss_ref.compute_seg_loss([q.float().cpu() for q in outs], proto.float().cpu(), tg, masks,
                                            sd["model.24.anchors"], HYP_SCRATCH_LOW, True)
    loss.backward()
    return {k: v.grad for k, v in params.items() if v.requires_grad and v.grad is not None}


def test_training_step_vs_oracle_amp_yardstick(cuda):
    cfg, sd, m = _seg_model(cuda, seed=45)
    m.train()
    g = torch.Generator().manual_seed(46)
    img = (torch.rand(4, 3, 128, 128, generator=g) * 255).to(torch.uint8)
    tg, masks = _seg_batch(4, 128, 128, 47)
    g32 = _ref_step(cfg, sd, img, tg, masks, cuda, False)
    gamp = _ref_step(cfg, sd, img, tg, masks, cuda, True)
    crit = ComputeLoss(m, overlap=True)
    with torch.autocast("cuda", dtype=torch.float16):
        outs, proto = m(img.to(cuda))
    loss, items = crit((outs, proto), tg.to(cuda), masks.to(cuda))
    loss.backward()
    named = dict(m.named_parameters())
    ratios, worst = [], (0.0, None)
    for k, gr in g32.items():
        got = named[k].grad
        assert got is not None and bool(torch.isfinite(got).all()), k
        n = float(gr.norm())
        if n == 0:
            continue
        e, el = float((got.float() - gr).norm()) / n, float((gamp[k].float() - gr).norm()) / n
        r = e / (1e-3 + el)
        ratios.append(r)
        worst = max(worst, (r, k), key=lambda t: t[0])
    ratios.sort()
    print("seg train-step gradient ratios: median", ratios[len(ratios) // 2], "worst", worst)
    assert len(ratios) > 150
    assert worst[0] <= 2.5 and ratios[len(ratios) // 2] <= 1.25, (ratios[len(ratios) // 2], worst)


def test_sgd_steps_lower_the_loss(cuda):
    from yolov5_b200.utils.torch_utils import FusedSGD

    _, _, m = _seg_model(cuda, seed=48)
    m.train()
    g = torch.Generator().manual_seed(49)
    img = (torch.rand(2, 3, 128, 128, generator=g) * 255).to(torch.uint8).to(cuda)
    tg, masks = _seg_batch(2, 128, 128, 50)
    tg, masks = tg.to(cuda), masks.to(cuda)
    crit = ComputeLoss(m, overlap=True)
    opt = FusedSGD([q for q in m.parameters() if q.requires_grad], lr=0.01, momentum=0.9)
    hist = []
    for _ in range(6):
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.float16):
            pred = m(img)
        loss, items = crit(pred, tg, masks)
        loss.backward()
        opt.fused_step()
        hist.append((float(loss), float(items[1])))
    print("seg loss / lseg over steps", hist)
    assert hist[-1][0] < hist[0][0] and hist[-1][1] < hist[0][1], hist
