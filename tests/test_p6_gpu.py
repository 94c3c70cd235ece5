"""GPU: the P6 models (reference models/hub/yolov5{n,s,m,l,x}6.yaml): four Detect levels, a stride-64 level, 1280 inputs.

Reduced model.  The reference-pickled yolov5s6 at width 1/16 through attempt_load against the reference's stored fp32 forward
(fp32, fp16 and bf16 inputs), level by level; augment=True against the reference's TTA output and its _clip_augmented slicing;
one AMP training step against the reference's fp32 step, judged against torch's own autocast run of the same expressions;
GraphedTrainStep against the eager step; a DeviceValLoader rect batch built at stride 64 through forward, NMS and
val_batch_metrics.

Full size.  ComputeLoss with four levels per level and per term against the float64 loss of tests/loss64_ref.py; NMS on a 1280
yolov5n6 output (102 000 rows per image, past the 30 000 max_nms cut) against the oracle; yolov5n6 ... x6 planned, run and
graph-captured at 640 and 1280 against the fp32 oracle."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import loss_ref, model_ref
from tests import loss64_ref as R
from yolov5_b200.cfg import HYP_SCRATCH_LOW, model_cfg

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
CKPT = os.path.join(G, "ref_p6_tiny.pt")
F16, BF16, F32 = torch.float16, torch.bfloat16, torch.float32
STRIDES = (8, 16, 32, 64)
BALANCE4 = (4.0, 1.0, 0.25, 0.06)  # reference utils/loss.py: ComputeLoss.balance for nl = 4


def _fixture():
    return np.load(os.path.join(G, "p6_golden.npz"))


def _image(shape, seed):
    return torch.from_numpy(np.random.RandomState(seed).uniform(0, 1, shape).astype(np.float32))


def _uint8(shape, seed):
    return torch.from_numpy(np.random.RandomState(seed).randint(0, 256, shape).astype(np.uint8))


def _targets(bs, seed, nc=3):
    """COCO128-shaped labels plus one box of 55-95 % of the image per image, so the P6 anchors match at small sizes too."""
    tg = loss_ref.synth_targets(bs, seed=seed, nc=nc)
    rs = np.random.RandomState(seed + 1)
    big = np.stack([np.arange(bs), rs.randint(0, nc, bs), rs.uniform(0.45, 0.55, bs), rs.uniform(0.45, 0.55, bs),
                    rs.uniform(0.55, 0.9, bs), rs.uniform(0.6, 0.95, bs)], 1)
    return np.concatenate((tg, big), 0).astype(np.float32)


def _small_model(dev):
    """The reference checkpoint's weights in a freshly built fp32 model, in training mode with hyp.scratch-low."""
    from yolov5_b200 import compat
    from yolov5_b200.models.yolo import DetectionModel

    compat.install()
    ck = torch.load(CKPT, map_location="cpu", weights_only=False)
    m = DetectionModel(json.loads(str(_fixture()["small_cfg"])))
    m.load_state_dict({k: v.float() if v.is_floating_point() else v for k, v in ck["model"].state_dict().items()})
    m = m.to(dev).train()
    m.hyp = dict(HYP_SCRATCH_LOW)
    return m


def _loaded(dev, dtype):
    from yolov5_b200.models.experimental import attempt_load

    return attempt_load(CKPT, device=dev).to(dtype)


@pytest.mark.parametrize("mdt,xdt,tol", [(F16, F32, 2e-2), (F16, F16, 2e-2), (BF16, BF16, 6e-2)], ids=["fp16-fp32in", "fp16", "bf16"])
def test_forward_vs_reference_golden(cuda, mdt, xdt, tol):
    """z level by level: rows [r_l, r_l + 3 ny_l nx_l) of z are level l's decoded boxes, in the reference's order."""
    f = _fixture()
    _, _, h, w = (int(v) for v in f["x_shape"])
    m = _loaded(cuda, mdt)
    assert m.model[-1].nl == 4 and m.stride.tolist() == [8.0, 16.0, 32.0, 64.0]
    with torch.no_grad():
        z, raws = m(_image(tuple(f["x_shape"]), int(f["x_seed"])).to(cuda, xdt))
    zg = f["z"]
    assert z.dtype == mdt and z.shape == zg.shape == (1, 3 * sum((h // s) * (w // s) for s in STRIDES), 8)
    z = z.float().cpu().numpy()
    assert np.abs(z - zg).max() <= tol * np.abs(zg).max()
    r0 = 0
    for i, (r, s) in enumerate(zip(raws, STRIDES)):
        rg = f[f"raw{i}"]
        assert tuple(r.shape) == rg.shape == (1, 3, h // s, w // s, 8)
        assert np.abs(r.float().cpu().numpy() - rg).max() <= tol * np.abs(rg).max(), (mdt, i)
        n = 3 * (h // s) * (w // s)
        zl, zgl = z[:, r0 : r0 + n], zg[:, r0 : r0 + n]
        assert np.abs(zl - zgl).max() <= tol * np.abs(zgl).max(), (mdt, "z level", i)
        r0 += n


def test_augment_four_levels_vs_reference(cuda):
    """augment=True against the reference's TTA output, and its tails cut as the reference's _clip_augmented cuts them: the
    full-scale copy loses exactly its stride-64 rows, the 0.67 copy exactly its stride-8 rows."""
    from yolov5_b200.models.yolo import scale_img

    f = _fixture()
    x = _image(tuple(f["x_shape"]), int(f["x_seed"])).to(cuda, F16)
    m = _loaded(cuda, F16)
    with torch.no_grad():
        za, extra = m(x, augment=True)
        zg = f["z_aug"]
        assert extra is None and za.shape == zg.shape
        assert np.abs(za.float().cpu().numpy() - zg).max() <= 2e-2 * np.abs(zg).max()
        ys, level_rows = [], []
        for s, flip in zip((1, 0.83, 0.67), (None, 3, None)):
            xi = scale_img(x.flip(flip) if flip else x, s, gs=64)
            level_rows.append([3 * (xi.shape[2] // st) * (xi.shape[3] // st) for st in STRIDES])
            yi = m(xi)[0]
            yi[..., :4] /= s
            if flip == 3:
                yi[..., 0] = x.shape[3] - yi[..., 0]
            ys.append(yi)
    nl = 4
    g = sum(4**k for k in range(nl))  # reference models/yolo.py _clip_augmented, e = 1
    i0, i1 = ys[0].shape[1] // g, (ys[-1].shape[1] // g) * 4 ** (nl - 1)
    assert i0 == level_rows[0][3] and i1 == level_rows[2][0]
    assert torch.equal(za, torch.cat([ys[0][:, :-i0], ys[1], ys[-1][:, i1:]], 1))


def test_amp_training_step_vs_reference_amp_yardstick(cuda):
    """One fp16-autocast step against the reference's fp32 step (the fixture), with torch's own autocast execution of the same
    expressions (oracle model + oracle loss, four-level balance) as the yardstick: loss and the whole model's gradient within
    1e-3 + 1.5 x torch-AMP's distance, each gradient tensor within 1e-3 + 2.5 x, median ratio <= 1.25 (test_train_gpu.py).
    The whole-model gradient is judged by its relative L2 error, not by the difference of the two norms: this reduced network
    is ill-conditioned in fp16 (torch-AMP's own per-tensor errors are 2-35 %), and a difference of norms of vectors that far
    apart is a cancellation, measured at 0.6 % for torch-AMP and 1.7 % for the engine on the same step."""
    from yolov5_b200.utils.loss import ComputeLoss

    f = _fixture()
    img = _uint8(tuple(int(v) for v in f["train_shape"]), int(f["train_seed"])).to(cuda)
    targets = torch.from_numpy(f["targets"])
    m = _small_model(cuda)
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    with torch.autocast("cuda", dtype=F16):
        p = m(img)
    assert [tuple(q.shape[2:4]) for q in p] == [(32, 32), (16, 16), (8, 8), (4, 4)]
    loss, items = ComputeLoss(m)(p, targets.to(cuda))
    loss.backward()
    params = {k: v.to(cuda).clone().requires_grad_(v.is_floating_point() and "running" not in k and "anchors" not in k) for k, v in sd.items()}
    with torch.autocast("cuda", dtype=F16):
        pa = model_ref.forward(json.loads(str(f["small_cfg"])), params, img.float() / 255, training=True, bn_batch_stats=True)
    loss_a, items_a = loss_ref.compute_loss([q.float().cpu() for q in pa], targets, sd["model.33.anchors"], HYP_SCRATCH_LOW, balance=BALANCE4)
    loss_a.backward()
    lref = float(f["loss"][0])
    rep = {"loss": (abs(float(loss) - lref) / lref, abs(float(loss_a) - lref) / lref)}
    ratios, tot, mine, amp = [], 0.0, 0.0, 0.0
    for k, q in m.named_parameters():
        ref = torch.from_numpy(f[f"grad:{k}"]).double()
        g, ga = q.grad.double().cpu(), params[k].grad.double().cpu()
        n = float(ref.norm())
        tot, mine, amp = tot + n * n, mine + float((g - ref).norm()) ** 2, amp + float((ga - ref).norm()) ** 2
        if n > 0:
            e, el = float((g - ref).norm()) / n, float((ga - ref).norm()) / n
            rep[k] = (e, el)
            ratios.append(e / (1e-3 + el))
    rep["total_grad"] = ((mine / tot) ** 0.5, (amp / tot) ** 0.5)
    ratios.sort()
    print("P6 step vs reference (engine, torch-AMP):", {k: (f"{a:.2e}", f"{b:.2e}") for k, (a, b) in rep.items()},
          "items", items.tolist(), items_a.tolist(), f["items"].tolist(), "ratio median / max", ratios[len(ratios) // 2], ratios[-1])
    assert np.abs(f["grad:model.33.m.3.weight"]).max() > 0  # the fixture's P6 level carries matches
    for k, (e, el) in rep.items():
        assert e <= 1e-3 + (1.5 if k in ("loss", "total_grad") else 2.5) * el, (k, e, el)
    assert ratios[len(ratios) // 2] <= 1.25, ratios


# ---------------------------------------------------------------------------------------------------------------------
# ComputeLoss with nl = 4 against the float64 reference, per level and per term (criterion of test_loss_parity_gpu.py)
# ---------------------------------------------------------------------------------------------------------------------
U = {F32: 2.0**-24, F16: 2.0**-11, BF16: 2.0**-8}
Z = {F32: 0.0, F16: 2.0**-25, BF16: 0.0}


def _ulp(t, dtype):
    return 2 * U[dtype] * torch.exp2(torch.floor(torch.log2(t.clamp_min(torch.finfo(dtype).tiny))))


def _ratio(err, bound):
    r = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, torch.inf, 0.0))
    return float(r.max()) if r.numel() else 0.0


@pytest.mark.parametrize("dtype,scale", [(F16, 65536.0 * 8), (F32, 1.0)], ids=["fp16", "fp32"])
def test_four_level_loss_vs_float64(cuda, dtype, scale):
    """8 images of 1280 (P3 160x160 ... P6 20x20), nc 80, yolov5n6's anchors: build_targets bit-exact, loss and items within
    2e-5, every gradient element within the per-element rounding bound of tests/test_loss_parity_gpu.py."""
    from yolov5_b200.models.yolo import DetectionModel
    from yolov5_b200.utils.loss import ComputeLoss

    hm = DetectionModel("yolov5n6")
    hm.hyp = dict(HYP_SCRATCH_LOW)
    crit = ComputeLoss(hm)
    bs, size, no = 8, 1280, 85
    gen = torch.Generator(device=cuda).manual_seed(201)
    p = [(torch.randn(bs, 3, size // s, size // s, no, generator=gen, device=cuda) * 1.5).to(dtype) for s in STRIDES]
    tg = loss_ref.synth_targets(bs, seed=202)
    shapes = [tuple(t.shape[2:4]) for t in p]
    bt = R.targets_for(tg, hm.model[-1].anchors.numpy(), shapes, bs, HYP_SCRATCH_LOW["anchor_t"])
    assert all(len(d["b"]) > 0 for d in bt), [len(d["b"]) for d in bt]
    tgd = torch.from_numpy(tg).to(cuda)
    tcls, tbox, idx, _ = crit.build_targets(p, tgd)
    for i, d in enumerate(bt):
        got = np.stack([idx[i][q].cpu().numpy() for q in range(4)] + [tcls[i].cpu().numpy()])
        assert np.array_equal(got, np.stack([d[k] for k in ("b", "a", "gj", "gi", "tcls")])), i
        assert np.array_equal(tbox[i].cpu().numpy(), d["tbox"]), i
    leaves = [t.detach().requires_grad_(True) for t in p]
    loss, items = crit(leaves, tgd)
    (loss * scale).backward()
    obj, rows = R.leaves_from_maps(p, bt)
    res = R.loss64(obj, rows, bt, HYP_SCRATCH_LOW, 80, bs, dtype=dtype, scale=scale, balance=BALANCE4)
    got = torch.cat((loss.detach().double().cpu(), items.double().cpu()))
    ref = torch.cat((torch.tensor([res["loss"]], dtype=torch.float64), res["items"]))
    assert bool(((got - ref).abs() <= 2e-5 * ref.abs() + 1e-7).all()), (got.tolist(), ref.tolist())
    u, z = U[dtype], Z[dtype]
    worst = []
    for l, (t, d) in enumerate(zip(leaves, bt)):
        g = t.grad
        ucell = d["ucell"].to(cuda)
        rest = g.clone().reshape(-1, no)
        rest[:, 4] = 0
        rest[ucell] = 0
        assert not bool(rest.any()), (l, "gradient outside the objectness channel and the matched cells")
        go, gr = g[..., 4].double().cpu().reshape(-1), res["gobj"][l].reshape(-1)
        gsc = HYP_SCRATCH_LOW["obj"] * BALANCE4[l] * bs * scale / d["cells"]
        bound = u * gr.abs() + 1e-5 * float(gr.abs().max()) + z
        bound[d["ucell"]] += gsc * _ulp(res["tobj"][l], dtype)
        worst.append((l, "obj", _ratio((go - gr).abs(), bound)))
        grow = g.reshape(-1, no)[ucell].double().cpu()
        mult = d["mult"].double()[:, None]
        for term, sl in (("xy", slice(0, 2)), ("wh", slice(2, 4)), ("cls", slice(5, None))):
            e, a = res["grows"][l][:, sl], res["arows"][l][:, sl]
            s = float(e.abs().max()) if e.numel() else 0.0
            worst.append((l, term, _ratio((grow[:, sl] - e).abs(), mult * u * a + 1e-5 * s + z)))
    print("P6 loss parity", dtype, "matches", [len(d["b"]) for d in bt], [(f"P{l + 3}", t, f"{r:.3g}") for l, t, r in worst])
    assert all(r <= 1.0 for _, _, r in worst), worst


def test_graphed_train_step_matches_eager(cuda):
    """GraphedTrainStep captures the four-level step: its steps give the eager loop's loss items and weights."""
    from yolov5_b200.utils.loss import ComputeLoss
    from yolov5_b200.utils.torch_utils import GraphedTrainStep, smart_optimizer

    ma, mb = _small_model(cuda), _small_model(cuda)
    imgs = [_uint8((2, 3, 256, 256), 70 + i).to(cuda) for i in range(3)]
    tgts = [torch.from_numpy(_targets(2, 80 + 2 * i)).to(cuda) for i in range(3)]
    oa = smart_optimizer(ma, "SGD", lr=0.01, momentum=0.937, decay=5e-4)
    ob = smart_optimizer(mb, "SGD", lr=0.01, momentum=0.937, decay=5e-4)
    step = GraphedTrainStep(ma, ComputeLoss(ma), oa, batch=2, size=256)
    lb, sb = ComputeLoss(mb), torch.amp.GradScaler("cuda")
    w0 = torch.cat([v.detach().flatten() for v in ma.parameters()]).clone()
    for i in range(3):
        items_a = step(imgs[i], tgts[i]).clone()
        with torch.autocast("cuda", dtype=F16):
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


class _RectValDataset:
    """The attributes DeviceValLoader reads from the reference's LoadImagesAndLabels(rect=True, pad=0.5), with batch_shapes
    computed as its __init__ computes them for the model's maximum stride."""

    def __init__(self, srcs, labels, img_size, batch_size, stride):
        ar = np.array([s.shape[0] / s.shape[1] for s in srcs])
        order = ar.argsort()
        self.src, self.labels, ar = [srcs[i] for i in order], [labels[i] for i in order], ar[order]
        n = len(srcs)
        self.segments = [[] for _ in range(n)]
        self.img_size, self.augment, self.image_weights, self.rect, self.mosaic = img_size, False, False, True, False
        self.batch = np.floor(np.arange(n) / batch_size).astype(int)
        shapes = [[1, 1]] * (self.batch[-1] + 1)
        for i in range(len(shapes)):
            ari = ar[self.batch == i]
            mini, maxi = ari.min(), ari.max()
            if maxi < 1:
                shapes[i] = [maxi, 1]
            elif mini > 1:
                shapes[i] = [1, 1 / mini]
        self.batch_shapes = np.ceil(np.array(shapes) * img_size / stride + 0.5).astype(int) * stride
        self.indices, self.n = np.arange(n), n
        self.im_files = [f"im{k}.png" for k in range(n)]
        self.im_hw0 = [s.shape[:2] for s in self.src]
        self.ims = [None] * n

    def __len__(self):
        return self.n


def test_rect_val_batches_at_stride_64(cuda):
    """DeviceValLoader over rect batches built at stride 64 -> forward -> NMS -> val_batch_metrics: the loader's batches equal the
    oracle's (letterbox and labels), and `correct` equals the one computed from the oracle's batch."""
    from oracle import val_load_ref as V
    from tests import val_load_fixture as VF
    from yolov5_b200.utils import metrics
    from yolov5_b200.utils.dataloaders import DeviceValLoader
    from yolov5_b200.utils.general import nms_device

    rs = np.random.RandomState(90)
    hw = [(300, 500), (420, 330), (250, 640), (640, 480), (377, 377), (200, 520)]
    srcs = [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in hw]
    labels = []
    for _ in hw:
        k = rs.randint(1, 6)
        labels.append(np.concatenate((rs.randint(0, 3, (k, 1)), rs.uniform(0.3, 0.7, (k, 2)), rs.uniform(0.05, 0.5, (k, 2))), 1).astype(np.float32))
    ds = _RectValDataset(srcs, labels, 320, 3, 64)
    assert (ds.batch_shapes % 64 == 0).all() and any(s[0] != s[1] for s in ds.batch_shapes)
    m = _loaded(cuda, F16)
    iouv = torch.linspace(0.5, 0.95, 10, device=cuda)

    def step(imgs, targets, shapes):
        h, w = imgs.shape[2:]
        x = imgs.half() / 255 if imgs.dtype == torch.uint8 else imgs
        rows, _, count = nms_device(m(x)[0], 0.001, 0.6, max_det=300)
        tg = targets.clone()
        tg[:, 2:] *= torch.tensor((w, h, w, h), device=cuda)
        return metrics.val_batch_metrics(rows, count, tg, (h, w), shapes, iouv)[1], count

    loader = DeviceValLoader(ds, 3, device=cuda, dtype=torch.uint8, workers=2, decode=VF.decode)
    nb = 0
    for bi, (imgs, targets, _, shapes) in enumerate(loader):
        items = [V.get_item(V.load_resize(ds.src[k], 320), ds.im_hw0[k], ds.labels[k], ds.batch_shapes[ds.batch[k]])
                 for k in range(3 * bi, min(3 * bi + 3, ds.n))]
        ri, rt, rsh = V.get_batch(items)
        assert tuple(imgs.shape[2:]) == tuple(ds.batch_shapes[bi]) and np.array_equal(imgs.cpu().numpy(), ri), bi
        assert np.array_equal(targets.cpu().numpy(), rt), bi
        got, gc = step(imgs, targets, shapes)
        want, wc = step(torch.from_numpy(ri).to(cuda), torch.from_numpy(rt).to(cuda), rsh)
        assert int(gc.min()) > 0 and torch.equal(gc, wc) and torch.equal(got, want), bi
        nb += 1
    assert nb == 2


def _synth_model(name, dev, seed, head_bias="init"):
    from yolov5_b200.models.yolo import DetectionModel

    sd = model_ref.synth_state_dict(model_cfg(name), seed=seed, head_bias=head_bias)
    m = DetectionModel(name)
    m.load_state_dict(sd)
    return m.to(dev).half().eval(), sd


def test_nms_on_1280_output_vs_oracle(cuda):
    """yolov5n6 at 2 x 1280: 102 000 rows per image, every one a candidate at val's conf_thres, so the max_nms cut applies;
    the public non_max_suppression equals the oracle row for row and index for index."""
    from oracle import nms_ref
    from yolov5_b200.utils.general import non_max_suppression

    m, _ = _synth_model("yolov5n6", cuda, 40, head_bias="hot")
    with torch.no_grad():
        z = m(_image((2, 3, 1280, 1280), 41).to(cuda, F16))[0]
    assert z.shape == (2, 3 * (160**2 + 80**2 + 40**2 + 20**2), 85) == (2, 102000, 85)
    conf = z[..., 4:5].float() * z[..., 5:].float()
    assert int(((z[..., 4].float() > 0.001) & (conf.amax(-1) > 0.001)).sum(1).min()) > 30000
    for conf_thres, iou_thres in ((0.001, 0.6), (0.25, 0.45)):
        dets, idx = non_max_suppression(z, conf_thres, iou_thres, max_det=300, return_indices=True)
        for b in range(2):
            ref, ridx = nms_ref.non_max_suppression(z[b : b + 1].float().cpu().numpy(), conf_thres, iou_thres, max_det=300, dtype="fp16",
                                                    return_index=True)
            assert len(ref[0]) > 0
            assert np.array_equal(idx[b].cpu().numpy(), ridx[0]) and np.array_equal(dets[b].cpu().numpy(), ref[0]), (conf_thres, b)


@pytest.mark.parametrize("size", [640, 1280])
@pytest.mark.parametrize("scale", "nsmlx")
def test_full_size_models_plan_run_capture(cuda, scale, size):
    """yolov5{n..x}6 fp16 at batch 1: z and the four raw maps against the fp32 oracle on the device (TF32 off), within
    1e-3 + 1.5 x the error of torch's own fp16 run of the same expressions (test_model_gpu.py's criterion); the CUDA graph replays
    to the same bytes."""
    name = f"yolov5{scale}6"
    m, sd = _synth_model(name, cuda, 50, head_bias="hot")
    cfg = model_cfg(name)
    x = _image((1, 3, size, size), 51).to(cuda)
    with torch.no_grad():
        z, raws = m(x.half())
        z2 = m(x.half())[0]
        assert torch.equal(z, z2)
        with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
            ref = model_ref.forward(cfg, {k: v.to(cuda) for k, v in sd.items()}, x.half().float(), fused=True)
        low = model_ref.forward(cfg, {k: v.to(cuda, F16) if v.is_floating_point() else v.to(cuda) for k, v in sd.items()}, x.half(), fused=True)
    assert [tuple(r.shape[2:4]) for r in raws] == [(size // s, size // s) for s in STRIDES]
    report = {}
    for tag, got, r, lo in [("z", z, ref[0], low[0])] + [(f"raw{l}", a, b, c) for l, (a, b, c) in enumerate(zip(raws, ref[1], low[1]))]:
        assert got.shape == r.shape, (tag, got.shape, r.shape)
        sc = float(r.abs().max())
        e, el = float((got.float() - r).abs().max()), float((lo.float() - r).abs().max())
        report[tag] = (f"{e / sc:.2e}", f"{el / sc:.2e}")
        assert e <= 1e-3 * sc + 1.5 * el, (name, size, tag, e / sc, el / sc)
    print("P6 full-size parity", name, size, report)
