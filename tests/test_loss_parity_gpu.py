"""GPU: ComputeLoss (y5_loss_fwd_bwd_scaled) forward and backward vs the float64 reference tests/loss64_ref.py, per level
and per term, at the training shape, in the looping regime of the match / class kernels, at the edges of build_targets,
on CIoU ties, with non-default hyper-parameters and class counts.

build_targets is compared bit-exactly with oracle.loss_ref.  Loss and items: |got - ref| <= 2e-5 |ref| + 1e-7.  Every
gradient element of term T (xy = channels 0-1, wh = 2-3, obj = 4, cls = 5..) of a level satisfies
    |g - g_ref| <= m u_D A + 1e-5 S + z_D
with u_D the unit roundoff of the logits dtype, m the matches summed into the element, A the sum of their absolute
contributions (each atomic add rounds), S the largest |g_ref| of that level and term, z_D half the fp16 subnormal
spacing (0 otherwise).  At matched objectness cells one dtype ulp of tobj (times the objectness gradient's scale) is
added: the kernel's fp32 IoU and the reference's float64 IoU can round to neighbouring values.  Every other gradient
element is exactly zero.  The worst err / bound of every case, level and term is printed (run with -s to see it).
"""
import numpy as np
import pytest
import torch

from oracle import loss_ref
from tests import loss64_ref as R
from tests.golden import make_seg_golden as mg
from yolov5_b200.cfg import HYP_SCRATCH_LOW
from yolov5_b200.utils.loss import ComputeLoss

pytestmark = pytest.mark.gpu

F16, BF16, F32 = torch.float16, torch.bfloat16, torch.float32
U = {F32: 2.0**-24, F16: 2.0**-11, BF16: 2.0**-8}
Z = {F32: 0.0, F16: 2.0**-25, BF16: 0.0}
ROW_TERMS = (("xy", slice(0, 2)), ("wh", slice(2, 4)), ("cls", slice(5, None)))


def _crit(nc=80, **hyp):
    m = mg.LossModel(nc)
    m.hyp.update(hyp)
    return ComputeLoss(m)


def _maps(dev, dtype, bs, h, w, no, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return [(torch.randn(bs, 3, h // s, w // s, no, generator=g, device=dev) * 1.5).to(dtype) for s in (8, 16, 32)]


def _ulp(t, dtype):
    return 2 * U[dtype] * torch.exp2(torch.floor(torch.log2(t.clamp_min(torch.finfo(dtype).tiny))))


def _ratio(err, bound):
    r = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, torch.inf, 0.0))
    return float(r.max()) if r.numel() else 0.0


def check(case, p, tg, crit, scale=1.0, ref_tg=None):
    """Runs ComputeLoss(p, tg) forward and backward(loss * scale) and checks it against the float64 reference of `ref_tg`
    (default `tg`).  Returns (reference targets, reference result, head-map gradients)."""
    dev, dtype, bs, no = p[0].device, p[0].dtype, p[0].shape[0], p[0].shape[-1]
    hyp, nc = crit.hyp, crit.nc
    shapes = [tuple(t.shape[2:4]) for t in p]
    bt = R.targets_for(tg if ref_tg is None else ref_tg, mg.anchors_grid().numpy(), shapes, bs, hyp["anchor_t"])
    tgd = torch.from_numpy(tg).to(dev)
    tcls, tbox, idx, _ = crit.build_targets(p, tgd)
    for i, d in enumerate(bt):
        got = np.stack([idx[i][q].cpu().numpy() for q in range(4)] + [tcls[i].cpu().numpy()])
        assert got.dtype == np.int64 and np.array_equal(got, np.stack([d[k] for k in ("b", "a", "gj", "gi", "tcls")])), (case, i)
        assert np.array_equal(tbox[i].cpu().numpy(), d["tbox"]), (case, i)
    leaves = [t.detach().requires_grad_(True) for t in p]
    loss, items = crit(leaves, tgd)
    (loss * scale).backward()
    obj, rows = R.leaves_from_maps(p, bt)
    res = R.loss64(obj, rows, bt, hyp, nc, bs, dtype=dtype, scale=scale)
    got = torch.cat((loss.detach().double().cpu(), items.double().cpu()))
    ref = torch.cat((torch.tensor([res["loss"]], dtype=torch.float64), res["items"]))
    assert bool(((got - ref).abs() <= 2e-5 * ref.abs() + 1e-7).all()), (case, got.tolist(), ref.tolist())
    u, z = U[dtype], Z[dtype]
    pwf = max(1.0, hyp["obj_pw"])
    worst = []
    for l, (t, d) in enumerate(zip(leaves, bt)):
        g = t.grad
        ucell = d["ucell"].to(dev)
        rest = g.clone().reshape(-1, no)
        rest[:, 4] = 0
        rest[ucell] = 0
        assert not bool(rest.any()), (case, l, "gradient outside the objectness channel and the matched cells")
        # objectness: one store per element, and one ulp of tobj at the matched cells
        go, gr = g[..., 4].double().cpu().reshape(-1), res["gobj"][l].reshape(-1)
        gs = hyp["obj"] * R.BALANCE[l] * bs * scale / d["cells"]
        bound = u * gr.abs() + 1e-5 * float(gr.abs().max()) + z
        if len(d["ucell"]):
            bound[d["ucell"]] += pwf * gs * _ulp(res["tobj"][l], dtype)
        worst.append((l, "obj", _ratio((go - gr).abs(), bound)))
        grow = g.reshape(-1, no)[ucell].double().cpu()
        m = d["mult"].double()[:, None]
        for term, sl in ROW_TERMS:
            e, a = res["grows"][l][:, sl], res["arows"][l][:, sl]
            s = float(e.abs().max()) if e.numel() else 0.0
            worst.append((l, term, _ratio((grow[:, sl] - e).abs(), m * u * a + 1e-5 * s + z)))
    counts = [len(d["b"]) for d in bt]
    print()
    for l, term, r in worst:
        print(f"loss-parity {case:<28} P{l + 3} {term:<3} matches {counts[l]:>6}  worst err/bound {r:.3g}")
    bad = [(l, term, r) for l, term, r in worst if not r <= 1.0]
    assert not bad, (case, bad)
    return bt, res, [t.grad for t in leaves]


# ---------------------------------------------------------------------------------------------------------------------
# the training shape: 16 images of 640 x 640, COCO-like labels, nc 80 (bench.py's yolov5s / yolov5m training workloads)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,scale", [(F16, 65536.0 * 8), (BF16, 8.0), (F32, 1.0)], ids=["fp16", "bf16", "fp32"])
def test_training_shape(cuda, dtype, scale):
    p = _maps(cuda, dtype, 16, 640, 640, 85, seed=101)
    tg = loss_ref.synth_targets(16, seed=102)
    bt, _, _ = check(f"train16x640-{dtype}".replace("torch.", ""), p, tg, _crit(), scale)
    assert all(len(d["b"]) > 0 for d in bt)


def test_training_shape_padded_targets(cuda):
    """GraphedTrainStep pads the labels with zero rows up to max_targets = 64 x batch: they match nothing."""
    p = _maps(cuda, F16, 16, 640, 640, 85, seed=103)
    tg = loss_ref.synth_targets(16, seed=104)
    padded = np.zeros((64 * 16, 6), np.float32)
    padded[: len(tg)] = tg
    check("train16x640-padded-float16", p, padded, _crit(), 65536.0 * 8, ref_tg=tg)


def test_training_shape_no_targets(cuda):
    p = _maps(cuda, F16, 16, 640, 640, 85, seed=105)
    _, res, _ = check("train16x640-nt0-float16", p, np.zeros((0, 6), np.float32), _crit(), 65536.0)
    assert float(res["items"][0]) == 0.0 and float(res["items"][2]) == 0.0


# ---------------------------------------------------------------------------------------------------------------------
# crowded: more than 32,768 matches at P3, so loss_match_kernel's grid-stride loop and loss_cls_kernel's warp loop run
# more than one round
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [F32, F16], ids=["fp32", "fp16"])
def test_crowded_looping(cuda, dtype):
    p = _maps(cuda, dtype, 4, 640, 640, 85, seed=106)
    tg = R.crowded_targets(4, 2000, 640, seed=107)
    scale = 65536.0 * 8 if dtype == F16 else 8.0  # fp16 under GradScaler's scale, as it trains
    bt, _, _ = check(f"crowded4x640-{dtype}".replace("torch.", ""), p, tg, _crit(), scale)
    counts = [len(d["b"]) for d in bt]
    print(f"loss-parity crowded matches per level {counts}, duplicate cells at P3 {int((bt[0]['mult'] > 1).sum())}")
    assert counts[0] > 32768 and counts[0] > 256 * 8


# ---------------------------------------------------------------------------------------------------------------------
# geometry edges on small grids (64 x 64: P3 8 x 8, P4 4 x 4, P5 2 x 2)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [F32, BF16], ids=["fp32", "bf16"])
def test_geometry_edges(cuda, dtype):
    p = _maps(cuda, dtype, 2, 64, 64, 85, seed=108)
    tg = R.edge_targets()
    bt, _, _ = check(f"edges-{dtype}".replace("torch.", ""), p, tg, _crit(), 4.0)
    assert sum(int((d["mult"] > 1).sum()) for d in bt) > 0


@pytest.mark.parametrize("dtype", [F32, BF16], ids=["fp32", "bf16"])
def test_out_of_range_rows_are_ignored(cuda, dtype):
    """Rows with class >= nc or < 0, image >= batch or < 0 are ignored: the loss is the reference's over the others."""
    p = _maps(cuda, dtype, 2, 64, 64, 85, seed=109)
    good = R.edge_targets()
    tg = np.concatenate((good[:5], R.invalid_rows(2, 80), good[5:]))
    check(f"invalid-rows-{dtype}".replace("torch.", ""), p, tg, _crit(), 1.0, ref_tg=good)


def test_single_target(cuda):
    p = _maps(cuda, F32, 2, 64, 64, 85, seed=110)
    check("one-target-float32", p, np.array([[1, 7, 0.4, 0.6, 0.3, 0.2]], np.float32), _crit())


# ---------------------------------------------------------------------------------------------------------------------
# CIoU ties: box logits 0 in image 0, so every predicted box there is (0.5, 0.5, aw, ah); targets on that box (full
# overlap), sharing one edge with it, and touching it.  torch splits min / max gradients on a tie and passes clamp(0)'s at 0
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [F32, BF16], ids=["fp32", "bf16"])
def test_ciou_ties(cuda, dtype):
    p = _maps(cuda, dtype, 2, 64, 64, 85, seed=111)
    for t in p:
        t[0, ..., 0:4] = 0
    other = loss_ref.synth_targets(2, seed=112)
    tg = np.concatenate((R.tie_targets(), other[other[:, 0] == 1]))
    bt, res, grads = check(f"ties-{dtype}".replace("torch.", ""), p, tg, _crit(), 1.0)
    # the full-overlap match (P3 anchor 0, cell (2, 3)): the IoU is at its maximum, its w / h gradient ~0
    d = bt[0]
    k = int(np.nonzero((d["b"] == 0) & (d["a"] == 0) & (d["gi"] == 2) & (d["gj"] == 3))[0][0])
    g = grads[0][0, 0, 3, 2, 0:4].float().cpu()
    gbox = HYP_SCRATCH_LOW["box"] * 2 / len(d["b"])
    assert float(g.abs().max()) <= 1e-5 * gbox, (g.tolist(), res["grows"][0][d["inv"][k]][0:4].tolist())


# ---------------------------------------------------------------------------------------------------------------------
# hyper-parameters: label smoothing, pos weights, class counts
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nc,dtype", [(1, F32), (3, F32), (80, F32), (80, BF16)], ids=["nc1-fp32", "nc3-fp32", "nc80-fp32", "nc80-bf16"])
def test_hyper_parameters(cuda, nc, dtype):
    p = _maps(cuda, dtype, 4, 128, 160, 5 + nc, seed=113)
    tg = loss_ref.synth_targets(4, seed=114, nc=nc)
    crit = _crit(nc, label_smoothing=0.1, cls_pw=1.3, obj_pw=1.3)
    _, res, grads = check(f"smooth-pw1.3-nc{nc}-{dtype}".replace("torch.", ""), p, tg, crit, 8.0)
    if nc == 1:
        assert float(res["items"][2]) == 0.0
        assert not any(bool(g[..., 5].any()) for g in grads)


# ---------------------------------------------------------------------------------------------------------------------
# call forms
# ---------------------------------------------------------------------------------------------------------------------
def test_repeated_calls_are_bit_identical(cuda):
    p = _maps(cuda, F16, 8, 320, 320, 85, seed=115)
    tg = torch.from_numpy(loss_ref.synth_targets(8, seed=116)).to(cuda)
    crit = _crit()
    a, ia = crit(p, tg)
    b, ib = crit(p, tg)
    assert torch.equal(a, b) and torch.equal(ia, ib)


@pytest.mark.parametrize("dtype", [F32, F16], ids=["fp32", "fp16"])
def test_non_contiguous_head_maps(cuda, dtype):
    """A permuted view (B, na, ny, nx, no) of a (B, ny, nx, na, no) buffer gives the loss and gradients of its copy."""
    g = torch.Generator(device=cuda).manual_seed(117)
    base = [(torch.randn(4, 128 // s, 160 // s, 3, 85, generator=g, device=cuda) * 1.5).to(dtype).requires_grad_(True) for s in (8, 16, 32)]
    views = [b.permute(0, 3, 1, 2, 4) for b in base]
    assert not any(v.is_contiguous() for v in views)
    copies = [v.detach().contiguous().requires_grad_(True) for v in views]
    tg = torch.from_numpy(loss_ref.synth_targets(4, seed=118)).to(cuda)
    crit = _crit()
    la, ia = crit(views, tg)
    (la * 8).backward()
    lb, ib = crit(copies, tg)
    (lb * 8).backward()
    assert torch.equal(la, lb) and torch.equal(ia, ib)
    for b, c in zip(base, copies):
        ga, gb = b.grad.permute(0, 3, 1, 2, 4).float(), c.grad.float()
        # matched cells sum their matches with atomics, in any order: equal to the rounding of each add
        assert bool(((ga - gb).abs() <= 4 * U[dtype] * gb.abs()).all())
