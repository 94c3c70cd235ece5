"""GPU: the segmentation ComputeLoss (y5_seg_loss_fwd_bwd_scaled) forward and backward vs the float64 reference
tests/seg_loss64_ref.py, per level and per term, at the shapes segmentation trains with and at the mask term's edges.

build_targets: all six lists bit-exact with seg_loss_ref.build_targets_seg.  Loss and items [loss, lbox, lseg, lobj, lcls]:
|got - ref| <= 2e-5 |ref| + 1e-7.  Gradients (u_D the unit roundoff of the logits dtype, u32 fp32's, S the largest
|ref| of that level and term, z_D half the fp16 subnormal spacing, m the matches of the cell, A the sum of their absolute
contributions):
- xy / wh / obj / cls channels: test_loss_parity_gpu's bounds, m u_D A + 1e-5 S + z_D (one dtype ulp of tobj times the
  objectness gradient's scale added at matched objectness cells, u_D |ref| + 1e-5 S + z_D elsewhere);
- mask-coefficient channels 5+nc .. 5+nc+nm of matched cells:
      sum_j u32 (k_j acoef_j + ecoef_j) + m u_D A + 1e-5 S + z_D
  seg_match_kernel runs one 256-thread CTA per match j: each thread sums g_p proto_kp over its crop pixels p = tid,
  tid + 256, ... with one FMA each (ceil(npix_j / 256) roundings), then a 5-step warp shuffle tree and a serial sum of the
  8 warps: k_j = ceil(npix_j / 256) + 5 + 8 roundings, each at most u32 of a partial sum <= acoef_j = |g_j| @ |proto|^T.
  ecoef_j = E_j @ |proto|^T carries the fp32 error of g_p itself (the logit's nm-term FMA chain, __expf, __fdividef,
  sigmoid - gt, the scale; seg_loss64_ref's docstring derives E).  The result is rounded to the dtype and atomically
  added into the cell, once per match: m u_D A;
- dproto: u_D |ref| + (n_cover + 1) u32 aproto + u32 eproto + z_D.  seg_proto_kernel writes every element once (no
  atomics): one fp32 FMA g_jp coef_jk per match j whose crop covers p, in list order (n_cover roundings of partial sums
  <= aproto = sum_j |coef_j| |g_jp|), the error of each g_jp (eproto), then one rounding to the proto dtype.
Every other gradient element is exactly 0: the mask channels of unmatched cells, every channel but objectness outside the
matched cells, and dproto wherever no crop of the image covers the pixel.  Just before the backward call a NaN-filled block
of every gradient's size is allocated and freed, so the caching allocator hands that memory to the gradients and "exactly
0" means the kernels wrote it.  fp16: where the float64 value rounds to inf, the kernel must give inf of the same sign.

The worst err / bound of every case, level and term is printed (run with -s to see it).
"""
import numpy as np
import pytest
import torch

from tests import seg_loss64_ref as S
from tests.golden import make_seg_golden as mg
from yolov5_b200.utils.segment.loss import ComputeLoss

pytestmark = pytest.mark.gpu

F16, BF16, F32 = torch.float16, torch.bfloat16, torch.float32
AMP = 65536.0 * 8  # GradScaler's initial scale, times the batch-size factor of the loss


def _crit(nc, nm, overlap):
    m = mg.LossModel(nc)
    m.model[-1].nm = nm
    return ComputeLoss(m, overlap=overlap)


def run(name, case, dev, dtype, scale=1.0, channels_last=False):
    """ComputeLoss forward, backward(loss * scale) on the case's inputs in `dtype`; checked against the float64 reference.
    Returns the reference result."""
    nc, nm, overlap = case["nc"], case["proto"].shape[1], case["overlap"]
    p = [torch.from_numpy(a).to(dev, dtype) for a in case["p"]]
    proto = torch.from_numpy(case["proto"]).to(dev, dtype)
    if channels_last:
        proto = proto.contiguous(memory_format=torch.channels_last)
    tg = torch.from_numpy(case["targets"]).to(dev)
    masks = torch.from_numpy(case["masks"]).to(dev)
    crit = _crit(nc, nm, overlap)
    ref = S.reference(p, proto, case["targets"], masks, overlap, crit.hyp, dtype=dtype, scale=scale)

    tcls, tbox, indices, anch, tidxs, xywhn = crit.build_targets(p, tg)
    for i, d in enumerate(ref["bt"]):
        got = np.stack([indices[i][q].cpu().numpy() for q in range(4)] + [tcls[i].cpu().numpy(), tidxs[i].cpu().numpy()])
        assert got.dtype == np.int64 and np.array_equal(got, np.stack([d[k] for k in ("b", "a", "gj", "gi", "tcls", "tidx")])), (name, i)
        assert np.array_equal(tbox[i].cpu().numpy(), d["tbox"]) and np.array_equal(xywhn[i].cpu().numpy(), d["xywhn"]), (name, i)
        assert np.array_equal(anch[i].cpu().numpy(), d["anch"]), (name, i)

    leaves = [t.detach().requires_grad_(True) for t in p]
    pl = proto.detach().requires_grad_(True)
    loss, items = crit((leaves, pl), tg, masks)
    junk = [torch.full_like(t, float("nan")) for t in leaves + [pl]]
    del junk
    (loss * scale).backward()
    assert pl.grad.dtype == dtype and pl.grad.stride() == pl.stride()

    no = p[0].shape[-1]
    outside, obj, rows = 0, [], []
    for t, d in zip(leaves, ref["bt"]):
        g = t.grad.reshape(-1, no)
        ucell = d["ucell"].to(dev)
        rest = g.clone()
        rest[:, 4] = 0
        rest[ucell] = 0
        outside += int((rest != 0).sum())
        obj.append(t.grad[..., 4].double().cpu())
        rows.append(g[ucell].double().cpu())
    got = dict(loss=float(loss), items=items.double().cpu(), obj=obj, rows=rows, proto=pl.grad.double(), outside=outside)
    table = S.ratios(got, ref)
    counts = [len(d["b"]) for d in ref["bt"]]
    print()
    for where, term, r in table:
        print(f"seg-loss-parity {name:<30} {where:<5} {term:<7} matches {counts}  worst err/bound {r:.3g}")
    bad = [(where, term, r) for where, term, r in table if not r <= 1.0]
    assert not bad, (name, bad)
    return ref


def _matches(ref):
    return [len(d["b"]) for d in ref["bt"]]


# ---------------------------------------------------------------------------------------------------------------------
# the training shape: 16 images of 640 x 640, nc 80, nm 32, overlap masks at 160 x 160
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,scale", [(F16, AMP), (BF16, 8.0), (F32, 1.0)], ids=["fp16", "bf16", "fp32"])
def test_training_shape(cuda, dtype, scale):
    ref = run(f"train16x640-{dtype}".replace("torch.", ""), S.training_case(), cuda, dtype, scale)
    # seg_match_kernel's grid is min(cap, 4 SMs) CTAs: some level takes a second round of its grid-stride loop
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    assert max(_matches(ref)) > 4 * sms, (_matches(ref), sms)


def test_no_overlap(cuda):
    """--no-overlap: one mask per target row, with holes."""
    ref = run("nonoverlap16x640-float16", S.no_overlap_case(), cuda, F16, AMP)
    assert all(n > 0 for n in _matches(ref))


@pytest.mark.parametrize("ratio,dtype", [(1, F16), (8, F16), (1, F32), (8, F32)], ids=["r1-fp16", "r8-fp16", "r1-fp32", "r8-fp32"])
def test_mask_ratio(cuda, ratio, dtype):
    """Masks at 640^2 (downsampled by 4 in the read) and at 80^2 (upsampled by 2) for a 160^2 proto."""
    case = S.mask_ratio_case(ratio)
    assert case["masks"].shape[-1] == 640 // ratio and case["proto"].shape[-1] == 160
    run(f"ratio{ratio}-16x640-{dtype}".replace("torch.", ""), case, cuda, dtype, AMP if dtype == F16 else 1.0)


@pytest.mark.parametrize("shape", [(16, 480, 640), (8, 320, 256)], ids=["16x480x640", "8x320x256"])
@pytest.mark.parametrize("channels_last", [False, True], ids=["nchw", "nhwc"])
def test_rect(cuda, shape, channels_last):
    """Non-square maps and protos (120 x 160: a partial 16-pixel tile row; 80 x 64: taller than wide)."""
    case = S.rect_case(*shape)
    mh, mw = case["proto"].shape[2:]
    assert mh != mw
    if shape[1] == 480:
        assert mh % S.TILE != 0
    run(f"rect{'x'.join(map(str, shape))}-{'nhwc' if channels_last else 'nchw'}-float16", case, cuda, F16, AMP, channels_last)


@pytest.mark.parametrize("dtype,scale", [(F16, AMP), (F32, 1.0)], ids=["fp16", "fp32"])
def test_crowded(cuda, dtype, scale):
    """300 labels per image in int32 masks: tidx past 255, many grid-stride rounds, many 32-match batches per tile."""
    case = S.crowded_case()
    assert case["masks"].dtype == np.int32
    ref = run(f"crowded4x640-{dtype}".replace("torch.", ""), case, cuda, dtype, scale)
    assert max(int(d["tidx"].max()) for d in ref["bt"]) > 255
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    assert max(_matches(ref)) > 8 * sms
    # the most matches whose crop meets one 16 x 16 proto tile of one image
    mh, mw = case["proto"].shape[2:]
    ty = torch.arange(0, mh, S.TILE)[:, None, None]
    tx = torch.arange(0, mw, S.TILE)[None, :, None]
    most = 0
    crop = torch.cat(ref["mask"]["crop"])
    b = torch.cat([torch.from_numpy(d["b"]) for d in ref["bt"]])
    for bi in range(case["proto"].shape[0]):
        x0, x1, y0, y1 = crop[b == bi].T
        hit = (torch.maximum(x0, tx) < torch.minimum(x1, tx + S.TILE)) & (torch.maximum(y0, ty) < torch.minimum(y1, ty + S.TILE))
        most = max(most, int(hit.sum(-1).max()))
    print(f"seg-loss-parity crowded: matches {_matches(ref)}, most matches on one tile {most}")
    assert most > 32


@pytest.mark.parametrize("dtype,scale", [(F32, 1.0), (BF16, 8.0), (F16, AMP)], ids=["fp32", "bf16", "fp16"])
def test_edges(cuda, dtype, scale):
    """Integer crop edges, boxes over the map border, a crop with no pixel, and the smallest P3 box alone in its image:
    its mask-gradient scale is the largest there is, and under fp16 at GradScaler's scale its gradients overflow."""
    case = S.edges_case()
    ref = run(f"edges2x640-{dtype}".replace("torch.", ""), case, cuda, dtype, scale)
    m = ref["mask"]
    npix = torch.cat(m["npix"]).cpu()
    assert int((npix == 0).sum()) > 0, "no empty crop"
    xy = S.crop_xyxy(np.concatenate([d["xywhn"] for d in ref["bt"]]), 160, 160)
    integer = (xy == torch.floor(xy)).all(1) & (xy[:, 2:] < 160).all(1) & (npix > 0)
    assert bool(integer.any()), "no integer-edge crop"
    assert int(m["nimg"][0, 1]) == 1, "the smallest box is not alone at P3 in image 1"
    if dtype == F16:
        assert float(ref["gproto"].abs().max()) >= S.F16_OVERFLOW
        assert float(ref["grows"][0][:, 5 + case["nc"]:].abs().max()) >= S.F16_OVERFLOW


def test_batch_layout(cuda):
    """Images without labels first, in the middle and last; targets shuffled; uint8 masks: tidx is positional."""
    case = S.batch_layout_case()
    tg = case["targets"]
    assert case["masks"].dtype == np.uint8 and not np.all(np.diff(tg[:, 0]) >= 0)
    ref = run("layout8x320-float32", case, cuda, F32, 1.0)
    for bi in (0, 3, 7):
        assert int(ref["mask"]["nimg"][:, bi].sum()) == 0


@pytest.mark.parametrize("nm,nc,dtype", [(1, 1, F32), (1, 3, BF16), (16, 1, BF16), (16, 3, F32)],
                         ids=["nm1-nc1-fp32", "nm1-nc3-bf16", "nm16-nc1-bf16", "nm16-nc3-fp32"])
def test_nm_and_nc(cuda, nm, nc, dtype):
    """Segment(nm=...) below 32 (the kernels' k < nm guards) and nc 1 (no class term)."""
    ref = run(f"nm{nm}-nc{nc}-4x256x320-{dtype}".replace("torch.", ""), S.nm_case(nm, nc), cuda, dtype, 8.0)
    if nc == 1:
        assert float(ref["items"][3]) == 0.0


def test_invalid_rows(cuda):
    """Non-overlap with class >= nc and image >= batch rows in the middle: ignored, but still owning their mask slot."""
    case = S.invalid_rows_case()
    ref = run("invalid-rows4x320-float32", case, cuda, F32, 1.0)
    k = (len(case["targets"]) - 3) // 2  # the three ignored rows are k, k + 1, k + 2
    tidx = set(np.concatenate([d["tidx"] for d in ref["bt"]]).tolist())
    assert not tidx & {k, k + 1, k + 2} and max(tidx) > k + 2  # the rows after them keep their global index
