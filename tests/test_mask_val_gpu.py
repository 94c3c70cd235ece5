"""GPU: mask-IoU matching of segment/val.py on the device (csrc/mask_metrics.cu through yolov5_b200.utils.metrics).

Bit rows against np.packbits of the oracle's masks for every source mode, mask_iou bit-equal to the fp32 torch expression,
process_batch(masks=True) bit-equal to the reference fixture, the batched seg_val_batch_metrics against the per-image oracle
(overlap, non-overlap, resize, retina, duplicated labels, several staging chunks) and as a replayed CUDA graph."""
import numpy as np
import pytest
import torch

from tests import mask_val_ref
from tests.seg_loss_ref import paint_masks
from yolov5_b200.utils import metrics
from yolov5_b200.utils.general import scale_meta
from yolov5_b200.utils.segment.general import process_mask_batch

pytestmark = pytest.mark.gpu

GOLDEN = np.load(mask_val_ref.__file__.replace("mask_val_ref.py", "golden/mask_val.npz"))


def _bits(t):
    return t.cpu().numpy().view("<i4")


def _engine_pack(src, src_hw, out_hw, n_rows, overlap=False, targets=None, batch=1):
    dev = src.device
    nonbin = torch.zeros(1, dtype=torch.int32, device=dev)
    li = torch.empty(batch + 1 + 2 * n_rows, dtype=torch.int32, device=dev) if targets is not None else None
    bits, pop = metrics._pack(src, src_hw, out_hw, n_rows, nonbin, overlap=overlap, targets=targets, batch=batch, label_index=li)
    torch.cuda.synchronize()
    return _bits(bits), pop.cpu().numpy(), int(nonbin.item()), (li.cpu().numpy() if li is not None else None)


@pytest.mark.parametrize("tag", list(mask_val_ref.CASES))
def test_pack_gt_equals_oracle_bits(cuda, tag):
    det, labels, pred, gt, overlap = mask_val_ref.case_inputs(tag)
    nl = labels.shape[0]
    out_hw = pred.shape[1:]
    ref, vals = mask_val_ref.expand_gt(gt, nl, overlap, out_hw)
    bits, pop, nonbin, _ = _engine_pack(torch.from_numpy(gt).to(cuda), gt.shape[1:], out_hw, nl, overlap=overlap)
    want = mask_val_ref.pack_bits(ref)
    if tag == "odd_ratio":  # DESIGN row f2's criterion: only pixels within 1e-5 of 0.5 may differ
        got = np.unpackbits(bits.view(np.uint8), axis=1, bitorder="little")[:, : out_hw[0] * out_hw[1]].reshape(ref.shape)
        off = got != ref
        assert not off.any() or np.abs(vals[off] - 0.5).max() < 1e-5
    else:
        assert np.array_equal(bits, want)
        assert np.array_equal(pop, ref.reshape(nl, -1).sum(1).astype(np.int32))
    assert nonbin == 0
    if vals is not None and (vals == 0.5).any():  # strict > 0.5: exactly-half pixels come out 0
        assert not ref[vals == 0.5].any()


@pytest.mark.parametrize("dtype", [torch.uint8, torch.bool, torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("shape", [(5, 37, 41), (0, 16, 16), (3, 1, 257), (2, 1280, 1280)])
def test_pack_direct_dtypes_and_odd_sizes(cuda, dtype, shape):
    g = torch.Generator().manual_seed(sum(shape))
    m = torch.rand(shape, generator=g) > 0.6
    bits, pop, nonbin, _ = _engine_pack(m.to(cuda, dtype), shape[1:], shape[1:], shape[0])
    assert np.array_equal(bits, mask_val_ref.pack_bits(m.numpy()))  # words beyond the last pixel are zero
    assert np.array_equal(pop, m.reshape(shape[0], shape[1] * shape[2]).sum(1).numpy().astype(np.int32)) and nonbin == 0


def test_pack_overlap_batched_label_rows(cuda):
    """Targets in any image order: image b's labels become rows li[b].. in target order, label k of b = index value k + 1."""
    rs = np.random.RandomState(3)
    b, h, w = 4, 48, 40
    img = np.array([2, 0, 2, 1, 0, 2, 3, 2, 0, 7, 1.5], np.float32)  # 7 and 1.5: no image
    tg = np.zeros((len(img), 6), np.float32)
    tg[:, 0] = img
    masks = rs.randint(0, 6, (b, h, w)).astype(np.float32)
    masks[1, :3, :3] = 2.5
    for out_hw in ((h, w), (24, 20), (96, 80)):
        bits, pop, nonbin, li = _engine_pack(torch.from_numpy(masks).to(cuda), (h, w), out_hw, len(img), overlap=True,
                                             targets=torch.from_numpy(tg).to(cuda), batch=b)
        off, row_t, row_i = li[: b + 1], li[b + 1: b + 1 + len(img)], li[b + 1 + len(img):]
        assert off.tolist() == [0, 3, 4, 8, 9]
        rows = []
        for bi in range(b):
            ts = np.nonzero(img == bi)[0]
            assert row_t[off[bi]:off[bi + 1]].tolist() == ts.tolist() and (row_i[off[bi]:off[bi + 1]] == bi).all()
            rows.append(mask_val_ref.expand_gt(masks[bi:bi + 1], len(ts), True, out_hw)[0])
        assert sorted(row_t[off[b]:].tolist()) == [9, 10] and (row_i[off[b]:] == -1).all()
        want = mask_val_ref.pack_bits(np.concatenate(rows + [np.zeros((2,) + out_hw, np.float32)]))
        assert np.array_equal(bits, want) and nonbin == 0


def test_pack_counts_non_binary_values(cuda):
    m = torch.zeros(3, 20, 20, device=cuda)
    m[0, 1, 1], m[2, 5, 5], m[2, 6, 6] = 0.5, 2.0, float("nan")
    assert _engine_pack(m, (20, 20), (20, 20), 3)[2] == 3
    assert _engine_pack(m, (20, 20), (10, 10), 3)[2] == 0  # resized values are thresholded, as the reference does


@pytest.mark.parametrize("n,m,px", [(7, 300, 25600), (1, 1, 1), (3, 5, 100), (40, 33, 409600), (17, 9, 257), (0, 4, 64), (6, 0, 64)])
def test_mask_iou_bit_equal_torch(cuda, n, m, px):
    g = torch.Generator().manual_seed(n * 1000 + m + px)
    a = (torch.rand(n, px, generator=g) > torch.rand(n, 1, generator=g)).float().to(cuda)
    b = (torch.rand(m, px, generator=g) > torch.rand(m, 1, generator=g)).float().to(cuda)
    if n > 2 and m > 2:
        a[0], b[0], b[1] = 0, 0, a[1]  # empty unions and an identical pair
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        inter = torch.matmul(a, b.T).clamp_(0)
        want = inter / ((a.sum(1)[:, None] + b.sum(1)[None]) - inter + 1e-7)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    got = metrics.mask_iou(a, b)
    assert got.dtype == torch.float32 and got.shape == (n, m) and got.device == a.device
    assert torch.equal(got, want)


def test_mask_iou_single_pixel_keeps_eps(cuda):
    """union 1: fl(1 + 1e-7) = 1 + 2^-23, so the IoU of two equal one-pixel masks is 1 - 2^-23 rather than 1."""
    a = torch.zeros(1, 64, device=cuda)
    a[0, 5] = 1
    got = metrics.mask_iou(a, a.clone())
    assert got.item() == np.float32(1) / (np.float32(1) + np.float32(1e-7)) and got.item() < 1.0
    assert metrics.mask_iou(a, a, eps=0.0).item() == 1.0


@pytest.mark.parametrize("tag", list(mask_val_ref.CASES))
def test_process_batch_masks_equals_fixture(cuda, tag):
    det, labels, pred, gt, overlap = mask_val_ref.case_inputs(tag)
    iouv = torch.from_numpy(mask_val_ref.IOUV).to(cuda)
    got = metrics.process_batch(torch.from_numpy(det).to(cuda), torch.from_numpy(labels).to(cuda), iouv,
                                torch.from_numpy(pred).to(cuda), torch.from_numpy(gt).to(cuda), overlap=overlap, masks=True)
    assert got.dtype == torch.bool and got.device == iouv.device
    assert np.array_equal(got.cpu().numpy(), GOLDEN[f"{tag}.correct"])


def test_process_batch_masks_rejects_non_binary(cuda):
    det, labels, pred, gt, _ = mask_val_ref.case_inputs("nonov")
    gt = gt.copy()
    gt[0, 50, 50] = 0.7
    with pytest.raises(ValueError):
        metrics.process_batch(torch.from_numpy(det).to(cuda), torch.from_numpy(labels).to(cuda), torch.from_numpy(mask_val_ref.IOUV).to(cuda),
                              torch.from_numpy(pred).to(cuda), torch.from_numpy(gt).to(cuda), overlap=False, masks=True)


# ---------------------------------------------------------------------------------------------------------------------
# the batched step
# ---------------------------------------------------------------------------------------------------------------------
def _seg_batch(dev, overlap, gt_hw, seed, im_hw=(128, 160), max_det=48, bs=6, dup=True):
    """Synthetic NMS output (rows (B,max_det,38), count), protos whose channel 0 makes each mask its (cropped) box, targets
    (nt,6) in network-input pixels and dataloader-style gt masks at gt_hw."""
    rs = np.random.RandomState(seed)
    ih, iw = im_hw
    mh, mw = ih // 4, iw // 4
    tg = []
    for b in range(bs):
        k = [0, 1, 3, 5, 8, 12][b % 6]
        xy = rs.uniform(0.25, 0.75, (k, 2))
        wh = rs.uniform(0.1, 0.4, (k, 2))
        cls = rs.randint(0, 3, k)
        for i in range(k):
            tg.append([b, cls[i], *xy[i], *wh[i]])
        if dup and k >= 2:
            tg.append(list(tg[-1]))  # a duplicated polygon: same box, same class
    tg = np.array(tg, np.float32)
    tg = tg[rs.permutation(len(tg))]  # targets in any image order
    if overlap:
        masks = np.zeros((bs,) + gt_hw, np.float32)
        for b in range(bs):
            rows = np.nonzero(tg[:, 0] == b)[0]
            masks[b] = paint_masks(gt_hw, tg[rows, 2:6], np.arange(1, len(rows) + 1))
    else:
        masks = np.stack([paint_masks(gt_hw, tg[i:i + 1, 2:6], [1.0]) * (rs.uniform(size=gt_hw) > 0.1) for i in range(len(tg))]).astype(np.float32)
    px = tg.copy()
    px[:, 2:6] *= np.array([iw, ih, iw, ih], np.float32)
    rows = rs.normal(0, 50, (bs, max_det, 38)).astype(np.float32)  # padding rows keep garbage
    count = rs.randint(0, max_det + 1, bs).astype(np.int32)
    count[0], count[1] = 0, max_det
    for b in range(bs):
        lab = px[px[:, 0] == b]
        for d in range(count[b]):
            if len(lab) and rs.uniform() < 0.8:
                c = lab[rs.randint(len(lab))]
                box = c[2:6] + rs.normal(0, 2.0, 4)
                cls = c[1] if rs.uniform() < 0.9 else rs.randint(0, 3)
            else:
                box = np.array([rs.uniform(20, iw - 20), rs.uniform(20, ih - 20), rs.uniform(8, 60), rs.uniform(8, 60)])
                cls = rs.randint(0, 3)
            rows[b, d, :4] = [box[0] - box[2] / 2, box[1] - box[3] / 2, box[0] + box[2] / 2, box[1] + box[3] / 2]
            rows[b, d, 4:6] = [rs.uniform(0.001, 1), cls]
            rows[b, d, 6:] = rs.normal(0, 0.3, 32)
            rows[b, d, 6] = 1.0
    protos = rs.normal(0, 1.0, (bs, 32, mh, mw)).astype(np.float32)
    protos[:, 0] = 8.0
    shapes = [((ih - 8 * b, iw), ) for b in range(bs)]
    t = lambda a: torch.from_numpy(a).to(dev)  # noqa: E731
    return t(rows), t(count), t(protos).half(), t(px), t(masks), im_hw, shapes


def _per_image_oracle(rows, count, protos, targets, masks, im_hw, overlap, native, iouv):
    out = []
    tg = targets.cpu().numpy()
    for b in range(rows.shape[0]):
        n = int(count[b])
        lab = tg[tg[:, 0] == b]
        corr = np.zeros((rows.shape[1], len(iouv)), bool)
        if n and len(lab):
            r = rows[b, :n]
            pm = process_mask_batch(protos[b], r[:, 6:], r[:, :4], None, im_hw, out_dtype=torch.uint8, native=native).cpu().numpy()
            gt = masks[b:b + 1] if overlap else masks[torch.from_numpy(tg[:, 0] == b).to(masks.device)]
            corr[:n] = mask_val_ref.process_batch_masks(r.cpu().numpy(), lab[:, 1:], iouv, pm, gt.cpu().numpy(), overlap)[0]
        out.append(corr)
    return np.stack(out)


@pytest.mark.parametrize("mode", ["overlap", "overlap_resize", "nonoverlap", "nonoverlap_resize", "retina", "retina_overlap_resize",
                                  "chunked"])
def test_seg_val_batch_metrics_vs_per_image_oracle(cuda, mode, monkeypatch):
    overlap = mode.startswith(("overlap", "retina_overlap", "chunked"))
    native = mode.startswith("retina")
    im_hw = (128, 160)
    gt_hw = im_hw if mode in ("overlap_resize", "nonoverlap_resize", "retina") else (32, 40)
    rows, count, protos, tg, masks, im_hw, shapes = _seg_batch(cuda, overlap, gt_hw, seed=len(mode))
    if mode == "chunked":  # two images per staged chunk
        monkeypatch.setattr(metrics, "_STAGE_BYTES", rows.shape[1] * 32 * 40 * 2)
    iouv = torch.from_numpy(mask_val_ref.IOUV).to(cuda)
    predn, cb, cm = metrics.seg_val_batch_metrics(rows, count, protos, tg, masks, im_hw, shapes, iouv, overlap, native=native, check=True)
    pn_box, cb_box = metrics.val_batch_metrics(rows, count, tg, im_hw, shapes, iouv)
    assert torch.equal(cb, cb_box) and torch.equal(predn, pn_box)
    want = _per_image_oracle(rows, count, protos, tg, masks, im_hw, overlap, native, mask_val_ref.IOUV)
    got = cm.cpu().numpy()
    assert cm.dtype == torch.bool and got.shape == want.shape
    for b in range(rows.shape[0]):
        assert not got[b, int(count[b]):].any(), "padding rows must be False"
    assert np.array_equal(got, want)
    assert got.any(), "the synthetic batch must produce true positives"


@pytest.mark.parametrize("overlap", [True, False])
@pytest.mark.parametrize("native", [False, True])
def test_seg_val_batch_metrics_without_labels(cuda, overlap, native):
    """An all-background batch (nt == 0): segment/val.py never calls process_batch, so every row stays False."""
    rows, count, protos, tg, masks, im_hw, shapes = _seg_batch(cuda, overlap, (32, 40), seed=5)
    tg = tg[:0]
    masks = torch.zeros_like(masks) if overlap else masks[:0]
    iouv = torch.from_numpy(mask_val_ref.IOUV).to(cuda)
    predn, cb, cm = metrics.seg_val_batch_metrics(rows, count, protos, tg, masks, im_hw, shapes, iouv, overlap, native=native, check=True)
    torch.cuda.synchronize()
    assert cm.shape == (rows.shape[0], rows.shape[1], 10) and not cm.any() and not cb.any()
    assert torch.equal(predn, metrics.val_batch_metrics(rows, count, tg, im_hw, shapes, iouv)[0])


def test_seg_val_batch_metrics_cuda_graph(cuda):
    """Capture fails on any host synchronisation: the batched step captures, and its replay equals the eager result."""
    rows, count, protos, tg, masks, im_hw, shapes = _seg_batch(cuda, True, (128, 160), seed=21)
    iouv = torch.from_numpy(mask_val_ref.IOUV).to(cuda)
    meta = scale_meta(im_hw, [s[0] for s in shapes]).to(cuda)
    eager = metrics.seg_val_batch_metrics(rows, count, protos, tg, masks, im_hw, meta, iouv, True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        metrics.seg_val_batch_metrics(rows, count, protos, tg, masks, im_hw, meta, iouv, True)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = metrics.seg_val_batch_metrics(rows, count, protos, tg, masks, im_hw, meta, iouv, True)
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(out, eager):
        assert torch.equal(a, b)
    assert eager[2].any()
