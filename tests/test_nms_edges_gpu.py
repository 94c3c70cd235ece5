"""GPU: y5_nms_batched where it can go wrong, bit for bit against the oracle (rows and candidate ids) and, for the cases in
tests/golden/nms_edges.npz, against the reference-generated rows:

- the max_nms cut in single- and multi-label mode, at the real 30000 on 1280-pixel inputs and at 1..1000 on small inputs,
  with ties straddling the cut across segments and warps, and fp32 scores that share their top 16 bits;
- one launch holding images over, under, exactly at and one above the cut, and an empty one;
- greedy suppression chains across the 64-candidate chunks, and max_det from 1 to 4096;
- conf_thres / iou_thres edges: scores at and one or two ulps around the dtype-rounded threshold, IoUs at and around the
  fp32 threshold the binding derives;
- class counts 1..4096 with `classes=` filters, agnostic mode and mask columns;
- NaN / inf inputs; repeated calls on a reused workspace and on a side stream.
"""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from oracle import nms_ref
from yolov5_b200 import _lib
from yolov5_b200.utils.general import MAX_NMS, MAX_WH, _iou_threshold_f32, non_max_suppression

from .test_nms_edges_cpu import edge_pred

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore:invalid value:RuntimeWarning")]
G = os.path.join(os.path.dirname(__file__), "golden")
TDT = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}
DTYPES = ["fp32", "fp16", "bf16"]


def run_nms(pred, dtype, dev, max_nms=MAX_NMS, conf_thres=0.25, iou_thres=0.45, classes=None, agnostic=False,
            multi_label=False, max_det=300, nm=0):
    """One y5_nms_batched launch with NmsParams filled here, so max_nms can differ from the reference's 30000.  `pred` is a
    numpy array (copied to the device in `dtype`) or a device tensor.  Returns per-image numpy rows and candidate ids."""
    t = pred if isinstance(pred, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(pred)).to(dev, TDT[dtype])
    bs, n, no = t.shape
    lib = _lib.lib()
    p = _lib.NmsParams()
    p.batch, p.n_rows, p.no, p.nc, p.nm = bs, n, no, no - 5 - nm, nm
    p.dtype = _lib.dtype_code(t.dtype)
    p.conf_thres, p.iou_thres = float(conf_thres), _iou_threshold_f32(iou_thres)
    p.multi_label, p.agnostic = int(multi_label), int(agnostic)
    p.max_det, p.max_nms, p.max_wh = max_det, max_nms, MAX_WH
    cls_t = torch.as_tensor(list(classes), dtype=torch.int32, device=dev) if classes is not None else None
    p.classes, p.n_classes = (cls_t.data_ptr(), cls_t.numel()) if cls_t is not None else (None, 0)
    need = lib.y5_nms_workspace_bytes(C.byref(p))
    assert need > 0
    ws = torch.empty(need + 256, dtype=torch.uint8, device=dev)
    rows = torch.empty(bs, max_det, 6 + nm, dtype=torch.float32, device=dev)
    idx = torch.empty(bs, max_det, dtype=torch.int64, device=dev)
    count = torch.empty(bs, dtype=torch.int32, device=dev)
    _lib.check(lib.y5_nms_batched(C.byref(p), t.data_ptr(), rows.data_ptr(), idx.data_ptr(), count.data_ptr(),
                                  (ws.data_ptr() + 255) & ~255, need, C.c_void_p(_lib.stream_ptr(dev))), "nms_batched")
    cnt = count.tolist()
    return [rows[b, :c].cpu().numpy() for b, c in enumerate(cnt)], [idx[b, :c].cpu().numpy() for b, c in enumerate(cnt)]


def assert_oracle(pred, dtype, got, max_nms=MAX_NMS, what="", **kw):
    """Rows and candidate ids of every image equal the oracle's, bit for bit (NaN where the oracle has NaN)."""
    ref, ridx = nms_ref.non_max_suppression(pred, dtype=dtype, return_index=True, max_nms=max_nms, **kw)
    rows, idx = got
    assert len(rows) == len(ref)
    for b in range(len(ref)):
        assert np.array_equal(idx[b], ridx[b]), (what, b, "ids", len(idx[b]), len(ridx[b]))
        assert rows[b].shape == ref[b].shape and np.array_equal(rows[b], ref[b], equal_nan=True), (what, b, "rows")
    return ref


def candidates(pred, dtype, conf_thres, multi_label, nc):
    """Per image, the number of candidates the reference forms before its max_nms cut."""
    thr = nms_ref.round_to(np.float32(conf_thres), dtype)
    out = []
    for x in pred:
        x = x[x[:, 4] > thr]
        with np.errstate(invalid="ignore"):
            conf = nms_ref.round_to(x[:, 5 : 5 + nc] * x[:, 4:5], dtype)
        out.append(int((conf > thr).sum()) if multi_label and nc > 1 else int((conf.max(1, initial=-np.inf) > thr).sum()))
    return out


def quantized(bs, n, nc, seed, dtype, levels=16, nm=0, img=640.0):
    """synth_predictions with objectness >= 0.5 and class scores on a 1/levels grid: few distinct scores, so equal-score runs
    straddle any cut and span many 32-row segments."""
    p = nms_ref.synth_predictions(bs, n, nc, nm, seed, dtype, img=img)
    p[..., 4] = np.maximum(p[..., 4], 0.5)
    p[..., 5 : 5 + nc] = np.round(p[..., 5 : 5 + nc] ** 0.25 * levels) / levels
    return nms_ref.round_to(p, dtype)


def _nudge(v, dtype, k):
    """v (representable in dtype) moved by k representable steps."""
    v = np.float32(v)
    for _ in range(abs(k)):
        if dtype == "fp32":
            v = np.nextafter(v, np.float32(np.inf if k > 0 else -np.inf))
        elif dtype == "fp16":
            v = np.float32(np.nextafter(np.float16(v), np.float16(np.inf if k > 0 else -np.inf)))
        else:
            u = int(np.array([v], np.float32).view(np.uint32)[0])
            if v == 0:
                u = 0x00010000 if k > 0 else 0x80010000
            else:
                u += (0x10000 if (k > 0) == (v > 0) else -0x10000)
            v = np.array([u], np.uint32).view(np.float32)[0]
    return v


# ---------------------------------------------------------------------------------------------------------- the fixture

def test_edge_fixture_bit_exact(cuda):
    """Every case of nms_edges.npz through the public entry point: bf16 val / segment-val with the cut, 1280-pixel
    single-label with the cut, NaN / inf / degenerate inputs.  Rows equal the reference-generated ones, ids the oracle's."""
    g = np.load(os.path.join(G, "nms_edges.npz"))
    for c in json.loads(str(g["meta"])):
        pred = edge_pred(g, c)
        t = torch.from_numpy(pred).to(cuda, TDT[c["dtype"]])
        out, idx = non_max_suppression(t, return_indices=True, **c["kw"])
        got = ([o.cpu().numpy() for o in out], [i.cpu().numpy() for i in idx])
        assert_oracle(pred, c["dtype"], got, what=c["tag"], **c["kw"])
        for b in range(c["bs"]):
            ref = g[f"{c['tag']}.{b}"]
            assert got[0][b].shape == ref.shape and np.array_equal(got[0][b], ref, equal_nan=True), (c["tag"], b)


@pytest.mark.parametrize("multi_label", [False, True])
def test_nan_class_score_drops_the_row(cuda, multi_label):
    """torch.max propagates NaN, so a row with any NaN class score has a NaN best score and is no candidate in single-label
    mode, wherever the NaN sits among the row's classes; in multi-label mode only the NaN class goes."""
    rs = np.random.RandomState(5)
    for nc in (3, 8, 9, 20, 80):
        n = 8 * nc + 3
        x = np.zeros((1, n, 5 + nc), np.float32)
        x[0, :, 0] = 20.0 + 40.0 * (np.arange(n) % 32)
        x[0, :, 1] = 20.0 + 40.0 * (np.arange(n) // 32)
        x[0, :, 2:4] = 16
        x[0, :, 4] = rs.uniform(0.6, 1.0, n)
        x[0, :, 5:] = rs.uniform(0.5, 1.0, (n, nc))
        for r in range(n - 3):
            x[0, r, 5 + r % nc] = np.nan  # row r: NaN at class r % nc, including the row's would-be best
        x[0, n - 3, 5 + nc - 1] = np.nan
        for dtype in DTYPES:
            p = nms_ref.round_to(x, dtype)
            got = run_nms(p, dtype, cuda, multi_label=multi_label, max_det=4096)
            ref = assert_oracle(p, dtype, got, what=(nc, dtype), multi_label=multi_label, max_det=4096)
            if not multi_label:
                assert len(ref[0]) == 2, (nc, dtype)  # only the two rows without a NaN


# --------------------------------------------------------------------------------------------------------------- the cut

@pytest.mark.parametrize("dtype", DTYPES)
def test_cut_at_1280_multi_label(cuda, dtype):
    """100800 rows, multi-label, quantized scores: several hundred thousand candidates, a tie run across the 30000 cut."""
    p = quantized(1, 100800, 16, 50 + DTYPES.index(dtype), dtype, img=1280.0)
    kw = dict(conf_thres=0.001, iou_thres=0.6, multi_label=True, max_det=300)
    assert candidates(p, dtype, 0.001, True, 16)[0] > 2 * MAX_NMS
    assert_oracle(p, dtype, run_nms(p, dtype, cuda, **kw), what=dtype, **kw)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("multi_label", [False, True])
def test_cut_small_max_nms(cuda, dtype, multi_label):
    """max_nms in {1, 2, 63, 64, 1000} on 2 x 1237 rows with 1/8-grid scores: the radix select, its tie count and the
    ordered compaction decide which equal-score candidates make the cut."""
    p = quantized(2, 1237, 7, 60, dtype, levels=8)
    kw = dict(conf_thres=0.1, iou_thres=0.5, multi_label=multi_label, max_det=4096)
    assert min(candidates(p, dtype, 0.1, multi_label, 7)) > 1000
    for max_nms in (1, 2, 63, 64, 1000):
        assert_oracle(p, dtype, run_nms(p, dtype, cuda, max_nms=max_nms, **kw), max_nms=max_nms, what=max_nms, **kw)


def test_cut_scores_share_top_16_bits(cuda):
    """fp32 scores that all fall in one level-1 histogram bin (equal top 16 bits), with repeated low halves: the level-2
    histogram alone decides the threshold and how many == T candidates survive."""
    rs = np.random.RandomState(7)
    n = 40000
    p = np.zeros((1, n, 6), np.float32)
    p[0, :, 0] = rs.uniform(0, 1280, n)
    p[0, :, 1] = rs.uniform(0, 1280, n)
    p[0, :, 2:4] = rs.uniform(2, 40, (n, 2))
    p[0, :, 4] = 1.0
    lo = rs.randint(0, 3000, n).astype(np.uint32)
    p[0, :, 5] = ((np.uint32(0x3F40) << 16) | lo).view(np.float32)
    kw = dict(conf_thres=0.25, iou_thres=0.45, max_det=1000)
    assert_oracle(p, "fp32", run_nms(p, "fp32", cuda, **kw), what="30000", **kw)
    for max_nms in (1, 64, 1000, 29999):
        assert_oracle(p, "fp32", run_nms(p, "fp32", cuda, max_nms=max_nms, **kw), max_nms=max_nms, what=max_nms, **kw)


@pytest.mark.parametrize("max_nms", [64, MAX_NMS])
def test_mixed_batch_one_launch(cuda, max_nms):
    """Images over the cut, under it, at exactly max_nms candidates, at max_nms + 1, and empty, in one launch."""
    rs = np.random.RandomState(8)
    n = max_nms + max_nms // 6 + 37
    want = [n - 5, max_nms // 2, max_nms, max_nms + 1, 0]
    p = np.zeros((len(want), n, 8), np.float32)
    for b, k in enumerate(want):
        p[b, :, 0:2] = rs.uniform(0, 1280, (n, 2))
        p[b, :, 2:4] = rs.uniform(4, 64, (n, 2))
        rows = rs.permutation(n)[:k]
        p[b, rows, 4] = np.round(rs.uniform(0.6, 1.0, k) * 32) / 32
        p[b, rows, 5:] = np.round(rs.uniform(0.6, 1.0, (k, 3)) * 32) / 32
    p = nms_ref.round_to(p, "fp16")
    kw = dict(conf_thres=0.25, iou_thres=0.45, max_det=300)
    assert candidates(p, "fp16", 0.25, False, 3) == want
    assert_oracle(p, "fp16", run_nms(p, "fp16", cuda, max_nms=max_nms, **kw), max_nms=max_nms, **kw)


# ------------------------------------------------------------------------------------------------------------ the greedy

def chain_pred(n, head, dtype, nc=1):
    """`head` isolated boxes, then a chain of n - head boxes along x where box k overlaps box k-1 at IoU 12/28 and box k-2
    at 4/36, lines of 200; scores fall with the row, so score order is row order and survivors alternate along the chain."""
    p = np.zeros((1, n, 5 + nc), np.float32)
    k = np.arange(n)
    p[0, :, 0] = 20 + 8 * (k % 200)
    p[0, :, 1] = 20 + 40 * (k // 200)
    p[0, :head, 1] = 20000 + 40 * np.arange(head)  # far away from everything
    p[0, :, 2] = 20
    p[0, :, 3] = 10
    p[0, :, 4] = 1.0
    p[0, :, 5] = np.linspace(1.0, 0.3, n)
    return nms_ref.round_to(p, dtype)


@pytest.mark.parametrize("dtype", ["fp32", "fp16"])
def test_greedy_chains_across_chunks(cuda, dtype):
    """Chains starting at sorted positions 0, 63, 64, 65, 127 and 128, so chunk boundaries fall inside them and the kept
    list grows past its 16-way split."""
    kw = dict(conf_thres=0.25, iou_thres=0.3, max_det=4096)
    for head in (0, 63, 64, 65, 127, 128):
        p = chain_pred(head + 330, head, dtype)
        ref = assert_oracle(p, dtype, run_nms(p, dtype, cuda, **kw), what=head, **kw)
        assert head + 150 < len(ref[0]) < head + 200  # about every other chain box survives


@pytest.mark.parametrize("dtype", ["fp32", "fp16"])
def test_greedy_max_det(cuda, dtype):
    """More survivors than max_det for max_det in {1, 63, 64, 65, 300, 4096}: the early exit mid-chunk and the output."""
    p = chain_pred(9000, 100, dtype)
    for max_det in (1, 63, 64, 65, 300, 4096):
        kw = dict(conf_thres=0.25, iou_thres=0.3, max_det=max_det)
        ref = assert_oracle(p, dtype, run_nms(p, dtype, cuda, **kw), what=max_det, **kw)
        assert len(ref[0]) == max_det


# ------------------------------------------------------------------------------------------------------ threshold edges

@pytest.mark.parametrize("dtype", DTYPES)
def test_conf_threshold_edges(cuda, dtype):
    """Objectness and obj * cls at, one and two steps above and below the dtype-rounded conf_thres, and products that round
    onto it, for conf_thres 0, 0.001, 0.25, 0.45 and 1."""
    for ct in (0.0, 0.001, 0.25, 0.45, 1.0):
        thr = nms_ref.round_to(np.float32(ct), dtype)
        edge = [_nudge(thr, dtype, k) for k in (-2, -1, 0, 1, 2)]
        ones = [_nudge(1.0, dtype, k) for k in (-1, 0, 1)]
        pairs = [(o, c) for o in edge for c in ones] + [(o, c) for o in ones for c in edge] + [(o, c) for o in edge for c in edge]
        n = len(pairs)
        p = np.zeros((1, n, 8), np.float32)
        p[0, :, 0] = 20.0 + 40.0 * (np.arange(n) % 32)
        p[0, :, 1] = 20.0 + 40.0 * (np.arange(n) // 32)
        p[0, :, 2:4] = 16
        p[0, :, 4] = [o for o, _ in pairs]
        p[0, np.arange(n), 5 + np.arange(n) % 3] = [c for _, c in pairs]
        p = nms_ref.round_to(p, dtype)
        for multi_label in (False, True):
            kw = dict(conf_thres=ct, iou_thres=0.45, multi_label=multi_label, max_det=4096)
            assert_oracle(p, dtype, run_nms(p, dtype, cuda, **kw), what=(ct, multi_label), **kw)


def _iou_pairs(target):
    """(k, c) with fl32(k / c) == target: box [1, k+1] x [0, 1] against [0, c] x [0, 1] has inter k and union c."""
    c = np.arange(4, 1 << 22, dtype=np.int64)  # near 9/20, 3/5 or 7/10 the k / c that round onto one ulp need large c
    for dk in (0, 1, -1):
        k = np.round(np.float64(target) * c).astype(np.int64) + dk
        ok = (k >= 1) & (k + 1 < c) & ((k.astype(np.float32) / c.astype(np.float32)) == np.float32(target))
        if ok.any():
            i = int(np.nonzero(ok)[0][0])
            return int(k[i]), int(c[i])
    raise AssertionError(target)


@pytest.mark.parametrize("iou_thres", [0.0, 0.45, 0.6, 0.7, 1.0])
def test_iou_threshold_edges(cuda, iou_thres):
    """Box pairs whose fp32 IoU is exactly the adjusted threshold, one and two ulps either side: the higher-scored box
    suppresses the other only above it (torchvision's CPU kernel compares the fp32 IoU against the threshold as a double).
    At 0 any overlap suppresses, at 1 nothing does, not even an identical box."""
    tf = np.float32(_iou_threshold_f32(iou_thres))
    targets = [_nudge(tf, "fp32", k) for k in (-2, -1, 0, 1, 2)] if 0 < iou_thres < 1 else []
    pairs = [_iou_pairs(t) for t in targets] + [(1, 50000), (5, 7), (10, 12)]  # IoU 2e-5, 5/7, 10/12
    n = 2 * len(pairs) + 2
    p = np.zeros((1, n, 6), np.float32)
    for q, (k, c) in enumerate(pairs):
        y = 0.5 + 10.0 * q
        p[0, 2 * q] = [c / 2, y, c, 1, 1.0, 0.9]                  # [0, c] x [y - 0.5, y + 0.5]
        p[0, 2 * q + 1] = [1 + k / 2, y, k, 1, 1.0, 0.8]          # [1, k + 1]
    p[0, n - 2] = [50, 5000, 20, 20, 1.0, 0.7]
    p[0, n - 1] = [50, 5000, 20, 20, 1.0, 0.6]                    # identical: IoU exactly 1
    kw = dict(conf_thres=0.25, iou_thres=iou_thres, max_det=300)
    got = run_nms(p, "fp32", cuda, **kw)
    ref = assert_oracle(p, "fp32", got, what=iou_thres, **kw)
    kept = set(got[1][0].tolist())
    for q, t in enumerate(targets):
        assert ((2 * q + 1) in kept) == (float(t) <= iou_thres), (q, float(t))
    assert ((2 * len(targets) + 1) in kept) == (iou_thres > 0)  # the 2e-5 overlap
    assert ((n - 1) in kept) == (iou_thres == 1.0)                # the identical box
    if iou_thres == 1.0:
        assert len(ref[0]) == n


# ------------------------------------------------------------------------------------------------ classes, masks, nc

@pytest.mark.parametrize("nc", [1, 3, 7, 33, 365, 4096])
def test_class_counts_filters_agnostic(cuda, nc):
    """nc from 1 to 4096 on row counts that are not multiples of 32, single- and multi-label, with `classes=` holding
    duplicates and out-of-range ids, agnostic mode, and the cut."""
    n = 517 if nc >= 365 else 1999
    p = quantized(2, n, nc, 70 + nc, "fp16", levels=8)
    classes = sorted({0, nc - 1, nc // 2}) + [0, nc - 1, -1, nc, nc + 7]
    for multi_label in (False, True):
        for cls in (None, classes):
            for agnostic in (False, True):
                for max_nms in (MAX_NMS, 64):
                    kw = dict(conf_thres=0.05, iou_thres=0.5, multi_label=multi_label, classes=cls, agnostic=agnostic, max_det=300)
                    assert_oracle(p, "fp16", run_nms(p, "fp16", cuda, max_nms=max_nms, **kw), max_nms=max_nms,
                                  what=(multi_label, cls is not None, agnostic, max_nms), **kw)


@pytest.mark.parametrize("dtype", ["fp16", "bf16"])
def test_mask_columns_with_the_cut(cuda, dtype):
    """nm = 32 in multi-label mode with the cut at 30000 (segment/val.py at 640) and at 1000: mask columns follow their
    candidates through the select, compaction and sort."""
    p = quantized(2, 25200, 80, 80, dtype, nm=32)
    kw = dict(conf_thres=0.001, iou_thres=0.6, multi_label=True, max_det=300, nm=32)
    assert min(candidates(p, dtype, 0.001, True, 80)) > MAX_NMS
    for max_nms in (MAX_NMS, 1000):
        assert_oracle(p, dtype, run_nms(p, dtype, cuda, max_nms=max_nms, **kw), max_nms=max_nms, what=max_nms, **kw)


# --------------------------------------------------------------------------------------------------------- repeat calls

def test_repeat_calls_reused_workspace_and_stream(cuda):
    """The same result on a second call, after a larger call of another shape has left its data in the cached workspace,
    and on a non-default stream."""
    small = quantized(2, 3001, 80, 90, "fp16")
    big = quantized(3, 25200, 80, 91, "fp16")
    kw = dict(conf_thres=0.001, iou_thres=0.6, multi_label=True, max_det=300)
    ts, tb = (torch.from_numpy(x).to(cuda, torch.float16) for x in (small, big))

    def public(t):
        out, idx = non_max_suppression(t, return_indices=True, **kw)
        return [o.cpu().numpy() for o in out], [i.cpu().numpy() for i in idx]

    first = public(ts)
    assert_oracle(small, "fp16", first, what="first", **kw)
    assert_oracle(big, "fp16", public(tb), what="big", **kw)
    for what, got in (("again", public(ts)), ("after big", public(ts))):
        for b in range(2):
            assert np.array_equal(got[1][b], first[1][b]) and np.array_equal(got[0][b], first[0][b]), (what, b)
    side = torch.cuda.Stream(cuda)
    side.wait_stream(torch.cuda.current_stream(cuda))
    with torch.cuda.stream(side):
        got_b = public(tb)
        got_s = public(ts)
    torch.cuda.current_stream(cuda).wait_stream(side)
    assert_oracle(big, "fp16", got_b, what="side big", **kw)
    for b in range(2):
        assert np.array_equal(got_s[1][b], first[1][b]) and np.array_equal(got_s[0][b], first[0][b]), ("side", b)
