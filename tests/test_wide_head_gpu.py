"""GPU: Detect / Segment heads with more than 128 outputs per anchor (no = 5 + nc + nm up to 8192, nc up to 4096).

The head GEMM gives each anchor tpa = ceil(no / 128) N tiles: the packed weights and bias hold npad = 128 * tpa rows per anchor,
anchor a in rows [a npad, a npad + no).  Head-level cases (integer operands: raw exact, z within decode_bound, mask columns passed
through, guarded outputs) cover a one-column second tile, the 16-byte / 4-byte / 2-byte copy-out paths, mask columns across the
tile boundary, na 1..4, M tails and tiles straddling images; every fp16 / normal bf16 value goes through unit-vector weights at
no = 370; three levels share one z.  Whole models (yolov5n nc = 365, yolov5n-seg nc = 100, yolov5l nc = 365) are measured against
the oracle as test_model_gpu.py does and against the reference's output in tests/golden/wide_head.npz; NMS, process_batch,
ap_per_class and ConfusionMatrix run on the nc = 365 predictions against their oracles.  Shapes beyond the limits are refused."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import ap_ref, confusion_ref, model_ref, nms_ref, post_ref
from yolov5_b200 import _lib
from yolov5_b200.models.yolo import DetectionModel, SegmentationModel
from yolov5_b200.utils.general import non_max_suppression
from yolov5_b200.utils.metrics import ConfusionMatrix, ap_per_class, process_batch

from .conv_exact_ref import all_values, decode64, decode_bound
from .test_conv_exact_gpu import ANCHORS, SENTINEL, _check_level, _guarded, _guards_intact, _rint
from .test_model_gpu import _torch_lowp_reference
from .test_wide_head_cpu import wide_case

pytestmark = pytest.mark.gpu
DTYPES = [torch.float16, torch.bfloat16]
DT_IDS = ["f16", "bf16"]
HEAD_N = 128
G = os.path.join(os.path.dirname(__file__), "golden")


def _pack_wide(w, bias, na, no, block_k, dtype):
    """(na*no, cin) weight and (na*no,) bias -> [na*npad][cin_pad] / [na*npad], anchor a in rows [npad a, npad a + no)."""
    npad = -(-no // HEAD_N) * HEAD_N
    cin = w.shape[1]
    ipad = (cin + block_k - 1) // block_k * block_k
    wp = torch.zeros(na * npad, ipad, dtype=dtype)
    bp = torch.zeros(na * npad, dtype=torch.float32)
    for a in range(na):
        wp[a * npad : a * npad + no, :cin] = w[a * no : (a + 1) * no].to(dtype)
        bp[a * npad : a * npad + no] = bias[a * no : (a + 1) * no]
    return wp, bp


def _desc(dtype, in_ptr, pitch, B, ny, nx, cin, wp, bp, na, no, nc, stride, block_k, z_rows, z_row0):
    d = _lib.DetectDesc()
    d.inp, d.in_pitch = in_ptr, pitch
    d.batch, d.ny, d.nx, d.in_c = B, ny, nx, cin
    d.weight, d.bias = wp.data_ptr(), bp.data_ptr()
    d.z_rows, d.z_row0 = z_rows, z_row0
    d.na, d.no, d.nc = na, no, nc
    d.stride = stride
    for q, v in enumerate((ANCHORS[:na] * stride / 8).reshape(-1).tolist()):
        d.anchor_wh[q] = v
    d.dtype, d.block_k = _lib.dtype_code(dtype), block_k
    return d


class WideHead:
    """One Detect level packed with npad rows per anchor: input view (channels [8, 8 + cin) of pitch cin + 16), plan."""

    def __init__(self, dev, dtype, x, w, bias, na, nc, stride, block_k, z_rows=0, z_row0=0):
        B, ny, nx, cin = x.shape
        self.na, self.no, self.nc, self.stride = na, w.shape[0] // na, nc, stride
        self.B, self.ny, self.nx = B, ny, nx
        self.z_rows, self.z_row0 = z_rows or na * ny * nx, z_row0
        self.dev, self.dtype = dev, dtype
        self.x, self.w, self.bias = x, w, bias
        pitch = (cin + 7) // 8 * 8 + 16
        self.ibuf = torch.full((B, ny, nx, pitch), 3.0, dtype=dtype, device=dev)
        self.ibuf[..., 8 : 8 + cin] = x.to(dev, dtype)
        wp, bp = _pack_wide(w, bias, na, self.no, block_k, dtype)
        self.wp, self.bp = wp.to(dev), bp.to(dev)
        self.anchors = ANCHORS[:na] * stride / 8
        d = _desc(dtype, self.ibuf.data_ptr() + 8 * self.ibuf.element_size(), pitch, B, ny, nx, cin, self.wp, self.bp, na, self.no, nc,
                  stride, block_k, self.z_rows, z_row0)
        self.plan = C.c_void_p()
        _lib.check(_lib.lib().y5_detect_plan_create(C.byref(d), C.byref(self.plan)), "detect_plan_create")

    def close(self):
        _lib.lib().y5_detect_plan_destroy(self.plan)

    def run_to(self, raw_ptr, z_ptr):
        _lib.check(_lib.lib().y5_detect_plan_run_to(self.plan, C.c_void_p(raw_ptr), C.c_void_p(z_ptr), C.c_void_p(_lib.stream_ptr(self.dev))),
                   "detect")
        torch.cuda.synchronize()

    def reference(self):
        """raw (B, na, ny, nx, no) float64, z, per-element bound on z."""
        x = self.x.double().to(self.dev).reshape(-1, self.x.shape[-1])
        raw = x @ self.w.double().to(self.dev).t() + self.bias.double().to(self.dev)
        raw = raw.reshape(self.B, self.ny, self.nx, self.na, self.no).permute(0, 3, 1, 2, 4).contiguous()
        z, grid = decode64(raw, self.nc, self.stride, self.anchors)
        return raw, z, decode_bound(z, grid, self.stride, self.dtype)


def _run_single(h: WideHead, what, shift=0):
    """Outputs inside guarded buffers; `shift` half-words moves both output pointers off 16-byte alignment."""
    guard = 64 + shift
    rbuf, raw = _guarded(h.B * h.na * h.ny * h.nx * h.no, h.dev, guard)
    zbuf, z = _guarded(h.B * h.z_rows * h.no, h.dev, guard)
    h.run_to(raw.data_ptr(), z.data_ptr())
    assert _guards_intact(rbuf, guard) and _guards_intact(zbuf, guard), f"{what}: wrote outside raw / z"
    _check_level(h, raw.view(h.dtype).double().view(h.B, h.na, h.ny, h.nx, h.no), z.view(h.dtype).double(), what)


WIDE_CASES = [
    # id, B, ny, nx, cin, na, nc, nm, block_k, shift
    ("no129_one_column_tile", 2, 9, 11, 64, 3, 124, 0, 64, 0),          # odd no: half-word copy-out; M = 198, tiles straddle images
    ("no256_vector", 2, 16, 16, 96, 3, 251, 0, 64, 0),                  # two full tiles, 16-byte copy-out
    ("no256_unaligned_4byte", 2, 5, 7, 64, 3, 251, 0, 32, 2),           # no % 8 == 0 but outputs 4-byte aligned only
    ("no370_objects365", 3, 7, 9, 128, 3, 365, 0, 64, 0),               # Objects365: 3 tiles per anchor, 4-byte copy-out
    ("no205_odd_scalar", 2, 13, 10, 48, 3, 200, 0, 32, 0),              # half-word copy-out
    ("seg_nc120_nm32", 2, 8, 12, 64, 3, 120, 32, 64, 0),                # no = 157: mask columns 125..156 straddle column 128
    ("na1_no370_bk16", 3, 6, 10, 16, 1, 365, 0, 16, 0),                 # one anchor, 16-channel K blocks
    ("na4_no264_masks", 2, 11, 13, 128, 4, 227, 32, 64, 0),             # four anchors, 16-byte copy-out
    ("na2_no1029_tail", 1, 3, 5, 64, 2, 1024, 0, 64, 0),                # 9 tiles per anchor, one 15-row M tile
]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("case", WIDE_CASES, ids=[c[0] for c in WIDE_CASES])
def test_wide_head_integer(cuda, dtype, case):
    """Integer weights / inputs / bias: raw exact, z within the bound, mask columns passed through, nothing written outside."""
    name, B, ny, nx, cin, na, nc, nm, bk, shift = case
    no = 5 + nc + nm
    g = torch.Generator().manual_seed(11)
    x, w, b = _rint(g, -2, 2, B, ny, nx, cin), _rint(g, -2, 2, na * no, cin), _rint(g, -8, 8, na * no)
    h = WideHead(cuda, dtype, x, w, b.float(), na, nc, 16.0, bk)
    try:
        _run_single(h, name, shift)
    finally:
        h.close()


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_wide_head_every_value(cuda, dtype):
    """Unit-vector weights at no = 370: output column (a, o) copies input channel a*no + o, so raw reproduces every fp16 (normal
    bf16) value bit for bit in every column of all three tiles of an anchor, and z is its float64 decode within the bound."""
    na, nc = 3, 365
    no = 5 + nc
    cin = na * no
    B, ny, nx = 2, 5, 6
    vals = all_values(dtype)
    assert vals.numel() <= B * ny * nx * cin
    x = torch.zeros(B * ny * nx * cin, dtype=dtype)
    x[: vals.numel()] = vals
    h = WideHead(cuda, dtype, x.view(B, ny, nx, cin), torch.eye(cin), torch.zeros(cin), na, nc, 8.0, 64)
    try:
        _run_single(h, "every value no 370")
    finally:
        h.close()


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_wide_three_levels_one_z(cuda, dtype):
    """Three no = 370 levels into one z buffer with z_rows / z_row0 as engine.lower_detect sets them: after each level its rows
    are right, the rows of the levels still to run keep their sentinels, and nothing around the buffers is written."""
    B, na, nc = 2, 3, 365
    no = 5 + nc
    levels = [(12, 16, 64, 8.0, 64), (6, 8, 128, 16.0, 32), (3, 4, 256, 32.0, 16)]  # ny, nx, cin, stride, block_k
    z_rows = sum(na * ny * nx for ny, nx, *_ in levels)
    g = torch.Generator().manual_seed(13)
    heads, row0 = [], 0
    try:
        for ny, nx, cin, stride, bk in levels:
            x, w, b = _rint(g, -2, 2, B, ny, nx, cin), _rint(g, -2, 2, na * no, cin), _rint(g, -8, 8, na * no)
            heads.append(WideHead(cuda, dtype, x, w, b.float(), na, nc, stride, bk, z_rows=z_rows, z_row0=row0))
            row0 += na * ny * nx
        zbuf, z = _guarded(B * z_rows * no, cuda)
        z3 = z.view(B, z_rows, no)
        for i, h in enumerate(heads):
            rbuf, raw = _guarded(B * na * h.ny * h.nx * no, cuda)
            h.run_to(raw.data_ptr(), z.data_ptr())
            assert _guards_intact(rbuf) and _guards_intact(zbuf), f"level {i}: wrote outside raw / z"
            lo, hi = h.z_row0, h.z_row0 + na * h.ny * h.nx
            assert bool((z3[:, hi:] == SENTINEL).all()), f"level {i} wrote rows of a later level"
            _check_level(h, raw.view(dtype).double().view(B, na, h.ny, h.nx, no), z3[:, lo:hi].view(dtype).double(), f"level {i}")
    finally:
        for h in heads:
            h.close()


# ------------------------------------------------------------------------------------------------------------------------------
# whole models
def _check_wide_model(name, cfg, sd, x, dtype, dev):
    """test_model_gpu._check_model's criterion for a model built with cfg["nc"]: every output within 1e-3 of the fp32 oracle's
    scale plus 1.5 times the error of the reference's expressions evaluated by torch in the same dtype."""
    with torch.no_grad():
        ref = model_ref.forward(cfg, sd, x.to(dtype).float(), fused=True)
    seg = name.endswith("-seg")
    m = (SegmentationModel if seg else DetectionModel)(name, nc=cfg["nc"])
    m.load_state_dict(sd)
    m = m.to(dev, dtype).eval()
    out = m(x.to(dev, dtype))
    low = _torch_lowp_reference(cfg, sd, x, dtype, dev)
    pairs = [("z", out[0], ref[0], low[0])]
    raws, rraws, lraws = (out[2], ref[2], low[2]) if seg else (out[1], ref[1], low[1])
    pairs += [(f"raw{l}", a, b, c) for l, (a, b, c) in enumerate(zip(raws, rraws, lraws))]
    if seg:
        pairs.append(("proto", out[1], ref[1], low[1]))
    for tag, got, r, lo in pairs:
        got, lo = got.float().cpu(), lo.float().cpu()
        assert got.shape == r.shape, (tag, got.shape, r.shape)
        scale = float(r.abs().max())
        e_eng, e_low = float((got - r).abs().max()), float((lo - r).abs().max())
        assert e_eng <= 1e-3 * scale + 1.5 * e_low, (name, tag, e_eng / scale, e_low / scale)
    return out


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("name", ["yolov5n", "yolov5n-seg"])
def test_wide_model_vs_oracle_and_golden(cuda, name, dtype):
    """yolov5n at nc = 365 (no = 370) and yolov5n-seg at nc = 100 (no = 137): against the oracle and the reference's z."""
    cfg, sd, x = wide_case(name)
    out = _check_wide_model(name, cfg, sd, x, dtype, cuda)
    g = np.load(os.path.join(G, "wide_head.npz"))
    z = out[0].float().cpu().numpy()
    assert z.shape == tuple(g[f"{name}.z_shape"])
    gz = g[f"{name}.z_sample"]
    assert np.abs(z[:, :: int(g["sample"])] - gz).max() <= 2e-2 * np.abs(gz).max()


def test_wide_model_yolov5l_640_bf16(cuda):
    from yolov5_b200.cfg import model_cfg

    cfg = dict(model_cfg("yolov5l"), nc=365)
    sd = model_ref.synth_state_dict(cfg, seed=5, head_bias="hot")
    x = torch.from_numpy(np.random.RandomState(105).uniform(0, 1, (2, 3, 640, 640)).astype(np.float32))
    _check_wide_model("yolov5l", cfg, sd, x, torch.bfloat16, cuda)


def test_wide_model_nms_and_val_metrics(cuda):
    """nc = 365 predictions of the engine (fp16) through non_max_suppression (bit-exact with oracle/nms_ref, indices included, as
    test_nms_gpu.py compares), then process_batch, ap_per_class and ConfusionMatrix against their oracles, with labels spread
    over all 365 classes."""
    cfg, sd, x = wide_case("yolov5n")
    nc = cfg["nc"]
    m = DetectionModel("yolov5n", nc=nc)
    m.load_state_dict(sd)
    m = m.to(cuda, torch.float16).eval()
    xb = torch.cat([x, x.flip(2)]).to(cuda, torch.float16)
    z = m(xb)[0]
    zn = z.float().cpu().numpy()
    for kw in (dict(conf_thres=0.25, iou_thres=0.45, max_det=300), dict(conf_thres=0.001, iou_thres=0.6, max_det=300)):
        dets, idx = non_max_suppression(z, return_indices=True, **kw)
        ref, ridx = nms_ref.non_max_suppression(zn, dtype="fp16", return_index=True, **kw)
        for b in range(z.shape[0]):
            assert np.array_equal(idx[b].cpu().numpy(), ridx[b]), (kw, b, "indices")
            assert np.array_equal(dets[b].cpu().numpy(), ref[b]), (kw, b)
            assert ref[b].shape[0] > 10 and ref[b][:, 5].max() > 127, (kw, b, ref[b].shape)
    # labels: jittered copies of some detections, classes over [0, 365)
    rs = np.random.RandomState(3)
    iouv = np.linspace(0.5, 0.95, 10).astype(np.float32)
    cm = ConfusionMatrix(nc=nc)
    cm_ref = np.zeros((nc + 1, nc + 1))
    stats = []
    for b in range(z.shape[0]):
        det = ref[b]
        pick = rs.choice(det.shape[0], det.shape[0] // 2, replace=False)
        boxes = det[pick, :4] + rs.normal(0, 2, (len(pick), 4)).astype(np.float32)
        cls = np.where(rs.uniform(size=len(pick)) < 0.7, det[pick, 5], rs.randint(0, nc, len(pick))).astype(np.float32)
        lab = np.concatenate((cls[:, None], boxes), 1).astype(np.float32)
        correct = process_batch(torch.from_numpy(det).to(cuda), torch.from_numpy(lab).to(cuda), torch.from_numpy(iouv).to(cuda))
        want = post_ref.process_batch(det, lab, iouv)
        assert np.array_equal(correct.cpu().numpy(), want), b
        stats.append((want, det[:, 4], det[:, 5], lab[:, 0]))
        cm.process_batch(torch.from_numpy(det).to(cuda), torch.from_numpy(lab).to(cuda))
        confusion_ref.process_batch(cm_ref, det, lab, nc)
    assert np.array_equal(cm.matrix, cm_ref)
    tp, conf, pc, tc = (np.concatenate([s[i] for s in stats]) for i in range(4))
    got = ap_per_class(tp, conf, pc, tc)
    want, _, gap = ap_ref.ap_per_class(tp, conf, pc, tc, return_index=True)
    index_free = gap < 1e-12 and gap != 0.0  # the two largest smoothed mean-F1 values tie: either max-F1 index is right
    for k, a, w in zip(("tp", "fp", "p", "r", "f1", "ap", "classes"), got, want):
        if index_free and k not in ("ap", "classes"):
            continue
        assert a.shape == w.shape and a.dtype == w.dtype and np.array_equal(a, w, equal_nan=True), k


# ------------------------------------------------------------------------------------------------------------------------------
# limits
@pytest.mark.parametrize("nc,nm", [(4096, 4092), (4097, 0)], ids=["no8193", "nc4097"])
def test_plan_refuses_beyond_the_limit(cuda, nc, nm):
    """no <= 8192 and nc <= 4096: the plan refuses beyond with Y5_E_UNSUPPORTED (-2) and a message naming the limits."""
    na, no, cin, bk = 1, 5 + nc + nm, 16, 16
    wp, bp = torch.zeros(na * 8320, bk, dtype=torch.float16, device=cuda), torch.zeros(na * 8320, device=cuda)
    x = torch.zeros(1, 2, 2, cin, dtype=torch.float16, device=cuda)
    d = _desc(torch.float16, x.data_ptr(), cin, 1, 2, 2, cin, wp, bp, na, no, nc, 8.0, bk, na * 4, 0)
    plan = C.c_void_p()
    code = _lib.lib().y5_detect_plan_create(C.byref(d), C.byref(plan))
    assert code == -2 and not plan.value
    msg = _lib.lib().y5_last_error().decode()
    assert "no <= 8192" in msg and "nc <= 4096" in msg, msg


def test_engine_refuses_beyond_the_limit(cuda):
    m = DetectionModel("yolov5n", nc=4097).to(cuda, torch.float16).eval()
    with pytest.raises(NotImplementedError, match=r"no <= 8192 .* nc <= 4096"):
        m(torch.zeros(1, 3, 64, 64, dtype=torch.float16, device=cuda))
