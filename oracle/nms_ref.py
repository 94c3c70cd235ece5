"""ORACLE (test infrastructure, never on the product path): numpy restatement of non_max_suppression.

Follows reference utils/general.py:658-767 step by step, including its dtype flow: while the rows are still
in the *input* dtype (fp16 / bf16 / fp32) every compare / multiply / subtract rounds to that dtype; the
``torch.cat(..., j.float())`` at :728/:731 promotes to fp32 and everything after (class offset, IoU) is fp32.
Low precision is emulated as "compute in fp32, round to the dtype" which is what torch's CPU and CUDA
elementwise kernels do.

Third-party pieces (source not under /root/reference):
  * ultralytics.utils.ops.xywh2xyxy (>= 8.4.118, requirements.txt:16): [cx-w/2, cy-h/2, cx+w/2, cy+h/2] in the
    input dtype -- restated, parity unpinned by any reference test;
  * torchvision.ops.nms (0.26.0 installed): greedy, stable score order, strict '>' -- restated in
    oracle/oracle_c.c and PINNED against the installed CPU op by tests/golden/make_golden.py.
Tie rule: ``argsort(descending=True)`` at :745 is taken as stable (equal scores keep candidate order), which is
what torch's CPU sort and CUDA radix sort do in practice.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build_c() -> str:
    so = os.path.join(_HERE, "liboracle.so")
    src = os.path.join(_HERE, "oracle_c.c")
    if not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-B", "liboracle.so"], stdout=subprocess.DEVNULL)
    return so


def _lib():
    global _LIB
    if _LIB is None:
        _LIB = ctypes.CDLL(build_c())
        _LIB.y5o_nms_greedy.restype = ctypes.c_int64
        _LIB.y5o_nms_greedy.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_double, ctypes.c_int64, ctypes.c_void_p]
        _LIB.y5o_box_iou.restype = None
        _LIB.y5o_box_iou.argtypes = [
            ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_float, ctypes.c_void_p,
        ]
    return _LIB


def round_to(x: np.ndarray, dtype: str) -> np.ndarray:
    """Round an fp32 array to fp32 | fp16 | bf16 (round-to-nearest-even) and return it as fp32."""
    x = np.asarray(x, np.float32)
    if dtype == "fp32":
        return x
    if dtype == "fp16":
        with np.errstate(over="ignore"):
            return x.astype(np.float16).astype(np.float32)
    if dtype == "bf16":
        shape = x.shape
        x = np.atleast_1d(x)
        u = x.view(np.uint32).astype(np.uint64)
        u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
        r = u.astype(np.uint32).view(np.float32).copy()
        r[np.isnan(x)] = np.nan
        return r.reshape(shape)
    raise ValueError(dtype)


def nms_greedy(boxes: np.ndarray, thr: float, max_keep: int | None = None) -> np.ndarray:
    """Greedy NMS over boxes (n,4) already in score-descending order; returns kept positions (int64)."""
    boxes = np.ascontiguousarray(boxes, np.float32)
    n = boxes.shape[0]
    keep = np.empty(max(n, 1), np.int64)
    k = _lib().y5o_nms_greedy(boxes.ctypes.data, n, float(thr), n if max_keep is None else max_keep, keep.ctypes.data)
    return keep[:k].copy()


def box_iou(a: np.ndarray, b: np.ndarray, eps: float = 1e-7) -> np.ndarray:
    a = np.ascontiguousarray(a, np.float32)
    b = np.ascontiguousarray(b, np.float32)
    out = np.empty((a.shape[0], b.shape[0]), np.float32)
    _lib().y5o_box_iou(a.ctypes.data, a.shape[0], b.ctypes.data, b.shape[0], np.float32(eps), out.ctypes.data)
    return out


def non_max_suppression(
    prediction: np.ndarray,
    conf_thres: float = 0.25,
    iou_thres: float = 0.45,
    classes=None,
    agnostic: bool = False,
    multi_label: bool = False,
    max_det: int = 300,
    nm: int = 0,
    dtype: str = "fp32",
    return_index: bool = False,
    labels=(),
    max_nms: int = 30000,
):
    """prediction: (B, N, 5+nc+nm) fp32 array holding values exactly representable in ``dtype``.

    ``labels`` (autolabelling, reference :706-712): per image an (m,5) array [cls, x, y, w, h]; its rows are appended to the
    image's candidates with obj = class score = 1.  The reference's ``torch.cat((x, v), 0)`` with an fp32 ``v`` promotes that
    image's rows to fp32, so everything after the first objectness test (:686) runs in fp32 for such an image.

    ``max_nms`` is the reference's hard-coded cap on the candidates that reach the greedy pass (:691); it is a keyword here
    so that the cut can be checked on small inputs.

    Returns a list of B fp32 arrays (n_i, 6+nm) = [x1,y1,x2,y2,conf,cls,(masks)]; with ``return_index`` also the
    list of int64 arrays of candidate ids ``row*nc + cls`` of the kept detections (the integer result).
    """
    assert 0 <= conf_thres <= 1 and 0 <= iou_thres <= 1
    pred = np.asarray(prediction, np.float32)
    bs, _, no = pred.shape
    nc = no - nm - 5
    mi = 5 + nc
    max_wh = 7680.0
    multi_label = multi_label and nc > 1
    thr = round_to(np.float32(conf_thres), dtype)  # python scalar is rounded to the tensor dtype before comparing
    outs, idxs = [], []
    for xi in range(bs):
        x = pred[xi]
        rows = np.nonzero(x[:, 4] > thr)[0]  # :686, :703
        empty = (np.zeros((0, 6 + nm), np.float32), np.zeros((0,), np.int64))
        x = x[rows]
        idt, ithr = dtype, thr  # dtype / threshold of this image from here on
        if labels and xi < len(labels) and len(labels[xi]):  # :706-712
            lb = np.asarray(labels[xi], np.float32)
            v = np.zeros((len(lb), no), np.float32)
            v[:, :4] = lb[:, 1:5]
            v[:, 4] = 1.0
            v[np.arange(len(lb)), lb[:, 0].astype(np.int64) + 5] = 1.0
            x = np.concatenate((x, v), 0)
            rows = np.concatenate((rows, pred.shape[1] + np.arange(len(lb))))  # appended rows get ids past the last prediction row
            idt, ithr = "fp32", np.float32(conf_thres)
        if x.shape[0] == 0:
            outs.append(empty[0]); idxs.append(empty[1]); continue
        dtype_i = idt
        scaled = round_to(x[:, 5:] * x[:, 4:5], dtype_i)  # :719  (cls AND mask columns are scaled by obj)
        half = round_to(x[:, 2:4] / np.float32(2), dtype_i)  # xywh2xyxy in the input dtype
        box = np.concatenate((round_to(x[:, 0:2] - half, dtype_i), round_to(x[:, 0:2] + half, dtype_i)), 1)
        cls_conf, mask = scaled[:, :nc], scaled[:, nc:]
        thr_i = ithr
        if multi_label:
            i, j = np.nonzero(cls_conf > thr_i)  # row-major (i, j) order, like Tensor.nonzero  :727
            conf = cls_conf[i, j]
        else:
            j = cls_conf.argmax(1)  # first maximum
            conf = cls_conf[np.arange(len(j)), j]
            i = np.nonzero(conf > thr_i)[0]  # :731
            j, conf = j[i], conf[i]
        cand = rows[i].astype(np.int64) * nc + j.astype(np.int64)
        det = np.concatenate((box[i], conf[:, None], j[:, None].astype(np.float32), mask[i]), 1).astype(np.float32)
        if classes is not None:
            sel = np.isin(det[:, 5], np.asarray(classes, np.float32))
            det, cand = det[sel], cand[sel]
        if det.shape[0] == 0:
            outs.append(empty[0]); idxs.append(empty[1]); continue
        order = np.argsort(-det[:, 4], kind="stable")[:max_nms]  # :745
        det, cand = det[order], cand[order]
        c = det[:, 5:6] * np.float32(0.0 if agnostic else max_wh)  # :748
        boxes = (det[:, :4] + c).astype(np.float32)
        keep = nms_greedy(boxes, iou_thres, max_det)  # :750-751
        outs.append(det[keep]); idxs.append(cand[keep])
    return (outs, idxs) if return_index else outs


def synth_predictions(bs: int, n_rows: int = 25200, nc: int = 80, nm: int = 0, seed: int = 2, dtype: str = "fp32",
                      img: float = 640.0) -> np.ndarray:
    """Seeded NMS input in the shape of Detect's decoded output (SURVEY.md section 8d): per image 5..40 objects,
    each spawning 5..30 near-duplicate rows, the rest low-objectness background.  Values are rounded to
    ``dtype`` and returned as fp32."""
    rs = np.random.RandomState(seed)
    no = 5 + nc + nm
    out = np.empty((bs, n_rows, no), np.float32)
    for b in range(bs):
        x = np.empty((n_rows, no), np.float32)
        x[:, 0:2] = rs.uniform(0, img, (n_rows, 2))
        x[:, 2:4] = np.exp(rs.uniform(np.log(4), np.log(img / 2), (n_rows, 2)))
        x[:, 4] = rs.uniform(0, 0.01, n_rows)
        x[:, 5 : 5 + nc] = rs.uniform(0, 1, (n_rows, nc)) ** 8
        if nm:
            x[:, 5 + nc :] = rs.normal(0, 1, (n_rows, nm))
        k = rs.randint(5, 41)
        free = rs.permutation(n_rows)
        pos = 0
        for _ in range(k):
            m = rs.randint(5, 31)
            cxy = rs.uniform(0.1 * img, 0.9 * img, 2)
            wh = np.exp(rs.uniform(np.log(16), np.log(img / 3), 2))
            cls = rs.randint(0, nc)
            r = free[pos : pos + m]
            pos += m
            m = len(r)
            if m == 0:
                break
            x[r, 0:2] = cxy * (1 + rs.uniform(-0.03, 0.03, (m, 2)))
            x[r, 2:4] = wh * (1 + rs.uniform(-0.10, 0.10, (m, 2)))
            x[r, 4] = rs.uniform(0.3, 1.0, m)
            x[r, 5 + cls] = rs.uniform(0.5, 1.0, m)
        out[b] = x
    return round_to(out, dtype)
