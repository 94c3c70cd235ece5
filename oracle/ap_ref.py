"""numpy restatement of ap_per_class (reference utils/metrics.py:25-126) with every order the result depends on written out:

- rows are ordered by np.argsort(-conf, kind="stable") (ties keep input order, NaN last).  The reference calls the default,
  unstable argsort, whose tie order depends on the host; `stable=False` replays that call;
- np.interp as `interp` (the rule of numpy's compiled interp, searchsorted for its binary search);
- np.trapezoid's sum as `pairwise_sum` (numpy's pairwise summation: 8 running accumulators for 8..128 terms);
- f1.mean(0) as `mean0` (the classes summed one after the other in class order, then divided by nc).

ultralytics' `smooth` (a 101-tap box filter through np.convolve) is kept as numpy computes it: its BLAS summation order is
not reproducible, so only its argmax is compared, never the smoothed values.
"""
from __future__ import annotations

import numpy as np

PX = np.linspace(0, 1, 1000)  # ap_per_class's p / r / f1 curve grid
X101 = np.linspace(0, 1, 101)  # compute_ap's 101-point COCO grid


def interp(x, xp, fp, left=None, right=None):
    """np.interp(x, xp, fp, left, right) for ascending xp: j = the largest index with xp[j] <= x; fp[j] where x == xp[j] or j
    is the last index; else s*(x - xp[j]) + fp[j], s = (fp[j+1] - fp[j]) / (xp[j+1] - xp[j]), and when that is NaN
    s*(x - xp[j+1]) + fp[j+1], and when that is NaN too while fp[j] == fp[j+1], fp[j]."""
    x, xp, fp = (np.asarray(a, np.float64) for a in (x, xp, fp))
    n = xp.shape[0]
    lval = fp[0] if left is None else np.float64(left)
    rval = fp[-1] if right is None else np.float64(right)
    j = np.searchsorted(xp, x, side="right") - 1
    jc = np.clip(j, 0, max(n - 2, 0))
    with np.errstate(all="ignore"):
        if n > 1:
            s = (fp[jc + 1] - fp[jc]) / (xp[jc + 1] - xp[jc])
            y = s * (x - xp[jc]) + fp[jc]
            y2 = s * (x - xp[jc + 1]) + fp[jc + 1]
            nan = np.isnan(y)
            y = np.where(nan, y2, y)
            y = np.where(nan & np.isnan(y2) & (fp[jc] == fp[jc + 1]), fp[jc], y)
        else:
            y = np.full(x.shape, fp[0])
    jx = np.clip(j, 0, n - 1)
    y = np.where((xp[jx] == x) | (j == n - 1), fp[jx], y)
    y = np.where(x < xp[0], lval, y)
    return np.where(x > xp[-1], rval, y)


def pairwise_sum(t):
    """np.add.reduce of a contiguous float64 vector of at most 128 terms (numpy's pairwise_sum)."""
    t = np.asarray(t, np.float64)
    n = t.shape[0]
    assert n <= 128
    if n < 8:
        res = np.float64(0.0)
        for v in t:
            res = res + v
        return res
    r = t[:8].copy()
    m = n - n % 8
    for i in range(8, m, 8):
        r = r + t[i:i + 8]
    res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
    for i in range(m, n):
        res = res + t[i]
    return res


def trapezoid(y, x):
    """np.trapezoid(y, x) of a 1-D curve: sum of d * (y[1:] + y[:-1]) / 2.0 in pairwise order."""
    d = x[1:] - x[:-1]
    return pairwise_sum(d * (y[1:] + y[:-1]) / 2.0)


def mean0(a):
    """a.mean(0) of a C-contiguous 2-D float64 array: rows added one after the other, then divided by the row count."""
    with np.errstate(all="ignore"):
        if a.shape[0] == 0:
            return np.full(a.shape[1:], np.nan)
        acc = a[0].copy()
        for row in a[1:]:
            acc = acc + row
        return acc / a.shape[0]


def smooth(y, f=0.05):
    """ultralytics.utils.metrics.smooth: box filter of nf = round(len(y) * f * 2) // 2 + 1 taps, edges padded with copies."""
    nf = round(len(y) * f * 2) // 2 + 1
    p = np.ones(nf // 2)
    yp = np.concatenate((p * y[0], y, p * y[-1]), 0)
    return np.convolve(yp, np.ones(nf) / nf, mode="valid")


def compute_ap(recall, precision):
    """compute_ap (reference utils/metrics.py:98-126, method "interp") with the restated interp and trapezoid."""
    mrec = np.concatenate(([0.0], recall, [1.0]))
    mpre = np.concatenate(([1.0], precision, [0.0]))
    mpre = np.flip(np.maximum.accumulate(np.flip(mpre)))
    return trapezoid(interp(X101, mrec, mpre), X101)


def ap_per_class(tp, conf, pred_cls, target_cls, eps=1e-16, stable=True, return_index=False):
    """Returns (tp, fp, p, r, f1, ap, unique_classes) as the reference does; with return_index also the max-F1 index i and the
    gap between the two largest smoothed mean-F1 values (a gap under 1e-12 makes i depend on np.convolve's summation order)."""
    tp = np.asarray(tp).astype(bool)
    conf = np.asarray(conf)
    pred_cls = np.asarray(pred_cls)
    i = np.argsort(-conf, kind="stable") if stable else np.argsort(-conf)
    tp, conf, pred_cls = tp[i], conf[i], pred_cls[i]
    unique_classes, nt = np.unique(target_cls, return_counts=True)
    nc = unique_classes.shape[0]
    ap, p, r = np.zeros((nc, tp.shape[1])), np.zeros((nc, 1000)), np.zeros((nc, 1000))
    for ci, c in enumerate(unique_classes):
        sel = pred_cls == c
        n_l, n_p = nt[ci], sel.sum()
        if n_p == 0 or n_l == 0:
            continue
        fpc = (1 - tp[sel]).cumsum(0)
        tpc = tp[sel].cumsum(0)
        recall = tpc / (n_l + eps)
        r[ci] = interp(-PX, -conf[sel], recall[:, 0], left=0)
        precision = tpc / (tpc + fpc)
        p[ci] = interp(-PX, -conf[sel], precision[:, 0], left=1)
        for j in range(tp.shape[1]):
            ap[ci, j] = compute_ap(recall[:, j], precision[:, j])
    with np.errstate(all="ignore"):
        f1 = 2 * p * r / (p + r + eps)
        s = smooth(mean0(f1), 0.1)
    k = int(s.argmax())
    p, r, f1 = p[:, k], r[:, k], f1[:, k]
    tp = (r * nt).round()
    with np.errstate(all="ignore"):
        fp = (tp / (p + eps) - tp).round()
    out = (tp, fp, p, r, f1, ap, unique_classes.astype(int))
    if return_index:
        top = np.sort(s[~np.isnan(s)])[-2:] if s.size else s
        gap = float(top[-1] - top[-2]) if top.size == 2 else np.inf
        return out, k, gap
    return out


def synth_stats(n_img, max_det=300, nc=80, mean_labels=7.3, niou=10, seed=0, ties=True, min_det=None):
    """COCO-val-like per-image stats, as val.py appends them: a list of (correct (n_i, niou) bool, conf (n_i,) float32,
    pred_cls (n_i,) float32, target_cls (m_i,) float32).  Poisson(mean_labels) labels per image with a skewed class mix;
    min_det (default max_det // 3) to max_det predictions per image, half of them of a class labelled in the image.
    Thresholds nest (correct at a stricter one implies correct at the looser ones) and no class of an image gets more true
    positives than it has labels.
    ties=True rounds confidences to fp16 (long runs of equal values); ties=False makes every confidence distinct."""
    rs = np.random.RandomState(seed)
    w = 1.0 / np.arange(1, nc + 1) ** 0.8
    w /= w.sum()
    sizes = rs.randint(max_det // 3 if min_det is None else min_det, max_det + 1, n_img) if max_det else np.zeros(n_img, int)
    distinct = (rs.permutation(int(sizes.sum())) + 0.5) / max(int(sizes.sum()), 1)
    at = 0
    stats = []
    for b in range(n_img):
        labels = rs.choice(nc, rs.poisson(mean_labels), p=w)
        n = int(sizes[b])
        own = rs.rand(n) < 0.5
        cls = np.where(own & (labels.size > 0), rs.choice(labels, n) if labels.size else 0, rs.choice(nc, n, p=w))
        if ties:
            conf = (rs.rand(n) ** 3).astype(np.float16).astype(np.float32)
        else:
            conf = distinct[at:at + n].astype(np.float32)
            at += n
        k = np.where(own, np.floor(rs.rand(n) * (niou + 1.5)).astype(int).clip(0, niou), 0)
        for c in np.unique(cls):  # at most as many true positives as labels of the class
            rows = np.nonzero((cls == c) & (k > 0))[0]
            k[rs.permutation(rows)[(labels == c).sum():]] = 0
        correct = np.arange(niou)[None, :] < k[:, None]
        stats.append((correct, conf, cls.astype(np.float32), labels.astype(np.float32)))
    return stats


def concat_stats(stats):
    """val.py:328: the per-image stats concatenated -> (tp, conf, pred_cls, target_cls)."""
    return tuple(np.concatenate([s[i] for s in stats], 0) for i in range(4))
