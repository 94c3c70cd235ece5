"""ComputeLoss with the reference's interface (reference utils/loss.py:101-247): ``ComputeLoss(model)(p, targets) ->
(loss (1,), items (3,))`` and ``.build_targets(p, targets)``.  build_targets, the gather/CIoU/scatter and both BCE
terms -- forward and backward -- run in liby5b200 (y5_loss_fwd_bwd_scaled); the returned loss carries a custom autograd
node that hands the kernel-computed gradient of every prediction level back to PyTorch.  ``CrossEntropyLoss`` is the
classification loss (nn.CrossEntropyLoss with label smoothing) on y5_cross_entropy.
"""
from __future__ import annotations

import ctypes as C

import torch
from torch import nn

from .. import _lib
from .._lib import LossParams
from .torch_utils import de_parallel


def smooth_bce(eps=0.1):
    return 1.0 - 0.5 * eps, 0.5 * eps


class _LossFn(torch.autograd.Function):
    """loss, items = ComputeLoss(p, targets).  The forward launch set computes the loss only; the backward one re-runs it with
    the gradient outputs enabled and the UPSTREAM gradient of the loss (GradScaler's factor x WORLD_SIZE x ..., a device
    scalar) multiplied in fp32 inside the kernels before anything is rounded to the prediction dtype -- exactly where
    autograd applies it for `scaler.scale(loss).backward()` (reference train.py:410).  Scaling fp16 gradients afterwards
    would overflow (65536 is not an fp16 number) and would already have flushed small objectness gradients to zero."""

    @staticmethod
    def forward(ctx, crit, targets, *p):
        out, _ = crit._run(p, targets, want_grad=False)
        ctx.crit, ctx.targets = crit, targets
        ctx.save_for_backward(*p)
        ctx.mark_non_differentiable(out[1])
        return out[0], out[1]

    @staticmethod
    def backward(ctx, g_loss, _g_items):
        p = ctx.saved_tensors
        if not any(ctx.needs_input_grad[2:]):
            return (None, None) + (None,) * len(p)
        scale = g_loss.detach().reshape(-1)[:1].to(p[0].device, torch.float32).contiguous()
        _, grads = ctx.crit._run(p, ctx.targets, want_grad=True, grad_scale=scale)
        return (None, None) + tuple(grads)


class _CrossEntropyFn(torch.autograd.Function):
    """loss = CrossEntropyLoss(label_smoothing)(logits, labels) on y5_cross_entropy.  As _LossFn: the forward launch computes the
    loss only; the backward re-launches the kernel with the upstream gradient (a device scalar) multiplied in fp32 before the
    gradient is rounded to the logits dtype -- where torch-autocast rounds it, since cross_entropy runs in fp32 under autocast."""

    @staticmethod
    def forward(ctx, eps, labels, logits):
        ctx.eps = eps
        ctx.save_for_backward(labels, logits)
        return _cross_entropy(logits, labels, eps)[0]

    @staticmethod
    def backward(ctx, g_loss):
        labels, logits = ctx.saved_tensors
        if not ctx.needs_input_grad[2]:
            return None, None, None
        scale = g_loss.detach().reshape(-1)[:1].to(logits.device, torch.float32).contiguous()
        return None, None, _cross_entropy(logits, labels, ctx.eps, grad_scale=scale)[1]


def _cross_entropy(logits, labels, eps, grad_scale=None):
    """(0-d fp32 loss, dlogits (B, nc) in the logits dtype or None) from one y5_cross_entropy call (no host synchronisation)."""
    b, nc = logits.shape
    if logits.stride(1) != 1:
        logits = logits.contiguous()
    dev = logits.device
    row_loss = torch.empty(b, dtype=torch.float32, device=dev)
    loss = torch.empty((), dtype=torch.float32, device=dev)
    grad = torch.empty(b, nc, dtype=logits.dtype, device=dev) if grad_scale is not None else None
    with _lib.on(dev):
        _lib.check(_lib.lib().y5_cross_entropy(logits.data_ptr(), _lib.dtype_code(logits.dtype), b, nc, logits.stride(0), labels.data_ptr(),
                                               float(eps), grad_scale.data_ptr() if grad_scale is not None else None,
                                               grad.data_ptr() if grad is not None else None, nc, row_loss.data_ptr(), loss.data_ptr(),
                                               C.c_void_p(_lib.stream_ptr(dev))), "cross_entropy")
    return loss, grad


class CrossEntropyLoss(nn.CrossEntropyLoss):
    """nn.CrossEntropyLoss(label_smoothing=eps) with reduction='mean' on class-index targets -- what smartCrossEntropyLoss
    returns to classify/train.py and classify/val.py -- computed forward and backward by y5_cross_entropy:
    mean_i[(1 - eps) (-log p_{i,y_i}) + (eps / nc) sum_c (-log p_{i,c})] in fp32 with a max-subtracted log-sum-exp.
    Logits (B, nc) in fp16 / bf16 / fp32; the loss is fp32, or the logits dtype outside autocast as torch returns it.
    A label outside [0, nc) -- ignore_index's -100 included -- gives a NaN loss and NaN gradients for its row (the reference
    stops at a device assert instead).  weight=, reduction != 'mean', a non-default ignore_index and probability targets are
    not implemented; CPU tensors are refused (no PyTorch fallback)."""

    def forward(self, input, target):
        if self.weight is not None:
            raise NotImplementedError("y5b200: CrossEntropyLoss(weight=...) is not implemented")
        if self.reduction != "mean":
            raise NotImplementedError(f"y5b200: CrossEntropyLoss(reduction='{self.reduction}') is not implemented (mean only)")
        if self.ignore_index != -100:
            raise NotImplementedError("y5b200: CrossEntropyLoss(ignore_index=...) is not implemented")
        if target.is_floating_point():
            raise NotImplementedError("y5b200: CrossEntropyLoss with class-probability targets is not implemented (class indices only)")
        if not (input.is_cuda and target.is_cuda):
            raise RuntimeError("y5b200: CrossEntropyLoss runs on CUDA tensors only (no CPU / PyTorch fallback)")
        if input.dim() != 2 or target.shape != input.shape[:1]:
            raise ValueError(f"y5b200: CrossEntropyLoss expects (B, nc) logits and (B,) labels, got {tuple(input.shape)} and {tuple(target.shape)}")
        labels = target if target.dtype == torch.int64 and target.is_contiguous() else target.long().contiguous()
        loss = _CrossEntropyFn.apply(float(self.label_smoothing), labels, input)
        if input.dtype != torch.float32 and not torch.is_autocast_enabled("cuda"):
            loss = loss.to(input.dtype)  # F.cross_entropy on fp16 / bf16 logits returns that dtype
        return loss


class ComputeLoss:
    sort_obj_iou = False

    def __init__(self, model, autobalance=False):
        if autobalance:
            raise NotImplementedError("y5b200: autobalance is outside the hot path (reference default False)")
        m = de_parallel(model).model[-1]
        h = model.hyp
        if h.get("fl_gamma", 0.0) > 0:
            raise NotImplementedError("y5b200: focal loss (fl_gamma > 0) is outside the hot path (default hyp uses 0)")
        self.hyp = h
        self.device = next(model.parameters()).device
        self.cp, self.cn = smooth_bce(eps=h.get("label_smoothing", 0.0))
        self.balance = {3: [4.0, 1.0, 0.4]}.get(m.nl, [4.0, 1.0, 0.25, 0.06, 0.02])
        self.na, self.nc, self.nl = m.na, m.nc, m.nl
        self.anchors = m.anchors
        self.gr = 1.0
        self._ws = None

    # -------------------------------------------------------------------------------------------------------------
    def _params(self, p, nt):
        q = LossParams()
        q.nl, q.batch, q.na, q.no, q.nc = self.nl, p[0].shape[0], self.na, p[0].shape[-1], self.nc
        for l, t in enumerate(p):
            q.ny[l], q.nx[l] = t.shape[2], t.shape[3]
            q.balance[l] = self.balance[l]
        q.dtype = _lib.dtype_code(p[0].dtype)
        q.nt = nt
        h = self.hyp
        q.anchor_t, q.box_gain, q.obj_gain, q.cls_gain = h["anchor_t"], h["box"], h["obj"], h["cls"]
        q.cls_pw, q.obj_pw, q.cp, q.cn = h["cls_pw"], h["obj_pw"], self.cp, self.cn
        q.grad_scale = 1.0
        return q

    def _check_shapes(self, p, targets, no):
        """Shape checks before any launch: the kernels take batch, dtype and grid strides from these tensors, so a level
        with another batch, anchor count, channel count or dtype would be read past its end."""
        if len(p) != self.nl:
            raise ValueError(f"y5b200: expected {self.nl} head maps, got {len(p)}")
        bs, dt = p[0].shape[0] if p[0].dim() else -1, p[0].dtype
        for t in p:
            if t.dim() != 5 or t.shape[0] != bs or t.shape[1] != self.na or t.shape[4] != no:
                raise ValueError(f"y5b200: head map {tuple(t.shape)} is not (B={bs}, na={self.na}, ny, nx, {no})")
            if t.dtype != dt:
                raise ValueError(f"y5b200: head maps must share one dtype, got {dt} and {t.dtype}")
        if targets.dim() != 2 or targets.shape[1] != 6:
            raise ValueError(f"y5b200: targets must be (n, 6) [image, class, x, y, w, h], got {tuple(targets.shape)}")
        return bs

    def _run(self, p, targets, want_grad, grad_scale=None):
        self._check_shapes(p, targets, 5 + self.nc)
        if not all(t.is_cuda for t in p):
            raise RuntimeError("y5b200: ComputeLoss runs on CUDA tensors only (no CPU / PyTorch fallback)")
        lib = _lib.lib()
        dev = p[0].device
        p = [t.contiguous() for t in p]
        tg = targets.to(dev, torch.float32).contiguous().view(-1, 6)
        q = self._params(p, tg.shape[0])
        need = int(lib.y5_loss_workspace_bytes(C.byref(q)))
        if need < 0:
            _lib.check(-1, "loss_workspace_bytes")
        key = (dev.index, _lib.stream_ptr(dev))  # scratch per (device, stream): concurrent streams never share it
        if self._ws is None:
            self._ws = {}
        ws = self._ws.get(key)
        if ws is None or ws.numel() < need + 256:
            ws = self._ws[key] = torch.empty(need + 256, dtype=torch.uint8, device=dev)
        ws_ptr = (ws.data_ptr() + 255) & ~255
        anchors = self.anchors.to(dev, torch.float32).contiguous()
        out = torch.empty(4, dtype=torch.float32, device=dev)
        grads = [torch.empty_like(t) for t in p] if want_grad else None
        pl = (C.c_void_p * self.nl)(*[t.data_ptr() for t in p])
        gl = (C.c_void_p * self.nl)(*[g.data_ptr() for g in grads]) if want_grad else None
        with _lib.on(dev):
            _lib.check(lib.y5_loss_fwd_bwd_scaled(C.byref(q), pl, tg.data_ptr(), anchors.data_ptr(), out.data_ptr(), gl,
                                                  grad_scale.data_ptr() if grad_scale is not None else None, ws_ptr, need,
                                                  C.c_void_p(_lib.stream_ptr(dev))), "loss_fwd_bwd")
        self._last = (q, ws_ptr)
        return (out[0:1], out[1:4]), grads

    def __call__(self, p, targets):
        loss, items = _LossFn.apply(self, targets, *p)
        return loss, items.detach()

    def build_targets(self, p, targets):
        """(tcls, tbox, indices, anch) like reference utils/loss.py:185-247 (int64 indices, fp32 boxes)."""
        self._run(p, targets, want_grad=False)
        q, ws_ptr = self._last
        lib = _lib.lib()
        dev = p[0].device
        cap = max(1, 5 * self.na * q.nt)
        tcls, tbox, indices, anch = [], [], [], []
        import numpy as np

        for l in range(self.nl):
            idx = np.empty((5, cap), np.int64)
            tb = np.empty((cap, 4), np.float32)
            cnt = C.c_int32()
            _lib.check(lib.y5_loss_read_targets(C.byref(q), ws_ptr, l, idx.ctypes.data, tb.ctypes.data, C.byref(cnt),
                                                C.c_void_p(_lib.stream_ptr(dev))), "loss_read_targets")
            n = cnt.value
            ii = torch.from_numpy(idx.reshape(-1)[: 5 * n].reshape(5, n).copy()).to(dev)
            indices.append((ii[0], ii[1], ii[2], ii[3]))
            tcls.append(ii[4])
            tbox.append(torch.from_numpy(tb[:n].copy()).to(dev))
            anch.append(self.anchors.to(dev)[l][ii[1]])
        return tcls, tbox, indices, anch
