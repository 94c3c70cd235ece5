"""Segmentation ComputeLoss with the reference's interface (reference utils/segment/loss.py:15-195):
``ComputeLoss(model, overlap=...)((p, proto), targets, masks) -> (loss (1,), items (4,) = [lbox, lseg, lobj, lcls])`` and
``.build_targets(p, targets) -> (tcls, tbox, indices, anch, tidxs, xywhn)``.  The box / objectness / class terms run
the detection loss's kernels; the mask term (BCE of ``coef @ proto`` inside each match's box crop, mean per image and
level) and its gradients for the head maps and for ``proto`` run in liby5b200 (y5_seg_loss_fwd_bwd_scaled) without a
host sync, visiting only the pixels inside the crops.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from ... import _lib
from ..loss import ComputeLoss as _DetComputeLoss
from ..torch_utils import de_parallel


class _SegLossFn(torch.autograd.Function):
    """loss, items = ComputeLoss((p, proto), targets, masks).  Like utils.loss._LossFn: the forward launch set computes the
    loss only, the backward one re-runs it with the gradient outputs and the upstream gradient of the loss (a device scalar)
    multiplied in fp32 inside the kernels before anything is rounded."""

    @staticmethod
    def forward(ctx, crit, targets, masks, proto, *p):
        out, _, _ = crit._run(p, proto, targets, masks, want_grad=False)
        ctx.crit, ctx.targets, ctx.masks = crit, targets, masks
        ctx.save_for_backward(proto, *p)
        ctx.mark_non_differentiable(out[1])
        return out[0], out[1]

    @staticmethod
    def backward(ctx, g_loss, _g_items):
        proto, *p = ctx.saved_tensors
        if not any(ctx.needs_input_grad[3:]):
            return (None, None, None, None) + (None,) * len(p)
        scale = g_loss.detach().reshape(-1)[:1].to(proto.device, torch.float32).contiguous()
        _, grads, gproto = ctx.crit._run(p, proto, ctx.targets, ctx.masks, want_grad=True, grad_scale=scale)
        return (None, None, None, gproto) + tuple(grads)


class ComputeLoss(_DetComputeLoss):
    def __init__(self, model, autobalance=False, overlap=False):
        super().__init__(model, autobalance=autobalance)
        self.overlap = overlap
        self.nm = de_parallel(model).model[-1].nm
        self._ws = None

    # -------------------------------------------------------------------------------------------------------------
    def _check(self, p, proto, targets, masks):
        bs = self._check_shapes(p, targets, 5 + self.nc + self.nm)
        if proto.dim() != 4 or proto.shape[0] != bs or proto.shape[1] != self.nm:
            raise ValueError(f"y5b200: proto {tuple(proto.shape)} is not (B={bs}, nm={self.nm}, mh, mw)")
        if masks.dim() != 3:
            raise ValueError(f"y5b200: masks must be (N, H, W), got {tuple(masks.shape)}")
        nt = targets.numel() // 6
        if self.overlap and masks.shape[0] != bs:
            raise ValueError(f"y5b200: overlap masks need one (H, W) map per image: {masks.shape[0]} != batch {bs}")
        if not self.overlap and masks.shape[0] < nt:
            raise ValueError(f"y5b200: {masks.shape[0]} masks for {nt} targets")
        if not all(t.is_cuda for t in p) or not proto.is_cuda:
            raise RuntimeError("y5b200: ComputeLoss runs on CUDA tensors only (no CPU / PyTorch fallback)")

    def _run(self, p, proto, targets, masks, want_grad, grad_scale=None):
        self._check(p, proto, targets, masks)
        lib = _lib.lib()
        dev = p[0].device
        p = [t.contiguous() for t in p]
        # the kernels address proto and dproto with proto's strides, so both must be dense: NCHW or channels_last
        # as given, any other view (channel slice, crop, step) copied first, channels innermost staying innermost
        if not (proto.is_contiguous() or proto.is_contiguous(memory_format=torch.channels_last)):
            proto = proto.contiguous(memory_format=torch.channels_last if proto.stride(1) == 1 else torch.contiguous_format)
        tg = targets.to(dev, torch.float32).contiguous().view(-1, 6)
        mk = masks.to(dev, torch.float32).contiguous()
        q = self._params(p, tg.shape[0])
        need = int(lib.y5_seg_loss_workspace_bytes(C.byref(q)))
        if need < 0:
            _lib.check(-1, "seg_loss_workspace_bytes")
        key = (dev.index, _lib.stream_ptr(dev))  # scratch per (device, stream): concurrent streams never share it
        if self._ws is None:
            self._ws = {}
        ws = self._ws.get(key)
        if ws is None or ws.numel() < need + 256:
            ws = self._ws[key] = torch.empty(need + 256, dtype=torch.uint8, device=dev)
        ws_ptr = (ws.data_ptr() + 255) & ~255
        anchors = self.anchors.to(dev, torch.float32).contiguous()
        out = torch.empty(5, dtype=torch.float32, device=dev)
        grads = [torch.empty_like(t) for t in p] if want_grad else None
        gproto = torch.empty_strided(proto.shape, proto.stride(), dtype=proto.dtype, device=dev) if want_grad else None
        pl = (C.c_void_p * self.nl)(*[t.data_ptr() for t in p])
        gl = (C.c_void_p * self.nl)(*[g.data_ptr() for g in grads]) if want_grad else None
        bs, nm, mh, mw = proto.shape
        with _lib.on(dev):
            _lib.check(lib.y5_seg_loss_fwd_bwd_scaled(
                C.byref(q), pl, tg.data_ptr(), anchors.data_ptr(), proto.data_ptr(), _lib.dtype_code(proto.dtype), *proto.stride(),
                nm, mh, mw, mk.data_ptr(), mk.shape[0], mk.shape[1], mk.shape[2], int(bool(self.overlap)), out.data_ptr(), gl,
                gproto.data_ptr() if want_grad else None, grad_scale.data_ptr() if grad_scale is not None else None, ws_ptr, need,
                C.c_void_p(_lib.stream_ptr(dev))), "seg_loss_fwd_bwd")
        self._last = (q, ws_ptr)
        return (out[0:1], out[1:5]), grads, gproto

    def __call__(self, preds, targets, masks):
        p, proto = preds
        loss, items = _SegLossFn.apply(self, targets, masks, proto, *p)
        return loss, items.detach()

    def build_targets(self, p, targets):
        """(tcls, tbox, indices, anch, tidxs, xywhn) like reference utils/segment/loss.py:122-195 (int64 indices and tidxs,
        fp32 tbox and xywhn)."""
        bs, nt = p[0].shape[0], targets.numel() // 6
        dev = p[0].device
        proto = torch.zeros(bs, self.nm, 1, 1, dtype=p[0].dtype, device=dev)  # the mask term is not needed here
        masks = torch.zeros(bs if self.overlap else max(nt, 1), 1, 1, device=dev)
        self._run(p, proto, targets, masks, want_grad=False)
        q, ws_ptr = self._last
        lib = _lib.lib()
        st = C.c_void_p(_lib.stream_ptr(dev))
        cap = max(1, 5 * self.na * q.nt)
        tcls, tbox, indices, anch, tidxs, xywhn = [], [], [], [], [], []
        for l in range(self.nl):
            idx = np.empty((5, cap), np.int64)
            tb = np.empty((cap, 4), np.float32)
            ti = np.empty(cap, np.int64)
            xy = np.empty((cap, 4), np.float32)
            cnt = C.c_int32()
            _lib.check(lib.y5_loss_read_targets(C.byref(q), ws_ptr, l, idx.ctypes.data, tb.ctypes.data, C.byref(cnt), st),
                       "loss_read_targets")
            _lib.check(lib.y5_seg_loss_read_targets(C.byref(q), ws_ptr, l, ti.ctypes.data, xy.ctypes.data, C.byref(cnt), st),
                       "seg_loss_read_targets")
            n = cnt.value
            ii = torch.from_numpy(idx.reshape(-1)[: 5 * n].reshape(5, n).copy()).to(dev)
            indices.append((ii[0], ii[1], ii[2], ii[3]))
            tcls.append(ii[4])
            tbox.append(torch.from_numpy(tb[:n].copy()).to(dev))
            anch.append(self.anchors.to(dev)[l][ii[1]])
            tidxs.append(torch.from_numpy(ti[:n].copy()).to(dev))
            xywhn.append(torch.from_numpy(xy[:n].copy()).to(dev))
        return tcls, tbox, indices, anch, tidxs, xywhn

