"""Training-mode execution of the hot path: Conv = act(BN_batchstats(conv(x))) forward and backward on liby5b200, act = SiLU,
LeakyReLU / ReLU or none.

Reference: models/common.py:86-88 (Conv.forward), :181 (Bottleneck), :246 (C3), :338-340 (SPPF), :453 (Concat),
models/yolo.py:95-98 (Detect in training returns the raw (B,na,ny,nx,no) maps), :160-170 (_forward_once routing);
train.py:401-410 (autocast forward, scaled backward).

What runs where
  * every convolution (forward, data gradient, weight gradient), BatchNorm batch statistics / normalise / backward and
    activation forward / backward: liby5b200 kernels (wgmma implicit GEMMs + HBM-bound passes), wrapped in
    torch.autograd.Function so gradients land in the ordinary ``.grad`` of the nn.Parameters (DDP's bucketed NCCL
    all-reduce -- smart_DDP -- works unchanged); a torch.nn.SyncBatchNorm that syncs (bn_sync_group) all-reduces its column
    sums between the split BN passes (train.py --sync-bn);
  * the glue between convolutions is liby5b200 too: channel concat = strided slice copies whose backward is a set of
    views, 2x nearest upsample and its 2x2-sum backward, SPPF's pooling chain and its arg-max backward, the Bottleneck
    shortcut as a residual operand of cv2's normalise+activate pass, GhostConv's depthwise half and its concat in one pass
    (y5_dwconv_fwd / y5_dwconv_wgrad).  What is left to torch autograd is bookkeeping: the
    graph itself, summing gradients of tensors with several consumers, the (B,na,ny,nx,no) permute of the head output.
    Activations are channels_last, so every op reads and writes the same NHWC bytes and no layout conversion exists.

Precision: activations and their gradients in fp16/bf16 (the autocast dtype, or the parameter dtype if the model was
cast), BN statistics / affine gradients / weight gradients in fp32 -- the reference's AMP recipe.
"""
from __future__ import annotations

import ctypes as C
import os
import weakref

import torch

from . import _lib
from .engine import (IMAGE_C, ConvInput, act_spec, conv_desc, image_nhwc, is_v6_stem, pack_weight, pad_image_weight, stem_buffer, stem_geom,
                     stem_s2d, stem_weight_narrow, stem_weight_wide, wgrad_desc)
from .engine import block_k as _block_k  # the shared, cached y5_conv_pick lookup


def _st(dev):
    return C.c_void_p(_lib.stream_ptr(dev))


def _cl(x: torch.Tensor) -> torch.Tensor:
    """dense channels_last (NHWC bytes) view / copy of a (B,C,H,W) tensor"""
    b, c, h, w = x.shape
    if x.stride() == (h * w * c, 1, w * c, c):
        return x
    y = torch.empty_strided((b, c, h, w), (h * w * c, 1, w * c, c), dtype=x.dtype, device=x.device)
    y.copy_(x)
    return y


def _nhwc(x: torch.Tensor):
    """(tensor, pitch) such that element (n,c,y,x) sits at data_ptr + (((n*H + y)*W + x)*pitch + c) elements: the tensor
    itself when it is channels_last or a channel slice of a channels_last buffer (what torch.cat's backward hands
    out), else a dense channels_last copy."""
    b, c, h, w = x.shape
    sn, sc, sh, sw = x.stride()
    if sc == 1 and sw >= c and sw % 8 == 0 and sh == w * sw and sn == h * sh and x.data_ptr() % 16 == 0:
        return x, sw
    return _cl(x), c


def _empty_cl(b, c, h, w, dtype, device):
    return torch.empty_strided((b, c, h, w), (h * w * c, 1, w * c, c), dtype=dtype, device=device)


_zero_bias_cache: dict = {}


def _zero_bias(n: int, device) -> torch.Tensor:
    key = (n, str(device))
    t = _zero_bias_cache.get(key)
    if t is None:
        t = _zero_bias_cache[key] = torch.zeros(n, dtype=torch.float32, device=device)
    return t


def pack_weights(w: torch.Tensor, dtype: torch.dtype, m_rows: int, want_fwd: bool = True, want_dgrad: bool = False):
    """OIHW master weights -> (fwd packing [O][k][k][I_pad], dgrad packing [I][k][k][O_pad]) in `dtype`, one launch
    (y5_weight_pack).  m_rows only steers the K-block choice."""
    lib = _lib.lib()
    w = w.detach()
    if not w.is_contiguous():
        w = w.contiguous()
    o, i, k, _ = w.shape
    fwd = dg = None
    ipad = opad = bk_f = bk_d = 0
    if want_fwd:
        bk_f = _block_k(i, o, m_rows)
        ipad = (i + bk_f - 1) // bk_f * bk_f
        fwd = torch.empty(o, k, k, ipad, dtype=dtype, device=w.device)
    if want_dgrad:
        bk_d = _block_k(o, i, m_rows)
        opad = (o + bk_d - 1) // bk_d * bk_d
        dg = torch.empty(i, k, k, opad, dtype=dtype, device=w.device)
    _lib.check(lib.y5_weight_pack(w.data_ptr(), _lib.dtype_code(w.dtype), o, i, k, fwd.data_ptr() if fwd is not None else None, ipad,
                                  dg.data_ptr() if dg is not None else None, opad, _lib.dtype_code(dtype), _st(w.device)), "weight_pack")
    return fwd, dg, bk_f, bk_d


class _PackEntry:
    __slots__ = ("weight", "wptr", "fwd", "dg", "ipad", "opad", "bk_f", "bk_d", "epoch")


class PackPlan:
    """The per-step re-packing of a model's fp32 master weights as ONE launch (y5_weight_pack_multi) into persistent buffers.

    The first training forward packs layer by layer (pack_weights) and registers every filter here together with the buffers
    it packed into; from the next forward on, `begin()` converts all registered filters in one launch before the first layer
    runs, and the layers just look their buffers up -- 1 launch and 1 library call per step instead of ~80, no allocations.
    The buffers are overwritten by the next forward's launch, which is stream-ordered after the backward that read them."""

    def __init__(self, device, dtype):
        self.device, self.dtype = device, dtype
        self.entries: dict = {}
        self.dirty = False
        self.epoch = 0
        self.table = None  # (items, chunk_item, chunk_index, n_chunks) in device memory
        self.keep: list = []  # replaced buffers stay alive: a captured CUDA graph may still write to them

    def __deepcopy__(self, memo):  # copy.deepcopy(model) (ModelEMA): the copy has other parameters, it starts an empty plan
        return PackPlan(self.device, self.dtype)

    def begin(self):
        """Start of a training forward: one launch packs every registered filter from the current master weights."""
        self.epoch += 1
        if not self.dirty and self.table is not None:
            for e in self.table[4]:  # a parameter whose storage was replaced (.to(), .data = ...): its table row points at the old one
                if e.wptr != e.weight.data_ptr():
                    self.dirty = True
                    break
        if self.dirty or self.table is None:
            if torch.cuda.is_current_stream_capturing():
                return  # no host-to-device table upload inside a capture: this forward packs layer by layer
            self._build()
        if self.table is None:
            return
        items, ci, cx, n, ents = self.table
        with _lib.on(self.device):
            _lib.check(_lib.lib().y5_weight_pack_multi(items.data_ptr(), ci.data_ptr(), cx.data_ptr(), n, _lib.dtype_code(self.dtype),
                                                       _st(self.device)), "weight_pack_multi")
        for e in ents:
            e.epoch = self.epoch

    def _build(self):
        ents = [e for e in self.entries.values() if e.wptr == e.weight.data_ptr()]
        self.dirty = False
        if not ents:
            self.table = None
            return
        chunk = int(_lib.lib().y5_weight_pack_chunk_elems())
        arr = (_lib.PackItem * len(ents))()
        ci, cx = [], []
        for t, e in enumerate(ents):
            o, i, k, _ = e.weight.shape
            it = arr[t]
            it.w, it.fwd, it.dgrad = e.wptr, e.fwd.data_ptr(), (e.dg.data_ptr() if e.dg is not None else None)
            it.w_dtype = _lib.dtype_code(e.weight.dtype)
            it.out_c, it.in_c, it.ksize, it.in_c_pad, it.out_c_pad = o, i, k, e.ipad, e.opad
            total = o * k * k * e.ipad + (i * k * k * e.opad if e.dg is not None else 0)
            n = (total + chunk - 1) // chunk
            ci += [t] * n
            cx += list(range(n))
        items = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(self.device)
        self.table = (items, torch.tensor(ci, dtype=torch.int32, device=self.device), torch.tensor(cx, dtype=torch.int32, device=self.device),
                      len(ci), ents)

    def lookup(self, weight, bk_f, bk_d, need_dx):
        """(fwd, dgrad) buffers holding THIS forward's packing of `weight`, or None (not registered / not packed this forward /
        another geometry)."""
        e = self.entries.get(id(weight))
        if (e is None or e.epoch != self.epoch or e.weight is not weight or e.wptr != weight.data_ptr() or e.bk_f != bk_f
                or (need_dx and (e.dg is None or e.bk_d != bk_d))):
            return None
        return e.fwd, e.dg

    def register(self, weight, fwd, dg, ipad, opad, bk_f, bk_d):
        if not weight.is_contiguous() or weight.device != self.device or fwd.dtype != self.dtype:
            return
        old = self.entries.get(id(weight))
        if old is not None:
            self.keep += [old.fwd, old.dg]
        e = _PackEntry()
        e.weight, e.wptr, e.fwd, e.dg, e.ipad, e.opad, e.bk_f, e.bk_d, e.epoch = weight, weight.data_ptr(), fwd, dg, ipad, opad, bk_f, bk_d, -1
        self.entries[id(weight)] = e
        self.dirty = True

    def tensors(self):
        """everything a captured graph's pack launch touches (GraphedTrainStep keeps these alive)"""
        out = list(self.keep)
        for e in self.entries.values():
            out += [e.fwd, e.dg]
        if self.table is not None:
            out += list(self.table[:3])
        return out


_cur_plan: PackPlan | None = None  # the plan of the forward_train that is running (None: layers pack for themselves)


def pack_plan_enabled() -> bool:
    return os.environ.get("Y5_TRAIN_PACK_PLAN", "1") != "0"


def pack_plan(model, dtype, device) -> PackPlan:
    plans = model.__dict__.setdefault("_y5_pack_plans", {})
    key = (str(device), dtype)
    if key not in plans:
        plans[key] = PackPlan(device, dtype)
    return plans[key]


def conv_packed(x: torch.Tensor, x_pitch: int, wp: torch.Tensor, block_k: int, bias32: torch.Tensor | None, cout: int, k: int, s: int, p: int,
                act: bool = False) -> torch.Tensor:
    """y = act(conv(x, w) + bias) through y5_conv_bn_silu_fwd.  x: (B,Cin,H,W) NHWC view with row pitch x_pitch; wp: K-major
    packed weights [cout][k][k][cin_pad]."""
    b, cin, h, w = x.shape
    ho, wo = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
    if cin % 8 or cout % 8:
        raise NotImplementedError(f"y5b200: training convs need channel counts that are multiples of 8 (got {cin} -> {cout})")
    bias32 = _zero_bias(cout, x.device) if bias32 is None else bias32
    y = _empty_cl(b, cout, ho, wo, x.dtype, x.device)
    d = conv_desc(ConvInput(x.data_ptr(), x_pitch, b, h, w, cin), wp, bias32, block_k, y.data_ptr(), cout, k, s, p, act, x.dtype)
    _lib.check(_lib.lib().y5_conv_bn_silu_fwd(C.byref(d), _st(x.device)), "conv fprop/dgrad")
    return y


def conv_raw(x: torch.Tensor, w_oihw: torch.Tensor, bias: torch.Tensor | None, k: int, s: int, p: int, act: bool = False) -> torch.Tensor:
    """One-off conv from OIHW weights (packs them first)."""
    x, pitch = _nhwc(x)
    b, cin, h, w = x.shape
    ho, wo = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
    wp, _, bk, _ = pack_weights(w_oihw, x.dtype, b * ho * wo)
    bias32 = None if bias is None else bias.detach().float().contiguous()
    return conv_packed(x, pitch, wp, bk, bias32, w_oihw.shape[0], k, s, p, act)


def conv_dgrad(dy: torch.Tensor, w_oihw: torch.Tensor | None, k: int, s: int, p: int, in_hw: tuple[int, int], wp_dgrad: torch.Tensor | None = None,
               cin: int | None = None, block_k: int = 0) -> torch.Tensor:
    """dx of y = conv(x, w): a stride-1 conv of dy with the flipped, transposed filter (stride-2 layers first expand dy
    with zeros).  dy: (B,Cout,Ho,Wo) NHWC view; pass either the OIHW weights or their dgrad packing."""
    lib = _lib.lib()
    dy, pitch = _nhwc(dy)
    b, cout, ho, wo = dy.shape
    if s == 2:
        if tuple(in_hw) != (2 * ho, 2 * wo):
            raise NotImplementedError("y5b200: stride-2 data gradient needs even input height/width")
        z = _empty_cl(b, cout, 2 * ho, 2 * wo, dy.dtype, dy.device)
        _lib.check(lib.y5_zero_stuff2x(dy.data_ptr(), pitch, z.data_ptr(), cout, b, ho, wo, cout, _lib.dtype_code(dy.dtype), _st(dy.device)),
                   "zero_stuff2x")
        dy, pitch = z, cout
    elif s != 1:
        raise NotImplementedError(f"y5b200: conv stride {s} backward")
    if wp_dgrad is None:
        _, wp_dgrad, _, block_k = pack_weights(w_oihw, dy.dtype, b * in_hw[0] * in_hw[1], want_fwd=False, want_dgrad=True)
        cin = w_oihw.shape[1]
    dx = conv_packed(dy, pitch, wp_dgrad, block_k, None, cin, k, 1, k - 1 - p, act=False)
    assert tuple(dx.shape[2:]) == tuple(in_hw), (dx.shape, in_hw)
    return dx


def conv_wgrad(x: torch.Tensor, dy: torch.Tensor, k: int, s: int, p: int) -> torch.Tensor:
    """fp32 dW (Cout,Cin,k,k) of y = conv(x, w) from NHWC views of x and dy."""
    x, xp = _nhwc(x)
    dy, dp = _nhwc(dy)
    b, cin, h, w = x.shape
    cout = dy.shape[1]
    dw = torch.empty(cout, k, k, cin, dtype=torch.float32, device=x.device)
    d = wgrad_desc(ConvInput(x.data_ptr(), xp, b, h, w, cin), dy.data_ptr(), dp, dw, k, s, p, x.dtype)
    _lib.check(_lib.lib().y5_conv_wgrad(C.byref(d), _st(x.device)), "conv_wgrad")
    if k == 1:
        return dw.view(cout, cin, 1, 1)  # KRSC == OIHW for 1x1 filters
    return dw.permute(0, 3, 1, 2).contiguous()  # gradients must be laid out like the parameter (DDP buckets, optimizers)


def stem_wide_enabled() -> bool:
    """Stem as a 3x1 conv over overlapping 48-channel "wide pixels" of the zero-padded space-to-depth image (the form the
    inference engine uses): 3 TMA rows per pixel instead of 9 for the forward and the weight gradient, which are bound by
    the TMA row rate on this 16-channel input.  On by default (Y5_TRAIN_STEM_WIDE=0 restores the 3x3x16 form)."""
    return os.environ.get("Y5_TRAIN_STEM_WIDE", "1") != "0"


def stem_conv_wide(buf: torch.Tensor, w3: torch.Tensor) -> torch.Tensor:
    """y = conv3x3/s1/p1(s2d image, w3) evaluated as a 3x1 conv over 48-channel wide pixels.  buf: stem_buffer; w3: (O,16,3,3)."""
    x = stem_geom(buf, wide=True)
    o = w3.shape[0]
    bk = _block_k(48, o, x.batch * x.in_h * x.in_w)
    wp = pack_weight(stem_weight_wide(w3.detach().float()), bk, buf.dtype)
    y = _empty_cl(x.batch, o, x.in_h, x.in_w, buf.dtype, buf.device)
    d = conv_desc(x, wp, _zero_bias(o, buf.device), bk, y.data_ptr(), o, 3, 1, 1, False, buf.dtype)
    _lib.check(_lib.lib().y5_conv_bn_silu_fwd(C.byref(d), _st(buf.device)), "stem conv (wide pixels)")
    return y


def stem_wgrad_wide(buf: torch.Tensor, dy: torch.Tensor) -> torch.Tensor:
    """fp32 gradient of the (O,16,3,3) space-to-depth stem filter from the stem_buffer and dy (B,O,H/2,W/2)."""
    dy, dp = _nhwc(dy)
    dw = torch.empty(dy.shape[1], 3, 1, 48, dtype=torch.float32, device=buf.device)
    d = wgrad_desc(stem_geom(buf, wide=True), dy.data_ptr(), dp, dw, 3, 1, 1, buf.dtype)
    _lib.check(_lib.lib().y5_conv_wgrad(C.byref(d), _st(buf.device)), "stem wgrad (wide pixels)")
    return stem_weight_narrow(dw.permute(0, 3, 1, 2))  # KRSC -> (O,48,3,1) -> (O,16,3,3)


_stem_idx_cache: dict = {}


def _stem_index(device):
    """gather indices between the (3,6,6) stem filter and its (16,3,3) space-to-depth form (see stem_weight_s2d):
    fwd[j] = flat (c,ky,kx) source of s2d element j (108 = the appended zero), inv[i] = s2d element holding source i."""
    key = str(device)
    if key not in _stem_idx_cache:
        fwd = torch.full((16 * 9,), 108, dtype=torch.long)
        inv = torch.zeros(108, dtype=torch.long)
        for dy in range(2):
            for dx in range(2):
                for c in range(3):
                    for r in range(3):
                        for q in range(3):
                            src = (c * 6 + (2 * r + dy)) * 6 + (2 * q + dx)
                            dst = (((dy * 2 + dx) * 3 + c) * 3 + r) * 3 + q
                            fwd[dst] = src
                            inv[src] = dst
        _stem_idx_cache[key] = (fwd.to(device), inv.to(device))
    return _stem_idx_cache[key]


class _ZeroArena:
    """fp64 scratch for the per-channel sums of the BN passes.  The kernels want it zero on entry; instead of one memset
    per layer the whole arena is cleared once at the start of a training forward and handed out in slices (forward and
    backward of the step both draw from it).  Outside a forward_train (single layers), or when it runs out, slices are
    freshly zeroed tensors and the arena grows at the next reset."""

    def __init__(self):
        self.buf = None
        self.off = 0
        self.want = 1 << 15

    def reset(self, device):
        if self.buf is None or self.buf.device != device or self.buf.numel() < self.want:
            self.buf = torch.zeros(self.want, dtype=torch.float64, device=device)
        else:
            self.buf.zero_()
        self.off = 0

    def take(self, n: int, device) -> torch.Tensor:
        n = (n + 1) // 2 * 2  # keep 16-byte alignment
        if self.buf is not None and self.buf.device == device and self.off + n <= self.buf.numel():
            v = self.buf[self.off : self.off + n]
            self.off += n
            return v
        self.want = max(self.want, 2 * (self.off + n))
        self.off += n
        return torch.zeros(n, dtype=torch.float64, device=device)


_arena = _ZeroArena()


def _bn_ws(c: int, device) -> torch.Tensor:
    return _arena.take(2 * c, device)


# ---------------------------------------------------------------------------------------------------------------------
# Weight gradients off the critical path.  Per layer the backward is  bn_bwd -> {dgrad, wgrad}; only dgrad feeds the next
# layer.  With `set_async_wgrad(True)` the weight-gradient kernels (and the KRSC -> OIHW copy behind them) are issued on a side
# stream that waits for the layer's dy; the calling stream joins it once, in a callback the autograd engine runs at the end of
# the backward pass (on the caller's stream).  Inside a captured CUDA graph that is a fork per layer and one join: the ~80
# small, latency-bound wgrad launches fill SMs the main chain leaves idle instead of extending it.  Off by default because
# anything that READS parameter gradients while backward is still running (DistributedDataParallel's bucket hooks, user
# hooks) would race with the side stream; GraphedTrainStep -- which takes plain modules only -- turns it on.
# ---------------------------------------------------------------------------------------------------------------------
_async_wgrad = False
_side_streams: dict = {}
_pending: list = []  # operands of in-flight side-stream work: freed only after the join, so the allocator cannot recycle them early
_join_armed = False


def set_async_wgrad(on: bool) -> bool:
    global _async_wgrad
    old, _async_wgrad = _async_wgrad, bool(on)
    return old


def _side_stream(dev) -> "torch.cuda.Stream":
    s = _side_streams.get(dev.index)
    if s is None:
        s = _side_streams[dev.index] = torch.cuda.Stream(dev)
    return s


def _join_side(dev) -> None:
    global _join_armed
    torch.cuda.current_stream(dev).wait_stream(_side_stream(dev))
    _pending.clear()
    _join_armed = False


def finish_async(dev) -> None:
    """join the side stream if a backward pass left it un-joined (it raised before the engine ran the callback)"""
    if _join_armed:
        _join_side(dev)


def _wgrad_async(dev, fn, keep):
    """run fn() (wgrad launches) on the side stream after everything queued so far; arm the end-of-backward join"""
    global _join_armed
    side = _side_stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        out = fn()
    # only the OPERANDS are parked: an extra reference to the gradient itself would make autograd's AccumulateGrad clone it
    # instead of adopting it -- a copy kernel on the calling stream, reading the gradient before the side stream has written it
    # (measured: exactly that race, the graph-captured step walked the weights differently from the eager one)
    _pending.append(keep)
    if os.environ.get("Y5_ASYNC_WGRAD_JOIN_NOW"):  # diagnostic: same streams, no concurrency
        torch.cuda.current_stream(dev).wait_stream(side)
    if not _join_armed:
        _join_armed = True
        torch.autograd.Variable._execution_engine.queue_callback(lambda: _join_side(dev))
    return out


def _bn_act_fwd(y, z_ptr: int, z_pitch: int, gamma, beta, running_mean, running_var, res: tuple, act, eps, momentum, training, pg):
    """z = act(BN(y)) + residual for the raw conv output y (dense NHWC): batch statistics in training (SyncBatchNorm's all-reduced
    ones when pg is set), running statistics otherwise.  z: element pointer and pitch of the output view; res: (pointer or None,
    pitch).  Returns (mean, invstd, gamma, beta as fp32, the all-rank row count or None) for _bn_act_bwd."""
    lib = _lib.lib()
    dev = y.device
    b, c, ho, wo = y.shape
    rows = b * ho * wo
    code = _lib.dtype_code(y.dtype)
    count = n_rows = None
    if training:
        mean = torch.empty(c, dtype=torch.float32, device=dev)
        invstd = torch.empty(c, dtype=torch.float32, device=dev)
        # the kernel updates fp32 running statistics in place; a model cast to fp16/bf16 goes through fp32 copies
        rm = running_mean if running_mean is None or running_mean.dtype == torch.float32 else running_mean.float()
        rv = running_var if running_var is None or running_var.dtype == torch.float32 else running_var.float()
        if pg is None:
            ws = _bn_ws(c, dev)
        else:  # SyncBatchNorm: [column sums | row count] of every rank in one all-reduce, then the statistics of all rows
            ws = _arena.take(2 * c + 1, dev)
            count = ws[2 * c :].data_ptr()
        _lib.check(lib.y5_bn_stats(y.data_ptr(), c, rows, c, code, ws.data_ptr(), count, _st(dev)), "bn_stats")
        if pg is not None:
            _all_reduce(ws[: 2 * c + 1], pg)
            n_rows = ws[2 * c : 2 * c + 1].clone()  # N for the backward: the arena is cleared by the next forward
        sums = ws.data_ptr()
    else:
        mean = running_mean.float().contiguous()
        invstd = torch.rsqrt(running_var.float() + eps)
        rm = rv = sums = None
    g32, b32 = gamma.detach().float().contiguous(), beta.detach().float().contiguous()
    _lib.check(lib.y5_bn_act_fwd(y.data_ptr(), c, z_ptr, z_pitch, rows, c, code, mean.data_ptr(), invstd.data_ptr(), g32.data_ptr(),
                                 b32.data_ptr(), *act, sums, count, eps, momentum, rm.data_ptr() if rm is not None else None,
                                 rv.data_ptr() if rv is not None else None, res[0], res[1], _st(dev)), "bn_act_fwd")
    if training:
        if rm is not running_mean:
            running_mean.copy_(rm)
        if rv is not running_var:
            running_var.copy_(rv)
    return mean, invstd, g32, b32, n_rows


def _bn_act_bwd(y, dz_ptr: int, dz_pitch: int, mean, invstd, g32, b32, act, pg, n_rows):
    """Backward of _bn_act_fwd in training: (dy like y, fp32 dgamma, fp32 dbeta) from the gradient view dz (pointer, pitch)."""
    lib = _lib.lib()
    dev = y.device
    b, c, ho, wo = y.shape
    rows = b * ho * wo
    code = _lib.dtype_code(y.dtype)
    dy = torch.empty_like(y)
    dgamma = torch.empty(c, dtype=torch.float32, device=dev)
    dbeta = torch.empty(c, dtype=torch.float32, device=dev)
    ws = _bn_ws(c, dev)
    if pg is None:
        _lib.check(lib.y5_bn_act_bwd(y.data_ptr(), c, dz_ptr, dz_pitch, dy.data_ptr(), c, rows, c, code, mean.data_ptr(),
                                     invstd.data_ptr(), g32.data_ptr(), b32.data_ptr(), *act, dgamma.data_ptr(), dbeta.data_ptr(),
                                     ws.data_ptr(), _st(dev)), "bn_act_bwd")
    else:  # SyncBatchNorm: dgamma / dbeta stay this rank's sums (DDP averages them); dy uses the sums of every rank over N
        _lib.check(lib.y5_bn_act_bwd_reduce(y.data_ptr(), c, dz_ptr, dz_pitch, dy.data_ptr(), c, rows, c, code, mean.data_ptr(),
                                            invstd.data_ptr(), g32.data_ptr(), b32.data_ptr(), *act, dgamma.data_ptr(),
                                            dbeta.data_ptr(), ws.data_ptr(), _st(dev)), "bn_act_bwd_reduce")
        _all_reduce(ws[: 2 * c], pg)
        _lib.check(lib.y5_bn_act_bwd_apply(y.data_ptr(), c, dz_ptr, dz_pitch, dy.data_ptr(), c, rows, c, code, mean.data_ptr(),
                                           invstd.data_ptr(), g32.data_ptr(), act[0], ws.data_ptr(), n_rows.data_ptr(),
                                           _st(dev)), "bn_act_bwd_apply")
    return dy, dgamma, dbeta


class _ConvBnAct(torch.autograd.Function):
    """z = act(BN(conv(x, w)))  with batch statistics (training) or running statistics (eval inside a training graph); act is
    engine.act_spec's (code, slope) pair."""

    @staticmethod
    def forward(ctx, x, weight, gamma, beta, running_mean, running_var, residual, k, s, p, act, eps, momentum, training, stem, pg=None):
        dev = x.device
        if stem == STEM_IMAGE:  # x is the image_input buffer; weight is the (O,3,k,k) filter, zero-padded to its channels
            w_eff, ke, se, pe = pad_image_weight(weight.detach()), k, s, p
        elif stem:  # x is already the 16-channel space-to-depth image; weight is the (O,3,6,6) stem filter
            fwd_idx, _ = _stem_index(dev)
            wf = weight.detach().flatten(1)
            w_eff = torch.cat((wf, wf.new_zeros(wf.shape[0], 1)), 1)[:, fwd_idx].view(-1, 16, 3, 3)
            ke, se, pe = 3, 1, 1
        else:
            w_eff, ke, se, pe = weight, k, s, p
        wide = stem == 2  # x is the (B, H/2, W/2 + 2, 16) zero-padded NHWC buffer of stem_input
        if wide:
            y = stem_conv_wide(x, w_eff)
            wp_dg, bk_d = None, 0
        else:
            x, xp = _nhwc(x)
            bsz, _, h, w_ = x.shape
            m_rows = bsz * ((h + 2 * pe - ke) // se + 1) * ((w_ + 2 * pe - ke) // se + 1)
            need_dx = ctx.needs_input_grad[0] and not stem
            hit = None
            if _cur_plan is not None and not stem and _cur_plan.dtype == x.dtype:
                bk_f = _block_k(w_eff.shape[1], w_eff.shape[0], m_rows)
                bk_d = _block_k(w_eff.shape[0], w_eff.shape[1], m_rows) if need_dx else 0
                hit = _cur_plan.lookup(weight, bk_f, bk_d, need_dx)
            if hit is not None:  # packed by this forward's y5_weight_pack_multi launch
                wp, wp_dg = hit
                if not need_dx:
                    wp_dg = None
            else:
                wp, wp_dg, bk_f, bk_d = pack_weights(w_eff, x.dtype, m_rows, True, need_dx)
                if _cur_plan is not None and not stem and _cur_plan.dtype == x.dtype and isinstance(weight, torch.nn.Parameter):
                    _cur_plan.register(weight, wp, wp_dg, wp.shape[3], wp_dg.shape[3] if wp_dg is not None else 0, bk_f, bk_d)
            y = conv_packed(x, xp, wp, bk_f, None, w_eff.shape[0], ke, se, pe, act=False)
        z = torch.empty_like(y)
        res = (None, 0) if residual is None else _nhwc(residual)
        mean, invstd, g32, b32, n_rows = _bn_act_fwd(y, z.data_ptr(), y.shape[1], gamma, beta, running_mean, running_var,
                                                     (res[0].data_ptr() if res[0] is not None else None, res[1]), act, eps, momentum,
                                                     training, pg)
        ctx.save_for_backward(x, weight, y, mean, invstd, g32, b32, wp_dg)
        ctx.cfg = (k, s, p, act, training, stem, ke, se, pe)
        ctx.bk_d = bk_d
        ctx.wide = wide
        ctx.pdtypes = (gamma.dtype, beta.dtype)
        ctx.pg, ctx.n_rows = pg, n_rows
        return z

    @staticmethod
    def backward(ctx, dz):
        x, weight, y, mean, invstd, g32, b32, wp_dg = ctx.saved_tensors
        k, s, p, act, training, stem, ke, se, pe = ctx.cfg
        if not training:
            raise NotImplementedError("y5b200: backward through eval-mode BatchNorm")
        dev = y.device
        dz_in = dz
        dz, dzp = _nhwc(dz if dz.dtype == y.dtype else dz.to(y.dtype))
        dy, dgamma, dbeta = _bn_act_bwd(y, dz.data_ptr(), dzp, mean, invstd, g32, b32, act, ctx.pg, ctx.n_rows)

        def wgrad():
            g = stem_wgrad_wide(x, dy) if ctx.wide else conv_wgrad(x, dy, ke, se, pe)
            if stem == STEM_IMAGE:  # the image buffer's padding channels carry no filter taps
                g = g[:, : weight.shape[1]].contiguous()
            elif stem:  # (O,16,3,3) gradient of the space-to-depth filter -> (O,3,6,6)
                _, inv_idx = _stem_index(dev)
                g = g.reshape(g.shape[0], -1)[:, inv_idx].view(weight.shape)
            return g.to(weight.dtype)

        # (an existing .grad would be accumulated into by autograd on the calling stream right after this function returns)
        dw = _wgrad_async(dev, wgrad, (x, dy)) if (_async_wgrad and weight.grad is None) else wgrad()
        dx = None
        if ctx.needs_input_grad[0]:
            if stem:
                raise NotImplementedError("y5b200: gradient w.r.t. the input image")
            dx = conv_dgrad(dy, None, k, s, p, (x.shape[2], x.shape[3]), wp_dgrad=wp_dg, cin=x.shape[1], block_k=ctx.bk_d)
        dres = dz_in if ctx.needs_input_grad[6] else None  # z = residual + act(bn(y)): the shortcut's gradient is dz itself
        return (dx, dw, dgamma.to(ctx.pdtypes[0]), dbeta.to(ctx.pdtypes[1]), None, None, dres, None, None, None, None, None,
                None, None, None, None)


class _GhostDw(torch.autograd.Function):
    """GhostConv's second half with its concat in training: out = cat(y + res[:, :c], act(BN(dw(y))) + res[:, c:]), dw the depthwise
    5x5 conv of GhostConv.cv2 and res an optional (B,2c,H,W) residual (GhostBottleneck's input).  One y5_dwconv_fwd launch writes
    the raw dw(y) and the first half; the BN passes of _ConvBnAct write the second half.  Backward: the BN backward gives d_raw,
    the same kernel with the taps rotated gives dy = dw^T(d_raw) + dout[:, :c] in one pass, and y5_dwconv_wgrad the weight
    gradient (on the side stream, as _ConvBnAct's)."""

    @staticmethod
    def forward(ctx, y, weight, gamma, beta, running_mean, running_var, residual, act, eps, momentum, training, pg=None):
        lib = _lib.lib()
        y, yp = _nhwc(y)
        b, c, h, w = y.shape
        dev, code = y.device, _lib.dtype_code(y.dtype)
        wp = torch.empty(c, 5, 5, 1, dtype=y.dtype, device=dev)  # [c][5][5]: the fp32 master filter rounded once
        wm = weight.detach().contiguous()
        _lib.check(lib.y5_weight_pack(wm.data_ptr(), _lib.dtype_code(wm.dtype), c, 1, 5, wp.data_ptr(), 1, None, 0, code, _st(dev)),
                   "weight_pack (depthwise)")
        out = _empty_cl(b, 2 * c, h, w, y.dtype, dev)
        raw = _empty_cl(b, c, h, w, y.dtype, dev)
        res, rp = (None, 0) if residual is None else _nhwc(residual)
        es = out.element_size()
        _lib.check(lib.y5_dwconv_fwd(y.data_ptr(), yp, wp.data_ptr(), None, raw.data_ptr(), c, None, 0, res.data_ptr() if res is not None else None,
                                     rp, out.data_ptr(), 2 * c, b, h, w, c, 5, 1, _lib.ACT_NONE, 0.0, 0, code, _st(dev)), "dwconv_fwd")
        mean, invstd, g32, b32, n_rows = _bn_act_fwd(raw, out.data_ptr() + c * es, 2 * c, gamma, beta, running_mean, running_var,
                                                     (res.data_ptr() + c * es if res is not None else None, rp), act, eps, momentum,
                                                     training, pg)
        ctx.save_for_backward(y, weight, raw, mean, invstd, g32, b32, wp)
        ctx.cfg = (act, training, pg, n_rows, gamma.dtype, beta.dtype)
        return out

    @staticmethod
    def backward(ctx, dout):
        lib = _lib.lib()
        y, weight, raw, mean, invstd, g32, b32, wp = ctx.saved_tensors
        act, training, pg, n_rows, gdt, bdt = ctx.cfg
        if not training:
            raise NotImplementedError("y5b200: backward through eval-mode BatchNorm")
        b, c, h, w = y.shape
        dev, code = y.device, _lib.dtype_code(y.dtype)
        dout_in = dout
        dout, dp = _nhwc(dout if dout.dtype == y.dtype else dout.to(y.dtype))
        es = dout.element_size()
        d_raw, dgamma, dbeta = _bn_act_bwd(raw, dout.data_ptr() + c * es, dp, mean, invstd, g32, b32, act, pg, n_rows)
        yp = _nhwc(y)[1]

        def wgrad():
            dw = torch.empty(c, 1, 5, 5, dtype=torch.float32, device=dev)
            _lib.check(lib.y5_dwconv_wgrad(y.data_ptr(), yp, d_raw.data_ptr(), c, dw.data_ptr(), b, h, w, c, 5, 1, code, _st(dev)),
                       "dwconv_wgrad")
            return dw.to(weight.dtype)

        dw = _wgrad_async(dev, wgrad, (y, d_raw)) if (_async_wgrad and weight.grad is None) else wgrad()
        dy = None
        if ctx.needs_input_grad[0]:
            dy = _empty_cl(b, c, h, w, y.dtype, dev)
            _lib.check(lib.y5_dwconv_fwd(d_raw.data_ptr(), c, wp.data_ptr(), None, dy.data_ptr(), c, dout.data_ptr(), dp, None, 0, None, 0,
                                         b, h, w, c, 5, 1, _lib.ACT_NONE, 0.0, 1, code, _st(dev)), "dwconv_fwd (data gradient)")
        dres = dout_in if ctx.needs_input_grad[6] else None  # out = ... + residual: the residual's gradient is dout itself
        return dy, dw, dgamma.to(gdt), dbeta.to(bdt), None, None, dres, None, None, None, None, None


def dwconv_module(m, y, residual=None):
    """GhostConv.cv2 (depthwise conv + BN + act) on y, concatenated after y, + residual: _GhostDw with conv_module's BN rules."""
    bn = getattr(m, "bn", None)
    if bn is None:
        raise RuntimeError("y5b200: cannot train a fused model (Conv without BatchNorm); build it unfused")
    act = act_spec(m.act)
    if bn.training and bn.track_running_stats and bn.num_batches_tracked is not None:
        bn.num_batches_tracked += 1
    mom = bn.momentum if bn.momentum is not None else 0.1
    return _GhostDw.apply(y, m.conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, residual, act, float(bn.eps), float(mom),
                          bn.training, bn_sync_group(bn))


def _ghost(m, x, residual=None):
    """GhostConv: cat(y, cv2(y)) + residual with y = cv1(x)."""
    from .models.common import ghost_dw_channels

    ghost_dw_channels(m)
    return dwconv_module(m.cv2, conv_module(m.cv1, x), residual)


class _ConvBias(torch.autograd.Function):
    """Detect.m[i]: 1x1 conv with bias, output channels padded to a multiple of 8; returns NHWC (B,H,W,Cpad)."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        x, _ = _nhwc(x)
        cout = weight.shape[0]
        cpad = (cout + 7) // 8 * 8
        wpad = torch.zeros(cpad, *weight.shape[1:], dtype=torch.float32, device=x.device)
        wpad[:cout] = weight.detach().float()
        bpad = torch.zeros(cpad, dtype=torch.float32, device=x.device)
        bpad[:cout] = bias.detach().float()
        y = conv_raw(x, wpad, bpad, 1, 1, 0, act=False)  # (B,cpad,H,W) channels_last
        ctx.save_for_backward(x, wpad)
        ctx.cout = cout
        ctx.wdtype, ctx.bdtype = weight.dtype, bias.dtype
        return y.permute(0, 2, 3, 1)  # NHWC view, dense

    @staticmethod
    def backward(ctx, dy_nhwc):
        lib = _lib.lib()
        x, wpad = ctx.saved_tensors
        cout = ctx.cout
        dy = _cl(dy_nhwc.to(x.dtype).permute(0, 3, 1, 2))
        b, cpad, h, w = dy.shape
        dev = x.device
        db = torch.empty(cpad, dtype=torch.float32, device=dev)
        ws = _bn_ws(cpad, dev)
        _lib.check(lib.y5_col_sum(dy.data_ptr(), cpad, b * h * w, cpad, _lib.dtype_code(dy.dtype), db.data_ptr(), ws.data_ptr(), _st(dev)),
                   "col_sum")
        dw = conv_wgrad(x, dy, 1, 1, 0)[:cout]
        dx = conv_dgrad(dy, wpad, 1, 1, 0, (h, w)) if ctx.needs_input_grad[0] else None
        return dx, dw.to(ctx.wdtype), db[:cout].to(ctx.bdtype)


class _Linear(torch.autograd.Function):
    """y = x W^T (+ bias) (+ residual) over the pixels of an NHWC (B,C,H,W) view: a 1x1 conv on the conv kernels, the residual
    added in its epilogue.  Backward: y5_conv_wgrad, the data-gradient conv and y5_col_sum, as _ConvBias does."""

    @staticmethod
    def forward(ctx, x, weight, bias, residual):
        x, xp = _nhwc(x)
        b, cin, h, w = x.shape
        cout = weight.shape[0]
        wp, _, bk, _ = pack_weights(weight.view(cout, cin, 1, 1), x.dtype, b * h * w)
        bias32 = _zero_bias(cout, x.device) if bias is None else bias.detach().float().contiguous()
        res, resp = (None, 0) if residual is None else _nhwc(residual)
        y = _empty_cl(b, cout, h, w, x.dtype, x.device)
        d = conv_desc(ConvInput(x.data_ptr(), xp, b, h, w, cin), wp, bias32, bk, y.data_ptr(), cout, 1, 1, 0, False, x.dtype,
                      res.data_ptr() if res is not None else None, resp)
        _lib.check(_lib.lib().y5_conv_bn_silu_fwd(C.byref(d), _st(x.device)), "linear")
        ctx.save_for_backward(x, weight)
        ctx.has_bias = bias is not None
        ctx.dtypes = (weight.dtype, bias.dtype if bias is not None else None)
        return y

    @staticmethod
    def backward(ctx, dy_in):
        x, weight = ctx.saved_tensors
        b, cin, h, w = x.shape
        cout = weight.shape[0]
        dy, dp = _nhwc(dy_in if dy_in.dtype == x.dtype else dy_in.to(x.dtype))
        dw = conv_wgrad(x, dy, 1, 1, 0).view(cout, cin).to(ctx.dtypes[0])
        db = None
        if ctx.has_bias:
            db = torch.empty(cout, dtype=torch.float32, device=x.device)
            _lib.check(_lib.lib().y5_col_sum(dy.data_ptr(), dp, b * h * w, cout, _lib.dtype_code(dy.dtype), db.data_ptr(),
                                             _bn_ws(cout, x.device).data_ptr(), _st(x.device)), "col_sum")
            db = db.to(ctx.dtypes[1])
        dx = conv_dgrad(dy, weight.view(cout, cin, 1, 1), 1, 1, 0, (h, w)) if ctx.needs_input_grad[0] else None
        return dx, dw, db, (dy_in if ctx.needs_input_grad[3] else None)


class _Attention(torch.autograd.Function):
    """Per image and head, softmax(q k^T / sqrt(dh)) v over the H*W tokens of NHWC (B,c,H,W) views (y5_attention_fwd, which
    saves the row logsumexp); the backward recomputes P from it (y5_attention_bwd) and returns dq, dk, dv as channel slices
    of one (B,3c,H,W) buffer."""

    @staticmethod
    def forward(ctx, q, k, v, heads, dh):
        q, k, v = (_cl(t) for t in (q, k, v))
        b, c, h, w = q.shape
        seq, dev = h * w, q.device
        o = _empty_cl(b, c, h, w, q.dtype, dev)
        lse = torch.empty(b * heads * seq, dtype=torch.float32, device=dev)
        _lib.check(_lib.lib().y5_attention_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), c, o.data_ptr(), c, lse.data_ptr(), b, seq, heads, dh,
                                               dh ** -0.5, _lib.dtype_code(q.dtype), _st(dev)), "attention_fwd")
        ctx.save_for_backward(q, k, v, o, lse)
        ctx.cfg = (heads, dh)
        return o

    @staticmethod
    def backward(ctx, do):
        q, k, v, o, lse = ctx.saved_tensors
        heads, dh = ctx.cfg
        b, c, h, w = q.shape
        seq, dev = h * w, q.device
        do = _cl(do if do.dtype == q.dtype else do.to(q.dtype))
        dqkv = _empty_cl(b, 3 * c, h, w, q.dtype, dev)
        delta = torch.empty(b * heads * seq, dtype=torch.float32, device=dev)
        p, es = dqkv.data_ptr(), dqkv.element_size()
        _lib.check(_lib.lib().y5_attention_bwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), c, o.data_ptr(), c, do.data_ptr(), c, lse.data_ptr(),
                                               delta.data_ptr(), p, p + c * es, p + 2 * c * es, 3 * c, b, seq, heads, dh, dh ** -0.5,
                                               _lib.dtype_code(q.dtype), _st(dev)), "attention_bwd")
        return dqkv[:, :c], dqkv[:, c : 2 * c], dqkv[:, 2 * c :], None, None


def _transformer(tb, x):
    """TransformerBlock (reference models/common.py:115-161) in training: nothing is folded, so every Linear, the in- and
    out-projections and the position embedding get their own gradients."""
    from .models.common import transformer_spec

    heads, dh = transformer_spec(tb, training=True)
    c = tb.c2
    x = _Linear.apply(x, tb.linear.weight, tb.linear.bias, x)  # p + linear(p)
    for layer in tb.tr:
        ma = layer.ma
        wi, bi = ma.in_proj_weight, ma.in_proj_bias
        q, k, v = (_Linear.apply(_Linear.apply(x, lin.weight, None, None), wi[i * c : (i + 1) * c], bi[i * c : (i + 1) * c], None)
                   for i, lin in enumerate((layer.q, layer.k, layer.v)))
        x = _Linear.apply(_Attention.apply(q, k, v, heads, dh), ma.out_proj.weight, ma.out_proj.bias, x)
        x = _Linear.apply(_Linear.apply(x, layer.fc1.weight, None, None), layer.fc2.weight, None, x)
    return x


# ---------------------------------------------------------------------------------------------------------------------
# module-level training forward
# ---------------------------------------------------------------------------------------------------------------------
def train_dtype(model) -> torch.dtype:
    """Activation dtype of the training forward: the autocast dtype when autocast is on (train.py:401), else the
    parameter dtype if the model was cast to fp16/bf16."""
    if torch.is_autocast_enabled("cuda"):
        dt = torch.get_autocast_dtype("cuda")
    else:
        dt = next(model.parameters()).dtype
    if dt not in (torch.float16, torch.bfloat16):
        raise RuntimeError("y5b200: the training forward computes in fp16/bf16 with fp32 statistics and weight gradients -- run it under "
                           "torch.autocast('cuda') (as reference train.py:401 does) or cast the model with .half()/.bfloat16()")
    return dt


def _all_reduce(t: torch.Tensor, pg) -> None:
    """SUM all-reduce of a slice of BN sums, ordered on the calling stream like the kernels around it"""
    import torch.distributed as dist

    dist.all_reduce(t, group=pg)


def bn_process_group(bn):
    """The group a torch.nn.SyncBatchNorm reduces over in training -- `bn.process_group` or WORLD -- when torch.distributed is
    initialised and that group has more than one rank; else None (plain BatchNorm2d, and every other BatchNorm, never syncs)."""
    if not isinstance(bn, torch.nn.SyncBatchNorm):
        return None
    import torch.distributed as dist

    if not (dist.is_available() and dist.is_initialized()):
        return None
    pg = bn.process_group or dist.group.WORLD
    return pg if dist.get_world_size(pg) > 1 else None


def bn_sync_group(bn):
    """torch.nn.SyncBatchNorm's rule for when it syncs: in training mode, with bn_process_group(bn) set.  Otherwise the layer
    is plain batch norm and takes the BatchNorm2d path, launch for launch."""
    return bn_process_group(bn) if bn.training else None


STEM_IMAGE = 3  # conv_module(stem=...): a plain first layer over the image_input buffer


def _check_conv(m, stem: int = 0):
    if m.conv.groups != 1 or m.conv.dilation[0] != 1:
        raise NotImplementedError("y5b200: grouped / dilated convolutions are outside the YOLOv5 n..x hot path")
    k, s, p = m.conv.kernel_size[0], m.conv.stride[0], m.conv.padding[0]
    if stem in (0, STEM_IMAGE) and (k, s, p) not in ((1, 1, 0), (3, 1, 1), (3, 2, 1)):
        raise NotImplementedError(f"y5b200: training conv k{k} s{s} p{p}")
    return k, s, p


def conv_module(m, x, stem: int = 0, residual=None):  # stem: 0 no, 1 space-to-depth 3x3x16, 2 wide-pixel 3x1x48, STEM_IMAGE
    bn = getattr(m, "bn", None)
    if bn is None:
        raise RuntimeError("y5b200: cannot train a fused model (Conv without BatchNorm); build it unfused")
    act = act_spec(m.act)
    k, s, p = _check_conv(m, stem)
    training = bn.training
    if training and bn.track_running_stats and bn.num_batches_tracked is not None:
        bn.num_batches_tracked += 1
    mom = bn.momentum if bn.momentum is not None else 0.1
    return _ConvBnAct.apply(x, m.conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, residual, k, s, p, act, float(bn.eps),
                            float(mom), training, stem, bn_sync_group(bn))


class _Upsample2x(torch.autograd.Function):
    """nn.Upsample(scale_factor=2, mode='nearest') (models/yolov5s.yaml:36,41) and its backward (sum of each 2x2 block)."""

    @staticmethod
    def forward(ctx, x):
        x, xp = _nhwc(x)
        b, c, h, w = x.shape
        y = _empty_cl(b, c, 2 * h, 2 * w, x.dtype, x.device)
        _lib.check(_lib.lib().y5_upsample2x(x.data_ptr(), xp, y.data_ptr(), c, b, h, w, c, _lib.dtype_code(x.dtype), _st(x.device)), "upsample2x")
        return y

    @staticmethod
    def backward(ctx, dy):
        dy, dp = _nhwc(dy)
        b, c, h2, w2 = dy.shape
        dx = _empty_cl(b, c, h2 // 2, w2 // 2, dy.dtype, dy.device)
        _lib.check(_lib.lib().y5_upsample2x_bwd(dy.data_ptr(), dp, dx.data_ptr(), c, b, h2 // 2, w2 // 2, c, _lib.dtype_code(dy.dtype),
                                                _st(dy.device)), "upsample2x_bwd")
        return dx


class _SppfPoolCat(torch.autograd.Function):
    """cat(a, m(a), m(m(a)), m(m(m(a)))) of SPPF (models/common.py:338-340), m = MaxPool2d(k, 1, k//2): one pooling launch
    writes the three pooled slices next to a copy of `a`; the backward routes gradients through the arg-max chain."""

    @staticmethod
    def forward(ctx, a, k):
        lib = _lib.lib()
        a, ap = _nhwc(a)
        b, c, h, w = a.shape
        code = _lib.dtype_code(a.dtype)
        cat = _empty_cl(b, 4 * c, h, w, a.dtype, a.device)
        es = cat.element_size()
        _lib.check(lib.y5_copy_view(a.data_ptr(), ap, cat.data_ptr(), 4 * c, b * h * w, c, code, _st(a.device)), "copy_view")
        _lib.check(lib.y5_sppf_pool(a.data_ptr(), ap, cat.data_ptr() + c * es, cat.data_ptr() + 2 * c * es, cat.data_ptr() + 3 * c * es, 4 * c,
                                    b, h, w, c, k, code, _st(a.device)), "sppf_pool")
        ctx.save_for_backward(cat)
        ctx.k = k
        return cat

    @staticmethod
    def backward(ctx, dcat):
        lib = _lib.lib()
        (cat,) = ctx.saved_tensors
        b, c4, h, w = cat.shape
        c = c4 // 4
        dcat, dp = _nhwc(dcat)
        da = _empty_cl(b, c, h, w, cat.dtype, cat.device)
        ws = torch.empty(3 * b * h * w * c, dtype=torch.float32, device=cat.device)
        _lib.check(lib.y5_sppf_pool_bwd(cat.data_ptr(), c4, dcat.data_ptr(), dp, da.data_ptr(), c, b, h, w, c, ctx.k, _lib.dtype_code(cat.dtype),
                                        ws.data_ptr(), _st(cat.device)), "sppf_pool_bwd")
        return da, None


class _SppPoolCat(_SppfPoolCat):
    """cat(a, mp_k(a), mp_2k-1(a), mp_3k-2(a)) of SPP: the forward is SPPF's (the pools compose exactly); the backward routes each
    pool's gradient to the first maximum of its own window of `a` (y5_spp_pool_bwd), as torch does, not through SPPF's chain."""

    @staticmethod
    def backward(ctx, dcat):
        lib = _lib.lib()
        (cat,) = ctx.saved_tensors
        b, c4, h, w = cat.shape
        c = c4 // 4
        dcat, dp = _nhwc(dcat)
        da = _empty_cl(b, c, h, w, cat.dtype, cat.device)
        ws = torch.empty(lib.y5_spp_bwd_workspace_bytes(b, h, w, c), dtype=torch.uint8, device=cat.device)
        _lib.check(lib.y5_spp_pool_bwd(cat.data_ptr(), c4, dcat.data_ptr(), dp, da.data_ptr(), c, b, h, w, c, ctx.k, _lib.dtype_code(cat.dtype),
                                       ws.data_ptr(), _st(cat.device)), "spp_pool_bwd")
        return da, None


class _MaxPool(torch.autograd.Function):
    """nn.MaxPool2d(2, 2, 0), or nn.ZeroPad2d((0, 1, 0, 1)) + nn.MaxPool2d(2, 1, 0) (mode: y5_maxpool2d's), forward and backward."""

    @staticmethod
    def forward(ctx, x, mode):
        x, xp = _nhwc(x)
        b, c, h, w = x.shape
        ho, wo = (h // 2, w // 2) if mode == _lib.POOL_K2S2 else (h, w)
        y = _empty_cl(b, c, ho, wo, x.dtype, x.device)
        _lib.check(_lib.lib().y5_maxpool2d(x.data_ptr(), xp, y.data_ptr(), c, b, h, w, c, mode, _lib.dtype_code(x.dtype), _st(x.device)),
                   "maxpool2d")
        ctx.save_for_backward(x)
        ctx.cfg = (xp, mode)
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        xp, mode = ctx.cfg
        b, c, h, w = x.shape
        dy, dp = _nhwc(dy if dy.dtype == x.dtype else dy.to(x.dtype))
        dx = _empty_cl(b, c, h, w, x.dtype, x.device)
        _lib.check(_lib.lib().y5_maxpool2d_bwd(x.data_ptr(), xp, dy.data_ptr(), dp, dx.data_ptr(), c, b, h, w, c, mode, _lib.dtype_code(x.dtype),
                                               _st(x.device)), "maxpool2d_bwd")
        return dx, None


class _Concat(torch.autograd.Function):
    """Channel concat (models/common.py:453) as strided slice copies; the backward hands out channel-slice views of the
    incoming gradient, which the consumers' kernels read in place through their pitch argument."""

    @staticmethod
    def forward(ctx, *xs):
        lib = _lib.lib()
        b, _, h, w = xs[0].shape
        cs = [x.shape[1] for x in xs]
        if any(c % 8 for c in cs):
            raise NotImplementedError(f"y5b200: concat of channel counts {cs} (multiples of 8 only)")
        out = _empty_cl(b, sum(cs), h, w, xs[0].dtype, xs[0].device)
        es, off = out.element_size(), 0
        for x, c in zip(xs, cs):
            x, xp = _nhwc(x)
            _lib.check(lib.y5_copy_view(x.data_ptr(), xp, out.data_ptr() + off * es, out.shape[1], b * h * w, c, _lib.dtype_code(out.dtype),
                                        _st(out.device)), "copy_view")
            off += c
        ctx.cs = cs
        return out

    @staticmethod
    def backward(ctx, dout):
        outs, off = [], 0
        for c in ctx.cs:
            outs.append(dout[:, off : off + c])
            off += c
        return tuple(outs)


class _GlobalAvgPool(torch.autograd.Function):
    """nn.AdaptiveAvgPool2d(1) of Classify (models/common.py:1140): (B,C,H,W) NHWC view -> (B,C,1,1) channels_last, summed in
    fp32 and rounded once (y5_global_avg_pool); the backward spreads dy / (H*W) over every pixel (y5_global_avg_pool_bwd)."""

    @staticmethod
    def forward(ctx, x):
        x, xp = _nhwc(x)
        b, c, h, w = x.shape
        y = _empty_cl(b, c, 1, 1, x.dtype, x.device)
        _lib.check(_lib.lib().y5_global_avg_pool(x.data_ptr(), xp, y.data_ptr(), c, b, h, w, c, _lib.dtype_code(x.dtype), _st(x.device)),
                   "global_avg_pool")
        ctx.hw = (h, w)
        return y

    @staticmethod
    def backward(ctx, dy):
        dy, dp = _nhwc(dy)
        b, c = dy.shape[:2]
        h, w = ctx.hw
        dx = _empty_cl(b, c, h, w, dy.dtype, dy.device)
        _lib.check(_lib.lib().y5_global_avg_pool_bwd(dy.data_ptr(), dp, dx.data_ptr(), c, b, h, w, c, _lib.dtype_code(dy.dtype), _st(dy.device)),
                   "global_avg_pool_bwd")
        return dx


def _classify(m, x):
    """Classify (models/common.py:1138-1140) in training: conv + batch-statistics BN + SiLU, pool, Linear as _ConvBias."""
    if isinstance(x, list):
        raise NotImplementedError("y5b200: Classify behind a Concat (list input) is outside the engine's hot path")
    if m.drop.p > 0 and m.drop.training:
        raise NotImplementedError("y5b200: Dropout(p > 0) in training is not implemented (its mask cannot follow torch's RNG); "
                                  "train with the reference default dropout_p=0.0")
    pooled = _GlobalAvgPool.apply(conv_module(m.conv, x))
    nc, cin = m.linear.weight.shape
    y = _ConvBias.apply(pooled, m.linear.weight.view(nc, cin, 1, 1), m.linear.bias)  # (B,1,1,ncpad) NHWC
    return y.reshape(y.shape[0], -1)[:, :nc]


def image_input(img: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """(B,3,H,W) uint8 / float image -> a (B,IMAGE_C,H,W) channels_last tensor, channels 3.. zero: the input of a plain first layer."""
    b, c, h, w = img.shape
    if c != 3:
        raise ValueError(f"y5b200: expected a (B,3,H,W) image batch, got {tuple(img.shape)}")
    out = _empty_cl(b, IMAGE_C, h, w, dtype, img.device)
    image_nhwc(img, out.permute(0, 2, 3, 1))
    return out


def stem_input(img: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """(B,3,H,W) uint8 / float image -> its space-to-depth cells (12 of 16 channels used): a stem_buffer for the wide-pixel stem,
    else a (B,16,H/2,W/2) channels_last tensor."""
    b, c, h, w = img.shape
    if c != 3 or h % 2 or w % 2:
        raise ValueError(f"y5b200: expected a (B,3,even,even) image batch, got {tuple(img.shape)}")
    if stem_wide_enabled():
        out = stem_buffer(b, h, w, dtype, img.device)
        stem_s2d(img, out)
        return out
    out = _empty_cl(b, 16, h // 2, w // 2, dtype, img.device)
    stem_s2d(img, out.permute(0, 2, 3, 1))
    return out


def _run(m, x, dt):
    from .models import common as mc
    from .models import yolo as my

    if isinstance(m, mc.Conv):
        return conv_module(m, x)
    if isinstance(m, mc.Bottleneck):  # the shortcut add rides on cv2's normalise+activate pass
        return conv_module(m.cv2, conv_module(m.cv1, x), residual=x if m.add else None)
    if isinstance(m, mc.GhostConv):
        return _ghost(m, x)
    if isinstance(m, mc.GhostBottleneck):  # cat(u, dw(u)) + x with u = g2.cv1(g1(x)): the add rides the depthwise pass, as in eval
        g1, g2 = mc.ghost_bottleneck_convs(m)
        return _ghost(g2, _ghost(g1, x), residual=x)
    if isinstance(m, mc.C3TR):
        return conv_module(m.cv3, _Concat.apply(_transformer(m.m, conv_module(m.cv1, x)), conv_module(m.cv2, x)))
    if isinstance(m, mc.C3):
        a = conv_module(m.cv1, x)
        for bt in m.m:
            a = _run(bt, a, dt)
        return conv_module(m.cv3, _Concat.apply(a, conv_module(m.cv2, x)))
    if isinstance(m, mc.SPPF):
        k = m.m.kernel_size if isinstance(m.m.kernel_size, int) else m.m.kernel_size[0]
        return conv_module(m.cv2, _SppfPoolCat.apply(conv_module(m.cv1, x), k))
    if isinstance(m, mc.SPP):
        return conv_module(m.cv2, _SppPoolCat.apply(conv_module(m.cv1, x), mc.spp_kernel(m)))
    if isinstance(m, torch.nn.Upsample):
        if float(m.scale_factor) != 2.0 or m.mode != "nearest":
            raise NotImplementedError("y5b200: only nn.Upsample(scale_factor=2, mode='nearest')")
        return _Upsample2x.apply(x)
    if isinstance(m, mc.Concat):
        if m.d != 1:
            raise NotImplementedError("y5b200: Concat along a dimension other than channels")
        return _Concat.apply(*x)
    if isinstance(m, mc.Proto):
        return conv_module(m.cv3, conv_module(m.cv2, _Upsample2x.apply(conv_module(m.cv1, x))))
    if isinstance(m, torch.nn.Sequential):
        for sub in m:
            x = _run(sub, x, dt)
        return x
    if isinstance(m, mc.Classify):
        return _classify(m, x)
    if isinstance(m, my.Detect):
        outs = []
        for i, xi in enumerate(x):
            yi = _ConvBias.apply(xi, m.m[i].weight, m.m[i].bias)  # (B,ny,nx,cpad)
            b, ny, nx, _ = yi.shape
            outs.append(yi[..., : m.na * m.no].reshape(b, ny, nx, m.na, m.no).permute(0, 3, 1, 2, 4).contiguous())
        if isinstance(m, my.Segment):
            return outs, _run(m.proto, x[0], dt)
        return outs
    raise NotImplementedError(f"y5b200: module {type(m).__name__} is outside the engine's hot path")


_grouped_checked: "weakref.WeakKeyDictionary" = weakref.WeakKeyDictionary()  # model -> ids of the layer list check_grouped_convs passed


def forward_train(model, img: torch.Tensor):
    """Training-mode DetectionModel / SegmentationModel forward: list of raw (B,na,ny,nx,no) maps (Segment: (list, proto)),
    differentiable w.r.t. every parameter."""
    from .models import common as mc

    dt = train_dtype(model)
    layers = list(model.model)
    first = layers[0]
    if not (isinstance(first, mc.Conv) and first.conv.in_channels == 3):
        raise NotImplementedError("y5b200: the first layer must be a Conv reading the 3-channel image")
    stem = is_v6_stem(first)
    if not stem:
        _check_conv(first, STEM_IMAGE)
    pools = mc.pool_modes(layers, model.save)  # every refusal before the first launch
    key = tuple(map(id, layers))  # the walk over every module costs ~0.5 ms: once per layer list (the lowerings check again)
    if _grouped_checked.get(model) != key:
        mc.check_grouped_convs(model)
        _grouped_checked[model] = key
    # every op below picks its dtype explicitly; autocast's own casting rules must not touch the glue ops
    global _cur_plan
    with torch.autocast("cuda", enabled=False):
        _arena.reset(img.device)
        _cur_plan = pack_plan(model, dt, img.device) if pack_plan_enabled() else None
        try:
            if _cur_plan is not None:
                _cur_plan.begin()  # every registered filter -> forward / data-gradient packings, one launch
            ys = []
            x = None
            for i, m in enumerate(layers):
                if i == 0 and stem:
                    x = conv_module(m, stem_input(img, dt), stem=2 if stem_wide_enabled() else 1)
                elif i == 0:
                    x = conv_module(m, image_input(img, dt), stem=STEM_IMAGE)
                else:
                    if m.f != -1:
                        x = ys[m.f] if isinstance(m.f, int) else [x if j == -1 else ys[j] for j in m.f]
                    if isinstance(m, torch.nn.MaxPool2d):
                        x = _MaxPool.apply(x, pools[i])
                    elif not isinstance(m, torch.nn.ZeroPad2d):  # a ZeroPad2d runs inside the max-pool after it
                        x = _run(m, x, dt)
                ys.append(x if i in model.save else None)
        finally:
            _cur_plan = None
    return x
