"""Layer zoo of the hot path with the reference's class names, constructor signatures, attribute names and
state_dict keys (reference models/common.py:62-92,115-181,230-270,318-340,443-453,1104-1140), so checkpoints and
state_dicts move between the two unchanged.  The modules only *hold* parameters: executing one (``forward``) lowers it
to liby5b200 kernels through yolov5_b200.engine.Program (eval) or yolov5_b200.train_ops (training: batch-statistics
BatchNorm, autograd) -- there is no torch.nn convolution behind them and CPU tensors are rejected.
"""
from __future__ import annotations

import torch
from torch import nn


def autopad(k, p=None, d=1):
    """'same' padding for kernel k (dilation d); reference models/common.py:62-71."""
    if d > 1:
        k = d * (k - 1) + 1 if isinstance(k, int) else [d * (x - 1) + 1 for x in k]
    if p is None:
        p = k // 2 if isinstance(k, int) else [x // 2 for x in k]
    return p


class _EngineLayer(nn.Module):
    """Runs a single layer through a cached single-layer Program (keyed by input shape / dtype / training flag)."""

    def _engine_forward(self, x: torch.Tensor) -> torch.Tensor:
        from ..engine import Program

        if not (isinstance(x, torch.Tensor) and x.is_cuda):
            raise RuntimeError(
                f"y5b200: {type(self).__name__} executes only on CUDA tensors through liby5b200 (no CPU/PyTorch fallback)"
            )
        if self.training:  # batch-statistics BatchNorm + autograd: yolov5_b200/train_ops.py
            from ..train_ops import _run, train_dtype

            dt = train_dtype(self)
            with torch.autocast("cuda", enabled=False):
                return _run(self, x.to(dt), dt)
        key = (tuple(x.shape), x.dtype, x.device.index, _param_version(self))
        b, c, h, w = x.shape
        with _lib_on(x.device):
            return _cached_program(self, key, lambda: Program(self, b, h, w, x.dtype, x.device, in_channels=c)).run_layer(x)

    def forward(self, x):
        return self._engine_forward(x)

    def __getstate__(self):  # programs hold raw pointers: never pickle them (checkpoints pickle whole modules)
        d = self.__dict__.copy()
        d.pop("_y5_programs", None)
        d.pop("_y5_tensors", None)
        d.pop("_y5_pack_plans", None)  # persistent packed-weight buffers of the training path (train_ops.PackPlan)
        return d

    def _apply(self, fn, *a, **k):
        _drop_engine_cache(self)
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        _drop_engine_cache(self)
        return super().load_state_dict(*a, **k)


def _lib_on(device):
    from .. import _lib

    return _lib.on(device)


def _param_version(m: nn.Module) -> int:
    """In-place edits of parameters / buffers (optimizer steps, BN statistics, manual surgery) invalidate the packed weights
    of a cached Program.  The tensor list is gathered once per module (walking ~350 sub-modules per forward cost more than the
    yolov5n forward itself); `_apply` / `load_state_dict` / `fuse` drop it together with the programs."""
    ts = m.__dict__.get("_y5_tensors")
    if ts is None:
        ts = m.__dict__["_y5_tensors"] = list(m.parameters()) + list(m.buffers())
    v = 0
    for t in ts:
        v += t._version
    return v


def _drop_engine_cache(m: nn.Module) -> None:
    m.__dict__.pop("_y5_programs", None)
    m.__dict__.pop("_y5_tensors", None)


PROGRAM_CACHE = 8  # cached Programs per module (least recently used one is dropped)


def _cached_program(m: nn.Module, key, build):
    from collections import OrderedDict

    cache = m.__dict__.get("_y5_programs")
    if cache is None:
        cache = m.__dict__["_y5_programs"] = OrderedDict()
    prog = cache.get(key)
    if prog is None:
        # programs of an older parameter version can never be hit again: drop them first
        for k in [k for k in cache if k[-1] != key[-1]]:
            del cache[k]
        while len(cache) >= PROGRAM_CACHE:
            cache.popitem(last=False)
        prog = cache[key] = build()
    else:
        cache.move_to_end(key)
    return prog


class Conv(_EngineLayer):
    """conv(bias=False) -> BatchNorm2d -> SiLU, executed as one fused kernel."""

    default_act = nn.SiLU()

    def __init__(self, c1, c2, k=1, s=1, p=None, g=1, d=1, act=True):
        super().__init__()
        self.conv = nn.Conv2d(c1, c2, k, s, autopad(k, p, d), groups=g, dilation=d, bias=False)
        self.bn = nn.BatchNorm2d(c2)
        self.act = self.default_act if act is True else act if isinstance(act, nn.Module) else nn.Identity()

    def forward_fuse(self, x):
        return self._engine_forward(x)


class Bottleneck(_EngineLayer):
    def __init__(self, c1, c2, shortcut=True, g=1, e=0.5):
        super().__init__()
        c_ = int(c2 * e)
        self.cv1 = Conv(c1, c_, 1, 1)
        self.cv2 = Conv(c_, c2, 3, 1, g=g)
        self.add = shortcut and c1 == c2


class C3(_EngineLayer):
    def __init__(self, c1, c2, n=1, shortcut=True, g=1, e=0.5):
        super().__init__()
        c_ = int(c2 * e)
        self.cv1 = Conv(c1, c_, 1, 1)
        self.cv2 = Conv(c1, c_, 1, 1)
        self.cv3 = Conv(2 * c_, c2, 1)
        self.m = nn.Sequential(*(Bottleneck(c_, c_, shortcut, g, e=1.0) for _ in range(n)))


class TransformerLayer(nn.Module):
    """x = ma(q(x), k(x), v(x)) + x;  x = fc2(fc1(x)) + x  (no LayerNorm, no activation).  `ma` is a real nn.MultiheadAttention
    because it holds the in- and out-projection parameters under the reference's keys; its forward never runs: the layer is
    lowered inside C3TR (engine: folded GEMMs around y5_attention_fwd; training: train_ops)."""

    def __init__(self, c, num_heads):
        super().__init__()
        self.q = nn.Linear(c, c, bias=False)
        self.k = nn.Linear(c, c, bias=False)
        self.v = nn.Linear(c, c, bias=False)
        self.ma = nn.MultiheadAttention(embed_dim=c, num_heads=num_heads)
        self.fc1 = nn.Linear(c, c, bias=False)
        self.fc2 = nn.Linear(c, c, bias=False)

    def forward(self, x):
        raise RuntimeError("y5b200: TransformerLayer runs inside C3TR (GEMMs and y5_attention kernels)")


class TransformerBlock(nn.Module):
    """Learnable position embedding p + linear(p) followed by `num_layers` TransformerLayers over the H*W tokens of each image.
    `conv` exists only when c1 != c2 (as in the reference); no model dict builds that case and the engine refuses it."""

    def __init__(self, c1, c2, num_heads, num_layers):
        super().__init__()
        self.conv = None
        if c1 != c2:
            self.conv = Conv(c1, c2)
        self.linear = nn.Linear(c2, c2)  # learnable position embedding
        self.tr = nn.Sequential(*(TransformerLayer(c2, num_heads) for _ in range(num_layers)))
        self.c2 = c2

    def forward(self, x):
        raise RuntimeError("y5b200: TransformerBlock runs inside C3TR (GEMMs and y5_attention kernels)")


ATTN_HEAD_DIMS = (32, 64, 96, 128, 160)  # the head dims y5_attention_fwd / _bwd are built for


def transformer_spec(tb: TransformerBlock, training: bool) -> tuple[int, int]:
    """(heads, head dim) of a TransformerBlock the kernels run; NotImplementedError naming any other configuration."""
    if tb.conv is not None:
        raise NotImplementedError("y5b200: TransformerBlock with c1 != c2 (its input Conv) is not built; C3TR never creates one")
    heads = dh = None
    for j, layer in enumerate(tb.tr):
        ma = layer.ma
        if not isinstance(ma, nn.MultiheadAttention):
            raise NotImplementedError(f"y5b200: TransformerLayer {j}: attention module {type(ma).__name__}")
        if (not ma._qkv_same_embed_dim or ma.batch_first or ma.bias_k is not None or ma.add_zero_attn or ma.in_proj_bias is None
                or ma.out_proj.bias is None or ma.embed_dim != tb.c2):
            raise NotImplementedError(f"y5b200: TransformerLayer {j}: nn.MultiheadAttention configuration (kdim/vdim != embed_dim, "
                                      "batch_first, add_bias_kv, add_zero_attn or no bias) outside nn.MultiheadAttention(c, heads)")
        if ma.head_dim not in ATTN_HEAD_DIMS:
            raise NotImplementedError(f"y5b200: attention head dim {ma.head_dim} (built: {ATTN_HEAD_DIMS})")
        if training and ma.dropout > 0:
            raise NotImplementedError(f"y5b200: attention dropout {ma.dropout} in training (its mask cannot follow torch's RNG)")
        if heads is not None and (ma.num_heads, ma.head_dim) != (heads, dh):
            raise NotImplementedError("y5b200: TransformerLayers with different head counts in one block")
        heads, dh = ma.num_heads, ma.head_dim
    if tb.linear.bias is None:
        raise NotImplementedError("y5b200: TransformerBlock position embedding without bias")
    return heads, dh


class C3TR(C3):
    """C3 whose `m` is a TransformerBlock(c_, c_, 4, n) (reference models/common.py:261-270)."""

    def __init__(self, c1, c2, n=1, shortcut=True, g=1, e=0.5):
        super().__init__(c1, c2, n, shortcut, g, e)
        c_ = int(c2 * e)
        self.m = TransformerBlock(c_, c_, 4, n)


class GhostConv(_EngineLayer):
    """cat(y, cv2(y)) with y = cv1(x) (reference models/common.py GhostConv): cv2 is the depthwise 5x5 conv Conv(c_, c_, 5, 1,
    None, c_), which runs on y5_dwconv_fwd.  Not a Conv subclass, as in the reference, so isinstance tests and state_dict keys
    (cv1.*, cv2.*) behave the same."""

    def __init__(self, c1, c2, k=1, s=1, g=1, act=True):
        super().__init__()
        c_ = c2 // 2
        self.cv1 = Conv(c1, c_, k, s, None, g, act=act)
        self.cv2 = Conv(c_, c_, 5, 1, None, c_, act=act)


class GhostBottleneck(_EngineLayer):
    """conv(x) + x with conv = GhostConv(c1, c2 // 2) -> Identity -> GhostConv(c2 // 2, c2, act=False) (reference models/common.py
    GhostBottleneck).  The stride-2 form puts a depthwise k x k conv in both branches; it is built here for its state_dict keys
    (the reference's DWConv holds conv / bn / act like Conv), and the engine refuses it: no reference model dict uses it."""

    def __init__(self, c1, c2, k=3, s=1):
        super().__init__()
        c_ = c2 // 2
        self.conv = nn.Sequential(GhostConv(c1, c_, 1, 1), Conv(c_, c_, k, s, g=c_, act=False) if s == 2 else nn.Identity(),
                                  GhostConv(c_, c2, 1, 1, act=False))
        self.shortcut = (nn.Sequential(Conv(c1, c1, k, s, g=c1, act=False), Conv(c1, c2, 1, 1, act=False)) if s == 2 else nn.Identity())


class C3Ghost(C3):
    """C3 whose `m` is a chain of GhostBottleneck(c_, c_) (reference models/common.py C3Ghost).  Like the reference it ignores
    `shortcut`: every GhostBottleneck adds its input."""

    def __init__(self, c1, c2, n=1, shortcut=True, g=1, e=0.5):
        super().__init__(c1, c2, n, shortcut, g, e)
        c_ = int(c2 * e)
        self.m = nn.Sequential(*(GhostBottleneck(c_, c_) for _ in range(n)))


def ghost_dw_channels(m: GhostConv) -> int:
    """Channel count of a GhostConv's depthwise half when y5_dwconv runs it: Conv2d(c, c, 5, 1, 2, groups=c) with c a multiple
    of 8; NotImplementedError naming the configuration otherwise."""
    d = m.cv2.conv
    c = d.in_channels
    if not (d.out_channels == c == d.groups and tuple(d.kernel_size) == (5, 5) and tuple(d.stride) == (1, 1)
            and tuple(d.padding) == (2, 2) and tuple(d.dilation) == (1, 1)):
        raise NotImplementedError(f"y5b200: GhostConv.cv2 {d!r} (built: the depthwise Conv2d(c, c, 5, 1, 2, groups=c))")
    if c % 8:
        raise NotImplementedError(f"y5b200: GhostConv with a depthwise conv of {c} channels (built: multiples of 8)")
    if m.cv1.conv.out_channels != c:
        raise NotImplementedError(f"y5b200: GhostConv whose cv1 gives {m.cv1.conv.out_channels} channels to a {c}-channel cv2")
    return c


def ghost_bottleneck_convs(m: GhostBottleneck) -> tuple[GhostConv, GhostConv]:
    """The two GhostConvs of a stride-1 GhostBottleneck; NotImplementedError for the stride-2 form."""
    if not (isinstance(m.conv[1], nn.Identity) and isinstance(m.shortcut, nn.Identity)):
        raise NotImplementedError("y5b200: GhostBottleneck(s=2) (built: the stride-1 form that C3Ghost uses)")
    return m.conv[0], m.conv[2]


def check_grouped_convs(root: nn.Module) -> None:
    """Refuse, before anything runs, every grouped convolution the kernels do not build: any GhostBottleneck other than the
    stride-1 form, any GhostConv whose cv2 is not the 5x5 depthwise conv, and every other Conv2d with groups != 1."""
    built = set()
    for name, m in root.named_modules():
        if isinstance(m, GhostBottleneck):
            ghost_bottleneck_convs(m)
        elif isinstance(m, GhostConv):
            ghost_dw_channels(m)
            built.add(id(m.cv2.conv))
    for name, m in root.named_modules():
        if isinstance(m, nn.Conv2d) and m.groups != 1 and id(m) not in built:
            raise NotImplementedError(f"y5b200: grouped convolution '{name}' {m!r} (built: only GhostConv's depthwise 5x5 conv)")


class SPPF(_EngineLayer):
    def __init__(self, c1, c2, k=5):
        super().__init__()
        c_ = c1 // 2
        self.cv1 = Conv(c1, c_, 1, 1)
        self.cv2 = Conv(c_ * 4, c2, 1, 1)
        self.m = nn.MaxPool2d(kernel_size=k, stride=1, padding=k // 2)


class SPP(_EngineLayer):
    """Spatial pyramid pooling of yolov3-spp (reference models/common.py SPP): cv2(cat(x, mp_k0(x), mp_k1(x), mp_k2(x))) with
    x = cv1(input) and stride-1 'same' max-pools.  The engine runs k = (k, 2k-1, 3k-2) -- the default (5, 9, 13) -- because
    those pools are SPPF's chain mp_k, mp_k^2, mp_k^3 exactly; spp_kernel refuses any other k."""

    def __init__(self, c1, c2, k=(5, 9, 13)):
        super().__init__()
        c_ = c1 // 2
        self.cv1 = Conv(c1, c_, 1, 1)
        self.cv2 = Conv(c_ * (len(k) + 1), c2, 1, 1)
        self.m = nn.ModuleList([nn.MaxPool2d(kernel_size=x, stride=1, padding=x // 2) for x in k])


def _pool_arg(v):
    return v if isinstance(v, int) else (v[0] if len(set(v)) == 1 else None)


def maxpool_form(m: nn.MaxPool2d) -> tuple[int, int, int] | None:
    """(kernel, stride, padding) of a square, undilated nn.MaxPool2d without ceil_mode / return_indices, else None."""
    k, s, p, d = (_pool_arg(m.kernel_size), _pool_arg(m.stride if m.stride is not None else m.kernel_size), _pool_arg(m.padding),
                  _pool_arg(m.dilation))
    if None in (k, s, p) or d != 1 or m.ceil_mode or m.return_indices:
        return None
    return k, s, p


def spp_kernel(m: SPP) -> int:
    """SPPF kernel size k of an SPP whose pools are stride-1 'same' max-pools of sizes (k, 2k-1, 3k-2), k odd; NotImplementedError
    naming the configuration otherwise."""
    forms = [maxpool_form(p) if isinstance(p, nn.MaxPool2d) else None for p in m.m]
    if len(forms) == 3 and None not in forms:
        k = forms[0][0]
        if k % 2 and forms == [(k, 1, k // 2), (2 * k - 1, 1, k - 1), (3 * k - 2, 1, 3 * (k // 2))]:
            return k
    raise NotImplementedError(f"y5b200: SPP pools {[p for p in m.m]} (built: three stride-1 'same' max-pools of sizes k, 2k-1, 3k-2, "
                              "k odd, such as (5, 9, 13))")


def pool_mode(m: nn.MaxPool2d, pad: nn.ZeroPad2d | None) -> int:
    """y5_maxpool2d mode of nn.MaxPool2d(2, 2, 0), or of nn.ZeroPad2d((0, 1, 0, 1)) followed by nn.MaxPool2d(2, 1, 0) (yolov3-tiny);
    NotImplementedError naming any other pool or pad."""
    from .. import _lib

    form = maxpool_form(m)
    if pad is None and form == (2, 2, 0):
        return _lib.POOL_K2S2
    if pad is not None and form == (2, 1, 0):
        if tuple(pad.padding) == (0, 1, 0, 1):
            return _lib.POOL_K2S1_ZPAD
        raise NotImplementedError(f"y5b200: {pad!r} before a max-pool (built: nn.ZeroPad2d((0, 1, 0, 1)))")
    raise NotImplementedError(f"y5b200: {m!r}{' after ' + repr(pad) if pad is not None else ''} (built: nn.MaxPool2d(2, 2, 0), and "
                              "nn.MaxPool2d(2, 1, 0) after nn.ZeroPad2d((0, 1, 0, 1)); no ceil_mode, dilation or return_indices)")


def pool_modes(layers, save) -> dict[int, int]:
    """y5_maxpool2d mode of every nn.MaxPool2d in a model's layer list.  Checks, before anything runs, that each nn.ZeroPad2d
    feeds only the max-pool right after it (the pair runs as one kernel, so nothing else may read the padded map) and that
    every SPP has pools the engine builds; NotImplementedError naming the layer otherwise."""
    modes = {}
    for i, m in enumerate(layers):
        if isinstance(m, nn.ZeroPad2d):
            nxt = layers[i + 1] if i + 1 < len(layers) else None
            if not (isinstance(nxt, nn.MaxPool2d) and nxt.f == -1) or i in save:
                raise NotImplementedError(f"y5b200: layer {i} {m!r} must feed only an nn.MaxPool2d(2, 1, 0) right after it")
        elif isinstance(m, nn.MaxPool2d):
            pad = layers[i - 1] if i > 0 and m.f == -1 and isinstance(layers[i - 1], nn.ZeroPad2d) else None
            modes[i] = pool_mode(m, pad)
        elif isinstance(m, SPP):
            spp_kernel(m)
    return modes


class Concat(nn.Module):
    """Channel concatenation.  Inside a model it costs nothing (producers write into slices of one buffer); called on
    its own it has no arithmetic to offload and simply concatenates."""

    def __init__(self, dimension=1):
        super().__init__()
        self.d = dimension

    def forward(self, x):
        return torch.cat(x, self.d)


class Proto(_EngineLayer):
    """Segmentation prototype branch: Conv3x3 -> 2x nearest upsample -> Conv3x3 -> Conv1x1."""

    def __init__(self, c1, c_=256, c2=32):
        super().__init__()
        self.cv1 = Conv(c1, c_, k=3)
        self.upsample = nn.Upsample(scale_factor=2, mode="nearest")
        self.cv2 = Conv(c_, c_, k=3)
        self.cv3 = Conv(c_, c2)


class Classify(nn.Module):
    """Classification head (reference models/common.py:1120-1140): Conv(c1, 1280) -> global average pool -> Dropout ->
    Linear(1280, c2).  Inside ClassificationModel.forward it runs as conv_gemm + y5_global_avg_pool + conv_gemm (the Linear
    as a 1x1 conv with bias); Dropout is the identity in eval, and p > 0 is refused in training."""

    def __init__(self, c1, c2, k=1, s=1, p=None, g=1, dropout_p=0.0):
        super().__init__()
        c_ = 1280  # efficientnet_b0 size
        self.conv = Conv(c1, c_, k, s, autopad(k, p), g)
        self.pool = nn.AdaptiveAvgPool2d(1)
        self.drop = nn.Dropout(p=dropout_p, inplace=True)
        self.linear = nn.Linear(c_, c2)

    def forward(self, x):
        raise RuntimeError("y5b200: Classify runs inside ClassificationModel.forward (conv, pool and linear as liby5b200 kernels)")
