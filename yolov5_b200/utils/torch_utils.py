"""Hot-path edges of the reference's utils/torch_utils.py: BatchNorm folding, the DDP wrapper, the fused optimizers and EMA,
and the classification helpers (smartCrossEntropyLoss, reshape_classifier_output)."""
from __future__ import annotations

import ctypes as C
import math
import os
from copy import deepcopy

import torch
from torch import nn

from .. import _lib


def fuse_conv_and_bn(conv: nn.Conv2d, bn: nn.BatchNorm2d) -> nn.Conv2d:
    """Conv2d + eval BatchNorm2d -> one Conv2d with bias; same algebra as reference utils/torch_utils.py:224-254
    (W' = diag(g / sqrt(var + eps)) W,  b' = beta + (b - mean) g / sqrt(var + eps))."""
    fused = nn.Conv2d(conv.in_channels, conv.out_channels, conv.kernel_size, conv.stride, conv.padding, conv.dilation,
                      conv.groups, bias=True).requires_grad_(False).to(conv.weight.device, conv.weight.dtype)
    scale = bn.weight / torch.sqrt(bn.running_var + bn.eps)
    fused.weight.copy_(conv.weight * scale.view(-1, 1, 1, 1))
    b0 = conv.bias if conv.bias is not None else torch.zeros_like(scale)
    fused.bias.copy_(bn.bias + (b0 - bn.running_mean) * scale)
    return fused


def smartCrossEntropyLoss(label_smoothing=0.0):
    """nn.CrossEntropyLoss(label_smoothing=...) as reference utils/torch_utils.py:52-57 returns it, on the engine's
    y5_cross_entropy kernel (yolov5_b200.utils.loss.CrossEntropyLoss, an nn.CrossEntropyLoss subclass)."""
    from .loss import CrossEntropyLoss

    return CrossEntropyLoss(label_smoothing=label_smoothing)


def reshape_classifier_output(model, n=1000):
    """Give the last layer `n` outputs (reference utils/torch_utils.py:72-93) for a Classify head or a plain nn.Linear, and drop
    the engine caches: the cached Programs and the parameter list behind _param_version still name the replaced Linear."""
    from ..models.common import Classify, _drop_engine_cache

    name, m = list((model.model if hasattr(model, "model") else model).named_children())[-1]
    if isinstance(m, Classify):
        if m.linear.out_features != n:
            m.linear = nn.Linear(m.linear.in_features, n)
    elif isinstance(m, nn.Linear):
        if m.out_features != n:
            setattr(model, name, nn.Linear(m.in_features, n))
    elif isinstance(m, nn.Sequential):
        types = [type(x) for x in m]
        if nn.Linear in types:
            i = len(types) - 1 - types[::-1].index(nn.Linear)
            if m[i].out_features != n:
                m[i] = nn.Linear(m[i].in_features, n)
        elif nn.Conv2d in types:
            i = len(types) - 1 - types[::-1].index(nn.Conv2d)
            if m[i].out_channels != n:
                m[i] = nn.Conv2d(m[i].in_channels, n, m[i].kernel_size, m[i].stride, bias=m[i].bias is not None)
    for mod in model.modules():
        _drop_engine_cache(mod)


def smart_DDP(model):
    """The path's one collective: gradient all-reduce through DistributedDataParallel over NCCL
    (reference utils/torch_utils.py:61-70)."""
    from torch.nn.parallel import DistributedDataParallel as DDP

    local_rank = int(os.getenv("LOCAL_RANK", -1))
    return DDP(model, device_ids=[local_rank], output_device=local_rank, static_graph=True)


def de_parallel(model):
    return model.module if isinstance(model, (nn.parallel.DataParallel, nn.parallel.DistributedDataParallel)) else model


def copy_attr(a, b, include=(), exclude=()):
    """Copy attributes b -> a (ultralytics.utils.torch_utils.copy_attr, used by ModelEMA.update_attr)."""
    for k, v in b.__dict__.items():
        if (len(include) and k not in include) or k.startswith("_") or k in exclude:
            continue
        setattr(a, k, v)


_OPT_DTYPE = None


def _opt_dtype():
    """numpy mirror of y5_opt_tensor (include/y5b200.h; layout checked against gcc by tests/test_abi.py)."""
    global _OPT_DTYPE
    if _OPT_DTYPE is None:
        import numpy as np

        _OPT_DTYPE = np.dtype([("param", "<u8"), ("grad", "<u8"), ("mom", "<u8"), ("ema", "<u8"), ("numel", "<i8"), ("group", "<i4"),
                               ("reserved", "<i4")])
        assert _OPT_DTYPE.itemsize == C.sizeof(_lib.OptTensor)
    return _OPT_DTYPE


class _OptTable:
    """Device-side description of a set of tensors for y5_opt_step: one y5_opt_tensor per tensor and the (tensor, chunk) list
    that maps thread blocks to 16K-element pieces.  The host copy lives in pinned memory so that the gradient-pointer column
    can be refreshed and re-uploaded per step without a synchronisation (gradients are fresh tensors after
    `zero_grad(set_to_none=True)`; inside a captured CUDA graph their addresses repeat, and the captured upload re-reads the
    same pinned table)."""

    def __init__(self, entries, device):
        # entries: list of (param, mom | None, ema | None, group); gradient pointers are filled in by set_grads()
        import numpy as np

        lib = _lib.lib()
        chunk = int(lib.y5_opt_chunk_elems())
        n = len(entries)
        self.host = torch.zeros(n * _opt_dtype().itemsize, dtype=torch.uint8).pin_memory()
        self.np = self.host.numpy().view(_opt_dtype())
        ct, ci = [], []
        for t, (p, m, e, grp) in enumerate(entries):
            for x in (p, m, e):
                if x is not None and (x.dtype != torch.float32 or not x.is_contiguous() or x.device != device):
                    raise TypeError("y5b200: the fused optimizer / EMA step handles contiguous fp32 tensors on one device (fp32 master weights)")
            self.np[t] = (p.data_ptr(), 0, m.data_ptr() if m is not None else 0, e.data_ptr() if e is not None else 0, p.numel(), grp, 0)
            n_chunks = (p.numel() + chunk - 1) // chunk
            ct += [t] * n_chunks
            ci += list(range(n_chunks))
        self.table = torch.empty(n * _opt_dtype().itemsize, dtype=torch.uint8, device=device)
        self.chunk_tensor = torch.tensor(ct, dtype=torch.int32, device=device)
        self.chunk_index = torch.tensor(ci, dtype=torch.int32, device=device)
        self.n_chunks = len(ct)
        self.partial = torch.zeros(2 * max(self.n_chunks, 1), dtype=torch.float32, device=device)
        self.keep = entries  # the table holds raw addresses: keep the tensors alive
        self.upload()

    def set_grads(self, ptrs):
        self.np["grad"][: len(ptrs)] = ptrs

    def upload(self):
        self.table.copy_(self.host, non_blocking=True)


class ModelEMA:
    """Exponential moving average of everything floating point in the model's state_dict (reference
    utils/torch_utils.py:343-375): ``ema = d * ema + (1 - d) * model`` with ``d = decay * (1 - exp(-updates / tau))``.
    `update` is ONE multi-tensor launch (y5_opt_step with the EMA branch only) instead of two foreach passes over ~350
    tensors; `FusedSGD.fused_step(ema=...)` folds it into the optimizer step so the new weights are not re-read at all."""

    def __init__(self, model, decay=0.9999, tau=2000, updates=0):
        self.ema = deepcopy(de_parallel(model)).eval()
        self.updates = updates
        self.decay_base, self.tau = float(decay), float(tau)
        self.decay = lambda x: decay * (1 - math.exp(-x / tau))
        for p in self.ema.parameters():
            p.requires_grad_(False)
        self._table = None
        self._hyper = None

    def pairs(self, model):
        """[(model tensor, ema tensor)] over floating-point state_dict entries, in state_dict order."""
        msd, esd = de_parallel(model).state_dict(), self.ema.state_dict()
        return [(msd[k], v) for k, v in esd.items() if v.dtype.is_floating_point]

    def hyper_init(self, hyper: torch.Tensor):
        hyper[_lib.OPT_EMA_DECAY] = self.decay_base
        hyper[_lib.OPT_EMA_TAU] = self.tau
        hyper[_lib.OPT_EMA_UPDATES] = float(self.updates)

    def update(self, model):
        pairs = self.pairs(model)
        if not pairs:
            return
        dev = pairs[0][0].device
        if not pairs[0][0].is_cuda:
            raise RuntimeError("y5b200: ModelEMA.update runs on CUDA tensors only (no CPU / PyTorch fallback)")
        key = tuple(t.data_ptr() for pr in pairs for t in pr)
        if self._table is None or self._key != key:
            self._table = _OptTable([(m.detach(), None, e, 0) for m, e in pairs], dev)
            self._key = key
            self._hyper = torch.zeros(_lib.OPT_GROUPS + 4, dtype=torch.float32, device=dev)
        self.hyper_init(self._hyper)  # host mirror of the counter is authoritative for the standalone path
        t = self._table
        with _lib.on(dev):
            _lib.check(_lib.lib().y5_opt_step(t.table.data_ptr(), t.chunk_tensor.data_ptr(), t.chunk_index.data_ptr(), t.n_chunks,
                                              self._hyper.data_ptr(), t.partial.data_ptr(), 0, 1, 0, C.c_void_p(_lib.stream_ptr(dev))), "ema_update")
        self.updates += 1

    def update_attr(self, model, include=(), exclude=("process_group", "reducer")):
        copy_attr(self.ema, model, include, exclude)


class _FusedOptimizer(torch.optim.Optimizer):
    """What FusedSGD and FusedAdam share: the device tables of every parameter (+ the EMA's tensors), the data-parallel
    gradient arena, the device-side GradScaler handling, the per-step hyper-parameter upload and the step's device outputs.
    A subclass owns its state buffers (`_bind_state`), its per-group hyper-parameters (`_fill_groups` / `_upload_groups`), the
    update launch (`_launch`) and `zero_state`."""

    def __init__(self, params, defaults):
        super().__init__(params, defaults)
        self._tab = None
        self._tab_key = None
        self._dp = None  # (process group, world size) once data_parallel() was called

    # ------------------------------------------------------------------ data parallel
    def data_parallel(self, model, process_group=None, src: int = 0):
        """Turn the step into the data-parallel one (what reference train.py gets from smart_DDP, utils/torch_utils.py:61-70):
        parameters and buffers are broadcast from rank `src` once; from then on `fused_step` copies every gradient into one
        contiguous fp32 arena (y5_grad_pack, one launch), all-reduces the arena with ONE NCCL call (average over ranks, like
        DDP) and updates from the averaged arena.  No autograd hooks, buckets or copy-backs, and nothing but the all-reduce
        itself touches the link.  `model` must be the plain module (not wrapped in DistributedDataParallel); gradient
        accumulation needs no `no_sync()`: ranks only talk inside `fused_step`.  BatchNorm statistics stay per rank unless the
        model was converted with torch.nn.SyncBatchNorm.convert_sync_batchnorm (train.py --sync-bn): those layers all-reduce
        their batch statistics and BN gradients over their process group inside the forward and backward."""
        import torch.distributed as dist

        name = type(self).__name__
        if not (dist.is_available() and dist.is_initialized()):
            raise RuntimeError(f"y5b200: {name}.data_parallel needs an initialised torch.distributed process group")
        if isinstance(model, (nn.parallel.DataParallel, nn.parallel.DistributedDataParallel)):
            raise TypeError(f"y5b200: pass the plain module to {name}.data_parallel (DistributedDataParallel would all-reduce a second time)")
        world = dist.get_world_size(process_group)
        with torch.no_grad():
            for t in list(model.parameters()) + list(model.buffers()):
                dist.broadcast(t.data, src=dist.get_global_rank(process_group, src) if process_group is not None else src, group=process_group)
        self._dp = (process_group, world)
        self._tab = None  # rebuild the tables with the arena
        return self

    # ------------------------------------------------------------------ tables
    def _params(self):
        return [(gi, p) for gi, g in enumerate(self.param_groups) for p in g["params"] if p.requires_grad]

    def _ensure(self, ema, model):
        ps = self._params()
        key = (tuple(id(p) for _, p in ps), id(ema))
        if self._tab is not None and self._tab_key == key:
            return
        dev = ps[0][1].device
        if not ps[0][1].is_cuda:
            raise RuntimeError(f"y5b200: {type(self).__name__} runs on CUDA parameters only (no CPU / PyTorch fallback)")
        ema_pairs = ema.pairs(model) if ema is not None else []
        ema_of = {m_t.data_ptr(): e_t for m_t, e_t in ema_pairs}
        seen = {p.data_ptr() for _, p in ps}
        buffers = [(m_t, e_t) for m_t, e_t in ema_pairs if m_t.data_ptr() not in seen]  # BN running statistics: EMA only
        self._plist = [p for _, p in ps]
        moms = self._bind_state(ps, len(ps) + len(buffers), dev)
        entries = [(p.detach(), m, ema_of.get(p.data_ptr()), gi) for (gi, p), m in zip(ps, moms)]
        entries += [(m_t.detach(), None, e_t, 0) for m_t, e_t in buffers]
        self._tab = _OptTable(entries, dev)
        self._tab_arena = None
        if self._dp is not None:
            # data-parallel mode: the gradients' home for the all-reduce and the update.  Tensor t sits at a 16-byte aligned
            # offset; the second table is the first with its gradient column pointing into the arena (fixed addresses).
            offs, o = [], 0
            for e in entries:
                offs.append(o if e[1] is not None else 0)
                if e[1] is not None:
                    o += (e[0].numel() + 3) // 4 * 4
            # [gradients | one "had a gradient on this rank" float per table entry]: one buffer, one all-reduce
            self._arena_all = torch.zeros(max(o, 4) + len(entries), dtype=torch.float32, device=dev)
            self._arena = self._arena_all[: max(o, 4)]
            self._present = self._arena_all[max(o, 4) :]
            self._arena_off = torch.tensor(offs, dtype=torch.int64, device=dev)
            self._tab_arena = _OptTable(entries, dev)
            self._tab_arena.set_grads([self._arena.data_ptr() + 4 * off if e[1] is not None else 0 for e, off in zip(entries, offs)])
            self._tab_arena.upload()
        self._tab_key = key
        n = _lib.OPT_GROUPS + self._GROUP_FLOATS * len(self.param_groups)
        self._hyper = torch.zeros(n, dtype=torch.float32, device=dev)
        self._hyper_host = torch.zeros(n, dtype=torch.float32).pin_memory()
        self._hyper[_lib.OPT_INV_SCALE] = 1.0
        if ema is not None:
            ema.hyper_init(self._hyper)

    def fill_hyper_host(self, max_norm):
        """Write the clip norm and every group's hyper-parameters into the pinned staging buffers."""
        self._hyper_host[_lib.OPT_MAX_NORM] = float(max_norm) if max_norm else 0.0
        self._fill_groups()

    def _upload_hyper(self, max_norm):
        self.fill_hyper_host(max_norm)
        h = self._hyper_host
        self._hyper[_lib.OPT_MAX_NORM : _lib.OPT_MAX_NORM + 1].copy_(h[_lib.OPT_MAX_NORM : _lib.OPT_MAX_NORM + 1], non_blocking=True)
        self._upload_groups()

    # ------------------------------------------------------------------ steps
    @torch.no_grad()
    def fused_step(self, scaler=None, max_norm=10.0, ema=None, model=None):
        """train.py:413-421 (minus zero_grad) in one call: un-scale by `scaler`'s current factor, clip to `max_norm`, update
        every parameter that has a gradient, and -- with `ema` (+ the `model` it tracks) -- ModelEMA.update.  `scaler` is a
        torch GradScaler: its scale is read, and its growth / back-off state advanced, on the device (what scaler.step +
        scaler.update do, without their host synchronisation); a non-finite gradient skips the update.  `last_grad_norm` /
        `last_step_skipped` read the device-side results (they synchronise)."""
        if ema is not None and model is None:
            model = getattr(self, "_ema_model", None)
            if model is None:
                raise ValueError(f"{type(self).__name__}.fused_step(ema=...) needs model= (the module the EMA tracks)")
        self._ema_model = model
        self._ensure(ema, model)
        dev = self._hyper.device
        self._upload_hyper(max_norm)
        t = self._tab
        t.set_grads([p.grad.data_ptr() if p.grad is not None else 0 for p in self._plist])
        for p in self._plist:
            if p.grad is not None and (p.grad.dtype != torch.float32 or not p.grad.is_contiguous()):
                raise TypeError(f"y5b200: {type(self).__name__} needs contiguous fp32 gradients")
        t.upload()
        use_scaler = scaler is not None and scaler.is_enabled() and getattr(scaler, "_scale", None) is not None
        if use_scaler:
            torch.reciprocal(scaler._scale.reshape(1).float(), out=self._hyper[_lib.OPT_INV_SCALE : _lib.OPT_INV_SCALE + 1])
        if self._dp is not None:
            import torch.distributed as dist

            with _lib.on(dev):
                _lib.check(_lib.lib().y5_grad_pack(t.table.data_ptr(), t.chunk_tensor.data_ptr(), t.chunk_index.data_ptr(), t.n_chunks,
                                                   self._arena_off.data_ptr(), self._arena.data_ptr(), self._present.data_ptr(),
                                                   C.c_void_p(_lib.stream_ptr(dev))), "grad_pack")
            if self._dp[1] > 1:
                dist.all_reduce(self._arena_all, op=dist.ReduceOp.AVG, group=self._dp[0])
            t = self._tab_arena
            with _lib.on(dev):
                _lib.check(_lib.lib().y5_grad_bind(t.table.data_ptr(), len(t.keep), self._arena_off.data_ptr(), self._arena.data_ptr(),
                                                   self._present.data_ptr(), C.c_void_p(_lib.stream_ptr(dev))), "grad_bind")
        with _lib.on(dev):
            self._launch(t, 1 if ema is not None else 0, C.c_void_p(_lib.stream_ptr(dev)))
        if ema is not None:
            ema.updates += 1
        if use_scaler:  # what scaler.update() does after scaler.step(): back off on overflow, grow after growth_interval clean steps
            torch._amp_update_scale_(scaler._scale, scaler._growth_tracker, self._hyper[_lib.OPT_OUT_SKIPPED : _lib.OPT_OUT_SKIPPED + 1],
                                     scaler.get_growth_factor(), scaler.get_backoff_factor(), scaler.get_growth_interval())

    @torch.no_grad()
    def step(self, closure=None):
        """Plain optimizer.step(): the update only (no un-scaling, clipping or EMA), for code that drives those itself."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        self.fused_step(scaler=None, max_norm=None, ema=None)
        return loss

    @property
    def last_grad_norm(self) -> float:
        return float(self._hyper[_lib.OPT_OUT_NORM])

    @property
    def last_step_skipped(self) -> bool:
        return bool(self._hyper[_lib.OPT_OUT_SKIPPED] != 0)


class FusedSGD(_FusedOptimizer):
    """SGD with momentum / Nesterov over parameter groups (what reference smart_optimizer builds, utils/torch_utils.py:256-289)
    whose whole step -- GradScaler un-scale, clip_grad_norm_, weight decay, momentum, update, zero_grad and optionally
    ModelEMA.update (reference train.py:413-421) -- is two multi-tensor launches of liby5b200 (y5_opt_step).

    `param_groups` carry lr / momentum / weight_decay / nesterov exactly like torch.optim.SGD, so LambdaLR schedulers and the
    warm-up code that edits them (train.py:368-376) work unchanged; their values are uploaded each step (a captured CUDA graph
    replays that upload, so schedules keep working under GraphedTrainStep).  Gradients are read where autograd left them
    (`zero_grad(set_to_none=True)` semantics: no extra accumulate kernels); only their addresses are refreshed per step.

        opt.fused_step(scaler=scaler, max_norm=10.0, ema=ema)     # == train.py:413-421
        opt.step()                                                # plain optimizer.step() (no clipping / scaling / EMA)
    """

    _GROUP_FLOATS = 4  # lr, momentum, weight_decay, nesterov at Y5_OPT_GROUPS + 4g of `hyper`

    def __init__(self, params, lr=1e-3, momentum=0.0, weight_decay=0.0, nesterov=False):
        if nesterov and momentum <= 0:
            raise ValueError("Nesterov momentum requires a momentum")
        super().__init__(params, dict(lr=lr, momentum=momentum, weight_decay=weight_decay, nesterov=nesterov))

    def _bind_state(self, ps, n_entries, dev):
        total = sum(p.numel() for _, p in ps)
        flat_m = torch.zeros(total, dtype=torch.float32, device=dev)  # momentum buffers: one allocation, fixed addresses
        off, moms = 0, []
        for _, p in ps:
            n = p.numel()
            st = self.state[p]
            m = flat_m[off : off + n].view_as(p)
            if st.get("momentum_buffer") is not None:
                m.copy_(st["momentum_buffer"])
            st["momentum_buffer"] = m
            moms.append(m)
            off += n
        self._flat_m = flat_m
        return moms

    def _fill_groups(self):
        h = self._hyper_host
        for gi, g in enumerate(self.param_groups):
            o = _lib.OPT_GROUPS + 4 * gi
            h[o], h[o + 1], h[o + 2], h[o + 3] = g["lr"], g["momentum"], g["weight_decay"], 1.0 if g["nesterov"] else 0.0

    def _upload_groups(self):
        self._hyper[_lib.OPT_GROUPS :].copy_(self._hyper_host[_lib.OPT_GROUPS :], non_blocking=True)

    def _launch(self, t, do_ema, stream):
        _lib.check(_lib.lib().y5_opt_step(t.table.data_ptr(), t.chunk_tensor.data_ptr(), t.chunk_index.data_ptr(), t.n_chunks,
                                          self._hyper.data_ptr(), t.partial.data_ptr(), 1, do_ema, 0, stream), "opt_step")

    def zero_state(self):
        """Zero the momentum buffers in place (their device addresses, which a captured graph holds, stay)."""
        self._flat_m.zero_()


class FusedAdam(_FusedOptimizer):
    """torch.optim.Adam (decoupled_weight_decay=False) or AdamW (True) over parameter groups -- what reference smart_optimizer
    builds for `--optimizer Adam | AdamW` (utils/torch_utils.py:276-279) -- with the same fused train.py:413-421 step as
    FusedSGD: three multi-tensor launches of liby5b200 (y5_adam_step).  The arithmetic is torch's foreach CUDA path, with the
    bias corrections computed in double like torch's Python scalars; amsgrad and maximize are not implemented.

    `param_groups` carry torch.optim.Adam's keys and no `momentum` (train.py's warm-up leaves the betas alone, as it does for the
    reference); lr / betas / eps / weight_decay are uploaded each step, also under GraphedTrainStep.  Each parameter's step
    count is an fp32 counter on the device that advances when the parameter had a gradient and the step was not skipped; it is
    never read back while training.  `state_dict()` / `load_state_dict()` use torch's Adam format (`step` a 0-d fp32 CPU
    tensor, `exp_avg`, `exp_avg_sq`), so optimizer states move both ways between this class and torch.optim.Adam / AdamW."""

    _GROUP_FLOATS = 0  # the per-group block is y5_adam_step's fp64 `group_hyper`

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, *, maximize=False,
                 decoupled_weight_decay=False):
        if amsgrad:
            raise NotImplementedError("y5b200: Adam(amsgrad=True) is outside the fused optimizer (reference smart_optimizer never sets it)")
        if maximize:
            raise NotImplementedError("y5b200: Adam(maximize=True) is outside the fused optimizer (reference smart_optimizer never sets it)")
        if not 0.0 <= lr or not 0.0 <= eps or not 0.0 <= weight_decay or not all(0.0 <= b < 1.0 for b in betas):
            raise ValueError(f"invalid Adam hyper-parameters lr={lr} betas={betas} eps={eps} weight_decay={weight_decay}")
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, amsgrad=False, maximize=False, foreach=None,
                                      capturable=False, differentiable=False, fused=None, decoupled_weight_decay=decoupled_weight_decay))

    def add_param_group(self, param_group):
        for k in ("amsgrad", "maximize"):
            if param_group.get(k):
                raise NotImplementedError(f"y5b200: Adam({k}=True) is outside the fused optimizer")
        super().add_param_group(param_group)

    def _bind_state(self, ps, n_entries, dev):
        self._total = sum(p.numel() for _, p in ps)
        self._flat = torch.zeros(2 * self._total, dtype=torch.float32, device=dev)  # [exp_avg | exp_avg_sq]: fixed addresses
        self._steps = torch.zeros(n_entries, dtype=torch.float32, device=dev)       # step count per table entry
        n_groups = len(self.param_groups)
        self._ghyper = torch.zeros(_lib.ADAM_STRIDE * n_groups, dtype=torch.float64, device=dev)
        self._ghyper_host = torch.zeros(_lib.ADAM_STRIDE * n_groups, dtype=torch.float64).pin_memory()
        self._adopt_state()
        return [self.state[p]["exp_avg"] for p in self._plist]

    def _adopt_state(self):
        """Move every parameter's state (fresh, loaded from a state_dict, or already ours) into the flat device buffers and
        point `state` at them: exp_avg / exp_avg_sq views and `step` a 0-d view of the device counter."""
        steps, off = [], 0
        for i, p in enumerate(self._plist):
            n = p.numel()
            st = self.state[p]
            m = self._flat[off : off + n].view_as(p)
            v = self._flat[self._total + off : self._total + off + n].view_as(p)
            for key, buf in (("exp_avg", m), ("exp_avg_sq", v)):
                if st.get(key) is not None:
                    buf.copy_(st[key])
                else:
                    buf.zero_()
            steps.append(float(st["step"]) if "step" in st else 0.0)
            st["exp_avg"], st["exp_avg_sq"], st["step"] = m, v, self._steps[i]
            off += n
        self._steps[: len(steps)].copy_(torch.tensor(steps, dtype=torch.float32))

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        if self._tab is not None:  # the tables hold the flat buffers' addresses: copy the loaded state into them
            self._adopt_state()

    def state_dict(self):
        sd = super().state_dict()
        if self._tab is not None:  # torch's format: `step` as a 0-d fp32 CPU tensor (one device-to-host copy for all)
            host = self._steps.cpu()
            row = {id(p): i for i, p in enumerate(self._plist)}
            flat = [p for g in self.param_groups for p in g["params"]]
            sd["state"] = {k: dict(st, step=host[row[id(flat[k])]].clone()) if id(flat[k]) in row else st for k, st in sd["state"].items()}
        return sd

    def _fill_groups(self):
        h = self._ghyper_host
        for gi, g in enumerate(self.param_groups):
            o = _lib.ADAM_STRIDE * gi
            h[o + _lib.ADAM_LR], h[o + _lib.ADAM_EPS], h[o + _lib.ADAM_WEIGHT_DECAY] = g["lr"], g["eps"], g["weight_decay"]
            h[o + _lib.ADAM_BETA1], h[o + _lib.ADAM_BETA2] = g["betas"]
            h[o + _lib.ADAM_DECOUPLED] = 1.0 if g["decoupled_weight_decay"] else 0.0

    def _upload_groups(self):
        self._ghyper.copy_(self._ghyper_host, non_blocking=True)

    def _launch(self, t, do_ema, stream):
        _lib.check(_lib.lib().y5_adam_step(t.table.data_ptr(), len(t.keep), t.chunk_tensor.data_ptr(), t.chunk_index.data_ptr(), t.n_chunks,
                                           self._hyper.data_ptr(), self._ghyper.data_ptr(), self._total, self._steps.data_ptr(),
                                           t.partial.data_ptr(), do_ema, 0, stream), "adam_step")

    def zero_state(self):
        """Zero both moments and the step counters in place (their device addresses, which a captured graph holds, stay): the
        next step is step 1 with the full bias correction."""
        self._flat.zero_()
        self._steps.zero_()


class FusedAdamW(FusedAdam):
    """torch.optim.AdamW on the fused step: FusedAdam with decoupled weight decay and AdamW's default weight_decay=1e-2."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False, *, maximize=False):
        super().__init__(params, lr, betas, eps, weight_decay, amsgrad, maximize=maximize, decoupled_weight_decay=True)


def smart_optimizer(model, name="Adam", lr=0.001, momentum=0.9, decay=1e-5):
    """Three parameter groups like reference utils/torch_utils.py:256-289 -- biases (no decay), BatchNorm weights (no decay),
    other weights (decay) -- on the fused step: SGD-Nesterov, Adam(betas=(momentum, 0.999)) or AdamW(betas=(momentum, 0.999),
    weight_decay=0 for the bias group).  RMSProp (not offered by train.py's --optimizer) is not implemented."""
    if name not in ("SGD", "Adam", "AdamW"):
        raise NotImplementedError(f"y5b200: optimizer {name} is outside the hot path (train.py offers SGD, Adam and AdamW)")
    g = [], [], []
    bn = tuple(v for k, v in nn.__dict__.items() if "Norm" in k)  # every torch.nn normalisation layer, SyncBatchNorm included
    for v in model.modules():
        for p_name, p in v.named_parameters(recurse=False):
            if p_name == "bias":
                g[2].append(p)
            elif p_name == "weight" and isinstance(v, bn):
                g[1].append(p)
            else:
                g[0].append(p)
    if name == "Adam":
        opt = FusedAdam(g[2], lr=lr, betas=(momentum, 0.999))
    elif name == "AdamW":
        opt = FusedAdamW(g[2], lr=lr, betas=(momentum, 0.999), weight_decay=0.0)
    else:
        opt = FusedSGD(g[2], lr=lr, momentum=momentum, nesterov=True)
    opt.add_param_group({"params": g[0], "weight_decay": decay})
    opt.add_param_group({"params": g[1], "weight_decay": 0.0})
    return opt


class GraphedTrainStep:
    """One optimisation step -- forward (batch-statistics BN), ComputeLoss, scaled backward, un-scale + gradient clipping +
    SGD / Adam / AdamW + zero_grad + EMA (reference train.py:401-421) -- captured once in a CUDA graph and replayed per batch.

    The training path never synchronises with the host, so the whole step is capturable; replaying it removes the Python /
    launch-issue time that bounds the eager step.  Numerically it is the reference's AMP recipe: with fp16 autocast the loss
    is multiplied by a dynamic loss scale kept ON THE DEVICE (GradScaler semantics: init 65536, x0.5 on overflow with the step
    skipped, x2 after 2000 clean steps -- y5_opt_step reports overflow, torch._amp_update_scale_ advances the scale, both
    inside the graph); bf16 autocast needs no scaling.  The optimizer's group hyper-parameters (lr, momentum or betas, ...) are re-read from
    `optimizer.param_groups` at every call (uploaded through a pinned buffer the captured copy node reads at replay time), so
    warm-up and schedulers work.  Shapes are fixed at construction: `batch` uint8 images of `size` and up to `max_targets`
    label rows; shorter label tensors are padded with zero-size boxes, which build_targets can never match (the anchor ratio
    test of utils/loss.py:219 fails for w = h = 0).  Data parallel: pass an optimizer on which `data_parallel(model)` was called
    -- its one NCCL all-reduce of the packed gradient arena is captured with the rest of the step (every rank constructs and
    calls the object in lock-step; the loss is multiplied by the world size like train.py:405).  A model wrapped in
    DistributedDataParallel is not capturable (autograd hooks, buckets).

        opt = smart_optimizer(model, "SGD", lr, momentum, decay); ema = ModelEMA(model)
        step = GraphedTrainStep(model, ComputeLoss(model), opt, batch=16, size=640, ema=ema)
        for imgs_u8, targets in loader:          # (B,3,H,W) uint8 on any device, (nt,6) float
            loss_items = step(imgs_u8, targets)  # (3,) tensor on the GPU, valid after the replay (stream-ordered)
    """

    def __init__(self, model, compute_loss, optimizer, batch: int, size, max_targets: int | None = None, amp_dtype=torch.float16,
                 max_norm: float | None = 10.0, warmup_steps: int = 3, ema=None, init_scale: float = 65536.0):
        if not isinstance(optimizer, _FusedOptimizer):
            raise TypeError("GraphedTrainStep needs a fused optimizer (yolov5_b200.utils.torch_utils.smart_optimizer / FusedSGD / FusedAdam): its "
                            "overflow-skipping step is what makes the loss-scaled update capturable")
        dev = next(model.parameters()).device
        h, w = (size, size) if isinstance(size, int) else size
        self.max_targets = max_targets or 64 * batch
        self.img = torch.zeros(batch, 3, h, w, dtype=torch.uint8, device=dev)
        self.tgt = torch.zeros(self.max_targets, 6, dtype=torch.float32, device=dev)
        self.items = torch.zeros(3, dtype=torch.float32, device=dev)
        self.optimizer, self.max_norm = optimizer, max_norm
        self.scaler = torch.amp.GradScaler("cuda", init_scale=init_scale, enabled=amp_dtype == torch.float16)
        scaler = self.scaler
        if isinstance(model, (nn.parallel.DataParallel, nn.parallel.DistributedDataParallel)):
            raise TypeError("GraphedTrainStep: pass the plain module; for data parallel use FusedSGD.data_parallel(model), whose single "
                            "all-reduce is capturable")
        world = optimizer._dp[1] if optimizer._dp is not None else 1

        from .. import train_ops

        syncing = [n for n, m in model.named_modules() if train_ops.bn_process_group(m) is not None]
        if syncing:
            raise NotImplementedError(f"GraphedTrainStep: {len(syncing)} SyncBatchNorm layers (first: {syncing[0]}) all-reduce their batch "
                                      "statistics inside the forward and backward, which this step does not capture; train such a model "
                                      "with the eager step, or convert it back to BatchNorm2d")

        def step():
            with torch.autocast("cuda", dtype=amp_dtype):
                pred = model(self.img)
            loss, items = compute_loss(pred, self.tgt)
            if world > 1:
                loss = loss * world  # train.py:405: the all-reduce averages over ranks, the reference rescales
            # weight gradients on a side stream, joined at the end of backward: a fork per layer in the captured graph
            prev = train_ops.set_async_wgrad(os.environ.get("Y5_ASYNC_WGRAD", "1") != "0")
            try:
                scaler.scale(loss).backward()
            finally:
                train_ops.set_async_wgrad(prev)
                train_ops.finish_async(dev)
            optimizer.fused_step(scaler=scaler, max_norm=max_norm, ema=ema, model=model)
            optimizer.zero_grad(set_to_none=True)  # gradients return to the graph's private pool: same addresses at every replay
            self.items.copy_(items)

        # warm-up on a side stream (lazy initialisation, optimizer tables, allocator pools), then capture.  The warm-up steps
        # run on the zero batch with a zero learning rate; everything they touch is restored below.
        lrs = [g["lr"] for g in optimizer.param_groups]
        state = {k: v.clone() for k, v in model.state_dict().items()}
        ema_state = {k: v.clone() for k, v in ema.ema.state_dict().items()} if ema is not None else None
        ema_updates = ema.updates if ema is not None else 0
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for g in optimizer.param_groups:
                g["lr"] = 0.0
            for _ in range(warmup_steps):
                step()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        for g, lr in zip(optimizer.param_groups, lrs):
            g["lr"] = lr
        self.graph = torch.cuda.CUDAGraph()
        # with a process group alive, NCCL's watchdog thread issues CUDA calls of its own: only this thread's calls belong to the capture
        with torch.cuda.graph(self.graph, capture_error_mode="thread_local" if world > 1 else "global"):
            step()
        # the capture baked in the address of the BN-sum arena (allocated during warm-up, outside the graph's pool): keep it
        # alive even if a later eager forward of another shape makes the arena grow
        self._arena_buf = train_ops._arena.buf
        self._pack_plans = list(model.__dict__.get("_y5_pack_plans", {}).values())  # persistent packed-weight buffers + tables
        # undo what warm-up and capture touched: weights are unchanged (lr 0 / capture does not execute), BN running statistics
        # and batch counters, the optimizer state (momentum / moments and step counts), the EMA and its counter, the loss scale
        model.load_state_dict(state)
        optimizer.zero_state()
        if ema is not None:
            ema.ema.load_state_dict(ema_state)
            ema.updates = ema_updates
            ema.hyper_init(optimizer._hyper)
        if self.scaler.is_enabled():
            self.scaler._scale.fill_(init_scale)
            self.scaler._growth_tracker.zero_()
        self.ema = ema

    def __call__(self, imgs_u8: torch.Tensor, targets: torch.Tensor) -> torch.Tensor:
        nt = targets.shape[0]
        if nt > self.max_targets:
            raise ValueError(f"GraphedTrainStep: {nt} label rows > max_targets {self.max_targets}")
        self.img.copy_(imgs_u8, non_blocking=True)
        self.tgt.zero_()
        if nt:
            self.tgt[:nt].copy_(targets, non_blocking=True)
        self.optimizer.fill_hyper_host(self.max_norm)  # the captured copy nodes read this pinned buffer at replay time
        self.graph.replay()
        if self.ema is not None:
            self.ema.updates += 1
        return self.items
