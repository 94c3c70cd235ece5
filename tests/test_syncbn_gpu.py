"""-m gpu: SyncBatchNorm on the training path (train.py --sync-bn converts the model with
torch.nn.SyncBatchNorm.convert_sync_batchnorm, reference train.py:268-271).

The defining property: k ranks synchronised on shards of a batch compute what one rank computes on the whole batch.
  * the split passes (y5_bn_stats / y5_bn_act_fwd with a row count, y5_bn_act_bwd_reduce / y5_bn_act_bwd_apply) with no
    all-reduce between them give exactly what y5_bn_stats + y5_bn_act_fwd without one and y5_bn_act_bwd give;
  * shards of one batch whose workspaces are added (fp64, exact on integer-valued data) stand in for the all-reduce: each
    shard's z / dy are the full batch's rows bit for bit, and so are the running statistics;
  * two processes on one GPU (gloo) train a converted yolov5n like one process on the whole batch;
  * on two GPUs (NCCL) a step under smart_DDP and under FusedSGD.data_parallel leaves both ranks identical;
  * a SyncBatchNorm that does not sync is BatchNorm2d, launch for launch; eval and checkpoints fold it like BatchNorm2d.
"""
import ctypes as C
import os
import time

import pytest
import torch

from yolov5_b200 import _lib, train_ops

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
EPS, MOM = 1e-3, 0.03


def _st(dev):
    return C.c_void_p(_lib.stream_ptr(dev))


def _ints(shape, seed, dev, lo=-2, hi=2):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randint(lo, hi + 1, shape, generator=g, device=dev, dtype=torch.float32)


def _slice(rows, c, extra, fill, dtype, dev):
    """(buffer [rows][c + extra + 8], pointer of the channel view at offset 8, pitch): channel-slice views as the model has"""
    buf = torch.full((rows, c + extra + 8), fill, dtype=dtype, device=dev)
    return buf, buf.data_ptr() + 8 * buf.element_size(), buf.shape[1]


def _bits(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.contiguous().view(-1).view(torch.uint8), b.contiguous().view(-1).view(torch.uint8))


class _Layer:
    """one BN layer's operands on channel-slice views: y, dz (+ residual), gamma / beta and running statistics"""

    def __init__(self, y, dz, gamma, beta, res, dtype, dev):
        rows, ch = y.shape
        self.rows, self.ch, self.dtype, self.dev = rows, ch, dtype, dev
        self.ybuf, self.yp, self.ypitch = _slice(rows, ch, 24, 9.0, dtype, dev)
        self.ybuf[:, 8 : 8 + ch] = y.to(dtype)
        self.dzbuf, self.dzp, self.dzpitch = _slice(rows, ch, 8, 11.0, dtype, dev)
        self.dzbuf[:, 8 : 8 + ch] = dz.to(dtype)
        self.rbuf, self.rp, self.rpitch = None, None, 0
        if res is not None:
            self.rbuf, self.rp, self.rpitch = _slice(rows, ch, 40, 3.0, dtype, dev)
            self.rbuf[:, 8 : 8 + ch] = res.to(dtype)
        self.gamma, self.beta = gamma, beta

    def view(self, r0, r1):
        """the same layer restricted to rows [r0, r1): a shard of the batch"""
        sub = _Layer.__new__(_Layer)
        sub.__dict__.update(self.__dict__)
        sub.rows = r1 - r0
        es = self.ybuf.element_size()
        sub.yp, sub.dzp = self.yp + r0 * self.ypitch * es, self.dzp + r0 * self.dzpitch * es
        sub.rp = self.rp + r0 * self.rpitch * es if self.rp is not None else None
        return sub


def _forward(L, act, sync, rm, rv, ws, eps=EPS):
    """stats + normalise/activate; returns (z buffer, mean, invstd).  `ws` is the workspace (2C, or 2C + 1 for sync, whose
    slot 2C is the row count)."""
    lib, code, st = _lib.lib(), _lib.dtype_code(L.dtype), _st(L.dev)
    mean, invstd = torch.empty(L.ch, device=L.dev), torch.empty(L.ch, device=L.dev)
    zbuf, zp, zpitch = _slice(L.rows, L.ch, 16, -7.0, L.dtype, L.dev)

    def count(w):
        return w[2 * L.ch :].data_ptr() if sync else None

    _lib.check(lib.y5_bn_stats(L.yp, L.ypitch, L.rows, L.ch, code, ws.data_ptr(), count(ws), st), "stats")
    return zbuf, zp, zpitch, mean, invstd, lambda sums: _lib.check(
        lib.y5_bn_act_fwd(L.yp, L.ypitch, zp, zpitch, L.rows, L.ch, code, mean.data_ptr(), invstd.data_ptr(), L.gamma.data_ptr(),
                          L.beta.data_ptr(), act, 0.0, sums.data_ptr(), count(sums), eps, MOM, rm.data_ptr(), rv.data_ptr(), L.rp, L.rpitch,
                          st), "fwd")


def _fused(L, act, rm, rv, eps=EPS):
    """today's path: y5_bn_stats + y5_bn_act_fwd, y5_bn_act_bwd"""
    lib, code, st = _lib.lib(), _lib.dtype_code(L.dtype), _st(L.dev)
    ws = torch.zeros(2 * L.ch, dtype=torch.float64, device=L.dev)
    zbuf, _, _, mean, invstd, fwd = _forward(L, act, False, rm, rv, ws, eps)
    fwd(ws)
    dybuf, dyp, dypitch = _slice(L.rows, L.ch, 32, -13.0, L.dtype, L.dev)
    dg, db = torch.empty(L.ch, device=L.dev), torch.empty(L.ch, device=L.dev)
    wsb = torch.zeros(2 * L.ch, dtype=torch.float64, device=L.dev)
    _lib.check(lib.y5_bn_act_bwd(L.yp, L.ypitch, L.dzp, L.dzpitch, dyp, dypitch, L.rows, L.ch, code, mean.data_ptr(), invstd.data_ptr(),
                                 L.gamma.data_ptr(), L.beta.data_ptr(), act, 0.0, dg.data_ptr(), db.data_ptr(), wsb.data_ptr(), st), "bwd")
    torch.cuda.synchronize()
    return dict(z=zbuf, mean=mean, invstd=invstd, rm=rm, rv=rv, dy=dybuf, dgamma=dg, dbeta=db)


def _sharded(L, act, bounds, rm0, rv0, eps=EPS):
    """The sync passes on the shards [bounds[i], bounds[i+1]) of L, with the all-reduce emulated by adding the shards'
    workspaces in fp64 (torch.stack(...).sum(0)).  Returns one result dict per shard."""
    lib, code, st = _lib.lib(), _lib.dtype_code(L.dtype), _st(L.dev)
    shards = [L.view(a, b) for a, b in zip(bounds[:-1], bounds[1:])]
    c = L.ch
    outs, launches, wss = [], [], []
    for S in shards:
        ws = torch.zeros(2 * c + 1, dtype=torch.float64, device=L.dev)
        rm, rv = rm0.clone(), rv0.clone()
        zbuf, _, _, mean, invstd, fwd = _forward(S, act, True, rm, rv, ws, eps)
        wss.append(ws)
        launches.append(fwd)
        outs.append(dict(z=zbuf, mean=mean, invstd=invstd, rm=rm, rv=rv))
    total = torch.stack(wss).sum(0)  # the SUM all-reduce of [sums | count]
    assert float(total[2 * c]) == L.rows
    for fwd in launches:
        fwd(total)
    n = total[2 * c : 2 * c + 1].clone()
    bws = []
    for S, o in zip(shards, outs):
        o["dy"], o["dyp"], o["dypitch"] = _slice(S.rows, c, 32, -13.0, L.dtype, L.dev)
        o["dgamma"], o["dbeta"] = torch.empty(c, device=L.dev), torch.empty(c, device=L.dev)
        ws = torch.zeros(2 * c, dtype=torch.float64, device=L.dev)
        _lib.check(lib.y5_bn_act_bwd_reduce(S.yp, S.ypitch, S.dzp, S.dzpitch, o["dyp"], o["dypitch"], S.rows, c, code, o["mean"].data_ptr(),
                                            o["invstd"].data_ptr(), L.gamma.data_ptr(), L.beta.data_ptr(), act, 0.0, o["dgamma"].data_ptr(),
                                            o["dbeta"].data_ptr(), ws.data_ptr(), st), "bwd_reduce")
        bws.append(ws)
    btotal = torch.stack(bws).sum(0)
    for S, o in zip(shards, outs):
        _lib.check(lib.y5_bn_act_bwd_apply(S.yp, S.ypitch, S.dzp, S.dzpitch, o["dyp"], o["dypitch"], S.rows, c, code, o["mean"].data_ptr(),
                                           o["invstd"].data_ptr(), L.gamma.data_ptr(), act, btotal.data_ptr(), n.data_ptr(), st), "bwd_apply")
    torch.cuda.synchronize()
    return outs


def _check_views_untouched(L, r):
    c = L.ch
    for name, buf, fill in (("z", r["z"], -7.0), ("dy", r["dy"], -13.0)):
        assert bool((buf[:, :8] == fill).all() and (buf[:, 8 + c :] == fill).all()), (name, "wrote outside its channel view")


# ---------------------------------------------------------------------------------------------------------------------
# 1. split == fused, bit for bit, with no all-reduce
# ---------------------------------------------------------------------------------------------------------------------
BN_SHAPES = [  # (channels, rows, residual): the shapes test_train_kernels_gpu.py trains the BN passes at
    (8, 7, False), (40, 7, True), (1280, 7, False),
    (48, 4099, True), (80, 10007, False), (1280, 3001, True),
    (40, 1_600_003, True),
]


def _layer(ch, rows, residual, dtype, dev, seed, integer=True):
    g = torch.Generator(device=dev).manual_seed(seed)
    if integer:
        y, dz = _ints((rows, ch), seed, dev), _ints((rows, ch), seed + 1, dev)
    else:
        y = (torch.rand(rows, ch, generator=g, device=dev) * 4 - 2) * torch.linspace(0.5, 2, ch, device=dev) + 0.3
        dz = torch.rand(rows, ch, generator=g, device=dev) * 2 - 1
    gamma = torch.rand(ch, generator=g, device=dev) + 0.5
    beta = torch.rand(ch, generator=g, device=dev) - 0.5
    res = _ints((rows, ch), seed + 2, dev) if residual else None
    return _Layer(y, dz, gamma, beta, res, dtype, dev)


def _running(ch, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.rand(ch, generator=g, device=dev), torch.rand(ch, generator=g, device=dev) + 0.5


@pytest.mark.parametrize("ch,rows,residual", BN_SHAPES)
@pytest.mark.parametrize("act", [0, 1])
@pytest.mark.parametrize("dtype", DTYPES)
def test_sync_passes_equal_plain(cuda, ch, rows, residual, act, dtype):
    L = _layer(ch, rows, residual, dtype, cuda, ch + rows)
    rm0, rv0 = _running(ch, cuda, rows)
    ref = _fused(L, act, rm0.clone(), rv0.clone())
    (got,) = _sharded(L, act, [0, rows], rm0, rv0)
    for k in ("z", "mean", "invstd", "rm", "rv", "dy", "dgamma", "dbeta"):
        assert _bits(got[k], ref[k]), (k, "the passes with a row count differ from y5_bn_stats + y5_bn_act_fwd / y5_bn_act_bwd without one")
    _check_views_untouched(L, got)


@pytest.mark.parametrize("act", [0, 1])
@pytest.mark.parametrize("dtype", DTYPES)
def test_sync_passes_random_data(cuda, act, dtype):
    """random data: the fp64 column sums may add in another order, so equal to a few ulps (dy: one activation-dtype ulp)"""
    ch, rows = 80, 10007
    L = _layer(ch, rows, True, dtype, cuda, 5, integer=False)
    rm0, rv0 = _running(ch, cuda, 6)
    ref = _fused(L, act, rm0.clone(), rv0.clone())
    (got,) = _sharded(L, act, [0, rows], rm0, rv0)
    for k in ("mean", "invstd", "rm", "rv", "dgamma", "dbeta"):
        torch.testing.assert_close(got[k], ref[k], rtol=4 * 2.0 ** -23, atol=1e-7, msg=k)
    ulp = 2.0 ** -10 if dtype == torch.float16 else 2.0 ** -7
    for k in ("z", "dy"):
        a, b = got[k][:, 8 : 8 + ch].float(), ref[k][:, 8 : 8 + ch].float()
        assert float((a - b).abs().max()) <= ulp * float(b.abs().max()), k


def test_sync_passes_validate_arguments(cuda):
    lib = _lib.lib()
    y = torch.zeros(16, 8, dtype=torch.float16, device=cuda)
    f = torch.zeros(8, device=cuda)
    ws = torch.zeros(17, dtype=torch.float64, device=cuda)
    p = y.data_ptr()
    n = ws[16:].data_ptr()
    assert lib.y5_bn_stats(p, 8, 16, 8, _lib.Y5_F32, ws.data_ptr(), n, None) != 0
    assert lib.y5_bn_stats(p + 2, 8, 16, 8, _lib.Y5_F16, ws.data_ptr(), n, None) != 0  # misaligned view
    assert lib.y5_bn_act_fwd(p, 8, p, 8, 16, 8, _lib.Y5_F16, f.data_ptr(), f.data_ptr(), f.data_ptr(), f.data_ptr(), 1, 0.0, None, n, EPS, MOM,
                             None, None, None, 0, None) != 0  # a row count requires the sums
    assert b"bn_act_fwd" in lib.y5_last_error()
    assert lib.y5_bn_act_bwd_apply(p, 8, p, 8, p, 8, 16, 8, _lib.Y5_F16, f.data_ptr(), f.data_ptr(), f.data_ptr(), 1, ws.data_ptr(), None,
                                   None) != 0  # count is required
    assert lib.y5_bn_act_bwd_reduce(p, 8, p, 8, p, 8, 16, 8, _lib.Y5_F16, f.data_ptr(), f.data_ptr(), f.data_ptr(), f.data_ptr(), 1, 0.0,
                                    None, f.data_ptr(), ws.data_ptr(), None) != 0  # dgamma is required


# ---------------------------------------------------------------------------------------------------------------------
# 2. emulated ranks in one process: uneven shards, workspaces added in fp64
# ---------------------------------------------------------------------------------------------------------------------
SHARDS = {2: [0.37], 3: [0.21, 0.70], 4: [0.1, 0.45, 0.52]}


def _bounds(rows, k):
    return [0] + [max(1, int(rows * f)) for f in SHARDS[k]] + [rows]


@pytest.mark.parametrize("k", [2, 3, 4])
@pytest.mark.parametrize("ch,rows,residual", [(40, 4099, True), (1280, 3001, False), (80, 10007, True)])
@pytest.mark.parametrize("dtype", DTYPES)
def test_emulated_rank_shards_forward_exact(cuda, k, ch, rows, residual, dtype):
    """Integer data: every fp64 sum is exact in any order, so the shards' statistics are the full batch's: z rows, mean,
    invstd and the running statistics (1/N and N/(N-1) formed on the device from the summed count) bit for bit.
    dgamma / dbeta are per-shard fp32 sums of non-integer terms: their sum over shards matches to a few fp32 ulps."""
    L = _layer(ch, rows, residual, dtype, cuda, 17 * k + ch)
    rm0, rv0 = _running(ch, cuda, ch)
    ref = _fused(L, 1, rm0.clone(), rv0.clone())
    b = _bounds(rows, k)
    outs = _sharded(L, 1, b, rm0, rv0)
    for (r0, r1), o in zip(zip(b[:-1], b[1:]), outs):
        for key in ("mean", "invstd", "rm", "rv"):
            assert _bits(o[key], ref[key]), (key, r0, r1)
        assert _bits(o["z"][:, 8 : 8 + ch], ref["z"][r0:r1, 8 : 8 + ch]), ("z", r0, r1)
    for key in ("dgamma", "dbeta"):
        s = torch.stack([o[key].double() for o in outs]).sum(0)
        err = float((s - ref[key].double()).abs().max() / ref[key].double().abs().max())
        assert err <= 1e-6, (key, err)


@pytest.mark.parametrize("k", [2, 3, 4])
@pytest.mark.parametrize("act,rows", [(0, 10007), (1, 390)])
@pytest.mark.parametrize("ch", [40, 1280])
@pytest.mark.parametrize("dtype", DTYPES)
def test_emulated_rank_shards_backward_exact(cuda, k, act, rows, ch, dtype):
    """dy needs both backward sums exact whatever the shard boundaries.  Every column holds +1 and -1 equally often and
    eps = 0, so mean = 0, invstd = 1 and x_hat = y exactly; dz is an integer.  Linear layers then sum integers.  SiLU layers
    sum du = round(dz * silu'(t)) with t = +-gamma + beta in [-3, 3]: multiples of 2^-14 below 2^10 in magnitude over 390
    rows, which fp32 holds exactly."""
    gen = torch.Generator(device=cuda).manual_seed(rows + ch + k)
    half = rows // 2
    col = torch.cat((torch.ones(half, device=cuda), -torch.ones(half, device=cuda)))
    y = torch.stack([col[torch.randperm(2 * half, generator=gen, device=cuda)] for _ in range(ch)], 1)
    dz = _ints((2 * half, ch), rows + 1, cuda)
    gamma = torch.randint(1, 3, (ch,), generator=gen, device=cuda).float()
    beta = torch.randint(-1, 2, (ch,), generator=gen, device=cuda).float()
    L = _Layer(y, dz, gamma, beta, None, dtype, cuda)
    rm0, rv0 = _running(ch, cuda, 3)
    ref = _fused(L, act, rm0.clone(), rv0.clone(), eps=0.0)
    assert bool((ref["invstd"] == 1).all()) and bool((ref["mean"] == 0).all())
    b = _bounds(2 * half, k)
    outs = _sharded(L, act, b, rm0, rv0, eps=0.0)
    for (r0, r1), o in zip(zip(b[:-1], b[1:]), outs):
        for key in ("rm", "rv"):
            assert _bits(o[key], ref[key]), (key, r0, r1)
        for key in ("z", "dy"):
            assert _bits(o[key][:, 8 : 8 + ch], ref[key][r0:r1, 8 : 8 + ch]), (key, r0, r1)
        _check_views_untouched(L, o)
    for key in ("dgamma", "dbeta"):  # exact here: integer-valued or exactly summed terms
        s = torch.stack([o[key].double() for o in outs]).sum(0)
        assert torch.equal(s, ref[key].double()), key


# ---------------------------------------------------------------------------------------------------------------------
# model-level helpers
# ---------------------------------------------------------------------------------------------------------------------
def _model(dev, seed=31, sync=False, head_bias="init"):
    from oracle import model_ref
    from yolov5_b200.cfg import HYP_SCRATCH_LOW, model_cfg
    from yolov5_b200.models.yolo import DetectionModel

    m = DetectionModel("yolov5n")
    m.load_state_dict(model_ref.synth_state_dict(model_cfg("yolov5n"), seed=seed, head_bias=head_bias))
    if sync:
        m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(m)
    m = m.to(dev).train()
    m.hyp = dict(HYP_SCRATCH_LOW)
    return m


MAP_SHAPES = [(3, 128 // s, 128 // s, 85) for s in (8, 16, 32)]  # yolov5n's head maps of a 128x128 image (na, ny, nx, no)


def _batch(dev, n=4, size=128, seed=100):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(n, 3, size, size, generator=g) * 255).to(torch.uint8).to(dev)


def _dzs(shapes, dev, seed=7):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(s, generator=g) * 1e-2).to(dev) for s in shapes]


def _linear_step(m, img, dzs, dtype=torch.float16):
    """train-mode forward of `img`, backward of sum(head maps * dzs); returns (maps, {name: grad})"""
    for q in m.parameters():
        q.grad = None
    with torch.autocast("cuda", dtype=dtype):
        p = m(img)
    sum((q.float() * d).sum() for q, d in zip(p, dzs)).backward()
    torch.cuda.synchronize()
    return [q.detach().float() for q in p], {k: q.grad.detach().clone() for k, q in m.named_parameters()}


def _buffers(m):
    return {k: v.detach().clone() for k, v in m.named_buffers() if "running" in k}


def _rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


# ---------------------------------------------------------------------------------------------------------------------
# 3. two processes on one GPU (gloo, which all-reduces CUDA tensors)
# ---------------------------------------------------------------------------------------------------------------------
def _gloo_worker(rank, world, store, out_dir):
    import torch.distributed as dist

    from yolov5_b200.utils.torch_utils import GraphedTrainStep, smart_optimizer
    from yolov5_b200.utils.loss import ComputeLoss

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", init_method=f"file://{store}", rank=rank, world_size=world)
    try:
        m = _model(dev, sync=True)
        assert sum(isinstance(x, torch.nn.SyncBatchNorm) for x in m.modules()) > 50
        img = _batch(dev)[2 * rank : 2 * rank + 2]
        dzs = [d[2 * rank : 2 * rank + 2] for d in _dzs([(4, *s) for s in MAP_SHAPES], dev)]
        maps, grads = _linear_step(m, img, dzs)
        refused = ""
        try:
            opt = smart_optimizer(m, "SGD", lr=0.01, momentum=0.9, decay=5e-4)
            GraphedTrainStep(m, ComputeLoss(m), opt, batch=2, size=128)
        except NotImplementedError as e:
            refused = str(e)
        torch.save({"maps": [q.cpu() for q in maps], "grads": {k: v.cpu() for k, v in grads.items()},
                    "buffers": {k: v.cpu() for k, v in _buffers(m).items()}, "refused": refused}, os.path.join(out_dir, f"r{rank}.pt"))
    finally:
        dist.destroy_process_group()


def _spawn(fn, world, args, timeout=600):
    """start `world` ranks, join them within `timeout` seconds; on failure or timeout no rank outlives the call"""
    import torch.multiprocessing as mp

    ctx = mp.spawn(fn, args=(world, *args), nprocs=world, join=False)
    deadline = time.monotonic() + timeout
    try:
        while not ctx.join(timeout=5):
            if time.monotonic() > deadline:
                raise TimeoutError(f"ranks did not finish within {timeout} s")
    finally:
        for p in ctx.processes:
            if p.is_alive():
                p.terminate()
            p.join(10)
            if p.is_alive():
                p.kill()
                p.join()


def test_two_processes_one_gpu_match_one_process(cuda, tmp_path):
    world = 2
    _spawn(_gloo_worker, world, (str(tmp_path / "store"), str(tmp_path)))
    rs = [torch.load(tmp_path / f"r{r}.pt") for r in range(world)]
    # one process, the four images, plain BatchNorm2d, same weights
    m = _model(cuda)
    img = _batch(cuda)
    dzs = _dzs([(4, *s) for s in MAP_SHAPES], cuda)
    maps, grads = _linear_step(m, img, dzs)
    bufs = _buffers(m)
    for r, out in enumerate(rs):
        for a, b in zip(out["maps"], maps):
            for i in range(2):
                err = _rel_l2(a[i], b[2 * r + i].cpu())
                assert err < 1e-2, ("head map", r, i, err)
        assert "SyncBatchNorm" in out["refused"], out["refused"]
    # Running buffers: identical on both ranks.  Against the single process, the convolutions of a 2-image and a 4-image
    # batch may round an fp16 output differently (another tile plan), so deeper layers see slightly different inputs: the
    # one-step update of each buffer (new - initial) is compared like the head maps.
    init = _buffers(_model(cuda))
    worst = (0.0, "")
    for k, v in bufs.items():
        assert torch.equal(rs[0]["buffers"][k], rs[1]["buffers"][k]), (k, "running buffers differ between ranks")
        err = _rel_l2(rs[0]["buffers"][k] - init[k].cpu(), (v - init[k]).cpu())
        worst = max(worst, (err, k))
    print(f"running-buffer updates, worst relative L2 vs one process: {worst}")
    assert worst[0] < 1e-2, worst
    # gradients: the sum over ranks is the whole batch's.  Without the sync the same two halves give another gradient.
    g_sum = torch.cat([(rs[0]["grads"][k] + rs[1]["grads"][k]).float().flatten() for k in grads])
    g_ref = torch.cat([grads[k].float().flatten().cpu() for k in grads])
    halves = [_linear_step(_model(cuda), img[2 * r : 2 * r + 2], [d[2 * r : 2 * r + 2] for d in dzs])[1] for r in range(2)]
    g_local = torch.cat([(halves[0][k] + halves[1][k]).float().flatten().cpu() for k in grads])
    _, g_again = _linear_step(_model(cuda), img, dzs)
    assert torch.isfinite(g_sum).all()
    err, err_local = _rel_l2(g_sum, g_ref), _rel_l2(g_local, g_ref)
    noise = _rel_l2(torch.cat([g_again[k].float().flatten().cpu() for k in grads]), g_ref)
    # float64 gradient of the same loss through the reference's expressions (CPU): the synced sum must be as close to it as
    # the one-process gradient is
    from oracle import model_ref
    from yolov5_b200.cfg import model_cfg

    sd64 = {k: v.double().requires_grad_(k in grads) for k, v in _model("cpu").state_dict().items()}
    maps64 = model_ref.forward(model_cfg("yolov5n"), sd64, img.cpu().double() / 255, training=True, bn_batch_stats=True)
    sum((q * d.cpu().double()).sum() for q, d in zip(maps64, dzs)).backward()
    g64 = torch.cat([sd64[k].grad.flatten() for k in grads])
    e_one, e_sync = _rel_l2(g_ref, g64), _rel_l2(g_sum, g64)
    print(f"gradient sum over ranks vs one process: rel L2 {err:.3e}; unsynced halves {err_local:.3e}; run to run {noise:.3e}; "
          f"vs float64: one process {e_one:.3e}, ranks {e_sync:.3e}")
    # The 2- and 4-image convolutions round their fp16 outputs differently (another tile plan), and with gradients that cancel
    # over the batch this leaves the two fp16 gradients 3.5e-2 apart (measured on an H100); each is 0.12 from float64.  The
    # sync is what brings the sum to the whole batch: without it the same halves are 1.5 away.
    assert err < 5e-2, err
    assert err < err_local / 20, (err, err_local)
    assert e_sync < 1.25 * e_one, (e_sync, e_one)


# ---------------------------------------------------------------------------------------------------------------------
# 4. two GPUs, NCCL: smart_DDP and FusedSGD.data_parallel
# ---------------------------------------------------------------------------------------------------------------------
def _nccl_worker(rank, world, port, out_dir):
    import torch.distributed as dist

    from oracle import loss_ref
    from yolov5_b200.utils.loss import ComputeLoss
    from yolov5_b200.utils.torch_utils import smart_DDP, smart_optimizer

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        img = _batch(dev, n=2, seed=100 + rank)
        tgt = torch.from_numpy(loss_ref.synth_targets(2, seed=200 + rank)).float().to(dev)
        out = {}
        for mode in ("ddp", "native"):
            m = _model(dev, sync=True)
            opt = smart_optimizer(m, "SGD", lr=0.01, momentum=0.9, decay=5e-4)
            net = m
            if mode == "ddp":
                net = smart_DDP(m)
            else:
                opt.data_parallel(m)
            with torch.autocast("cuda", dtype=torch.float16):
                p = net(img)
            loss, _ = ComputeLoss(m)(p, tgt)
            (loss * world).backward()
            opt.fused_step(max_norm=10.0)
            torch.cuda.synchronize()
            out[mode] = {"params": torch.cat([q.detach().flatten() for q in m.parameters()]).cpu(),
                         "buffers": torch.cat([b.detach().float().flatten() for k, b in m.named_buffers() if "running" in k]).cpu()}
        torch.save(out, os.path.join(out_dir, f"n{rank}.pt"))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_ddp_and_data_parallel(cuda, tmp_path):
    _spawn(_nccl_worker, 2, (29691, str(tmp_path)))
    a, b = torch.load(tmp_path / "n0.pt"), torch.load(tmp_path / "n1.pt")
    start = torch.cat([q.detach().flatten() for q in _model("cpu").parameters()])
    for mode in ("ddp", "native"):
        assert torch.isfinite(a[mode]["params"]).all(), mode
        assert not torch.equal(a[mode]["params"], start), mode
        assert torch.equal(a[mode]["params"], b[mode]["params"]), (mode, "parameters differ between ranks")
        assert torch.equal(a[mode]["buffers"], b[mode]["buffers"]), (mode, "running buffers differ between ranks")


# ---------------------------------------------------------------------------------------------------------------------
# 5. single process: a SyncBatchNorm that does not sync is BatchNorm2d
# ---------------------------------------------------------------------------------------------------------------------
def test_single_process_sync_bn_is_batchnorm(cuda):
    import torch.distributed as dist

    from oracle import loss_ref
    from yolov5_b200.utils.loss import ComputeLoss

    assert not dist.is_initialized()
    img = _batch(cuda, n=2)
    tgt = torch.from_numpy(loss_ref.synth_targets(2, seed=3)).float().to(cuda)

    def step(m):
        for q in m.parameters():
            q.grad = None
        torch.cuda.synchronize()
        n0 = _lib.launch_count()
        with torch.autocast("cuda", dtype=torch.float16):
            p = m(img)
        loss, items = ComputeLoss(m)(p, tgt)
        loss.backward()
        torch.cuda.synchronize()
        return (_lib.launch_count() - n0, items.detach().clone(), {k: q.grad.detach().clone() for k, q in m.named_parameters()},
                _buffers(m))

    plain, plain2, conv = _model(cuda), _model(cuda), _model(cuda, sync=True)
    assert all(train_ops.bn_sync_group(x) is None for x in conv.modules())
    for mm in (plain, plain2, conv):  # first forward: weight packing registers every filter
        step(mm)
        mm.load_state_dict(_model(cuda).state_dict())
    na, ia, ga, ba = step(plain)
    nb, ib, gb, _ = step(plain2)
    nc, ic, gc, bc = step(conv)
    assert na == nb == nc, ("launches per step", na, nb, nc)  # the sync path would add a finalize launch per BN layer
    torch.testing.assert_close(ic, ia, rtol=1e-4, atol=1e-6)
    for k in ba:  # batch statistics: fp64 column sums, equal up to their summation order
        torch.testing.assert_close(bc[k], ba[k], rtol=1e-5, atol=1e-6, msg=k)
    noise = {k: _rel_l2(gb[k], ga[k]) for k in ga}  # weight gradients: fp32 atomics, different run to run
    bad = [(k, _rel_l2(gc[k], ga[k]), noise[k]) for k in ga if _rel_l2(gc[k], ga[k]) > 2 * noise[k] + 1e-6]
    assert not bad, bad[:5]


# ---------------------------------------------------------------------------------------------------------------------
# 6. eval and checkpoints
# ---------------------------------------------------------------------------------------------------------------------
def _detect(m, img):
    from yolov5_b200.utils.general import non_max_suppression

    with torch.no_grad():
        z = m(img.half() / 255)[0]
    return z, non_max_suppression(z, 0.001, 0.6, max_det=300)


def test_converted_model_eval_and_checkpoint(cuda, tmp_path):
    from yolov5_b200.models.experimental import attempt_load

    img = _batch(cuda, n=2)
    plain = _model(cuda, seed=20, head_bias="hot")
    conv = _model(cuda, seed=20, sync=True, head_bias="hot")
    assert any(isinstance(x, torch.nn.SyncBatchNorm) for x in conv.modules())
    zp, dp = _detect(plain.half().eval(), img)
    zc, dc = _detect(conv.half().eval(), img)
    assert torch.equal(zc, zp)
    for a, b in zip(dc, dp):
        assert torch.equal(a, b)
    # checkpoints as train.py saves them with --sync-bn: the whole module pickled, SyncBatchNorm layers included
    for name, m in (("plain", _model("cpu", seed=20, head_bias="hot")), ("sync", _model("cpu", seed=20, sync=True, head_bias="hot"))):
        torch.save({"model": m.half(), "ema": None}, tmp_path / f"{name}.pt")
    lp = attempt_load(str(tmp_path / "plain.pt"), device=cuda).half()
    ls = attempt_load(str(tmp_path / "sync.pt"), device=cuda).half()
    zlp, dlp = _detect(lp, img)
    zls, dls = _detect(ls, img)
    assert torch.equal(zls, zlp)
    for a, b in zip(dls, dlp):
        assert torch.equal(a, b)
    assert len(dlp[0]) > 0
