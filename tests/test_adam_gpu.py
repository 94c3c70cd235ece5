"""GPU: `--optimizer Adam | AdamW` on the fused step (FusedAdam / y5_adam_step) -- against the oracle and the reference-generated
fixture, against torch.optim.Adam / AdamW with GradScaler + clip_grad_norm_ over real yolov5n steps, through plain step(),
state_dict round trips with torch, GraphedTrainStep replay and the data-parallel gradient arena."""
import os
from copy import deepcopy

import numpy as np
import pytest
import torch

from oracle import adam_ref
from tests.test_optim_gpu import _train_setup
from yolov5_b200.utils.loss import ComputeLoss
from yolov5_b200.utils.torch_utils import FusedAdam, FusedAdamW, GraphedTrainStep, ModelEMA, smart_optimizer

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")


def _steps(opt, params):
    """Step counts of `params` as opt.state_dict() reports them (0-d fp32 CPU tensors, keyed by position in param_groups)."""
    state = opt.state_dict()["state"]
    index = {id(p): i for i, p in enumerate(q for g in opt.param_groups for q in g["params"])}
    out = []
    for p in params:
        st = state[index[id(p)]]["step"]
        assert st.device.type == "cpu" and st.dtype == torch.float32 and st.dim() == 0
        out.append(float(st))
    return out


@pytest.mark.parametrize("ci", range(len(adam_ref.CASES)))
def test_fused_adam_vs_oracle_and_reference_fixture(cuda, ci):
    g = np.load(os.path.join(G, "adam.npz"))
    case = adam_ref.CASES[ci]
    params, running, m0, v0 = adam_ref.synth_net(50 + ci)
    net = adam_ref.make_net(params, running).to(cuda)
    ps = list(net.parameters())

    def build():
        return smart_optimizer(net, case["opt"], case["lr"], case["momentum"], case["decay"])

    opt = build()
    if "start_step" in case:  # a state loaded before the tables exist
        for i, p in enumerate(ps):
            opt.state[p] = dict(step=torch.tensor(float(case["start_step"])), exp_avg=torch.from_numpy(m0[i].copy()).to(cuda),
                                exp_avg_sq=torch.from_numpy(v0[i].copy()).to(cuda))
    ema = ModelEMA(net, decay=0.9999, tau=2000, updates=adam_ref.EMA_UPDATES0)
    scaler = torch.amp.GradScaler("cuda", init_scale=1.0, growth_interval=1000)
    scaler.scale(torch.zeros(1, device=cuda))  # lazy-init the device scale
    for k, spec in enumerate(case["steps"]):
        if case.get("resume_after") == k:  # smart_resume into a fresh optimizer
            sd = deepcopy(opt.state_dict())
            opt = build()
            opt.load_state_dict(sd)
        for p, gr in zip(ps, adam_ref.synth_grads(50 + ci, k, spec)):
            p.grad = None if gr is None else torch.from_numpy(gr).to(cuda)
        scaler._scale.fill_(1.0 / spec.get("inv_scale", 1.0))
        opt.fused_step(scaler=scaler, max_norm=spec["max_norm"], ema=ema, model=net)
        opt.zero_grad()
        assert opt.last_step_skipped == bool(g[f"c{ci}.skipped"][k]), k
        if "poison" in spec:  # GradScaler.update: halved on the overflow step
            assert float(scaler.get_scale()) == 0.5 / spec["inv_scale"]
    want = adam_ref.run_case(ci)
    s = adam_ref.FIXTURE_STRIDE
    ema_ps = list(ema.ema.parameters())
    for i, p in enumerate(ps):
        st = opt.state[p]
        for tag, got, ref in (("p", p.detach(), want["params"][i]), ("m", st["exp_avg"], want["exp_avgs"][i]),
                              ("v", st["exp_avg_sq"], want["exp_avg_sqs"][i]), ("e", ema_ps[i], want["emas"][i])):
            got = got.cpu().numpy()
            assert np.allclose(got, ref, rtol=3e-6, atol=2e-7), (ci, tag, i, np.abs(got - ref).max())
            assert np.allclose(got.reshape(-1)[::s], g[f"c{ci}.{tag}{i}"], rtol=3e-6, atol=2e-7), (ci, tag, i)  # the real reference
    for j, b in enumerate((ema.ema.bn.running_mean, ema.ema.bn.running_var)):
        assert np.allclose(b.cpu().numpy(), g[f"c{ci}.ebuf{j}"], rtol=3e-6, atol=2e-7)
    assert _steps(opt, ps) == list(g[f"c{ci}.steps"]) == want["steps"]
    assert ema.updates == adam_ref.EMA_UPDATES0 + len(case["steps"])


@pytest.mark.parametrize("decoupled", [False, True])
def test_first_steps_use_fp64_bias_correction(cuda, decoupled):
    """From zero weights the update IS the new weight, so it is compared at 1e-6: torch's bias corrections are Python doubles
    (an fp32 1 - 0.999 alone is 1.3e-5 off)."""
    rs = np.random.RandomState(3)
    p = torch.nn.Parameter(torch.zeros(40000, device=cuda))
    opt = (FusedAdamW if decoupled else FusedAdam)([p], lr=0.01, betas=(0.9, 0.999), weight_decay=0.0)
    pn, m, v, steps = [np.zeros(40000, np.float32)], [np.zeros(40000, np.float32)], [np.zeros(40000, np.float32)], [0.0]
    hyper = [dict(lr=0.01, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, decoupled_weight_decay=decoupled)]
    for k in range(2):
        gr = rs.normal(0, 1, 40000).astype(np.float32)
        before = p.detach().cpu().numpy()
        p.grad = torch.from_numpy(gr).to(cuda)
        opt.step()
        prev = pn[0]
        pn, m, v, steps, _, _ = adam_ref.adam_step(pn, [gr], m, v, steps, [0], hyper, max_norm=None)
        got = p.detach().cpu().numpy() - before
        want = pn[0] - prev
        # step 1 starts from zero weights (exact); at step 2 the weight's own rounding (about 1e-9) sits on top
        assert np.allclose(got, want, rtol=1e-6, atol=0 if k == 0 else 2e-8), (k, np.abs(got - want).max())
        assert np.allclose(opt.state[p]["exp_avg_sq"].cpu().numpy(), v[0], rtol=1e-6, atol=0)
    assert _steps(opt, [p]) == [2.0]


def test_every_block_sees_the_same_step_count(cuda):
    """A tensor of more thread blocks than the GPU holds at once: late blocks must still see the pre-step count."""
    torch.manual_seed(0)
    pa = torch.nn.Parameter(torch.randn(24_000_000, device=cuda) * 0.1)
    pb = torch.nn.Parameter(pa.detach().clone())
    oa = FusedAdam([pa], lr=0.01, betas=(0.9, 0.999))
    ob = torch.optim.Adam([pb], lr=0.01, betas=(0.9, 0.999))
    for _ in range(3):
        gr = torch.randn_like(pa)
        pa.grad, pb.grad = gr, gr.clone()
        oa.step()
        ob.step()
    assert torch.allclose(pa, pb, rtol=1e-5, atol=1e-7), float((pa - pb).abs().max())
    assert _steps(oa, [pa]) == [3.0]


def _torch_twin(m, name, lr, momentum, decay):
    groups = [[], [], []]
    for v in m.modules():
        for n, p in v.named_parameters(recurse=False):
            groups[2 if n == "bias" else 1 if isinstance(v, torch.nn.BatchNorm2d) and n == "weight" else 0].append(p)
    if name == "Adam":
        opt = torch.optim.Adam(groups[2], lr=lr, betas=(momentum, 0.999))
    else:
        opt = torch.optim.AdamW(groups[2], lr=lr, betas=(momentum, 0.999), weight_decay=0.0)
    opt.add_param_group({"params": groups[0], "weight_decay": decay})
    opt.add_param_group({"params": groups[1], "weight_decay": 0.0})
    return opt


@pytest.mark.parametrize("name", ["Adam", "AdamW"])
def test_fused_adam_tracks_torch_adam_clip_gradscaler_over_real_steps(cuda, name):
    """Three real yolov5n steps (fp16 autocast, GradScaler) drive smart_optimizer(m, name).fused_step and, on the same scaled
    gradients, torch.optim.Adam / AdamW in the reference's three groups with the train.py:413-421 sequence.  One step overflows."""
    ma, imgs, tgts = _train_setup(cuda)
    mb, _, _ = _train_setup(cuda)
    la = ComputeLoss(ma)
    oa = smart_optimizer(ma, name, lr=0.01, momentum=0.937, decay=5e-2)
    ob = _torch_twin(mb, name, lr=0.01, momentum=0.937, decay=5e-2)
    sa, sb = torch.amp.GradScaler("cuda"), torch.amp.GradScaler("cuda")
    sb.scale(torch.zeros(1, device=cuda))
    ea, eb = ModelEMA(ma), ModelEMA(mb)
    pa, pb = list(ma.parameters()), list(mb.parameters())
    for i in range(3):
        with torch.autocast("cuda", dtype=torch.float16):
            pred = ma(imgs[i])
        loss_a, _ = la(pred, tgts[i])
        sa.scale(loss_a).backward()
        for qa, qb in zip(pa, pb):
            qb.grad = qa.grad.clone()
        if i == 1:
            pa[5].grad.view(-1)[0] = float("inf")
            pb[5].grad.view(-1)[0] = float("inf")
        oa.fused_step(scaler=sa, max_norm=10.0, ema=ea, model=ma)
        oa.zero_grad()
        sb.unscale_(ob)
        torch.nn.utils.clip_grad_norm_(pb, max_norm=10.0)
        sb.step(ob)
        sb.update()
        ob.zero_grad()
        with torch.no_grad():
            for (_, ba), (_, bb) in zip(ma.named_buffers(), mb.named_buffers()):
                bb.copy_(ba)
        eb.update(mb)
        assert float(sa.get_scale()) == float(sb.get_scale()), i
        assert oa.last_step_skipped == (i == 1)
    assert float(sa.get_scale()) == 32768.0
    for (k, a), b in zip(ma.named_parameters(), pb):
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-7), (k, float((a - b).abs().max()))
        for key in ("exp_avg", "exp_avg_sq"):
            assert torch.allclose(oa.state[a][key], ob.state[b][key], rtol=1e-5, atol=1e-7), (k, key)
    assert _steps(oa, pa) == [float(ob.state[b]["step"]) for b in pb] and set(_steps(oa, pa)) == {2.0}
    for (k, a), b in zip(ea.ema.state_dict().items(), eb.ema.state_dict().values()):
        if a.dtype.is_floating_point:
            assert torch.allclose(a, b, rtol=1e-5, atol=1e-7), k


def _grad_net(cuda, seed=0):
    params, running, _, _ = adam_ref.synth_net(seed)
    return adam_ref.make_net(params, running).to(cuda)


def _set_grads(nets, k, drop=()):
    rs = np.random.RandomState(500 + k)
    for i, ps in enumerate(zip(*[list(n.parameters()) for n in nets])):
        gr = torch.from_numpy(rs.normal(0, 2.0, ps[0].shape).astype(np.float32) * 1024).to(ps[0].device)
        for p in ps:
            p.grad = None if i in drop else gr.clone()


def test_plain_step_under_unmodified_train_loop_equals_fused_step(cuda):
    """train.py's own calls -- scaler.unscale_(opt), clip_grad_norm_, scaler.step(opt), scaler.update() -- on FusedAdamW equal
    fused_step(scaler, 10.0) on a twin."""
    na, nb = _grad_net(cuda), _grad_net(cuda)
    oa = smart_optimizer(na, "AdamW", 0.01, 0.9, 0.05)
    ob = smart_optimizer(nb, "AdamW", 0.01, 0.9, 0.05)
    sa = torch.amp.GradScaler("cuda", init_scale=1024.0)
    sb = torch.amp.GradScaler("cuda", init_scale=1024.0)
    sa.scale(torch.zeros(1, device=cuda))
    sb.scale(torch.zeros(1, device=cuda))
    for k in range(3):
        _set_grads([na, nb], k, drop=(4,) if k == 1 else ())
        sa.unscale_(oa)
        torch.nn.utils.clip_grad_norm_(na.parameters(), max_norm=10.0)
        sa.step(oa)
        sa.update()
        oa.zero_grad()
        ob.fused_step(scaler=sb, max_norm=10.0)
        ob.zero_grad()
    for a, b in zip(na.parameters(), nb.parameters()):
        # equal up to clip_grad_norm_'s own norm (torch's reduction order, not the kernel's) and its separate multiply
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-7), float((a - b).abs().max())
        assert torch.allclose(oa.state[a]["exp_avg"], ob.state[b]["exp_avg"], rtol=1e-5, atol=1e-7)
    assert _steps(oa, na.parameters()) == _steps(ob, nb.parameters()) == [3.0, 3.0, 3.0, 3.0, 2.0, 3.0, 3.0]


@pytest.mark.parametrize("name", ["Adam", "AdamW"])
def test_state_dict_round_trips_with_torch(cuda, name):
    """A torch Adam / AdamW state loads into an engine optimizer whose tables already exist, and the next step matches torch's;
    the engine's state loads into torch and its next step matches the engine's."""
    ne, nt = _grad_net(cuda), _grad_net(cuda)
    oe = smart_optimizer(ne, name, 0.01, 0.9, 0.05)
    ot = _torch_twin(nt, name, 0.01, 0.9, 0.05)
    _set_grads([ne], 7)
    oe.step()  # tables built, state that the load must replace
    for k in range(2):
        _set_grads([nt], k, drop=(2,) if k == 0 else ())
        ot.step()
    with torch.no_grad():
        for a, b in zip(ne.parameters(), nt.parameters()):
            a.copy_(b)
    oe.load_state_dict(deepcopy(ot.state_dict()))
    assert _steps(oe, ne.parameters()) == [2.0, 2.0, 1.0, 2.0, 2.0, 2.0, 2.0]
    for k in (2, 3):
        _set_grads([ne, nt], k)
        oe.step()
        ot.step()
        for a, b in zip(ne.parameters(), nt.parameters()):
            assert torch.allclose(a, b, rtol=1e-5, atol=1e-7), (k, float((a - b).abs().max()))
    # the reverse direction: the engine's state into a fresh torch optimizer
    sd = oe.state_dict()
    ot2 = _torch_twin(nt, name, 0.01, 0.9, 0.05)
    ot2.load_state_dict(deepcopy(sd))
    _set_grads([ne, nt], 4)
    oe.step()
    ot2.step()
    for a, b in zip(ne.parameters(), nt.parameters()):
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-7), float((a - b).abs().max())
    assert _steps(oe, ne.parameters()) == [float(ot2.state[b]["step"]) for b in nt.parameters()] == [5.0, 5.0, 4.0, 5.0, 5.0, 5.0, 5.0]


def test_graphed_train_step_with_adamw(cuda):
    """GraphedTrainStep with AdamW = the eager fused loop: loss items, scale and counters, the first replayed step is step 1,
    and the learning rate is changed between replays (criteria of the SGD graph test)."""
    ma, imgs, tgts = _train_setup(cuda, seed=1)
    mb, _, _ = _train_setup(cuda, seed=1)
    oa = smart_optimizer(ma, "AdamW", lr=0.001, momentum=0.937, decay=5e-4)
    ob = smart_optimizer(mb, "AdamW", lr=0.001, momentum=0.937, decay=5e-4)
    ea, eb = ModelEMA(ma), ModelEMA(mb)
    step = GraphedTrainStep(ma, ComputeLoss(ma), oa, batch=2, size=128, ema=ea)
    assert set(_steps(oa, ma.parameters())) == {0.0} and float(oa._flat.abs().max()) == 0.0  # warm-up state undone
    lb, sb = ComputeLoss(mb), torch.amp.GradScaler("cuda")
    w0 = torch.cat([v.detach().flatten() for v in ma.parameters()]).clone()
    for i in range(3):
        lr = 0.001 * (1 + i)
        for g_ in oa.param_groups + ob.param_groups:
            g_["lr"] = lr
        items_a = step(imgs[i], tgts[i]).clone()
        torch.cuda.synchronize()
        if i == 0:
            assert set(_steps(oa, ma.parameters())) == {1.0}
        with torch.autocast("cuda", dtype=torch.float16):
            pb = mb(imgs[i])
        loss_b, items_b = lb(pb, tgts[i])
        sb.scale(loss_b).backward()
        ob.fused_step(scaler=sb, max_norm=10.0, ema=eb, model=mb)
        ob.zero_grad()
        assert torch.allclose(items_a, items_b, rtol=3e-2, atol=1e-4), (i, items_a, items_b)
        if i == 0:
            # Adam's first step moves every weight by about lr whatever its gradient: compare relative to that
            wa = torch.cat([v.detach().flatten() for v in ma.parameters()])
            wb = torch.cat([v.detach().flatten() for v in mb.parameters()])
            moved = float((wb - w0).norm())
            assert moved > 0 and float((wa - wb).norm()) <= 0.05 * moved, (float((wa - wb).norm()), moved)
    assert ea.updates == eb.updates == 3 and float(step.scaler.get_scale()) == float(sb.get_scale())
    assert _steps(oa, ma.parameters()) == _steps(ob, mb.parameters())
    assert all(bool(torch.isfinite(v).all()) for v in ma.parameters())


def test_data_parallel_mode_world1_steps_identically(cuda):
    """FusedAdam.data_parallel in a one-rank group: the step from the gradient arena is bit-identical to the plain step,
    including a parameter without a gradient (its step count stays behind)."""
    import torch.distributed as dist

    own_group = not dist.is_initialized()
    if own_group:
        dist.init_process_group("nccl", init_method="tcp://127.0.0.1:29687", rank=0, world_size=1, device_id=cuda)
    try:
        torch.manual_seed(5)
        shapes = [(33, 7, 3, 3), (33,), (1,), (64, 33, 1, 1), (5,), (70001,)]
        ma = torch.nn.ParameterList([torch.nn.Parameter(torch.randn(s, device=cuda)) for s in shapes])
        mb = torch.nn.ParameterList([torch.nn.Parameter(p.detach().clone()) for p in ma])
        oa = FusedAdamW(list(ma), lr=0.05, weight_decay=1e-2)
        ob = FusedAdamW(list(mb), lr=0.05, weight_decay=1e-2)
        oa.data_parallel(ma)
        for it in range(3):
            for i, (pa, pb) in enumerate(zip(ma, mb)):
                if i == 4 and it == 2:
                    pa.grad = pb.grad = None
                    continue
                g = torch.randn_like(pa) * (10.0 if it == 1 else 1.0)
                pa.grad, pb.grad = g, g.clone()
            oa.fused_step(max_norm=10.0)
            ob.fused_step(max_norm=10.0)
            for pa, pb in zip(ma, mb):
                assert torch.equal(pa, pb)
                assert torch.equal(oa.state[pa]["exp_avg_sq"], ob.state[pb]["exp_avg_sq"])
            assert oa.last_grad_norm == ob.last_grad_norm
            oa.zero_grad()
            ob.zero_grad()
        assert _steps(oa, ma) == _steps(ob, mb) == [3.0, 3.0, 3.0, 3.0, 2.0, 3.0]
    finally:
        if own_group:
            dist.destroy_process_group()
