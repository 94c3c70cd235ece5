"""ORACLE (test infrastructure, never on the product path): numpy restatement of the step right after backward with
`--optimizer Adam | AdamW` -- reference train.py:413-421:  scaler.unscale_(optimizer); clip_grad_norm_(params, 10.0);
scaler.step(optimizer); optimizer.zero_grad(); ema.update(model)  with optimizer = torch.optim.Adam(betas=(momentum, 0.999))
or AdamW(betas=(momentum, 0.999), weight_decay=0) plus the two decay groups of utils/torch_utils.py:257-290, and ModelEMA.update
of utils/torch_utils.py:359-368.  float32 arithmetic; the bias corrections, 1 - beta and 1 - lr * weight_decay in float64,
rounded to float32 where torch rounds its Python scalars.

Only tests/ may import this.  Pinned: tests/golden/adam.npz holds the result of the real reference objects (its
smart_optimizer, torch.nn.utils.clip_grad_norm_ and ModelEMA through tests/golden/refshim.py) on the seeded problems below;
tests/golden/make_adam_golden.py asserts that this file equals them, tests/test_adam_cpu.py checks it against the fixture.
"""
from __future__ import annotations

import math

import numpy as np

F = np.float32

# the test network: (parameter name, shape, parameter group of the reference's smart_optimizer: 0 biases, 1 decayed weights,
# 2 BatchNorm weights -- param_groups order [g[2], g[0], g[1]]).  lin.weight spans two 16K-element chunks; fc.weight gets
# gradients small enough that eps shapes its update.
NET = (("conv.weight", (16, 8, 3, 3), 1), ("bn.weight", (16,), 2), ("bn.bias", (16,), 0), ("fc.weight", (32, 16, 1, 1), 1),
       ("fc.bias", (32,), 0), ("lin.weight", (100, 170), 1), ("lin.bias", (100,), 0))
SMALL_GRAD = 3  # index of fc.weight
EMA_UPDATES0 = 100

# each case: optimizer, smart_optimizer's lr / momentum / decay, per-step dicts (inv_scale, max_norm, drop = indices without a
# gradient, poison = index with an inf gradient), optional resume_after (a state_dict round trip before that step) and
# start_step (every parameter starts with this step count and seeded moments)
CASES = (
    dict(opt="Adam", lr=0.01, momentum=0.937, decay=5e-4, steps=[dict(inv_scale=1 / 1024, max_norm=10.0)] * 3),
    dict(opt="AdamW", lr=0.01, momentum=0.9, decay=0.05, steps=[dict(max_norm=1e9), dict(max_norm=1e9, drop=(2, 6)), dict(max_norm=1e9)]),
    dict(opt="Adam", lr=0.002, momentum=0.8, decay=1e-3, steps=[dict(max_norm=10.0, drop=(5,)), dict(inv_scale=1 / 8, max_norm=10.0, poison=4),
                                                                 dict(inv_scale=1 / 4, max_norm=10.0)]),
    dict(opt="AdamW", lr=0.01, momentum=0.937, decay=0.01, steps=[dict(max_norm=10.0)] * 3, resume_after=2),
    dict(opt="Adam", lr=0.001, momentum=0.9, decay=5e-4, steps=[dict(max_norm=1e9)]),
    dict(opt="AdamW", lr=0.001, momentum=0.9, decay=5e-4, steps=[dict(max_norm=1e9)], start_step=9999),
)


def group_of():
    return [g for _, _, g in NET]


def hyper(case):
    """Per parameter group (smart_optimizer's order): dicts of lr, betas, eps, weight_decay, decoupled_weight_decay."""
    decoupled = case["opt"] == "AdamW"
    base = dict(lr=case["lr"], betas=(case["momentum"], 0.999), eps=1e-8, decoupled_weight_decay=decoupled)
    return [dict(base, weight_decay=0.0), dict(base, weight_decay=case["decay"]), dict(base, weight_decay=0.0)]


def synth_net(seed: int):
    """Seeded parameters, BN running statistics and initial optimizer state (float32)."""
    rs = np.random.RandomState(seed)
    params = [rs.normal(0, 0.3, s).astype(F) for _, s, _ in NET]
    running = [rs.normal(0, 1, 16).astype(F), rs.uniform(0.5, 2, 16).astype(F)]
    exp_avgs = [rs.normal(0, 0.05, s).astype(F) for _, s, _ in NET]
    exp_avg_sqs = [(rs.normal(0, 0.05, s) ** 2).astype(F) for _, s, _ in NET]
    return params, running, exp_avgs, exp_avg_sqs


def synth_grads(seed: int, step: int, spec: dict):
    """Gradients of one step as the scaled backward leaves them (divide by inv_scale); None where the step drops them."""
    rs = np.random.RandomState(1000 * seed + step)
    inv = spec.get("inv_scale", 1.0)
    grads = []
    for i, (_, s, _) in enumerate(NET):
        g = (rs.normal(0, 1e-4 if i == SMALL_GRAD else 2.0, s) / inv).astype(F)
        grads.append(None if i in spec.get("drop", ()) else g)
    if "poison" in spec:
        grads[spec["poison"]].flat[7] = np.inf
    return grads


def adam_step(params, grads, exp_avgs, exp_avg_sqs, steps, groups, hyper, inv_scale=1.0, max_norm=10.0):
    """One step.  grads[i] None: no gradient (parameter and state untouched).  Returns updated copies
    (params, exp_avgs, exp_avg_sqs, steps, grad_norm, skipped)."""
    g = [None if x is None else F(inv_scale) * x.astype(F) for x in grads]                         # scaler.unscale_
    present = [x for x in g if x is not None]
    finite = all(np.isfinite(x).all() for x in present)
    total = F(math.sqrt(sum(float((x.astype(np.float64) ** 2).sum()) for x in present)))       # clip_grad_norm_
    coef = F(1.0)
    if max_norm and max_norm > 0:
        coef = min(F(max_norm) / (total + F(1e-6)), F(1.0))
    p_out, m_out, v_out, s_out = [x.copy() for x in params], [x.copy() for x in exp_avgs], [x.copy() for x in exp_avg_sqs], list(steps)
    if not finite:                                                                               # GradScaler.step skips
        return p_out, m_out, v_out, s_out, float(total), True
    for i, (p, gi, m, v, grp) in enumerate(zip(params, g, exp_avgs, exp_avg_sqs, groups)):
        if gi is None:
            continue
        h = hyper[grp]
        lr, (b1, b2), eps, wd = h["lr"], h["betas"], h["eps"], h["weight_decay"]
        d = gi * coef
        step = float(F(steps[i]) + F(1))
        if wd != 0:
            if h["decoupled_weight_decay"]:
                p = p * F(1 - lr * wd)
            else:
                d = d + F(wd) * p
        w1 = F(1 - b1)
        m = m + w1 * (d - m) if w1 < 0.5 else d - (d - m) * (F(1) - w1)                          # torch's lerp
        v = v * F(b2) + F(1 - b2) * (d * d)
        step_size = F(-(lr / (1 - b1 ** step)))
        bc2_sqrt = F(math.sqrt(1 - b2 ** step))
        den = np.sqrt(v) / bc2_sqrt + F(eps)
        p_out[i], m_out[i], v_out[i], s_out[i] = (p + step_size * (m / den)).astype(F), m.astype(F), v.astype(F), step
    return p_out, m_out, v_out, s_out, float(total), False


def ema_update(emas, values, updates, decay=0.9999, tau=2000.0):
    """ModelEMA.update after `updates` earlier updates: e = d * e + (1 - d) * value, d = decay * (1 - exp(-(updates + 1) / tau))."""
    dec = F(decay * (1 - math.exp(-(updates + 1) / tau)))
    return [(dec * e + (F(1) - dec) * x).astype(F) for e, x in zip(emas, values)]


def run_case(ci: int):
    """The whole case on the oracle: returns dict(params, exp_avgs, exp_avg_sqs, steps, emas (parameters then running mean /
    var), norms, skipped) after its last step."""
    case = CASES[ci]
    params, running, m0, v0 = synth_net(50 + ci)
    n = len(NET)
    if "start_step" in case:
        m, v, steps = m0, v0, [float(case["start_step"])] * n
    else:
        m, v, steps = [np.zeros_like(x) for x in params], [np.zeros_like(x) for x in params], [0.0] * n
    emas = [x.copy() for x in params] + [x.copy() for x in running]
    norms, skipped = [], []
    for k, spec in enumerate(case["steps"]):
        grads = synth_grads(50 + ci, k, spec)
        params, m, v, steps, gn, sk = adam_step(params, grads, m, v, steps, group_of(), hyper(case), spec.get("inv_scale", 1.0), spec["max_norm"])
        emas = ema_update(emas, params + running, EMA_UPDATES0 + k)
        norms.append(gn)
        skipped.append(sk)
    return dict(params=params, exp_avgs=m, exp_avg_sqs=v, steps=steps, emas=emas, norms=norms, skipped=skipped)


def make_net(params, running):
    """The torch module of NET holding `params` and the BN running statistics (CPU, float32)."""
    import torch
    from torch import nn

    class Net(nn.Module):
        def __init__(self):
            super().__init__()
            self.conv = nn.Conv2d(8, 16, 3, bias=False)
            self.bn = nn.BatchNorm2d(16)
            self.fc = nn.Conv2d(16, 32, 1)
            self.lin = nn.Linear(170, 100)

    net = Net()
    sd = {name: torch.from_numpy(p.copy()) for (name, _, _), p in zip(NET, params)}
    sd["bn.running_mean"], sd["bn.running_var"] = torch.from_numpy(running[0].copy()), torch.from_numpy(running[1].copy())
    sd["bn.num_batches_tracked"] = torch.tensor(0)
    net.load_state_dict(sd)
    assert [n for n, _ in net.named_parameters()] == [n for n, _, _ in NET]
    return net


FIXTURE_STRIDE = 5  # tests/golden/adam.npz keeps every 5th element of each result (flattened) to stay small
