"""Generate tests/golden/adam.npz by running the UNMODIFIED reference (/root/reference) with `--optimizer Adam | AdamW`.

Runs only in the build container (the GPU box has no /root/reference):
    python tests/golden/make_adam_golden.py
The reference is imported through tests/golden/refshim.py.  Every case of oracle/adam_ref.py runs through the reference's own
smart_optimizer (torch.optim.Adam / AdamW in its three groups), the train.py:413-421 sequence -- `p.grad.mul_(inv_scale)` for
scaler.unscale_, clip_grad_norm_, the step unless a gradient is non-finite, zero_grad, the reference's ModelEMA.update -- and
the oracle is asserted equal to it.  The fixture keeps the reference's outputs (strided) and its parameter-group layout on
yolov5n.
"""
from __future__ import annotations

import json
import os
import sys
from copy import deepcopy

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import refshim  # noqa: E402

refshim.install()

import torch  # noqa: E402

from oracle import adam_ref  # noqa: E402

RTOL, ATOL = 2e-6, 1e-7


def run_reference(ci):
    from utils.torch_utils import ModelEMA, smart_optimizer

    case = adam_ref.CASES[ci]
    params, running, m0, v0 = adam_ref.synth_net(50 + ci)
    net = adam_ref.make_net(params, running)
    ps = list(net.parameters())

    def build():
        return smart_optimizer(net, case["opt"], case["lr"], case["momentum"], case["decay"])

    opt = build()
    if "start_step" in case:
        for i, p in enumerate(ps):
            opt.state[p] = dict(step=torch.tensor(float(case["start_step"])), exp_avg=torch.from_numpy(m0[i].copy()),
                                exp_avg_sq=torch.from_numpy(v0[i].copy()))
    ema = ModelEMA(net, decay=0.9999, tau=2000, updates=adam_ref.EMA_UPDATES0)
    norms, skipped = [], []
    for k, spec in enumerate(case["steps"]):
        if case.get("resume_after") == k:  # smart_resume: a fresh optimizer loads the saved state_dict
            sd = deepcopy(opt.state_dict())
            opt = build()
            opt.load_state_dict(sd)
        for p, g in zip(ps, adam_ref.synth_grads(50 + ci, k, spec)):
            p.grad = None if g is None else torch.from_numpy(g.copy())
        # train.py:413-421
        for p in ps:
            if p.grad is not None:
                p.grad.mul_(spec.get("inv_scale", 1.0))                 # scaler.unscale_
        found_inf = not all(bool(torch.isfinite(p.grad).all()) for p in ps if p.grad is not None)
        norm = torch.nn.utils.clip_grad_norm_(ps, max_norm=spec["max_norm"])
        if not found_inf:                                               # scaler.step skips on overflow
            opt.step()
        opt.zero_grad()
        ema.update(net)
        norms.append(float(norm))
        skipped.append(found_inf)
    return net, opt, ema, norms, skipped


def state_of(opt, p):
    st = opt.state.get(p, {})
    if not st:
        return np.zeros(p.shape, np.float32), np.zeros(p.shape, np.float32), 0.0
    return st["exp_avg"].numpy(), st["exp_avg_sq"].numpy(), float(st["step"])


def layout(name):
    """The reference's parameter groups on yolov5n: per group the parameter sizes, the keys, betas and weight decay."""
    from models.yolo import DetectionModel
    from utils.torch_utils import smart_optimizer

    torch.manual_seed(0)
    m = DetectionModel(f"{refshim.REFERENCE_ROOT}/models/yolov5n.yaml")
    opt = smart_optimizer(m, name, 0.01, 0.937, 5e-4)
    return [dict(numel=[p.numel() for p in g["params"]], keys=sorted(k for k in g if k != "params"), betas=list(g["betas"]),
                 weight_decay=g["weight_decay"], decoupled_weight_decay=g["decoupled_weight_decay"]) for g in opt.param_groups]


def main():
    store = {}
    s = adam_ref.FIXTURE_STRIDE
    for ci in range(len(adam_ref.CASES)):
        net, opt, ema, norms, skipped = run_reference(ci)
        want = adam_ref.run_case(ci)
        assert skipped == want["skipped"], (ci, skipped, want["skipped"])
        for gn, ref in zip(want["norms"], norms):
            assert np.isinf(ref) or abs(gn - ref) <= 1e-5 * ref, (ci, gn, ref)
        esd = [v for v in ema.ema.state_dict().values() if v.dtype.is_floating_point]
        ema_ref = [esd[i] for i in (0, 1, 2, 5, 6, 7, 8)] + [esd[3], esd[4]]  # parameters in NET order, then running mean / var
        steps = []
        for i, p in enumerate(net.parameters()):
            m, v, step = state_of(opt, p)
            steps.append(step)
            for tag, got, ref in (("p", p.detach().numpy(), want["params"][i]), ("m", m, want["exp_avgs"][i]), ("v", v, want["exp_avg_sqs"][i]),
                                  ("e", ema_ref[i].numpy(), want["emas"][i])):
                assert np.allclose(got, ref, rtol=RTOL, atol=ATOL), (ci, tag, i, np.abs(got - ref).max())
                store[f"c{ci}.{tag}{i}"] = got.reshape(-1)[::s].copy()
        for j in (0, 1):
            got = ema_ref[len(adam_ref.NET) + j].numpy()
            assert np.allclose(got, want["emas"][len(adam_ref.NET) + j], rtol=RTOL, atol=ATOL), (ci, "ebuf", j)
            store[f"c{ci}.ebuf{j}"] = got.copy()
        assert steps == want["steps"], (ci, steps, want["steps"])
        store[f"c{ci}.steps"] = np.array(steps, np.float32)
        store[f"c{ci}.skipped"] = np.array(skipped)
        store[f"c{ci}.norms"] = np.array(norms)
    store["layout"] = np.array(json.dumps({name: layout(name) for name in ("Adam", "AdamW")}))
    np.savez_compressed(f"{HERE}/adam.npz", **store)
    print(f"Adam / AdamW step: oracle == reference smart_optimizer + clip_grad_norm_ + ModelEMA on {len(adam_ref.CASES)} cases")


if __name__ == "__main__":
    main()
