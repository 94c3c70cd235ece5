"""CPU: the Adam / AdamW step's oracle against the reference-generated fixture, smart_optimizer's parameter groups against the
reference's, and what the fused Adam refuses (bad y5_adam_step arguments, RMSProp, amsgrad, maximize) -- no GPU needed."""
import json
import os

import numpy as np
import pytest

from oracle import adam_ref
from yolov5_b200 import _lib
from yolov5_b200.models.yolo import DetectionModel
from yolov5_b200.utils.torch_utils import FusedAdam, FusedAdamW, smart_optimizer

G = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("ci", range(len(adam_ref.CASES)))
def test_oracle_matches_reference_fixture(ci):
    g = np.load(os.path.join(G, "adam.npz"))
    want = adam_ref.run_case(ci)
    s = adam_ref.FIXTURE_STRIDE
    for i in range(len(adam_ref.NET)):
        for tag, got in (("p", want["params"][i]), ("m", want["exp_avgs"][i]), ("v", want["exp_avg_sqs"][i]), ("e", want["emas"][i])):
            assert np.allclose(got.reshape(-1)[::s], g[f"c{ci}.{tag}{i}"], rtol=2e-6, atol=1e-7), (ci, tag, i)
    for j in (0, 1):
        assert np.allclose(want["emas"][len(adam_ref.NET) + j], g[f"c{ci}.ebuf{j}"], rtol=2e-6, atol=1e-7)
    assert np.array_equal(np.array(want["steps"], np.float32), g[f"c{ci}.steps"])
    assert list(g[f"c{ci}.skipped"]) == want["skipped"]


@pytest.mark.parametrize("name", ["Adam", "AdamW"])
def test_smart_optimizer_groups_match_the_reference(name):
    ref = json.loads(str(np.load(os.path.join(G, "adam.npz"))["layout"]))[name]
    opt = smart_optimizer(DetectionModel("yolov5n"), name, 0.01, 0.937, 5e-4)
    assert type(opt) is (FusedAdam if name == "Adam" else FusedAdamW)
    assert len(opt.param_groups) == len(ref) == 3
    for g, r in zip(opt.param_groups, ref):
        assert [p.numel() for p in g["params"]] == r["numel"]
        assert sorted(k for k in g if k != "params") == r["keys"]
        assert "momentum" not in g  # train.py's warm-up only touches groups that have one
        assert list(g["betas"]) == r["betas"] and g["weight_decay"] == r["weight_decay"]
        assert g["decoupled_weight_decay"] == r["decoupled_weight_decay"]
        assert g["amsgrad"] is False and g["maximize"] is False


def test_adam_defaults_follow_torch():
    import torch

    p = [torch.nn.Parameter(torch.zeros(3))]
    for ours, theirs in ((FusedAdam(p), torch.optim.Adam(p)), (FusedAdamW(p), torch.optim.AdamW(p))):
        a, b = ours.param_groups[0], theirs.param_groups[0]
        assert {k: v for k, v in a.items() if k != "params"} == {k: v for k, v in b.items() if k != "params"}


def test_out_of_scope_options_raise():
    import torch

    m = DetectionModel("yolov5n")
    with pytest.raises(NotImplementedError):
        smart_optimizer(m, "RMSProp", 0.01, 0.937, 5e-4)
    p = [torch.nn.Parameter(torch.zeros(3))]
    with pytest.raises(NotImplementedError):
        FusedAdam(p, amsgrad=True)
    with pytest.raises(NotImplementedError):
        FusedAdamW(p, maximize=True)
    opt = FusedAdam(p)
    with pytest.raises(NotImplementedError):
        opt.add_param_group({"params": [torch.nn.Parameter(torch.zeros(2))], "amsgrad": True})


def test_adam_step_argument_validation_without_gpu(built_lib):
    lib = built_lib
    assert lib.y5_adam_step(None, 4, None, None, 0, None, None, 0, None, None, 1, 0, None) == 0  # nothing to do
    assert lib.y5_adam_step(None, 4, None, None, 4, None, None, 0, None, None, 1, 0, None) == -1
    assert b"null" in lib.y5_last_error()
    # every pointer but one set: still refused before any launch
    args = [4096, 4, 4096, 4096, 4, 4096, 4096, 0, 4096, 4096, 1, 0, None]
    for k in (0, 2, 3, 5, 6, 8, 9):
        bad = list(args)
        bad[k] = None
        assert lib.y5_adam_step(*bad) == -1, k
    bad = list(args)
    bad[7] = -1  # negative exp_avg_sq offset
    assert lib.y5_adam_step(*bad) == -1 and b"sq_offset" in lib.y5_last_error()
    bad = list(args)
    bad[1] = 0
    assert lib.y5_adam_step(*bad) == -1
    assert _lib.ADAM_STRIDE >= _lib.ADAM_DECOUPLED + 1
