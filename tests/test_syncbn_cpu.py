"""CPU: the device-free parts of SyncBatchNorm on the training path -- when a layer syncs (torch.nn.SyncBatchNorm's rule),
smart_optimizer's parameter groups of a converted model (reference utils/torch_utils.py:263), GraphedTrainStep's refusal,
and the argument checks of the split BN entry points."""
import types

import pytest
from torch import nn

from yolov5_b200 import _lib, train_ops


def _model(sync=False):
    from oracle import model_ref
    from yolov5_b200.cfg import model_cfg
    from yolov5_b200.models.yolo import DetectionModel

    m = DetectionModel("yolov5n")
    m.load_state_dict(model_ref.synth_state_dict(model_cfg("yolov5n"), seed=3))
    return nn.SyncBatchNorm.convert_sync_batchnorm(m) if sync else m


@pytest.fixture
def fake_world(monkeypatch):
    """torch.distributed as an initialised WORLD of `size[0]` ranks, without a process group"""
    import torch.distributed as dist

    size = [2]
    monkeypatch.setattr(dist, "is_available", lambda: True)
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "group", types.SimpleNamespace(WORLD=object()))
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: size[0] if group is not None else -1)
    return size


def test_no_sync_without_torch_distributed():
    import torch.distributed as dist

    assert not dist.is_initialized()
    for bn in (nn.SyncBatchNorm(8), nn.BatchNorm2d(8)):
        assert train_ops.bn_process_group(bn) is None
        assert train_ops.bn_sync_group(bn.train()) is None


def test_sync_rule(fake_world):
    import torch.distributed as dist

    bn = nn.SyncBatchNorm(8).train()
    assert dist.group.WORLD is not None
    assert train_ops.bn_sync_group(bn) is dist.group.WORLD
    assert train_ops.bn_sync_group(bn.eval()) is None  # eval: running statistics, no collective
    assert train_ops.bn_process_group(bn) is dist.group.WORLD
    own = object()
    bn.process_group = own
    assert train_ops.bn_sync_group(bn.train()) is own  # the layer's own group takes precedence over WORLD
    fake_world[0] = 1
    assert train_ops.bn_sync_group(bn) is None  # a group of one rank is plain batch norm
    fake_world[0] = 2
    assert train_ops.bn_sync_group(nn.BatchNorm2d(8).train()) is None  # only SyncBatchNorm syncs


def test_smart_optimizer_groups_follow_the_reference_rule():
    from yolov5_b200.utils.torch_utils import smart_optimizer

    norm = tuple(v for k, v in nn.__dict__.items() if "Norm" in k)  # reference utils/torch_utils.py:263

    def reference_groups(m):
        g = [], [], []
        for v in m.modules():
            for p_name, p in v.named_parameters(recurse=False):
                if p_name == "bias":
                    g[2].append(p)
                elif p_name == "weight" and isinstance(v, norm):
                    g[1].append(p)
                else:
                    g[0].append(p)
        return g

    plain, conv = _model(), _model(sync=True)
    assert sum(isinstance(v, nn.SyncBatchNorm) for v in conv.modules()) > 50
    names = {}
    for m in (plain, conv):
        ids = {id(p): k for k, p in m.named_parameters()}
        opt = smart_optimizer(m, "SGD", lr=0.01, momentum=0.9, decay=5e-4)
        got = [[ids[id(p)] for p in g["params"]] for g in opt.param_groups]  # biases, decayed weights, norm weights
        ref = reference_groups(m)
        assert got == [[ids[id(p)] for p in ref[i]] for i in (2, 0, 1)]
        assert [g["weight_decay"] for g in opt.param_groups] == [0.0, 5e-4, 0.0]
        names[m is conv] = got
    assert names[True] == names[False]  # the converted model gets the unconverted model's three groups
    assert all(".bn.weight" in k for k in names[True][2]) and not any(".bn." in k for k in names[True][1])


def test_graphed_train_step_refuses_a_syncing_model(fake_world):
    from yolov5_b200.utils.torch_utils import FusedSGD, GraphedTrainStep

    m = _model(sync=True).train()
    opt = FusedSGD(m.parameters(), lr=0.01, momentum=0.9)
    with pytest.raises(NotImplementedError, match="SyncBatchNorm"):
        GraphedTrainStep(m, None, opt, batch=2, size=64)


def test_sync_passes_check_arguments_without_gpu(built_lib):
    lib = built_lib
    f16 = _lib.Y5_F16
    n = 4096  # a non-NULL row count: SyncBatchNorm's forms of the passes
    assert lib.y5_bn_stats(None, 64, 10, 64, f16, None, n, None) == -1 and b"bn_stats" in lib.y5_last_error()
    assert lib.y5_bn_act_fwd(None, 64, None, 64, 10, 64, f16, None, None, None, None, 1, 0.0, None, n, 1e-3, 0.03, None, None, None, 0, None) == -1
    assert b"bn_act_fwd y" in lib.y5_last_error()
    assert lib.y5_bn_act_bwd_reduce(None, 64, None, 64, None, 64, 10, 64, f16, None, None, None, None, 1, 0.0, None, None, None, None) == -1
    assert b"bn_act_bwd_reduce y" in lib.y5_last_error()
    assert lib.y5_bn_act_bwd_apply(None, 64, None, 64, None, 64, 10, 64, f16, None, None, None, 1, None, None, None) == -1
    assert b"bn_act_bwd_apply y" in lib.y5_last_error()
    # the plain forms
    assert lib.y5_bn_act_fwd(None, 64, None, 64, 10, 64, f16, None, None, None, None, 1, 0.0, None, None, 1e-3, 0.03, None, None, None, 0, None) == -1
    assert b"bn_act_fwd y" in lib.y5_last_error()
    assert lib.y5_bn_act_bwd(None, 64, None, 64, None, 64, 10, 64, f16, None, None, None, None, 1, 0.0, None, None, None, None) == -1
    assert b"bn_act_bwd y" in lib.y5_last_error()
    # a row count needs the column sums it divides: refused before anything is launched (the pointers are never read)
    p = 4096
    assert lib.y5_bn_act_fwd(p, 64, p, 64, 10, 64, f16, p, p, p, p, 1, 0.0, None, n, 1e-3, 0.03, None, None, None, 0, None) == -1
    assert b"bn_act_fwd: count needs the column sums" in lib.y5_last_error()
