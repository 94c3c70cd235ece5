"""CPU: the YOLOv3 models (reference models/hub/yolov3.yaml, yolov3-spp.yaml, yolov3-tiny.yaml) without a GPU -- the built-in
names against the reference YAMLs' digests, parameter counts, state_dict keys, Detect strides and anchors against the reference's
models, the SPP = chained SPPF identity, the pooling oracle's tie rule against torch CPU autograd, the reference-pickled
checkpoints, the refusals (raised before anything is launched) and the pool entry points' argument checks."""
import hashlib
import json
import os
from copy import deepcopy

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch import nn

from oracle import pool_ref
from yolov5_b200 import _lib
from yolov5_b200.cfg import model_cfg, model_names
from yolov5_b200.models import common as mc

G = os.path.join(os.path.dirname(__file__), "golden")
NAMES = ("yolov3", "yolov3-spp", "yolov3-tiny")


def _fixture(name):
    return np.load(os.path.join(G, f"{name.replace('-', '_')}_golden.npz"))


@pytest.mark.parametrize("name", NAMES)
def test_builtin_names_match_reference_yaml(name):
    cfg = model_cfg(name)
    assert hashlib.sha256(json.dumps(cfg, sort_keys=True).encode()).hexdigest() == str(_fixture(name)["digest"])
    assert model_cfg(f"{name}.yaml") == cfg == model_cfg(f"models/hub/{name}.yaml")
    assert name not in model_names()


@pytest.mark.parametrize("name", NAMES)
def test_parameters_keys_strides_anchors_match_reference(name):
    from yolov5_b200.models.yolo import DetectionModel

    f = _fixture(name)
    m = DetectionModel(name)
    assert sum(p.numel() for p in m.parameters()) == int(f["n_params"])
    assert list(m.state_dict().keys()) == json.loads(str(f["keys"]))
    det = m.model[-1]
    assert det.stride.tolist() == f["stride"].tolist()
    assert torch.equal(det.anchors, torch.from_numpy(f["anchors"]))
    small = DetectionModel(json.loads(str(f["small_cfg"])))
    assert list(small.state_dict().keys()) == json.loads(str(f["small_keys"]))


def test_spp_module_matches_reference_signature():
    m = mc.SPP(64, 32)
    assert [type(p) for p in m.m] == [nn.MaxPool2d] * 3 and [p.kernel_size for p in m.m] == [5, 9, 13]
    assert m.cv1.conv.out_channels == 32 and m.cv2.conv.in_channels == 128
    assert set(m.state_dict()) == {f"cv{i}.{k}" for i in (1, 2) for k in ("conv.weight", "bn.weight", "bn.bias", "bn.running_mean",
                                                                             "bn.running_var", "bn.num_batches_tracked")}
    assert mc.spp_kernel(m) == 5 and mc.spp_kernel(mc.SPP(64, 32, (3, 5, 7))) == 3


def _tied(shape, seed, lo=-4, hi=5):
    """integer values in a narrow range: many ties in every window"""
    return torch.from_numpy(np.random.RandomState(seed).randint(lo, hi, shape)).float()


def test_spp_pools_are_chained_sppf_pools():
    """mp_{2k-1} = mp_k . mp_k and mp_{3k-2} = mp_k . mp_k . mp_k exactly (values), with -inf padding at the edges; NaN and -inf
    inputs included."""
    for k, shape, seed in ((5, (2, 3, 13, 11), 0), (3, (1, 4, 7, 9), 1), (5, (1, 2, 20, 20), 2)):
        x = _tied(shape, seed)
        x[0, 0, 0, 0] = float("-inf")
        x[0, 1, shape[2] // 2, 3] = float("nan")
        m = lambda t, kk: F.max_pool2d(t, kk, 1, kk // 2)  # noqa: E731
        a1 = m(x, k)
        assert torch.allclose(m(x, 2 * k - 1), m(a1, k), equal_nan=True, rtol=0, atol=0)
        assert torch.allclose(m(x, 3 * k - 2), m(m(a1, k), k), equal_nan=True, rtol=0, atol=0)
        assert torch.allclose(pool_ref.spp(x, (k, 2 * k - 1, 3 * k - 2)), torch.cat([x, a1, m(a1, k), m(m(a1, k), k)], 1).double(),
                              equal_nan=True, rtol=0, atol=0)


def _torch_grad(fn, x, dy):
    x = x.double().clone().requires_grad_(True)
    y = fn(x)
    y.backward(dy.double())
    return y.detach(), x.grad


@pytest.mark.parametrize("case", ["k2s2", "zpad", "k2s2_odd"])
def test_pool_oracle_tie_rule_matches_torch_autograd(case):
    shape = {"k2s2": (2, 3, 8, 10), "zpad": (2, 3, 7, 6), "k2s2_odd": (1, 2, 9, 7)}[case]
    x = _tied(shape, 3, lo=-3, hi=2)  # negative values reach the zero-pad border
    if case == "zpad":
        fn, ref = (lambda t: F.max_pool2d(F.pad(t, (0, 1, 0, 1)), 2, 1)), (lambda t: pool_ref.maxpool(t, 2, 1, 0, 1))
    else:
        fn, ref = (lambda t: F.max_pool2d(t, 2, 2)), (lambda t: pool_ref.maxpool(t, 2, 2))
    y, idx = ref(x)
    dy = _tied(tuple(y.shape), 4, lo=-8, hi=9)
    yt, gt = _torch_grad(fn, x, dy)
    assert torch.equal(y, yt) and torch.equal(pool_ref.maxpool_backward(idx, dy, x.shape), gt)
    if case == "zpad":
        assert (idx < 0).any()  # some border windows chose a pad cell


def test_spp_oracle_backward_matches_torch_autograd():
    x = _tied((2, 4, 9, 11), 5, lo=-2, hi=3)
    ks = (5, 9, 13)
    dcat = _tied((2, 16, 9, 11), 6, lo=-8, hi=9)

    def fn(t):
        return torch.cat([t] + [F.max_pool2d(t, k, 1, k // 2) for k in ks], 1)

    yt, gt = _torch_grad(fn, x, dcat)
    assert torch.equal(pool_ref.spp(x, ks), yt)
    assert torch.equal(pool_ref.spp_backward(x, dcat, ks), gt)
    # SPPF's chain routes mp9's and mp13's gradients through intermediate arg-maxes: a different element on ties

    def chained(t):
        p1 = F.max_pool2d(t, 5, 1, 2)
        p2 = F.max_pool2d(p1, 5, 1, 2)
        return torch.cat([t, p1, p2, F.max_pool2d(p2, 5, 1, 2)], 1)

    assert not torch.equal(gt, _torch_grad(chained, x, dcat)[1])


@pytest.mark.parametrize("name", NAMES)
def test_reference_checkpoint_loads_through_compat(name):
    from yolov5_b200 import compat

    assert compat.install()
    ck = torch.load(os.path.join(G, f"ref_{name}_tiny.pt"), map_location="cpu", weights_only=False)
    m = ck["model"]
    assert type(m).__module__ == "yolov5_b200.models.yolo"
    assert list(m.state_dict().keys()) == json.loads(str(_fixture(name)["small_keys"]))
    if name == "yolov3-spp":
        assert type(m.model[12]).__name__ == "SPP" and type(m.model[12]).__module__ == "yolov5_b200.models.common"


def _small(name):
    from yolov5_b200.models.yolo import DetectionModel

    return DetectionModel(json.loads(str(_fixture(name)["small_cfg"])))


def _refused(model, match):
    """both the inference planner and the training forward refuse `model` before anything runs (CPU tensors: any launch would fail
    with another error)"""
    from yolov5_b200.engine import Program
    from yolov5_b200.train_ops import forward_train

    with pytest.raises(NotImplementedError, match=match):
        Program(model.half(), 1, 64, 64, torch.float16, "cpu")
    with pytest.raises(NotImplementedError, match=match):
        forward_train(model.half(), torch.zeros(1, 3, 64, 64, dtype=torch.uint8))


@pytest.mark.parametrize("pool", [nn.MaxPool2d(2, 2, 0, ceil_mode=True), nn.MaxPool2d(2, 2, 0, dilation=2), nn.MaxPool2d(2, 2, 0, return_indices=True),
                                  nn.MaxPool2d(3, 2, 1), nn.MaxPool2d(2, 1, 0), nn.MaxPool2d((2, 3), 2)], ids=str)
def test_refuses_other_pools(built_lib, pool):
    m = _small("yolov3-tiny")
    pool.i, pool.f = 1, -1
    m.model[1] = pool
    _refused(m, "MaxPool2d")


@pytest.mark.parametrize("pad", [(0, 1, 1, 0), (1, 1, 1, 1), (0, 2, 0, 2)])
def test_refuses_other_zero_pads(built_lib, pad):
    m = _small("yolov3-tiny")
    p = nn.ZeroPad2d(pad)
    p.i, p.f = 11, -1
    m.model[11] = p
    _refused(m, "ZeroPad2d")


def test_refuses_zero_pad_without_its_pool(built_lib):
    m = _small("yolov3-tiny")
    conv = m.model[13]
    m.model[12] = deepcopy(m.model[10])  # a Conv after the pad instead of MaxPool2d(2, 1, 0)
    m.model[12].i, m.model[12].f = 12, -1
    m.model[12].conv = nn.Conv2d(conv.conv.in_channels, conv.conv.in_channels, 3, 1, 1, bias=False)
    _refused(m, "ZeroPad2d")


@pytest.mark.parametrize("ks", [(5, 9, 12), (5, 7, 9), (4, 7, 10), (5, 9)])
def test_refuses_other_spp_kernels(built_lib, ks):
    m = _small("yolov3-spp")
    old = m.model[12]
    spp = mc.SPP(old.cv1.conv.in_channels, old.cv2.conv.out_channels, ks)
    spp.i, spp.f = 12, -1
    m.model[12] = spp
    _refused(m, "SPP")


def test_pool_entry_points_check_arguments(built_lib):
    lib = built_lib
    buf = 4096  # never dereferenced: every call below fails its argument checks first
    assert lib.y5_maxpool2d(buf, 8, buf, 8, 1, 4, 4, 8, 7, _lib.Y5_F16, None) == -2 and b"mode" in lib.y5_last_error()
    assert lib.y5_maxpool2d(buf, 8, buf, 8, 1, 4, 4, 12, _lib.POOL_K2S2, _lib.Y5_F16, None) == -2
    assert lib.y5_maxpool2d(buf + 2, 8, buf, 8, 1, 4, 4, 8, _lib.POOL_K2S2, _lib.Y5_F16, None) == -1
    assert lib.y5_maxpool2d(buf, 8, buf, 8, 1, 1, 1, 8, _lib.POOL_K2S2, _lib.Y5_F16, None) == -1  # empty output
    assert lib.y5_maxpool2d(buf, 8, buf, 8, 1, 4, 4, 8, _lib.POOL_K2S2, _lib.Y5_U8, None) == -2
    assert lib.y5_maxpool2d_bwd(buf, 8, None, 8, buf, 8, 1, 4, 4, 8, _lib.POOL_K2S1_ZPAD, _lib.Y5_F32, None) == -1
    assert lib.y5_spp_bwd_workspace_bytes(2, 20, 20, 128) == 3 * 2 * 20 * 20 * 128 * 2
    assert lib.y5_spp_pool_bwd(buf, 8, buf, 32, buf, 8, 1, 4, 4, 8, 4, _lib.Y5_F16, buf, None) == -2  # even k
    assert lib.y5_spp_pool_bwd(buf, 8, buf, 16, buf, 8, 1, 4, 4, 8, 5, _lib.Y5_F16, buf, None) == -1  # dcat pitch < 4c
    assert lib.y5_spp_pool_bwd(buf, 8, buf, 32, buf, 8, 1, 4, 4, 8, 5, _lib.Y5_F16, None, None) == -1
    assert lib.y5_image_nhwc(buf, _lib.Y5_U8, buf, _lib.Y5_F16, 1, 4, 4, 12, None) == -1
    assert lib.y5_image_nhwc(buf, _lib.Y5_U8, buf, _lib.Y5_F32, 1, 4, 4, 16, None) == -2
    assert lib.y5_image_nhwc(buf, 9, buf, _lib.Y5_F16, 1, 4, 4, 16, None) == -2
