"""CPU: yolov5s-ghost (reference models/hub/yolov5s-ghost.yaml) without a GPU -- the built-in name against the reference YAML's
digest; the full model's parameter count, state_dict keys, Detect strides and anchors against the reference's model; the module
signatures; the reference-pickled checkpoint through compat.install(); the oracle (oracle/ghost_ref.py) against the reference's
stored forward and training gradients; the refusals of grouped convolutions the kernels do not build (raised before anything is
launched, by the planner and by the training forward); and the depthwise entry points' argument checks."""
import hashlib
import json
import os
from copy import deepcopy

import numpy as np
import pytest
import torch
from torch import nn

from oracle import ghost_ref, loss_ref
from yolov5_b200 import _lib
from yolov5_b200.cfg import HYP_SCRATCH_LOW, model_cfg, model_names
from yolov5_b200.models import common as mc

G = os.path.join(os.path.dirname(__file__), "golden")
NAME = "yolov5s-ghost"


def _fixture():
    return np.load(os.path.join(G, "ghost_golden.npz"))


def test_builtin_name_matches_reference_yaml():
    cfg = model_cfg(NAME)
    assert hashlib.sha256(json.dumps(cfg, sort_keys=True).encode()).hexdigest() == str(_fixture()["digest"])
    assert model_cfg(f"{NAME}.yaml") == cfg == model_cfg(f"models/hub/{NAME}.yaml")
    assert NAME not in model_names()


def test_parameters_keys_strides_anchors_match_reference():
    from yolov5_b200.models.yolo import DetectionModel

    f = _fixture()
    m = DetectionModel(NAME)
    assert sum(p.numel() for p in m.parameters()) == int(f["n_params"]) == 3897605
    assert list(m.state_dict().keys()) == json.loads(str(f["keys"]))
    det = m.model[-1]
    assert det.stride.tolist() == f["stride"].tolist() == [8.0, 16.0, 32.0]  # the GhostConv(c, 3, 2) layers downsample
    assert torch.equal(det.anchors, torch.from_numpy(f["anchors"]))
    small = DetectionModel(json.loads(str(f["small_cfg"])))
    assert list(small.state_dict().keys()) == json.loads(str(f["small_keys"]))
    dws = [c for c in m.modules() if isinstance(c, nn.Conv2d) and c.groups > 1]
    assert len(dws) == 30 and all(c.kernel_size == (5, 5) and c.groups == c.in_channels == c.out_channels for c in dws)
    assert sorted({c.in_channels for c in dws}) == [8, 16, 32, 64, 128, 256]


def test_module_signatures_match_reference():
    g = mc.GhostConv(16, 32, 3, 2)
    assert not isinstance(g, mc.Conv)
    assert g.cv1.conv.stride == (2, 2) and g.cv1.conv.out_channels == 16 and g.cv2.conv.groups == 16 and g.cv2.conv.kernel_size == (5, 5)
    assert isinstance(mc.GhostConv(16, 32, act=False).cv2.act, nn.Identity)
    b = mc.GhostBottleneck(32, 32)
    assert isinstance(b.conv[1], nn.Identity) and isinstance(b.shortcut, nn.Identity)
    assert isinstance(b.conv[2].cv1.act, nn.Identity) and isinstance(b.conv[0].cv2.act, nn.SiLU)
    assert [k for k in b.state_dict() if k.endswith("conv.weight")] == ["conv.0.cv1.conv.weight", "conv.0.cv2.conv.weight",
                                                                          "conv.2.cv1.conv.weight", "conv.2.cv2.conv.weight"]
    s2 = mc.GhostBottleneck(32, 64, 3, 2)  # built for its keys (the reference's DWConv / Conv), refused by the engine
    assert {k.rsplit(".", 1)[0] for k in s2.state_dict()} >= {"conv.1.conv", "shortcut.0.conv", "shortcut.1.conv"}
    c3 = mc.C3Ghost(64, 64, 2, False)
    assert isinstance(c3, mc.C3) and len(c3.m) == 2 and all(isinstance(x, mc.GhostBottleneck) for x in c3.m)


def test_smart_optimizer_decays_depthwise_weights():
    from yolov5_b200.models.yolo import DetectionModel
    from yolov5_b200.utils.torch_utils import smart_optimizer

    m = DetectionModel(json.loads(str(_fixture()["small_cfg"])))
    opt = smart_optimizer(m, "SGD", lr=0.01, momentum=0.937, decay=5e-4)
    decayed = {id(p) for g in opt.param_groups if g["weight_decay"] > 0 for p in g["params"]}
    dw = [c.weight for c in m.modules() if isinstance(c, nn.Conv2d) and c.groups > 1]
    assert dw and all(id(w) in decayed for w in dw)


def test_reference_checkpoint_loads_through_compat():
    from yolov5_b200 import compat

    assert compat.install()
    ck = torch.load(os.path.join(G, "ref_ghost_tiny.pt"), map_location="cpu", weights_only=False)
    m = ck["model"]
    assert type(m).__module__ == "yolov5_b200.models.yolo"
    assert list(m.state_dict().keys()) == json.loads(str(_fixture()["small_keys"]))
    for i, name in ((1, "GhostConv"), (2, "C3Ghost")):
        assert type(m.model[i]).__name__ == name and type(m.model[i]).__module__ == "yolov5_b200.models.common"
    assert type(m.model[2].m[0]) is mc.GhostBottleneck


def _small_sd(dtype=torch.float64):
    ck = torch.load(os.path.join(G, "ref_ghost_tiny.pt"), map_location="cpu", weights_only=False)
    return {k: v.to(dtype) if v.is_floating_point() else v for k, v in ck["model"].state_dict().items()}


def test_oracle_matches_reference_forward():
    f = _fixture()
    cfg = json.loads(str(f["small_cfg"]))
    x = torch.from_numpy(np.random.RandomState(int(f["x_seed"])).uniform(0, 1, tuple(f["x_shape"])).astype(np.float32))
    z, raws = ghost_ref.forward(cfg, _small_sd(), x.double())
    # the fixture's forward ran on the fp32 model the checkpoint was saved from; the checkpoint holds it in fp16
    assert np.abs(z.numpy() - f["z"]).max() <= 1e-2 * np.abs(f["z"]).max()
    assert len(raws) == 3 and all(r.shape == f[f"raw{i}"].shape for i, r in enumerate(raws))


def test_oracle_matches_reference_training_gradients():
    """The oracle's batch-statistics forward, loss_ref's ComputeLoss and float64 autograd against the reference's fp32 step."""
    f = _fixture()
    cfg = json.loads(str(f["small_cfg"]))
    shape, (s_img, s_tgt) = tuple(f["train_shape"]), f["train_seeds"].tolist()
    img = torch.from_numpy(np.random.RandomState(s_img).randint(0, 256, shape).astype(np.uint8)).double() / 255
    sd = _small_sd()
    for k, v in sd.items():
        if v.is_floating_point() and not k.endswith(("running_mean", "running_var", "anchors")):
            v.requires_grad_(True)
    p = ghost_ref.forward(cfg, sd, img, training=True, bn_batch_stats=True)
    loss, items = loss_ref.compute_loss(p, loss_ref.synth_targets(shape[0], seed=s_tgt, nc=3), sd["model.24.anchors"], HYP_SCRATCH_LOW)
    loss.sum().backward()
    assert np.allclose(np.asarray(items, dtype=np.float64), f["items"], rtol=1e-4, atol=1e-6)
    num = den = 0.0
    for k in (k for k in f.files if k.startswith("grad:")):
        g = torch.from_numpy(f[k].astype(np.float64))
        num += float((sd[k[5:]].grad - g).norm()) ** 2
        den += float(g.norm()) ** 2
    assert (num / den) ** 0.5 <= 2e-3  # the fixture stores fp16-rounded gradients


def _small():
    from yolov5_b200.models.yolo import DetectionModel

    return DetectionModel(json.loads(str(_fixture()["small_cfg"])))


def _refused(model, match):
    """both the inference planner and the training forward refuse `model` before anything runs (CPU tensors: any launch would fail
    with another error)"""
    from yolov5_b200.engine import Program
    from yolov5_b200.train_ops import forward_train

    with pytest.raises(NotImplementedError, match=match):
        Program(model.half(), 1, 64, 64, torch.float16, "cpu")
    with pytest.raises(NotImplementedError, match=match):
        forward_train(model.half(), torch.zeros(1, 3, 64, 64, dtype=torch.uint8))


@pytest.mark.parametrize("k,s,d,groups", [(3, 1, 1, "c"), (5, 2, 1, "c"), (5, 1, 2, "c"), (5, 1, 1, "c/2"), (5, 1, 1, "1")],
                         ids=["k3", "s2", "dilation2", "groups_c/2", "groups_1"])
def test_refuses_other_ghost_cheap_convs(built_lib, k, s, d, groups):
    m = _small()
    g = m.model[1]  # GhostConv(64, 64, 3, 2): cv2 is Conv(32, 32, 5, 1, None, 32)
    c = g.cv2.conv.in_channels
    g.cv2 = mc.Conv(c, c, k, s, None, {"c": c, "c/2": c // 2, "1": 1}[groups], d)
    _refused(m, "GhostConv.cv2")


def test_refuses_stride2_ghost_bottleneck(built_lib):
    m = _small()
    c = m.model[2].m[0].conv[0].cv1.conv.in_channels
    m.model[2].m[0] = mc.GhostBottleneck(c, c, 3, 2)
    _refused(m, r"GhostBottleneck\(s=2\)")


def test_refuses_other_grouped_convs(built_lib):
    m = _small()
    old = m.model[9].cv1  # SPPF.cv1 as a grouped 1x1 conv
    m.model[9].cv1 = mc.Conv(old.conv.in_channels, old.conv.out_channels, 1, 1, g=2)
    _refused(m, "grouped convolution 'model.9.cv1.conv'")
    single = deepcopy(m.model[9]).half()
    from yolov5_b200.engine import Program

    with pytest.raises(NotImplementedError, match="grouped convolution"):
        Program(single, 1, 8, 8, torch.float16, "cpu", in_channels=old.conv.in_channels)


def test_dwconv_entry_points_check_arguments(built_lib):
    lib = built_lib
    buf, w = 4096, 8192  # never dereferenced: every call below fails its argument checks first
    F16 = _lib.Y5_F16

    def fwd(x=buf, xp=8, wt=w, y=buf + 1024, yp=8, res=None, rp=0, xr=None, xrp=0, xo=None, xop=0, c=8, k=5, s=1, act=0, slope=0.0, dt=F16):
        return lib.y5_dwconv_fwd(x, xp, wt, None, y, yp, res, rp, xr, xrp, xo, xop, 1, 4, 4, c, k, s, act, slope, 0, dt, None)

    assert fwd(c=12) == -1 and b"multiple of 8" in lib.y5_last_error()
    assert fwd(xp=4) == -1 and b"pitch" in lib.y5_last_error()
    assert fwd(yp=12) == -1
    assert fwd(x=buf + 2) == -1 and b"aligned" in lib.y5_last_error()
    assert fwd(res=buf + 8, rp=8) == -1
    assert fwd(wt=w + 1) == -1
    assert fwd(k=3) == -1 and b"kernel size 3" in lib.y5_last_error()
    assert fwd(s=2) == -1 and b"stride 2" in lib.y5_last_error()
    assert fwd(xr=buf + 2048, xrp=8) == -1  # x_res without x_out
    assert fwd(y=buf) == -1  # in place over x
    assert fwd(act=7) == -1
    assert fwd(act=_lib.ACT_LEAKY, slope=float("nan")) == -1
    assert fwd(dt=_lib.Y5_F32) == -2
    assert lib.y5_dwconv_wgrad(buf, 8, buf, 8, w, 1, 4, 4, 12, 5, 1, F16, None) == -1
    assert lib.y5_dwconv_wgrad(buf, 4, buf, 8, w, 1, 4, 4, 8, 5, 1, F16, None) == -1
    assert lib.y5_dwconv_wgrad(buf + 4, 8, buf, 8, w, 1, 4, 4, 8, 5, 1, F16, None) == -1
    assert lib.y5_dwconv_wgrad(buf, 8, buf, 8, w + 2, 1, 4, 4, 8, 5, 1, F16, None) == -1
    assert lib.y5_dwconv_wgrad(buf, 8, buf, 8, w, 1, 4, 4, 8, 3, 1, F16, None) == -1
    assert lib.y5_dwconv_wgrad(buf, 8, buf, 8, w, 1, 4, 4, 8, 5, 2, F16, None) == -1
