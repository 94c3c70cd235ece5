"""CPU: yolov5s-transformer (C3TR, reference models/common.py:115-161, 261-270) without a GPU -- the model dict and built-in name
against the reference YAML's digest, the modules' keys and signatures, the reference-pickled checkpoint, the float64 oracle
against the reference's stored forward, the refusals, and the attention entry points' argument checks."""
import ctypes as C
import hashlib
import inspect
import json
import os

import numpy as np
import pytest
import torch
from torch import nn

from yolov5_b200 import _lib
from yolov5_b200.cfg import model_cfg
from yolov5_b200.models import common as mc

G = os.path.join(os.path.dirname(__file__), "golden")


def _fixture(width):
    return np.load(os.path.join(G, f"transformer_forward_w{int(width * 100)}.npz"))


def test_builtin_name_matches_reference_yaml_digest():
    cfg = model_cfg("yolov5s-transformer")
    for width in (0.5, 0.25):
        assert hashlib.sha256(json.dumps(cfg, sort_keys=True).encode()).hexdigest() == str(_fixture(width)["digest"])
    assert model_cfg("models/hub/yolov5s-transformer.yaml") == cfg


def test_yaml_builds_with_reference_keys_and_signatures():
    from yolov5_b200.models.yolo import DetectionModel

    for w in (0.5, 0.25):
        cfg = model_cfg("yolov5s-transformer")
        cfg["width_multiple"] = w
        m = DetectionModel(cfg)
        assert list(m.state_dict().keys()) == json.loads(str(_fixture(w)["keys"]))
        c3tr = m.model[8]
        assert isinstance(c3tr, mc.C3TR) and isinstance(c3tr.m, mc.TransformerBlock) and len(c3tr.m.tr) == 1
        assert c3tr.m.tr[0].ma.num_heads == 4 and c3tr.m.tr[0].ma.head_dim == int(1024 * w) // 8
    assert list(inspect.signature(mc.C3TR).parameters) == ["c1", "c2", "n", "shortcut", "g", "e"]
    assert list(inspect.signature(mc.TransformerBlock).parameters) == ["c1", "c2", "num_heads", "num_layers"]
    assert list(inspect.signature(mc.TransformerLayer).parameters) == ["c", "num_heads"]


def test_optimizer_groups_follow_reference_rule():
    from yolov5_b200.models.yolo import DetectionModel
    from yolov5_b200.utils.torch_utils import smart_optimizer

    m = DetectionModel("yolov5s-transformer")
    opt = smart_optimizer(m, "SGD", lr=0.01, momentum=0.9, decay=5e-4)
    ids = [{id(p) for p in grp["params"]} for grp in opt.param_groups]  # [bias, decay, no-decay BN weights]
    ma = m.model[8].m.tr[0].ma
    assert id(ma.in_proj_bias) in ids[1] and id(ma.in_proj_weight) in ids[1]
    assert id(ma.out_proj.bias) in ids[0] and id(m.model[8].m.linear.bias) in ids[0]


def test_reference_checkpoint_loads():
    from yolov5_b200 import compat

    compat.install()
    ck = torch.load(os.path.join(G, "ref_transformer_tiny.pt"), map_location="cpu", weights_only=False)
    m = ck["model"]
    f = np.load(os.path.join(G, "ref_transformer_tiny_forward.npz"))
    assert type(m.model[8]) is mc.C3TR and list(m.state_dict().keys()) == json.loads(str(f["keys"]))


@pytest.mark.parametrize("width", [0.5, 0.25])
def test_oracle_reproduces_reference_forward(width):
    from oracle import transformer_ref

    g = _fixture(width)
    cfg = model_cfg("yolov5s-transformer")
    cfg["width_multiple"] = width
    sd = {k: v.double() if v.is_floating_point() else v for k, v in transformer_ref.synth_state_dict(cfg, seed=int(g["seed"][0])).items()}
    x = torch.from_numpy(np.random.RandomState(int(g["seed"][1])).uniform(0, 1, tuple(g["shape"])).astype(np.float32)).double()
    with torch.no_grad():
        z, raws = transformer_ref.forward(cfg, sd, x, fused=True)
    assert np.allclose(z.numpy(), g["z"], rtol=1e-4, atol=1e-4)
    for l, r in enumerate(raws):
        assert np.allclose(r.numpy(), g[f"raw{l}"], rtol=1e-4, atol=1e-4)


def test_refusals():
    tb = mc.TransformerBlock(128, 128, 4, 1)
    assert mc.transformer_spec(tb, training=True) == (4, 32)
    with pytest.raises(NotImplementedError, match="c1 != c2"):
        mc.transformer_spec(mc.TransformerBlock(64, 128, 4, 1), training=False)
    with pytest.raises(NotImplementedError, match="head dim 16"):
        mc.transformer_spec(mc.TransformerBlock(64, 64, 4, 1), training=False)
    tb.tr[0].ma.dropout = 0.1
    assert mc.transformer_spec(tb, training=False) == (4, 32)  # dropout is the identity in eval
    with pytest.raises(NotImplementedError, match="dropout"):
        mc.transformer_spec(tb, training=True)
    for kw in (dict(kdim=64), dict(batch_first=True), dict(add_bias_kv=True), dict(add_zero_attn=True), dict(bias=False)):
        tb = mc.TransformerBlock(128, 128, 4, 1)
        tb.tr[0].ma = nn.MultiheadAttention(128, 4, **kw)
        with pytest.raises(NotImplementedError, match="MultiheadAttention configuration"):
            mc.transformer_spec(tb, training=False)


def test_attention_entry_points_reject_bad_arguments(built_lib):
    lib = _lib.lib()
    buf = (C.c_uint8 * 4096)()
    base = (C.addressof(buf) + 15) // 16 * 16
    lse = base
    f16, st = _lib.dtype_code(torch.float16), None

    def fwd(q=base, pitch=3 * 128, o=base, o_pitch=128, seq=4, heads=2, dh=64, scale=0.125, dtype=f16):
        return lib.y5_attention_fwd(q, q, q, pitch, o, o_pitch, lse, 1, seq, heads, dh, scale, dtype, st)

    def bwd(q=base, pitch=3 * 128, seq=4, heads=2, dh=64, dq=base):
        return lib.y5_attention_bwd(q, q, q, pitch, base, 128, base, 128, lse, lse, dq, dq, dq, pitch, 1, seq, heads, dh, 0.125, f16, st)

    cases = [(lambda: fwd(dh=48), "head_dim 48"), (lambda: fwd(dh=256), "head_dim 256"), (lambda: fwd(seq=0), "seq < 1"),
             (lambda: fwd(q=base + 2), "16-byte aligned"), (lambda: fwd(pitch=100), "qkv_pitch"), (lambda: fwd(o_pitch=64), "o must be"),
             (lambda: fwd(dtype=5), "dtype"), (lambda: fwd(scale=0.0), "scale"), (lambda: bwd(dh=80), "head_dim 80"),
             (lambda: bwd(seq=-1), "seq < 1"), (lambda: bwd(dq=base + 8), "16-byte aligned"), (lambda: bwd(pitch=130), "qkv_pitch")]
    for call, msg in cases:
        assert call() != 0, msg
        assert msg in lib.y5_last_error().decode(), (msg, lib.y5_last_error())
    assert lib.y5_attention_bwd(base, base, base, 384, base, 128, base, 128, None, lse, base, base, base, 384, 1, 4, 2, 64, 0.125, f16, st) != 0
