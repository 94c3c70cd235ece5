"""Per-launch timing of one forward program (CUDA events behind a queued blocker) with algorithmic bytes / FLOPs.
    python tools/layer_profile.py [model] [batch] [size] [dtype]"""
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from yolov5_b200 import _lib, engine
from yolov5_b200.models.yolo import DetectionModel

name = sys.argv[1] if len(sys.argv) > 1 else "yolov5s"
bs = int(sys.argv[2]) if len(sys.argv) > 2 else 32
size = int(sys.argv[3]) if len(sys.argv) > 3 else 640
dt = {"fp16": torch.float16, "bf16": torch.bfloat16}[sys.argv[4] if len(sys.argv) > 4 else "fp16"]
dev = torch.device("cuda:0")

# record per-conv metadata by wrapping Program.emit_conv
meta = {}
_orig = engine.Program.emit_conv


def emit_conv(self, d, name, keep):
    n0 = len(self.ops)
    _orig(self, d, name, keep)
    k, s, n = d.ksize, d.stride, d.out_c
    kw, pad_w = (d.kw, d.pad_w) if d.kw else (k, d.pad)
    m = d.batch * ((d.in_h + 2 * d.pad - k) // s + 1) * ((d.in_w + 2 * pad_w - kw) // s + 1)
    if d.in_x_stride:  # stem: count the real 6x6x3 filter and the image
        cin, kk, in_el = 3, 36, self.B * self.H * self.W * 3
    else:
        cin, kk, in_el = d.in_c, k * k, d.batch * d.in_h * d.in_w * d.in_c
    meta[n0] = dict(name=name, M=m, N=n, K=cin * kk, k=k, s=s, flops=2 * m * n * cin * kk,
                    bytes=2 * (in_el + m * n) + 2 * n * cin * kk + (2 * m * n if d.residual else 0))


engine.Program.emit_conv = emit_conv
torch.manual_seed(0)
m = DetectionModel(name).to(dev, dt).eval()
x = torch.rand(bs, 3, size, size, device=dev).to(dt)
prog = m._program(x)
m(x)
torch.cuda.synchronize()
st = _lib.stream_ptr(dev)
evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in prog.ops]
acc = [0.0] * len(prog.ops)
reps = 5
for _ in range(reps):
    torch.cuda._sleep(40_000_000)
    for op, (s, e) in zip(prog.ops, evs):
        s.record(); op.run(st); e.record()
    torch.cuda.synchronize()
    for i, (s, e) in enumerate(evs):
        acc[i] += s.elapsed_time(e) / reps
tot = sum(acc)


def plan_cols(op):
    """tile (rows x cols), pipeline stages a/b and the epilogue (tma | direct) of a conv launch"""
    if op.fn is not prog.lib.y5_conv_plan_run:
        return ""
    info = _lib.PlanInfo()
    _lib.check(prog.lib.y5_conv_plan_info(op.args[0], C.byref(info)), "conv_plan_info")
    return f"{128 * info.mt:>4d}x{info.block_n:<4d} {info.a_stages}/{info.b_stages} {'tma' if info.tma_epi else 'direct'}"


# floors: NVIDIA's H100 SXM data-sheet rates (989 TFLOP/s dense fp16/bf16, 3.35 TB/s HBM3), not measured ones
props = torch.cuda.get_device_properties(dev)
smi = os.popen("nvidia-smi --query-gpu=power.limit,clocks.max.sm --format=csv,noheader -i 0").read().strip()
print(f"{props.name} ({smi})")
print(f"{name} bs={bs} {size} {dt}: fixed ops {tot:.3f} ms ({len(prog.ops)} launches)")
print(f"{'op':28s} {'M':>8s} {'N':>5s} {'K':>5s} {'us':>8s} {'GB/s':>7s} {'TF/s':>6s} {'tensor-floor':>12s} {'hbm-floor':>9s}  tile      st  epilogue")
for i, op in enumerate(prog.ops):
    md = meta.get(i)
    if md:
        us = acc[i] * 1e3
        print(f"{md['name']:28s} {md['M']:8d} {md['N']:5d} {md['K']:5d} {us:8.1f} {md['bytes'] / us / 1e3:7.0f} {md['flops'] / us / 1e6:6.1f} "
              f"{md['flops'] / 989e6:12.1f} {md['bytes'] / 3350e3:9.1f}  {plan_cols(op)}")
    else:
        print(f"{op.name:28s} {'':8s} {'':5s} {'':5s} {acc[i] * 1e3:8.1f}")
# Detect-head GEMMs (they run outside the captured graph: fresh output tensors per call)
no = prog.det_shapes[0][-1]
zbuf = torch.empty(prog.B, prog.z_rows, no, dtype=prog.dtype, device=dev)
raws = [torch.empty(sh, dtype=prog.dtype, device=dev) for sh in prog.det_shapes]
hev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in prog.head_ops]
hacc = [0.0] * len(prog.head_ops)
for _ in range(reps):
    torch.cuda._sleep(40_000_000)
    for plan, raw, (s, e) in zip(prog.head_ops, raws, hev):
        s.record()
        _lib.check(prog.lib.y5_detect_plan_run_to(plan, raw.data_ptr(), zbuf.data_ptr(), C.c_void_p(st)), "detect")
        e.record()
    torch.cuda.synchronize()
    for i, (s, e) in enumerate(hev):
        hacc[i] += s.elapsed_time(e) / reps
for i, sh in enumerate(prog.det_shapes):
    mrows = sh[0] * sh[2] * sh[3]
    byt = 2 * (mrows * prog.outs[[17, 20, 23][i]].c + 2 * mrows * sh[1] * sh[4]) if len(prog.outs) > 23 else 0
    print(f"{'detect.' + str(i):28s} {mrows:8d} {sh[1] * sh[4]:5d} {'':5s} {hacc[i] * 1e3:8.1f} {byt / max(hacc[i], 1e-9) / 1e6:7.0f} {'':6s} {'':12s} {byt / 3350e3:9.1f}")
print(f"fixed ops + head {tot + sum(hacc):.3f} ms")
# head + stem timing
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
torch.cuda.synchronize()
e0.record()
for _ in range(10):
    m(x)
e1.record()
torch.cuda.synchronize()
print(f"full forward (graph + stem + head) {e0.elapsed_time(e1) / 10:.3f} ms")
