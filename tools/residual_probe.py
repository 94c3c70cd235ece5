"""Cost of the Bottleneck residual add in the conv epilogue, per residual layer shape of yolov5l (64 x 640², bf16) and
yolov5s (32 x 640², fp16).  Each shape is planned three ways with the library's default choices and timed with CUDA events:
no residual, the residual in a separate buffer, and the residual in place (residual == out, as the engine lowers a C3
Bottleneck: both are the first c_ channels of the C3's concat buffer).  The variants are interleaved round by round.
    python tools/residual_probe.py [--reps 200] [--rounds 5]"""
import argparse
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from yolov5_b200 import _lib
from yolov5_b200.engine import ConvInput, conv_desc, pack_weight

# (model, batch, dtype, [(map size, c_)]) -- the 3x3 c_ -> c_ m{j}.cv2 convs of backbone layers 2, 4, 6 and 8
SHAPES = [("yolov5l", 64, torch.bfloat16, [(160, 64), (80, 128), (40, 256), (20, 512)]),
          ("yolov5s", 32, torch.float16, [(160, 32), (80, 64), (40, 128), (20, 256)])]
VARIANTS = ("none", "separate", "in-place")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0) + ", power limit not read"


def copy_bandwidth(dev):
    """bytes moved per second by a 1 GiB device-to-device copy (read + write)"""
    a = torch.empty(1 << 29, dtype=torch.float16, device=dev)
    b = torch.empty_like(a)
    for _ in range(3):
        b.copy_(a)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        b.copy_(a)
    e1.record()
    torch.cuda.synchronize()
    return 2 * a.numel() * 2 * 20 / (e0.elapsed_time(e1) * 1e-3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200, help="launches per timed window")
    ap.add_argument("--rounds", type=int, default=5, help="interleaved windows per variant (the median is reported)")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    lib = _lib.lib()
    st = _lib.stream_ptr(dev)
    bw = copy_bandwidth(dev)
    print(f"card: {card()}; lib: {_lib.LIB_PATH}; measured copy bandwidth {bw / 1e12:.2f} TB/s")
    print(f"{'model':8s} {'map':>4s} {'c_':>4s} {'M':>8s} {'variant':9s} {'us':>8s} {'TFLOP/s':>8s} {'floor us':>9s} {'x floor':>8s}")
    g = torch.Generator(device=dev).manual_seed(0)
    for model, bs, dt, layers in SHAPES:
        for hw, c in layers:
            M, K = bs * hw * hw, 9 * c
            x = (torch.rand(bs, hw, hw, c, generator=g, device=dev) - 0.5).to(dt)
            cat = (torch.rand(bs, hw, hw, 2 * c, generator=g, device=dev) - 0.5).to(dt) * 0.01  # out / residual: channels [0, c)
            sep = (torch.rand(bs, hw, hw, 2 * c, generator=g, device=dev) - 0.5).to(dt) * 0.01
            w = (torch.rand(c, c, 3, 3, generator=g, device=dev) - 0.5) / K ** 0.5
            bk, bn = C.c_int32(), C.c_int32()
            _lib.check(lib.y5_conv_pick(c, c, M, C.byref(bk), C.byref(bn)))
            wp = pack_weight(w, bk.value, dt)
            bias = torch.zeros(c, dtype=torch.float32, device=dev)
            plans = {}
            for v in VARIANTS:
                res = {"none": (None, 0), "separate": (sep.data_ptr(), 2 * c), "in-place": (cat.data_ptr(), 2 * c)}[v]
                d = conv_desc(ConvInput(x.data_ptr(), c, bs, hw, hw, c), wp, bias, bk.value, cat.data_ptr(), 2 * c, 3, 1, 1, True, dt, *res)
                plan = C.c_void_p()
                _lib.check(lib.y5_conv_plan_create(C.byref(d), C.byref(plan)), "plan")
                plans[v] = plan
            times = {v: [] for v in VARIANTS}
            for v in VARIANTS:  # warm-up
                for _ in range(5):
                    _lib.check(lib.y5_conv_plan_run(plans[v], C.c_void_p(st)), "run")
            for _ in range(a.rounds):
                for v in VARIANTS:
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(a.reps):
                        lib.y5_conv_plan_run(plans[v], C.c_void_p(st))
                    e1.record()
                    torch.cuda.synchronize()
                    times[v].append(e0.elapsed_time(e1) * 1e3 / a.reps)
            for v in VARIANTS:
                us = sorted(times[v])[len(times[v]) // 2]
                byt = 2 * (M * c + M * c + (M * c if v != "none" else 0) + c * K)  # input, output, residual, weights
                floor = byt / bw * 1e6
                print(f"{model:8s} {hw:4d} {c:4d} {M:8d} {v:9s} {us:8.1f} {2 * M * c * K / us / 1e6:8.1f} {floor:9.1f} {us / floor:8.2f}")
            for v in VARIANTS:
                lib.y5_conv_plan_destroy(plans[v])
            del x, cat, sep


if __name__ == "__main__":
    main()
