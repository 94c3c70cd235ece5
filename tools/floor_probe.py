"""Per-launch floor / per-tile slope of conv_gemm: times back-to-back launches of one plan inside a CUDA graph.

usage: python tools/floor_probe.py            (on an H100)
For each (N, K, ksize) the row count M is swept in whole waves of <SM count> x 128-row tiles; the intercept of time vs waves is
the fixed cost of a launch, the slope the steady-state cost of one tile per CTA.
"""
import ctypes as C
import sys, os

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from yolov5_b200 import _lib
from yolov5_b200.engine import ConvInput, conv_desc, pack_weight


def plan_for(dev, dtype, M, cin, cout, k):
    lib = _lib.lib()
    W = 128
    H = M // W
    x = torch.randn(1, H, W, cin, device=dev, dtype=dtype)
    y = torch.empty(1, H, W, cout, device=dev, dtype=dtype)
    bk, bn = C.c_int32(), C.c_int32()
    _lib.check(lib.y5_conv_pick(cin, cout, M, C.byref(bk), C.byref(bn)))
    w = torch.randn(cout, cin, k, k) / (cin * k * k) ** 0.5
    wp = pack_weight(w, bk.value, dtype).to(dev)
    b = torch.zeros(cout, device=dev)
    d = conv_desc(ConvInput(x.data_ptr(), cin, 1, H, W, cin), wp, b, bk.value, y.data_ptr(), cout, k, 1, k // 2, True, dtype)
    plan = C.c_void_p()
    _lib.check(lib.y5_conv_plan_create(C.byref(d), C.byref(plan)))
    return plan, (x, y, wp, b)


def time_plan(plan, reps=20, iters=10):
    lib = _lib.lib()
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for _ in range(3):
            lib.y5_conv_plan_run(plan, C.c_void_p(st.cuda_stream))
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            for _ in range(reps):
                lib.y5_conv_plan_run(plan, C.c_void_p(st.cuda_stream))
        g.replay()
        st.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for _ in range(iters):
            g.replay()
        e1.record(st)
        st.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (reps * iters)


def main():
    dev = torch.device("cuda:0")
    dtype = torch.float16
    print(f"{'N':>5} {'K':>5} {'k':>2} | " + " ".join(f"{w:>7}w" for w in (1, 2, 3, 4, 8, 16)) + "   (us per launch; w = 128-row tiles per SM)")
    for cout, cin, k in ((32, 32, 1), (64, 64, 1), (128, 128, 1), (256, 256, 1), (512, 512, 1), (128, 128, 3), (256, 256, 3), (64, 64, 3), (512, 1024, 1)):
        row = []
        for waves in (1, 2, 3, 4, 8, 16):
            M = 128 * torch.cuda.get_device_properties(0).multi_processor_count * waves
            plan, keep = plan_for(dev, dtype, M, cin, cout, k)
            row.append(time_plan(plan))
            _lib.lib().y5_conv_plan_destroy(plan)
            del keep
        print(f"{cout:>5} {cin:>5} {k:>2} | " + " ".join(f"{t:>8.2f}" for t in row), flush=True)


if __name__ == "__main__":
    main()
