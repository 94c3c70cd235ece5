"""Per-shape timing of the training kernels (BN statistics / apply / backward, wgrad) on an H100, inside a CUDA graph of
20 back-to-back launches.   python tools/train_kernel_probe.py [batch]"""
import ctypes as C
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from yolov5_b200 import _lib, train_ops


def graph_time(fn, reps=20, iters=5):
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for _ in range(2):
            fn()
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            for _ in range(reps):
                fn()
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
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 16
    dev = torch.device("cuda:0")
    lib = _lib.lib()
    dt = torch.float16
    code = _lib.dtype_code(dt)
    print(f"{'rows':>9} {'C':>4} | {'stats':>7} {'fwd':>7} {'bwd_red':>7} {'bwd_app':>7}  us   (GB/s of the pass in brackets)")
    shapes = ((320, 32), (160, 64), (160, 32), (80, 128), (80, 64), (40, 256), (40, 128), (20, 512), (20, 256))
    if os.environ.get("PROBE_SHAPES") == "m":  # yolov5m's channel widths
        shapes = ((320, 48), (160, 96), (160, 48), (80, 192), (80, 96), (40, 384), (40, 192), (20, 768), (20, 384))
    for hw, c in shapes:
        rows = B * hw * hw
        y = torch.randn(rows, c, device=dev).to(dt)
        dz = torch.randn(rows, c, device=dev).to(dt)
        z = torch.empty_like(y)
        mean, invstd = torch.zeros(c, device=dev), torch.ones(c, device=dev)
        gamma, beta = torch.ones(c, device=dev), torch.zeros(c, device=dev)
        dg, db = torch.empty(c, device=dev), torch.empty(c, device=dev)
        ws = torch.empty(2 * c, dtype=torch.float64, device=dev)

        def st():
            return C.c_void_p(torch.cuda.current_stream().cuda_stream)

        t_stats = graph_time(lambda: lib.y5_bn_stats(y.data_ptr(), c, rows, c, code, ws.data_ptr(), None, st()))
        t_fwd = graph_time(lambda: lib.y5_bn_act_fwd(y.data_ptr(), c, z.data_ptr(), c, rows, c, code, mean.data_ptr(), invstd.data_ptr(),
                                                     gamma.data_ptr(), beta.data_ptr(), 1, 0.0, None, None, 1e-3, 0.03, None, None, None, 0,
                                                     st()))
        t_bwd = graph_time(lambda: lib.y5_bn_act_bwd(y.data_ptr(), c, dz.data_ptr(), c, z.data_ptr(), c, rows, c, code, mean.data_ptr(),
                                                     invstd.data_ptr(), gamma.data_ptr(), beta.data_ptr(), 1, 0.0, dg.data_ptr(), db.data_ptr(),
                                                     ws.data_ptr(), st()))
        nb = rows * c * 2
        print(f"{rows:>9} {c:>4} | {t_stats:7.1f} ({nb / t_stats / 1e3:5.0f}) {t_fwd:7.1f} ({2 * nb / t_fwd / 1e3:5.0f}) {t_bwd:7.1f} ({5 * nb / t_bwd / 1e3:5.0f})",
              flush=True)
    if os.environ.get("PROBE_BN_ONLY"):
        return
    print(f"\nwgrad: {'B,H,W':>12} {'cin':>4} {'cout':>4} k s |     us   TFLOP/s")
    for hw, cin, cout, k, s in ((320, 16, 32, 3, 1), (320, 32, 64, 3, 2), (160, 64, 64, 1, 1), (160, 32, 32, 3, 1), (160, 64, 128, 3, 2),
                                (80, 128, 128, 1, 1), (80, 64, 64, 3, 1), (80, 128, 256, 3, 2), (40, 256, 256, 1, 1), (40, 128, 128, 3, 1),
                                (40, 256, 512, 3, 2), (20, 512, 512, 1, 1), (20, 256, 256, 3, 1), (20, 1024, 512, 1, 1)):
        p = k // 2
        ho = (hw + 2 * p - k) // s + 1
        x = torch.randn(B, cin, hw, hw, device=dev).to(dt).contiguous(memory_format=torch.channels_last)
        dy = torch.randn(B, cout, ho, ho, device=dev).to(dt).contiguous(memory_format=torch.channels_last)
        t = graph_time(lambda: train_ops.conv_wgrad(x, dy, k, s, p))
        fl = 2.0 * B * ho * ho * cout * cin * k * k
        print(f"       {B:>3},{hw:>3},{hw:>3} {cin:>4} {cout:>4} {k} {s} | {t:7.1f}  {fl / t / 1e6:7.1f}", flush=True)


if __name__ == "__main__":
    main()
