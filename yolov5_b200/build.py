"""In-tree build of liby5b200.so (hand-written sm_90a kernels + C ABI) with nvcc.

    python -m yolov5_b200.build            # incremental
    python -m yolov5_b200.build --force

The shared object is written next to this file (yolov5_b200/liby5b200.so) so it travels with the repo snapshot to
the GPU machine; nvcc cross-compiles for sm_90a without a GPU.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "liby5b200.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden"]
# file -> extra flags.  nms.cu / loss.cu hold bit-exact integer/index paths: no FMA contraction there.
SOURCES = {
    "host_util.cu": [],
    "conv_gemm.cu": [],
    "conv_wgrad.cu": [],
    "aux_kernels.cu": [],
    "train_kernels.cu": [],
    "nms.cu": ["-fmad=false"],
    "loss.cu": ["-fmad=false"],
    "post_kernels.cu": ["-fmad=false"],
    "mask_metrics.cu": ["-fmad=false"],
    "optim_kernels.cu": [],
    "aug_kernels.cu": ["-fmad=false"],
    "seg_aug_kernels.cu": ["-fmad=false"],
    "cls_kernels.cu": [],
    "attention.cu": [],
    "pool_kernels.cu": [],
    "ap_metrics.cu": ["-fmad=false"],
}


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def _stale(target: str, deps: list[str]) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    headers.append(os.path.join(os.path.dirname(HERE), "include", "y5b200.h"))
    nvcc = _nvcc()
    jobs = []
    objs = []
    for src, extra in SOURCES.items():
        s = os.path.join(CSRC, src)
        if not os.path.exists(s):
            continue
        o = os.path.join(OBJ, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _stale(o, [s, __file__] + headers):
            jobs.append([nvcc, *ARCH, *COMMON, *extra, "-c", s, "-o", o])

    def run(cmd):
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed: {' '.join(cmd)}\n{r.stdout}\n{r.stderr}")
        return r

    with ThreadPoolExecutor(max_workers=max(1, min(len(jobs), os.cpu_count() or 1))) as ex:
        list(ex.map(run, jobs))
    if jobs or force or _stale(LIB, objs):
        run([nvcc, *ARCH, "-shared", "-o", LIB, *objs, "-cudart", "static"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
