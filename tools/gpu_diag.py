"""First-contact diagnostics on an H100: each stage runs in its own subprocess (a trapped kernel kills only its stage)
and prints error summaries rather than asserting.   python tools/gpu_diag.py [stage ...]"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

STAGES = {}


def stage(fn):
    STAGES[fn.__name__] = fn
    return fn


def _conv(label, *case, **kw):
    import torch

    from tests.gpu_util import conv_case, rel_err

    dev = torch.device("cuda:0")
    dtype = kw.pop("dtype", torch.float16)
    got, ref, untouched = conv_case(dev, dtype, *case, **kw)
    e = rel_err(got, ref)
    print(f"  {label:34s} case={case} rel_err={e:.3e} untouched={untouched}", flush=True)
    if e > 5e-3:
        d = (got - ref).abs()
        bad = (d > 5e-3 * ref.abs().max()).float()
        print("    bad fraction", float(bad.mean()), "per-channel bad frac (first 16):", bad.mean((0, 2, 3))[:16].tolist())
        print("    per-row(y) bad frac:", bad.mean((0, 1, 3))[:16].tolist())
        print("    got[0,:4,0,:6]", got[0, :4, 0, :6].tolist())
        print("    ref[0,:4,0,:6]", ref[0, :4, 0, :6].tolist())


@stage
def s1_gemm_1x1():
    _conv("1x1 K=64 N=64", 2, 16, 16, 64, 64, 1, 1, 0)
    _conv("1x1 K=128 N=256 Mtail", 1, 20, 20, 128, 256, 1, 1, 0)
    _conv("1x1 bk32", 3, 8, 12, 32, 32, 1, 1, 0)
    _conv("1x1 bk16", 3, 8, 12, 16, 32, 1, 1, 0)
    _conv("1x1 cin24", 2, 12, 12, 24, 48, 1, 1, 0)
    _conv("1x1 direct kernel", 2, 16, 16, 64, 64, 1, 1, 0, direct=True)


@stage
def s2_im2col():
    _conv("3x3 s1 bk64", 2, 20, 20, 64, 64, 3, 1, 1)
    _conv("3x3 s1 bk16", 2, 16, 16, 16, 32, 3, 1, 1)
    _conv("3x3 s2", 2, 16, 24, 32, 64, 3, 2, 1)
    _conv("3x3 s1 128ch", 1, 40, 40, 128, 128, 3, 1, 1)
    _conv("3x3 s2 deep", 2, 10, 10, 256, 512, 3, 2, 1)
    _conv("3x3 tiny (<128KiB tensor)", 1, 8, 8, 64, 64, 3, 1, 1)


@stage
def s2b_patch_mode():
    for a_mode in (1, 2):
        _conv(f"3x3 s1 a_mode={a_mode}", 2, 20, 20, 64, 64, 3, 1, 1, a_mode=a_mode)
        _conv(f"3x3 s1 80x80 a_mode={a_mode}", 1, 80, 80, 64, 64, 3, 1, 1, a_mode=a_mode)
        _conv(f"3x3 s1 13x27 res+slices a_mode={a_mode}", 3, 13, 27, 32, 64, 3, 1, 1, a_mode=a_mode, residual=True, in_extra=8, out_extra=24)
        _conv(f"3x3 s1 bk16 a_mode={a_mode}", 2, 16, 16, 16, 32, 3, 1, 1, a_mode=a_mode)
        _conv(f"3x3 s1 9x130 N=32 a_mode={a_mode}", 2, 9, 130, 64, 32, 3, 1, 1, a_mode=a_mode)


@stage
def s3_epilogue_variants():
    import torch

    _conv("residual+slices", 2, 20, 20, 64, 64, 3, 1, 1, residual=True, in_extra=24, out_extra=40)
    _conv("bf16", 2, 20, 20, 64, 64, 3, 1, 1, dtype=torch.bfloat16)
    for bn in (32, 64, 128, 256):
        _conv(f"block_n {bn}", 2, 20, 20, 64, 256, 3, 1, 1, block_n=bn)
    _conv("many tiles", 8, 80, 80, 64, 64, 3, 1, 1)
    for bn in (128, 256):
        _conv(f"MT=2 block_n {bn} im2col", 2, 20, 20, 64, 256, 3, 1, 1, block_n=bn, mt2=True, a_mode=1, residual=True)
        _conv(f"MT=2 block_n {bn} patch", 2, 20, 20, 64, 256, 3, 1, 1, block_n=bn, mt2=True, a_mode=2, residual=True)
        _conv(f"MT=2 block_n {bn} 1x1", 3, 16, 16, 128, 256, 1, 1, 0, block_n=bn, mt2=True)
        _conv(f"MT=2 block_n {bn} s2 N=384", 1, 40, 40, 128, 384, 3, 2, 1, block_n=bn, mt2=True)


@stage
def s3b_cluster():
    for bn, mt2 in ((128, False), (128, True), (256, False), (256, True)):
        _conv(f"cluster2 bn{bn} mt2={mt2} patch", 4, 40, 40, 64, 256, 3, 1, 1, block_n=bn, mt2=mt2, cluster=2, a_mode=2, residual=True)
        _conv(f"cluster2 bn{bn} mt2={mt2} 1x1 odd", 5, 24, 24, 128, 512, 1, 1, 0, block_n=bn, mt2=mt2, cluster=2)
        _conv(f"cluster2 bn{bn} mt2={mt2} s2", 3, 40, 40, 128, 384, 3, 2, 1, block_n=bn, mt2=mt2, cluster=2)


@stage
def s4_model():
    import numpy as np
    import torch

    from oracle import model_ref
    from yolov5_b200.cfg import model_cfg
    from yolov5_b200.models.yolo import DetectionModel

    dev = torch.device("cuda:0")
    for name, shape in (("yolov5n", (2, 3, 96, 128)), ("yolov5s", (1, 3, 64, 64)), ("yolov5s", (2, 3, 640, 640))):
        cfg = model_cfg(name)
        sd = model_ref.synth_state_dict(cfg, seed=10)
        x = torch.from_numpy(np.random.RandomState(1).uniform(0, 1, shape).astype(np.float32))
        with torch.no_grad():
            ref = model_ref.forward(cfg, sd, x.half().float(), fused=True)
        m = DetectionModel(name)
        m.load_state_dict(sd)
        m = m.to(dev).half().eval()
        os.environ["Y5_NO_GRAPH"] = "1"
        out = m(x.to(dev).half())
        torch.cuda.synchronize()
        z = out[0].float().cpu()
        print(f"  {name} {shape}: z rel err {float((z - ref[0]).abs().max() / ref[0].abs().max()):.3e}", flush=True)
        for l, (a, b) in enumerate(zip(out[1], ref[1])):
            print(f"     raw{l} rel err {float((a.float().cpu() - b).abs().max() / b.abs().max()):.3e}")
        os.environ["Y5_NO_GRAPH"] = "0"
        z2 = m(x.to(dev).half())[0].float().cpu()
        print(f"     graph replay == eager: {bool(torch.equal(z, z2))}")
        # per-layer check against the oracle intermediate activations
        prog = m._program(x.to(dev).half())
        print(f"     launches/forward {prog.launches_per_forward()}  GFLOP {prog.flops / 1e9:.2f}")


@stage
def s5_nms():
    import numpy as np
    import torch

    from oracle import nms_ref
    from yolov5_b200.utils.general import non_max_suppression

    dev = torch.device("cuda:0")
    for tag, dtype, kw, n, bs in (("detect fp16", "fp16", dict(conf_thres=0.25, iou_thres=0.45, max_det=1000), 25200, 3),
                                  ("val fp32", "fp32", dict(conf_thres=0.001, iou_thres=0.6, multi_label=True, max_det=300), 25200, 2),
                                  ("val fp16", "fp16", dict(conf_thres=0.001, iou_thres=0.6, multi_label=True, max_det=300), 25200, 2)):
        pred = nms_ref.synth_predictions(bs, n, 80, 0, 2, dtype)
        t = torch.from_numpy(pred).to(dev, {"fp16": torch.float16, "fp32": torch.float32}[dtype])
        out, idx = non_max_suppression(t, return_indices=True, **kw)
        ref, ridx = nms_ref.non_max_suppression(pred, dtype=dtype, return_index=True, **kw)
        for b in range(bs):
            o = out[b].cpu().numpy()
            same_idx = o.shape[0] == ref[b].shape[0] and np.array_equal(idx[b].cpu().numpy(), ridx[b])
            same = o.shape == ref[b].shape and np.array_equal(o, ref[b])
            print(f"  {tag} img{b}: n={o.shape[0]} ref={ref[b].shape[0]} idx_equal={same_idx} rows_equal={same}", flush=True)
            if not same_idx and o.shape[0] and ref[b].shape[0]:
                k = min(o.shape[0], ref[b].shape[0])
                gi, ri = idx[b].cpu().numpy()[:k], ridx[b][:k]
                first = int(np.argmax(gi != ri)) if np.any(gi != ri) else -1
                print("     first diff at", first, gi[max(0, first - 2):first + 3], ri[max(0, first - 2):first + 3])


@stage
def s6_loss():
    import numpy as np
    import torch

    from oracle import loss_ref, model_ref
    from yolov5_b200.cfg import HYP_SCRATCH_LOW, model_cfg
    from yolov5_b200.models.yolo import DetectionModel
    from yolov5_b200.utils.loss import ComputeLoss

    dev = torch.device("cuda:0")
    m = DetectionModel("yolov5n")
    m.load_state_dict(model_ref.synth_state_dict(model_cfg("yolov5n"), seed=30))
    m.hyp = dict(HYP_SCRATCH_LOW)
    m = m.to(dev)
    crit = ComputeLoss(m)
    anchors = m.model[-1].anchors.detach().cpu().numpy()
    rs = np.random.RandomState(31)
    pn = [rs.normal(0, 1.5, (4, 3, 128 // s, 160 // s, 85)).astype(np.float32) for s in (8, 16, 32)]
    tg = loss_ref.synth_targets(4, 31)
    p = [torch.from_numpy(a).to(dev).requires_grad_(True) for a in pn]
    loss, items = crit(p, torch.from_numpy(tg).to(dev))
    loss.backward()
    p2 = [torch.from_numpy(a).requires_grad_(True) for a in pn]
    lo, it = loss_ref.compute_loss(p2, tg, anchors, HYP_SCRATCH_LOW)
    lo.backward()
    print("  loss", loss.item(), lo.item(), "items", items.tolist(), it.tolist())
    for l, (a, b) in enumerate(zip(p, p2)):
        print(f"  grad{l} rel err {float((a.grad.cpu() - b.grad).abs().max() / b.grad.abs().max()):.3e}")
    bt = loss_ref.build_targets(tg, anchors, [tuple(t.shape[2:4]) for t in p], 4.0)
    tcls, tbox, indices, anch = crit.build_targets(p, torch.from_numpy(tg).to(dev))
    for l in range(3):
        ok = all(np.array_equal(indices[l][q].cpu().numpy(), bt[l][k]) for q, k in enumerate(("b", "a", "gj", "gi")))
        print(f"  targets{l}: n={len(tcls[l])} ref={len(bt[l]['b'])} idx_equal={ok} tbox_equal={np.array_equal(tbox[l].cpu().numpy(), bt[l]['tbox'])}")


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--run":
        STAGES[sys.argv[2]]()
        sys.exit(0)
    names = sys.argv[1:] or list(STAGES)
    for n in names:
        print(f"== {n}", flush=True)
        try:
            r = subprocess.run([sys.executable, __file__, "--run", n], timeout=420, capture_output=True, text=True, cwd=ROOT)
            print(r.stdout[-6000:])
            if r.returncode != 0:
                print(f"   STAGE FAILED rc={r.returncode}\n{r.stderr[-3000:]}")
        except subprocess.TimeoutExpired as e:
            print("   STAGE TIMED OUT", (e.stdout or b"")[-2000:] if isinstance(e.stdout, bytes) else e.stdout)
