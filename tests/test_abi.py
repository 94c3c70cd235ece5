"""CPU: the C-ABI library builds for sm_90a, loads, and exports every symbol include/y5b200.h declares
(no compute calls here -- there is no GPU in the build container)."""
import ctypes
import os
import re
import subprocess

from yolov5_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "y5b200.h")


def _declared():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(y5_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_the_entry_points():
    names = _declared()
    for must in ("y5_conv_plan_create", "y5_conv_plan_run", "y5_detect_plan_create", "y5_stem_s2d", "y5_sppf_pool",
                 "y5_upsample2x", "y5_nms_batched", "y5_box_iou", "y5_loss_fwd_bwd_scaled", "y5_last_error"):
        assert must in names


def test_library_exports_every_declared_symbol(built_lib):
    handle = ctypes.CDLL(_lib.LIB_PATH)
    missing = [n for n in _declared() if not hasattr(handle, n)]
    assert not missing, missing
    assert sorted(_lib.SIGNATURES) == _declared()  # the ctypes table mirrors the header one to one


def test_library_is_sm90a_with_wgmma_and_tma(built_lib):
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in sass
    for mnemonic in ("HGMMA.64x", "UTMALDG", "UTMALDG.4D.IM2COL"):  # wgmma, TMA, im2col TMA
        assert mnemonic in sass, mnemonic
    # the weight-gradient kernel is a wgmma kernel of its own (MN-major operands) with vector fp32 reductions
    wg = sass[sass.index("conv_wgrad_kernel"):]
    wg = wg[: wg.index("Function :", 10)] if "Function :" in wg[10:] else wg
    for mnemonic in ("HGMMA.64x64x16.F32", "UTMALDG", "REDG.E.ADD.F32x2"):
        assert mnemonic in wg, mnemonic


def test_wgrad_and_bn_pass_argument_validation_without_gpu(built_lib):
    lib = built_lib
    d = _lib.WgradDesc()
    assert lib.y5_conv_wgrad(ctypes.byref(d), None) == -1 and b"null" in lib.y5_last_error()
    assert lib.y5_bn_workspace_bytes(64) == 64 * 2 * 8
    assert lib.y5_sppf_bwd_workspace_bytes(2, 20, 20, 128) == 3 * 2 * 20 * 20 * 128 * 4
    assert lib.y5_bn_stats(None, 64, 10, 64, _lib.Y5_F16, None, None, None) == -1
    assert lib.y5_weight_pack(None, _lib.Y5_F32, 8, 8, 1, None, 8, None, 8, _lib.Y5_F16, None) == -1
    assert lib.y5_weight_pack_chunk_elems() > 0
    assert lib.y5_weight_pack_multi(None, None, None, 3, _lib.Y5_F16, None) == -1 and lib.y5_weight_pack_multi(None, None, None, 0, _lib.Y5_F16, None) == 0


def test_pre_post_optimizer_argument_validation_without_gpu(built_lib):
    """The section-8(f) entry points reject bad arguments before touching the device."""
    lib = built_lib
    assert lib.y5_letterbox(None, 1, 640, 640, 1, 114, None, _lib.Y5_U8, 0, 0, 0, None) == -1
    im = _lib.LetterboxImage()
    im.data, im.src_h, im.src_w, im.row_bytes, im.new_h, im.new_w, im.top, im.left = 4096, 480, 640, 1920, 480, 640, 100, 0
    assert lib.y5_letterbox(ctypes.byref(im), 1, 512, 640, 1, 114, 4096, _lib.Y5_U8, 0, 0, 0, None) == -1  # 100 + 480 > 512
    assert b"does not fit" in lib.y5_last_error()
    assert lib.y5_letterbox_max_images() >= 8
    assert lib.y5_process_mask_workspace_bytes(10, 160, 160, 0) == 0
    assert lib.y5_process_mask_workspace_bytes(10, 160, 160, 1) >= 10 * 160 * 160 * 4
    assert lib.y5_process_mask(4096, _lib.Y5_F16, 1, 128, 160, 160, 4096, 38, 4096, 38, None, 3, 640, 640, 0, None, 4096, _lib.Y5_F32, None,
                               0, None) == -2  # 128 prototype channels
    assert lib.y5_match_batch(4096, 1800, 6, None, 2, 5000, None, 0, 4096, 10, 1e-7, 4096, None) == -2  # max_det cap
    assert lib.y5_scale_boxes(None, 6, 10, None, 0, None, None, None) == -1
    assert lib.y5_opt_chunk_elems() > 0 and lib.y5_opt_step(None, None, None, 4, None, None, 1, 1, 1, None) == -1
    assert lib.y5_grad_pack(None, None, None, 4, None, None, None, None) == -1 and lib.y5_grad_pack(None, None, None, 0, None, None, None, None) == 0
    assert lib.y5_grad_bind(None, 4, None, None, None, None) == -1 and lib.y5_grad_bind(None, 0, None, None, None, None) == 0
    assert lib.y5_fold_pack(None, _lib.Y5_F32, 8, 8, 1, 1, None, None, None, None, None, _lib.Y5_F32, 1e-3, None, 8, 8, None, _lib.Y5_F16, None) == -1
    assert lib.y5_loss_fwd_bwd_scaled(None, None, None, None, None, None, None, None, 0, None) == -1


def test_abi_version_and_argument_validation_without_gpu(built_lib):
    lib = built_lib
    assert lib.y5_version() == 2
    d = _lib.ConvDesc()  # all null
    plan = ctypes.c_void_p()
    assert lib.y5_conv_plan_create(ctypes.byref(d), ctypes.byref(plan)) == -1  # Y5_E_INVALID
    assert b"null" in lib.y5_last_error()
    p = _lib.NmsParams()
    p.batch, p.n_rows, p.no, p.nc, p.nm, p.dtype = 2, 100, 85, 80, 0, _lib.Y5_F16
    p.conf_thres, p.iou_thres, p.max_det, p.max_nms = 0.25, 0.45, 300, 30000
    assert lib.y5_nms_workspace_bytes(ctypes.byref(p)) > 0
    p.no = 84
    assert lib.y5_nms_workspace_bytes(ctypes.byref(p)) == -1
    bk, bn = ctypes.c_int32(), ctypes.c_int32()
    assert lib.y5_conv_pick(128, 256, 51200, ctypes.byref(bk), ctypes.byref(bn)) == 0
    assert bk.value == 64 and bn.value in (128, 256)


PLAIN_TAGS = ("y5_conv_plan_info",)


def _header_structs():
    """{struct name: [field names in declaration order]} parsed from include/y5b200.h (typedefs and plain struct tags)"""
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    out = {}
    found = re.findall(r"typedef struct \w+ \{(.*?)\}\s*(\w+);", src, flags=re.S)
    # plain struct tags whose C type name is taken by a function of the same name
    found += [(body, name) for name, body in re.findall(r"(?<!typedef )struct (\w+) \{(.*?)\};", src, flags=re.S)
              if name in PLAIN_TAGS]
    for body, name in found:
        fields = []
        for decl in body.split(";"):
            decl = decl.strip()
            if not decl:
                continue
            first, *rest = decl.split(",")
            names = [first.split()[-1]] + [r.strip() for r in rest]
            fields += [re.sub(r"\[.*\]", "", n).lstrip("*").strip() for n in names]
        out[name] = fields
    return out


def test_ctypes_structs_match_the_c_layout(tmp_path):
    """sizeof / offsetof of every struct in the header (compiled by gcc) == the ctypes mirrors in yolov5_b200/_lib.py."""
    mirrors = {"y5_conv_desc": _lib.ConvDesc, "y5_detect_desc": _lib.DetectDesc, "y5_nms_params": _lib.NmsParams,
               "y5_loss_params": _lib.LossParams, "y5_wgrad_desc": _lib.WgradDesc, "y5_letterbox_image": _lib.LetterboxImage,
               "y5_opt_tensor": _lib.OptTensor, "y5_pack_item": _lib.PackItem,
               "y5_conv_plan_info": _lib.PlanInfo}
    structs = _header_structs()
    assert sorted(structs) == sorted(mirrors), (sorted(structs), sorted(mirrors))
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{HEADER}"', "int main(void) {"]
    for s, fields in structs.items():
        t = f"struct {s}" if s in PLAIN_TAGS else s
        lines.append(f'  printf("{s} %zu", sizeof({t}));')
        for f in fields:
            lines.append(f'  printf(" %zu", offsetof({t}, {f}));')
        lines.append('  printf("\\n");')
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-o", str(exe), str(src)], check=True)
    got = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.strip().splitlines()
    for line in got:
        name, size, *offs = line.split()
        cls = mirrors[name]
        assert int(size) == ctypes.sizeof(cls), (name, size, ctypes.sizeof(cls))
        py = [getattr(cls, f).offset for f, _ in cls._fields_]
        assert [int(o) for o in offs] == py, (name, offs, py)
