"""The ctypes mirrors in make-it-3d_b200/_lib.py and nerf/sd.py against include/mi3d.h, field by field: a C program compiled from the header with
gcc prints sizeof / offsetof of every struct member; they must equal what ctypes lays out.  (The C ABI passes these structs by pointer:
a drifted mirror corrupts arguments silently.)  CPU only."""
import ctypes
import importlib
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PAIRS = [("mi3d_hashgrid", "_lib", "HashGrid"), ("mi3d_raygen", "_lib", "RayGen"), ("mi3d_mlp", "_lib", "Mlp"), ("mi3d_epilogue", "_lib", "Epilogue"),
         ("mi3d_field_cfg", "_lib", "FieldCfg"), ("mi3d_field_io", "_lib", "FieldIO"), ("mi3d_view_segs", "_lib", "ViewSegs"),
         ("mi3d_adan_cfg", "_lib", "AdanCfg"), ("mi3d_render_args", "_lib", "RenderArgs"), ("mi3d_render_eval_args", "_lib", "RenderEvalArgs"),
         ("mi3d_render_ws", "_lib", "RenderWs"), ("mi3d_op_gemm_args", "_lib", "OpGemmArgs"), ("mi3d_unet_cfg", "nerf.sd", "UNetCfg"), ("mi3d_vae_cfg", "nerf.sd", "VaeCfg")]


def test_ctypes_mirrors_match_the_header_layout(tmp_path):
    classes = []
    for cname, mod, pyname in PAIRS:
        m = importlib.import_module("make-it-3d_b200." + mod)
        classes.append((cname, getattr(m, pyname)))
    src = ['#include <stdio.h>', '#include <stddef.h>', '#include "mi3d.h"', 'int main(void) {']
    for cname, cls in classes:
        src.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, *_ in cls._fields_:
            src.append(f'  printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    src += ['  return 0;', '}']
    c = tmp_path / "layout.c"
    c.write_text("\n".join(src))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(exe)], check=True)
    out = dict(l.split() for l in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines())
    for cname, cls in classes:
        assert int(out[cname]) == ctypes.sizeof(cls), (cname, out[cname], ctypes.sizeof(cls))
        for fname, *_ in cls._fields_:
            assert int(out[f"{cname}.{fname}"]) == getattr(cls, fname).offset, (cname, fname)


def test_enum_values_match_the_header():
    L = importlib.import_module("make-it-3d_b200._lib")
    hdr = open(os.path.join(ROOT, "include", "mi3d.h")).read()
    import re
    vals = {k: int(v) for k, v in re.findall(r"(MI3D_[A-Z0-9_]+)\s*=\s*(\d+)", hdr)}
    for name, v in L.SHADING.items():
        assert vals["MI3D_SHADING_" + name.upper()] == v
