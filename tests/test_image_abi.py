"""The descriptor records of the batched image kernels (mn_lq_crop, mn_sr_piece): the ctypes layouts follow the header."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _fields(header, name):
    body = re.search(r"typedef struct \{([^{}]*)\}\s*" + name + ";", header).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = []
    for decl in body.split(";"):
        parts = [p.strip() for p in decl.strip().split(",") if p.strip()]
        names += [re.findall(r"[A-Za-z_0-9]+$", p)[0] for p in parts]
    return names


@pytest.mark.parametrize("c_name,py_name,size", [("mn_lq_crop", "LqCrop", 56), ("mn_sr_piece", "SrPiece", 32)])
def test_descriptor_structs_match_header_field_order(c_name, py_name, size):
    from marconet_b200 import _lib
    header = open(os.path.join(ROOT, "include", "marconet_b200.h")).read()
    cls = getattr(_lib, py_name)
    assert _fields(header, c_name) == [f[0] for f in cls._fields_]
    assert ctypes.sizeof(cls) == size        # x86-64 / aarch64 natural alignment, as nvcc lays the struct out on the device


def test_batched_image_kernels_build_without_spills(tmp_path):
    """ptxas -v for sm_90a: the crop and stitch kernels keep everything in registers."""
    import subprocess
    from marconet_b200 import build
    src = os.path.join(ROOT, "marconet_b200", "csrc", "image_ops.cu")
    r = subprocess.run([build.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-DMN_BUILD", "-Xptxas", "-v",
                        "-cubin", src, "-o", str(tmp_path / "image_ops.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    for kernel in ("preprocess_lq_crops_kernel", "postprocess_sr_pieces_kernel"):
        props = re.search(kernel + r"[^\n]*\n[^\n]*Function properties for [^\n]*" + kernel + r"[^\n]*\n([^\n]*)", r.stderr)
        assert props, f"no ptxas report for {kernel}"
        assert "0 bytes spill stores, 0 bytes spill loads" in props.group(1), props.group(1)
