"""ptxas -v for sm_90a: every instantiation of the wgmma convolution keeps its roles in registers (setmaxnreg budgets) and keeps
its wgmma groups asynchronous.  The ctypes layouts of the convolution's C ABI records follow the header."""
import ctypes
import os
import re
import subprocess

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


@pytest.mark.parametrize("c_name,py_name,size", [("mn_conv_params", "ConvParams", 296), ("mn_conv_plan", "ConvPlan", 60)])
def test_conv_structs_match_header(c_name, py_name, size):
    from marconet_b200 import _lib
    header = open(os.path.join(ROOT, "include", "marconet_b200.h")).read()
    cls = getattr(_lib, py_name)
    assert _fields(header, c_name) == [f[0] for f in cls._fields_]
    assert ctypes.sizeof(cls) == size        # x86-64 / aarch64 natural alignment, as the library is compiled


def test_conv_tc2_kernels_build_without_spills(tmp_path):
    from marconet_b200 import build
    src = os.path.join(ROOT, "marconet_b200", "csrc", "conv_tc2.cu")
    r = subprocess.run([build.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-DMN_BUILD", "-Xptxas", "-v",
                        "-cubin", src, "-o", str(tmp_path / "conv_tc2.cubin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    props = re.findall(r"Function properties for (\S*conv_tc2_kernel\S*)\n([^\n]*)", r.stderr)
    # GroupNorm transform on / off x three precision modes (x the work-item widths)
    assert len(props) >= 6, r.stderr[-2000:]
    for kernel, line in props:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, f"{kernel}: {line}"
    # C7513: ptxas had to serialize the wgmma instructions (a wait after every MMA)
    assert "C7513" not in r.stderr, r.stderr[-2000:]
