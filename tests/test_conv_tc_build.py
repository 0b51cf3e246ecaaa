"""ptxas -v for sm_90a: every instantiation of the wgmma convolution keeps its roles in registers (setmaxnreg budgets) and keeps
its wgmma groups asynchronous."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


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
