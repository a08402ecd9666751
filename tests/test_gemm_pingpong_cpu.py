"""The ping-pong GEMM kernel keeps its accumulators in registers: ptxas reports no spills for any of its instances, and
(with test_build_cpu) no wgmma serialization."""
import os
import re
import subprocess

import pytest

from libai_b200.ops import build as ops_build


def pingpong_reports(log):
    """{mangled kernel name: the ptxas lines reported for it} for every gemm_pingpong_kernel instance of a log."""
    reports, name = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            name = m.group(1) if "gemm_pingpong_kernel" in m.group(1) else None
            if name:
                reports[name] = []
        elif name and "ptxas info" in line and "Function properties" in line:
            continue
        elif name:
            reports[name].append(line)
    return reports


def test_pingpong_reports_parse():
    log = ("ptxas info    : Compiling entry function '_ZN2lb20gemm_pingpong_kernelILb0EEEv' for 'sm_90a'\n"
           "ptxas info    : Function properties for _ZN2lb20gemm_pingpong_kernelILb0EEEv\n"
           "    0 bytes stack frame, 8 bytes spill stores, 8 bytes spill loads\n"
           "ptxas info    : Used 168 registers, used 16 barriers\n"
           "ptxas info    : Compiling entry function '_ZN2lb11gemm_kernelILi64ELb0ELb0ELi0ELb0EEEv' for 'sm_90a'\n"
           "    0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads\n")
    reports = pingpong_reports(log)
    assert list(reports) == ["_ZN2lb20gemm_pingpong_kernelILb0EEEv"]
    assert any("8 bytes spill stores" in ln for ln in reports["_ZN2lb20gemm_pingpong_kernelILb0EEEv"])


@pytest.mark.skipif(not os.path.exists(ops_build.NVCC), reason="needs nvcc")
def test_pingpong_kernels_do_not_spill(tmp_path):
    res = subprocess.run([ops_build.NVCC, *ops_build.NVCC_FLAGS, "-I", ops_build.CSRC, "-c",
                          os.path.join(ops_build.CSRC, "gemm_sm90.cu"), "-o", str(tmp_path / "gemm_sm90.o")],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    reports = pingpong_reports(res.stdout)
    assert len(reports) == 2, list(reports)      # NT and NN
    for name, lines in reports.items():
        spills = [ln for ln in lines if "spill" in ln]
        assert spills, (name, lines)
        for ln in spills:
            assert re.search(r"\b0 bytes spill stores, 0 bytes spill loads", ln), (name, ln)
        assert not any("stack frame" in ln and not ln.strip().startswith("0 bytes") for ln in lines), (name, lines)
