"""Kernels that issue wgmma must keep it asynchronous: ptxas reports C7510 when it had to make every wgmma wait for
the previous one (for example because of a function call in the kernel), and the build treats that as an error."""
import os
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor

import pytest

from libai_b200.ops import build as ops_build

C7510_LOG = (
    "ptxas info    : (C7510) Potential Performance Loss: wgmma.mma_async instructions are serialized due to wgmma "
    "pipeline crossing function boundary at a function call in the function '_ZN2lb17spin_timeout_trapEPKjjii'\n"
    "ptxas info    : Used 168 registers, used 2 barriers, 32 bytes cumulative stack size\n"
)


def test_serialized_wgmma_names_the_function_and_the_reason():
    lines = ops_build.serialized_wgmma(C7510_LOG + C7510_LOG)
    assert len(lines) == 1
    assert "function call" in lines[0]
    if shutil.which("c++filt"):
        assert "lb::spin_timeout_trap(" in lines[0]
    assert ops_build.serialized_wgmma("ptxas info    : Used 168 registers, used 2 barriers\n") == []


@pytest.mark.skipif(not os.path.exists(ops_build.NVCC), reason="needs nvcc")
def test_wgmma_kernels_compile_without_serialization(tmp_path):
    def compile_log(src):
        res = subprocess.run([ops_build.NVCC, *ops_build.NVCC_FLAGS, "-I", ops_build.CSRC, "-c",
                              os.path.join(ops_build.CSRC, src), "-o", str(tmp_path / (src + ".o"))],
                             stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert res.returncode == 0, res.stdout
        return res.stdout

    sources = ["gemm_sm90.cu", "attention_sm90.cu"]
    with ThreadPoolExecutor(len(sources)) as ex:
        logs = dict(zip(sources, ex.map(compile_log, sources)))
    for src, log in logs.items():
        assert "Compiling entry function" in log, src   # -Xptxas -v is among the build flags
        assert ops_build.serialized_wgmma(log) == [], (src, ops_build.serialized_wgmma(log))
