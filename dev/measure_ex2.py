"""Measures the relative error of ex2.approx.ftz.f32 (fast_exp2 in libai_b200/csrc/common.cuh) over every fp32 x in
[-126, 0], the exponents the attention kernels give it, against the fp64 2^x computed on the device.  The result backs
EX2_APPROX in tests/attention_ref.py.  Usage: python dev/measure_ex2.py (needs a GPU; compiles a small extension into
a temporary directory)."""
import math
import os
import tempfile

import torch
from torch.utils.cpp_extension import load_inline

CUDA_SRC = r"""
#include <torch/extension.h>
#include <cstdint>

__global__ void ex2_err_kernel(uint32_t first, uint32_t last, unsigned long long* worst) {
  unsigned long long best = 0;   // max relative error, as the bits of a non-negative double (monotone as integers)
  for (uint64_t u = first + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; u <= last;
       u += (uint64_t)gridDim.x * blockDim.x) {
    const float x = __uint_as_float((uint32_t)u);
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    const double ref = exp2((double)x);
    const double rel = fabs((double)y / ref - 1.0);
    const unsigned long long bits = (unsigned long long)__double_as_longlong(rel);
    best = bits > best ? bits : best;
  }
  atomicMax(worst, best);
}

torch::Tensor ex2_max_rel_err(int64_t first, int64_t last) {
  auto worst = torch::zeros({1}, torch::dtype(torch::kInt64).device(torch::kCUDA));
  ex2_err_kernel<<<4096, 256>>>((uint32_t)first, (uint32_t)last, (unsigned long long*)worst.data_ptr<int64_t>());
  return worst;
}
"""
CPP_SRC = "torch::Tensor ex2_max_rel_err(int64_t first, int64_t last);"


def main():
    with tempfile.TemporaryDirectory() as build_dir:
        mod = load_inline("measure_ex2", cpp_sources=CPP_SRC, cuda_sources=CUDA_SRC, functions=["ex2_max_rel_err"],
                          extra_cuda_cflags=["-gencode", "arch=compute_90a,code=sm_90a"], build_directory=build_dir,
                          verbose=False)
        import struct

        # negative fp32 values from -0 (0x80000000) down to -126 (0xC2FC0000): bit patterns increase as x decreases;
        # results below 2^-126 are flushed, so x < -126 is outside the range where a relative error means anything
        first, last = 0x80000000, struct.unpack("<I", struct.pack("<f", -126.0))[0]
        bits = int(mod.ex2_max_rel_err(first, last).item())
        torch.cuda.synchronize()
    err = struct.unpack("<d", struct.pack("<q", bits))[0]
    name = torch.cuda.get_device_name()
    print(f"{name}: max |ex2.approx(x) / 2^x - 1| over fp32 x in [-126, 0] = {err:.4e} = 2^{math.log2(err):.2f}")


if __name__ == "__main__":
    os.environ.setdefault("TORCH_EXTENSIONS_DIR", tempfile.gettempdir())
    main()
