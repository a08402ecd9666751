"""Measures the relative error of sqrt.approx.ftz.f32 (what `sqrtf` compiles to under --use_fast_math: MUFU.SQRT in the
fused Adam update) over every positive normal fp32 x, against the fp64 square root computed on the device.  The result
backs SQRT_APPROX in tests/train_ref.py.  Usage: python dev/measure_sqrt_approx.py (needs a GPU; compiles a small
extension into a temporary directory)."""
import math
import os
import struct
import tempfile

import torch
from torch.utils.cpp_extension import load_inline

CUDA_SRC = r"""
#include <torch/extension.h>
#include <cstdint>

__global__ void sqrt_err_kernel(uint32_t first, uint32_t last, unsigned long long* worst) {
  unsigned long long best = 0;   // max relative error, as the bits of a non-negative double (monotone as integers)
  for (uint64_t u = first + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; u <= last;
       u += (uint64_t)gridDim.x * blockDim.x) {
    const float x = __uint_as_float((uint32_t)u);
    float y;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    const double rel = fabs((double)y / sqrt((double)x) - 1.0);
    const unsigned long long bits = (unsigned long long)__double_as_longlong(rel);
    best = bits > best ? bits : best;
  }
  atomicMax(worst, best);
}

torch::Tensor sqrt_max_rel_err(int64_t first, int64_t last) {
  auto worst = torch::zeros({1}, torch::dtype(torch::kInt64).device(torch::kCUDA));
  sqrt_err_kernel<<<4096, 256>>>((uint32_t)first, (uint32_t)last, (unsigned long long*)worst.data_ptr<int64_t>());
  return worst;
}
"""
CPP_SRC = "torch::Tensor sqrt_max_rel_err(int64_t first, int64_t last);"


def main():
    with tempfile.TemporaryDirectory() as build_dir:
        mod = load_inline("measure_sqrt_approx", cpp_sources=CPP_SRC, cuda_sources=CUDA_SRC,
                          functions=["sqrt_max_rel_err"], extra_cuda_cflags=["-gencode", "arch=compute_90a,code=sm_90a"],
                          build_directory=build_dir, verbose=False)
        # every positive normal fp32: 2^-126 (0x00800000) up to the largest finite value (0x7F7FFFFF)
        bits = int(mod.sqrt_max_rel_err(0x00800000, 0x7F7FFFFF).item())
        torch.cuda.synchronize()
    from measure_fp8_acc import card     # (this directory)

    err = struct.unpack("<d", struct.pack("<q", bits))[0]
    print(f"{card()}: max |sqrt.approx(x) / sqrt(x) - 1| over every positive normal fp32 x = {err:.4e} = "
          f"2^{math.log2(err):.2f}")


if __name__ == "__main__":
    os.environ.setdefault("TORCH_EXTENSIONS_DIR", tempfile.gettempdir())
    main()
