"""Writes libai_b200/csrc/wgmma.cuh: the inline-PTX wgmma.mma_async wrappers for every tile width the kernels use."""
import os
out = ["// sm_90a warpgroup MMA wrappers (wgmma.mma_async), one per tile width N used by the kernels (written by tools/gen_wgmma.py).",
       "// Accumulator fragment of m64nN (fp32): thread t of the warpgroup holds rows 16 * (t / 32) + (t % 32) / 4 + {0, 8},",
       "// columns 8 j + 2 (t % 4) + {0, 1}: d[4 j + 2 h + c] = (row + 8 h, column 8 j + 2 (t % 4) + c).",
       "#pragma once", "#include <stdint.h>", "", "namespace lb {", ""]
def regs(n):
    return ", ".join(f"%{i}" for i in range(n))
def outs(n):
    return ", ".join(f'"+f"(d[{i}])' for i in range(n))
for N in (64, 128, 192, 256):
    R = N // 2
    # SS bf16 with transpose immediates
    out.append(f"template <int TA, int TB>")
    out.append(f"__device__ __forceinline__ void wgmma_bf16_ss_n{N}(float (&d)[{R}], uint64_t da, uint64_t db, uint32_t acc) {{")
    out.append("  asm volatile(")
    out.append('      "{\\n.reg .pred p;\\nsetp.ne.b32 p, %' + str(R + 2) + ', 0;\\n"')
    out.append(f'      "wgmma.mma_async.sync.aligned.m64n{N}k16.f32.bf16.bf16 {{{regs(R)}}}, %{R}, %{R+1}, p, 1, 1, %{R+3}, %{R+4};\\n}}\\n"')
    out.append(f'      : {outs(R)}')
    out.append(f'      : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB));')
    out.append("}")
    # SS e4m3 (K-major only)
    out.append(f"__device__ __forceinline__ void wgmma_e4m3_ss_n{N}(float (&d)[{R}], uint64_t da, uint64_t db, uint32_t acc) {{")
    out.append("  asm volatile(")
    out.append('      "{\\n.reg .pred p;\\nsetp.ne.b32 p, %' + str(R + 2) + ', 0;\\n"')
    out.append(f'      "wgmma.mma_async.sync.aligned.m64n{N}k32.f32.e4m3.e4m3 {{{regs(R)}}}, %{R}, %{R+1}, p, 1, 1;\\n}}\\n"')
    out.append(f'      : {outs(R)}')
    out.append(f'      : "l"(da), "l"(db), "r"(acc));')
    out.append("}")
    # RS bf16: A from registers
    out.append(f"template <int TB>")
    out.append(f"__device__ __forceinline__ void wgmma_bf16_rs_n{N}(float (&d)[{R}], const uint32_t (&a)[4], uint64_t db, uint32_t acc) {{")
    out.append("  asm volatile(")
    out.append('      "{\\n.reg .pred p;\\nsetp.ne.b32 p, %' + str(R + 5) + ', 0;\\n"')
    out.append(f'      "wgmma.mma_async.sync.aligned.m64n{N}k16.f32.bf16.bf16 {{{regs(R)}}}, {{%{R}, %{R+1}, %{R+2}, %{R+3}}}, %{R+4}, p, 1, 1, %{R+6};\\n}}\\n"')
    out.append(f'      : {outs(R)}')
    out.append(f'      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc), "n"(TB));')
    out.append("}")
    out.append("")
# dispatchers
out.append("template <int N, int TA, int TB>")
out.append("__device__ __forceinline__ void wgmma_bf16_ss(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t acc) {")
for i, N in enumerate((64, 128, 192, 256)):
    kw = "if" if i == 0 else "else if"
    out.append(f"  {kw} constexpr (N == {N}) wgmma_bf16_ss_n{N}<TA, TB>(d, da, db, acc);")
out.append("}")
out.append("template <int N>")
out.append("__device__ __forceinline__ void wgmma_e4m3_ss(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t acc) {")
for i, N in enumerate((64, 128, 192, 256)):
    kw = "if" if i == 0 else "else if"
    out.append(f"  {kw} constexpr (N == {N}) wgmma_e4m3_ss_n{N}(d, da, db, acc);")
out.append("}")
out.append("template <int N, int TB>")
out.append("__device__ __forceinline__ void wgmma_bf16_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t db, uint32_t acc) {")
for i, N in enumerate((64, 128, 192, 256)):
    kw = "if" if i == 0 else "else if"
    out.append(f"  {kw} constexpr (N == {N}) wgmma_bf16_rs_n{N}<TB>(d, a, db, acc);")
out.append("}")
out.append("")
out.append("}  // namespace lb")
open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "libai_b200", "csrc", "wgmma.cuh"), "w").write("\n".join(out) + "\n")
