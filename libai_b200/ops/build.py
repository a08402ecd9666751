"""In-tree build of the native extension ``libai_b200/_C.so`` (and the C++ dataset helpers).

    python -m libai_b200.ops.build [--force] [--verbose]

CUDA sources are compiled for sm_90a only (``-gencode arch=compute_90a,code=sm_90a -lineinfo``);
nvcc cross-compiles without a GPU.  Objects are cached under ``libai_b200/csrc/build`` keyed by
source mtime.  ``--sass`` additionally dumps ``cuobjdump -sass`` listings into ``profiles/sass``.
"""
from __future__ import annotations

import argparse
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "csrc")
BUILD = os.path.join(CSRC, "build")
SO_PATH = os.path.join(ROOT, "_C.so")
CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")
NVCC = os.path.join(CUDA_HOME, "bin", "nvcc")

CU_SOURCES = ["gemm_sm90.cu", "norm.cu", "elementwise.cu", "attention_sm90.cu", "comm_kernels.cu",
              "decode_attention_sm90.cu", "window_attention_sm90.cu"]
CPP_SOURCES = ["bindings.cpp", "symm_mem.cpp"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "--use_fast_math", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v",
]


def _run(cmd, verbose):
    if verbose:
        print(" ".join(cmd), flush=True)
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"command failed ({res.returncode}): {' '.join(cmd)}\n{res.stdout}")
    return res.stdout


def serialized_wgmma(log: str) -> list:
    """ptxas warning C7510 means that it made every wgmma of a kernel wait for the previous one to complete (for
    example because the kernel contains a function call), which turns the asynchronous tensor-core pipeline into a
    serial one.  Returns the distinct such warnings of a ptxas log, demangled; each names the function it blames."""
    lines = list(dict.fromkeys(ln.split("(C7510)", 1)[-1].strip() for ln in log.splitlines() if "C7510" in ln))
    if lines:
        try:
            lines = subprocess.run(["c++filt"], input="\n".join(lines), stdout=subprocess.PIPE, text=True,
                                   check=True).stdout.splitlines()
        except (OSError, subprocess.CalledProcessError):
            pass
    return lines


def _stale(src, obj, deps=()):
    if not os.path.exists(obj):
        return True
    t = os.path.getmtime(obj)
    return any(os.path.getmtime(p) > t for p in (src,) + tuple(deps) if os.path.exists(p))


def build(force: bool = False, verbose: bool = False, sass: bool = False) -> str:
    import torch
    from torch.utils import cpp_extension

    os.makedirs(BUILD, exist_ok=True)
    headers = tuple(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h")))
    cu = [s for s in CU_SOURCES if os.path.exists(os.path.join(CSRC, s))]
    cpp = [s for s in CPP_SOURCES if os.path.exists(os.path.join(CSRC, s))]
    jobs, objs, logs = [], [], {}
    for s in cu:
        src, obj = os.path.join(CSRC, s), os.path.join(BUILD, s + ".o")
        objs.append(obj)
        if force or _stale(src, obj, headers):
            jobs.append((s, [NVCC, *NVCC_FLAGS, "-I", CSRC, "-c", src, "-o", obj]))
    inc = []
    for p in cpp_extension.include_paths(device_type="cuda"):
        inc += ["-isystem", p]
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    for s in cpp:
        src, obj = os.path.join(CSRC, s), os.path.join(BUILD, s + ".o")
        objs.append(obj)
        if force or _stale(src, obj, headers):
            jobs.append((s, ["g++", "-O2", "-std=c++17", "-fPIC", f"-D_GLIBCXX_USE_CXX11_ABI={abi}",
                             "-DTORCH_EXTENSION_NAME=_C", *inc, "-I", os.path.join(CUDA_HOME, "include"),
                             "-I", CSRC, "-c", src, "-o", obj]))
    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for (name, _), out in zip(jobs, ex.map(lambda j: _run(j[1], verbose), jobs)):
                logs[name] = out
        os.makedirs(os.path.join(os.path.dirname(ROOT), "profiles"), exist_ok=True)
        with open(os.path.join(BUILD, "ptxas.log"), "w") as f:
            for name, out in logs.items():
                f.write(f"==== {name}\n{out}\n")
        serialized = {name: serialized_wgmma(out) for name, out in logs.items()}
        serialized = {name: lines for name, lines in serialized.items() if lines}
        if serialized:
            for name in serialized:   # the next build must compile them again, not link the serialized objects
                os.remove(os.path.join(BUILD, name + ".o"))
            raise RuntimeError("ptxas serialized wgmma (C7510); kernels that issue wgmma must not contain a function "
                               "call:\n" + "\n".join(f"{name}: {ln}" for name, lines in serialized.items()
                                                    for ln in lines))
    if jobs or force or not os.path.exists(SO_PATH):
        tlib = os.path.join(os.path.dirname(torch.__file__), "lib")
        _run(["g++", "-shared", "-o", SO_PATH, *objs, f"-L{tlib}", "-lc10", "-ltorch_cpu", "-ltorch", "-lc10_cuda",
              "-ltorch_cuda", f"-L{os.path.join(CUDA_HOME, 'lib64')}", "-lcudart",
              f"-Wl,-rpath,{tlib}", f"-Wl,-rpath,{os.path.join(CUDA_HOME, 'lib64')}"], verbose)
    if sass:
        dump_sass()
    return SO_PATH


def dump_sass():
    """Write SASS listings + a mnemonic summary (HGMMA / UTMALDG ...) to profiles/sass."""
    out_dir = os.path.join(os.path.dirname(ROOT), "profiles", "sass")
    os.makedirs(out_dir, exist_ok=True)
    summary = []
    for s in CU_SOURCES:
        obj = os.path.join(BUILD, s + ".o")
        if not os.path.exists(obj):
            continue
        text = subprocess.run([os.path.join(CUDA_HOME, "bin", "cuobjdump"), "-sass", obj], stdout=subprocess.PIPE,
                              text=True).stdout
        counts = {}
        # HGMMA / QGMMA = wgmma (bf16 / fp8); UTMALDG / UTMASTG / UTMAREDG / UBLKCP = TMA tensor + bulk copies and
        # reductions; LDGMC = multimem.ld_reduce (NVLS in-switch reduction; multimem.st is a STG.*.STRONG.SYS on a
        # multicast address); USETMAXREG = setmaxnreg
        for key in ("HGMMA", "QGMMA", "UTMALDG", "UTMASTG", "UTMAREDG", "UBLKCP", "SYNCS", "LDGMC", "USETMAXREG", "RED.E",
                    "REDG", "LDG.E", "STG.E"):
            counts[key] = text.count(key)
        summary.append((s, counts))
        keep = [ln for ln in text.splitlines() if "Function :" in ln or any(k in ln for k in ("GMMA", "UTMA", "UBLKCP", "LDGMC", "USETMAXREG"))]
        with open(os.path.join(out_dir, s + ".sass.txt"), "w") as f:
            f.write("\n".join(keep) + "\n")
    with open(os.path.join(out_dir, "SUMMARY.md"), "w") as f:
        f.write("# SASS mnemonic counts per translation unit (cuobjdump -sass, sm_90a)\n\n")
        for s, c in summary:
            f.write(f"* `{s}`: " + ", ".join(f"{k}={v}" for k, v in c.items() if v) + "\n")
    return summary


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--verbose", action="store_true")
    ap.add_argument("--sass", action="store_true")
    a = ap.parse_args()
    print(build(a.force, a.verbose, a.sass))
