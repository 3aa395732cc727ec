"""Builds tinsel_b200/libtinsel_b200.so (CUDA kernels + C ABI) in-tree with nvcc for sm_90a (H100).

Numerics-critical flags (see csrc/tb_math.cuh): no FMA contraction on the device (-fmad=false) or
the host (-ffp-contract=off), IEEE division and square root, no flush-to-zero, no fast-math.
"""
import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libtinsel_b200.so")

SOURCES = ["kernels.cu", "api.cu", "snapshot.cpp", "bvh_build.cu"]
HEADERS = ["tb_math.cuh", "tb_scene.cuh", "tb_shade.cuh", "tb_film.cuh", "tb_kernels.cuh", "wf2_common.cuh", "wf2_lanes.cuh", "wf2_rings.cuh", "tb_query.cuh", "tb_probe.cuh"]

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]

NVCC_FLAGS = [
    *ARCH,
    "-O3", "-std=c++17", "-lineinfo",
    "-fmad=false", "-prec-div=true", "-prec-sqrt=true", "-ftz=false",
    "-Xcompiler", "-fPIC,-ffp-contract=off,-O2",
    "--expt-relaxed-constexpr",
]


def _nvcc():
    path = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(path):
        raise RuntimeError("nvcc not found")
    return path


def _host_compiler():
    # the image exports CXX=/opt/gcc/bin/g++, a wrapper that links libstdc++ statically; a second C++
    # runtime inside a python process that already loaded libstdc++.so.6 crashes, so use the system g++
    return "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else (shutil.which("g++") or "g++")


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in SOURCES + HEADERS]
    deps += [os.path.join(ROOT, "include", "tinsel_b200.h"), os.path.join(ROOT, "include", "tb200_detmath.h")]
    deps.append(os.path.abspath(__file__))   # flags and target architecture
    return any(os.path.getmtime(d) > t for d in deps)


def build_native(force=False, verbose=False, extra_flags=(), out=None):
    """out: alternative library name (development variants, selected with TINSEL_B200_LIB)."""
    lib = os.path.join(PKG, out) if out else LIB
    if not force and not out and not needs_build():
        return LIB
    objs = []
    tag = (out or "default").replace(".", "_")
    os.makedirs(os.path.join(PKG, "build", tag), exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(PKG, "build", tag, src + ".o")
        cmd = [_nvcc(), "-ccbin", _host_compiler(), *NVCC_FLAGS, *extra_flags, "-I", os.path.join(ROOT, "include"),
               "-I", CSRC, "-c", os.path.join(CSRC, src), "-o", obj]
        if src.endswith(".cpp"):
            cmd.insert(1, "-x")
            cmd.insert(2, "cu")
        if verbose:
            print(" ".join(cmd), flush=True)
        subprocess.check_call(cmd)
        objs.append(obj)
    cmd = [_nvcc(), "-ccbin", _host_compiler(), *ARCH, "-shared", "-o", lib, *objs,
           "-lcudart"]
    if verbose:
        print(" ".join(cmd), flush=True)
    subprocess.check_call(cmd)
    return lib


if __name__ == "__main__":
    argv = sys.argv[1:]
    out = None
    if "--out" in argv:
        i = argv.index("--out")
        out = argv[i + 1]
        del argv[i:i + 2]
    extra = [a for a in argv if a not in ("-f", "-V")]
    print(build_native(force="-f" in argv, verbose="-V" in argv, extra_flags=extra, out=out))
