"""Build libpsb200.so (hand-written CUDA for sm_90a, H100) in-tree with nvcc. No torch dependency."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libpsb200.so")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def headers():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    hs.append(os.path.join(os.path.dirname(HERE), "include", "psb200.h"))
    return hs


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(p) > t for p in sources() + headers())


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    os.makedirs(LIBDIR, exist_ok=True)
    cmd = ["nvcc", *ARCH, "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-shared"]
    if verbose:
        cmd += ["-Xptxas", "-v"]
    cmd += ["-o", LIB, *sources()]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc failed building libpsb200.so")
    if verbose:
        sys.stderr.write(r.stderr)
    return LIB


TORCH_SRC = os.path.join(HERE, "csrc_torch", "rasterize_points.cpp")
TORCH_LIB = os.path.join(LIBDIR, "libcuda_rasterizer.so")


def build_torch_shim(force=False):
    """libcuda_rasterizer.so: the reference's B1/B2 C++ symbols on top of libpsb200.so (host-only C++/LibTorch)."""
    build()
    if not force and os.path.exists(TORCH_LIB) and os.path.getmtime(TORCH_LIB) >= max(os.path.getmtime(TORCH_SRC), os.path.getmtime(LIB)):
        return TORCH_LIB
    import torch
    ti = os.path.dirname(torch.__file__)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    cmd = [cxx, "-O2", "-std=c++17", "-fPIC", "-shared", f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}",
           f"-I{ti}/include", f"-I{ti}/include/torch/csrc/api/include", "-I/usr/local/cuda/include", TORCH_SRC, "-o", TORCH_LIB,
           f"-L{LIBDIR}", "-lpsb200", f"-L{ti}/lib", "-ltorch", "-ltorch_cpu", "-lc10", "-lc10_cuda", "-ltorch_cuda",
           "-Wl,-rpath,$ORIGIN", f"-Wl,-rpath,{ti}/lib"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("g++ failed building libcuda_rasterizer.so")
    return TORCH_LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
    if "--torch" in sys.argv:
        print(build_torch_shim(force="--force" in sys.argv))
