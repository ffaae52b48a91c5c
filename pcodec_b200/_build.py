"""Builds pcodec_b200/libcpcodec.so (CUDA kernels + C-ABI) in-tree with nvcc for sm_90a (H100)."""
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
INCLUDE = os.path.join(HERE, "..", "include")
LIB = os.path.join(HERE, "libcpcodec.so")
SOURCES = ["host_api.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared", "--fmad=false", "-cudart", "static",
]


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libcpcodec.so is a CUDA library and cannot be built without it")


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    return any(os.path.getmtime(d) > t for d in deps)


def build_variant(name, defines, verbose=False):
    """Experiment builds: pcodec_b200/libcpcodec_<name>.so with extra -D flags (select with PCOB200_LIB)."""
    out = os.path.join(HERE, f"libcpcodec_{name}.so")
    ccbin = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
    cmd = [_nvcc(), "-ccbin", ccbin] + NVCC_FLAGS + [f"-D{d}" for d in defines] + (["-Xptxas", "-v"] if verbose else []) + ["-o", out] + SOURCES
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    if verbose:
        print(res.stderr)
    return out


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    # the image exports CXX=/opt/gcc/bin/g++ (links libstdc++ statically); use the system g++ as nvcc's host compiler
    ccbin = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
    tmp = LIB + f".tmp{os.getpid()}"  # linked beside the target and renamed into place: a reader never sees a half-written library
    cmd = [_nvcc(), "-ccbin", ccbin] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", tmp] + SOURCES
    res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    if res.returncode != 0:
        if os.path.exists(tmp):
            os.remove(tmp)
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    os.replace(tmp, LIB)
    if verbose:
        print(res.stderr)
    return LIB
