"""In-tree build of the CUDA library: nvcc -> jssenv_b200/libjss_b200.so (sm_90a only)."""
import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
SRCS = [os.path.join(PKG, "csrc", "jss_api.cu"), os.path.join(PKG, "csrc", "jss_host.cpp")]
OUT = os.path.join(PKG, "libjss_b200.so")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-shared", "-Xcompiler", "-fPIC"]


def find_nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def needs_build():
    if not os.path.exists(OUT):
        return True
    deps = [os.path.join(PKG, "csrc", f) for f in os.listdir(os.path.join(PKG, "csrc"))]
    deps.append(os.path.join(PKG, "..", "include", "jss_b200.h"))
    return os.path.getmtime(OUT) < max(os.path.getmtime(d) for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return OUT
    cmd = [find_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", OUT] + SRCS
    subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
