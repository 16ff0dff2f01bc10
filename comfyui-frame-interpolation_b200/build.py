"""Compile libvfi_b200.so in-tree with nvcc for sm_90a (no other architecture, no JIT cache)."""
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libvfi_b200.so")
SOURCES = ["tapconv.cu", "elementwise.cu", "ops.cu", "ops_extra.cu", "rife46.cu", "streamconv.cu", "film_elem.cu", "film.cu", "sepconv_elem.cu", "sepconv.cu", "gmops.cu", "flavr_elem.cu", "flavr.cu", "ifrnet_elem.cu", "ifrnet.cu", "cain_elem.cu", "cain.cu", "ifunet_elem.cu", "ifunet.cu"]
HEADERS = ["ptx.cuh", "vfi_internal.h", "hoststage.h", os.path.join("..", "..", "include", "vfi_b200.h")]


def _nvcc():
    return shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS]
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
           "--threads", "4", "-Xcompiler", "-fPIC,-mavx2", "-shared", "-o", LIB] + [os.path.join(CSRC, s) for s in SOURCES]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    if verbose:
        print(r.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose=True))
