"""Builds libcchess_b200.so (the C-ABI engine library) in-tree with nvcc for sm_90a (H100)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = [os.path.join(HERE, "csrc", "cz_engine.cu"), os.path.join(HERE, "csrc", "cz_net.cu"), os.path.join(HERE, "csrc", "cz_tower.cu"),
       os.path.join(HERE, "csrc", "cz_host.cu")]
DEPS = SRC + [os.path.join(HERE, "csrc", "cz_rules.cuh"), os.path.join(HERE, "csrc", "cz_wgmma.cuh"), os.path.join(HERE, "csrc", "cz_exp.h"),
        os.path.join(os.path.dirname(HERE), "include", "cchess_b200.h")]
LIB = os.path.join(HERE, "libcchess_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "--fmad=false",
         "-Xcompiler", "-fPIC", "-Xcompiler", "-ffp-contract=off", "-shared", "-Xptxas", "-v"]


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(p) > t for p in DEPS)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    tmp = "%s.tmp.%d" % (LIB, os.getpid())          # build beside the target, then rename: never a half-written library
    cmd = [NVCC] + FLAGS + ["-o", tmp] + SRC
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or r.returncode:
        sys.stderr.write(r.stdout + r.stderr)
    if r.returncode:
        if os.path.exists(tmp):
            os.remove(tmp)
        raise RuntimeError("nvcc failed: " + " ".join(cmd))
    os.replace(tmp, LIB)
    return LIB


if __name__ == "__main__":
    build(force=True, verbose=True)
    print(LIB)
