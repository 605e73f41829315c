"""Builds rapid_b200/librapid_b200.so in-tree with nvcc for sm_90a, the H100 (no JIT cache, no torch extension:
the library is a plain C-ABI shared object)."""
import os
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "librapid_b200.so")
SOURCES = ["api.cu", "view.cu", "overlay.cu", "cd_core.cu", "cd_census.cu", "cd_prepare.cu", "cd_bucketed.cu", "fast_paxos.cu", "classic_paxos.cu", "wire.cu", "wire_encode.cu", "fd.cu"]
HEADERS = ["common.cuh", "cd_internal.cuh", "nccl_api.cuh", "scan.cuh", "radix.cuh", "wire_internal.cuh", os.path.join("..", "..", "include", "rapid_b200.h")]
ARCH = "sm_90a"
GENCODE = ["-gencode", "arch=compute_90a,code=" + ARCH]
NVCC_FLAGS = GENCODE + ["-lineinfo", "-O3", "-std=c++17",
                         "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden"]


def _nvcc():
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found: librapid_b200.so cannot be built (there is no CPU fallback)")


def _stale(out, deps):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    return any(os.path.getmtime(d) > t for d in deps)


def build_native(force=False, verbose=False):
    nvcc = _nvcc()
    objdir = os.path.join(HERE, "build", ARCH)      # objects of another architecture are never linked in
    os.makedirs(objdir, exist_ok=True)
    hdrs = [os.path.join(CSRC, h) for h in HEADERS]

    def compile_one(src):
        s = os.path.join(CSRC, src)
        o = os.path.join(objdir, src.replace(".cu", ".o"))
        if force or _stale(o, [s] + hdrs):
            cmd = [nvcc] + NVCC_FLAGS + ["-c", s, "-o", o]
            if verbose:
                print(" ".join(cmd))
            subprocess.check_call(cmd)
        return o

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    if force or _stale(LIB, objs):
        cmd = [nvcc, "-shared", "-o", LIB] + objs + GENCODE + ["-ldl"]
        if verbose:
            print(" ".join(cmd))
        subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build_native(verbose=True))
