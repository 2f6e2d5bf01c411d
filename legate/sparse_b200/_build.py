"""In-tree nvcc build of libb200sparse.so (sm_90a only).

The reference builds through scikit-build + rapids-cmake + a CPM fetch of legate.core
(install.py, CMakeLists.txt); here the whole native side is a handful of .cu files compiled
straight into one shared library that sits next to this file, so it travels with the tree.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_NAME = "libb200sparse.so"
LIB_PATH = os.path.join(HERE, LIB_NAME)
SOURCES = ["capi.cu", "spmv.cu", "spmv_f32.cu", "spmv_f64.cu", "spmm.cu", "spmm_tma.cu", "vecops.cu", "spgemm.cu", "peer.cu", "probe.cu", "comm.cu", "convert.cu", "elementwise.cu", "sddmm.cu", "tropical.cu", "reduce.cu", "index.cu", "construct.cu", "csc.cu", "dia.cu", "random.cu"]
HEADERS = ["common.cuh", "scan.cuh", "spmv_common.cuh", "spmv_kernels.cuh", os.path.join("..", "..", "..", "include", "b200sparse.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
]


def _nvcc() -> str:
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found; libb200sparse.so cannot be built")
    return nvcc


def _host_compiler_args():
    # the image exports CXX=/opt/gcc/bin/g++ (a wrapper); the system g++ is the one nvcc supports
    for cand in ("/usr/bin/g++",):
        if os.path.exists(cand):
            return ["-ccbin", cand]
    return []


def needs_build() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, s) for s in SOURCES] + [os.path.normpath(os.path.join(CSRC, h)) for h in HEADERS]
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False, ptxas_info: bool = False) -> str:
    """Compile every .cu under csrc/ for sm_90a and link libb200sparse.so in-tree."""
    if not force and not needs_build():
        return LIB_PATH
    # one builder at a time (torchrun imports the package on every rank at once): the others wait on the lock and
    # then find the library up to date; the link goes to a temporary name and is renamed into place atomically
    import fcntl

    lock = open(os.path.join(HERE, ".build.lock"), "w")
    fcntl.flock(lock, fcntl.LOCK_EX)
    try:
        if not force and not needs_build():
            return LIB_PATH
        return _build_locked(verbose, ptxas_info)
    finally:
        fcntl.flock(lock, fcntl.LOCK_UN)
        lock.close()


def _build_locked(verbose: bool, ptxas_info: bool) -> str:
    nvcc = _nvcc()
    objs = []
    build_dir = os.path.join(HERE, "build")
    os.makedirs(build_dir, exist_ok=True)
    procs = []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(build_dir, s.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [nvcc, *NVCC_FLAGS, *_host_compiler_args(), "-c", src, "-o", obj]
        if ptxas_info:
            cmd += ["-Xptxas", "-v"]
        if verbose:
            print(" ".join(cmd), file=sys.stderr)
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {s}:\n{out}")
        if (verbose or ptxas_info) and out:
            print(out, file=sys.stderr)
    tmp = LIB_PATH + f".tmp{os.getpid()}"
    cmd = [nvcc, "-shared", *_host_compiler_args(), "-o", tmp, *objs, "-lcudart", "-ldl"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    os.replace(tmp, LIB_PATH)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True, ptxas_info="--ptxas" in sys.argv))
