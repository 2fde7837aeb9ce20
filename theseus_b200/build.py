"""Build libthb200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

    python -m theseus_b200.build [--force]

The .so is git-ignored but travels to the GPU box with the repo snapshot.  nvcc cross-compiles without
a GPU.  No JIT, no torch.utils.cpp_extension: the library has no torch dependency (plain C ABI).
"""
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIBNAME = "libthb200.so"
SOURCES = ["thb_costs.cu", "thb_gram.cu", "thb_chol_dense.cu", "thb_sparse.cu", "thb_sparse_lane.cu", "thb_symbolic.cu", "thb_lie_ops.cu", "thb_front.cu", "thb_gram_dense.cu"]
HEADERS = ["thb_common.cuh", "thb_lie.cuh", os.path.join("..", "..", "include", "thb200.h")]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-DTHB_ARCH=90",
]


def _nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; libthb200 cannot be built")


def _digest():
    h = hashlib.sha256()
    for f in SOURCES + HEADERS:
        p = os.path.join(CSRC, f)
        if os.path.exists(p):
            with open(p, "rb") as fh:
                h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def lib_path():
    return os.path.join(LIBDIR, LIBNAME)


def build(force=False, verbose=True):
    os.makedirs(LIBDIR, exist_ok=True)
    stamp = os.path.join(LIBDIR, "build.stamp")
    dig = _digest()
    if not force and os.path.exists(lib_path()) and os.path.exists(stamp) and open(stamp).read().strip() == dig:
        return lib_path()
    nvcc = _nvcc()
    objs = []
    procs = []
    for src in SOURCES:
        sp = os.path.join(CSRC, src)
        if not os.path.exists(sp):
            continue
        obj = os.path.join(LIBDIR, src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [nvcc] + NVCC_FLAGS + ["-c", sp, "-o", obj]
        if verbose:
            print(" ".join(cmd), flush=True)
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{out}")
        if verbose and out.strip():
            print(out)
    cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", lib_path()] + objs + ["-lcudart"]
    if verbose:
        print(" ".join(cmd), flush=True)
    subprocess.check_call(cmd)
    with open(stamp, "w") as fh:
        fh.write(dig)
    return lib_path()


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
