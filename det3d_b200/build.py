"""In-tree nvcc build of the det3d_b200 C-ABI library (sm_90a only: H100).

`python -m det3d_b200.build` (or `__graft_entry__.build()`) cross-compiles
every CUDA translation unit under `det3d_b200/csrc/` into
`det3d_b200/lib/libdet3d_b200.so`.  The library is a git-ignored build product
of the source tree; nothing is JIT-compiled at import time.
"""
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libdet3d_b200.so")
STAMP = os.path.join(LIB_DIR, "build.stamp")

NVCC_FLAGS = [
    "-O3",
    "-std=c++17",
    "-gencode",
    "arch=compute_90a,code=sm_90a",
    "-lineinfo",
    "-Xcompiler",
    "-fPIC",
    "--expt-relaxed-constexpr",
]


def _nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found; det3d_b200 needs the CUDA 12.9 toolkit to build")
    return exe


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest():
    h = hashlib.sha256()
    files = sources() + sorted(
        os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))
    )
    files.append(os.path.join(ROOT, "include", "det3d_b200.h"))
    for f in files:
        h.update(f.encode())
        with open(f, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def is_fresh():
    if not (os.path.exists(LIB_PATH) and os.path.exists(STAMP)):
        return False
    with open(STAMP) as fh:
        return fh.read().strip() == _digest()


def build(force=False, verbose=False):
    """Compile the library if sources changed. Returns the .so path."""
    os.makedirs(LIB_DIR, exist_ok=True)
    if not force and is_fresh():
        return LIB_PATH
    objs = []
    obj_dir = os.path.join(LIB_DIR, "obj")
    os.makedirs(obj_dir, exist_ok=True)
    procs = []
    for src in sources():
        obj = os.path.join(obj_dir, os.path.basename(src)[:-3] + ".o")
        cmd = [_nvcc()] + NVCC_FLAGS + ["-I", os.path.join(ROOT, "include"), "-I", CSRC, "-c", src, "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        text = out.decode(errors="replace")
        if p.returncode != 0:
            failed = True
            sys.stderr.write("nvcc failed on %s:\n%s\n" % (src, text))
        elif verbose and text.strip():
            sys.stderr.write(text)
    if failed:
        raise RuntimeError("det3d_b200: CUDA build failed")
    # libcuda is NOT linked: CPU-only hosts must be able to dlopen the library
    # (driver entry points, if needed, are resolved with cudaGetDriverEntryPoint).
    link = [_nvcc(), "-shared", "-Wno-deprecated-gpu-targets", "-o", LIB_PATH] + objs
    subprocess.run(link, check=True)
    with open(STAMP, "w") as fh:
        fh.write(_digest())
    return LIB_PATH


def build_debug():
    """Development library with soft wait time-outs (-DD3B_SOFT_TIMEOUT): lib/libdet3d_b200_dbg.so, selected at run
    time with D3B_LIB=<path>.  Never loaded by default."""
    os.makedirs(os.path.join(LIB_DIR, "obj_dbg"), exist_ok=True)
    out = os.path.join(LIB_DIR, "libdet3d_b200_dbg.so")
    objs, procs = [], []
    for src in sources():
        obj = os.path.join(LIB_DIR, "obj_dbg", os.path.basename(src)[:-3] + ".o")
        cmd = [_nvcc()] + NVCC_FLAGS + ["-DD3B_SOFT_TIMEOUT", "-I", os.path.join(ROOT, "include"), "-I", CSRC, "-c", src, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(obj)
    for src, p in procs:
        text, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError("nvcc failed on %s:\n%s" % (src, text.decode(errors="replace")))
    subprocess.run([_nvcc(), "-shared", "-Wno-deprecated-gpu-targets", "-o", out] + objs, check=True)
    return out


if __name__ == "__main__":
    if "--debug" in sys.argv:
        print(build_debug())
    else:
        print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
