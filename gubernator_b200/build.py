"""Builds libgubernator_b200.so in-tree with nvcc for sm_90a (H100) (no torch involved: the library is plain CUDA runtime)."""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libgubernator_b200.so")
SOURCES = [os.path.join(CSRC, f) for f in ("gub_api.cu", "host_util.cpp", "host_v1.cpp")]
DEPS = SOURCES + [os.path.join(CSRC, f) for f in ("gub_kernels.cuh", "gub_batch.cuh", "gub_global.cuh", "gub_p2p.cuh", "gub_store.cuh", "gub_proto.cuh", "bucket_math.cuh")] + \
    [os.path.join(ROOT, "include", f) for f in ("gubernator_b200.h", "gubernator_b200_host.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--fmad=false",              # Go on amd64 never fuses multiply-add; the float64 leaky-bucket math must be bit-exact
    "-Xcompiler", "-fPIC,-O2,-Wall,-ffp-contract=off",
    "-shared", "-cudart", "static", "-lpthread",
]


def nvcc_path():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in DEPS)


def build(force=False, verbose=False, out=None, defines=()):
    """out / defines: build an experimental variant next to the product library (e.g. out="libgub_onepass.so",
    defines=("GUB_GROUP_ONEPASS=1",)); load it with GUB_LIB=<path> (gubernator_b200.native)."""
    srcs = [s for s in SOURCES if os.path.exists(s)]
    target = os.path.join(HERE, out) if out else LIB
    if not out and not force and not needs_build():
        return LIB
    extra = os.environ.get("GUB_NVCC_EXTRA", "").split() + [f"-D{d}" for d in defines]
    cmd = [nvcc_path()] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + ["-o", target] + srcs
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("nvcc failed building libgubernator_b200.so")
    if verbose:
        sys.stderr.write(res.stdout + res.stderr)
    return target


if __name__ == "__main__":
    print(build(force=True, verbose="-v" in sys.argv))
