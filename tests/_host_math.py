"""Builds/loads the TEST-ONLY host compilation of gubernator_b200/csrc/bucket_math.cuh (tests/host_math_harness.cpp), and the
TEST-ONLY device compilation of the same header (tests/bucket_math_dev.cu, built by build_dev() from build())."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SO = os.path.join(HERE, "libhostmath_test.so")
SRC = [os.path.join(HERE, "host_math_harness.cpp"), os.path.join(ROOT, "gubernator_b200", "csrc", "bucket_math.cuh"),
       os.path.join(ROOT, "include", "gubernator_b200.h")]
DEV_SO = os.path.join(HERE, "libbucketmath_dev_test.so")
DEV_SRC = [os.path.join(HERE, "bucket_math_dev.cu")] + SRC[1:]

CLOCK_DTYPE = np.dtype([("now_ms", "<i8"), ("greg_expire", "<i8", (6,)), ("greg_duration", "<i8", (6,))])
BUCKET_DTYPE = np.dtype([("key", "<u8"), ("tag", "<u8"), ("limit", "<i8"), ("duration", "<i8"), ("rem", "<u8"),
                         ("stamp", "<i8"), ("burst", "<i8"), ("expire", "<i8"), ("flags", "<u4"), ("_pad", "<u4")])
DELTA_DTYPE = np.dtype([("over", "<u4"), ("hit", "<u4"), ("miss", "<u4")])
F_LEAKY, F_OVER, F_LIVE = 1, 2, 4

_lib = None
_dev_lib = None


def _elementwise(L):
    vp, sz = C.c_void_p, C.c_size_t
    L.hm_f2i.argtypes = [vp, vp, sz]; L.hm_f2i.restype = None
    L.hm_apply_one.argtypes = [vp, vp, vp, sz, vp, vp]; L.hm_apply_one.restype = None
    L.hm_run_to_rank.argtypes = [vp, vp, vp, vp, sz, vp, vp]; L.hm_run_to_rank.restype = None
    L.hm_sizeof_bucket.restype = C.c_size_t
    assert L.hm_sizeof_bucket() == BUCKET_DTYPE.itemsize


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO) or any(os.path.getmtime(s) > os.path.getmtime(SO) for s in SRC):
            subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-msse2", "-ffp-contract=off",
                                   "-x", "c++", SRC[0], "-o", SO])
        L = C.CDLL(SO)
        L.hm_table_new.restype = C.c_void_p
        L.hm_table_free.argtypes = [C.c_void_p]
        L.hm_apply_seq.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
        L.hm_plan_check.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
        L.hm_rank_check.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
        _elementwise(L)
        _lib = L
    return _lib


def build_dev(force=False):
    """nvcc with the product library's flags (so the device build sees the same --fmad=false and sm_90a) -> DEV_SO."""
    from gubernator_b200 import build as B
    if force or not os.path.exists(DEV_SO) or any(os.path.getmtime(s) > os.path.getmtime(DEV_SO) for s in DEV_SRC):
        subprocess.check_call([B.nvcc_path()] + B.NVCC_FLAGS + ["-o", DEV_SO, DEV_SRC[0]])
    return DEV_SO


def dev_lib():
    """The device build; a missing library is an error (build() makes it)."""
    global _dev_lib
    if _dev_lib is None:
        if not os.path.exists(DEV_SO):
            raise FileNotFoundError(f"{DEV_SO} is missing: __graft_entry__.build() builds it")
        L = C.CDLL(DEV_SO)
        _elementwise(L)
        L.bmd_f2i_bare.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]; L.bmd_f2i_bare.restype = None
        L.bmd_add.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]; L.bmd_add.restype = None
        _dev_lib = L
    return _dev_lib


def _checked(L):
    if hasattr(L, "bmd_error"):
        assert L.bmd_error() == 0, f"CUDA error {L.bmd_error()}"


def f2i(L, x, fn="hm_f2i"):
    x = np.ascontiguousarray(x, dtype=np.float64)
    out = np.zeros(len(x), dtype=np.int64)
    getattr(L, fn)(x.ctypes.data, out.ctypes.data, len(x))
    _checked(L)
    return out


def apply_one(L, buckets, reqs, clk):
    """(responses, buckets after, deltas) of one apply_one() per (bucket, request) pair."""
    import oracle_py as O
    b = np.ascontiguousarray(buckets).copy()
    reqs = np.ascontiguousarray(reqs)
    out, d = np.zeros(len(b), dtype=O.HRESP_DTYPE), np.zeros(len(b), dtype=DELTA_DTYPE)
    L.hm_apply_one(b.ctypes.data, reqs.ctypes.data, clk.ctypes.data, len(b), out.ctypes.data, d.ctypes.data)
    _checked(L)
    return out, b, d


def run_to_rank(L, buckets, reqs, targets, clk):
    import oracle_py as O
    b = np.ascontiguousarray(buckets).copy()
    reqs = np.ascontiguousarray(reqs)
    t = np.ascontiguousarray(targets, dtype=np.uint32)
    out, d = np.zeros(len(b), dtype=O.HRESP_DTYPE), np.zeros(len(b), dtype=DELTA_DTYPE)
    L.hm_run_to_rank(b.ctypes.data, reqs.ctypes.data, t.ctypes.data, clk.ctypes.data, len(b), out.ctypes.data, d.ctypes.data)
    _checked(L)
    return out, b, d


class HostTable:
    def __init__(self):
        self._t = lib().hm_table_new()

    def apply_seq(self, reqs, clk):
        import oracle_py as O
        out = np.zeros(len(reqs), dtype=O.HRESP_DTYPE)
        ctr = np.zeros(3, dtype=np.uint64)
        lib().hm_apply_seq(self._t, reqs.ctypes.data, len(reqs), clk.ctypes.data, out.ctypes.data, ctr.ctypes.data)
        return out, dict(over_limit=int(ctr[0]), cache_hit=int(ctr[1]), cache_miss=int(ctr[2]))

    def __del__(self):
        try:
            lib().hm_table_free(self._t)
        except Exception:
            pass


def plan_check(bucket, req, m, clk, cap=16):
    npieces = C.c_uint32(0)
    covered = C.c_uint32(0)
    rc = lib().hm_plan_check(bucket.ctypes.data, req.ctypes.data, m, clk.ctypes.data, cap, C.byref(npieces), C.byref(covered))
    return rc, npieces.value, covered.value


def rank_check(bucket, req, m, clk, stride=1):
    return lib().hm_rank_check(bucket.ctypes.data, req.ctypes.data, m, clk.ctypes.data, stride)
