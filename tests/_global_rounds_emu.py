"""Builds/loads the TEST-ONLY CPU emulation of the GLOBAL tick's rounds (tests/global_rounds_emu_harness.cpp: the kernel emulation of
tests/kernel_emu_harness.cpp plus k_gq_hist, gq_plan_rounds, k_gq_partition and gq_round_span).  Its own library, so the one of
tests/_kernel_emu.py is untouched."""
import ctypes as C
import os
import subprocess

import numpy as np

import _kernel_emu as E

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SO = os.path.join(HERE, "libglobal_rounds_emu_test.so")
SRC = [os.path.join(HERE, "global_rounds_emu_harness.cpp")] + E.SRC

_libs = {}


def lib():
    if "L" not in _libs:
        if not os.path.exists(SO) or any(os.path.getmtime(s) > os.path.getmtime(SO) for s in SRC):
            subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-msse2", "-ffp-contract=off", "-Wno-unknown-pragmas",
                                   "-Wl,-Bsymbolic", "-I", os.path.join(ROOT, "include"), "-x", "c++", SRC[0], "-o", SO])
        L = C.CDLL(SO)
        vp, u32 = C.c_void_p, C.c_uint32
        L.emu_gq_bins.argtypes = []; L.emu_gq_bins.restype = u32
        L.emu_gq_hist.argtypes = [vp, u32, vp]; L.emu_gq_hist.restype = None
        L.emu_gq_plan.argtypes = [vp, u32, u32, vp, u32]; L.emu_gq_plan.restype = u32
        L.emu_gq_partition.argtypes = [vp, u32, vp, u32, vp, u32, vp, vp, vp]; L.emu_gq_partition.restype = None
        _libs["L"] = L
    return _libs["L"]


def bins():
    return int(lib().emu_gq_bins())


def hist(recs):
    """k_gq_hist over the records (an HREQ_DTYPE array) -> uint32 [GQ_BINS]."""
    recs = np.ascontiguousarray(recs)
    h = np.zeros(bins(), dtype=np.uint32)
    lib().emu_gq_hist(recs.ctypes.data if len(recs) else None, len(recs), h.ctypes.data)
    return h


def plan(hists, cap):
    """gq_plan_rounds over the sources' histograms -> int64 [R, 3] of (lo, hi, slice)."""
    hs = np.ascontiguousarray(np.stack(hists), dtype=np.uint32)
    cap_rounds = 1 << 20
    out = np.zeros((cap_rounds, 3), dtype=np.uint32)
    n = lib().emu_gq_plan(hs.ctypes.data, len(hists), int(cap), out.ctypes.data, cap_rounds)
    assert n <= cap_rounds
    return out[:n].astype(np.int64)


def partition(recs, h, cap, rounds):
    """k_gq_partition of one source's records -> (records in round order, offset [R], count [R]) of every round."""
    recs = np.ascontiguousarray(recs)
    out = np.zeros(max(len(recs), 1), dtype=recs.dtype)
    rr = np.ascontiguousarray(rounds, dtype=np.uint32)
    offs, counts = np.zeros(max(len(rr), 1), dtype=np.uint32), np.zeros(max(len(rr), 1), dtype=np.uint32)
    h = np.ascontiguousarray(h, dtype=np.uint32)
    lib().emu_gq_partition(recs.ctypes.data if len(recs) else None, len(recs), h.ctypes.data, int(cap), rr.ctypes.data, len(rr), out.ctypes.data,
                           offs.ctypes.data, counts.ctypes.data)
    return out[:len(recs)], offs[:len(rr)].astype(np.int64), counts[:len(rr)].astype(np.int64)
