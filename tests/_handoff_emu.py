"""Builds/loads the TEST-ONLY CPU emulation of the single-table pipeline with two grouping scratch sets and k_group's early path
(tests/handoff_emu_harness.cpp: the kernel emulation of tests/kernel_emu_harness.cpp plus a launcher like launch_chunk of gub_api.cu).
Its own library, so the one of tests/_kernel_emu.py is untouched."""
import ctypes as C
import os
import subprocess

import numpy as np

import _kernel_emu as E

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SO = os.path.join(HERE, "libhandoff_emu_test.so")
SRC = [os.path.join(HERE, "handoff_emu_harness.cpp")] + E.SRC

_libs = {}


def lib():
    if "L" not in _libs:
        if not os.path.exists(SO) or any(os.path.getmtime(s) > os.path.getmtime(SO) for s in SRC):
            subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-msse2", "-ffp-contract=off", "-Wno-unknown-pragmas",
                                   "-Wl,-Bsymbolic", "-I", os.path.join(ROOT, "include"), "-x", "c++", SRC[0], "-o", SO])
        L = C.CDLL(SO)
        vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32
        L.emu_handoff_create.argtypes = [u64, u32]; L.emu_handoff_create.restype = vp
        L.emu_handoff_destroy.argtypes = [vp]; L.emu_handoff_destroy.restype = None
        L.emu_handoff_submit.argtypes = [vp, vp, C.c_size_t, vp, vp, u32]
        L.emu_handoff_chain_done.argtypes = [vp]; L.emu_handoff_chain_done.restype = u32
        L.emu_set_epoch.argtypes = [vp, u32]; L.emu_set_epoch.restype = None
        L.emu_counters.argtypes = [vp, vp]; L.emu_counters.restype = None
        L.emu_scan.argtypes = [vp, vp, u64]; L.emu_scan.restype = u64
        _libs["L"] = L
    return _libs["L"]


class HandoffTable(E.EmuTable):
    """E.EmuTable's surface (counters, scan, set_epoch) on a table with two scratch sets; submit(early=True) makes every k_group block
    take the early path."""

    def __init__(self, capacity_slots, max_batch=65536):
        self._L = lib()
        self._h = self._L.emu_handoff_create(int(capacity_slots), int(max_batch))
        self.capacity = int(capacity_slots)
        self.fused = False

    def submit(self, reqs, clk, resp_dtype, early=True):
        out = np.zeros(len(reqs), dtype=resp_dtype)
        reqs = np.ascontiguousarray(reqs)
        assert reqs.dtype.itemsize == 64 and out.dtype.itemsize == 32
        self._L.emu_handoff_submit(self._h, reqs.ctypes.data, len(reqs), clk.ctypes.data, out.ctypes.data, 1 if early else 0)
        return out

    def chain_done(self):
        return int(self._L.emu_handoff_chain_done(self._h))

    def __del__(self):
        try:
            self._L.emu_handoff_destroy(self._h)
        except Exception:
            pass
