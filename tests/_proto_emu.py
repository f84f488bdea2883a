"""Builds/loads the TEST-ONLY CPU emulation of the wire-format entry (tests/proto_emu_harness.cpp: the kernel emulation of
tests/kernel_emu_harness.cpp plus the kernels of gub_proto.cuh, run in gub_submit_proto_async's order).  Its own library, so the one of
tests/_kernel_emu.py is untouched."""
import ctypes as C
import os
import subprocess

import numpy as np

import _kernel_emu as E

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SO = os.path.join(HERE, "libproto_emu_test.so")
SRC = [os.path.join(HERE, "proto_emu_harness.cpp"), os.path.join(ROOT, "gubernator_b200", "csrc", "gub_proto.cuh")] + E.SRC

_libs = {}


def lib():
    if "L" not in _libs:
        if not os.path.exists(SO) or any(os.path.getmtime(s) > os.path.getmtime(SO) for s in SRC):
            subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-msse2", "-ffp-contract=off", "-Wno-unknown-pragmas",
                                   "-Wl,-Bsymbolic", "-I", os.path.join(ROOT, "include"), "-x", "c++", SRC[0], "-o", SO])
        L = C.CDLL(SO)
        vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32
        L.emu_create.argtypes = [u64, u32]; L.emu_create.restype = vp
        L.emu_destroy.argtypes = [vp]; L.emu_destroy.restype = None
        L.emu_set_fused.argtypes = [u32]; L.emu_set_fused.restype = None
        L.emu_submit.argtypes = [vp, vp, C.c_size_t, vp, vp]
        L.emu_counters.argtypes = [vp, vp]; L.emu_counters.restype = None
        L.emu_scan.argtypes = [vp, vp, u64]; L.emu_scan.restype = u64
        L.emu_submit_proto.argtypes = [vp, vp, u64, u32, vp, vp, u64, vp, vp]
        _libs["L"] = L
    return _libs["L"]


class ProtoEmuTable(E.EmuTable):
    """E.EmuTable on this library, plus submit_proto()."""

    def __init__(self, capacity_slots, max_batch=65536):
        self._L = lib()
        self._h = self._L.emu_create(int(capacity_slots), int(max_batch))
        self.capacity = int(capacity_slots)
        self.fused = False

    def submit_proto(self, packed, n_msgs, clk, out_cap, guard=64):
        """(statuses, [response bytes per message], raw output buffer with `guard` bytes on each side)."""
        raw = np.full(out_cap + 2 * guard, 0xA5, dtype=np.uint8)
        off = np.zeros(n_msgs + 1, dtype=np.uint64)
        st = np.full(max(n_msgs, 1), 0xEE, dtype=np.uint32)
        rc = self._L.emu_submit_proto(self._h, packed.ctypes.data, len(packed), n_msgs, clk.ctypes.data, raw[guard:].ctypes.data, out_cap,
                                      off.ctypes.data, st.ctypes.data)
        assert rc == 0, "the host-side checks refused the call"
        out = raw[guard:guard + out_cap]
        return st[:n_msgs].tolist(), [out[int(off[m]):int(off[m + 1])].tobytes() for m in range(n_msgs)], raw, off
