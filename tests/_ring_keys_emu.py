"""Builds/loads the TEST-ONLY CPU emulation of the ring fed with key strings (tests/ring_keys_emu_harness.cpp: the kernel emulation of
tests/kernel_emu_harness.cpp plus a step whose phase 1 is k_p2p_route_keys).  Its own library, so the one of tests/_kernel_emu.py is
untouched; both clusters a test compares (keys and records) live in this one."""
import ctypes as C
import os
import subprocess

import numpy as np

import _kernel_emu as E

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SO = os.path.join(HERE, "libring_keys_emu_test.so")
SRC = [os.path.join(HERE, "ring_keys_emu_harness.cpp")] + E.SRC

_libs = {}


def lib():
    if "L" not in _libs:
        if not os.path.exists(SO) or any(os.path.getmtime(s) > os.path.getmtime(SO) for s in SRC):
            subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-msse2", "-ffp-contract=off", "-Wno-unknown-pragmas",
                                   "-Wl,-Bsymbolic", "-I", os.path.join(ROOT, "include"), "-x", "c++", SRC[0], "-o", SO])
        L = C.CDLL(SO)
        vp, u64, u32, i64 = C.c_void_p, C.c_uint64, C.c_uint32, C.c_int64
        L.emu_set_finish_cap.argtypes = [u32]; L.emu_set_finish_cap.restype = None
        L.emu_set_fused.argtypes = [u32]; L.emu_set_fused.restype = None
        L.emu_p2p_create.argtypes = [u32, u32, u64, u32, vp, vp, u32]; L.emu_p2p_create.restype = vp
        L.emu_p2p_step.argtypes = [vp, vp, vp, vp, vp, u32, vp]
        L.emu_p2p_step_keys.argtypes = [vp, vp, vp, vp, vp, u32, i64, vp, vp, u32, vp, vp]
        L.emu_p2p_route_state.argtypes = [vp, u32, vp, vp, vp]; L.emu_p2p_route_state.restype = None
        _libs["L"] = L
    return _libs["L"]


class KeysP2PCluster(E.EmuP2PCluster):
    """E.EmuP2PCluster (step() with records) on this library, plus step_keys() and route_state()."""

    def __init__(self, world, cap, capacity_slots, pts, peers, max_batch=4096, finish_cap=132, fused=False):
        self.world, self.cap = world, cap
        self.fused = bool(fused)
        self.capacity_slots = int(capacity_slots)
        self._L = lib()
        self._finish_cap = finish_cap
        pts, peers = np.ascontiguousarray(pts, dtype=np.uint64), np.ascontiguousarray(peers, dtype=np.int32)
        self._h = self._L.emu_p2p_create(world, cap, int(capacity_slots), int(max_batch), pts.ctypes.data, peers.ctypes.data, len(pts))

    def step_keys(self, packed, params, created_base, clk, resp_dtype, n, global_mode=False, req_dtype=None):
        """step() with key strings: packed[r] = shard r's batch (a uint8 array in the layout of gub_keys_layout, or (address, size)
        of one), n[r] its request count, params the PARAMS_DTYPE table.  global_mode: also returns every request's ring owner and
        (as req_dtype) its expanded record."""
        W = self.world
        ptrs, sizes = [], []
        for b in packed:
            if isinstance(b, tuple):
                ptrs.append(b[0]); sizes.append(b[1])
            else:
                ptrs.append(b.ctypes.data if len(b) else None); sizes.append(len(b))
        n = np.array(n, dtype=np.uint32)
        outs = [np.zeros(max(int(k), 1), dtype=resp_dtype) for k in n]
        owners = [np.zeros(max(int(k), 1), dtype=np.uint8) for k in n]
        expanded = [np.zeros(max(int(k), 1), dtype=req_dtype or np.dtype((np.void, 64))) for k in n]
        params = np.ascontiguousarray(params)
        bs = np.array(sizes, dtype=np.uint64)
        pp = (C.c_void_p * W)(*ptrs)
        op = (C.c_void_p * W)(*[o.ctypes.data for o in outs])
        wp = (C.c_void_p * W)(*[o.ctypes.data for o in owners])
        ep = (C.c_void_p * W)(*[e.ctypes.data for e in expanded])
        self._L.emu_set_finish_cap(self._finish_cap)
        self._L.emu_set_fused(1 if self.fused else 0)
        try:
            rc = self._L.emu_p2p_step_keys(self._h, pp, bs.ctypes.data, n.ctypes.data, params.ctypes.data if len(params) else None, len(params),
                                           int(created_base), clk.ctypes.data, op, 1 if global_mode else 0, wp if global_mode else None,
                                           ep if global_mode else None)
        finally:
            self._L.emu_set_finish_cap(132)
            self._L.emu_set_fused(0)
        assert rc == 0, "a mailbox flag wait timed out"
        res = [o[:int(k)] for o, k in zip(outs, n)]
        if global_mode:
            return res, [o[:int(k)] for o, k in zip(owners, n)], [e[:int(k)] for e, k in zip(expanded, n)]
        return res

    def route_state(self, rank, req_dtype):
        """(request mailbox block [2 x W x cap], perm [cap], counts [W]) of shard `rank` as the last routing left them."""
        mb = np.zeros(2 * self.world * self.cap, dtype=req_dtype)
        perm, counts = np.zeros(self.cap, dtype=np.uint32), np.zeros(self.world, dtype=np.uint32)
        self._L.emu_p2p_route_state(self._h, rank, mb.ctypes.data, perm.ctypes.data, counts.ctypes.data)
        return mb, perm, counts
