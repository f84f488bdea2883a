"""Builds/loads the TEST-ONLY CPU emulation of the wire-format entry on the ring (tests/ring_proto_emu_harness.cpp: the kernel emulation of
tests/kernel_emu_harness.cpp plus the kernels of gub_proto.cuh, run in gub_p2p_step_proto_local_all's order).  Its own library, so the
ones of tests/_kernel_emu.py and tests/_proto_emu.py are untouched; both clusters a test compares (wire bytes and records) live in this one."""
import ctypes as C
import os
import subprocess

import numpy as np

import _kernel_emu as E

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SO = os.path.join(HERE, "libring_proto_emu_test.so")
SRC = [os.path.join(HERE, "ring_proto_emu_harness.cpp"), os.path.join(ROOT, "gubernator_b200", "csrc", "gub_proto.cuh")] + E.SRC

_libs = {}


def lib():
    if "L" not in _libs:
        if not os.path.exists(SO) or any(os.path.getmtime(s) > os.path.getmtime(SO) for s in SRC):
            subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-msse2", "-ffp-contract=off", "-Wno-unknown-pragmas",
                                   "-Wl,-Bsymbolic", "-I", os.path.join(ROOT, "include"), "-x", "c++", SRC[0], "-o", SO])
        L = C.CDLL(SO)
        vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32
        L.emu_set_finish_cap.argtypes = [u32]; L.emu_set_finish_cap.restype = None
        L.emu_set_fused.argtypes = [u32]; L.emu_set_fused.restype = None
        L.emu_p2p_create.argtypes = [u32, u32, u64, u32, vp, vp, u32]; L.emu_p2p_create.restype = vp
        L.emu_p2p_table.argtypes = [vp, u32]; L.emu_p2p_table.restype = vp
        L.emu_p2p_step.argtypes = [vp, vp, vp, vp, vp, u32, vp]
        L.emu_p2p_step_proto.argtypes = [vp, vp, vp, vp, u32, vp, vp, vp, vp, vp, u32, vp, vp, vp, vp]
        L.emu_p2p_epoch.argtypes = [vp]; L.emu_p2p_epoch.restype = u32
        L.emu_scan.argtypes = [vp, vp, u64]; L.emu_scan.restype = u64
        L.emu_counters.argtypes = [vp, vp]; L.emu_counters.restype = None
        L.emu_install_updates.argtypes = [vp, vp, u32, C.c_int64]; L.emu_install_updates.restype = None
        _libs["L"] = L
    return _libs["L"]


class ProtoP2PCluster(E.EmuP2PCluster):
    """E.EmuP2PCluster (step() with records) on this library, plus step_proto() and epoch()."""

    def __init__(self, world, cap, capacity_slots, pts, peers, max_batch=4096, finish_cap=132, fused=False):
        self.world, self.cap = world, cap
        self.fused = bool(fused)
        self.capacity_slots = int(capacity_slots)
        self._L = lib()
        self._finish_cap = finish_cap
        pts, peers = np.ascontiguousarray(pts, dtype=np.uint64), np.ascontiguousarray(peers, dtype=np.int32)
        self._h = self._L.emu_p2p_create(world, cap, int(capacity_slots), int(max_batch), pts.ctypes.data, peers.ctypes.data, len(pts))

    def epoch(self):
        return int(self._L.emu_p2p_epoch(self._h))

    def step_proto(self, packed, n_msgs, clk, out_caps=None, force_global=False, global_mode=False, timeouts=None, guard=64):
        """packed[r] = shard r's pack_proto() buffer, n_msgs[r] its message count.  Returns (steps, [(statuses, [response bytes per
        message]) per shard]), or None when the host-side checks refuse the call.  timeouts[r]: dense-batch indices of shard r answered
        GUB_ERR_PEER_TIMEOUT.  global_mode: each shard's result also carries the ring owner of every item of its dense batch.  Each output
        has `guard` bytes of 0xA5 on both sides, checked here."""
        W = self.world
        caps = [int(c) for c in out_caps]
        raws = [np.full(c + 2 * guard, 0xA5, dtype=np.uint8) for c in caps]
        offs = [np.zeros(int(k) + 1, dtype=np.uint64) for k in n_msgs]
        sts = [np.full(max(int(k), 1), 0xEE, dtype=np.uint32) for k in n_msgs]
        tos = [np.ascontiguousarray(t if t is not None else [], dtype=np.uint32) for t in (timeouts or [None] * W)]
        pp = (C.c_void_p * W)(*[b.ctypes.data if len(b) else None for b in packed])
        pb = np.array([len(b) for b in packed], dtype=np.uint64)
        nm = np.array(n_msgs, dtype=np.uint32)
        oc = np.array(caps, dtype=np.uint64)
        op = (C.c_void_p * W)(*[r[guard:].ctypes.data for r in raws])
        fp = (C.c_void_p * W)(*[o.ctypes.data for o in offs])
        sp = (C.c_void_p * W)(*[s.ctypes.data for s in sts])
        tp = (C.c_void_p * W)(*[t.ctypes.data if len(t) else None for t in tos])
        tn = np.array([len(t) for t in tos], dtype=np.uint32)
        owners = [np.zeros(len(b) // 2 + 1, dtype=np.uint8) for b in packed]  # (a dense batch has at most one item per 2 message bytes)
        wp = (C.c_void_p * W)(*[o.ctypes.data for o in owners])
        steps = C.c_uint32(0)
        self._L.emu_set_finish_cap(self._finish_cap)
        self._L.emu_set_fused(1 if self.fused else 0)
        try:
            rc = self._L.emu_p2p_step_proto(self._h, pp, pb.ctypes.data, nm.ctypes.data, 1 if force_global else 0, clk.ctypes.data, op,
                                            oc.ctypes.data, fp, sp, 1 if global_mode else 0, tp, tn.ctypes.data, wp if global_mode else None,
                                            C.byref(steps))
        finally:
            self._L.emu_set_finish_cap(132)
            self._L.emu_set_fused(0)
        if rc == -1:
            return None
        assert rc == 0, "a mailbox flag wait timed out"
        res = []
        for r in range(W):
            raw = raws[r]
            assert (raw[:guard] == 0xA5).all() and (raw[guard + caps[r]:] == 0xA5).all(), f"shard {r}: a guard byte was overwritten"
            out = raw[guard:guard + caps[r]]
            k = int(n_msgs[r])
            one = (sts[r][:k].tolist(), [out[int(offs[r][m]):int(offs[r][m + 1])].tobytes() for m in range(k)])
            res.append(one + (owners[r],) if global_mode else one)  # (owners: trimmed by the caller, who knows n_r)
        return int(steps.value), res
