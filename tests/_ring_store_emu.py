"""Builds/loads the TEST-ONLY CPU emulation of the ring's Store step (tests/ring_store_emu_harness.cpp: the kernel emulation with the
Store passes of tests/store_emu_harness.cpp plus a ring step driven like gub_p2p_step_keys_store_local_all).  Its own library, so
those of tests/_kernel_emu.py and tests/_store_emu.py are untouched."""
import ctypes as C
import os
import subprocess

import numpy as np

import _kernel_emu as E
import _store_emu as SE

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SO = os.path.join(HERE, "libring_store_emu_test.so")
SRC = [os.path.join(HERE, "ring_store_emu_harness.cpp"), os.path.join(HERE, "store_emu_harness.cpp")] + SE.SRC[1:]

# gub_store_rec with the ring's naming fields (the same 104 bytes as _store_emu.REC_DTYPE)
REC_DTYPE = np.dtype([("first", "<u4"), ("last", "<u4"), ("flags", "<u4"), ("first_shard", "<u2"), ("last_shard", "<u2"), ("item", SE.ITEM_DTYPE)])
assert REC_DTYPE.itemsize == SE.REC_DTYPE.itemsize

_libs = {}


def lib():
    if "L" not in _libs:
        if not os.path.exists(SO) or any(os.path.getmtime(s) > os.path.getmtime(SO) for s in SRC):
            subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-msse2", "-ffp-contract=off", "-Wno-unknown-pragmas",
                                   "-Wl,-Bsymbolic", "-I", os.path.join(ROOT, "include"), "-x", "c++", SRC[0], "-o", SO])
        L = C.CDLL(SO)
        vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32
        L.emu_set_finish_cap.argtypes = [u32]; L.emu_set_finish_cap.restype = None
        L.emu_p2p_create.argtypes = [u32, u32, u64, u32, vp, vp, u32]; L.emu_p2p_create.restype = vp
        L.emu_p2p_table.argtypes = [vp, u32]; L.emu_p2p_table.restype = vp
        L.emu_ring_store_step.argtypes = [vp, vp, vp, vp, SE.GET_FN, vp, vp, vp, vp]
        L.emu_ring_store_set_epoch.argtypes = [vp, u32, u32]; L.emu_ring_store_set_epoch.restype = None
        L.emu_ring_store_epoch.argtypes = [vp, u32]; L.emu_ring_store_epoch.restype = u32
        L.emu_ring_ovf_count.argtypes = [vp, u32]; L.emu_ring_ovf_count.restype = u32
        L.emu_counters.argtypes = [vp, vp]; L.emu_counters.restype = None
        L.emu_scan.argtypes = [vp, vp, u64]; L.emu_scan.restype = u64
        _libs["L"] = L
    return _libs["L"]


class StoreRingCluster:
    """W shards in one process stepping with a Store, phase by phase (ring_store_emu_harness.cpp)."""

    def __init__(self, world, cap, capacity_slots, pts, peers, max_batch, finish_cap=3):
        self.world, self.cap, self.capacity = world, cap, int(capacity_slots)
        self._L = lib()
        self._finish_cap = finish_cap
        pts, peers = np.ascontiguousarray(pts, dtype=np.uint64), np.ascontiguousarray(peers, dtype=np.int32)
        self._h = self._L.emu_p2p_create(world, cap, self.capacity, int(max_batch), pts.ctypes.data, peers.ctypes.data, len(pts))

    def step(self, batches, clk, resp_dtype, get):
        """batches[r] = shard r's ingest (request records); get: None or a callable(misses) -> int over REC_DTYPE misses.
        Returns (rc, responses per shard, change log per owner)."""
        W = self.world
        batches = [np.ascontiguousarray(b) for b in batches]
        n = np.array([len(b) for b in batches], dtype=np.uint32)
        outs = [np.zeros(max(len(b), 1), dtype=resp_dtype) for b in batches]
        changes = [np.zeros(W * self.cap, dtype=REC_DTYPE) for _ in range(W)]
        n_changes = np.zeros(W, dtype=np.uint32)
        cb = SE.GET_FN()
        if get is not None:
            cb = SE.GET_FN(lambda _u, p, m: int(get(np.frombuffer((C.c_char * (m * REC_DTYPE.itemsize)).from_address(p), dtype=REC_DTYPE)) or 0))
        self._L.emu_set_finish_cap(self._finish_cap)
        try:
            rc = self._L.emu_ring_store_step(self._h, (C.c_void_p * W)(*[b.ctypes.data for b in batches]), n.ctypes.data, clk.ctypes.data, cb, None,
                                             (C.c_void_p * W)(*[o.ctypes.data for o in outs]), (C.c_void_p * W)(*[c.ctypes.data for c in changes]),
                                             n_changes.ctypes.data)
        finally:
            self._L.emu_set_finish_cap(132)
        return rc, [o[:len(b)] for o, b in zip(outs, batches)], [c[:int(k)].copy() for c, k in zip(changes, n_changes)]

    def counters(self, rank):
        c = np.zeros(len(E.COUNTER_NAMES), dtype=np.uint64)
        self._L.emu_counters(self._L.emu_p2p_table(self._h, rank), c.ctypes.data)
        return dict(zip(E.COUNTER_NAMES, (int(v) for v in c)))

    def scan(self, rank, item_dtype):
        out = np.zeros(self.capacity, dtype=item_dtype)
        k = self._L.emu_scan(self._L.emu_p2p_table(self._h, rank), out.ctypes.data, len(out))
        out = out[:k]
        return out[np.lexsort((out["key_fnv1"], out["key_xxh64"]))]

    def ovf_count(self, rank):
        """Inserts the last step parked on owner `rank` (the next step's k_group places them)."""
        return int(self._L.emu_ring_ovf_count(self._h, rank))

    def set_store_epoch(self, rank, e):
        self._L.emu_ring_store_set_epoch(self._h, rank, int(e))

    def store_epoch(self, rank):
        return int(self._L.emu_ring_store_epoch(self._h, rank))
