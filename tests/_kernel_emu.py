"""Builds/loads the TEST-ONLY CPU emulation of the CUDA kernels (tests/kernel_emu_harness.cpp on tests/cuda_emu.h): the
kernel source of gubernator_b200/csrc/gub_kernels.cuh, compiled with g++ and run with fibers standing in for threads."""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SO = os.path.join(HERE, "libkernel_emu_test.so")
SRC = [os.path.join(HERE, "kernel_emu_harness.cpp"), os.path.join(HERE, "cuda_emu.h"),
       os.path.join(ROOT, "gubernator_b200", "csrc", "gub_kernels.cuh"), os.path.join(ROOT, "gubernator_b200", "csrc", "bucket_math.cuh"),
       os.path.join(ROOT, "gubernator_b200", "csrc", "gub_batch.cuh"), os.path.join(ROOT, "gubernator_b200", "csrc", "gub_p2p.cuh"),
       os.path.join(ROOT, "gubernator_b200", "csrc", "gub_global.cuh"),
       os.path.join(ROOT, "include", "gubernator_b200.h")]
COUNTER_NAMES = ["over_limit", "cache_hit", "cache_miss", "inserts", "table_full", "requests", "batches", "dup_groups", "mixed_groups",
                 "serial_fallbacks", "unexpired_evictions", "swept", "gq_dropped"]

_libs = {}


def lib():
    if "L" not in _libs:
        so = SO
        if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in SRC):
            subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-msse2", "-ffp-contract=off", "-Wno-unknown-pragmas",
                                   "-I", os.path.join(ROOT, "include"), "-x", "c++", SRC[0], "-o", so])
        L = C.CDLL(so)
        vp, u64, u32, i64 = C.c_void_p, C.c_uint64, C.c_uint32, C.c_int64
        L.emu_create.argtypes = [u64, u32]; L.emu_create.restype = vp
        L.emu_destroy.argtypes = [vp]; L.emu_destroy.restype = None
        L.emu_set_epoch.argtypes = [vp, u32]; L.emu_set_epoch.restype = None
        L.emu_set_finish_cap.argtypes = [u32]; L.emu_set_finish_cap.restype = None
        L.emu_set_fused.argtypes = [u32]; L.emu_set_fused.restype = None
        L.emu_set_grid.argtypes = [vp, u32]; L.emu_set_grid.restype = None
        L.emu_set_sweep.argtypes = [vp, u32]; L.emu_set_sweep.restype = None
        L.emu_submit.argtypes = [vp, vp, C.c_size_t, vp, vp]
        L.emu_submit_compact.argtypes = [vp, vp, C.c_size_t, vp, C.c_size_t, i64, vp, vp]
        L.emu_counters.argtypes = [vp, vp]; L.emu_counters.restype = None
        L.emu_scan.argtypes = [vp, vp, u64]; L.emu_scan.restype = u64
        L.emu_add_items.argtypes = [vp, vp, u32]; L.emu_add_items.restype = u32
        L.emu_get_items.argtypes = [vp, vp, vp, u32, i64, vp, vp]; L.emu_get_items.restype = None
        L.emu_sweep.argtypes = [vp, i64]; L.emu_sweep.restype = u64
        L.emu_sweep_range.argtypes = [vp, u64, u64, i64]; L.emu_sweep_range.restype = u64
        L.emu_random_rmw.argtypes = [vp, u64]; L.emu_random_rmw.restype = None
        L.emu_hash_keys.argtypes = [vp, vp, u32, vp, vp]; L.emu_hash_keys.restype = None
        L.emu_route.argtypes = [vp, u32, vp, vp, u32, u32, vp, vp, vp, vp]; L.emu_route.restype = None
        L.emu_unroute.argtypes = [vp, vp, u32, vp]; L.emu_unroute.restype = None
        L.emu_gq_create.argtypes = [u32, u32]; L.emu_gq_create.restype = vp
        L.emu_gq_accumulate.argtypes = [vp, vp, u32, vp, u32, u64]; L.emu_gq_accumulate.restype = None
        L.emu_gq_drain.argtypes = [vp, vp, u32, u32]; L.emu_gq_drain.restype = u32
        L.emu_make_updates.argtypes = [vp, vp, u32, vp]; L.emu_make_updates.restype = u32
        L.emu_p2p_create.argtypes = [u32, u32, u64, u32, vp, vp, u32]; L.emu_p2p_create.restype = vp
        L.emu_p2p_table.argtypes = [vp, u32]; L.emu_p2p_table.restype = vp
        L.emu_p2p_step.argtypes = [vp, vp, vp, vp, vp, u32, vp]
        L.emu_install_updates.argtypes = [vp, vp, u32, i64]; L.emu_install_updates.restype = None
        assert L.emu_counter_count() == len(COUNTER_NAMES)
        _libs["L"] = L
    return _libs["L"]


class EmuTable:
    """Same surface as gubernator_b200.native.Table for what the CPU tests need."""

    def __init__(self, capacity_slots, max_batch=65536, fused=False, grid=6, sweep=0):
        """fused: evaluate with the persistent kernel k_batch (what rings use) instead of the four-kernel pipeline; grid = its CTAs
        (every emulated CTA costs 512 fibers; the kernel takes any grid, more rounds make up for it); sweep = slots every CTA of
        k_batch sweeps per round."""
        self._L = lib()
        self._h = self._L.emu_create(int(capacity_slots), int(max_batch))
        self.capacity = int(capacity_slots)
        self.fused = bool(fused)
        self._L.emu_set_grid(self._h, int(grid))
        self._L.emu_set_sweep(self._h, int(sweep))

    def submit(self, reqs, clk, resp_dtype):
        out = np.zeros(len(reqs), dtype=resp_dtype)
        reqs = np.ascontiguousarray(reqs)
        assert reqs.dtype.itemsize == 64 and out.dtype.itemsize == 32
        self._L.emu_set_fused(1 if self.fused else 0)
        self._L.emu_submit(self._h, reqs.ctypes.data, len(reqs), clk.ctypes.data, out.ctypes.data)
        return out

    def submit_compact(self, creqs, params, created_base, clk, resp_dtype):
        out = np.zeros(len(creqs), dtype=resp_dtype)
        self._L.emu_set_fused(1 if self.fused else 0)
        self._L.emu_submit_compact(self._h, creqs.ctypes.data, len(creqs), params.ctypes.data, len(params), int(created_base), clk.ctypes.data,
                                 out.ctypes.data)
        return out

    def set_epoch(self, e):
        self._L.emu_set_epoch(self._h, int(e))

    def counters(self):
        c = np.zeros(len(COUNTER_NAMES), dtype=np.uint64)
        self._L.emu_counters(self._h, c.ctypes.data)
        return dict(zip(COUNTER_NAMES, (int(v) for v in c)))

    def scan(self, item_dtype):
        out = np.zeros(self.capacity, dtype=item_dtype)
        n = self._L.emu_scan(self._h, out.ctypes.data, len(out))
        return out[:n]

    def add_items(self, items):
        items = np.ascontiguousarray(items)
        assert items.dtype.itemsize == 88
        assert self._L.emu_add_items(self._h, items.ctypes.data, len(items)) == 0, "table full"

    def get_items(self, key_xxh64, key_fnv1, now_ms, item_dtype):
        kx = np.ascontiguousarray(key_xxh64, dtype=np.uint64)
        kf = np.ascontiguousarray(key_fnv1, dtype=np.uint64)
        out, found = np.zeros(len(kx), dtype=item_dtype), np.zeros(len(kx), dtype=np.uint8)
        self._L.emu_get_items(self._h, kx.ctypes.data, kf.ctypes.data, len(kx), int(now_ms), out.ctypes.data, found.ctypes.data)
        return out, found.astype(bool)

    def sweep(self, now_ms):
        return int(self._L.emu_sweep(self._h, int(now_ms)))

    def sweep_range(self, lo, hi, now_ms):
        return int(self._L.emu_sweep_range(self._h, int(lo), int(hi), int(now_ms)))

    def random_rmw(self, accesses):
        self._L.emu_random_rmw(self._h, int(accesses))

    def __del__(self):
        try:
            if getattr(self, "_owned", True):  # (a handle borrowed from an EmuP2PCluster belongs to the cluster)
                self._L.emu_destroy(self._h)
        except Exception:
            pass


def hash_keys(keys):
    """XXH64 and FNV-1 of every key (bytes) through k_hash_keys."""
    blob = b"".join(keys)
    offs = np.zeros(len(keys) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum([len(k) for k in keys])
    buf = np.frombuffer(blob + b"\0", dtype=np.uint8)
    xx, fv = np.zeros(len(keys), dtype=np.uint64), np.zeros(len(keys), dtype=np.uint64)
    lib().emu_hash_keys(buf.ctypes.data, offs.ctypes.data, len(keys), xx.ctypes.data, fv.ctypes.data)
    return xx, fv


def route(reqs, pts, peers, nshards):
    """(partitioned requests, perm, counts, owner) as gub_route_device produces them."""
    n = len(reqs)
    out = np.zeros(max(n, 1), dtype=reqs.dtype)
    perm, counts, owner = np.zeros(max(n, 1), dtype=np.uint32), np.zeros(nshards, dtype=np.uint32), np.zeros(max(n, 1), dtype=np.uint8)
    pts, peers = np.ascontiguousarray(pts, dtype=np.uint64), np.ascontiguousarray(peers, dtype=np.int32)
    reqs = np.ascontiguousarray(reqs)
    lib().emu_route(reqs.ctypes.data, n, pts.ctypes.data, peers.ctypes.data, len(pts), nshards, out.ctypes.data, perm.ctypes.data, counts.ctypes.data,
                    owner.ctypes.data)
    return out[:n], perm[:n], counts, owner[:n]


def unroute(resps, perm):
    out = np.zeros(len(resps), dtype=resps.dtype)
    resps = np.ascontiguousarray(resps)
    if len(resps):
        lib().emu_unroute(resps.ctypes.data, perm.ctypes.data, len(resps), out.ctypes.data)
    return out


class EmuP2PCluster:
    """W shards in one process stepping through gub_p2p_step's kernels phase by phase (see kernel_emu_harness.cpp)."""

    def __init__(self, world, cap, capacity_slots, pts, peers, max_batch=4096, finish_cap=132, fused=False):
        """fused: owners evaluate with the persistent kernel k_batch (GUB_PATH=fused) instead of the pipeline in ring mode."""
        self.world = world
        self.fused = bool(fused)
        self.capacity_slots = int(capacity_slots)
        self._L = lib()
        self._finish_cap = finish_cap
        pts, peers = np.ascontiguousarray(pts, dtype=np.uint64), np.ascontiguousarray(peers, dtype=np.int32)
        self._h = self._L.emu_p2p_create(world, cap, int(capacity_slots), int(max_batch), pts.ctypes.data, peers.ctypes.data, len(pts))

    def step(self, batches, clk, resp_dtype, global_mode=False):
        """batches: one request array per shard (what that shard ingests); returns one response array per shard.  global_mode (after
        gub_p2p_enable_global): GLOBAL requests a shard does not own stay with it; also returns every request's ring owner."""
        batches = [np.ascontiguousarray(b) for b in batches]
        outs = [np.zeros(max(len(b), 1), dtype=resp_dtype) for b in batches]
        owners = [np.zeros(max(len(b), 1), dtype=np.uint8) for b in batches]
        rp = (C.c_void_p * self.world)(*[b.ctypes.data if len(b) else None for b in batches])
        op = (C.c_void_p * self.world)(*[o.ctypes.data for o in outs])
        wp = (C.c_void_p * self.world)(*[o.ctypes.data for o in owners])
        n = np.array([len(b) for b in batches], dtype=np.uint32)
        self._L.emu_set_finish_cap(self._finish_cap)
        self._L.emu_set_fused(1 if self.fused else 0)
        try:
            rc = self._L.emu_p2p_step(self._h, rp, n.ctypes.data, clk.ctypes.data, op, 1 if global_mode else 0, wp if global_mode else None)
        finally:
            self._L.emu_set_finish_cap(132)
            self._L.emu_set_fused(0)
        assert rc == 0, "a mailbox flag wait timed out"
        res = [o[:len(b)] for o, b in zip(outs, batches)]
        return (res, [o[:len(b)] for o, b in zip(owners, batches)]) if global_mode else res

    def table(self, rank):
        """The shard's table as an EmuTable-like handle (submit / scan on it go through the single-table path)."""
        t = EmuTable.__new__(EmuTable)
        t._L, t._h, t.fused, t._owned, t.capacity = self._L, self._L.emu_p2p_table(self._h, rank), self.fused, False, self.capacity_slots
        return t

    def install(self, rank, items, now_ms):
        items = np.ascontiguousarray(items)
        self._L.emu_install_updates(self._L.emu_p2p_table(self._h, rank), items.ctypes.data if len(items) else None, len(items), int(now_ms))


class EmuGq:
    """gub_gq_* (the GLOBAL manager's hits / updates queues) over the emulated kernels."""

    def __init__(self, capacity=1 << 12, keep_latest=False):
        self._L = lib()
        self._h = self._L.emu_gq_create(int(capacity), 1 if keep_latest else 0)

    def accumulate(self, reqs, owner, self_index, seq_base):
        reqs = np.ascontiguousarray(reqs)
        op = None
        if owner is not None:
            owner = np.ascontiguousarray(owner, dtype=np.uint8)
            op = owner.ctypes.data
        self._L.emu_gq_accumulate(self._h, reqs.ctypes.data, len(reqs), op, int(self_index), int(seq_base))

    def drain(self, req_dtype, as_status_query, cap=1 << 12):
        out = np.zeros(cap, dtype=req_dtype)
        n = self._L.emu_gq_drain(self._h, out.ctypes.data, cap, 1 if as_status_query else 0)
        return out[:n]


def make_updates(queries, resps, item_dtype):
    out = np.zeros(max(len(queries), 1), dtype=item_dtype)
    queries, resps = np.ascontiguousarray(queries), np.ascontiguousarray(resps)
    n = lib().emu_make_updates(queries.ctypes.data, resps.ctypes.data, len(queries), out.ctypes.data)
    return out[:n]
