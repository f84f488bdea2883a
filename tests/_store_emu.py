"""Builds/loads the TEST-ONLY CPU emulation of the Store plugin's pre- and post-pass around the pipeline (tests/store_emu_harness.cpp: the
kernel emulation of tests/kernel_emu_harness.cpp plus gubernator_b200/csrc/gub_store.cuh, driven like gub_submit_keys_store_async), and
the host layer's Store rule (csrc/host_v1.cpp submit_with_store) restated over the oracle, which both the emulated and the GPU tests
compare with.  Its own library, so the one of tests/_kernel_emu.py is untouched."""
import ctypes as C
import os
import subprocess

import numpy as np

import _kernel_emu as E
import oracle_py as O

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SO = os.path.join(HERE, "libstore_emu_test.so")
SRC = [os.path.join(HERE, "store_emu_harness.cpp"), os.path.join(ROOT, "gubernator_b200", "csrc", "gub_store.cuh")] + E.SRC

STORE_FOUND, STORE_REMOVE, STORE_CHANGE = 1, 2, 4
ITEM_DTYPE = np.dtype([("key_xxh64", "<u8"), ("key_fnv1", "<u8"), ("algorithm", "<i4"), ("status", "<i4"), ("limit", "<i8"),
                       ("duration", "<i8"), ("remaining", "<i8"), ("remaining_f", "<f8"), ("stamp", "<i8"), ("burst", "<i8"),
                       ("expire_at", "<i8"), ("invalid_at", "<i8")])
REC_DTYPE = np.dtype([("first", "<u4"), ("last", "<u4"), ("flags", "<u4"), ("_pad", "<u4"), ("item", ITEM_DTYPE)])
GET_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_size_t)

_libs = {}


def lib():
    if "L" not in _libs:
        if not os.path.exists(SO) or any(os.path.getmtime(s) > os.path.getmtime(SO) for s in SRC):
            subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-msse2", "-ffp-contract=off", "-Wno-unknown-pragmas",
                                   "-Wl,-Bsymbolic", "-I", os.path.join(ROOT, "include"), "-x", "c++", SRC[0], "-o", SO])
        L = C.CDLL(SO)
        vp, u64, u32 = C.c_void_p, C.c_uint64, C.c_uint32
        L.emu_store_create.argtypes = [u64, u32]; L.emu_store_create.restype = vp
        L.emu_store_destroy.argtypes = [vp]; L.emu_store_destroy.restype = None
        L.emu_store_submit.argtypes = [vp, vp, C.c_size_t, vp, GET_FN, vp, vp, vp, vp]
        L.emu_store_set_epoch.argtypes = [vp, u32]; L.emu_store_set_epoch.restype = None
        L.emu_store_epoch.argtypes = [vp]; L.emu_store_epoch.restype = u32
        L.emu_ovf_count.argtypes = [vp]; L.emu_ovf_count.restype = u32
        L.emu_counters.argtypes = [vp, vp]; L.emu_counters.restype = None
        L.emu_scan.argtypes = [vp, vp, u64]; L.emu_scan.restype = u64
        _libs["L"] = L
    return _libs["L"]


class StoreTable(E.EmuTable):
    """E.EmuTable's surface (counters, scan) plus submit_store(): one batch through the Store's pre-pass, the four kernels and the post-pass."""

    def __init__(self, capacity_slots, max_batch=65536):
        self._L = lib()
        self._h = self._L.emu_store_create(int(capacity_slots), int(max_batch))
        self.capacity = int(capacity_slots)
        self.fused = False

    def submit_store(self, reqs, clk, resp_dtype, get):
        """get: None or a callable(misses) -> int, as native.Table.submit_keys_store_async takes it.  Returns (rc, responses, records)."""
        reqs = np.ascontiguousarray(reqs)
        out = np.zeros(len(reqs), dtype=resp_dtype)
        changes = np.zeros(max(len(reqs), 1), dtype=REC_DTYPE)
        n_changes = np.zeros(1, dtype=np.uint32)
        cb = GET_FN()
        if get is not None:
            cb = GET_FN(lambda _u, p, m: int(get(np.frombuffer((C.c_char * (m * REC_DTYPE.itemsize)).from_address(p), dtype=REC_DTYPE)) or 0))
        rc = self._L.emu_store_submit(self._h, reqs.ctypes.data, len(reqs), clk.ctypes.data, cb, None, out.ctypes.data, changes.ctypes.data,
                                      n_changes.ctypes.data)
        return rc, out, changes[:int(n_changes[0])].copy()

    def set_store_epoch(self, e):
        self._L.emu_store_set_epoch(self._h, int(e))

    def store_epoch(self):
        return int(self._L.emu_store_epoch(self._h))

    def ovf_count(self):
        return int(self._L.emu_ovf_count(self._h))

    def __del__(self):
        try:
            self._L.emu_store_destroy(self._h)
        except Exception:
            pass


# ---- the host layer's rule (csrc/host_v1.cpp submit_with_store) over the oracle -------------------------------------------------------
def oracle_to_item(it, kx, kf):
    """An oracle CacheItem as gub_get_items reports it: token buckets carry no burst / float remaining, leaky ones no status / int remaining."""
    r = np.zeros(1, dtype=ITEM_DTYPE)[0]
    leaky = it.value_kind == 2
    r["key_xxh64"], r["key_fnv1"] = kx, kf
    r["algorithm"] = 1 if leaky else 0
    r["status"] = 0 if leaky else it.status
    r["limit"], r["duration"], r["stamp"], r["expire_at"], r["invalid_at"] = it.limit, it.duration, it.stamp, it.expire_at, it.invalid_at
    r["remaining"] = 0 if leaky else it.remaining_i
    r["remaining_f"] = it.remaining_f if leaky else 0.0
    r["burst"] = it.burst if leaky else 0
    return r


def item_to_oracle(r):
    """A gub_item as gub_add_items installs it (to_dev of gub_api.cu), as an oracle CacheItem."""
    it = O.Item()
    leaky = int(r["algorithm"]) == 1
    it.algorithm = int(r["algorithm"]); it.value_kind = 2 if leaky else 1
    it.expire_at = int(r["expire_at"]); it.invalid_at = int(r["invalid_at"])
    it.status = 0 if leaky else int(r["status"]); it.limit = int(r["limit"]); it.duration = int(r["duration"])
    it.remaining_i = 0 if leaky else int(r["remaining"]); it.remaining_f = float(r["remaining_f"]) if leaky else 0.0
    it.stamp = int(r["stamp"]); it.burst = int(r["burst"]) if leaky else 0
    return it


def model_batch(pool, reqs, now, store_items):
    """One batch the way submit_with_store runs it, on the oracle.  store_items: {(kx, kf): ITEM_DTYPE record} (what Store.Get finds).
    Returns (misses, responses, records) with misses / records as REC_DTYPE arrays ordered by `first`."""
    pool.set_now(now)
    first, last, reset = {}, {}, {}
    for j in range(len(reqs)):
        k = (int(reqs["key_xxh64"][j]), int(reqs["key_fnv1"][j]))
        first.setdefault(k, j)
        last[k] = j
        if int(reqs["algorithm"][j]) == 0 and int(reqs["behavior"][j]) & O.RESET_REMAINING:
            reset[k] = True
    keys = sorted(first, key=first.get)
    had, before, misses = {}, {}, []
    for k in keys:
        it = pool.get_item_hashed(*k)
        if it is not None:
            had[k], before[k] = 1, (1 if it.value_kind == 2 else 0)
            continue
        m = np.zeros(1, dtype=REC_DTYPE)[0]
        m["first"], m["last"] = first[k], last[k]
        m["item"]["key_xxh64"], m["item"]["key_fnv1"] = k
        misses.append(m)
        if k in store_items:
            li = store_items[k].copy()
            li["key_xxh64"], li["key_fnv1"] = k
            had[k], before[k] = (2 if int(li["expire_at"]) >= now else 0), int(li["algorithm"])
            if int(li["algorithm"]) in (0, 1):
                pool.add_item_hashed(k[0], k[1], item_to_oracle(li))
    resp = pool.submit_hashed(np.ascontiguousarray(reqs))
    recs = []
    for k in keys:
        jf, jl = first[k], last[k]
        alg = int(reqs["algorithm"][jf])
        flags = 0
        if had.get(k, 0) and ((before[k] != alg and alg <= 1) or reset.get(k, False)):
            flags |= STORE_REMOVE
        after = pool.get_item_hashed(*k)
        if after is not None and int(resp["err_code"][jl]) == 0 and int(reqs["behavior"][jl]) & O.REQ_IS_OWNER:
            flags |= STORE_CHANGE
        if not flags:
            continue
        r = np.zeros(1, dtype=REC_DTYPE)[0]
        r["first"], r["last"], r["flags"] = jf, jl, flags
        r["item"]["key_xxh64"], r["item"]["key_fnv1"] = k
        if flags & STORE_CHANGE:
            r["item"] = oracle_to_item(after, *k)
        recs.append(r)
    return np.array(misses, dtype=REC_DTYPE), resp, np.array(recs, dtype=REC_DTYPE)


def store_item(rng, now, kind):
    """An item a Store could hold: 'token' / 'leaky' (live), 'expired', 'invalid' (past InvalidAt), 'pending' (InvalidAt ahead), 'bad'
    (an algorithm the cache cannot hold)."""
    r = np.zeros(1, dtype=ITEM_DTYPE)[0]
    leaky = kind == "leaky" or (kind not in ("token",) and rng.random() < 0.5)
    r["algorithm"] = 1 if leaky else 0
    r["limit"], r["duration"] = int(rng.choice([5, 10, 100])), int(rng.choice([1000, 60000]))
    r["remaining"] = int(rng.integers(0, 5))
    r["remaining_f"] = float(rng.integers(0, 5)) + (0.5 if leaky else 0.0)
    r["status"] = int(rng.integers(0, 2)) if not leaky else 0
    r["stamp"] = now - int(rng.integers(0, 500))
    r["burst"] = int(r["limit"]) if leaky else 0
    r["expire_at"] = now + int(rng.integers(1, 50000))
    if kind == "expired":
        r["expire_at"] = now - int(rng.integers(1, 1000))
    elif kind == "invalid":
        r["invalid_at"] = now - int(rng.integers(1, 1000))
    elif kind == "pending":
        r["invalid_at"] = now + int(rng.integers(1, 1000))
    elif kind == "bad":
        r["algorithm"] = 5
    return r


def fill_store(rng, reqs, now, frac=0.3, kinds=("token", "leaky", "expired", "invalid", "pending", "bad")):
    """Store items for about `frac` of the batch's keys, of every kind."""
    out = {}
    for kx, kf in set(zip(reqs["key_xxh64"].tolist(), reqs["key_fnv1"].tolist())):
        if rng.random() < frac:
            out[(int(kx), int(kf))] = store_item(rng, now, kinds[int(rng.integers(0, len(kinds)))])
    return out


def found_filler(store_items, calls=None):
    """A Get callback over store_items; `calls` (a list) receives a copy of every miss list it was handed."""
    def get(misses):
        if calls is not None:
            calls.append(misses.copy())
        for m in misses:
            k = (int(m["item"]["key_xxh64"]), int(m["item"]["key_fnv1"]))
            if k in store_items:
                it = store_items[k].copy()
                it["key_xxh64"], it["key_fnv1"] = k
                m["item"] = it
                m["flags"] |= STORE_FOUND
        return 0
    return get
