"""ctypes binding of libgubernator_b200.so (include/gubernator_b200.h).  No fallbacks: a missing library is an error."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# GUB_LIB=<path>: load an experimental build variant instead (gubernator_b200.build.build(out=..., defines=...)); unset = the product library
LIB_PATH = os.environ.get("GUB_LIB") or os.path.join(_HERE, "libgubernator_b200.so")

TOKEN_BUCKET, LEAKY_BUCKET = 0, 1
UNDER_LIMIT, OVER_LIMIT = 0, 1
NO_BATCHING, GLOBAL, DURATION_IS_GREGORIAN, RESET_REMAINING, MULTI_REGION, DRAIN_OVER_LIMIT = 1, 2, 4, 8, 16, 32
REQ_IS_OWNER = 0x100
ERR_UNIQUE_KEY_EMPTY, ERR_NAMESPACE_EMPTY, ERR_INVALID_ALGORITHM, ERR_GREGORIAN_WEEKS, ERR_GREGORIAN_INVALID, ERR_TABLE_FULL, ERR_PEER_TIMEOUT = 1, 2, 3, 4, 5, 6, 7

REQ_DTYPE = np.dtype([("key_xxh64", "<u8"), ("key_fnv1", "<u8"), ("hits", "<i8"), ("limit", "<i8"), ("duration", "<i8"),
                      ("burst", "<i8"), ("created_at", "<i8"), ("algorithm", "<u4"), ("behavior", "<u4")])
RESP_DTYPE = np.dtype([("status", "<u4"), ("err_code", "<u4"), ("limit", "<i8"), ("remaining", "<i8"), ("reset_time", "<i8")])
CLOCK_DTYPE = np.dtype([("now_ms", "<i8"), ("greg_expire", "<i8", (6,)), ("greg_duration", "<i8", (6,))])
ITEM_DTYPE = np.dtype([("key_xxh64", "<u8"), ("key_fnv1", "<u8"), ("algorithm", "<i4"), ("status", "<i4"), ("limit", "<i8"),
                       ("duration", "<i8"), ("remaining", "<i8"), ("remaining_f", "<f8"), ("stamp", "<i8"), ("burst", "<i8"),
                       ("expire_at", "<i8"), ("invalid_at", "<i8")])
COUNTER_FIELDS = ("over_limit", "cache_hit", "cache_miss", "inserts", "table_full", "requests", "batches", "dup_groups",
                  "mixed_groups", "serial_fallbacks", "unexpired_evictions", "swept", "gq_dropped")
CREQ_DTYPE = np.dtype([("key_xxh64", "<u8"), ("key_fnv1", "<u8"), ("hits", "<i8"), ("params", "<u4"), ("created_delta", "<i4")])
PARAMS_DTYPE = np.dtype([("limit", "<i8"), ("duration", "<i8"), ("burst", "<i8"), ("algorithm", "<u4"), ("behavior", "<u4")])
assert CREQ_DTYPE.itemsize == 32 and PARAMS_DTYPE.itemsize == 32
assert REQ_DTYPE.itemsize == 64 and RESP_DTYPE.itemsize == 32 and CLOCK_DTYPE.itemsize == 104 and ITEM_DTYPE.itemsize == 88
STORE_FOUND, STORE_REMOVE, STORE_CHANGE = 1, 2, 4
STORE_REC_DTYPE = np.dtype([("first", "<u4"), ("last", "<u4"), ("flags", "<u4"), ("first_shard", "<u2"), ("last_shard", "<u2"),
                            ("item", ITEM_DTYPE)])  # gub_store_rec
assert STORE_REC_DTYPE.itemsize == 104
# gub_store_get_fn: (user, misses, n) -> 0 = ok
STORE_GET_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_size_t)


def _store_get_fn(get):
    """A STORE_GET_FN over get(misses) -> None | int (misses: a STORE_REC_DTYPE view of the library's miss list, valid during the call)."""
    if get is None:
        return STORE_GET_FN()

    def _get(_user, misses_ptr, m):
        return int(get(np.frombuffer((C.c_char * (m * STORE_REC_DTYPE.itemsize)).from_address(misses_ptr), dtype=STORE_REC_DTYPE)) or 0)
    return STORE_GET_FN(_get)


EXPORTS = ["gub_create", "gub_destroy", "gub_last_error", "gub_abi_version", "gub_submit", "gub_submit_device", "gub_submit_device_n", "gub_submit_compact", "gub_submit_compact_async",
           "gub_pipeline_depth", "gub_submit_async", "gub_wait", "gub_host_alloc", "gub_host_free", "gub_clock_fill",
           "gub_add_items", "gub_get_items", "gub_scan", "gub_size", "gub_sweep", "gub_get_counters", "gub_probe_random_access", "gub_set_profiling", "gub_get_profile", "gub_hash_keys", "gub_hash_keys_device",
           "gub_xxh64", "gub_fnv1_64", "gub_fnv1a_64", "gub_ring_create", "gub_ring_destroy", "gub_ring_add", "gub_ring_size",
           "gub_ring_get", "gub_ring_get_by_hash", "gub_ring_points", "gub_route_device", "gub_unroute_device", "gub_gq_create",
           "gub_gq_destroy", "gub_gq_accumulate_device", "gub_gq_drain_device", "gub_make_updates_device", "gub_add_items_device",
           "gub_route_owner_device", "gub_route_global_device", "gub_p2p_create", "gub_p2p_destroy", "gub_p2p_export", "gub_p2p_connect",
           "gub_p2p_connect_local", "gub_p2p_step", "gub_p2p_step_streams", "gub_p2p_status", "gub_p2p_enable_global", "gub_nccl_unique_id",
           "gub_p2p_nccl_init", "gub_p2p_nccl_init_local", "gub_global_tick", "gub_gq_dropped", "gub_set_sweep", "gub_set_trace", "gub_get_trace", "gub_get_trace_raw", "gub_get_ktrace", "gub_keys_layout", "gub_submit_keys_async", "gub_global_tick_local_all", "gub_p2p_step_local_all",
           "gub_p2p_step_keys", "gub_p2p_step_keys_local_all", "gub_p2p_step_mixed_local_all",
           "gub_submit_keys_store_async", "gub_p2p_step_keys_store_local_all", "gub_proto_layout", "gub_submit_proto_async",
           "gub_p2p_step_proto_local_all"]


class Config(C.Structure):
    _fields_ = [("capacity_slots", C.c_uint64), ("max_batch", C.c_uint32), ("device", C.c_int32)]


class GubError(RuntimeError):
    pass


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise GubError(f"{LIB_PATH} is missing: build it with `python -m gubernator_b200.build` (there is no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        vp, u64, i64, sz, i32 = C.c_void_p, C.c_uint64, C.c_int64, C.c_size_t, C.c_int
        L.gub_create.argtypes = [C.POINTER(Config), C.POINTER(vp)]
        L.gub_destroy.argtypes = [vp]; L.gub_destroy.restype = None
        L.gub_last_error.restype = C.c_char_p
        L.gub_submit.argtypes = [vp, vp, sz, vp, vp]
        L.gub_submit_device.argtypes = [vp, vp, sz, vp, vp, vp]
        L.gub_submit_device_n.argtypes = [vp, vp, sz, vp, vp, vp, vp]
        L.gub_submit_compact.argtypes = [vp, vp, sz, vp, sz, i64, vp, vp]
        L.gub_submit_compact_async.argtypes = [vp, vp, sz, vp, sz, i64, vp, vp, C.POINTER(i32)]
        L.gub_pipeline_depth.argtypes = [vp]
        L.gub_submit_async.argtypes = [vp, vp, sz, vp, vp, C.POINTER(i32)]
        L.gub_wait.argtypes = [vp, i32]
        L.gub_host_alloc.argtypes = [sz]; L.gub_host_alloc.restype = vp
        L.gub_host_free.argtypes = [vp]; L.gub_host_free.restype = None
        L.gub_clock_fill.argtypes = [i64, vp]
        L.gub_add_items.argtypes = [vp, vp, sz]
        L.gub_get_items.argtypes = [vp, vp, vp, sz, i64, vp, vp]
        L.gub_scan.argtypes = [vp, vp, sz, C.POINTER(sz)]
        L.gub_size.argtypes = [vp, C.POINTER(sz)]
        L.gub_sweep.argtypes = [vp, i64, C.POINTER(sz)]
        L.gub_get_counters.argtypes = [vp, vp]
        L.gub_set_profiling.argtypes = [vp, i32]
        L.gub_get_profile.argtypes = [vp, vp, vp, i32]
        L.gub_hash_keys.argtypes = [vp, vp, sz, vp, vp]
        L.gub_hash_keys_device.argtypes = [vp, vp, vp, sz, vp, vp, vp, vp]
        L.gub_xxh64.argtypes = [C.c_char_p, sz, u64]; L.gub_xxh64.restype = u64
        L.gub_fnv1_64.argtypes = [C.c_char_p, sz]; L.gub_fnv1_64.restype = u64
        L.gub_fnv1a_64.argtypes = [C.c_char_p, sz]; L.gub_fnv1a_64.restype = u64
        L.gub_ring_create.argtypes = [i32, i32]; L.gub_ring_create.restype = vp
        L.gub_ring_destroy.argtypes = [vp]; L.gub_ring_destroy.restype = None
        L.gub_ring_add.argtypes = [vp, C.c_char_p]
        L.gub_ring_size.argtypes = [vp]
        L.gub_ring_get.argtypes = [vp, C.c_char_p, sz]
        L.gub_ring_get_by_hash.argtypes = [vp, u64]
        L.gub_ring_points.argtypes = [vp, vp, vp, sz]; L.gub_ring_points.restype = sz
        L.gub_route_device.argtypes = [vp, vp, vp, sz, vp, vp, vp, vp]
        L.gub_unroute_device.argtypes = [vp, vp, vp, sz, vp, vp]
        L.gub_gq_create.argtypes = [i32, C.c_uint32, i32, C.POINTER(vp)]
        L.gub_gq_destroy.argtypes = [vp]; L.gub_gq_destroy.restype = None
        L.gub_gq_accumulate_device.argtypes = [vp, vp, sz, vp, C.c_uint32, u64, vp]
        L.gub_gq_drain_device.argtypes = [vp, vp, sz, vp, i32, vp]
        L.gub_make_updates_device.argtypes = [vp, vp, vp, sz, vp, vp, vp]
        L.gub_add_items_device.argtypes = [vp, vp, sz, i64, vp]
        L.gub_route_owner_device.argtypes = [vp, vp, vp, sz, vp, vp]
        L.gub_route_global_device.argtypes = [vp, vp, C.c_uint32, vp, sz, vp, vp, vp, vp, vp]
        L.gub_p2p_create.argtypes = [vp, vp, C.c_uint32, C.c_uint32, C.POINTER(vp)]
        L.gub_p2p_destroy.argtypes = [vp]; L.gub_p2p_destroy.restype = None
        L.gub_p2p_export.argtypes = [vp, vp]
        L.gub_p2p_connect.argtypes = [vp, vp]
        L.gub_p2p_connect_local.argtypes = [vp, C.POINTER(vp)]
        L.gub_p2p_step.argtypes = [vp, vp, sz, vp, vp, vp]
        L.gub_probe_random_access.argtypes = [vp, C.c_uint64, C.POINTER(C.c_double)]
        L.gub_p2p_step_streams.argtypes = [vp, vp, sz, vp, vp, vp, vp]
        L.gub_p2p_status.argtypes = [vp, C.POINTER(C.c_int)]
        L.gub_p2p_enable_global.argtypes = [vp, C.c_uint32]
        L.gub_nccl_unique_id.argtypes = [vp]
        L.gub_p2p_nccl_init.argtypes = [vp, vp]
        L.gub_p2p_nccl_init_local.argtypes = [C.POINTER(vp), C.c_uint32]
        L.gub_global_tick.argtypes = [vp, vp, i64, vp, vp]
        L.gub_p2p_step_local_all.argtypes = [C.POINTER(vp), C.c_uint32, C.POINTER(vp), C.POINTER(sz), vp, C.POINTER(vp), C.POINTER(vp)]
        L.gub_global_tick_local_all.argtypes = [C.POINTER(vp), C.c_uint32, vp, i64, C.POINTER(vp), vp]
        L.gub_gq_dropped.argtypes = [vp, C.POINTER(u64)]
        L.gub_set_sweep.argtypes = [vp, C.c_uint32]
        L.gub_set_trace.argtypes = [vp, i32]
        L.gub_get_trace.argtypes = [vp, vp, vp]
        L.gub_get_trace_raw.argtypes = [vp, vp]
        L.gub_get_ktrace.argtypes = [vp, vp, i32]
        L.gub_submit_keys_async.argtypes = [vp, vp, sz, sz, vp, sz, i64, vp, vp, C.POINTER(C.c_int)]
        L.gub_keys_layout.argtypes = [sz, sz, C.POINTER(sz), C.POINTER(sz), C.POINTER(sz)]
        _lib = L
    return _lib


_vp, _sz, _pvp, _psz = C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)
# The ring's key-string entries are bound when first called, so that a library built without them (the CPU emulation of the C ABI
# that the host-layer tests load) still loads; calling one that a library lacks raises.
_LATE_ARGTYPES = {
    "gub_p2p_step_keys": [_vp, _vp, _sz, _sz, _vp, _sz, C.c_int64, _vp, _vp, _vp, _vp],
    "gub_p2p_step_keys_local_all": [_pvp, C.c_uint32, _pvp, _psz, _psz, _vp, _sz, C.c_int64, _vp, _pvp, _pvp],
    "gub_p2p_step_mixed_local_all": [_pvp, C.c_uint32, _pvp, _pvp, _psz, _psz, _vp, _sz, C.c_int64, _vp, _pvp, _pvp],
    "gub_submit_keys_store_async": [_vp, _vp, _sz, _sz, _vp, _sz, C.c_int64, _vp, STORE_GET_FN, _vp, _vp, _vp, _vp, C.POINTER(C.c_int)],
    "gub_p2p_step_keys_store_local_all": [_pvp, C.c_uint32, _pvp, _psz, _psz, _vp, _sz, C.c_int64, _vp, STORE_GET_FN, _vp, _pvp, _pvp, _pvp, _pvp],
    "gub_proto_layout": [_sz, _sz, _psz, _psz, _psz, _psz],
    "gub_submit_proto_async": [_vp, _vp, _sz, _sz, _vp, _vp, _sz, _vp, _vp, C.POINTER(C.c_int)],
    "gub_p2p_step_proto_local_all": [_pvp, C.c_uint32, _pvp, _psz, _psz, C.c_int, _vp, _pvp, _psz, _pvp, _pvp, _pvp],
}


def _entry(name):
    fn = getattr(lib(), name)
    if fn.argtypes is None:
        fn.argtypes = _LATE_ARGTYPES[name]
    return fn


def _check(rc, what):
    if rc != 0:
        raise GubError(f"{what}: {lib().gub_last_error().decode()}")


def xxh64(b: bytes, seed=0):
    return lib().gub_xxh64(b, len(b), seed)


def fnv1_64(b: bytes):
    return lib().gub_fnv1_64(b, len(b))


def fnv1a_64(b: bytes):
    return lib().gub_fnv1a_64(b, len(b))


def hash_keys(keys):
    """keys: list of bytes -> (xxh64 array, fnv1 array); one library call over the packed bytes."""
    n = len(keys)
    offs = np.zeros(n + 1, dtype=np.uint64)
    if n:
        offs[1:] = np.cumsum([len(k) for k in keys])
    blob = b"".join(keys)
    xx = np.zeros(n, dtype=np.uint64)
    fv = np.zeros(n, dtype=np.uint64)
    buf = C.create_string_buffer(blob, len(blob) + 1)
    _check(lib().gub_hash_keys(C.addressof(buf), offs.ctypes.data, n, xx.ctypes.data, fv.ctypes.data), "gub_hash_keys")
    return xx, fv


def compact_batch(reqs: np.ndarray):
    """gub_req records -> (gub_creq records, gub_params table, created_base): what a shim that knows its limit
    configurations fills directly.  created_base is the smallest created_at (deltas must fit int32)."""
    cfg = np.zeros(len(reqs), dtype=PARAMS_DTYPE)
    for f in ("limit", "duration", "burst", "algorithm", "behavior"):
        cfg[f] = reqs[f]
    params, inv = np.unique(cfg, return_inverse=True)
    base = int(reqs["created_at"].min()) if len(reqs) else 0
    delta = reqs["created_at"] - base
    if len(reqs) and (delta.max() > 0x7FFFFFFF):
        raise ValueError("created_at spread does not fit the compact record")
    c = np.zeros(len(reqs), dtype=CREQ_DTYPE)
    c["key_xxh64"], c["key_fnv1"], c["hits"] = reqs["key_xxh64"], reqs["key_fnv1"], reqs["hits"]
    c["params"] = inv.astype(np.uint32).reshape(-1)
    c["created_delta"] = delta.astype(np.int32)
    return c, np.ascontiguousarray(params), base


def clock_fill(now_ms):
    clk = np.zeros(1, dtype=CLOCK_DTYPE)
    _check(lib().gub_clock_fill(int(now_ms), clk.ctypes.data), "gub_clock_fill")
    return clk


Clock = clock_fill


class PinnedArray:
    """numpy view over page-locked memory from gub_host_alloc."""

    def __init__(self, n, dtype):
        self.nbytes = int(n) * np.dtype(dtype).itemsize
        self.ptr = lib().gub_host_alloc(max(self.nbytes, 64))
        if not self.ptr:
            raise GubError("gub_host_alloc failed")
        buf = (C.c_char * max(self.nbytes, 64)).from_address(self.ptr)
        self.array = np.frombuffer(buf, dtype=dtype, count=int(n))

    def free(self):
        if self.ptr:
            self.array = None
            lib().gub_host_free(self.ptr)
            self.ptr = None


class Table:
    """One GPU's shard: the device-resident bucket table + batch evaluation (WorkerPool replacement)."""

    def __init__(self, capacity_slots, max_batch=65536, device=0):
        cfg = Config(int(capacity_slots), int(max_batch), int(device))
        h = C.c_void_p()
        _check(lib().gub_create(C.byref(cfg), C.byref(h)), "gub_create")
        self._h = h
        self.device = device
        self.capacity = int(capacity_slots)

    def close(self):
        if getattr(self, "_h", None):
            lib().gub_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- hot path
    def submit(self, reqs: np.ndarray, clk: np.ndarray, out: np.ndarray = None):
        assert reqs.dtype == REQ_DTYPE and reqs.flags.c_contiguous
        if out is None:
            out = np.zeros(len(reqs), dtype=RESP_DTYPE)
        _check(lib().gub_submit(self._h, reqs.ctypes.data, len(reqs), clk.ctypes.data, out.ctypes.data), "gub_submit")
        return out

    def submit_async(self, reqs_ptr, n, clk: np.ndarray, out_ptr):
        ticket = C.c_int(-1)
        _check(lib().gub_submit_async(self._h, reqs_ptr, n, clk.ctypes.data, out_ptr, C.byref(ticket)), "gub_submit_async")
        return ticket.value

    def wait(self, ticket):
        _check(lib().gub_wait(self._h, ticket), "gub_wait")

    def submit_compact(self, creqs: np.ndarray, params: np.ndarray, created_base, clk: np.ndarray, out: np.ndarray = None):
        assert creqs.dtype == CREQ_DTYPE and params.dtype == PARAMS_DTYPE and creqs.flags.c_contiguous and params.flags.c_contiguous
        if out is None:
            out = np.zeros(len(creqs), dtype=RESP_DTYPE)
        _check(lib().gub_submit_compact(self._h, creqs.ctypes.data, len(creqs), params.ctypes.data, len(params), int(created_base),
                                        clk.ctypes.data, out.ctypes.data), "gub_submit_compact")
        return out

    def submit_compact_async(self, creqs_ptr, n, params_ptr, n_params, created_base, clk: np.ndarray, out_ptr):
        ticket = C.c_int(-1)
        _check(lib().gub_submit_compact_async(self._h, creqs_ptr, n, params_ptr, n_params, int(created_base), clk.ctypes.data, out_ptr,
                                              C.byref(ticket)), "gub_submit_compact_async")
        return ticket.value

    def probe_random_access(self, accesses=1 << 26):
        """GB/s of random 64-byte read-modify-write over this table's slots (contents unchanged); synchronises the device."""
        gbs = C.c_double(0.0)
        _check(lib().gub_probe_random_access(self._h, int(accesses), C.byref(gbs)), "gub_probe_random_access")
        return gbs.value

    def submit_device(self, d_reqs_ptr, n, clk: np.ndarray, d_out_ptr, stream=0):
        _check(lib().gub_submit_device(self._h, d_reqs_ptr, n, clk.ctypes.data, d_out_ptr, stream), "gub_submit_device")

    # ---- maintenance
    def add_items(self, items: np.ndarray):
        assert items.dtype == ITEM_DTYPE and items.flags.c_contiguous
        _check(lib().gub_add_items(self._h, items.ctypes.data, len(items)), "gub_add_items")

    def get_items(self, key_xxh64, key_fnv1, now_ms):
        kx = np.ascontiguousarray(key_xxh64, dtype=np.uint64)
        kf = np.ascontiguousarray(key_fnv1, dtype=np.uint64)
        out = np.zeros(len(kx), dtype=ITEM_DTYPE)
        found = np.zeros(len(kx), dtype=np.uint8)
        _check(lib().gub_get_items(self._h, kx.ctypes.data, kf.ctypes.data, len(kx), int(now_ms), out.ctypes.data, found.ctypes.data), "gub_get_items")
        return out, found.astype(bool)

    def size(self):
        n = C.c_size_t(0)
        _check(lib().gub_size(self._h, C.byref(n)), "gub_size")
        return n.value

    def scan(self):
        n = self.size()
        out = np.zeros(max(n, 1), dtype=ITEM_DTYPE)
        m = C.c_size_t(0)
        _check(lib().gub_scan(self._h, out.ctypes.data, len(out), C.byref(m)), "gub_scan")
        return out[:min(m.value, len(out))]

    def sweep(self, now_ms):
        n = C.c_size_t(0)
        _check(lib().gub_sweep(self._h, int(now_ms), C.byref(n)), "gub_sweep")
        return n.value

    def counters(self):
        c = np.zeros(len(COUNTER_FIELDS), dtype=np.uint64)
        _check(lib().gub_get_counters(self._h, c.ctypes.data), "gub_get_counters")
        return {k: int(v) for k, v in zip(COUNTER_FIELDS, c)}

    def hash_keys_device(self, d_bytes_ptr, d_offsets_ptr, n, d_xxh_ptr, d_fnv_ptr, d_reqs_ptr=None, stream=0):
        _check(lib().gub_hash_keys_device(self._h, d_bytes_ptr, d_offsets_ptr, n, d_xxh_ptr, d_fnv_ptr, d_reqs_ptr, stream), "gub_hash_keys_device")

    def submit_keys_async(self, packed_ptr, packed_bytes, n, params_ptr, n_params, created_base, clk, out_ptr):
        """Key strings in (packed: see pack_keys), responses out; hashing runs on the device.  Returns a ticket for wait()."""
        tk = C.c_int(-1)
        _check(lib().gub_submit_keys_async(self._h, packed_ptr, packed_bytes, n, params_ptr, n_params, int(created_base), clk.ctypes.data, out_ptr, C.byref(tk)),
               "gub_submit_keys_async")
        return tk.value

    def submit_keys_store_async(self, packed_ptr, packed_bytes, n, params_ptr, n_params, created_base, clk, get, out_ptr, changes_ptr, n_changes_ptr):
        """submit_keys_async with a Store plugin (gub_submit_keys_store_async).  get: None (a store that never reads) or a callable
        get(misses) -> None | int that fills misses["item"] and sets STORE_FOUND in misses["flags"] for the keys the store has (misses:
        a STORE_REC_DTYPE view of the library's miss list, valid during the call only); a non-zero return fails the submission.
        changes_ptr (room for n STORE_REC_DTYPE records) and n_changes_ptr (uint32) must be page-locked (PinnedArray); after wait(),
        they hold one record per key with STORE_REMOVE and/or STORE_CHANGE, ordered by `first`.  Returns a ticket for wait()."""
        cb = _store_get_fn(get)
        tk = C.c_int(-1)
        _check(_entry("gub_submit_keys_store_async")(self._h, packed_ptr, packed_bytes, n, params_ptr, n_params, int(created_base), clk.ctypes.data,
                                                     cb, None, out_ptr, changes_ptr, n_changes_ptr, C.byref(tk)),
               "gub_submit_keys_store_async")
        return tk.value

    def submit_proto_async(self, packed_ptr, packed_bytes, n_msgs, clk, out_ptr, out_cap, out_off_ptr, status_ptr):
        """GetRateLimitsReq wire bytes in (packed: see pack_proto), GetRateLimitsResp wire bytes out (gub_submit_proto_async).  out_ptr
        (out_cap bytes, at least pack_proto's bound), out_off_ptr (n_msgs + 1 uint64) and status_ptr (n_msgs uint32) must be page-locked
        (PinnedArray).  After wait(): message m's response is out[out_off[m]:out_off[m + 1]], its status PROTO_OK / PROTO_TOO_LARGE /
        PROTO_MALFORMED.  Returns a ticket for wait()."""
        tk = C.c_int(-1)
        _check(_entry("gub_submit_proto_async")(self._h, packed_ptr, packed_bytes, n_msgs, clk.ctypes.data, out_ptr, out_cap, out_off_ptr, status_ptr,
                                            C.byref(tk)), "gub_submit_proto_async")
        return tk.value

    def set_sweep(self, slots_per_cta):
        _check(lib().gub_set_sweep(self._h, int(slots_per_cta)), "gub_set_sweep")

    def set_trace(self, on):
        _check(lib().gub_set_trace(self._h, 1 if on else 0), "gub_set_trace")

    TRACE_MARKS = ("entry", "tile_issued", "tile_landed", "phase1_done", "barrier_passed", "probe_done", "entries_read", "evaluated",
                   "checked_in", "uniform_finished", "mixed_finished", "counters_flushed")

    def get_trace(self):
        mx, mean = np.zeros(12), np.zeros(12)
        _check(lib().gub_get_trace(self._h, mx.ctypes.data, mean.ctypes.data), "gub_get_trace")
        return {"max_us": dict(zip(self.TRACE_MARKS, (round(float(v), 2) for v in mx))), "mean_us": dict(zip(self.TRACE_MARKS, (round(float(v), 2) for v in mean)))}

    def get_trace_raw(self):
        raw = np.zeros((256, 12), dtype=np.uint64)
        _check(lib().gub_get_trace_raw(self._h, raw.ctypes.data), "gub_get_trace_raw")
        return raw

    def get_ktrace(self, reset=True):
        """Pipeline kernels' time stamps [kernel 0..3][block][mark 0..7] in ns (0 = never), see gub_get_ktrace."""
        raw = np.zeros((4, 1024, 8), dtype=np.uint64)
        _check(lib().gub_get_ktrace(self._h, raw.ctypes.data, 1 if reset else 0), "gub_get_ktrace")
        return raw

    def set_profiling(self, on):
        _check(lib().gub_set_profiling(self._h, 1 if on else 0), "gub_set_profiling")

    def get_profile(self, reset=True):
        ms = np.zeros(4, dtype=np.float64)
        n = C.c_uint64(0)
        _check(lib().gub_get_profile(self._h, ms.ctypes.data, C.byref(n), 1 if reset else 0), "gub_get_profile")
        return dict(k_group_ms=float(ms[0]), k_rank_ms=float(ms[1]), k_eval_ms=float(ms[2]), k_finish_ms=float(ms[3]), launches=int(n.value))

    # ---- multi-GPU routing
    def route_device(self, ring, d_reqs_ptr, n, d_out_reqs_ptr, d_perm_ptr, d_counts_ptr, stream=0):
        _check(lib().gub_route_device(self._h, ring._r, d_reqs_ptr, n, d_out_reqs_ptr, d_perm_ptr, d_counts_ptr, stream), "gub_route_device")

    def route_global_device(self, ring, self_index, d_reqs_ptr, n, d_out_reqs_ptr, d_perm_ptr, d_counts_ptr, d_owner_ptr, stream=0):
        _check(lib().gub_route_global_device(self._h, ring._r, self_index, d_reqs_ptr, n, d_out_reqs_ptr, d_perm_ptr, d_counts_ptr, d_owner_ptr,
                                             stream), "gub_route_global_device")

    def route_owner_device(self, ring, d_reqs_ptr, n, d_owner_ptr, stream=0):
        _check(lib().gub_route_owner_device(self._h, ring._r, d_reqs_ptr, n, d_owner_ptr, stream), "gub_route_owner_device")

    def make_updates_device(self, d_queries_ptr, d_resps_ptr, n, d_items_ptr, d_count_ptr, stream=0):
        _check(lib().gub_make_updates_device(self._h, d_queries_ptr, d_resps_ptr, n, d_items_ptr, d_count_ptr, stream), "gub_make_updates_device")

    def add_items_device(self, d_items_ptr, n, now_ms, stream=0):
        _check(lib().gub_add_items_device(self._h, d_items_ptr, n, int(now_ms), stream), "gub_add_items_device")

    def unroute_device(self, d_resp_in_ptr, d_perm_ptr, n, d_resp_out_ptr, stream=0):
        _check(lib().gub_unroute_device(self._h, d_resp_in_ptr, d_perm_ptr, n, d_resp_out_ptr, stream), "gub_unroute_device")


class P2P:
    """Fused routing over NVLink peer memory (gub_p2p_*): one per shard."""

    def __init__(self, table, ring, rank, cap):
        h = C.c_void_p()
        _check(lib().gub_p2p_create(table._h, ring._r, rank, cap, C.byref(h)), "gub_p2p_create")
        self._h, self.table, self.ring, self.world, self.rank = h, table, ring, ring.size(), rank

    def export(self) -> bytes:
        buf = C.create_string_buffer(64)
        _check(lib().gub_p2p_export(self._h, buf), "gub_p2p_export")
        return buf.raw

    def connect(self, handles):
        """handles: list of `world` 64-byte handles in rank order (from other processes)."""
        blob = C.create_string_buffer(b"".join(handles), 64 * self.world)
        _check(lib().gub_p2p_connect(self._h, blob), "gub_p2p_connect")

    def connect_local(self, peers):
        arr = (C.c_void_p * self.world)(*[p._h for p in peers])
        _check(lib().gub_p2p_connect_local(self._h, arr), "gub_p2p_connect_local")

    def step(self, d_reqs_ptr, n, clk, d_out_ptr, stream=0, ingest_stream=None):
        if ingest_stream is None:
            _check(lib().gub_p2p_step(self._h, d_reqs_ptr, n, clk.ctypes.data, d_out_ptr, stream), "gub_p2p_step")
        else:
            _check(lib().gub_p2p_step_streams(self._h, d_reqs_ptr, n, clk.ctypes.data, d_out_ptr, ingest_stream, stream), "gub_p2p_step_streams")

    def step_keys(self, d_packed_ptr, packed_bytes, n, params, created_base, clk, d_out_ptr, stream=0, ingest_stream=None):
        """One step fed with key strings (gub_p2p_step_keys): d_packed_ptr = a pack_keys() buffer on this shard's device, params = the
        PARAMS_DTYPE table (host).  ingest_stream None: one stream for the whole step."""
        params = _params_array(params)
        _check(_entry("gub_p2p_step_keys")(self._h, d_packed_ptr, packed_bytes, n, params.ctypes.data if len(params) else None, len(params), int(created_base),
                                       clk.ctypes.data, d_out_ptr, stream if ingest_stream is None else ingest_stream, stream), "gub_p2p_step_keys")

    def status(self):
        """Raises when a bounded device-side wait of an earlier step gave up (a shard of the ring is not answering)."""
        e = C.c_int(0)
        _check(lib().gub_p2p_status(self._h, C.byref(e)), "gub_p2p_status")
        return e.value

    def enable_global(self, capacity=1 << 16):
        _check(lib().gub_p2p_enable_global(self._h, int(capacity)), "gub_p2p_enable_global")

    def nccl_init(self, unique_id: bytes):
        _check(lib().gub_p2p_nccl_init(self._h, C.create_string_buffer(unique_id, 128)), "gub_p2p_nccl_init")

    def tick(self, clk, now_ms, stream=0):
        """One GLOBAL sync (gub_global_tick).  Returns dict(hits_sent, updates_made, installed, gathered_bytes)."""
        st = (C.c_uint64 * 4)()
        _check(lib().gub_global_tick(self._h, clk.ctypes.data, int(now_ms), stream, st), "gub_global_tick")
        return dict(hits_sent=int(st[0]), updates_made=int(st[1]), installed=int(st[2]), gathered_bytes=int(st[3]))

    def close(self):
        if getattr(self, "_h", None):
            lib().gub_p2p_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


KREQ_DTYPE = np.dtype([("hits", "<i8"), ("params", "<u4"), ("created_delta", "<i4")])


def pack_keys(keys, hits, params_idx, created_delta):
    """The one-buffer layout of gub_submit_keys_async: [gub_kreq x n][uint32 offsets x (n + 1)][key bytes] -> np.uint8 array."""
    n = len(keys)
    lens = np.fromiter((len(k) for k in keys), dtype=np.int64, count=n)
    blob = b"".join(keys)
    o_at, b_at, tot = C.c_size_t(), C.c_size_t(), C.c_size_t()
    _check(lib().gub_keys_layout(n, len(blob), C.byref(o_at), C.byref(b_at), C.byref(tot)), "gub_keys_layout")
    buf = np.zeros(tot.value, dtype=np.uint8)
    kr = buf[:n * 16].view(KREQ_DTYPE)
    kr["hits"] = hits; kr["params"] = params_idx; kr["created_delta"] = created_delta
    offs = buf[o_at.value:o_at.value + 4 * (n + 1)].view(np.uint32)
    offs[1:] = np.cumsum(lens)
    buf[b_at.value:b_at.value + len(blob)] = np.frombuffer(blob, dtype=np.uint8)
    return buf


PROTO_OK, PROTO_TOO_LARGE, PROTO_MALFORMED = 0, 1, 2


def proto_layout(n_msgs, msg_bytes):
    """(offsets_at, bytes_at, total, out_bound) of gub_proto_layout."""
    v = [C.c_size_t() for _ in range(4)]
    _check(_entry("gub_proto_layout")(n_msgs, msg_bytes, *[C.byref(x) for x in v]), "gub_proto_layout")
    return tuple(x.value for x in v)


def pack_proto(messages, created_at, out=None):
    """The one-buffer layout of gub_submit_proto_async: [int64 created_at x n][uint32 offsets x (n + 1)][message bytes].  messages: the
    GetRateLimitsReq wire bytes of each RPC; created_at: one default per message (or one for all).  out: an array to pack into (e.g. a
    PinnedArray's view), else a new np.uint8 array.  Returns (buffer, out_bound)."""
    n = len(messages)
    lens = np.fromiter((len(m) for m in messages), dtype=np.int64, count=n)
    blob = b"".join(messages)
    o_at, b_at, tot, bound = proto_layout(n, len(blob))
    buf = np.zeros(tot, dtype=np.uint8) if out is None else out[:tot]
    buf[:o_at].view(np.int64)[:] = created_at
    offs = buf[o_at:o_at + 4 * (n + 1)].view(np.uint32)
    offs[0] = 0
    offs[1:] = np.cumsum(lens)
    buf[b_at:b_at + len(blob)] = np.frombuffer(blob, dtype=np.uint8)
    buf[b_at + len(blob):] = 0
    return buf, bound


def nccl_unique_id() -> bytes:
    buf = C.create_string_buffer(128)
    _check(lib().gub_nccl_unique_id(buf), "gub_nccl_unique_id")
    return buf.raw


def p2p_step_local_all(p2ps, req_ptrs, ns, clk, out_ptrs, streams):
    """One step of every shard of this process from one host thread (gub_p2p_step_local_all)."""
    W = len(p2ps)
    _check(lib().gub_p2p_step_local_all((C.c_void_p * W)(*[p._h for p in p2ps]), W, (C.c_void_p * W)(*req_ptrs), (C.c_size_t * W)(*ns), clk.ctypes.data,
                                        (C.c_void_p * W)(*out_ptrs), (C.c_void_p * W)(*streams)), "gub_p2p_step_local_all")


def _params_array(params):
    params = np.ascontiguousarray(params)
    assert params.dtype == PARAMS_DTYPE
    return params


def p2p_step_keys_local_all(p2ps, packed_ptrs, packed_bytes, ns, params, created_base, clk, out_ptrs, streams):
    """p2p_step_local_all fed with key strings (gub_p2p_step_keys_local_all): packed_ptrs[r] = shard r's pack_keys() buffer on its device."""
    W = len(p2ps)
    params = _params_array(params)
    _check(_entry("gub_p2p_step_keys_local_all")((C.c_void_p * W)(*[p._h for p in p2ps]), W, (C.c_void_p * W)(*packed_ptrs), (C.c_size_t * W)(*packed_bytes),
                                             (C.c_size_t * W)(*ns), params.ctypes.data if len(params) else None, len(params), int(created_base),
                                             clk.ctypes.data, (C.c_void_p * W)(*out_ptrs), (C.c_void_p * W)(*streams)), "gub_p2p_step_keys_local_all")


def p2p_step_proto_local_all(p2ps, packed_ptrs, packed_bytes, n_msgs, clk, out_ptrs, out_caps, out_off_ptrs, status_ptrs, streams,
                             force_global=False):
    """GetRateLimitsReq wire bytes on every shard of this process (gub_p2p_step_proto_local_all): packed_ptrs[r] = shard r's pack_proto()
    buffer (host memory), n_msgs[r] its message count.  out_ptrs[r] (out_caps[r] bytes, at least pack_proto's bound), out_off_ptrs[r]
    (n_msgs[r] + 1 uint64) and status_ptrs[r] (n_msgs[r] uint32) must be page-locked (PinnedArray): shard r's responses, valid once
    streams[r] has completed the call.  force_global: Behaviors.ForceGlobal."""
    W = len(p2ps)
    _check(_entry("gub_p2p_step_proto_local_all")((C.c_void_p * W)(*[p._h for p in p2ps]), W, (C.c_void_p * W)(*packed_ptrs),
                                              (C.c_size_t * W)(*packed_bytes), (C.c_size_t * W)(*n_msgs), 1 if force_global else 0, clk.ctypes.data,
                                              (C.c_void_p * W)(*out_ptrs), (C.c_size_t * W)(*out_caps), (C.c_void_p * W)(*out_off_ptrs),
                                              (C.c_void_p * W)(*status_ptrs), (C.c_void_p * W)(*streams)), "gub_p2p_step_proto_local_all")


def p2p_step_mixed_local_all(p2ps, req_ptrs, packed_ptrs, packed_bytes, ns, params, created_base, clk, out_ptrs, streams):
    """Both kinds of ingest in one step (gub_p2p_step_mixed_local_all): shard r ingests key strings when packed_ptrs[r] is not None,
    else the records at req_ptrs[r]."""
    W = len(p2ps)
    params = _params_array(params)
    _check(_entry("gub_p2p_step_mixed_local_all")((C.c_void_p * W)(*[p._h for p in p2ps]), W, (C.c_void_p * W)(*req_ptrs), (C.c_void_p * W)(*packed_ptrs),
                                              (C.c_size_t * W)(*packed_bytes), (C.c_size_t * W)(*ns), params.ctypes.data if len(params) else None,
                                              len(params), int(created_base), clk.ctypes.data, (C.c_void_p * W)(*out_ptrs), (C.c_void_p * W)(*streams)),
           "gub_p2p_step_mixed_local_all")


def p2p_step_keys_store_local_all(p2ps, packed_ptrs, packed_bytes, ns, params, created_base, clk, get, out_ptrs, changes_ptrs, n_changes_ptrs,
                                  streams):
    """p2p_step_keys_local_all with a Store plugin (gub_p2p_step_keys_store_local_all).  get: None (a store that never reads) or a
    callable get(misses) -> None | int, called once per owner that has misses, in rank order, as for Table.submit_keys_store_async; a
    miss names its request by (first_shard, first).  changes_ptrs[r] (room for world x cap STORE_REC_DTYPE records) and
    n_changes_ptrs[r] (uint32) must be page-locked (PinnedArray): owner r's change log, valid once streams[r] has completed the step."""
    W = len(p2ps)
    params = _params_array(params)
    cb = _store_get_fn(get)
    _check(_entry("gub_p2p_step_keys_store_local_all")((C.c_void_p * W)(*[p._h for p in p2ps]), W, (C.c_void_p * W)(*packed_ptrs),
                                                   (C.c_size_t * W)(*packed_bytes), (C.c_size_t * W)(*ns), params.ctypes.data if len(params) else None,
                                                   len(params), int(created_base), clk.ctypes.data, cb, None, (C.c_void_p * W)(*out_ptrs),
                                                   (C.c_void_p * W)(*changes_ptrs), (C.c_void_p * W)(*n_changes_ptrs), (C.c_void_p * W)(*streams)),
           "gub_p2p_step_keys_store_local_all")


def global_tick_local_all(p2ps, clk, now_ms, streams):
    W = len(p2ps)
    st = (C.c_uint64 * (4 * W))()
    _check(lib().gub_global_tick_local_all((C.c_void_p * W)(*[p._h for p in p2ps]), W, clk.ctypes.data, int(now_ms), (C.c_void_p * W)(*streams), st),
           "gub_global_tick_local_all")
    return [dict(hits_sent=int(st[4 * r]), updates_made=int(st[4 * r + 1]), installed=int(st[4 * r + 2]), gathered_bytes=int(st[4 * r + 3])) for r in range(W)]


def p2p_nccl_init_local(p2ps):
    arr = (C.c_void_p * len(p2ps))(*[p._h for p in p2ps])
    _check(lib().gub_p2p_nccl_init_local(arr, len(p2ps)), "gub_p2p_nccl_init_local")


class GlobalQueue:
    """Device-side hits / updates queue of the GLOBAL manager (global.go:91-231)."""

    def __init__(self, device=0, capacity=1 << 16, keep_latest=False):
        h = C.c_void_p()
        _check(lib().gub_gq_create(int(device), int(capacity), 1 if keep_latest else 0, C.byref(h)), "gub_gq_create")
        self._h = h

    def accumulate_device(self, d_reqs_ptr, n, d_owner_ptr, self_index, seq_base, stream=0):
        _check(lib().gub_gq_accumulate_device(self._h, d_reqs_ptr, n, d_owner_ptr, self_index, int(seq_base), stream), "gub_gq_accumulate_device")

    def drain_device(self, d_out_ptr, cap, d_count_ptr, as_status_query, stream=0):
        _check(lib().gub_gq_drain_device(self._h, d_out_ptr, cap, d_count_ptr, 1 if as_status_query else 0, stream), "gub_gq_drain_device")

    def close(self):
        if getattr(self, "_h", None):
            lib().gub_gq_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Ring:
    """ReplicatedConsistentHash (replicated_hash.go:36-119)."""

    def __init__(self, hash_kind=0, replicas=512):
        self._r = C.c_void_p(lib().gub_ring_create(hash_kind, replicas))
        self.peers = []

    def add(self, addr: str):
        rc = lib().gub_ring_add(self._r, addr.encode())
        if rc < 0:
            raise GubError("gub_ring_add failed")
        self.peers.append(addr)
        return rc

    def size(self):
        return lib().gub_ring_size(self._r)

    def get(self, key: str):
        b = key.encode()
        return lib().gub_ring_get(self._r, b, len(b))

    def get_by_hash(self, h):
        return lib().gub_ring_get_by_hash(self._r, int(h))

    def points(self):
        n = lib().gub_ring_points(self._r, None, None, 0)
        hs = np.zeros(n, dtype=np.uint64)
        ps = np.zeros(n, dtype=np.int32)
        lib().gub_ring_points(self._r, hs.ctypes.data, ps.ctypes.data, n)
        return hs, ps

    def __del__(self):
        try:
            lib().gub_ring_destroy(self._r)
        except Exception:
            pass
