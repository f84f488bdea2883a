"""The ring fed with key strings (k_p2p_route_keys, gub_p2p.cuh) on the CPU emulation of the kernels: hashing, parameter expansion
and routing in one kernel must leave every owner's mailbox, perm and counts byte-identical to k_p2p_route on the same batch hashed
on the host, and answer like the per-shard oracles.  Malformed offsets are clamped to the buffer, which ends at a guard page here,
so an over-read fails the test process instead of passing silently."""
import ctypes as C
import mmap

import numpy as np
import pytest

import oracle_py as O
import _ring_keys_emu as K
from local_ring import per_shard_oracle_results
from workloads import T0, adversarial_batch, bench_key_bytes, make_clock, zipf_ids

PARAM_FIELDS = ("limit", "duration", "burst", "algorithm", "behavior")


@pytest.fixture(scope="module")
def G():
    import gubernator_b200 as g  # dtypes only; nothing here touches CUDA
    return g


def _oring(world):
    from gubernator_b200.sharded import shard_addresses
    oring = O.Ring(0, 512)
    for a in shard_addresses(world):
        oring.add(a)
    return oring


def pack(keys, kreq):
    """[gub_kreq x n][uint32 offsets x (n + 1)][key bytes], padded to 16 bytes (gub_keys_layout)."""
    n = len(keys)
    blob = b"".join(keys)
    bytes_at = n * 16 + (n + 1) * 4
    buf = np.zeros((bytes_at + len(blob) + 15) & ~15, dtype=np.uint8)
    buf[:n * 16] = np.ascontiguousarray(kreq).view(np.uint8)
    offs = buf[n * 16:bytes_at].view(np.uint32)
    offs[1:] = np.cumsum([len(k) for k in keys])
    buf[bytes_at:bytes_at + len(blob)] = np.frombuffer(blob, dtype=np.uint8)
    return buf


def odd_keys(rng, count):
    """Keys of length 0, 1, 31, 32, 33 and 100 (around XXH64's 32-byte stripe), with non-ASCII bytes, plus bench-like ones."""
    fixed = [b"", b"\xff", bytes(range(200, 231)), "ключ_".encode() * 2 + b"x" * 14, b"\x00" * 33, bytes(rng.integers(0, 256, 100, dtype=np.uint8))]
    assert [len(k) for k in fixed] == [0, 1, 31, 32, 33, 100]
    rest = [bytes(r) for r in bench_key_bytes(np.arange(count), prefix=b"keys_tk")]
    return fixed + rest


def key_step(G, batches, n_params, rng, unknown_at=3):
    """One step's (host records, key strings) per shard -> (packed batch per shard, the step's parameter table, created_base, the
    records as the host hashes and expands them).  The table holds at least n_params sets, shuffled; request `unknown_at` of every
    shard gets an index past the table (an unknown set: the in-band error record)."""
    allreq = np.concatenate([b for b, _ in batches])
    cfg = np.zeros(len(allreq), dtype=G.native.PARAMS_DTYPE)
    for f in PARAM_FIELDS:
        cfg[f] = allreq[f]
    uniq, inv = np.unique(cfg, return_inverse=True)
    inv = inv.reshape(-1)
    table = np.zeros(max(n_params, len(uniq)), dtype=G.native.PARAMS_DTYPE)
    table["limit"] = 7 + np.arange(len(table)); table["duration"] = 1000
    order = rng.permutation(len(table))
    table[order[:len(uniq)]] = uniq
    base = int(allreq["created_at"].min()) if len(allreq) else T0
    packed, host, at = [], [], 0
    for reqs, keys in batches:
        n = len(reqs)
        kreq = np.zeros(n, dtype=G.native.KREQ_DTYPE)
        kreq["hits"] = reqs["hits"]
        kreq["params"] = order[inv[at:at + n]]
        kreq["created_delta"] = (reqs["created_at"] - base).astype(np.int32)
        at += n
        h = np.ascontiguousarray(reqs).copy()
        h["key_xxh64"] = [O.xxh64(k) for k in keys]
        h["key_fnv1"] = [O.fnv1_64(k) for k in keys]
        if n > unknown_at:
            kreq["params"][unknown_at] = len(table) + 5
            for f in ("limit", "duration", "burst", "behavior"):
                h[f][unknown_at] = 0
            h["algorithm"][unknown_at] = 0xFFFFFFFF
        packed.append(pack(keys, kreq)); host.append(h)
    return packed, table, base, host


def _batch(G, rng, kind, n, now, keyset):
    if kind == "bench":
        ids = zipf_ids(rng, n, len(keyset), 1.1)
        reqs = np.zeros(n, dtype=O.HREQ_DTYPE)
        reqs["hits"] = 1; reqs["limit"] = 100; reqs["duration"] = 60000; reqs["created_at"] = now
        reqs["algorithm"] = ids & 1; reqs["behavior"] = O.REQ_IS_OWNER
        return reqs, [keyset[int(i)] for i in ids]
    reqs = adversarial_batch(rng, n, 41, now)
    _, key_id = np.unique(reqs["key_xxh64"], return_inverse=True)  # same key, same key string: the per-key structure survives
    return reqs, [keyset[int(i) % len(keyset)] for i in key_id.reshape(-1)]


CASES = [(w, p) for w in (1, 2, 4, 8) for p in ("pipeline", "fused")]


@pytest.mark.parametrize("world,path", CASES)
def test_keys_route_equals_record_route(G, world, path):
    oring = _oring(world)
    pts, peers = oring.points()
    cap = 1536
    kw = dict(cap=cap, capacity_slots=1 << 13, pts=pts, peers=peers, max_batch=2048, finish_cap=3, fused=(path == "fused"))
    keyed, twin = K.KeysP2PCluster(world, **kw), K.KeysP2PCluster(world, **kw)
    sim = [O.Pool(workers=2, cache_size=10**7, now_ms=T0) for _ in range(world)]
    sizes = [1100, 1, 0, 700, 1536, 513, 64, 900]
    for step, (kind, n_params) in enumerate([("bench", 3), ("adversarial", 40)]):
        now = T0 + step
        rng = np.random.default_rng(31 * world + step)
        keyset = odd_keys(rng, 400)
        batches = [_batch(G, rng, kind, sizes[(r + step) % len(sizes)], now, keyset) for r in range(world)]
        packed, table, base, host = key_step(G, batches, n_params, rng)
        assert (len(table) <= 32) == (n_params == 3)
        got = keyed.step_keys(packed, table, base, make_clock(now), O.HRESP_DTYPE, n=[len(h) for h in host])
        want_twin = twin.step([h.astype(G.REQ_DTYPE) for h in host], make_clock(now), O.HRESP_DTYPE)
        for r in range(world):
            a, b = keyed.route_state(r, G.REQ_DTYPE), twin.route_state(r, G.REQ_DTYPE)
            n = len(host[r])
            assert a[0].tobytes() == b[0].tobytes(), f"step {step}: owner {r}'s mailbox differs"
            assert np.array_equal(a[1][:n], b[1][:n]) and np.array_equal(a[2], b[2]), f"step {step} shard {r}: perm / counts differ"
        want = per_shard_oracle_results(oring, sim, host, now)
        for r in range(world):
            assert np.array_equal(got[r], want[r]), f"step {step} shard {r}: {int((got[r] != want[r]).sum())} responses differ from the oracle"
            assert np.array_equal(got[r], want_twin[r])
            if len(host[r]) > 3:
                assert got[r]["err_code"][3] == G.native.ERR_INVALID_ALGORITHM


def test_global_mode_queues_the_expanded_records(G):
    """GLOBAL mode: the keys kernel hands the hits queue the same records (and ring owners) the record path reads."""
    world = 4
    oring = _oring(world)
    pts, peers = oring.points()
    kw = dict(cap=1024, capacity_slots=1 << 13, pts=pts, peers=peers, max_batch=2048, finish_cap=3)
    keyed, twin = K.KeysP2PCluster(world, **kw), K.KeysP2PCluster(world, **kw)
    rng = np.random.default_rng(5)
    keyset = odd_keys(rng, 60)
    packed, host = [], []
    table = None
    for r in range(world):
        ids = rng.integers(0, len(keyset), 800)
        reqs = np.zeros(800, dtype=O.HREQ_DTYPE)
        reqs["hits"] = 1 + (ids % 3); reqs["limit"] = 50; reqs["duration"] = 60000; reqs["created_at"] = T0
        reqs["behavior"] = np.where(ids % 2 == 0, O.GLOBAL, 0).astype(np.uint32) | np.uint32(O.REQ_IS_OWNER)
        keys = [keyset[int(i)] for i in ids]
        cfg = np.zeros(2, dtype=G.native.PARAMS_DTYPE)
        cfg["limit"] = 50; cfg["duration"] = 60000; cfg["behavior"] = [O.REQ_IS_OWNER, O.GLOBAL | O.REQ_IS_OWNER]
        table = cfg
        kreq = np.zeros(800, dtype=G.native.KREQ_DTYPE)
        kreq["hits"] = reqs["hits"]; kreq["params"] = (ids % 2 == 0).astype(np.uint32)
        h = reqs.copy()
        h["key_xxh64"] = [O.xxh64(k) for k in keys]; h["key_fnv1"] = [O.fnv1_64(k) for k in keys]
        packed.append(pack(keys, kreq)); host.append(h)
    got, owners, expanded = keyed.step_keys(packed, table, T0, make_clock(T0), O.HRESP_DTYPE, n=[800] * world, global_mode=True, req_dtype=G.REQ_DTYPE)
    want, want_owners = twin.step([h.astype(G.REQ_DTYPE) for h in host], make_clock(T0), O.HRESP_DTYPE, global_mode=True)
    for r in range(world):
        assert np.array_equal(got[r], want[r]) and np.array_equal(owners[r], want_owners[r])
        assert expanded[r].tobytes() == host[r].astype(G.REQ_DTYPE).tobytes()


class GuardedBuffer:
    """`data` copied to the end of an anonymous mapping whose next page is PROT_NONE: one byte read past the end faults."""

    def __init__(self, data):
        libc = C.CDLL(None, use_errno=True)
        libc.mmap.restype = C.c_void_p
        libc.mmap.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_long]
        libc.mprotect.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
        libc.munmap.argtypes = [C.c_void_p, C.c_size_t]
        self._libc, page = libc, mmap.PAGESIZE
        self.size = (len(data) + page - 1) // page * page + page
        base = libc.mmap(None, self.size, mmap.PROT_READ | mmap.PROT_WRITE, mmap.MAP_PRIVATE | mmap.MAP_ANONYMOUS, -1, 0)
        assert base not in (None, C.c_void_p(-1).value)
        self.base = base
        guard = base + self.size - page
        assert libc.mprotect(guard, page, 0) == 0  # PROT_NONE
        self.ptr = guard - len(data)
        C.memmove(self.ptr, bytes(data), len(data))

    def close(self):
        self._libc.munmap(self.base, self.size)


def test_malformed_offsets_are_clamped_to_the_buffer(G):
    world, n = 2, 600
    oring = _oring(world)
    pts, peers = oring.points()
    cl = K.KeysP2PCluster(world, cap=1024, capacity_slots=1 << 13, pts=pts, peers=peers, max_batch=2048, finish_cap=3)
    rng = np.random.default_rng(11)
    keys = [bytes(rng.integers(0, 256, int(l), dtype=np.uint8)) for l in rng.integers(0, 70, n)]
    kreq = np.zeros(n, dtype=G.native.KREQ_DTYPE)
    kreq["hits"] = 1
    buf = pack(keys, kreq)
    bytes_at = n * 16 + (n + 1) * 4
    key_len = len(buf) - bytes_at                     # the buffer ends right here, at the guard page
    offs = buf[n * 16:bytes_at].view(np.uint32)
    offs[10] = offs[12] + 5                           # decreasing: offsets[10] > offsets[11]
    offs[50] = 0xFFFFFFFF                             # past the buffer (and the next key starts before it)
    offs[51] = key_len + 1
    offs[200:205] = [key_len - 3, key_len + 40, 7, key_len + 1000, key_len]
    offs[n] = key_len + 100000                        # the last key runs past the end
    table = np.zeros(1, dtype=G.native.PARAMS_DTYPE)
    table["limit"] = 10; table["duration"] = 60000
    g = GuardedBuffer(buf.tobytes())
    try:
        got = cl.step_keys([(g.ptr, len(buf)), np.zeros(0, dtype=np.uint8)], table, T0, make_clock(T0), O.HRESP_DTYPE, n=[n, 0])
    finally:
        g.close()
    blob = buf[bytes_at:].tobytes()
    want = np.zeros(n, dtype=O.HREQ_DTYPE)
    for i in range(n):
        hi = min(int(offs[i + 1]), key_len)
        lo = min(int(offs[i]), hi)
        want["key_xxh64"][i], want["key_fnv1"][i] = O.xxh64(blob[lo:hi]), O.fnv1_64(blob[lo:hi])
    want["hits"] = 1; want["limit"] = 10; want["duration"] = 60000; want["created_at"] = T0
    mbs = [cl.route_state(r, G.REQ_DTYPE) for r in range(world)]
    perm = mbs[0][1][:n]
    par = 1  # the first step's mailbox half
    for i in range(n):
        o, pos = int(perm[i]) >> 24, int(perm[i]) & 0xFFFFFF
        rec = mbs[o][0][(par * world + 0) * 1024 + pos]
        assert (int(rec["key_xxh64"]), int(rec["key_fnv1"])) == (int(want["key_xxh64"][i]), int(want["key_fnv1"][i])), i
    sim = [O.Pool(workers=2, cache_size=10**7, now_ms=T0) for _ in range(world)]
    exp = per_shard_oracle_results(oring, sim, [want, np.zeros(0, dtype=O.HREQ_DTYPE)], T0)
    assert np.array_equal(got[0], exp[0])
