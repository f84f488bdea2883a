"""The ring fed with key strings through the C ABI (gub_p2p_step_keys_local_all: k_p2p_route_keys hashes, expands and routes in one
launch), checked against one oracle per shard and against a twin ring fed the host-hashed records through gub_p2p_step_local_all:
same responses every step, same table contents at the end.  Well-formed buffers only; clamping of malformed offsets is covered on
the CPU emulator (tests/test_ring_keys_emulated.py)."""
import numpy as np
import pytest

import oracle_py as O
from local_ring import LocalRing, per_shard_oracle_results
from workloads import T0, adversarial_batch, bench_key_bytes, bench_key_hashes, zipf_ids

pytestmark = pytest.mark.gpu

PARAM_FIELDS = ("limit", "duration", "burst", "algorithm", "behavior")
N_KEYS = 3000


@pytest.fixture(autouse=True, params=["pipeline", "fused"])
def owner_kernel_path(request, monkeypatch):
    """Owners evaluate their mailboxes with the four-kernel pipeline in ring mode (default) or with the persistent kernel k_batch
    (GUB_PATH=fused); read when a table is created."""
    monkeypatch.setenv("GUB_PATH", request.param)
    return request.param


def _keyset():
    """Key id -> key string and its hashes: bench-like 16-byte keys, the first few replaced by keys of other lengths (non-ASCII too)."""
    keys = [bytes(k) for k in bench_key_bytes(np.arange(N_KEYS))]
    keys[:6] = [b"", b"\xfe", bytes(range(140, 171)), "ключ_".encode() * 2 + b"k" * 14, b"\x00" * 33, bytes(range(100))]
    xx, fv = bench_key_hashes(np.arange(N_KEYS))
    for i in range(6):
        xx[i], fv[i] = O.xxh64(keys[i]), O.fnv1_64(keys[i])
    return keys, xx, fv


KEYS, KXX, KFV = _keyset()


def _pack(G, ids, reqs, table_index, base):
    n = len(ids)
    kb = [KEYS[int(i)] for i in ids]
    blob = b"".join(kb)
    bytes_at = n * 16 + (n + 1) * 4
    buf = np.zeros((bytes_at + len(blob) + 15) & ~15, dtype=np.uint8)
    kr = buf[:n * 16].view(G.native.KREQ_DTYPE)
    kr["hits"] = reqs["hits"]; kr["params"] = table_index; kr["created_delta"] = (reqs["created_at"] - base).astype(np.int32)
    buf[n * 16:bytes_at].view(np.uint32)[1:] = np.cumsum([len(k) for k in kb])
    buf[bytes_at:bytes_at + len(blob)] = np.frombuffer(blob, dtype=np.uint8)
    return buf


def make_step(G, rng, world, step, now, cap, n_params=None, sizes=None):
    """Per shard: key ids and records (bench-like on even steps, adversarial on odd ones), then the step's parameter table (at least
    n_params sets: 3 on even steps, 40 on odd ones by default), the packed key batches and the host-hashed records."""
    sizes = sizes or [[3000, 1, 0, 8192, 5], [2000, 0, 0, 8192, 700], [1, 4000, 0, 100, 8192], [8192, 0, 0, 7, 300]]
    ids, recs = [], []
    for r in range(world):
        n = min(sizes[r % 4][step % 5], cap)
        if step % 2:
            rec = adversarial_batch(rng, n, 41, now)
            _, kid = np.unique(rec["key_xxh64"], return_inverse=True)
            i = (kid.reshape(-1) * 37) % N_KEYS
        else:
            i = zipf_ids(rng, n, N_KEYS, 1.1)
            rec = np.zeros(n, dtype=O.HREQ_DTYPE)
            rec["hits"] = 1; rec["limit"] = 100; rec["duration"] = 60000; rec["created_at"] = now
            rec["algorithm"] = i & 1; rec["behavior"] = O.REQ_IS_OWNER
        ids.append(np.asarray(i, dtype=np.int64)); recs.append(rec)
    allrec = np.concatenate(recs)
    cfg = np.zeros(len(allrec), dtype=G.native.PARAMS_DTYPE)
    for f in PARAM_FIELDS:
        cfg[f] = allrec[f]
    uniq, inv = np.unique(cfg, return_inverse=True)
    want_sets = n_params if n_params is not None else (40 if step % 2 else 3)
    table = np.zeros(max(want_sets, len(uniq)), dtype=G.native.PARAMS_DTYPE)
    table["limit"] = 1 + np.arange(len(table)); table["duration"] = 5000
    table[:len(uniq)] = uniq
    inv = inv.reshape(-1)
    base = int(allrec["created_at"].min()) if len(allrec) else now
    packed, host, at = [], [], 0
    for r in range(world):
        n = len(recs[r])
        packed.append(_pack(G, ids[r], recs[r], inv[at:at + n], base))
        h = recs[r].copy()
        h["key_xxh64"], h["key_fnv1"] = KXX[ids[r]], KFV[ids[r]]
        host.append(h)
        at += n
    return packed, table, base, host


class KeyRing:
    """A ring fed with key strings and its twin fed the same requests as host-hashed records."""

    def __init__(self, world, cap=8192, spread=False, global_capacity=0, capacity=1 << 16):
        self.keyed = LocalRing(world, capacity=capacity, cap=cap, global_capacity=global_capacity, spread_devices=spread)
        self.twin = LocalRing(world, capacity=capacity, cap=cap, global_capacity=global_capacity, spread_devices=spread)
        self.W, self.cap, self.g, self.torch = world, cap, self.keyed.g, self.keyed.torch

    def upload_keys(self, packed):
        torch, lr = self.torch, self.keyed
        bufs = [torch.from_numpy(p).to(torch.device("cuda", lr.devs[r])) if len(p) else torch.zeros(16, dtype=torch.uint8, device=torch.device("cuda", lr.devs[r]))
                for r, p in enumerate(packed)]
        outs = [torch.zeros((max(self.cap, 1), 32), dtype=torch.uint8, device=torch.device("cuda", lr.devs[r])) for r in range(self.W)]
        for d in set(lr.devs):
            torch.cuda.synchronize(d)
        return bufs, outs

    def enqueue_keys(self, bufs, packed, ns, table, base, now, outs):
        lr = self.keyed
        self.g.native.p2p_step_keys_local_all(lr.p2ps, [b.data_ptr() for b in bufs], [len(p) for p in packed], ns, table, base, self.g.clock_fill(now),
                                              [o.data_ptr() for o in outs], [s.cuda_stream for s in lr.streams])

    @staticmethod
    def read(outs, ns):
        return [outs[r][:ns[r]].cpu().numpy().reshape(-1).view(O.HRESP_DTYPE) for r in range(len(ns))]

    def step(self, packed, table, base, host, now):
        ns = [len(h) for h in host]
        bufs, outs = self.upload_keys(packed)
        self.enqueue_keys(bufs, packed, ns, table, base, now, outs)
        self.keyed.sync()
        return self.read(outs, ns), self.twin.step(host, now)

    def check_scans(self):
        for r in range(self.W):
            a, b = np.sort(self.keyed.tabs[r].scan(), order=["key_xxh64", "key_fnv1"]), np.sort(self.twin.tabs[r].scan(), order=["key_xxh64", "key_fnv1"])
            assert a.tobytes() == b.tobytes(), f"shard {r}: table contents differ from the twin's"


def _oring(world):
    from gubernator_b200.sharded import shard_addresses
    oring = O.Ring(0, 512)
    for a in shard_addresses(world):
        oring.add(a)
    return oring


def _check(got, twin, want, step):
    for r in range(len(got)):
        assert np.array_equal(got[r], want[r]), f"step {step} shard {r}: {int((got[r] != want[r]).sum())} differ from the oracle"
        assert np.array_equal(got[r], twin[r]), f"step {step} shard {r}: differs from the twin ring"


@pytest.mark.parametrize("spread", [False, True])
@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_key_steps_match_oracles_and_the_record_ring(world, spread):
    import gubernator_b200 as G
    import torch
    if spread and (torch.cuda.device_count() < 2 or world == 1):
        pytest.skip("needs >= 2 GPUs")
    kr = KeyRing(world, spread=spread)
    oring = _oring(world)
    sim = [O.Pool(workers=2, cache_size=10**7, now_ms=T0) for _ in range(world)]
    rng = np.random.default_rng(world)
    for step in range(10):
        now = T0 + step
        packed, table, base, host = make_step(G, rng, world, step, now, kr.cap)
        got, twin = kr.step(packed, table, base, host, now)
        _check(got, twin, per_shard_oracle_results(oring, sim, host, now), step)
    kr.check_scans()


def test_mixed_step_keys_and_records():
    """Even shards ingest key strings, odd shards ingest records, in the same steps (gub_p2p_step_mixed_local_all)."""
    import gubernator_b200 as G
    world = 4
    kr = KeyRing(world)
    oring = _oring(world)
    sim = [O.Pool(workers=2, cache_size=10**7, now_ms=T0) for _ in range(world)]
    rng = np.random.default_rng(44)
    lr = kr.keyed
    for step in range(6):
        now = T0 + step
        packed, table, base, host = make_step(G, rng, world, step, now, kr.cap)
        ns = [len(h) for h in host]
        kbufs, outs = kr.upload_keys(packed)
        rbufs, _ = lr.upload(host)
        keyed = [r % 2 == 0 for r in range(world)]
        G.native.p2p_step_mixed_local_all(lr.p2ps, [None if keyed[r] else rbufs[r].data_ptr() for r in range(world)],
                                          [kbufs[r].data_ptr() if keyed[r] else None for r in range(world)], [len(p) for p in packed], ns, table, base,
                                          G.clock_fill(now), [o.data_ptr() for o in outs], [s.cuda_stream for s in lr.streams])
        lr.sync()
        got, twin = kr.read(outs, ns), kr.twin.step(host, now)
        _check(got, twin, per_shard_oracle_results(oring, sim, host, now), step)
    kr.check_scans()


@pytest.mark.parametrize("world", [2, 4])
def test_key_steps_back_to_back(world):
    """Eight key-string steps enqueued with no host synchronisation in between, then every response of every step is checked."""
    import gubernator_b200 as G
    kr = KeyRing(world, cap=4096)
    oring = _oring(world)
    rng = np.random.default_rng(8 + world)
    STEPS = 8
    steps = [make_step(G, rng, world, s, T0 + s, 4096) for s in range(STEPS)]
    staged = [kr.upload_keys(s[0]) for s in steps]
    for s, (packed, table, base, host) in enumerate(steps):
        kr.enqueue_keys(staged[s][0], packed, [len(h) for h in host], table, base, T0 + s, staged[s][1])
    kr.keyed.sync()
    sim = [O.Pool(workers=2, cache_size=10**7, now_ms=T0) for _ in range(world)]
    for s, (packed, table, base, host) in enumerate(steps):
        want = per_shard_oracle_results(oring, sim, host, T0 + s)
        got = kr.read(staged[s][1], [len(h) for h in host])
        for r in range(world):
            assert np.array_equal(got[r], want[r]), f"step {s} shard {r}: {int((got[r] != want[r]).sum())} differ"


def test_parameter_tables_past_the_inline_limit():
    """40 parameter sets take the copy into the ring's device table; small and large tables alternate (the buffer is reused)."""
    import gubernator_b200 as G
    world = 2
    kr = KeyRing(world)
    oring = _oring(world)
    sim = [O.Pool(workers=2, cache_size=10**7, now_ms=T0) for _ in range(world)]
    rng = np.random.default_rng(40)
    for step, n_params in enumerate([40, 3, 40, 200, 40]):
        now = T0 + step
        packed, table, base, host = make_step(G, rng, world, step, now, kr.cap, n_params=n_params)
        assert len(table) >= n_params
        got, twin = kr.step(packed, table, base, host, now)
        _check(got, twin, per_shard_oracle_results(oring, sim, host, now), step)
    kr.check_scans()


def test_empty_batches():
    """Shards with n = 0 still step (the collective rule) and the others are answered."""
    import gubernator_b200 as G
    world = 3
    kr = KeyRing(world)
    oring = _oring(world)
    sim = [O.Pool(workers=2, cache_size=10**7, now_ms=T0) for _ in range(world)]
    rng = np.random.default_rng(3)
    for step, sizes in enumerate([[[0], [0], [0]], [[500], [0], [0]], [[0], [0], [7000]]]):
        now = T0 + step
        packed, table, base, host = make_step(G, rng, world, 0, now, kr.cap, sizes=[s * 5 for s in sizes] + [[0] * 5])
        assert [len(h) for h in host] == [s[0] for s in sizes]
        got, twin = kr.step(packed, table, base, host, now)
        _check(got, twin, per_shard_oracle_results(oring, sim, host, now), step)


def test_global_key_steps_match_the_record_ring():
    """GLOBAL behaviour (gub_p2p_enable_global, gub_global_tick_local_all) with key-string steps: responses, tick statistics and the
    final tables equal those of the twin ring fed host-hashed records."""
    import gubernator_b200 as G
    world = 3
    kr = KeyRing(world, cap=4096, global_capacity=4096, capacity=1 << 14)
    rng = np.random.default_rng(503)
    now = T0
    for step in range(14):
        now += int(rng.choice([0, 1, 5, 400]))
        ids, recs = [], []
        for r in range(world):
            n = int(rng.choice([0, 1, 700, 3000]))
            i = rng.integers(0, 300, n) + 6
            b = np.zeros(n, dtype=O.HREQ_DTYPE)
            b["limit"] = 20 + (i % 7) * 10; b["duration"] = 30000 + (i % 3) * 30000; b["algorithm"] = (i >> 1) & 1
            b["hits"] = np.where(i % 11 == 0, 0, 1 + (i % 3)); b["created_at"] = now
            glob = (i % 5) < 2
            b["behavior"] = np.where(glob, O.GLOBAL, 0).astype(np.uint32) | np.uint32(O.REQ_IS_OWNER)
            if step == 7:
                b["behavior"] |= np.where(glob & (i % 13 == 0), O.RESET_REMAINING, 0).astype(np.uint32)
            ids.append(i); recs.append(b)
        allrec = np.concatenate(recs)
        cfg = np.zeros(len(allrec), dtype=G.native.PARAMS_DTYPE)
        for f in PARAM_FIELDS:
            cfg[f] = allrec[f]
        table, inv = np.unique(cfg, return_inverse=True)
        if not len(table):
            table = np.zeros(1, dtype=G.native.PARAMS_DTYPE)
        inv = inv.reshape(-1)
        packed, host, at = [], [], 0
        for r in range(world):
            n = len(recs[r])
            packed.append(_pack(G, ids[r], recs[r], inv[at:at + n], now))
            h = recs[r].copy()
            h["key_xxh64"], h["key_fnv1"] = KXX[ids[r]], KFV[ids[r]]
            host.append(h)
            at += n
        got, twin = kr.step(packed, table, now, host, now)
        for r in range(world):
            assert np.array_equal(got[r], twin[r]), f"step {step} shard {r}: {int((got[r] != twin[r]).sum())} differ from the twin ring"
        if step % 3 == 2:
            assert kr.keyed.tick(now) == kr.twin.tick(now)
            assert kr.keyed.last_tick == kr.twin.last_tick
    kr.check_scans()
