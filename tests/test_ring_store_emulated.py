"""The ring's Store step (gub_p2p_step_keys_store_local_all: the *_ring Store kernels and k_store_orig of gub_store.cuh) on the CPU
emulation of the kernels.  Every owner's responses, miss list and change log must equal, bit for bit, those of the single-table Store
emulation (tests/_store_emu.py) fed that owner's pass, once pass indices are turned into (source shard, source index)."""
import numpy as np
import pytest

import oracle_py as O
import _ring_store_emu as R
import _store_emu as S
from workloads import T0, adversarial_batch, bench_requests, key_hashes, make_clock, zipf_ids

CAP = 512


def _oring(world):
    from gubernator_b200.sharded import shard_addresses
    oring = O.Ring(0, 512)
    for a in shard_addresses(world):
        oring.add(a)
    return oring


def _batch(rng, n, now, kind):
    """Zipf runs, or adversarial traffic (resets, switches, invalid algorithms, Hits 0 / negative, non-owners) plus keys seen once."""
    if n == 0:
        return np.zeros(0, dtype=O.HREQ_DTYPE)
    if kind == "zipf":
        return np.ascontiguousarray(bench_requests(zipf_ids(rng, n, 300, 1.1), now))
    if kind == "spread":
        # Many distinct long-lived keys, more than a small table holds.  Every key has its own duration, so no two entries share an
        # ExpireAt: which entry a full table evicts then has no tie to break.  (The ring-mode and single-table pipelines may break
        # such ties differently; that is the batch kernels' business, not the Store's.)
        ids = rng.integers(0, 900, n)
        reqs = np.zeros(n, dtype=O.HREQ_DTYPE)
        reqs["key_xxh64"], reqs["key_fnv1"] = key_hashes(ids, name="park")
        reqs["hits"], reqs["limit"], reqs["created_at"], reqs["behavior"] = 1, 50, now, O.REQ_IS_OWNER
        reqs["duration"] = 600000 + ids * 10
        return reqs
    adv = adversarial_batch(rng, max(n - n // 5, 1), int(rng.choice([20, 80])), now)
    once = np.zeros(n - len(adv), dtype=O.HREQ_DTYPE)
    once["key_xxh64"], once["key_fnv1"] = key_hashes(rng.integers(10**6, 10**7, len(once)), name="once")
    once["hits"], once["limit"], once["duration"], once["created_at"] = 1, 10, 60000, now
    once["algorithm"] = rng.integers(0, 2, len(once))
    once["behavior"] = O.REQ_IS_OWNER
    reqs = np.concatenate([adv, once])
    return np.ascontiguousarray(reqs[rng.permutation(len(reqs))])


def _passes(oring, batches, world):
    owners = [np.array([oring.get_by_hash(int(h)) for h in b["key_fnv1"]], dtype=np.int64) for b in batches]
    out = []
    for r in range(world):
        shard = np.concatenate([np.full(int((owners[s] == r).sum()), s, dtype=np.int64) for s in range(world)])
        idx = np.concatenate([np.nonzero(owners[s] == r)[0] for s in range(world)])
        out.append((shard, idx))
    return out


def _named(recs, shard, idx):
    r = recs.copy().view(R.REC_DTYPE)
    r["first_shard"], r["last_shard"] = shard[recs["first"]], shard[recs["last"]]
    r["first"], r["last"] = idx[recs["first"]], idx[recs["last"]]
    return r


def _eq(got, want, what):
    assert len(got) == len(want), f"{what}: {len(got)} records, want {len(want)}"
    assert got.tobytes() == want.tobytes(), f"{what}: records differ"


class Twins:
    """The ring and one single-table Store emulation per owner, fed the same steps."""

    def __init__(self, world, capacity, max_batch=2048):
        self.W, self.oring = world, _oring(world)
        pts, peers = self.oring.points()
        self.ring = R.StoreRingCluster(world, CAP, capacity, pts, peers, max_batch)
        self.tabs = [S.StoreTable(capacity, max_batch=max_batch) for _ in range(world)]

    def step(self, rng, now, kinds, frac=0.4, with_get=True, sizes=None):
        W = self.W
        sizes = sizes or [int(rng.choice([0, 1, 200, CAP])) for _ in range(W)]
        batches = [_batch(rng, sizes[r], now, kinds[r % len(kinds)]) for r in range(W)]
        allreq = np.concatenate(batches)
        items = S.fill_store(rng, allreq, now, frac) if with_get and len(allreq) else {}
        calls = []
        rc, got, recs = self.ring.step(batches, make_clock(now), O.HRESP_DTYPE, S.found_filler(items, calls) if with_get else None)
        assert rc == 0
        want = [np.zeros(len(b), dtype=O.HRESP_DTYPE) for b in batches]
        want_misses = []
        for r, (shard, idx) in enumerate(_passes(self.oring, batches, W)):
            pr = np.concatenate([batches[s][idx[shard == s]] for s in range(W)]) if len(idx) else np.zeros(0, dtype=O.HREQ_DTYPE)
            if len(pr) == 0:
                assert len(recs[r]) == 0
                continue
            tcalls = []
            trc, tresp, trecs = self.tabs[r].submit_store(pr, make_clock(now), O.HRESP_DTYPE, S.found_filler(items, tcalls) if with_get else None)
            assert trc == 0
            _eq(recs[r], _named(trecs, shard, idx), f"owner {r}: change log")
            want_misses += [_named(c, shard, idx) for c in tcalls]
            for s in range(W):
                want[s][idx[shard == s]] = tresp[shard == s]
        assert len(calls) == len(want_misses), "one Get per owner that has misses"
        for c, w in zip(calls, want_misses):
            _eq(c.view(R.REC_DTYPE), w, "miss list")
        for s in range(W):
            assert np.array_equal(got[s], want[s]), f"shard {s}: responses differ"
        return recs

    def check_tables(self):
        for r in range(self.W):
            assert self.ring.scan(r, S.ITEM_DTYPE).tobytes() == _sorted_scan(self.tabs[r]).tobytes(), f"owner {r}: table differs"


def _sorted_scan(tab):
    s = tab.scan(S.ITEM_DTYPE)
    return s[np.lexsort((s["key_fnv1"], s["key_xxh64"]))]


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_ring_store_matches_single_table_per_owner(world):
    rng = np.random.default_rng(60 + world)
    tw = Twins(world, 1 << 13)
    now, seen = T0, 0
    for step in range(4):
        now += int(rng.choice([0, 1, 700, 70000]))
        recs = tw.step(rng, now, ["zipf", "adv"] if step % 2 else ["adv", "zipf"])
        for rr in recs:
            seen |= int(np.bitwise_or.reduce(rr["flags"])) if len(rr) else 0
    assert seen == S.STORE_REMOVE | S.STORE_CHANGE
    tw.check_tables()


def test_small_table_parks_inserts():
    """A table too small for its owner's pass parks inserts.  The reference here is the plain ring fed the same steps, not a single
    table: once a table overflows, ring-mode and single-table pipelines may place and evict differently (with or without a Store).
    The Store step must answer exactly as the plain ring, and every OnChange item must be the state its key's last request left,
    read from the parked list where the table lacks the key."""
    import _kernel_emu as E
    world = 2
    rng = np.random.default_rng(5)
    oring = _oring(world)
    pts, peers = oring.points()
    ring = R.StoreRingCluster(world, CAP, 128, pts, peers, 2048)
    plain = E.EmuP2PCluster(world, CAP, 128, pts, peers, max_batch=2048, finish_cap=3)
    parked = 0
    for step in range(3):
        now = T0 + step
        batches = [_batch(rng, CAP, now, "spread") for _ in range(world)]
        rc, got, recs = ring.step(batches, make_clock(now), O.HRESP_DTYPE, S.found_filler({}))
        assert rc == 0
        want = plain.step(batches, make_clock(now), O.HRESP_DTYPE)
        for s in range(world):
            assert np.array_equal(got[s], want[s]), f"step {step} shard {s}: responses differ from the plain ring"
        for r in range(world):
            assert np.all(recs[r]["flags"] == S.STORE_CHANGE)
            last = np.array([got[int(x["last_shard"])][int(x["last"])] for x in recs[r]], dtype=O.HRESP_DTYPE)
            if len(last):
                assert np.array_equal(recs[r]["item"]["remaining"], last["remaining"])
                assert np.array_equal(recs[r]["item"]["expire_at"], last["reset_time"])
            parked += ring.ovf_count(r)
        keys = {(int(a), int(b)) for bt in batches for a, b in zip(bt["key_xxh64"], bt["key_fnv1"])}
        assert sum(len(x) for x in recs) == len(keys), "one record per key"
    assert parked > 0, "the tables took everything: no insert was parked"


def test_write_behind_store_without_get():
    rng = np.random.default_rng(6)
    tw = Twins(3, 1 << 13)
    for step in range(3):
        tw.step(rng, T0 + 10 * step, ["adv", "zipf"], with_get=False)
    tw.check_tables()


def test_failing_get_changes_nothing_and_keeps_the_ring_in_step():
    world = 3
    rng = np.random.default_rng(8)
    a, b = Twins(world, 1 << 13), Twins(world, 1 << 13)
    batches0 = [_batch(rng, 300, T0, "zipf") for _ in range(world)]
    for t in (a, b):
        assert t.ring.step(batches0, make_clock(T0), O.HRESP_DTYPE, S.found_filler({}))[0] == 0
    before = [(a.ring.scan(r, S.ITEM_DTYPE).tobytes(), a.ring.counters(r)) for r in range(world)]
    calls = []
    failed = [_batch(rng, 300, T0 + 1, "adv") for _ in range(world)]
    rc, _, _ = a.ring.step(failed, make_clock(T0 + 1), O.HRESP_DTYPE, lambda m: calls.append(len(m)) or 4)
    assert rc == 4 and len(calls) == 1
    assert [(a.ring.scan(r, S.ITEM_DTYPE).tobytes(), a.ring.counters(r)) for r in range(world)] == before
    batches2 = [_batch(rng, 400, T0 + 2, "adv") for _ in range(world)]
    items = S.fill_store(rng, np.concatenate(batches2), T0 + 2)
    ra = a.ring.step(batches2, make_clock(T0 + 2), O.HRESP_DTYPE, S.found_filler(items))
    rb = b.ring.step(batches2, make_clock(T0 + 2), O.HRESP_DTYPE, S.found_filler(items))
    assert ra[0] == rb[0] == 0
    for r in range(world):
        assert ra[1][r].tobytes() == rb[1][r].tobytes() and ra[2][r].tobytes() == rb[2][r].tobytes()


def test_dedup_epoch_wrap():
    """Steps across a wrap of every owner's dedup epoch (the scratch is cleared) match the single tables, which wrap too."""
    world = 2
    rng = np.random.default_rng(9)
    tw = Twins(world, 1 << 13)
    for r in range(world):
        tw.ring.set_store_epoch(r, 0xFFFFFFFE)
        tw.tabs[r].set_store_epoch(0xFFFFFFFE)
    for step in range(3):
        tw.step(rng, T0 + step, ["zipf", "adv"], sizes=[CAP, CAP])
    assert all(tw.ring.store_epoch(r) == 2 for r in range(world))
    tw.check_tables()
