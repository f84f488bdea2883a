"""The Store plugin's device passes (gubernator_b200/csrc/gub_store.cuh) on the CPU emulation, around the four batch kernels: the miss list
Store.Get receives, the responses and every Remove / OnChange record, bit for bit, against the host layer's rule restated over the oracle
(tests/_store_emu.py model_batch)."""
import numpy as np
import pytest

import oracle_py as O
import _store_emu as S
from workloads import T0, adversarial_batch, bench_requests, key_hashes, make_clock, zipf_ids


def _eq(got, want, what):
    assert len(got) == len(want), f"{what}: {len(got)} records, want {len(want)}"
    if got.tobytes() != want.tobytes():
        bad = [i for i in range(len(got)) if got[i].tobytes() != want[i].tobytes()]
        raise AssertionError(f"{what}: {len(bad)} differ; first {bad[0]}: got {got[bad[0]]} want {want[bad[0]]}")


def _mixed_batch(rng, now, n_adv_keys):
    """Adversarial runs (resets, switches, invalid algorithms, Hits 0 / negative, non-owners, Gregorian), keys seen once and Zipf runs."""
    adv = adversarial_batch(rng, 900, n_adv_keys, now)
    once = np.zeros(200, dtype=O.HREQ_DTYPE)
    once["key_xxh64"], once["key_fnv1"] = key_hashes(rng.integers(10**6, 10**7, 200), name="once")
    once["hits"], once["limit"], once["duration"], once["created_at"] = 1, 10, 60000, now
    once["algorithm"] = rng.integers(0, 2, 200)
    once["behavior"] = O.REQ_IS_OWNER
    zipf = bench_requests(zipf_ids(rng, 700, 300, 1.1), now)
    reqs = np.concatenate([adv, once, zipf])
    return np.ascontiguousarray(reqs[rng.permutation(len(reqs))])


def _run(tab, pool, rng, batches, frac=0.4, with_get=True):
    now, seen = T0, 0
    for b in range(batches):
        now += int(rng.choice([0, 1, 700, 70000]))
        reqs = _mixed_batch(rng, now, int(rng.choice([20, 80, 400])))
        items = S.fill_store(rng, reqs, now, frac if with_get else 0.0)
        calls = []
        rc, resp, recs = tab.submit_store(reqs, make_clock(now), O.HRESP_DTYPE, S.found_filler(items, calls) if with_get else None)
        assert rc == 0
        misses, want_resp, want_recs = S.model_batch(pool, reqs, now, items if with_get else {})
        if with_get:
            assert len(calls) == (1 if len(misses) else 0)
            if calls:
                _eq(calls[0], misses, f"batch {b}: miss list")
        assert np.array_equal(resp, want_resp), f"batch {b}: responses differ"
        _eq(recs, want_recs, f"batch {b}: records")
        assert np.all(np.diff(recs["first"].astype(np.int64)) > 0)
        seen |= int(np.bitwise_or.reduce(recs["flags"])) if len(recs) else 0
    assert seen == S.STORE_REMOVE | S.STORE_CHANGE


@pytest.mark.parametrize("seed", [0, 1])
def test_store_passes_match_the_host_layer_rule(seed):
    rng = np.random.default_rng(40 + seed)
    _run(S.StoreTable(1 << 14, max_batch=2048), O.Pool(now_ms=T0), rng, 4)


def test_write_behind_store_without_get():
    """get = NULL: no miss list, no call; the records are those of a store that never finds anything."""
    rng = np.random.default_rng(7)
    _run(S.StoreTable(1 << 14, max_batch=2048), O.Pool(now_ms=T0), rng, 3, with_get=False)


def test_dedup_scratch_epoch_wrap():
    """Stale entries from before the wrap of the dedup scratch's epoch must not alias this batch's keys."""
    rng = np.random.default_rng(11)
    tab = S.StoreTable(1 << 14, max_batch=2048)
    tab.set_store_epoch(0xFFFFFFFE)
    _run(tab, O.Pool(now_ms=T0), rng, 3)
    assert tab.store_epoch() == 2


def test_failing_get_evaluates_nothing():
    rng = np.random.default_rng(3)
    tab = S.StoreTable(1 << 14, max_batch=2048)
    now = T0
    reqs = _mixed_batch(rng, now, 50)
    assert tab.submit_store(reqs, make_clock(now), O.HRESP_DTYPE, None)[0] == 0
    scan, counters = tab.scan(S.ITEM_DTYPE), tab.counters()
    rc, _, _ = tab.submit_store(_mixed_batch(rng, now + 5, 50), make_clock(now + 5), O.HRESP_DTYPE, lambda misses: 9)
    assert rc == 9
    assert tab.counters() == counters
    assert tab.scan(S.ITEM_DTYPE).tobytes() == scan.tobytes()


def test_parked_inserts_are_seen_by_both_passes():
    """A table too small for the batch parks inserts: the post-pass reads them from the parked list, the next pre-pass finds them there."""
    rng = np.random.default_rng(5)
    tab, pool = S.StoreTable(512, max_batch=2048), O.Pool(now_ms=T0)
    now = T0
    for b in range(3):
        reqs = np.zeros(1200, dtype=O.HREQ_DTYPE)
        reqs["key_xxh64"], reqs["key_fnv1"] = key_hashes(rng.integers(0, 900, 1200), name="park")
        reqs["hits"], reqs["limit"], reqs["duration"], reqs["created_at"], reqs["behavior"] = 1, 50, 600000, now, O.REQ_IS_OWNER
        rc, resp, recs = tab.submit_store(reqs, make_clock(now), O.HRESP_DTYPE, S.found_filler({}))
        assert rc == 0 and tab.ovf_count() > 0
        assert np.all(recs["flags"] == S.STORE_CHANGE)
        assert len(recs) == len(set(zip(reqs["key_xxh64"].tolist(), reqs["key_fnv1"].tolist())))
        # the state each record reports is what the last request of its key answered
        last = resp[recs["last"]]
        assert np.array_equal(recs["item"]["remaining"], last["remaining"]) and np.array_equal(recs["item"]["expire_at"], last["reset_time"])
        now += 1
