"""The single-table pipeline with two grouping scratch sets and k_group's early path (grouping before griddepcontrol.wait, the parked-insert
drain after it), on the CPU emulation of the kernels (tests/handoff_emu_harness.cpp).  Checked against the oracle and against the
one-set pipeline of tests/kernel_emu_harness.cpp: responses, counters and final table, bit for bit.  griddepcontrol is a no-op here, so
these tests cover the data flow of both scratch parities and of the early path, not the overlap itself (the `-m gpu` tests do that)."""
import numpy as np
import pytest

import oracle_py as O
import _handoff_emu as H
import _kernel_emu as E
from workloads import T0, adversarial_batch, bench_requests, key_hashes, make_clock, zipf_ids


@pytest.fixture(scope="module")
def G():
    import gubernator_b200 as g  # dtypes only; nothing here touches CUDA
    return g


def _cmp(got, want, what=""):
    if not np.array_equal(got, want):
        bad = np.nonzero(got != want)[0]
        i = int(bad[0])
        raise AssertionError(f"{what}: {len(bad)} of {len(got)} responses differ; first at {i}: got {got[i]} want {want[i]}")


def _same_table(G, a, b):
    sa, sb = np.sort(a.scan(G.ITEM_DTYPE), order=["key_xxh64", "key_fnv1"]), np.sort(b.scan(G.ITEM_DTYPE), order=["key_xxh64", "key_fnv1"])
    assert len(sa) == len(sb) and sa.tobytes() == sb.tobytes()
    assert a.counters() == b.counters()


@pytest.mark.parametrize("early", [True, False])
def test_consecutive_batches_sharing_keys(G, early):
    """Batches whose keys repeat from one batch to the next, on both parities: Zipf batches (uniform runs) and adversarial ones
    (non-uniform groups, expiry, every behaviour bit)."""
    rng = np.random.default_rng(31)
    tab, ref, pool = H.HandoffTable(1 << 13, max_batch=2048), E.EmuTable(1 << 13, max_batch=2048), O.Pool(now_ms=T0)
    now, epoch = T0, 0
    for step in range(8):
        now += int(rng.choice([0, 1, 700, 70000]))
        pool.set_now(now)
        reqs = bench_requests(zipf_ids(rng, 3000, 1200, 1.1), now) if step % 2 == 0 else adversarial_batch(rng, 2500, 60, now)
        got = tab.submit(reqs, make_clock(now), O.HRESP_DTYPE, early=early)
        _cmp(got, pool.submit_hashed(reqs), f"step {step}")
        _cmp(got, ref.submit(reqs, make_clock(now), O.HRESP_DTYPE), f"step {step} vs one scratch set")
        epoch += -(-len(reqs) // 2048)  # one epoch per chunk of max_batch requests
        assert tab.chain_done() == epoch  # stored by the last k_finish block of the last chunk
    _same_table(G, tab, ref)
    assert tab.counters()["mixed_groups"] > 0 and tab.counters()["dup_groups"] > 0


def test_epoch_wrap_in_a_sequence(G):
    """65 535 -> 1 in the middle of a sequence: both aux sets are cleared, the batch at epoch 1 waits first."""
    rng = np.random.default_rng(5)
    tab, pool = H.HandoffTable(1 << 13, max_batch=1024), O.Pool(now_ms=T0)
    tab.set_epoch(65532)
    now = T0
    for step in range(6):
        now += 300
        pool.set_now(now)
        reqs = adversarial_batch(rng, 1000, 40, now) if step % 2 else bench_requests(zipf_ids(rng, 1000, 300, 1.1), now)
        _cmp(tab.submit(reqs, make_clock(now), O.HRESP_DTYPE), pool.submit_hashed(reqs), f"step {step}")
        assert tab.chain_done() == [65533, 65534, 65535, 1, 2, 3][step]


def test_parked_inserts_drain_after_the_wait(G):
    """A table far too small for the batch: keys whose probe window is full are parked, and the next batch's k_group places them after
    its wait — on the early path too — with the same responses, counters and final table as the one-set pipeline."""
    n = 1500
    reqs = np.zeros(n, dtype=G.REQ_DTYPE)
    xx, fv = key_hashes(np.arange(n), name="full")
    reqs["key_xxh64"], reqs["key_fnv1"] = xx, fv
    reqs["hits"] = 1; reqs["limit"] = 5; reqs["duration"] = 100000; reqs["created_at"] = T0 + np.arange(n)
    tab, ref = H.HandoffTable(64, max_batch=2048), E.EmuTable(64, max_batch=2048)
    _cmp(tab.submit(reqs, make_clock(T0), O.HRESP_DTYPE), ref.submit(reqs, make_clock(T0), O.HRESP_DTYPE), "first batch")
    c = tab.counters()
    assert c["inserts"] == 64 and c["table_full"] == n - 64 - 1024 and c["unexpired_evictions"] == 0  # parked, not placed yet
    _same_table(G, tab, ref)
    again = reqs[-8:].copy()
    again["created_at"] = T0 + 5
    got = tab.submit(again, make_clock(T0 + 5), O.HRESP_DTYPE)
    _cmp(got, ref.submit(again, make_clock(T0 + 5), O.HRESP_DTYPE), "second batch")
    assert tab.counters()["unexpired_evictions"] == 1024 and np.all(got["err_code"] == 0)
    _same_table(G, tab, ref)
