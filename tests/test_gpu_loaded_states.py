"""Loaded states on the GPU: every lattice state of edge_states.py installed with gub_add_items (and into the oracle bit for bit),
then driven by request plans aimed at each evaluation route, on both paths.  Responses, counters, gub_get_items and gub_scan
(remaining_f through its bits) must equal the oracle's."""
import numpy as np
import pytest

import edge_states as ES
import oracle_py as O

pytestmark = pytest.mark.gpu

BATCH = 65536


@pytest.fixture(autouse=True, params=["pipeline", "fused"])
def eval_path(request, monkeypatch):
    """Both evaluation paths of a single table: the four-kernel pipeline and the persistent kernel k_batch (GUB_PATH=fused)."""
    monkeypatch.setenv("GUB_PATH", request.param)
    return request.param


@pytest.fixture(scope="module")
def G():
    import gubernator_b200 as g
    return g


@pytest.fixture(scope="module")
def lattice(G):
    return ES.lattice(G.REQ_DTYPE)


def _cmp(got, want, what):
    if not np.array_equal(got, want):
        bad = np.nonzero(got != want)[0]
        i = int(bad[0])
        raise AssertionError(f"{what}: {len(bad)} of {len(got)} responses differ; first at {i}: got {got[i]} want {want[i]}")


def _loaded(G, its):
    tab = G.Table(1 << 16)
    pool = O.Pool(workers=4, cache_size=10_000_000, now_ms=ES.NOW)
    tab.add_items(its)
    for r in its:
        pool.add_item_hashed(r["key_xxh64"], r["key_fnv1"], ES.oracle_item(r))
    return tab, pool


def _check_items(G, tab, pool, its):
    """The counters, the whole gub_scan and gub_get_items of every key against the oracle's cache, byte for byte."""
    c, oc = tab.counters(), pool.counters()
    for k in ("over_limit", "cache_hit", "cache_miss"):
        assert c[k] == oc[k], (k, c, oc)
    scan, held = ES.keyed_scan(tab.scan(), pool.each())
    assert scan.keys() == held.keys()
    for k, it in held.items():
        want = ES.item_of_oracle(it, *k)
        assert scan[k].tobytes() == want.tobytes(), ("scan", k, scan[k], want)
    # after the scan: the oracle's GetItem removes what it finds expired
    kx, kf = its["key_xxh64"], its["key_fnv1"]
    got, found = tab.get_items(kx, kf, ES.NOW)
    for i in range(len(its)):
        it = pool.get_item_hashed(kx[i], kf[i])
        assert found[i] == (it is not None), (i, its[i])
        if it is not None:
            want = ES.item_of_oracle(it, kx[i], kf[i])
            assert got[i].tobytes() == want.tobytes(), ("get_items", i, its[i], got[i], want)


def test_loaded_states_in_full_batches(G, lattice):
    """All plans back to back in full 65 536-request batches (each plan's requests in order, plans shuffled)."""
    its, plans = lattice
    tab, pool = _loaded(G, its)
    order = np.random.default_rng(11).permutation(len(plans))
    reqs = np.concatenate([plans[i] for i in order])
    clk = G.clock_fill(ES.NOW)
    for off in range(0, len(reqs), BATCH):
        chunk = np.ascontiguousarray(reqs[off:off + BATCH])
        _cmp(tab.submit(chunk, clk), pool.submit_hashed(chunk), f"batch at {off}")
    _check_items(G, tab, pool, its)
    c = tab.counters()
    assert c["dup_groups"] > 0 and c["mixed_groups"] > 0 and c["serial_fallbacks"] > 0, c


def test_loaded_states_one_plan_at_a_time(G, lattice):
    """Every plan as a batch of its own: single requests are answered in k_rank, runs by the closed forms of k_eval / k_finish."""
    its, plans = lattice
    tab, pool = _loaded(G, its)
    clk = G.clock_fill(ES.NOW)
    for n, p in enumerate(plans):
        _cmp(tab.submit(p, clk), pool.submit_hashed(p), f"plan {n} on item {its[n]}")
    _check_items(G, tab, pool, its)
    c = tab.counters()
    assert c["dup_groups"] > 0 and c["mixed_groups"] > 0 and c["serial_fallbacks"] > 0, c
