"""The CUDA kernel source itself, on the CPU: gubernator_b200/csrc/gub_kernels.cuh and gub_batch.cuh compiled with g++ on top of tests/cuda_emu.h
(fibers standing in for the threads of a block; tests/kernel_emu_harness.cpp drives the launches exactly like gub_api.cu) and
checked against the oracle — responses, counters and final table, bit for bit.  This is NOT a product path (the library has no
CPU fallback) and not a replacement for the `-m gpu` parity tests: it explores one interleaving and no memory-model effects.
It keeps the grouping / rank / snapshot / segment logic, the routing kernels and the hashing kernel under test where there is
no GPU, and lets a kernel change be tried before GPU minutes are spent on it."""
import numpy as np
import pytest

import edge_states as ES
import oracle_py as O
import _kernel_emu as E
from workloads import T0, adversarial_batch, bench_requests, extreme_batch, key_hashes, make_clock, zipf_ids


# Both evaluation paths run the same bodies: "pipeline" = k_group / k_rank / k_eval / k_finish (what gub_submit* launches for a single
# table), "fused" = the persistent cooperative kernel k_batch (what rings launch; here on a 6-CTA grid, so most batches take rounds).
both_paths = pytest.mark.parametrize("path", ["pipeline", "fused"])


def Tab(path, capacity, **kw):
    return E.EmuTable(capacity, fused=(path == "fused"), **kw)


@pytest.fixture(scope="module")
def G():
    import gubernator_b200 as g  # dtypes and the host-side helpers only; nothing here touches CUDA
    return g


def _cmp(got, want, what=""):
    if not np.array_equal(got, want):
        bad = np.nonzero(got != want)[0]
        i = int(bad[0])
        raise AssertionError(f"{what}: {len(bad)} of {len(got)} responses differ; first at {i}: got {got[i]} want {want[i]}")


def _check_state(G, tab, pool):
    c, oc = tab.counters(), pool.counters()
    for k in ("over_limit", "cache_hit", "cache_miss"):
        assert c[k] == oc[k], (k, c, oc)
    items = pool.each()
    scan = tab.scan(G.ITEM_DTYPE)
    dev = {(int(s["key_xxh64"]), int(s["key_fnv1"]) >> 8): s for s in scan}
    assert len(dev) == len(scan) == len(items)
    for (kx, kf), it in items.items():
        s = dev[(kx if kx >= 2 else kx + 2, kf >> 8)]
        assert (int(s["limit"]), int(s["duration"]), int(s["stamp"]), int(s["expire_at"])) == (it.limit, it.duration, it.stamp, it.expire_at)
        if it.value_kind == 2:
            assert int(s["algorithm"]) == 1 and int(s["burst"]) == it.burst
            assert np.float64(s["remaining_f"]).view(np.uint64) == np.float64(it.remaining_f).view(np.uint64)
        else:
            assert int(s["algorithm"]) == 0 and int(s["remaining"]) == it.remaining_i and int(s["status"]) == it.status


@both_paths
@pytest.mark.parametrize("seed,n_keys,n", [(0, 3, 1500), (1, 40, 3000), (2, 2500, 3000), (3, 1, 700)])
def test_adversarial_batches_match_oracle(G, seed, n_keys, n, path):
    """Every behaviour bit, both algorithms, parameter changes mid-run, time steps that expire items: few keys exercise the
    non-uniform (segment) path of k_finish, many keys the singleton path of k_rank."""
    rng = np.random.default_rng(100 + seed)
    tab, pool = Tab(path, 1 << 13, max_batch=2048), O.Pool(now_ms=T0)
    now = T0
    for step in range(3):
        now += int(rng.choice([0, 1, 900, 70000]))
        pool.set_now(now)
        reqs = adversarial_batch(rng, n, n_keys, now)
        _cmp(tab.submit(reqs, make_clock(now), O.HRESP_DTYPE), pool.submit_hashed(reqs), f"step {step}")
    _check_state(G, tab, pool)


@both_paths
def test_zipf_uniform_runs_use_the_rank_path(G, path):
    """The bench workload's shape: identical requests per key, heavy repeats — run_to_rank per member, no non-uniform groups."""
    rng = np.random.default_rng(7)
    tab, pool = Tab(path, 1 << 13), O.Pool(now_ms=T0)
    for step in range(3):
        now = T0 + 400 * step
        pool.set_now(now)
        reqs = bench_requests(zipf_ids(rng, 4096, 1500, 1.1), now)
        _cmp(tab.submit(reqs, make_clock(now), O.HRESP_DTYPE), pool.submit_hashed(reqs), f"step {step}")
    c = tab.counters()
    assert c["mixed_groups"] == 0 and c["dup_groups"] > 0
    _check_state(G, tab, pool)


@both_paths
def test_numeric_extremes(G, path):
    rng = np.random.default_rng(31)
    tab, pool = Tab(path, 1 << 12), O.Pool(now_ms=T0)
    for step in range(2):
        now = T0 + 1000 * step
        pool.set_now(now)
        reqs = extreme_batch(rng, 2000, 30, now)
        _cmp(tab.submit(reqs, make_clock(now), O.HRESP_DTYPE), pool.submit_hashed(reqs), f"step {step}")
    _check_state(G, tab, pool)


@both_paths
def test_loaded_states_match_oracle(G, path):
    """Every state of edge_states.py installed with k_add_items (and into the oracle bit for bit), then its request plans: all
    short plans on every state, the long uniform runs and the chunk-crossing and one-request-segment runs on every 16th.
    Responses, counters, get_items and the scan (remaining_f as bits) equal the oracle's."""
    its, plans = ES.lattice(O.HREQ_DTYPE, lambda i, j, p: len(p) <= 40 or i % 16 == 0)
    tab, pool = Tab(path, 1 << 15), O.Pool(workers=4, cache_size=10_000_000, now_ms=ES.NOW)
    tab.add_items(its)
    for r in its:
        pool.add_item_hashed(r["key_xxh64"], r["key_fnv1"], ES.oracle_item(r))
    reqs = np.concatenate([plans[i] for i in np.random.default_rng(12).permutation(len(plans))])
    for off in range(0, len(reqs), 65536):
        chunk = np.ascontiguousarray(reqs[off:off + 65536])
        _cmp(tab.submit(chunk, make_clock(ES.NOW), O.HRESP_DTYPE), pool.submit_hashed(chunk), f"batch at {off}")
    c, oc = tab.counters(), pool.counters()
    assert all(c[k] == oc[k] for k in ("over_limit", "cache_hit", "cache_miss")), (c, oc)
    assert c["dup_groups"] > 0 and c["mixed_groups"] > 0 and c["serial_fallbacks"] > 0, c
    scan, held = ES.keyed_scan(tab.scan(G.ITEM_DTYPE), pool.each())
    assert scan.keys() == held.keys()
    for k, it in held.items():
        assert scan[k].tobytes() == ES.item_of_oracle(it, *k).tobytes(), ("scan", scan[k], ES.item_of_oracle(it, *k))
    got, found = tab.get_items(its["key_xxh64"], its["key_fnv1"], ES.NOW, G.ITEM_DTYPE)  # after the scan: GetItem removes expired items
    for i, r in enumerate(its):
        it = pool.get_item_hashed(r["key_xxh64"], r["key_fnv1"])
        assert found[i] == (it is not None), (i, r)
        assert it is None or got[i].tobytes() == ES.item_of_oracle(it, r["key_xxh64"], r["key_fnv1"]).tobytes(), ("get_items", i, r, got[i])


@both_paths
def test_many_segments_force_the_serial_walk(G, path):
    rng = np.random.default_rng(77)
    tab, pool = Tab(path, 4096), O.Pool(now_ms=T0)
    n = 1200
    reqs = np.zeros(n, dtype=G.REQ_DTYPE)
    xx, fv = key_hashes([1] * n, name="hot")
    reqs["key_xxh64"], reqs["key_fnv1"] = xx, fv
    reqs["hits"] = rng.integers(0, 3, n); reqs["limit"] = rng.choice([50, 100], n); reqs["duration"] = 60000
    reqs["created_at"] = T0 + rng.integers(0, 5, n); reqs["algorithm"] = 1; reqs["behavior"] = G.native.REQ_IS_OWNER
    _cmp(tab.submit(reqs, make_clock(T0), O.HRESP_DTYPE), pool.submit_hashed(reqs))
    walked = tab.counters()["serial_fallbacks"]  # chunks of the group that were mostly one-request segments: applied one by one
    assert walked >= 1
    reqs2 = reqs.copy()
    reqs2["hits"] = 1; reqs2["limit"] = 100; reqs2["created_at"] = T0 + 10 + (np.arange(n) // 200)  # six long uniform segments
    pool.set_now(T0 + 10)
    _cmp(tab.submit(reqs2, make_clock(T0 + 10), O.HRESP_DTYPE), pool.submit_hashed(reqs2))
    assert tab.counters()["serial_fallbacks"] == walked  # long segments are planned, not walked
    _check_state(G, tab, pool)


@both_paths
@pytest.mark.parametrize("algorithm", [0, 1])
def test_hot_key_with_differing_hits_many_segments(G, path, algorithm):
    """A hot key whose clients ask for different `hits`: hundreds of segments (runs of identical requests) per chunk of the group.
    The segment fold speculates that a range of segments leaves the bucket unchanged (true once the key is over its limit) and falls
    back, range by range, where the state moves: first batch walks the limit down (every range moves the state), later batches
    sit at the fixed point, the last one mixes in Hits = 0 queries, a limit change and negative hits (state moves again mid-way)."""
    rng = np.random.default_rng(5 + algorithm)
    tab, pool = Tab(path, 4096), O.Pool(now_ms=T0)
    n = 3000
    xx, fv = key_hashes([3] * n, name="hothetero")
    for b in range(4):
        now = T0 + 7 * b
        reqs = np.zeros(n, dtype=G.REQ_DTYPE)
        reqs["key_xxh64"], reqs["key_fnv1"] = xx, fv
        run = np.repeat(np.arange(n // 4 + 1), rng.integers(1, 9, n // 4 + 1))[:n]     # runs of 1..8 identical requests
        hits_of_run = rng.choice([1, 2, 3], run.max() + 1)
        reqs["hits"] = hits_of_run[run]
        reqs["limit"] = 4000 if b < 2 else 3000; reqs["duration"] = 60000; reqs["created_at"] = now
        reqs["algorithm"] = algorithm; reqs["behavior"] = G.native.REQ_IS_OWNER
        if b == 3:
            odd = rng.random(n) < 0.03
            reqs["hits"] = np.where(odd, rng.choice([0, -5, 1 << 20], n), reqs["hits"])
            reqs["limit"] = np.where(rng.random(n) < 0.01, 3500, reqs["limit"])
        pool.set_now(now)
        _cmp(tab.submit(reqs, make_clock(now), O.HRESP_DTYPE), pool.submit_hashed(reqs), f"batch {b}")
    if path == "pipeline":
        assert tab.counters()["mixed_groups"] >= 4
    _check_state(G, tab, pool)


def test_sweep_in_slices_equals_one_sweep(G):
    """The pipeline's incremental sweep (gub_api.cu maybe_sweep: one slice of the table between batches) frees exactly what one
    whole-table sweep frees, and the table keeps answering like the oracle afterwards (expired keys are misses either way)."""
    rng = np.random.default_rng(9)
    cap = 1 << 12
    tabs, pool = [Tab("pipeline", cap), Tab("pipeline", cap)], O.Pool(now_ms=T0)
    reqs = bench_requests(rng.permutation(1500), T0).astype(G.REQ_DTYPE)
    reqs["duration"] = np.where(np.arange(1500) % 3 == 0, 50, 60000)  # a third of the keys expire at T0 + 50
    want = pool.submit_hashed(reqs)
    for t in tabs:
        _cmp(t.submit(reqs, make_clock(T0), O.HRESP_DTYPE), want)
    now = T0 + 1000
    whole = tabs[0].sweep(now)
    parts = sum(tabs[1].sweep_range(lo, lo + cap // 8, now) for lo in range(0, cap, cap // 8))
    assert whole == parts == 500
    pool.set_now(now)
    reqs["created_at"] = now
    want = pool.submit_hashed(reqs)
    for t in tabs:
        _cmp(t.submit(reqs, make_clock(now), O.HRESP_DTYPE), want)


@both_paths
def test_token_reset_flipflop(G, path):
    tab, pool = Tab(path, 4096), O.Pool(now_ms=T0)
    n = 300
    reqs = np.zeros(n, dtype=G.REQ_DTYPE)
    xx, fv = key_hashes([7] * n, name="flip")
    reqs["key_xxh64"], reqs["key_fnv1"] = xx, fv
    reqs["hits"] = 1; reqs["limit"] = 10; reqs["duration"] = 60000; reqs["created_at"] = T0
    reqs["behavior"] = G.native.REQ_IS_OWNER | G.native.RESET_REMAINING
    _cmp(tab.submit(reqs, make_clock(T0), O.HRESP_DTYPE), pool.submit_hashed(reqs))
    _check_state(G, tab, pool)


@both_paths
def test_ragged_sizes_and_chunking(G, path):
    rng = np.random.default_rng(5)
    tab, pool = Tab(path, 1 << 12, max_batch=1024), O.Pool(now_ms=T0)
    assert len(tab.submit(np.zeros(0, dtype=G.REQ_DTYPE), make_clock(T0), O.HRESP_DTYPE)) == 0
    for n in (1, 2, 31, 32, 33, 255, 257, 1023, 1024, 1025, 2500):  # the last two cross the max_batch chunking
        reqs = adversarial_batch(rng, n, 50, T0)
        _cmp(tab.submit(reqs, make_clock(T0), O.HRESP_DTYPE), pool.submit_hashed(reqs), f"n={n}")
    _check_state(G, tab, pool)


@both_paths
def test_sentinel_hashes_table_full_and_sweep(G, path):
    tab, pool = Tab(path, 4096), O.Pool(now_ms=T0)
    reqs = np.zeros(8, dtype=G.REQ_DTYPE)
    reqs["key_xxh64"] = [0, 1, 2, 3, 0, 1, 2, 3]
    reqs["key_fnv1"] = [10 << 8, 11 << 8, 12 << 8, 13 << 8, 10 << 8, 11 << 8, 12 << 8, 13 << 8]
    reqs["hits"] = 1; reqs["limit"] = 5; reqs["duration"] = 1000; reqs["created_at"] = T0
    _cmp(tab.submit(reqs, make_clock(T0), O.HRESP_DTYPE), pool.submit_hashed(reqs))
    # a table far too small for the batch: the reference's LRU would evict (lrucache.go:98,138-149) and still answer every request;
    # so do we: keys whose probe window is full are parked and placed, with eviction, before the next batch reads the table
    small = Tab(path, 64)
    n = 1500
    reqs = np.zeros(n, dtype=G.REQ_DTYPE)
    xx, fv = key_hashes(np.arange(n), name="full")
    reqs["key_xxh64"], reqs["key_fnv1"] = xx, fv
    reqs["hits"] = 1; reqs["limit"] = 5; reqs["duration"] = 100000; reqs["created_at"] = T0 + np.arange(n)  # key i expires at T0 + 100000 + i
    big = O.Pool(now_ms=T0)
    out = small.submit(reqs, make_clock(T0), O.HRESP_DTYPE)
    _cmp(out, big.submit_hashed(reqs), "every request is answered as if the cache had room")
    c = small.counters()
    assert len(small.scan(G.ITEM_DTYPE)) == 64 and c["inserts"] == 64
    assert c["table_full"] == n - 64 - 1024  # beyond the 1024 parked keys the state is dropped, and counted
    # the next batch places the parked keys first: each evicts the entry of its window that expires first
    again = reqs[-8:].copy()
    again["created_at"] = T0 + 5
    out = small.submit(again, make_clock(T0 + 5), O.HRESP_DTYPE)
    c = small.counters()
    assert c["unexpired_evictions"] == 1024 and np.all(out["err_code"] == 0)
    items = small.scan(G.ITEM_DTYPE)
    assert len(items) == 64
    # what survives is what expires last among the placed keys (the dropped ones never made it)
    assert items["expire_at"].min() > T0 + 100000 + 64
    assert small.sweep(T0 + 300000) == 64 and len(small.scan(G.ITEM_DTYPE)) == 0
    assert np.all(small.submit(reqs[:64], make_clock(T0 + 300000), O.HRESP_DTYPE)["err_code"] == 0)


def test_epoch_wrap(G):
    """16-bit epoch tags of the grouping table: batches on both sides of the wrap (the launcher clears the table at 65535)."""
    rng = np.random.default_rng(41)
    tab, pool = E.EmuTable(1 << 12, max_batch=1024), O.Pool(now_ms=T0)
    reqs = adversarial_batch(rng, 64, 5, T0)
    clk = make_clock(T0)
    _cmp(tab.submit(reqs, clk, O.HRESP_DTYPE), pool.submit_hashed(reqs), "first")
    tab.set_epoch(65530)
    for b in range(12):
        _cmp(tab.submit(reqs, clk, O.HRESP_DTYPE), pool.submit_hashed(reqs), f"batch {b} after epoch 65530")


def test_epoch_wrap_with_mixed_groups(G):
    """The wrap 65535 -> 1 keeps the epoch parity, so the batch after it reuses the allocator pair the batch before it filled
    (ADVICE r1): several hundred requests on a few keys (non-uniform groups on both sides of the wrap), state and counters checked."""
    rng = np.random.default_rng(43)
    tab, pool = E.EmuTable(1 << 12, max_batch=1024), O.Pool(now_ms=T0)
    clk = make_clock(T0)
    tab.set_epoch(65530)
    for b in range(10):
        reqs = adversarial_batch(rng, 600, 5, T0)
        _cmp(tab.submit(reqs, clk, O.HRESP_DTYPE), pool.submit_hashed(reqs), f"batch {b} after epoch 65530")
    c = tab.counters()
    assert c["requests"] == 6000 and c["mixed_groups"] <= 50


@both_paths
def test_compact_records_expand_like_the_full_ones(G, path):
    rng = np.random.default_rng(61)
    a, b, pool = Tab(path, 1 << 13), Tab(path, 1 << 13), O.Pool(now_ms=T0)
    for n_sets in (2, 32, 33):  # <= 32 sets travel in the kernel arguments (k_expand_inline), more by pointer (k_expand)
        now = T0 + n_sets
        pool.set_now(now)
        ids = zipf_ids(rng, 3000, 800, 1.1)
        reqs = bench_requests(ids, now)
        reqs["limit"] = 50 + (ids % n_sets)
        reqs["algorithm"] = (ids % n_sets) & 1
        creqs, params, base = G.native.compact_batch(reqs.astype(G.REQ_DTYPE))
        assert len(params) == n_sets
        want = pool.submit_hashed(reqs)
        _cmp(a.submit(reqs, make_clock(now), O.HRESP_DTYPE), want, f"full, {n_sets} sets")
        _cmp(b.submit_compact(creqs, params, base, make_clock(now), O.HRESP_DTYPE), want, f"compact, {n_sets} sets")
    creqs, params, base = G.native.compact_batch(adversarial_batch(rng, 10, 3, T0).astype(G.REQ_DTYPE))
    creqs["params"][3] = 10_000  # unknown parameter set: in-band error
    assert b.submit_compact(creqs, params, base, make_clock(T0), O.HRESP_DTYPE)["err_code"][3] == G.native.ERR_INVALID_ALGORITHM


def test_hash_kernel_matches_oracle_hashes():
    rng = np.random.default_rng(9)
    keys = [b"", b"a", b"bench_k000000042", b"x" * 31, b"y" * 32, b"z" * 33, b"w" * 100] + [bytes(rng.integers(0, 256, int(l), dtype=np.uint8))
                                                                                           for l in rng.integers(0, 90, 200)]
    xx, fv = E.hash_keys(keys)
    for k, x, f in zip(keys, xx, fv):
        assert int(x) == O.xxh64(k) and int(f) == O.fnv1_64(k), k


@pytest.mark.parametrize("world", [1, 2, 8])
def test_route_kernels_partition_stably_by_ring_owner(G, world):
    from gubernator_b200.sharded import shard_addresses
    oring = O.Ring(0, 512)
    for a in shard_addresses(world):
        oring.add(a)
    pts, peers = oring.points()
    rng = np.random.default_rng(world)
    for n in (1, 1000, 1024, 3333):
        reqs = bench_requests(zipf_ids(rng, n, 5000, 1.1), T0).astype(G.REQ_DTYPE)
        out, perm, counts, owner = E.route(reqs, pts, peers, world)
        want_owner = np.array([oring.get_by_hash(int(h)) for h in reqs["key_fnv1"]], dtype=np.int64)
        assert np.array_equal(owner.astype(np.int64), want_owner)
        order = np.argsort(want_owner, kind="stable")  # the stable partition, by definition
        assert np.array_equal(perm.astype(np.int64), order) and out.tobytes() == reqs[order].tobytes()
        assert np.array_equal(counts.astype(np.int64), np.bincount(want_owner, minlength=world))
        resps = np.zeros(n, dtype=O.HRESP_DTYPE)
        resps["remaining"] = np.arange(n)
        back = E.unroute(resps, perm)
        assert np.array_equal(back["remaining"][order], np.arange(n))


@pytest.mark.parametrize("world,path", [(1, "pipeline"), (2, "pipeline"), (4, "pipeline"), (8, "pipeline"), (1, "fused"), (2, "fused"), (4, "fused")])
def test_mailbox_routing_kernels_match_per_shard_oracles(G, world, path):
    """gub_p2p.cuh (partition + stores into the owners' mailboxes, gather, device-side batch size, responses back, un-route)
    for W shards in one process: every response equals what one oracle per shard gives when it applies the records of source 0
    (in index order), then source 1, ... — the order tests/test_gpu_p2p.py checks on the GPU."""
    from gubernator_b200.sharded import shard_addresses
    oring = O.Ring(0, 512)
    for a in shard_addresses(world):
        oring.add(a)
    pts, peers = oring.points()
    cl = E.EmuP2PCluster(world, cap=2048, capacity_slots=1 << 13, pts=pts, peers=peers, max_batch=2048, finish_cap=3,
                         fused=(path == "fused"))  # inbox > max_batch: the pipeline takes it in several passes
    sim = [O.Pool(workers=2, cache_size=10**7, now_ms=T0) for _ in range(world)]
    sizes = [[900, 1, 0, 2048, 5], [600, 0, 0, 2048, 300], [1, 1500, 0, 100, 2048], [2048, 0, 0, 7, 300]]
    for step in range(5):
        now = T0 + step
        batches = []
        for r in range(world):
            rng = np.random.default_rng(77 * step + r)
            n = sizes[r % 4][step]
            if n == 0:
                batches.append(np.zeros(0, dtype=G.REQ_DTYPE))
            elif step % 2:
                batches.append(adversarial_batch(rng, n, 41, now).astype(G.REQ_DTYPE))
            else:
                batches.append(bench_requests(zipf_ids(rng, n, 3000, 1.1), now).astype(G.REQ_DTYPE))
        got = cl.step(batches, make_clock(now), O.HRESP_DTYPE)
        owners = [np.array([oring.get_by_hash(int(h)) for h in b["key_fnv1"]], dtype=np.int64) for b in batches]
        want = [np.zeros(len(b), dtype=O.HRESP_DTYPE) for b in batches]
        for gi in range(world):
            sim[gi].set_now(now)
            for s_ in range(world):
                idx = np.nonzero(owners[s_] == gi)[0]
                if len(idx):
                    want[s_][idx] = sim[gi].submit_hashed(np.ascontiguousarray(batches[s_][idx]))
        for r in range(world):
            _cmp(got[r], want[r], f"step {step} shard {r}")


def test_keys_colliding_in_the_grouping_table(G):
    """Two different keys that share the batch-wide grouping entry (same home position and the same 24-bit tag = top bits of the
    XXH64): they are grouped as one run, found different from the representative, and walked key by key in k_finish.  When both
    have requests in the same block, k_group has to fold their fragments into one (merge_colliding_fragments) — this test found
    that case broken (duplicate ranks) before the fold existed."""
    max_batch = 1024
    mask = 4 * max_batch - 1                          # aux entries - 1 (gub_create: next_pow2(4 * max_batch))
    rng = np.random.default_rng(2024)
    top = np.uint64(0xABCDEF) << np.uint64(40)
    lows = rng.integers(2, 1 << 40, 4000).astype(np.uint64)
    keys = top | lows
    home = ((keys ^ (keys >> np.uint64(29))) & np.uint64(mask)).astype(np.int64)
    order = np.argsort(home, kind="stable")
    same = np.nonzero(np.diff(home[order]) == 0)[0]
    assert len(same) > 0
    ka, kb = keys[order[same[0]]], keys[order[same[0] + 1]]
    assert ka != kb
    tab, pool = E.EmuTable(4096, max_batch=max_batch), O.Pool(now_ms=T0)
    for step in range(3):
        now = T0 + step
        pool.set_now(now)
        n = 600
        reqs = np.zeros(n, dtype=G.REQ_DTYPE)
        pick = rng.integers(0, 3, n)
        reqs["key_xxh64"] = np.where(pick == 0, ka, np.where(pick == 1, kb, keys[rng.integers(0, 50, n)]))
        reqs["key_fnv1"] = (reqs["key_xxh64"] * np.uint64(0x9E3779B97F4A7C15)) | np.uint64(0x100)
        reqs["hits"] = 1 if step < 2 else rng.integers(0, 3, n)
        reqs["limit"] = 500; reqs["duration"] = 60000; reqs["created_at"] = now
        reqs["algorithm"] = (reqs["key_xxh64"] & np.uint64(1)).astype(np.uint32); reqs["behavior"] = G.native.REQ_IS_OWNER
        _cmp(tab.submit(reqs, make_clock(now), O.HRESP_DTYPE), pool.submit_hashed(reqs), f"step {step}")
    assert tab.counters()["mixed_groups"] > 0
    _check_state(G, tab, pool)


def test_colliding_keys_in_few_long_segments(G):
    """The same collision, but each key's requests are contiguous: two segments, planned by plan_run with a cursor switch between them
    (the test above, with its random interleaving, ends in the serial walk)."""
    max_batch = 1024
    rng = np.random.default_rng(2024)
    keys = (np.uint64(0xABCDEF) << np.uint64(40)) | rng.integers(2, 1 << 40, 4000).astype(np.uint64)
    home = ((keys ^ (keys >> np.uint64(29))) & np.uint64(4 * max_batch - 1)).astype(np.int64)
    order = np.argsort(home, kind="stable")
    same = np.nonzero(np.diff(home[order]) == 0)[0]
    ka, kb = keys[order[same[0]]], keys[order[same[0] + 1]]
    tab, pool = E.EmuTable(4096, max_batch=max_batch), O.Pool(now_ms=T0)
    for step in range(2):
        now = T0 + step
        pool.set_now(now)
        n = 500
        reqs = np.zeros(n, dtype=G.REQ_DTYPE)
        reqs["key_xxh64"] = np.where(np.arange(n) < 230, ka, kb)  # both keys inside block 0, kb alone in block 1
        reqs["key_fnv1"] = (reqs["key_xxh64"] * np.uint64(0x9E3779B97F4A7C15)) | np.uint64(0x100)
        reqs["hits"] = 1; reqs["limit"] = 300; reqs["duration"] = 60000; reqs["created_at"] = now
        reqs["algorithm"] = step; reqs["behavior"] = G.native.REQ_IS_OWNER
        _cmp(tab.submit(reqs, make_clock(now), O.HRESP_DTYPE), pool.submit_hashed(reqs), f"step {step}")
    c = tab.counters()
    assert c["mixed_groups"] == 2 and c["serial_fallbacks"] == 0
    _check_state(G, tab, pool)


@both_paths
def test_probe_window_wraps_and_skips_tombstones(G, path):
    """Keys whose home slot is at the very end of a small table (the linear probe wraps to slot 0), expiring at different times:
    after a sweep the survivors are found behind tombstones and new keys reuse the freed slots."""
    cap = 256
    rng = np.random.default_rng(8)
    cand = rng.integers(2, 1 << 62, 200000).astype(np.uint64) | (np.uint64(0xFF) << np.uint64(56))  # home = (key * cap) >> 64 = 255
    keys = np.unique(cand)[:60]
    assert np.all((keys >> np.uint64(56)) == 255)
    tab, pool = Tab(path, cap), O.Pool(now_ms=T0)

    def batch(ks, now, duration):
        r = np.zeros(len(ks), dtype=G.REQ_DTYPE)
        r["key_xxh64"] = ks; r["key_fnv1"] = (ks * np.uint64(0x9E3779B97F4A7C15)) | np.uint64(0x100)
        r["hits"] = 1; r["limit"] = 10; r["duration"] = duration; r["created_at"] = now
        r["algorithm"] = (ks & np.uint64(1)).astype(np.uint32); r["behavior"] = G.native.REQ_IS_OWNER
        return r
    first = batch(keys[:40], T0, np.where(np.arange(40) % 2 == 0, 1000, 100000))  # every other item is short-lived
    _cmp(tab.submit(first, make_clock(T0), O.HRESP_DTYPE), pool.submit_hashed(first), "fill")
    now = T0 + 5000
    pool.set_now(now)
    assert tab.sweep(now) == 20
    again = batch(np.concatenate([keys[:40], keys[40:60]]), now, 100000)  # survivors, re-created short-lived ones, brand-new keys
    rng.shuffle(again)
    _cmp(tab.submit(again, make_clock(now), O.HRESP_DTYPE), pool.submit_hashed(again), "after the sweep")
    _check_state(G, tab, pool)


@pytest.mark.parametrize("seed,n_keys", [(0, 2500), (5, 1200)])
def test_fuzz_with_frequent_grouping_collisions(G, seed, n_keys):
    """Adversarial traffic over a key space with only 48 distinct 24-bit tags and a 4096-entry grouping table: several pairs (and
    triples) of different keys share a group entry in every batch, inside and across blocks."""
    rng, krng = np.random.default_rng(900 + seed), np.random.default_rng(seed)
    tags = krng.integers(0, 1 << 24, 48).astype(np.uint64)
    newk = (tags[krng.integers(0, len(tags), 8000)] << np.uint64(40)) | krng.integers(2, 1 << 40, 8000).astype(np.uint64)
    tab, pool = E.EmuTable(1 << 13, max_batch=1024), O.Pool(now_ms=T0)
    now = T0
    for step in range(3):
        now += int(rng.choice([0, 1, 900]))
        pool.set_now(now)
        reqs = adversarial_batch(rng, 3000, n_keys, now).astype(G.REQ_DTYPE)
        reqs["key_xxh64"] = newk[(reqs["key_xxh64"] % np.uint64(len(newk))).astype(np.int64)]
        reqs["key_fnv1"] = (reqs["key_xxh64"] * np.uint64(0x9E3779B97F4A7C15)) | np.uint64(0x100)
        _cmp(tab.submit(reqs, make_clock(now), O.HRESP_DTYPE), pool.submit_hashed(reqs), f"step {step}")
    _check_state(G, tab, pool)


# ---- the reference's own known-answer tables through the emulated kernels -----------------------------------------------------
class _EmuInstance:
    """The frozen-clock backend tests/kat_player.py expects, over the emulated kernels: the host-side steps of
    V1Instance.GetRateLimits (gubernator.go:203-220: field checks, CreatedAt default, HashKey) are restated here in Python; hashes
    come from the oracle's XXH64 / FNV-1, error strings from the product's gub_format_error."""

    def __init__(self, G, now_ms):
        import ctypes as C
        self.G, self.C, self._now = G, C, now_ms
        self.tab = E.EmuTable(1 << 12)
        self.L = G.native.lib()
        self.L.gub_format_error.argtypes = [C.c_int, C.c_char_p, C.c_int32, C.c_char_p, C.c_size_t]

    def now(self):
        return self._now

    def advance(self, ms):
        self._now += ms

    def _err(self, code, key, algorithm):
        buf = self.C.create_string_buffer(512)
        self.L.gub_format_error(code, key, algorithm, buf, 512)
        return buf.value.decode()

    def get_rate_limits(self, reqs):
        G = self.G
        out = [None] * len(reqs)
        rec, where = np.zeros(len(reqs), dtype=G.REQ_DTYPE), []
        for i, r in enumerate(reqs):
            name, uk = r.get("name", ""), r.get("unique_key", "")
            if uk == "" or name == "":  # unique_key is checked first (gubernator.go:208-217)
                code = G.native.ERR_UNIQUE_KEY_EMPTY if uk == "" else G.native.ERR_NAMESPACE_EMPTY
                out[i] = dict(status=0, limit=0, remaining=0, reset_time=0, error=self._err(code, b"", 0))
                continue
            key = (name + "_" + uk).encode()
            k = len(where)
            rec[k]["key_xxh64"], rec[k]["key_fnv1"] = O.xxh64(key), O.fnv1_64(key)
            for f in ("hits", "limit", "duration", "burst", "algorithm"):
                rec[k][f] = r.get(f, 0)
            rec[k]["behavior"] = r.get("behavior", 0) | G.native.REQ_IS_OWNER
            rec[k]["created_at"] = r.get("created_at", 0) or self._now
            where.append((i, key, r.get("algorithm", 0)))
        resp = self.tab.submit(rec[:len(where)], make_clock(self._now), O.HRESP_DTYPE)
        for (i, key, algo), o in zip(where, resp):
            err = self._err(int(o["err_code"]), key, algo) if o["err_code"] else ""
            out[i] = dict(status=int(o["status"]), limit=int(o["limit"]), remaining=int(o["remaining"]), reset_time=int(o["reset_time"]), error=err)
        return out


def test_reference_scenarios_through_the_emulated_kernels(G):
    """functional_test.go's tables (tests/golden/reference_kat.py) played against the CUDA kernel source on the CPU."""
    from golden import reference_kat as K
    from kat_player import play_missing_fields, play_scenario
    for sc in K.SCENARIOS:
        play_scenario(_EmuInstance(G, K.T0), sc)
    play_missing_fields(_EmuInstance(G, K.T0))


# ---- the bodies of GPU tests, run against the emulated kernels ----------------------------------------------------------------
class _TableLike:
    """gubernator_b200.native.Table's surface over the emulated kernels, so that test functions written for the GPU can be run
    here unchanged: it checks the test code and the kernel logic, not the hardware."""

    def __init__(self, G, capacity_slots, max_batch=65536, device=0):
        self._G, self._t = G, E.EmuTable(capacity_slots, max_batch=max_batch)

    def submit(self, reqs, clk, out=None):
        return self._t.submit(reqs, clk, self._G.RESP_DTYPE)

    def submit_compact(self, creqs, params, created_base, clk, out=None):
        return self._t.submit_compact(creqs, params, created_base, clk, self._G.RESP_DTYPE)

    def scan(self):
        return self._t.scan(self._G.ITEM_DTYPE)

    def size(self):
        return len(self.scan())

    def sweep(self, now_ms):
        return self._t.sweep(now_ms)

    def counters(self):
        return self._t.counters()

    def probe_random_access(self, accesses=1 << 26):
        self._t.random_rmw(accesses)
        return 1.0


def _fake_g(G):
    import types
    return types.SimpleNamespace(Table=lambda *a, **k: _TableLike(G, *a, **k), REQ_DTYPE=G.REQ_DTYPE, RESP_DTYPE=G.RESP_DTYPE, ITEM_DTYPE=G.ITEM_DTYPE,
                                 native=G.native, clock_fill=G.clock_fill)


# (test_compact_requests_equal_full_records and test_random_access_probe_leaves_table_unchanged run the same way — a minute of
# fibers between them; test_compact_records_expand_like_the_full_ones above covers the compact path at emulator size)
@pytest.mark.parametrize("name", ["test_keys_colliding_in_the_grouping_table"])
def test_gpu_test_bodies_on_the_emulator(G, name):
    """The GPU tests added after this round's last GPU run (any other function of tests/test_gpu_parity.py that only uses the Table
    surface above can be run the same way)."""
    import test_gpu_parity as gpu_tests
    getattr(gpu_tests, name)(_fake_g(G))


@pytest.mark.parametrize("keep_latest", [False, True])
def test_global_queues_match_the_reference_maps(G, keep_latest):
    """gub_global.cuh against a dict model of global.go: the hits queue (runAsyncHits, global.go:91-141) keeps the FIRST request of a
    key with Hits summed over the window and RESET_REMAINING OR-ed in, for keys this shard does not own; the updates queue
    (runBroadcasts, global.go:193-231) keeps the LATEST request seen.  Draining empties the queue."""
    N = G.native
    rng = np.random.default_rng(17 + keep_latest)
    q = E.EmuGq(capacity=256, keep_latest=keep_latest)
    self_index, seq = 1, 0
    for window in range(3):
        model = {}
        for batch in range(3):
            n = int(rng.choice([1, 40, 300]))
            reqs = np.zeros(n, dtype=G.REQ_DTYPE)
            ids = rng.integers(0, 25, n)
            reqs["key_xxh64"], reqs["key_fnv1"] = key_hashes(ids, name="gq")
            reqs["hits"] = rng.integers(-2, 4, n); reqs["limit"] = rng.integers(1, 50, n); reqs["duration"] = rng.choice([1000, 60000], n)
            reqs["created_at"] = T0 + rng.integers(0, 9, n); reqs["algorithm"] = ids & 1
            reqs["behavior"] = (rng.choice([0, N.GLOBAL, N.GLOBAL, N.GLOBAL | N.RESET_REMAINING], n) | N.REQ_IS_OWNER).astype(np.uint32)
            owner = rng.integers(0, 3, n).astype(np.uint8)
            q.accumulate(reqs, None if keep_latest else owner, self_index, seq)
            for i in range(n):
                r = reqs[i]
                if not (int(r["behavior"]) & N.GLOBAL) or int(r["hits"]) == 0:
                    continue
                if not keep_latest and int(owner[i]) == self_index:
                    continue
                k = int(r["key_xxh64"])
                if k not in model:
                    model[k] = dict(first=r.copy(), last=r.copy(), hits=0, reset=0)
                m = model[k]
                m["hits"] += int(r["hits"]); m["last"] = r.copy(); m["reset"] |= int(r["behavior"]) & N.RESET_REMAINING
            seq += n
        got = q.drain(G.REQ_DTYPE, as_status_query=keep_latest)
        assert len(got) == len(model) == len(set(got["key_xxh64"].tolist()))
        for e in got:
            m = model[int(e["key_xxh64"])]
            src = m["last"] if keep_latest else m["first"]
            for f in ("key_fnv1", "limit", "duration", "burst", "created_at", "algorithm"):
                assert e[f] == src[f], (f, e, src)
            if keep_latest:   # status query for the broadcast: Hits = 0, evaluated with IsOwner = false (global.go:238-245)
                assert int(e["hits"]) == 0 and int(e["behavior"]) == int(src["behavior"]) & ~N.REQ_IS_OWNER
            else:             # forwarded to the owner: summed hits, DRAIN_OVER_LIMIT added there (gubernator.go:510-512)
                assert int(e["hits"]) == m["hits"]
                assert int(e["behavior"]) == int(src["behavior"]) | m["reset"] | N.DRAIN_OVER_LIMIT | N.REQ_IS_OWNER
        assert len(q.drain(G.REQ_DTYPE, as_status_query=keep_latest)) == 0  # drained


def test_update_items_built_from_status_queries(G):
    """k_make_updates: the CacheItem a peer installs for an UpdatePeerGlobal (gubernator.go:427-451)."""
    q = np.zeros(3, dtype=G.REQ_DTYPE)
    q["key_xxh64"] = [11, 12, 13]; q["key_fnv1"] = [21 << 8, 22 << 8, 23 << 8]; q["duration"] = [1000, 2000, 3000]; q["algorithm"] = [0, 1, 7]
    r = np.zeros(3, dtype=O.HRESP_DTYPE)
    r["status"] = [1, 0, 0]; r["limit"] = [10, 20, 30]; r["remaining"] = [0, 7, 1]; r["reset_time"] = [T0 + 5, T0 + 6, T0 + 7]
    items = E.make_updates(q, r, G.ITEM_DTYPE)
    assert len(items) == 2  # the invalid algorithm is skipped (logged in the reference, global.go:246-249)
    by = {int(i["key_xxh64"]): i for i in items}
    t, l = by[11], by[12]
    assert (int(t["algorithm"]), int(t["status"]), int(t["limit"]), int(t["duration"]), int(t["remaining"]), int(t["expire_at"])) == (0, 1, 10, 1000, 0, T0 + 5)
    assert (int(l["algorithm"]), int(l["limit"]), int(l["duration"]), float(l["remaining_f"]), int(l["burst"]), int(l["expire_at"])) == (1, 20, 2000, 7.0, 20, T0 + 6)


def test_global_queue_overflow_drops_whole_keys(G):
    """More GLOBAL keys in one window than the queue has slots: the surplus keys are not queued (their hits are not synchronised in
    this window — the reference's map is unbounded, so size the queue for the hot set), the ones that are queued stay exact."""
    N = G.native
    q = E.EmuGq(capacity=64, keep_latest=False)
    n = 200
    reqs = np.zeros(n, dtype=G.REQ_DTYPE)
    reqs["key_xxh64"], reqs["key_fnv1"] = key_hashes(np.arange(100).repeat(2), name="gqo")
    reqs["hits"] = 3; reqs["limit"] = 9; reqs["duration"] = 1000; reqs["created_at"] = T0
    reqs["behavior"] = N.GLOBAL | N.REQ_IS_OWNER
    q.accumulate(reqs, np.zeros(n, dtype=np.uint8), 1, 0)
    got = q.drain(G.REQ_DTYPE, as_status_query=False)
    assert len(got) == 64 and len(set(got["key_xxh64"].tolist())) == 64
    assert np.all(got["hits"] == 6) and np.all(got["limit"] == 9)


@both_paths
def test_global_flow_on_bench_like_traffic_matches_the_cluster_model(G, path):
    """BASELINE config 5 in small: two shards, the hot keys (top of the Zipf ranking) carry GLOBAL, both algorithms, the clock
    advances 35 ms per step (limit 100 per 60 s: a leaky token per 600 ms), a sync tick after warm-up and two at the end.  The
    whole flow runs on the emulated kernels — routing with GLOBAL requests kept on the non-owner, the ring-mode pipeline, the hits /
    updates queues, status queries, k_make_updates, replica install — orchestrated like gub_global_tick, and is compared with the
    oracle cluster model (tests/global_model.py): every response of every step, and the answers of both shards to a Hits = 0 query
    on every hot key after the quiesced ticks."""
    import importlib.util
    import os
    from global_model import OracleCluster
    from gubernator_b200.sharded import shard_addresses
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(root, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    W, n_keys, per_step, dt = 2, 200000, 4096, 35
    steps = 60 if path == "pipeline" else 14  # (a persistent-kernel step costs several times the fibers)
    hot = n_keys // 100
    oring = O.Ring(0, 512)
    for a in shard_addresses(W):
        oring.add(a)
    pts, peers = oring.points()
    cl = E.EmuP2PCluster(W, cap=per_step, capacity_slots=1 << 16, pts=pts, peers=peers, max_batch=W * per_step, fused=(path == "fused"))
    model = OracleCluster(W, T0)
    hits_q = [E.EmuGq(capacity=1 << 13, keep_latest=False) for _ in range(W)]
    upd_q = [E.EmuGq(capacity=1 << 13, keep_latest=True) for _ in range(W)]
    rngs = [np.random.default_rng(900 + r) for r in range(W)]
    seq = [0]

    def evaluated_at(g, batches, owners):
        """The records shard g evaluated in a global-mode step, in evaluation order (source rank, then source index)."""
        parts = []
        for s_, b in enumerate(batches):
            is_global = (b["behavior"] & O.GLOBAL) != 0
            dest = np.where(is_global & (owners[s_] != s_), s_, owners[s_])
            sel = dest == g
            ev = b[sel].copy()
            local = (is_global & (owners[s_] != s_))[sel]
            ev["behavior"][local] = (ev["behavior"][local] | O.NO_BATCHING) & ~np.uint32(O.GLOBAL | O.REQ_IS_OWNER)
            parts.append(ev)
        return np.concatenate(parts) if parts else np.zeros(0, dtype=G.REQ_DTYPE)

    def step(batches, now):
        clk = make_clock(now)
        got, owners = cl.step(batches, clk, O.HRESP_DTYPE, global_mode=True)
        owners = [o.astype(np.int64) for o in owners]
        for r in range(W):
            hits_q[r].accumulate(batches[r], owners[r].astype(np.uint8), r, seq[0] << 32)
            upd_q[r].accumulate(evaluated_at(r, batches, owners), None, r, seq[0] << 32)
        seq[0] += 1
        return got

    def tick(now):
        clk = make_clock(now)
        recs = [hits_q[r].drain(G.REQ_DTYPE, False, cap=1 << 13) for r in range(W)]       # phase A: hits to their owners ...
        cl.step(recs, clk, O.HRESP_DTYPE)                                                   # ... evaluated there (phase B)
        owners = [np.array([oring.get_by_hash(int(h)) for h in b["key_fnv1"]], dtype=np.int64) for b in recs]
        for g in range(W):
            ev = np.concatenate([recs[s_][owners[s_] == g] for s_ in range(W)])
            upd_q[g].accumulate(ev, None, g, seq[0] << 32)
        seq[0] += 1
        for g in range(W):                                                                  # phase C + install
            q = upd_q[g].drain(G.REQ_DTYPE, True, cap=1 << 13)
            if not len(q):
                continue
            resp = cl.table(g).submit(q, clk, O.HRESP_DTYPE)
            items = E.make_updates(q, resp, G.ITEM_DTYPE)
            for p_ in range(W):
                if p_ != g:
                    cl.install(p_, items, now)

    def batch(r, now):
        return bench.gen_batch(rngs[r], per_step, n_keys, now, 1.1, G.REQ_DTYPE, global_hot=hot)[0]
    now = T0
    for b in range(steps):
        now = T0 + 1 + dt * b
        batches = [batch(r, now) for r in range(W)]
        got, want = step(batches, now), model.step([x.astype(O.HREQ_DTYPE) for x in batches], now)
        for r in range(W):
            _cmp(got[r], want[r], f"step {b} shard {r}")
        if b == 4:
            tick(now); model.tick(now)
    tick(now); model.tick(now)
    tick(now); model.tick(now)
    q = bench_requests(np.arange(hot, dtype=np.int64), now).astype(G.REQ_DTYPE)
    q["hits"] = 0
    q["behavior"] = np.uint32(O.GLOBAL | O.REQ_IS_OWNER)
    got = step([q.copy() for _ in range(W)], now)
    want = model.step([q.astype(O.HREQ_DTYPE) for _ in range(W)], now)
    for r in range(W):
        _cmp(got[r], want[r], f"convergence query shard {r}")
    tok = q["algorithm"] == 0
    assert np.array_equal(got[0][tok], got[1][tok])  # the reference's own consistency check (functional_test.go:1816-1821)
