"""CPU checks of the exact header the CUDA kernels include (gubernator_b200/csrc/bucket_math.cuh):
apply_one() against the oracle, and plan_run()/eval_piece() against repeated apply_one()."""
import numpy as np
import pytest

import edge_states as ES
import oracle_py as O
from _host_math import BUCKET_DTYPE, F_LEAKY, F_LIVE, F_OVER, HostTable, apply_one, lib, plan_check, rank_check
from workloads import T0, adversarial_batch, bench_batch, extreme_batch, make_clock


def _cmp(a, b):
    if not np.array_equal(a, b):
        bad = np.nonzero(a != b)[0]
        i = int(bad[0])
        raise AssertionError(f"{len(bad)} mismatches; first at {i}: got {a[i]} want {b[i]}")


@pytest.mark.parametrize("seed", range(6))
def test_apply_one_matches_oracle_adversarial(seed):
    rng = np.random.default_rng(100 + seed)
    pool = O.Pool(workers=4, cache_size=10_000_000, now_ms=T0)
    host = HostTable()
    now = T0
    for batch in range(12):
        now += int(rng.choice([0, 1, 7, 1000, 31000, 61000, 3_700_000]))
        pool.set_now(now)
        clk = make_clock(now)
        reqs = adversarial_batch(rng, 3000, int(rng.choice([3, 40, 400])), now)
        want = pool.submit_hashed(reqs)
        got, ctr = host.apply_seq(reqs, clk)
        _cmp(got, want)
        oc = pool.counters()
        assert (ctr["over_limit"], ctr["cache_hit"], ctr["cache_miss"]) == (oc["over_limit"], oc["cache_hit"], oc["cache_miss"])


def test_apply_one_matches_oracle_bench_traffic():
    rng = np.random.default_rng(5)
    pool = O.Pool(workers=8, cache_size=10_000_000, now_ms=T0)
    host = HostTable()
    for b in range(6):
        now = T0 + b * 20000
        pool.set_now(now)
        reqs, _ = bench_batch(rng, 20000, 5000, now, zipf_s=1.1, mixed=True)
        _cmp(host.apply_seq(reqs, make_clock(now))[0], pool.submit_hashed(reqs))


_EDGE = ES.buckets(BUCKET_DTYPE)


def _rand_bucket(rng, now):
    if rng.random() < 0.25:  # a state only a Store or Loader installs (edge_states.py)
        return _EDGE[int(rng.integers(0, len(_EDGE)))][None].copy()
    b = np.zeros(1, dtype=BUCKET_DTYPE)
    leaky = rng.random() < 0.5
    b["flags"] = (F_LIVE if rng.random() < 0.9 else 0) | (F_LEAKY if leaky else 0) | (F_OVER if (not leaky and rng.random() < 0.2) else 0)
    b["limit"] = int(rng.choice([0, 1, 5, 10, 100, 2000]))
    b["duration"] = int(rng.choice([0, 5, 1000, 60000]))
    if leaky:
        rem = float(rng.choice([0.0, 0.25, 1.0, 3.5, 9.999, 57.7, 100.0, 1999.5, -2.5, 5e15]))
        b["rem"] = np.float64(rem).view(np.uint64)
        b["burst"] = int(rng.choice([1, 5, 10, 100, 2000]))
    else:
        b["rem"] = np.int64(rng.choice([0, 1, 2, 7, 10, 99, 100, 2000, -5])).view(np.uint64)
    b["stamp"] = now - int(rng.choice([0, 1, 500, 59000, 10**7]))
    b["expire"] = now + int(rng.choice([-1, 0, 1, 1000, 60000]))
    return b


@pytest.mark.parametrize("seed", range(4))
def test_plan_run_equals_repeated_apply(seed):
    rng = np.random.default_rng(900 + seed)
    now = T0 + 777
    clk = make_clock(now)
    n_linear = 0
    for trial in range(6000):
        b = _rand_bucket(rng, now)
        rq = np.zeros(1, dtype=O.HREQ_DTYPE)
        leaky_req = rng.random() < 0.5
        rq["algorithm"] = int(leaky_req) if rng.random() < 0.97 else 3
        rq["hits"] = int(rng.choice([0, 1, 1, 1, 2, 3, 10, -1, 5000]))
        rq["limit"] = int(b["limit"][0]) if rng.random() < 0.7 else int(rng.choice([0, 1, 10, 100]))
        rq["duration"] = int(b["duration"][0]) if rng.random() < 0.7 else int(rng.choice([0, 1, 2, 3, 9, 1000, 60000]))
        rq["burst"] = int(rng.choice([0, 0, int(b["burst"][0]), 7]))
        rq["behavior"] = int(rng.choice([0, 0, 0, 8, 32, 4, 4 | 32])) | int(rng.choice([0, O.REQ_IS_OWNER]))
        rq["created_at"] = now + int(rng.choice([0, 0, 1, -70000, 100000]))
        m = int(rng.choice([1, 2, 3, 10, 100, 1000, 7300]))
        cap = int(rng.choice([2, 4, 16]))
        rc, npieces, covered = plan_check(b, rq, m, clk, cap)
        assert rc == 0, (trial, rc, b, rq, m, cap)
        rc = rank_check(b, rq, m, clk, stride=1 if m <= 100 else 37)
        assert rc == 0, ("run_to_rank", trial, rc, b, rq, m)
        if covered == m and npieces < m:
            n_linear += 1
    assert n_linear > 500  # the planner actually compresses runs


def test_plan_run_compresses_hot_key_run():
    # BASELINE config 3: hits=1, limit=100 on an existing bucket, 7300 identical requests
    now = T0
    clk = make_clock(now)
    for algo in (0, 1):
        b = np.zeros(1, dtype=BUCKET_DTYPE)
        rq = np.zeros(1, dtype=O.HREQ_DTYPE)
        rq["algorithm"] = algo; rq["hits"] = 1; rq["limit"] = 100; rq["duration"] = 60000; rq["created_at"] = now
        rq["behavior"] = O.REQ_IS_OWNER
        rc, npieces, covered = plan_check(b, rq, 7300, clk, 16)
        assert rc == 0 and covered == 7300 and npieces <= 6, (algo, rc, npieces, covered)
        assert rank_check(b, rq, 7300, clk, stride=1) == 0


@pytest.mark.parametrize("seed", range(3))
def test_apply_one_matches_oracle_on_numeric_extremes(seed):
    """int64 wrap-around, float64 beyond 2^52 / 2^63, Go's int64(float64) on overflow and NaN, negative limits/durations."""
    rng = np.random.default_rng(4000 + seed)
    pool = O.Pool(workers=3, cache_size=10_000_000, now_ms=T0)
    host = HostTable()
    now = T0
    for batch in range(10):
        now += int(rng.choice([0, 1, 1000, 61000]))
        pool.set_now(now)
        reqs = extreme_batch(rng, 4000, int(rng.choice([5, 60, 900])), now)
        want = pool.submit_hashed(reqs)
        got, ctr = host.apply_seq(reqs, make_clock(now))
        _cmp(got, want)
        oc = pool.counters()
        assert (ctr["over_limit"], ctr["cache_hit"], ctr["cache_miss"]) == (oc["over_limit"], oc["cache_hit"], oc["cache_miss"])


def _check_loaded_state(b, it, what):
    """A slot image after apply_one against the oracle's CacheItem for the same key, bit for bit."""
    assert (int(b["limit"]), int(b["duration"]), int(b["stamp"]), int(b["expire"])) == (it.limit, it.duration, it.stamp, it.expire_at), what
    if it.value_kind == 2:
        assert int(b["flags"]) & F_LEAKY and int(b["burst"]) == it.burst, what
        assert int(b["rem"]) == ES.oracle_rem_bits(it), (what, hex(int(b["rem"])), hex(ES.oracle_rem_bits(it)))
    else:
        assert not int(b["flags"]) & F_LEAKY and int(b["rem"]) == it.remaining_i % (1 << 64) and bool(int(b["flags"]) & F_OVER) == (it.status == 1), what


@pytest.mark.parametrize("seed", range(2))
def test_apply_one_matches_oracle_on_loaded_states(seed):
    """Every lattice state of edge_states.py, loaded into the oracle bit for bit, under requests drawn around it: one apply_one()
    per (state, request) pair gives the oracle's response, counters and stored item."""
    rng = np.random.default_rng(7100 + seed)
    b, rq, _, idx = ES.pairs(rng, 40000, BUCKET_DTYPE, O.HREQ_DTYPE)
    its = ES.items()
    pool = O.Pool(workers=4, cache_size=10_000_000, now_ms=ES.NOW)
    for i in range(len(rq)):
        pool.add_item_hashed(rq["key_xxh64"][i], rq["key_fnv1"][i], ES.oracle_item(its[idx[i]]))
    clk = make_clock(ES.NOW)
    got, after, d = apply_one(lib(), b, rq, clk)
    _cmp(got, pool.submit_hashed(rq))
    oc = pool.counters()
    assert (int(d["over"].sum()), int(d["hit"].sum()), int(d["miss"].sum())) == (oc["over_limit"], oc["cache_hit"], oc["cache_miss"])
    held = pool.each()
    live = (after["flags"] & F_LIVE) != 0
    assert len(held) == int(live.sum())
    for i in np.nonzero(live)[0]:
        _check_loaded_state(after[i], held[(int(rq["key_xxh64"][i]), int(rq["key_fnv1"][i]))], (i, b[i], rq[i]))
