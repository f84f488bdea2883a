"""Consecutive batches on one stream with no synchronisation in between, on the single-table pipeline: the next batch's k_group groups
its keys while the current batch is still evaluated (two grouping scratch sets, early hand-off from k_finish to k_group).  Responses
and the final table (by scan) are compared bit for bit with the oracle."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle_py as O
from workloads import T0, adversarial_batch, bench_requests, zipf_ids

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def G():
    if os.environ.get("GUB_PATH") == "fused":
        pytest.skip("the early hand-off is a property of the four-kernel pipeline")
    import gubernator_b200 as g
    return g


@pytest.fixture(scope="module")
def torch():
    import torch as t
    if not t.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return t


def _cmp(got, want, what=""):
    if not np.array_equal(got, want):
        bad = np.nonzero(got != want)[0]
        i = int(bad[0])
        raise AssertionError(f"{what}: {len(bad)} of {len(got)} responses differ; first at {i}: got {got[i]} want {want[i]}")


def _dev(torch, reqs):
    return torch.from_numpy(np.ascontiguousarray(reqs).view(np.uint8).reshape(len(reqs), 64)).cuda()


def _host(G, d_out, n):
    return d_out[:n].cpu().numpy().reshape(-1).view(G.RESP_DTYPE)


def _check_table(G, tab, pool):
    scan = tab.scan()
    items = pool.each()
    dev = {(int(s["key_xxh64"]), int(s["key_fnv1"]) >> 8): s for s in scan}
    assert len(dev) == len(scan) == len(items)
    for (kx, kf), it in items.items():
        s = dev[(kx if kx >= 2 else kx + 2, kf >> 8)]
        assert (int(s["limit"]), int(s["duration"]), int(s["stamp"]), int(s["expire_at"])) == (it.limit, it.duration, it.stamp, it.expire_at)
        if it.value_kind == 2:
            assert np.float64(s["remaining_f"]).view(np.uint64) == np.float64(it.remaining_f).view(np.uint64)
        else:
            assert int(s["remaining"]) == it.remaining_i and int(s["status"]) == it.status


def _zipf_steps(rng, steps, n, n_ids):
    """One batch per step over one id space (keys shared from batch to batch), stamped with the step's clock T0 + 10 b."""
    return [bench_requests(zipf_ids(rng, n, n_ids, 1.1), T0 + 10 * b) for b in range(steps)]


def test_back_to_back_zipf_batches(G, torch):
    """48 batches of 65 536 Zipf requests over 300 000 ids, submitted back to back on one stream."""
    rng = np.random.default_rng(101)
    tab, pool = G.Table(1 << 21), O.Pool(cache_size=10_000_000, now_ms=T0)
    steps = 48
    batches = _zipf_steps(rng, steps, 65536, 300_000)
    d_in = [_dev(torch, r) for r in batches]
    d_out = [torch.empty((65536, 32), dtype=torch.uint8, device="cuda") for _ in range(steps)]
    stream = torch.cuda.current_stream().cuda_stream
    for b in range(steps):
        tab.submit_device(d_in[b].data_ptr(), 65536, G.clock_fill(T0 + 10 * b), d_out[b].data_ptr(), stream)
    torch.cuda.synchronize()
    for b in range(steps):
        pool.set_now(T0 + 10 * b)
        _cmp(_host(G, d_out[b], 65536), pool.submit_hashed(batches[b]), f"batch {b}")
    _check_table(G, tab, pool)


def test_records_written_by_a_kernel_between_submissions(G, torch):
    """A torch kernel writes the next batch's records into the buffer the previous batch read, between every two submissions: k_group
    must see that k_finish of the previous batch has finished and wait before it reads them."""
    rng = np.random.default_rng(102)
    tab, pool = G.Table(1 << 21), O.Pool(cache_size=10_000_000, now_ms=T0)
    steps = 32
    batches = _zipf_steps(rng, steps, 65536, 300_000)
    src = [_dev(torch, r).view(torch.int64) for r in batches]
    cur = torch.empty((65536, 64), dtype=torch.uint8, device="cuda")
    d_out = [torch.empty((65536, 32), dtype=torch.uint8, device="cuda") for _ in range(steps)]
    stream = torch.cuda.current_stream().cuda_stream
    zero = torch.zeros((), dtype=torch.int64, device="cuda")
    for b in range(steps):
        torch.add(src[b], zero, out=cur.view(torch.int64))  # an elementwise kernel, not a copy
        tab.submit_device(cur.data_ptr(), 65536, G.clock_fill(T0 + 10 * b), d_out[b].data_ptr(), stream)
    torch.cuda.synchronize()
    for b in range(steps):
        pool.set_now(T0 + 10 * b)
        _cmp(_host(G, d_out[b], 65536), pool.submit_hashed(batches[b]), f"batch {b}")
    _check_table(G, tab, pool)


def test_mixed_groups_against_the_oracle(G, torch):
    """Adversarial batches (non-uniform groups, every behaviour bit, expiry) interleaved with Zipf ones, back to back."""
    rng = np.random.default_rng(103)
    tab, pool = G.Table(1 << 16, max_batch=4096), O.Pool(cache_size=10_000_000, now_ms=T0)
    now, reqs_all, nows = T0, [], []
    for b in range(40):
        now += int(rng.choice([0, 1, 900, 70000]))
        reqs_all.append(adversarial_batch(rng, 4096, 300, now) if b % 2 else bench_requests(zipf_ids(rng, 4096, 3000, 1.1), now))
        nows.append(now)
    d_in = [_dev(torch, r) for r in reqs_all]
    d_out = [torch.empty((4096, 32), dtype=torch.uint8, device="cuda") for _ in reqs_all]
    stream = torch.cuda.current_stream().cuda_stream
    for b, r in enumerate(reqs_all):
        tab.submit_device(d_in[b].data_ptr(), len(r), G.clock_fill(nows[b]), d_out[b].data_ptr(), stream)
    torch.cuda.synchronize()
    for b, r in enumerate(reqs_all):
        pool.set_now(nows[b])
        _cmp(_host(G, d_out[b], len(r)), pool.submit_hashed(r), f"batch {b}")
    assert tab.counters()["mixed_groups"] > 0
    _check_table(G, tab, pool)


def test_parked_inserts_and_sweep_back_to_back(G, torch):
    """A table far too small (inserts parked and placed with eviction at every batch), non-uniform groups and the scheduled sweep (a
    k_sweep launch between batches 1024 and 1025), 1100 batches back to back.  Every batch has keys of its own, repeated inside it, so
    its responses do not depend on which entries earlier batches evicted (the CAS races of a full window decide that): they equal the
    oracle's with room for all."""
    rng = np.random.default_rng(104)
    pool = O.Pool(cache_size=10_000_000, now_ms=T0)
    seq, nows = [], []
    for b in range(1100):
        now = T0 + 40 * b
        r = adversarial_batch(rng, 1024, 200, now)
        r["key_xxh64"] = r["key_xxh64"] * np.uint64(0x9E3779B97F4A7C15) + np.uint64(b)  # this batch's own keys (same grouping)
        r["duration"] = 100  # entries expire while the clock advances
        seq.append(r); nows.append(now)
    d_in = torch.cat([_dev(torch, r) for r in seq])
    tab = G.Table(1 << 10, max_batch=1024)
    tab.set_sweep(1)
    d_out = torch.empty((1024 * len(seq), 32), dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    for b in range(len(seq)):
        tab.submit_device(d_in[1024 * b:].data_ptr(), 1024, G.clock_fill(nows[b]), d_out[1024 * b:].data_ptr(), stream)
    torch.cuda.synchronize()
    out = d_out.cpu().numpy().reshape(-1).view(G.RESP_DTYPE)
    for b, r in enumerate(seq):
        pool.set_now(nows[b])
        _cmp(out[1024 * b:1024 * (b + 1)], pool.submit_hashed(r), f"batch {b}")
    c = tab.counters()
    assert c["unexpired_evictions"] > 0 and c["mixed_groups"] > 0


def test_submit_device_n_back_to_back(G, torch):
    """gub_submit_device_n: the batch size lives on the device and a torch kernel writes it (and the records) before every submission."""
    rng = np.random.default_rng(105)
    tab, pool = G.Table(1 << 21), O.Pool(cache_size=10_000_000, now_ms=T0)
    L = G.native.lib()
    sizes = [65536, 50000, 1, 256, 40961, 65535, 3000, 65536] * 3
    batches = _zipf_steps(rng, len(sizes), 65536, 300_000)
    src = [_dev(torch, r).view(torch.int64) for r in batches]
    cur = torch.empty((65536, 64), dtype=torch.uint8, device="cuda")
    counts = torch.tensor(sizes, dtype=torch.int32, device="cuda")
    d_n = torch.zeros(1, dtype=torch.int32, device="cuda")
    d_out = [torch.empty((65536, 32), dtype=torch.uint8, device="cuda") for _ in sizes]
    stream = torch.cuda.current_stream().cuda_stream
    zero = torch.zeros((), dtype=torch.int64, device="cuda")
    clks = [G.clock_fill(T0 + 10 * b) for b in range(len(sizes))]
    for b in range(len(sizes)):
        torch.add(src[b], zero, out=cur.view(torch.int64))
        d_n.copy_(counts[b:b + 1])
        rc = L.gub_submit_device_n(tab._h, C.c_void_p(cur.data_ptr()), 65536, C.c_void_p(d_n.data_ptr()), clks[b].ctypes.data,
                                   C.c_void_p(d_out[b].data_ptr()), C.c_void_p(stream))
        assert rc == 0, L.gub_last_error()
    torch.cuda.synchronize()
    for b, n in enumerate(sizes):
        pool.set_now(T0 + 10 * b)
        _cmp(_host(G, d_out[b], n), pool.submit_hashed(batches[b][:n]), f"batch {b} ({n} requests)")
    _check_table(G, tab, pool)
