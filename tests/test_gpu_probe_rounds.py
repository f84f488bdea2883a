"""The table probe in rounds on the GPU: long clusters of keys sharing one home slot (wrapping at the table's end, with tombstones
left by a sweep) through gub_submit_device on both evaluation paths, bit for bit against the oracle, then a full scan of the table
and a lookup of every key through the items kernels."""
import numpy as np
import pytest

import oracle_py as O
from workloads import T0

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, params=["pipeline", "fused"])
def eval_path(request, monkeypatch):
    """Both evaluation paths of a single table: the four-kernel pipeline and the persistent kernel k_batch (GUB_PATH=fused)."""
    monkeypatch.setenv("GUB_PATH", request.param)
    return request.param


@pytest.fixture(scope="module")
def G():
    import gubernator_b200 as g
    return g


def _cmp(got, want, what=""):
    if not np.array_equal(got, want):
        bad = np.nonzero(got != want)[0]
        i = int(bad[0])
        raise AssertionError(f"{what}: {len(bad)} of {len(got)} responses differ; first at {i}: got {got[i]} want {want[i]}")


def _check_table_equals_oracle(tab, pool):
    items = pool.each()
    scan = tab.scan()
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


def _keys_with_home(rng, h, cap, n):
    """n distinct keys whose home slot (key * cap) >> 64 is h."""
    lo = max(2, -(-(h << 64) // cap))
    hi = -(-((h + 1) << 64) // cap) - 1
    assert hi - lo < (1 << 62)
    out = set()
    while len(out) < n:
        out.add(lo + int(rng.integers(0, hi - lo + 1)))
    keys = np.array(sorted(out), dtype=np.uint64)
    rng.shuffle(keys)
    return keys


def _submit_device(G, tab, reqs, now):
    import torch
    dev = torch.device("cuda:0")
    n = len(reqs)
    d_reqs = torch.from_numpy(np.ascontiguousarray(reqs).view(np.uint8).reshape(n, 64)).to(dev)
    d_out = torch.zeros((n, 32), dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    tab.submit_device(d_reqs.data_ptr(), n, G.clock_fill(now), d_out.data_ptr(), st)
    torch.cuda.synchronize()
    return d_out.cpu().numpy().reshape(-1).view(G.RESP_DTYPE)


@pytest.mark.parametrize("length", [14, 66, 162])
def test_long_clusters_bit_exact(G, length):
    """`length` keys sharing a home 3 slots before the table's end (the cluster wraps), every other one short-lived; after a sweep the
    survivors sit behind tombstones, then survivors, re-created and new keys arrive in random order, then every key once more."""
    cap = 1 << 12
    rng = np.random.default_rng(length)
    keys = _keys_with_home(rng, cap - 3, cap, length + 40)
    tab, pool = G.Table(cap), O.Pool(now_ms=T0)

    def batch(ks, now, duration):
        r = np.zeros(len(ks), dtype=G.REQ_DTYPE)
        r["key_xxh64"] = ks; r["key_fnv1"] = (ks * np.uint64(0x9E3779B97F4A7C15)) | np.uint64(0x100)
        r["hits"] = 1; r["limit"] = 10; r["duration"] = duration; r["created_at"] = now
        r["algorithm"] = (ks & np.uint64(1)).astype(np.uint32); r["behavior"] = G.native.REQ_IS_OWNER
        return r
    first = batch(keys[:length], T0, np.where(np.arange(length) % 2 == 0, 1000, 100000))
    _cmp(_submit_device(G, tab, first, T0), pool.submit_hashed(first), "fill")
    now = T0 + 5000
    pool.set_now(now)
    assert tab.sweep(now) == (length + 1) // 2
    again = batch(keys, now, 100000)
    rng.shuffle(again)
    _cmp(_submit_device(G, tab, again, now), pool.submit_hashed(again), "after the sweep")
    now += 1
    pool.set_now(now)
    last = batch(keys[::-1].copy(), now, 100000)
    _cmp(_submit_device(G, tab, last, now), pool.submit_hashed(last), "all resident")
    c, oc = tab.counters(), pool.counters()
    for k in ("over_limit", "cache_hit", "cache_miss"):
        assert c[k] == oc[k], (k, c, oc)
    _check_table_equals_oracle(tab, pool)
    fv = (keys * np.uint64(0x9E3779B97F4A7C15)) | np.uint64(0x100)
    got, found = tab.get_items(keys, fv, now)
    assert found.all() and np.all(got["limit"] == 10)
    assert not tab.get_items(keys + np.uint64(1), fv ^ np.uint64(1 << 20), now)[1].any()
