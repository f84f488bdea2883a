"""GLOBAL sync ticks that carry more hit records than the ring's mailbox capacity (`cap`): the tick sends them in key-consistent rounds,
one mailbox epoch each.  W shards in one process (tests/local_ring.LocalRing, cap = 4096, global_capacity = 16384), checked bit for
bit against the oracle-side cluster model in tests/global_model.py, which applies a window's hits in one go."""
import os
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import oracle_py as O
from global_model import OracleCluster
from workloads import T0, key_hashes

pytestmark = pytest.mark.gpu

CAP, GCAP = 4096, 16384
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True, params=["pipeline", "fused"])
def owner_kernel_path(request, monkeypatch):
    """Owners evaluate their mailboxes with the four-kernel pipeline in ring mode (default) or with the persistent kernel k_batch
    (GUB_PATH=fused); read when a table is created."""
    monkeypatch.setenv("GUB_PATH", request.param)
    return request.param


def _ring(world, spread=False):
    from local_ring import LocalRing
    import torch
    if spread and torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    return LocalRing(world, capacity=1 << 17, cap=CAP, global_capacity=GCAP, spread_devices=spread)


def _batch(ids, src, window, now, glob_frac=5, reset=False, hits=None):
    """Requests for key ids: limits differ between sources, the algorithm is fixed per key (token and leaky buckets)."""
    n = len(ids)
    b = np.zeros(n, dtype=O.HREQ_DTYPE)
    xx, fv = key_hashes(ids, name="rounds")
    b["key_xxh64"], b["key_fnv1"] = xx, fv
    b["limit"] = 20 + ((ids + 3 * src + window) % 7) * 10
    b["duration"] = 30000 + (ids % 3) * 30000
    b["algorithm"] = (ids >> 1) & 1
    b["hits"] = np.where(ids % 11 == 0, 0, 1 + (ids % 3)) if hits is None else hits
    b["created_at"] = now
    glob = (ids % glob_frac) != 0
    b["behavior"] = np.where(glob, O.GLOBAL, 0).astype(np.uint32) | np.uint32(O.REQ_IS_OWNER)
    if reset:
        b["behavior"] |= np.where(glob & (ids % 13 == 0), O.RESET_REMAINING, 0).astype(np.uint32)
    return b


def _step(lr, model, batches, now, what):
    got, want = lr.step(batches, now), model.step(batches, now)
    for r in range(len(batches)):
        if not np.array_equal(got[r], want[r]):
            bad = np.nonzero(got[r] != want[r])[0]
            raise AssertionError(f"{what} shard {r}: {len(bad)} differ; first {bad[0]}: {got[r][bad[0]]} vs {want[r][bad[0]]}")
    return got


def _same_tables(lr, model):
    """Replicas and owners hold identical state on every shard (as test_gpu_global.test_global_random_traffic_matches_model)."""
    for r in range(lr.W):
        items = model.pools[r].each()
        dev = {(int(s["key_xxh64"]), int(s["key_fnv1"]) >> 8): s for s in lr.tabs[r].scan()}
        assert len(dev) == len(items)
        for (kx, kf), it in items.items():
            s = dev[(kx, kf >> 8)]
            assert int(s["limit"]) == it.limit and int(s["expire_at"]) == it.expire_at and int(s["stamp"]) == it.stamp, (r, s)
            if it.value_kind == 2:
                assert np.float64(s["remaining_f"]).view(np.uint64) == np.float64(it.remaining_f).view(np.uint64)
            else:
                assert int(s["remaining"]) == it.remaining_i and int(s["status"]) == it.status


def _dropped(lr):
    return sum(t.counters()["gq_dropped"] for t in lr.tabs)


def _window_traffic(rng, world, window, now, pool, steps=5):
    """`steps` steps of CAP requests per shard over a shared pool of key ids: about 3 x CAP distinct GLOBAL keys per shard."""
    out = []
    for step in range(steps):
        out.append([_batch(rng.choice(pool, CAP, replace=False), r, window, now + step, reset=(window == 1 and step == 2)) for r in range(world)])
    return out


@pytest.mark.parametrize("world,spread", [(1, False), (2, False), (4, False), (2, True)])
def test_rounds_random_traffic_match_model(world, spread):
    lr = _ring(world, spread)
    model = OracleCluster(world, T0)
    rng = np.random.default_rng(70 + world)
    pool = np.arange(1, 20000)
    now = T0
    for window in range(2):
        for i, batches in enumerate(_window_traffic(rng, world, window, now, pool)):
            _step(lr, model, batches, now + i, f"window {window} step {i}")
        now += 3
        lr.tick(now); model.tick(now)
        st = lr.last_tick
        if world > 1:
            assert max(s["hits_sent"] for s in st) > CAP, st  # several rounds ran
        else:
            assert st[0]["updates_made"] > CAP, st
        now += 400
    # replicas answer like the owners after the last tick
    probe = [_batch(rng.choice(pool, CAP, replace=False), r, 2, now, hits=0) for r in range(world)]
    _step(lr, model, probe, now, "probe")
    _same_tables(lr, model)
    assert _dropped(lr) == 0


def _owned_by(model, ids, shard, invert=False):
    b = _batch(ids, 0, 0, T0)
    own = model.owners(b)
    return ids[(own != shard) if invert else (own == shard)]


def test_skewed_shards():
    """Shard 0's window needs at least 4 rounds while shard 1 has no GLOBAL hits at all: every shard still runs every round."""
    world = 4
    lr, model = _ring(world), OracleCluster(world, T0)
    rng = np.random.default_rng(5)
    heavy = rng.permutation(_owned_by(model, np.arange(1, 40000), 0, invert=True))[:int(3.5 * CAP)]
    now = T0
    for i in range(4):
        ids = heavy[i * len(heavy) // 4:(i + 1) * len(heavy) // 4]
        batches = [_batch(ids, 0, 0, now, glob_frac=1 << 30)] + [_batch(np.arange(100000 + 50 * r, 100050 + 50 * r), r, 0, now, glob_frac=1)
                                                              for r in range(1, world)]
        _step(lr, model, batches, now, f"step {i}")
    lr.tick(now); model.tick(now)
    st = lr.last_tick
    sent = int(np.sum(heavy % 11 != 0))  # (Hits = 0 requests are never queued)
    assert st[0]["hits_sent"] == sent and sent > 3 * CAP
    assert all(s["hits_sent"] == 0 for s in st[1:])
    for p in lr.p2ps:
        assert p.status() == 0
    for i in range(3):  # the steps after a multi-round tick stay aligned, and every shard sees the owners' state
        batches = [_batch(rng.choice(heavy, 1000, replace=False), r, 0, now + 1 + i, glob_frac=1 << 30) for r in range(world)]
        _step(lr, model, batches, now + 1 + i, f"after tick {i}")
    lr.tick(now + 10); model.tick(now + 10)
    _same_tables(lr, model)
    assert _dropped(lr) == 0


def test_queue_overflow_still_counted():
    """More distinct keys than the queue holds: the overflow is counted in gq_dropped, and every key that was queued converges."""
    world = 2
    lr, model = _ring(world), OracleCluster(world, T0)
    ids = _owned_by(model, np.arange(1, 60000), 1)[:GCAP + CAP]
    assert len(ids) == GCAP + CAP
    now = T0
    empty = np.zeros(0, dtype=O.HREQ_DTYPE)

    def token(k, hits):
        b = _batch(k, 0, 0, now, glob_frac=1 << 30, hits=hits)
        b["algorithm"] = 0
        return b
    for i in range(0, len(ids), CAP):
        lr.step([token(ids[i:i + CAP], 1), empty], now)
    lr.tick(now)
    assert _dropped(lr) == len(ids) - GCAP
    assert lr.last_tick[0]["hits_sent"] == GCAP
    agree = 0
    for i in range(0, len(ids), CAP):
        q = token(ids[i:i + CAP], 0)
        a, b = lr.step([q, empty], now)[0], lr.step([empty, q], now)[1]
        agree += int(np.sum((a["status"] == b["status"]) & (a["remaining"] == b["remaining"]) & (a["limit"] == b["limit"])
                            & (a["reset_time"] == b["reset_time"])))
    assert agree == GCAP  # the queued keys: replica == owner; the dropped ones were never sent


def test_threaded_driver_matches_single_thread_driver():
    """gub_global_tick from one thread per shard gives what gub_global_tick_local_all gives."""
    world = 4
    one, many = _ring(world), _ring(world)
    rng = np.random.default_rng(11)
    pool = np.arange(1, 20000)
    now = T0
    pool_ex = ThreadPoolExecutor(world)
    for window in range(2):
        for i, batches in enumerate(_window_traffic(rng, world, window, now, pool, steps=3)):
            a, b = one.step(batches, now + i), many.step(batches, now + i)
            assert all(np.array_equal(x, y) for x, y in zip(a, b)), f"window {window} step {i}"
        now += 3
        one.tick(now)
        clk = many.g.clock_fill(now)
        stats = [f.result() for f in [pool_ex.submit(many.p2ps[r].tick, clk, now, many.streams[r].cuda_stream) for r in range(world)]]
        many.sync()
        assert stats == one.last_tick
        assert max(s["hits_sent"] for s in stats) > CAP
    for r in range(world):
        sa = np.sort(one.tabs[r].scan(), order=["key_xxh64"])
        sb = np.sort(many.tabs[r].scan(), order=["key_xxh64"])
        assert np.array_equal(sa, sb)
    pool_ex.shutdown()


def test_nccl_two_processes():
    """One process per GPU: the histograms and the items travel by NCCL all-gather (tests/global_rounds_worker.py)."""
    import subprocess
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    env = dict(os.environ, GUB_ROOT=ROOT, OMP_NUM_THREADS="1")
    port = 29900 + (os.getpid() % 90)
    res = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                          "--master-port", str(port), os.path.join(ROOT, "tests", "global_rounds_worker.py")], env=env, capture_output=True,
                         text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "rank 0 ok" in res.stdout and "rank 1 ok" in res.stdout
