"""gub_p2p_step_keys_store_local_all on the H100: every owner of a ring applies the Store rule to its pass (what it evaluates in a step, in
source-rank then source-index order).  Checked on three sides, step by step: the ring; one twin table per owner fed that owner's pass
through gub_submit_keys_store_async; the oracle model of the rule (tests/_store_emu.py model_batch) per owner.  Responses, the Store call
sequence (Get / Remove / OnChange with key strings and items), the final tables and the counters agree."""
import numpy as np
import pytest

import oracle_py as O
import _store_emu as S
from local_ring import LocalRing
from workloads import T0, adversarial_batch, bench_key_bytes, bench_key_hashes, zipf_ids

pytestmark = pytest.mark.gpu

N_KEYS = 3000
PARAM_FIELDS = ("limit", "duration", "burst", "algorithm", "behavior")
ITEM_FIELDS = ("algorithm", "status", "limit", "duration", "remaining", "remaining_f", "stamp", "burst", "expire_at")
KEYS = [bytes(k) for k in bench_key_bytes(np.arange(N_KEYS))]
KXX, KFV = bench_key_hashes(np.arange(N_KEYS))


_OPEN = []  # (p2ps, tables) made by a test: closed after it, rings before tables, whatever the test's outcome


def opened(p2ps, tabs):
    _OPEN.append((list(p2ps), list(tabs)))
    return p2ps


@pytest.fixture(autouse=True)
def _close_rings():
    yield
    while _OPEN:
        p2ps, tabs = _OPEN.pop()
        for p in p2ps:
            p.close()
        for t in tabs:
            t.close()


@pytest.fixture(scope="module")
def G():
    import os
    import gubernator_b200 as g
    if os.environ.get("GUB_PATH") == "fused":
        pytest.skip("the Store path runs on the four-kernel pipeline only")
    return g


def _oring(world):
    from gubernator_b200.sharded import shard_addresses
    oring = O.Ring(0, 512)
    for a in shard_addresses(world):
        oring.add(a)
    return oring


def make_step(G, rng, world, step, now, cap):
    """Per shard: key ids and hashed records (Zipf on even steps, adversarial traffic on odd ones), the step's parameter table and
    every shard's packed key batch."""
    ids, recs = [], []
    for r in range(world):
        n = int(min(cap, rng.choice([1, 700, 3000, cap])))
        if step % 2:
            rec = adversarial_batch(rng, n, 41, now)
            _, kid = np.unique(rec["key_xxh64"], return_inverse=True)
            i = (kid.reshape(-1) * 37) % N_KEYS
        else:
            i = zipf_ids(rng, n, N_KEYS, 1.1)
            rec = np.zeros(n, dtype=O.HREQ_DTYPE)
            rec["hits"] = 1; rec["limit"] = 100; rec["duration"] = 60000; rec["created_at"] = now
            rec["algorithm"] = i & 1; rec["behavior"] = O.REQ_IS_OWNER
        rec = rec.copy()
        rec["key_xxh64"], rec["key_fnv1"] = KXX[i], KFV[i]
        ids.append(np.asarray(i, dtype=np.int64)); recs.append(rec)
    allrec = np.concatenate(recs)
    cfg = np.zeros(len(allrec), dtype=G.native.PARAMS_DTYPE)
    for f in PARAM_FIELDS:
        cfg[f] = allrec[f]
    table, inv = np.unique(cfg, return_inverse=True)
    inv = inv.reshape(-1)
    base = int(allrec["created_at"].min())
    packed, pidx, at = [], [], 0
    for r in range(world):
        n = len(recs[r])
        pidx.append(inv[at:at + n])
        packed.append(G.native.pack_keys([KEYS[int(k)] for k in ids[r]], recs[r]["hits"], inv[at:at + n], (recs[r]["created_at"] - base).astype(np.int32)))
        at += n
    return dict(ids=ids, recs=recs, table=table, base=base, packed=packed, pidx=pidx)


class Ring:
    """The ring under test: LocalRing's shards stepped through gub_p2p_step_keys_store_local_all."""

    def __init__(self, G, world, cap=8192, spread=False, capacity=1 << 16):
        self.G, self.lr, self.W, self.cap = G, LocalRing(world, capacity=capacity, cap=cap, spread_devices=spread), world, cap
        opened(self.lr.p2ps, self.lr.tabs)
        self.ch = [G.native.PinnedArray(world * cap, G.native.STORE_REC_DTYPE) for _ in range(world)]
        self.nc = [G.native.PinnedArray(1, np.uint32) for _ in range(world)]

    def step(self, st, now, get):
        torch, lr = self.lr.torch, self.lr
        bufs = [torch.from_numpy(p).to(torch.device("cuda", lr.devs[r])) for r, p in enumerate(st["packed"])]
        outs = [torch.zeros((self.cap, 32), dtype=torch.uint8, device=torch.device("cuda", lr.devs[r])) for r in range(self.W)]
        for d in set(lr.devs):
            torch.cuda.synchronize(d)
        ns = [len(x) for x in st["recs"]]
        for a in self.nc:
            a.array[0] = 0xFFFFFFFF
        self.G.native.p2p_step_keys_store_local_all(lr.p2ps, [b.data_ptr() for b in bufs], [len(p) for p in st["packed"]], ns, st["table"], st["base"],
                                                    self.G.clock_fill(now), get, [o.data_ptr() for o in outs], [c.ptr for c in self.ch],
                                                    [c.ptr for c in self.nc], [s.cuda_stream for s in lr.streams])
        lr.sync()
        resp = [outs[r][:ns[r]].cpu().numpy().reshape(-1).view(O.HRESP_DTYPE) for r in range(self.W)]
        return resp, [self.ch[r].array[:int(self.nc[r].array[0])].copy() for r in range(self.W)]


def passes(oring, st, world):
    """Owner r's pass: (source shard, source index) of every request it evaluates, in source-rank then source-index order."""
    owners = [np.array([oring.get_by_hash(int(h)) for h in rec["key_fnv1"]], dtype=np.int64) for rec in st["recs"]]
    out = []
    for r in range(world):
        shard = np.concatenate([np.full(int((owners[s] == r).sum()), s, dtype=np.int64) for s in range(world)])
        idx = np.concatenate([np.nonzero(owners[s] == r)[0] for s in range(world)])
        out.append((shard, idx))
    return out


def named(recs, shard, idx):
    """Records of a single table fed a pass, with their pass indices turned into (source shard, source index) as the ring names them."""
    import gubernator_b200 as g
    r = recs.copy().view(g.native.STORE_REC_DTYPE)
    r["first_shard"], r["last_shard"] = shard[recs["first"]], shard[recs["last"]]
    r["first"], r["last"] = idx[recs["first"]], idx[recs["last"]]
    return r


def key_of(st, shard, i):
    return KEYS[int(st["ids"][int(shard)][int(i)])].decode("latin-1")


def calls_of(st, recs):
    """The Store calls the records ask for, with key strings and items, in order."""
    out = []
    for rec in recs:
        key = key_of(st, rec["first_shard"], rec["first"])
        if rec["flags"] & S.STORE_REMOVE:
            out.append(("Remove", key))
        if rec["flags"] & S.STORE_CHANGE:
            out.append(("OnChange", key, tuple(rec["item"][f].item() for f in ITEM_FIELDS)))
    return out


def _scan(tab):
    s = tab.scan()
    return s[np.lexsort((s["key_fnv1"], s["key_xxh64"]))]


def _counters(tab):
    c = dict(tab.counters())
    c.pop("batches")  # (a ring owner runs one batch per step even when its pass is empty; its twin gets none then)
    return c


def run_three_sides(G, world, steps, seed, spread=False, get=True, cap=8192):
    rng = np.random.default_rng(seed)
    ring = Ring(G, world, cap=cap, spread=spread)
    oring = _oring(world)
    twins = [G.Table(1 << 16) for _ in range(world)]
    opened([], twins)
    pools = [O.Pool(workers=2, cache_size=10**7, now_ms=T0) for _ in range(world)]
    now = T0
    for step in range(steps):
        now += int(rng.choice([0, 1, 900, 70000]))
        st = make_step(G, rng, world, step, now, cap)
        items = S.fill_store(rng, np.concatenate(st["recs"]), now) if get else {}
        ring_calls = []
        got, recs = ring.step(st, now, S.found_filler(items, ring_calls) if get else None)
        ring_gets = [key_of(st, m["first_shard"], m["first"]) for call in ring_calls for m in call]
        twin_gets, twin_resp, model_resp = [], [np.zeros(len(x), dtype=O.HRESP_DTYPE) for x in st["recs"]], [np.zeros(len(x), dtype=O.HRESP_DTYPE) for x in st["recs"]]
        for r, (shard, idx) in enumerate(passes(oring, st, world)):
            n = len(idx)
            if n == 0:
                assert len(recs[r]) == 0
                continue
            pr = np.concatenate([st["recs"][s][idx[shard == s]] for s in range(world)])
            pi = np.concatenate([st["pidx"][s][idx[shard == s]] for s in range(world)])
            packed = G.native.pack_keys([KEYS[int(st["ids"][s][i])] for s, i in zip(shard, idx)], pr["hits"], pi, (pr["created_at"] - st["base"]).astype(np.int32))
            out = G.native.PinnedArray(n, G.RESP_DTYPE)
            ch, nc = G.native.PinnedArray(n, G.native.STORE_REC_DTYPE), G.native.PinnedArray(1, np.uint32)
            tcalls = []
            twins[r].wait(twins[r].submit_keys_store_async(packed.ctypes.data, len(packed), n, st["table"].ctypes.data, len(st["table"]), st["base"],
                                                           G.clock_fill(now), S.found_filler(items, tcalls) if get else None, out.ptr, ch.ptr, nc.ptr))
            trecs = named(ch.array[:int(nc.array[0])].copy(), shard, idx)
            twin_gets += [key_of(st, shard[m["first"]], idx[m["first"]]) for call in tcalls for m in call]
            _, mresp, mrecs = S.model_batch(pools[r], pr, now, items)
            assert recs[r].tobytes() == trecs.tobytes(), f"step {step} owner {r}: change log differs from the twin table's"
            assert recs[r].tobytes() == named(mrecs, shard, idx).tobytes(), f"step {step} owner {r}: change log differs from the model"
            assert calls_of(st, recs[r]) == calls_of(st, trecs)
            for s in range(world):
                twin_resp[s][idx[shard == s]] = out.array[:n][shard == s]
                model_resp[s][idx[shard == s]] = mresp[shard == s]
        assert ring_gets == twin_gets, f"step {step}: Store.Get calls differ"
        for s in range(world):
            assert np.array_equal(got[s], twin_resp[s]), f"step {step} shard {s}: responses differ from the twin tables"
            assert np.array_equal(got[s], model_resp[s]), f"step {step} shard {s}: responses differ from the model"
    for r in range(world):
        assert _scan(ring.lr.tabs[r]).tobytes() == _scan(twins[r]).tobytes(), f"owner {r}: final table differs from its twin"
        assert _counters(ring.lr.tabs[r]) == _counters(twins[r]), f"owner {r}: counters differ from its twin"
    return ring


@pytest.mark.parametrize("spread", [False, True])
@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_ring_store_matches_twin_tables_and_model(G, world, spread):
    import torch
    if spread and (torch.cuda.device_count() < 2 or world == 1):
        pytest.skip("needs >= 2 GPUs")
    run_three_sides(G, world, steps=6, seed=100 + world, spread=spread)


def test_write_behind_store(G):
    """get = NULL: the step is gub_p2p_step_keys_local_all's, and the change logs are those of a store that finds nothing."""
    run_three_sides(G, 4, steps=4, seed=7, get=False)


def test_failing_get_keeps_the_ring_in_step(G):
    """A failing Get fails the call and changes no table; the ring stays in step, and the next step matches a twin ring that never saw
    the failed one."""
    world, cap = 4, 8192
    rng = np.random.default_rng(31)
    a, b = Ring(G, world, cap), Ring(G, world, cap)
    st0, st1, st2 = (make_step(G, rng, world, s, T0 + s, cap) for s in range(3))
    for ring in (a, b):
        ring.step(st0, T0, S.found_filler({}))
    before = [(_scan(t).tobytes(), t.counters()) for t in a.lr.tabs]
    calls = []

    def failing(misses):
        calls.append(len(misses))
        return 5
    with pytest.raises(G.native.GubError, match="get callback failed"):
        a.step(st1, T0 + 1, failing)
    a.lr.sync()
    assert len(calls) == 1
    assert [(_scan(t).tobytes(), t.counters()) for t in a.lr.tabs] == before
    items = S.fill_store(rng, np.concatenate(st2["recs"]), T0 + 2)
    got_a, recs_a = a.step(st2, T0 + 2, S.found_filler(items))
    got_b, recs_b = b.step(st2, T0 + 2, S.found_filler(items))
    for r in range(world):
        assert got_a[r].tobytes() == got_b[r].tobytes() and recs_a[r].tobytes() == recs_b[r].tobytes()
        assert _scan(a.lr.tabs[r]).tobytes() == _scan(b.lr.tabs[r]).tobytes()


def test_get_that_overwrites_the_request_names(G):
    """A get that writes the whole miss record, request names included, changes nothing: the library keeps its own copy."""
    world, cap = 4, 8192
    rng = np.random.default_rng(12)
    a, b = Ring(G, world, cap), Ring(G, world, cap)
    for step in range(3):
        st = make_step(G, rng, world, step, T0 + step, cap)
        items = S.fill_store(rng, np.concatenate(st["recs"]), T0 + step)
        clean = S.found_filler(items)

        def scribbler(misses):
            clean(misses)
            misses["first"], misses["last"], misses["first_shard"], misses["last_shard"] = 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFF, 0xFFFF
            return 0
        got_a, recs_a = a.step(st, T0 + step, clean)
        got_b, recs_b = b.step(st, T0 + step, scribbler)
        for r in range(world):
            assert got_a[r].tobytes() == got_b[r].tobytes() and recs_a[r].tobytes() == recs_b[r].tobytes()
    for r in range(world):
        assert _scan(a.lr.tabs[r]).tobytes() == _scan(b.lr.tabs[r]).tobytes()


def test_refusals(G, monkeypatch):
    rng = np.random.default_rng(3)
    ring = Ring(G, 2, 8192)
    st = make_step(G, rng, 2, 0, T0, 8192)
    lr = ring.lr
    bufs = [lr.torch.from_numpy(p).cuda() for p in st["packed"]]
    outs = [lr.torch.zeros((8192, 32), dtype=lr.torch.uint8, device="cuda") for _ in range(2)]
    ns = [len(x) for x in st["recs"]]

    def call(p2ps, ch_ptrs, nc_ptrs):
        G.native.p2p_step_keys_store_local_all(p2ps, [b.data_ptr() for b in bufs], [len(p) for p in st["packed"]], ns, st["table"], st["base"],
                                               G.clock_fill(T0), None, [o.data_ptr() for o in outs], ch_ptrs, nc_ptrs, [s.cuda_stream for s in lr.streams])
    pinned = ([c.ptr for c in ring.ch], [c.ptr for c in ring.nc])
    plain_ch, plain_nc = [np.zeros(2 * 8192, dtype=G.native.STORE_REC_DTYPE) for _ in range(2)], [np.zeros(1, dtype=np.uint32) for _ in range(2)]
    with pytest.raises(G.native.GubError, match="page-locked"):
        call(lr.p2ps, [c.ctypes.data for c in plain_ch], [c.ctypes.data for c in plain_nc])
    from gubernator_b200.sharded import shard_addresses

    tabs5 = [G.Table(1 << 14, max_batch=65536) for _ in range(5)]
    ring5 = G.Ring(0, 512)
    for a_ in shard_addresses(5):
        ring5.add(a_)
    p5 = [G.native.P2P(tabs5[r], ring5, r, 65536) for r in range(5)]  # 5 x 65 536 > the 262 144-request pass gub_p2p_create allows
    opened(p5, tabs5)
    for p in p5:
        p.connect_local(p5)
    ch5 = [G.native.PinnedArray(1, G.native.STORE_REC_DTYPE) for _ in range(5)]
    nc5 = [G.native.PinnedArray(1, np.uint32) for _ in range(5)]
    empty = np.zeros(16, dtype=np.uint8)
    eb = lr.torch.from_numpy(empty).cuda()
    with pytest.raises(G.native.GubError, match="exceeds an owner's pass"):
        G.native.p2p_step_keys_store_local_all(p5, [eb.data_ptr()] * 5, [16] * 5, [0] * 5, st["table"], st["base"], G.clock_fill(T0), None,
                                               [outs[0].data_ptr()] * 5, [c.ptr for c in ch5], [c.ptr for c in nc5], [0] * 5)
    unconnected = [G.native.P2P(G.Table(1 << 14), lr.ring, r, 8192) for r in range(2)]
    opened(unconnected, [p.table for p in unconnected])
    with pytest.raises(G.native.GubError, match="gub_p2p_connect_local"):
        call(unconnected, *pinned)
    glob = LocalRing(2, cap=8192, global_capacity=4096)
    opened(glob.p2ps, glob.tabs)
    with pytest.raises(G.native.GubError, match="GLOBAL"):
        call(glob.p2ps, *pinned)
    monkeypatch.setenv("GUB_PATH", "fused")
    fused = LocalRing(2, cap=8192)
    opened(fused.p2ps, fused.tabs)
    with pytest.raises(G.native.GubError, match="GUB_PATH=fused"):
        call(fused.p2ps, *pinned)
    monkeypatch.delenv("GUB_PATH")
    call(lr.p2ps, *pinned)  # and the ring still steps
    lr.sync()

