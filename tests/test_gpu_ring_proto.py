"""GetRateLimits wire bytes on the ring of this process (gub_p2p_step_proto_local_all) on the H100, checked byte for byte against a twin
ring fed the same items as records through gub_p2p_step_local_all (chunked by the call's rule: cap items per shard per step) and encoded
by the restatement (tests/_proto_wire.py), and, for a contiguous split on a non-GLOBAL ring, against gub_submit_proto_async on one table.
Outputs are page-locked with guard bytes on both sides.  The code-7 text of an owner that never answered is covered on the CPU
(tests/test_ring_proto_emulated.py): no test here waits out a silent peer."""
import numpy as np
import pytest

import oracle_py as O
import _proto_wire as W
from local_ring import LocalRing
from ring_proto_traffic import encode, spread_items
from workloads import T0

pytestmark = pytest.mark.gpu

GUARD = 256
N_KEYS = 1 << 20
GLOBAL = 2


@pytest.fixture(autouse=True, params=["pipeline", "fused"])
def owner_kernel_path(request, monkeypatch):
    """Owners evaluate with the four-kernel pipeline in ring mode (default) or the persistent kernel k_batch (GUB_PATH=fused)."""
    monkeypatch.setenv("GUB_PATH", request.param)
    return request.param


@pytest.fixture(scope="module")
def G():
    import gubernator_b200 as g
    return g


class Call:
    """One call's page-locked buffers for every shard, with GUARD bytes of 0xA5 before and after each output."""

    def __init__(self, G, shards):
        self.G, self.shards = G, shards
        self.n = [len(m) for m, _ in shards]
        self.pk, self.out, self.off, self.st, self.bound = [], [], [], [], []
        for (msgs, created), n in zip(shards, self.n):
            packed, bound = G.native.pack_proto(msgs, created)
            pk = G.native.PinnedArray(len(packed), np.uint8)
            pk.array[:] = packed
            out = G.native.PinnedArray(bound + 2 * GUARD, np.uint8)
            off = G.native.PinnedArray(n + 1 + 2 * GUARD // 8, np.uint64)
            st = G.native.PinnedArray(n + 2 * GUARD // 4, np.uint32)
            for a in (out, off, st):
                a.array.view(np.uint8)[:] = 0xA5
            self.pk.append(pk); self.out.append(out); self.off.append(off); self.st.append(st); self.bound.append(bound)

    def enqueue(self, lr, now, force_global=False):
        G = self.G
        G.native.p2p_step_proto_local_all(lr.p2ps, [p.ptr for p in self.pk], [len(p.array) for p in self.pk], self.n, G.clock_fill(now),
                                          [o.ptr + GUARD for o in self.out], self.bound, [o.ptr + GUARD for o in self.off],
                                          [s.ptr + GUARD for s in self.st], [s.cuda_stream for s in lr.streams], force_global=force_global)

    def result(self):
        res = []
        for r, n in enumerate(self.n):
            for a in (self.out[r], self.off[r], self.st[r]):
                b = a.array.view(np.uint8)
                assert (b[:GUARD] == 0xA5).all() and (b[len(b) - GUARD:] == 0xA5).all(), f"shard {r}: a guard byte was overwritten"
            off = self.off[r].array[GUARD // 8:GUARD // 8 + n + 1]
            out = self.out[r].array[GUARD:GUARD + self.bound[r]]
            res.append((self.st[r].array[GUARD // 4:GUARD // 4 + n].tolist(), [out[int(off[m]):int(off[m + 1])].tobytes() for m in range(n)]))
        return res

    def free(self):
        for lst in (self.pk, self.out, self.off, self.st):
            for a in lst:
                a.free()


def run(G, lr, shards, now, force_global=False):
    call = Call(G, shards)
    call.enqueue(lr, now, force_global)
    lr.sync()
    res = call.result()
    call.free()
    return res


def twin_run(twin, shards, now, force_global=False):
    """The twin ring's answer: the restatement's records of every shard, cap per shard per step, encoded per message."""
    plans, batches = [], []
    for msgs, created in shards:
        batch, plan = W.prepare(msgs, created)
        if force_global:
            batch["behavior"] |= np.uint32(GLOBAL)
        plans.append(plan); batches.append(batch)
    cap = twin.cap
    S = max((len(b) + cap - 1) // cap for b in batches)
    resp = [np.zeros(len(b), dtype=O.HRESP_DTYPE) for b in batches]
    for k in range(S):
        got = twin.step([b[k * cap:(k + 1) * cap] for b in batches], now)
        for r, g in enumerate(got):
            resp[r][k * cap:k * cap + len(g)] = g
    return [encode(p, r) for p, r in zip(plans, resp)], S


def _check(got, want, what):
    for r, ((st, outs), exp) in enumerate(zip(got, want)):
        assert st == [s for s, _ in exp], f"{what} shard {r}: statuses differ"
        for m, (b, (_, wb)) in enumerate(zip(outs, exp)):
            assert b == wb, f"{what} shard {r} message {m}: response bytes differ"


def _scan(tab):
    return np.sort(tab.scan(), order=["key_xxh64", "key_fnv1"])


def _same_rings(a, b):
    for r in range(a.W):
        assert _scan(a.tabs[r]).tobytes() == _scan(b.tabs[r]).tobytes(), f"shard {r}: table contents differ from the twin's"
        assert a.tabs[r].counters() == b.tabs[r].counters(), f"shard {r}: counters differ from the twin's"


def rpcs(rng, items, now, adversarial=False, n_keys=N_KEYS):
    """RPCs of 100-1000 items, `items` in all: bench-like (Zipf over n_keys) or adversarial (few hot keys, edge messages mixed in)."""
    msgs, left = [], items
    while left > 0:
        k = min(left, int(rng.integers(100, 1001)))
        msgs.append(W.message(spread_items(rng, k, n_keys=64 if adversarial else n_keys)))
        left -= k
    if adversarial:
        for _, m, _ in W.edge_messages(rng, now)[::3]:
            msgs.insert(int(rng.integers(0, len(msgs) + 1)), m)
    return msgs, np.array([now - int(rng.integers(0, 40)) for _ in msgs], dtype=np.int64)


@pytest.mark.parametrize("spread", [False, True])
@pytest.mark.parametrize("world", [1, 2, 4])
def test_calls_match_the_record_ring(G, world, spread):
    import torch
    if spread and (torch.cuda.device_count() < 2 or world == 1):
        pytest.skip("needs >= 2 GPUs")
    kw = dict(capacity=1 << 20, cap=65536, spread_devices=spread)
    lr, twin = LocalRing(world, **kw), LocalRing(world, **kw)
    rng = np.random.default_rng(100 + world)
    for c in range(3):
        now = T0 + 700 * c
        shards = [rpcs(rng, int(rng.integers(65536 // world // 2, 65536 // world)), now, adversarial=(c == 1)) for _ in range(world)]
        got = run(G, lr, shards, now)
        want, _ = twin_run(twin, shards, now)
        _check(got, want, f"call {c}")
    _same_rings(lr, twin)


@pytest.mark.parametrize("world", [1, 2, 4])
def test_contiguous_split_matches_one_table(G, world):
    """A non-GLOBAL ring fed a contiguous split with every n_r <= cap answers what gub_submit_proto_async answers on one table."""
    lr = LocalRing(world, capacity=1 << 21, cap=65536)
    tab = G.Table(1 << 22)
    rng = np.random.default_rng(7 + world)
    for c in range(3):
        now = T0 + 900 * c
        msgs, created = rpcs(rng, 60000, now, adversarial=(c == 2))
        cuts = np.linspace(0, len(msgs), world + 1).astype(int)
        got = run(G, lr, [(msgs[cuts[r]:cuts[r + 1]], created[cuts[r]:cuts[r + 1]]) for r in range(world)], now)
        one = Call(G, [(msgs, created)])
        tab.wait(tab.submit_proto_async(one.pk[0].ptr, len(one.pk[0].array), one.n[0], G.clock_fill(now), one.out[0].ptr + GUARD, one.bound[0],
                                        one.off[0].ptr + GUARD, one.st[0].ptr + GUARD))
        (st, outs), = one.result()
        one.free()
        assert sum((s for s, _ in got), []) == st
        assert sum((o for _, o in got), []) == outs, f"call {c}: response bytes differ from the single table's"
    ring_items = np.sort(np.concatenate([lr.tabs[r].scan() for r in range(world)]), order=["key_xxh64", "key_fnv1"])
    assert ring_items.tobytes() == _scan(tab).tobytes()
    for f in ("requests", "cache_hit", "cache_miss", "over_limit"):
        assert sum(lr.tabs[r].counters()[f] for r in range(world)) == tab.counters()[f], f


def test_several_steps_per_call(G):
    """cap = 8192: one shard's RPCs take S = 3 steps, another's one, a third has none."""
    lr, twin = LocalRing(3, capacity=1 << 18, cap=8192), LocalRing(3, capacity=1 << 18, cap=8192)
    rng = np.random.default_rng(31)
    for c in range(2):
        now = T0 + 50 * c
        shards = [rpcs(rng, 20000, now), rpcs(rng, 3000, now, adversarial=True), ([], np.zeros(0, dtype=np.int64))]
        got = run(G, lr, shards[c:] + shards[:c], now)
        want, S = twin_run(twin, shards[c:] + shards[:c], now)
        assert S >= 3
        _check(got, want, f"call {c}")
    _same_rings(lr, twin)


def test_force_global_with_ticks(G):
    """A GLOBAL ring with force_global: responses, tick results and tables equal those of the twin fed the records with GLOBAL set."""
    kw = dict(capacity=1 << 16, cap=8192, global_capacity=8192)
    lr, twin = LocalRing(3, **kw), LocalRing(3, **kw)
    rng = np.random.default_rng(503)
    now = T0
    for c in range(8):
        now += int(rng.choice([0, 1, 5, 400]))
        shards = [rpcs(rng, int(rng.integers(0, 5000)), now, n_keys=2000, adversarial=(c % 3 == 1)) for _ in range(3)]
        got = run(G, lr, shards, now, force_global=True)
        want, _ = twin_run(twin, shards, now, force_global=True)
        _check(got, want, f"call {c}")
        if c % 2 == 1:
            assert lr.tick(now) == twin.tick(now)
            assert lr.last_tick == twin.last_tick
    _same_rings(lr, twin)


def test_pipelined_calls_equal_calls_one_by_one(G):
    lr, one = LocalRing(2, capacity=1 << 18, cap=16384), LocalRing(2, capacity=1 << 18, cap=16384)
    rng = np.random.default_rng(12)
    calls = [(T0 + 300 * c, [rpcs(rng, int(rng.integers(2000, 20000)), T0 + 300 * c, adversarial=(c % 2 == 1)) for _ in range(2)]) for c in range(6)]
    want = [run(G, one, shards, now) for now, shards in calls]
    staged = [Call(G, shards) for _, shards in calls]
    for (now, _), call in zip(calls, staged):
        call.enqueue(lr, now)
    lr.sync()
    for c, call in enumerate(staged):
        assert call.result() == want[c], f"call {c}: pipelined result differs"
        call.free()
    _same_rings(lr, one)


def test_interleaved_with_record_and_key_steps(G):
    """Wire-bytes calls, record steps and key-string steps on the same ring with no synchronisation in between."""
    world = 2
    lr, twin = LocalRing(world, capacity=1 << 18, cap=8192), LocalRing(world, capacity=1 << 18, cap=8192)
    rng = np.random.default_rng(77)
    params = np.zeros(1, dtype=G.native.PARAMS_DTYPE)
    params["limit"] = 50; params["duration"] = 60000; params["behavior"] = O.REQ_IS_OWNER
    torch = lr.torch
    steps, expect = [], []
    for s in range(9):  # every step's input and the twin's answer first: uploading synchronises the device
        now = T0 + 10 * s
        kind = ("proto", "records", "keys")[s % 3]
        if kind == "proto":
            shards = [rpcs(rng, int(rng.integers(1000, 8000)), now, n_keys=5000) for _ in range(world)]
            steps.append((kind, now, Call(G, shards)))
            expect.append(twin_run(twin, shards, now)[0])
            continue
        keys = [[(b"ring_%09d" % int(i))[::-1] for i in rng.integers(0, 5000, int(rng.integers(0, 8000)))] for _ in range(world)]
        recs = []
        for ks in keys:
            b = np.zeros(len(ks), dtype=O.HREQ_DTYPE)
            b["key_xxh64"] = [O.xxh64(k) for k in ks]; b["key_fnv1"] = [O.fnv1_64(k) for k in ks]
            b["hits"] = 1; b["limit"] = 50; b["duration"] = 60000; b["created_at"] = now; b["behavior"] = O.REQ_IS_OWNER
            recs.append(b)
        ns = [len(b) for b in recs]
        if kind == "records":
            bufs, outs = lr.upload(recs)
            steps.append((kind, now, (bufs, outs, ns, None)))
        else:
            packed = [G.native.pack_keys(ks, 1, 0, 0) for ks in keys]
            bufs = [torch.from_numpy(p).to("cuda") for p in packed]
            outs = [torch.zeros((max(n, 1), 32), dtype=torch.uint8, device="cuda") for n in ns]
            steps.append((kind, now, (bufs, outs, ns, [len(p) for p in packed])))
        expect.append(twin.step(recs, now))
    torch.cuda.synchronize()
    for kind, now, x in steps:  # then every step enqueued back to back
        if kind == "proto":
            x.enqueue(lr, now)
        elif kind == "records":
            lr.enqueue(x[0], x[2], now, x[1])
        else:
            bufs, outs, ns, sizes = x
            G.native.p2p_step_keys_local_all(lr.p2ps, [b.data_ptr() for b in bufs], sizes, ns, params, now, G.clock_fill(now),
                                             [o.data_ptr() for o in outs], [s.cuda_stream for s in lr.streams])
    lr.sync()
    for s, ((kind, _, x), want) in enumerate(zip(steps, expect)):
        if kind == "proto":
            _check(x.result(), want, f"step {s}")
            x.free()
        else:
            _, outs, ns, _ = x
            got = [outs[r][:ns[r]].cpu().numpy().reshape(-1).view(O.HRESP_DTYPE) for r in range(world)]
            for r in range(world):
                assert np.array_equal(got[r], want[r]), f"step {s} ({kind}) shard {r} differs"
    _same_rings(lr, twin)


def test_rejected_call_then_a_normal_one(G):
    lr, twin = LocalRing(2, capacity=1 << 16, cap=8192), LocalRing(2, capacity=1 << 16, cap=8192)
    rng = np.random.default_rng(4)
    shards = [rpcs(rng, 3000, T0) for _ in range(2)]
    _check(run(G, lr, shards, T0), twin_run(twin, shards, T0)[0], "warm-up")
    before = [_scan(t).tobytes() for t in lr.tabs]
    bad = Call(G, [rpcs(rng, 2000, T0 + 1) for _ in range(2)])
    n = bad.n[1]
    bad.pk[1].array[8 * n + 4:8 * n + 8] = np.frombuffer(np.uint32(len(bad.pk[1].array)).tobytes(), dtype=np.uint8)
    with pytest.raises(G.native.GubError, match="shard 1: offsets"):
        bad.enqueue(lr, T0 + 1)
    bad.bound[0] -= 1
    with pytest.raises(G.native.GubError, match="out_cap"):
        bad.enqueue(lr, T0 + 1)
    bad.free()
    lr.sync()
    assert [_scan(t).tobytes() for t in lr.tabs] == before
    shards = [rpcs(rng, 4000, T0 + 2, adversarial=True) for _ in range(2)]
    _check(run(G, lr, shards, T0 + 2), twin_run(twin, shards, T0 + 2)[0], "after the refusals")
    _same_rings(lr, twin)


def test_plain_host_memory_is_refused(G):
    lr = LocalRing(2, capacity=1 << 12, cap=1024)
    packed, bound = G.native.pack_proto([W.message([W.item(b"a", b"b", hits=1)])], T0)
    out, off, st = np.zeros(bound, np.uint8), np.zeros(2, np.uint64), np.zeros(1, np.uint32)
    empty, _ = G.native.pack_proto([], T0)
    off0 = G.native.PinnedArray(1, np.uint64)
    with pytest.raises(G.native.GubError, match="page-locked"):
        G.native.p2p_step_proto_local_all(lr.p2ps, [packed.ctypes.data, empty.ctypes.data], [len(packed), len(empty)], [1, 0], G.clock_fill(T0),
                                          [out.ctypes.data, None], [bound, 0], [off.ctypes.data, off0.ptr], [st.ctypes.data, None],
                                          [s.cuda_stream for s in lr.streams])
    off0.free()
