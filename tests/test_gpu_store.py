"""gub_submit_keys_store_async on the H100: the Store plugin's miss list and change log computed on the device around the key-string path,
checked against the host layer (V1Instance + set_store on a twin table, csrc/host_v1.cpp) and the oracle model of its rule
(tests/_store_emu.py model_batch): responses, the ordered Store call sequence with its items, counters and the final table."""
import os

import numpy as np
import pytest

import oracle_py as O
import _store_emu as S
from workloads import T0, adversarial_batch, bench_requests, zipf_ids

pytestmark = pytest.mark.gpu

ITEM_FIELDS = ("algorithm", "status", "limit", "duration", "remaining", "remaining_f", "stamp", "burst", "expire_at")


@pytest.fixture(scope="module")
def G():
    import gubernator_b200 as g
    if os.environ.get("GUB_PATH") == "fused":
        pytest.skip("the Store path runs on the four-kernel pipeline only")
    return g


class MockStore:
    """MockStore2 of the reference (mock_store_test.go:28) keyed by key string: records the calls, returns programmed items."""

    def __init__(self, items=None):
        self.calls, self.items = [], dict(items or {})

    def get(self, req, key):
        self.calls.append(("Get", key))
        return self.items.get(key)

    def on_change(self, req, key, item):
        self.calls.append(("OnChange", key, item))

    def remove(self, key):
        self.calls.append(("Remove", key))


def _item_dict(rec_item):
    return {f: (float(rec_item[f]) if f == "remaining_f" else int(rec_item[f])) for f in ITEM_FIELDS}


class KeysBatch:
    """One batch as key strings (packed for the device), as records (for the oracle) and as V1Instance requests."""

    def __init__(self, G, names, uks, reqs):
        self.keys = [f"{a}_{b}".encode() for a, b in zip(names, uks)]
        self.reqs = reqs.copy()
        self.reqs["key_xxh64"] = [O.xxh64(k) for k in self.keys]
        self.reqs["key_fnv1"] = [O.fnv1_64(k) for k in self.keys]
        creqs, self.params, self.base = G.native.compact_batch(self.reqs.astype(G.REQ_DTYPE))
        self.packed = G.native.pack_keys(self.keys, self.reqs["hits"], creqs["params"], creqs["created_delta"])
        self.v1 = [dict(name=a, unique_key=b, hits=int(r["hits"]), limit=int(r["limit"]), duration=int(r["duration"]), burst=int(r["burst"]),
                        algorithm=int(r["algorithm"]), behavior=int(r["behavior"]) & 0xFF, created_at=int(r["created_at"]))
                   for a, b, r in zip(names, uks, self.reqs)]


def adv_batch(G, rng, n, n_keys, now, owner_only=False):
    reqs = adversarial_batch(rng, n, n_keys, now)
    if owner_only:
        reqs["behavior"] |= O.REQ_IS_OWNER
    ids = {}
    for i in range(n_keys):
        s = f"adv_k{i:09d}".encode()
        ids[(O.xxh64(s), O.fnv1_64(s))] = i
    uks = [f"k{ids[(int(a), int(b))]:09d}" for a, b in zip(reqs["key_xxh64"], reqs["key_fnv1"])]
    return KeysBatch(G, ["adv"] * n, uks, reqs)


def zipf_batch(G, rng, n, n_keys, now):
    ids = zipf_ids(rng, n, n_keys, 1.1)
    return KeysBatch(G, ["bench"] * n, [f"k{int(i):09d}" for i in ids], bench_requests(ids, now))


class Native:
    """The table plus the caller side of the new entry point: page-locked buffers, a Get callback over a MockStore, the replay."""

    def __init__(self, G, tab, store):
        self.G, self.tab, self.store = G, tab, store

    def submit(self, kb, now, get=True, failing=False):
        G, n = self.G, len(kb.keys)
        self.out = G.native.PinnedArray(max(n, 1), G.RESP_DTYPE)
        self.ch = G.native.PinnedArray(max(n, 1), G.native.STORE_REC_DTYPE)
        self.nc = G.native.PinnedArray(1, np.uint32)
        self.nc.array[0] = 12345

        def cb(misses):
            if failing:
                return 3
            for m in misses:
                key = kb.keys[int(m["first"])].decode()
                it = self.store.get(None, key)
                if it is not None:
                    for f in ITEM_FIELDS:
                        m["item"][f] = it.get(f, 0)
                    m["flags"] |= G.native.STORE_FOUND
            return 0
        tk = self.tab.submit_keys_store_async(kb.packed.ctypes.data, len(kb.packed), n, kb.params.ctypes.data, len(kb.params), kb.base,
                                              G.clock_fill(now), cb if get else None, self.out.ptr, self.ch.ptr, self.nc.ptr)
        return tk

    def finish(self, kb, tk):
        self.tab.wait(tk)
        n = len(kb.keys)
        recs = self.ch.array[:int(self.nc.array[0])].copy()
        for r in recs:
            key = kb.keys[int(r["first"])].decode()
            if r["flags"] & self.G.native.STORE_REMOVE:
                self.store.remove(key)
            if r["flags"] & self.G.native.STORE_CHANGE:
                self.store.on_change(None, key, _item_dict(r["item"]))
        return self.out.array[:n].copy(), recs


def _v1_resp(G, got):
    out = np.zeros(len(got), dtype=G.RESP_DTYPE)
    for i, o in enumerate(got):
        out[i] = (o["status"], o["err_code"], o["limit"], o["remaining"], o["reset_time"]) if not o["err_code"] else (0, o["err_code"], 0, 0, 0)
    return out


def _scan(tab):
    s = tab.scan()
    return s[np.lexsort((s["key_fnv1"], s["key_xxh64"]))]


@pytest.mark.parametrize("algo", [0, 1])
def test_store_call_sequences(G, algo):
    """The cases of store_test.go:127-533 (the host layer's test_store_plugin_call_sequences) through the new entry point."""
    key = "test_over_limit_account:1234"
    req = dict(name="test_over_limit", unique_key="account:1234", algorithm=algo, duration=1000, limit=10, hits=1, behavior=O.REQ_IS_OWNER)

    def run(items, reqs_list, now=T0):
        st = MockStore(items)
        nat = Native(G, G.Table(4096), st)
        res = []
        for r in reqs_list:
            a = np.zeros(1, dtype=O.HREQ_DTYPE)
            for f in ("hits", "limit", "duration", "burst", "algorithm", "behavior"):
                a[f] = r.get(f, 0)
            a["created_at"] = now
            kb = KeysBatch(G, [r["name"]], [r["unique_key"]], a)
            resp, _ = nat.finish(kb, nat.submit(kb, now))
            res.append(resp[0])
        return st, res

    def item(duration=1000, stamp=T0, expire=None, algorithm=algo):
        return dict(algorithm=algorithm, limit=10, duration=duration, remaining=10, remaining_f=10.0, stamp=stamp, burst=10,
                    expire_at=expire if expire is not None else stamp + duration)

    st, res = run({}, [req, req])
    assert (int(res[0]["limit"]), int(res[0]["status"])) == (10, 0)
    assert [c[0] for c in st.calls] == ["Get", "OnChange", "OnChange"] and st.calls[1][2]["limit"] == 10 and st.calls[1][2]["duration"] == 1000
    st, res = run({key: item()}, [req])
    assert (int(res[0]["limit"]), int(res[0]["status"]), int(res[0]["remaining"])) == (10, 0, 9)
    assert [c[0] for c in st.calls] == ["Get", "OnChange"]
    st, res = run({key: item(algorithm=1 - algo)}, [req])
    assert [c[0] for c in st.calls] == ["Get", "Remove", "OnChange"] and st.calls[2][2]["algorithm"] == algo
    if algo == 0:
        req2 = dict(req, duration=8000)
        st, res = run({key: item(duration=5000)}, [req2])
        it = st.calls[-1][2]
        assert st.calls[-1][0] == "OnChange" and it["expire_at"] == it["stamp"] + 8000 and it["duration"] == 8000 and it["limit"] == 10
        long_ago = T0 - 100000
        st, res = run({key: item(duration=500000, stamp=long_ago, expire=long_ago + 500000)}, [req2])
        it = st.calls[-1][2]
        assert it["expire_at"] == it["stamp"] + 8000 and it["stamp"] == T0 and it["duration"] == 8000


def _store_items(rng, kb, now, frac=0.35):
    items = {}
    for k in sorted(set(kb.keys)):
        if rng.random() < frac:
            kind = ("token", "leaky", "expired")[int(rng.integers(0, 3))]
            r = S.store_item(rng, now, kind)
            items[k.decode()] = {f: (float(r[f]) if f == "remaining_f" else int(r[f])) for f in ITEM_FIELDS}
    return items


def test_random_traffic_matches_host_layer_and_model(G):
    """Zipf and adversarial batches on three sides, each with its own mock store pre-filled alike: the new path, V1Instance + set_store
    on a twin table, the oracle model.  Same responses, Store calls and items, counters and final table."""
    rng = np.random.default_rng(2024)
    nat = Native(G, G.Table(1 << 15), MockStore())
    inst = G.V1Instance(capacity_slots=1 << 15, now_ms=T0)
    host = MockStore()
    inst.set_store(host)
    pool = O.Pool(now_ms=T0)
    now = T0
    for b in range(6):
        now += int(rng.choice([0, 1, 900, 70000]))
        kb = adv_batch(G, rng, 3000, int(rng.choice([40, 300])), now, owner_only=True) if b % 2 else zipf_batch(G, rng, 8000, 3000, now)
        items = _store_items(rng, kb, now)
        nat.store.items, host.items = dict(items), dict(items)
        nat.store.calls, host.calls = [], []
        got, recs = nat.finish(kb, nat.submit(kb, now))
        inst.set_now(now)
        want = _v1_resp(G, inst.get_rate_limits(kb.v1, unbounded=True))
        assert np.array_equal(got, want), f"batch {b}: responses differ from the host layer"
        assert nat.store.calls == host.calls, f"batch {b}: Store calls differ"
        model_items = {}
        for k, it in items.items():
            r = np.zeros(1, dtype=S.ITEM_DTYPE)[0]
            for f in ITEM_FIELDS:
                r[f] = it[f]
            model_items[(O.xxh64(k.encode()), O.fnv1_64(k.encode()))] = r
        _, mresp, mrecs = S.model_batch(pool, kb.reqs, now, model_items)
        assert np.array_equal(got, mresp), f"batch {b}: responses differ from the model"
        assert recs.tobytes() == mrecs.tobytes(), f"batch {b}: records differ from the model"
    assert nat.tab.counters() == inst.table.counters()
    assert _scan(nat.tab).tobytes() == _scan(inst.table).tobytes()


def test_write_behind_store_matches_plain_path_with_depth_in_flight(G):
    """get = NULL: responses byte-identical to gub_submit_keys_async on a twin table, records those of a store that finds nothing, with
    gub_pipeline_depth() submissions in flight."""
    rng = np.random.default_rng(5)
    tab, twin, pool = G.Table(1 << 15), G.Table(1 << 15), O.Pool(now_ms=T0)
    depth = G.native.lib().gub_pipeline_depth(tab._h)
    now = T0
    for round_ in range(2):
        pend = []
        for k in range(depth):
            now += int(rng.choice([0, 1, 900]))
            kb = adv_batch(G, rng, 2000, 200, now) if k % 2 else zipf_batch(G, rng, 6000, 2000, now)
            nat = Native(G, tab, MockStore())
            pend.append((kb, now, nat, nat.submit(kb, now, get=False)))
            tout = np.zeros(len(kb.keys), dtype=G.RESP_DTYPE)
            twin.wait(twin.submit_keys_async(kb.packed.ctypes.data, len(kb.packed), len(kb.keys), kb.params.ctypes.data, len(kb.params), kb.base,
                                             G.clock_fill(now), tout.ctypes.data))
            pend[-1] += (tout,)
        for kb, t, nat, tk, tout in pend:
            got, recs = nat.finish(kb, tk)
            assert got.tobytes() == tout.tobytes()
            _, mresp, mrecs = S.model_batch(pool, kb.reqs, t, {})
            assert np.array_equal(got, mresp) and recs.tobytes() == mrecs.tobytes()
    assert _scan(tab).tobytes() == _scan(twin).tobytes()


def test_failing_callback_changes_nothing(G):
    rng = np.random.default_rng(9)
    nat = Native(G, G.Table(1 << 14), MockStore())
    kb = zipf_batch(G, rng, 4000, 1500, T0)
    nat.finish(kb, nat.submit(kb, T0))
    scan, counters = _scan(nat.tab), nat.tab.counters()
    kb2 = zipf_batch(G, rng, 4000, 3000, T0 + 10)
    with pytest.raises(G.native.GubError, match="get callback failed"):
        nat.submit(kb2, T0 + 10, failing=True)
    assert nat.tab.counters() == counters and _scan(nat.tab).tobytes() == scan.tobytes()


def test_refusals_and_empty_batch(G, monkeypatch):
    rng = np.random.default_rng(1)
    tab = G.Table(1 << 14, max_batch=1024)
    nat = Native(G, tab, MockStore())
    with pytest.raises(G.native.GubError, match="exceeds max_batch"):
        nat.submit(zipf_batch(G, rng, 1025, 100, T0), T0)
    kb = zipf_batch(G, rng, 100, 10, T0)
    out = np.zeros(100, dtype=G.RESP_DTYPE)
    ch, nc = np.zeros(100, dtype=G.native.STORE_REC_DTYPE), np.zeros(1, dtype=np.uint32)
    with pytest.raises(G.native.GubError, match="page-locked"):
        tab.submit_keys_store_async(kb.packed.ctypes.data, len(kb.packed), 100, kb.params.ctypes.data, len(kb.params), kb.base, G.clock_fill(T0),
                                    None, out.ctypes.data, ch.ctypes.data, nc.ctypes.data)
    empty = KeysBatch(G, [], [], np.zeros(0, dtype=O.HREQ_DTYPE))
    empty.packed = np.zeros(16, dtype=np.uint8)
    empty.params = np.zeros(1, dtype=G.native.PARAMS_DTYPE)
    _, recs = nat.finish(empty, nat.submit(empty, T0))
    assert len(recs) == 0 and int(nat.nc.array[0]) == 0
    monkeypatch.setenv("GUB_PATH", "fused")
    fused = Native(G, G.Table(1 << 14), MockStore())
    with pytest.raises(G.native.GubError, match="GUB_PATH=fused"):
        fused.submit(kb, T0)


def test_parked_inserts_small_table(G):
    """A table too small for the batch parks inserts: responses equal the plain path's, each OnChange item is the state the batch left."""
    rng = np.random.default_rng(17)
    tab, twin = G.Table(512), G.Table(512)
    nat = Native(G, tab, MockStore())
    now = T0
    for b in range(3):
        kb = zipf_batch(G, rng, 2000, 1000, now)
        got, recs = nat.finish(kb, nat.submit(kb, now))
        tout = np.zeros(len(kb.keys), dtype=G.RESP_DTYPE)
        twin.wait(twin.submit_keys_async(kb.packed.ctypes.data, len(kb.packed), len(kb.keys), kb.params.ctypes.data, len(kb.params), kb.base,
                                         G.clock_fill(now), tout.ctypes.data))
        assert got.tobytes() == tout.tobytes()
        assert len(recs) == len(set(kb.keys)) and np.all(recs["flags"] == G.native.STORE_CHANGE)
        tok = recs[recs["item"]["algorithm"] == 0]  # (a token bucket's response shows its stored Remaining and ExpireAt)
        last = got[tok["last"]]
        assert len(tok) and np.array_equal(tok["item"]["remaining"], last["remaining"]) and np.array_equal(tok["item"]["expire_at"], last["reset_time"])
        now += 1
