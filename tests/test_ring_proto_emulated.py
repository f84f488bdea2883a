"""CPU: GetRateLimits wire bytes on the ring (gub_p2p_step_proto_local_all) through the emulated kernels (tests/ring_proto_emu_harness.cpp):
every shard's decode, S ring steps of cap items, every shard's encode.  The twin is an emulated record ring fed the restatement's records
(tests/_proto_wire.py prepare) chunked by the same rule, and its responses encoded by the restatement."""
import ctypes as C

import numpy as np
import pytest

import oracle_py as O
import _proto_wire as W
from _proto_emu import ProtoEmuTable
from _ring_proto_emu import ProtoP2PCluster
from ring_proto_traffic import PEER_TIMEOUT, encode, error_text, spread_items
from workloads import T0, make_clock

import gubernator_b200.native as N

GLOBAL = 2
COUNTED = ("requests", "cache_hit", "cache_miss", "over_limit")


def _points(world):
    from gubernator_b200.sharded import shard_addresses
    oring = O.Ring(0, 512)
    for a in shard_addresses(world):
        oring.add(a)
    return oring.points()


def _pair(world, cap, fused=False, capacity=1 << 13):
    pts, peers = _points(world)
    kw = dict(cap=cap, capacity_slots=capacity, pts=pts, peers=peers, max_batch=2048, finish_cap=3, fused=fused)
    return ProtoP2PCluster(world, **kw), ProtoP2PCluster(world, **kw)


def twin_call(twin, shards, now, force_global=False, global_mode=False, timeouts=None):
    """What the call must answer, from the twin record ring: shards[r] = (messages, created) of shard r.  Returns (S, per-shard
    [(status, bytes)], per-shard ring owners of the dense batch in GLOBAL mode)."""
    W_ = len(shards)
    plans, batches = [], []
    for msgs, created in shards:
        batch, plan = W.prepare(msgs, created)
        if force_global:
            batch["behavior"] |= np.uint32(GLOBAL)
        plans.append(plan); batches.append(batch)
    S = max((len(b) + twin.cap - 1) // twin.cap for b in batches)
    resp = [np.zeros(len(b), dtype=O.HRESP_DTYPE) for b in batches]
    owners = [np.zeros(len(b), dtype=np.uint8) for b in batches]
    for k in range(S):
        chunk = [b[k * twin.cap:(k + 1) * twin.cap] for b in batches]
        got = twin.step(chunk, make_clock(now), O.HRESP_DTYPE, global_mode=global_mode)
        if global_mode:
            got, own = got
            for r in range(W_):
                owners[r][k * twin.cap:k * twin.cap + len(chunk[r])] = own[r]
        for r in range(W_):
            resp[r][k * twin.cap:k * twin.cap + len(chunk[r])] = got[r]
    for r, idx in enumerate(timeouts or [None] * W_):
        if idx is not None and len(idx):
            resp[r][idx] = np.zeros(len(idx), dtype=O.HRESP_DTYPE)
            resp[r]["err_code"][idx] = PEER_TIMEOUT
    return S, [encode(p, r) for p, r in zip(plans, resp)], owners, [len(b) for b in batches]


def ring_call(ring, shards, now, **kw):
    packed = [N.pack_proto(m, c) for m, c in shards]
    return ring.step_proto([p for p, _ in packed], [len(m) for m, _ in shards], make_clock(now), out_caps=[b for _, b in packed], **kw)


def _check(got, want, what):
    for r, ((st, outs), exp) in enumerate(zip(got, want)):
        assert st == [s for s, _ in exp], f"{what} shard {r}: statuses differ"
        for m, (b, (_, wb)) in enumerate(zip(outs, exp)):
            assert b == wb, f"{what} shard {r} message {m}: response bytes differ"


def _scan(tab):
    return np.sort(tab.scan(N.ITEM_DTYPE), order=["key_xxh64", "key_fnv1"])


def _same_tables(a, b, world):
    for r in range(world):
        assert _scan(a.table(r)).tobytes() == _scan(b.table(r)).tobytes(), f"shard {r}: table contents differ from the twin's"
        assert a.table(r).counters() == b.table(r).counters(), f"shard {r}: counters differ from the twin's"


def traffic(rng, n_msgs, lo, hi, n_keys=400, edges=False, now=T0):
    msgs = [W.message(spread_items(rng, int(rng.integers(lo, hi)), n_keys=n_keys)) for _ in range(n_msgs)]
    if edges:
        picked = [m for n, m, _ in W.edge_messages(rng, now) if n != "malformed item past 1000"]
        for m in rng.choice(len(picked), 6, replace=False):
            msgs.insert(int(rng.integers(0, len(msgs) + 1)), picked[int(m)])
    created = np.array([now - int(rng.integers(0, 40)) for _ in msgs], dtype=np.int64)
    return msgs, created


@pytest.mark.parametrize("world", [1, 2, 4])
@pytest.mark.parametrize("path", ["pipeline", "fused"])
def test_calls_equal_the_record_ring(world, path):
    ring, twin = _pair(world, cap=512, fused=(path == "fused"))
    rng = np.random.default_rng(17 * world + (path == "fused"))
    for call in range(2):
        now = T0 + 300 * call
        shards = [traffic(rng, int(rng.integers(1, 5)), 0, 160, edges=(r + call) % 2 == 0, now=now) for r in range(world)]
        steps, got = ring_call(ring, shards, now)
        S, want, _, n_eval = twin_call(twin, shards, now)
        assert steps == S
        _check(got, want, f"call {call}")
    _same_tables(ring, twin, world)


@pytest.mark.parametrize("world", [2, 4])
def test_contiguous_split_equals_one_table(world):
    """n_r <= cap and a contiguous split: the bytes of gub_submit_proto_async on one table for the concatenated messages."""
    rng = np.random.default_rng(40 + world)
    ring, _ = _pair(world, cap=1024)
    one = ProtoEmuTable(1 << 15, max_batch=2048)
    for call in range(2):
        now = T0 + 500 * call
        msgs, created = traffic(rng, 3 * world, 10, 200, n_keys=300, edges=True, now=now)
        cuts = np.linspace(0, len(msgs), world + 1).astype(int)
        shards = [(msgs[cuts[r]:cuts[r + 1]], created[cuts[r]:cuts[r + 1]]) for r in range(world)]
        assert all(len(W.prepare(m, c)[0]) <= 1024 for m, c in shards)
        _, got = ring_call(ring, shards, now)
        packed, bound = N.pack_proto(msgs, created)
        st, outs, _, _ = one.submit_proto(packed, len(msgs), make_clock(now), bound)
        assert sum((s for s, _ in got), []) == st
        assert sum((o for _, o in got), []) == outs
    items = np.concatenate([_scan(ring.table(r)) for r in range(world)])
    assert np.sort(items, order=["key_xxh64", "key_fnv1"]).tobytes() == _scan(one).tobytes()
    for f in COUNTED:
        assert sum(ring.table(r).counters()[f] for r in range(world)) == one.counters()[f], f


def test_chunking_over_several_steps():
    """cap = 256, one shard with several cap of items, one with none, one with messages that evaluate nothing: S > 1, empty ingest in
    some steps."""
    world = 3
    ring, twin = _pair(world, cap=256)
    rng = np.random.default_rng(9)
    for call in range(2):
        now = T0 + 1000 * call
        big = traffic(rng, 5, 150, 260, now=now)
        bad = ([W.message([W.item(b"", b"u", hits=1)] * 20), W.message([W.item(b"x", b"\xff")])], np.full(2, now, dtype=np.int64))
        shards = [big, ([], np.zeros(0, dtype=np.int64)), bad] if call == 0 else [bad, big, traffic(rng, 2, 100, 200, now=now)]
        e0 = ring.epoch()
        steps, got = ring_call(ring, shards, now)
        S, want, _, n_eval = twin_call(twin, shards, now)
        assert steps == S and S == (max(n_eval) + 255) // 256 and S >= 3
        assert ring.epoch() == e0 + S
        _check(got, want, f"call {call}")
    _same_tables(ring, twin, world)


def test_no_evaluable_item_takes_no_step():
    """S = 0 (every message malformed or too large, or every item failing validation): the responses are written, no epoch advances,
    and the next call still matches the twin."""
    world = 2
    ring, twin = _pair(world, cap=512)
    rng = np.random.default_rng(21)
    warm = [traffic(rng, 2, 20, 100) for _ in range(world)]
    ring_call(ring, warm, T0)
    twin_call(twin, warm, T0)
    e0, t0 = ring.epoch(), twin.epoch()
    dead = [([W.message([W.item(b"x", b"y", hits=1)] * 1001), W.message([W.item(b"a", b"\xc0\xaf")])], np.full(2, T0, dtype=np.int64)),
            ([W.message([W.item(b"", b"u", hits=1), W.item(b"n", b"", hits=1), b""])], np.full(1, T0, dtype=np.int64))]
    steps, got = ring_call(ring, dead, T0 + 1)
    S, want, _, _ = twin_call(twin, dead, T0 + 1)
    assert steps == 0 and S == 0 and ring.epoch() == e0 and twin.epoch() == t0
    _check(got, want, "dead call")
    assert got[0][0] == [W.TOO_LARGE, W.MALFORMED] and got[1][0] == [W.OK] and len(got[1][1][0]) > 0
    nxt = [traffic(rng, 3, 20, 120, now=T0 + 2) for _ in range(world)]
    _, got = ring_call(ring, nxt, T0 + 2)
    _, want, _, _ = twin_call(twin, nxt, T0 + 2)
    _check(got, want, "next call")
    _same_tables(ring, twin, world)


def test_force_global_equals_global_records():
    """force_global on a GLOBAL ring: the twin fed the same records with GLOBAL set answers the same (replica answers for keys another
    shard owns), ends with the same tables, and routes every item to the same ring owner, which the hits queue reads."""
    world = 3
    ring, twin = _pair(world, cap=512)
    rng = np.random.default_rng(33)
    for call in range(3):
        now = T0 + 200 * call
        shards = [traffic(rng, 3, 30, 200, n_keys=120, now=now) for _ in range(world)]
        steps, got = ring_call(ring, shards, now, force_global=True, global_mode=True)
        S, want, owners, n_eval = twin_call(twin, shards, now, force_global=True, global_mode=True)
        assert steps == S
        _check([g[:2] for g in got], want, f"call {call}")
        for r in range(world):
            assert np.array_equal(got[r][2][:n_eval[r]], owners[r]), f"call {call} shard {r}: ring owners differ"
        assert len(np.unique(np.concatenate(owners))) == world, "every shard owns some of the keys"
    _same_tables(ring, twin, world)


def test_peer_timeout_is_answered_with_its_error_text():
    """Items whose owner never answered (GUB_ERR_PEER_TIMEOUT, as k_p2p_collect writes them) are encoded with gubernator.go:374's text."""
    world = 2
    ring, twin = _pair(world, cap=512)
    rng = np.random.default_rng(5)
    shards = [traffic(rng, 3, 20, 150) for _ in range(world)]
    n_eval = [len(W.prepare(m, c)[0]) for m, c in shards]
    timeouts = [np.sort(rng.choice(n, min(n, 25), replace=False)).astype(np.uint32) for n in n_eval]
    _, got = ring_call(ring, shards, T0, timeouts=timeouts)
    _, want, _, _ = twin_call(twin, shards, T0, timeouts=timeouts)
    _check(got, want, "timeout call")
    key = W.prepare(*shards[0])[1]
    texts = b"".join(got[0][1])
    first = next(k for st, per in key for _, j, k in per if j == int(timeouts[0][0]))
    assert b"Error while fetching rate limit '" + first + b"' from peer: context deadline exceeded" in texts
    L = N.lib()
    L.gub_format_error.argtypes = [C.c_int, C.c_char_p, C.c_int32, C.c_char_p, C.c_size_t]
    buf = C.create_string_buffer(256)
    L.gub_format_error(PEER_TIMEOUT, b"ns_key", 0, buf, 256)
    assert buf.value == b"Error while fetching rate limit 'ns_key' from peer: context deadline exceeded"
    assert len(error_text(PEER_TIMEOUT, b"", 0)) == 71


def test_refusals_leave_every_shard_untouched():
    world = 3
    ring, _ = _pair(world, cap=512)
    rng = np.random.default_rng(8)
    shards = [traffic(rng, 2, 20, 100) for _ in range(world)]
    ring_call(ring, shards, T0)
    e0 = ring.epoch()
    before = [_scan(ring.table(r)).tobytes() for r in range(world)]
    counters = [ring.table(r).counters() for r in range(world)]
    packed = [N.pack_proto(m, c) for m, c in shards]
    n = [len(m) for m, _ in shards]
    bad = packed[1][0].copy()
    bad[8 * n[1] + 4:8 * n[1] + 8] = np.frombuffer(np.uint32(len(bad)).tobytes(), dtype=np.uint8)  # offsets[1] past the buffer
    assert ring.step_proto([packed[0][0], bad, packed[2][0]], n, make_clock(T0 + 1), out_caps=[b for _, b in packed]) is None
    caps = [b for _, b in packed]
    caps[2] -= 1
    assert ring.step_proto([p for p, _ in packed], n, make_clock(T0 + 1), out_caps=caps) is None
    assert ring.epoch() == e0
    assert [_scan(ring.table(r)).tobytes() for r in range(world)] == before
    assert [ring.table(r).counters() for r in range(world)] == counters
