"""The table probe in rounds (cursor_open of gubernator_b200/csrc/gub_kernels.cuh), on the CPU.

cursor_open checks the home slot, then loads the key / tag pairs of PROBE_ROUND slots at once and scans them in probe order.  It
must give exactly what probing one slot after the other gives: the first matching slot, else the first tombstone or EMPTY seen, and
never a slot outside the window [home, home + MAX_PROBE).  tests/probe_rounds_emu_harness.cpp runs cursor_open over a table image
built here; _one_slot_probe restates the one-slot loop.  The end-to-end tests push long clusters through both evaluation paths of
the emulated kernels against the oracle."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import oracle_py as O
import _kernel_emu as E
from workloads import T0, make_clock

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SO = os.path.join(HERE, "libprobe_rounds_emu_test.so")
SRC = [os.path.join(HERE, "probe_rounds_emu_harness.cpp"), os.path.join(HERE, "cuda_emu.h"),
       os.path.join(ROOT, "gubernator_b200", "csrc", "gub_kernels.cuh"), os.path.join(ROOT, "gubernator_b200", "csrc", "bucket_math.cuh")]

EMPTY, TOMB = 0, 1
F_LIVE = 4
M64 = (1 << 64) - 1


@pytest.fixture(scope="module")
def L():
    if not os.path.exists(SO) or any(os.path.getmtime(s) > os.path.getmtime(SO) for s in SRC):
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-msse2", "-ffp-contract=off", "-Wno-unknown-pragmas",
                               "-I", os.path.join(ROOT, "include"), "-x", "c++", SRC[0], "-o", SO])
    lib = C.CDLL(SO)
    vp = C.c_void_p
    lib.emu_probe.argtypes = [vp, C.c_uint64, vp, vp, C.c_uint32, vp, vp, vp, vp, vp]
    lib.emu_probe.restype = None
    return lib


@pytest.fixture(scope="module")
def R(L):
    return int(L.emu_probe_round())


@pytest.fixture(scope="module")
def W(L):
    return int(L.emu_max_probe())


def _table(cap):
    """A zeroed (all EMPTY) table image of `cap` 64-byte slots, 64-byte aligned like the device table."""
    raw = np.zeros(cap * 8 + 8, dtype=np.uint64)
    off = (-raw.ctypes.data % 64) // 8
    t = raw[off:off + cap * 8].reshape(cap, 8)
    assert t.ctypes.data % 64 == 0
    return t


def _home(key, cap):
    return (key * cap) >> 64


def _key_with_home(rng, h, cap):
    """A key (>= 2) whose home slot in a table of `cap` slots is h."""
    lo = max(2, -(-(h << 64) // cap))
    hi = min(M64, -(-((h + 1) << 64) // cap) - 1)
    assert lo <= hi
    return rng.randint(lo, hi)


def _put(t, i, key, tag, rng):
    t[i, 0] = key
    t[i, 1] = (tag << 8) | F_LIVE
    t[i, 2:] = [rng.getrandbits(64) for _ in range(6)]


def _one_slot_probe(t, cap, key, tag, window):
    """cursor_open as it probed before the rounds: one slot per step."""
    idx = home = _home(key, cap)
    slot = -1
    for _ in range(window):
        w0, w1 = int(t[idx, 0]), int(t[idx, 1])
        if w0 == key and (w1 >> 8) == tag:
            return True, idx, home
        if w0 == EMPTY:
            if slot < 0:
                slot = idx
            break
        if w0 == TOMB and slot < 0:
            slot = idx
        idx = 0 if idx + 1 == cap else idx + 1
    return False, slot, home


def _check(L, t, keys, tags, window):
    cap = t.shape[0]
    n = len(keys)
    k = np.array(keys, dtype=np.uint64)
    g = np.array(tags, dtype=np.uint64)
    found, slot, home = np.zeros(n, np.uint8), np.zeros(n, np.int64), np.zeros(n, np.uint64)
    b, old_ok = np.zeros((n, 9), np.uint64), np.zeros(n, np.uint8)
    L.emu_probe(t.ctypes.data, cap, k.ctypes.data, g.ctypes.data, n, found.ctypes.data, slot.ctypes.data, home.ctypes.data, b.ctypes.data,
                old_ok.ctypes.data)
    hits = 0
    for i in range(n):
        want = _one_slot_probe(t, cap, int(k[i]), int(g[i]), window)
        got = (bool(found[i]), int(slot[i]), int(home[i]))
        assert got == want, f"key {i} ({int(k[i]):#x}, cap {cap}): got {got}, want {want}"
        assert old_ok[i]
        if want[0]:
            w = [int(v) for v in t[want[1]]]
            assert [int(v) for v in b[i]] == [w[0], w[1] >> 8, w[1] & 0xFF] + w[2:], f"key {i}: bucket"
            hits += 1
        else:
            assert [int(v) for v in b[i]] == [int(k[i]), int(g[i])] + [0] * 7, f"key {i}: miss bucket"
    return hits


@pytest.mark.parametrize("alpha", [0.3, 0.5, 0.7, 0.85, 0.95])
@pytest.mark.parametrize("cap", [4096, 1021])
def test_random_tables_with_tombstones(L, W, alpha, cap):
    """Random-order linear-probing inserts up to load factor alpha, then a tenth of the items removed (tombstones); lookups of resident
    keys, of removed ones, of resident keys under another tag, and of absent keys."""
    rng = random.Random(int(alpha * 100) * 7 + cap)
    t = _table(cap)
    live = []
    while len(live) < int(alpha * cap):
        key, tag = rng.randint(2, M64), rng.getrandbits(56)
        i, d = _home(key, cap), 0
        while int(t[i, 0]) > TOMB:
            i, d = (0 if i + 1 == cap else i + 1), d + 1
        if d >= W:  # inserts stay inside the probe window
            continue
        _put(t, i, key, tag, rng)
        live.append((key, tag, i))
    removed = rng.sample(live, len(live) // 10)
    for _, _, i in removed:
        t[i, 0] = TOMB
    keys = [(k, g) for k, g, _ in live] + [(k, g) for k, g, _ in removed]
    keys += [(k, g ^ 1) for k, g, _ in rng.sample(live, 100)] + [(rng.randint(2, M64), rng.getrandbits(56)) for _ in range(500)]
    hits = _check(L, t, [k for k, _ in keys], [g for _, g in keys], W)
    assert hits == len(live) - len(removed)


@pytest.mark.parametrize("home_at", ["middle", "end"])
def test_clusters_with_a_hole_at_every_position(L, R, W, home_at):
    """Keys sharing one home, in a run 3 rounds long plus one slot; one TOMB or EMPTY at each position of the run in turn (the first
    and last slot of every round included), a resident key under another tag in front; every key and an absent one looked up."""
    cap = 512
    rng = random.Random(11 if home_at == "middle" else 12)
    h = 200 if home_at == "middle" else cap - 2  # "end": the run wraps to slot 0
    run = 1 + 3 * R + 1
    for hole_kind in (TOMB, EMPTY):
        for q in range(run):
            t = _table(cap)
            keys = [_key_with_home(rng, h, cap) for _ in range(run)]
            tags = [rng.getrandbits(56) for _ in range(run)]
            for p in range(run):
                _put(t, (h + p) % cap, keys[p], tags[p], rng)
            t[(h + q) % cap, 0] = hole_kind
            t[(h + run) % cap, 0] = EMPTY
            look = keys + [keys[0], _key_with_home(rng, h, cap)]
            ltag = tags + [tags[0] ^ 2, rng.getrandbits(56)]
            _check(L, t, look, ltag, W)


def test_tombstones_before_the_key_and_past_the_empty(L, R, W):
    """Several tombstones in one round and across rounds (the first one is the reusable slot), a key behind them, and a key past an
    EMPTY (not reachable)."""
    cap = 256
    rng = random.Random(5)
    h = 17
    for layout in ("TTKx", "xTxTxTxK", "xxxxTxxxxxxxTxxxK", "xxKExK", "xxxxxxxxExxK", "TTTTTTTTTTTTTE"):
        t = _table(cap)
        keys, tags = [], []
        for p, c in enumerate(layout):
            k, g = _key_with_home(rng, h, cap), rng.getrandbits(56)
            if c in "xK":
                _put(t, h + p, k, g, rng)
            else:
                t[h + p, 0] = TOMB if c == "T" else EMPTY
            keys.append(k); tags.append(g)
        _check(L, t, keys + [_key_with_home(rng, h, cap)], tags + [1], W)


@pytest.mark.parametrize("cap", [1, 2, 3, 4, 5, 7, 8, 9])
def test_tables_smaller_than_a_round(L, R, W, cap):
    """Tables of fewer slots than one round (and around it): every index of a round wraps by itself, and a full table is walked around
    many times within the window, as before."""
    rng = random.Random(cap)
    for variant in range(4 * cap + 2):
        t = _table(cap)
        keys = [rng.randint(2, M64) for _ in range(cap)]
        tags = [rng.getrandbits(56) for _ in range(cap)]
        for i in range(cap):
            _put(t, i, keys[i], tags[i], rng)
        if variant % 2:
            t[variant % cap, 0] = TOMB
        if variant % 3 == 2:
            t[(variant // 3) % cap, 0] = EMPTY
        _check(L, t, keys + [rng.randint(2, M64) for _ in range(3)], tags + [rng.getrandbits(56) for _ in range(3)], W)


def test_full_window_and_its_last_slot(L, R, W):
    """No EMPTY in the window: a key in the window's last slot is found, one just past it is not, an absent key reports the first
    tombstone of the window or none; the same with the window wrapping at the table's end."""
    cap = 2 * W + 64
    rng = random.Random(3)
    for h in (100, cap - 37):
        t = _table(cap)
        for i in range(cap):
            _put(t, i, _key_with_home(rng, i, cap), rng.getrandbits(56), rng)
        last, past = _key_with_home(rng, h, cap), _key_with_home(rng, h, cap)
        _put(t, (h + W - 1) % cap, last, 7, rng)
        _put(t, (h + W) % cap, past, 8, rng)
        absent = _key_with_home(rng, h, cap)
        assert _check(L, t, [last, past, absent], [7, 8, 9], W) == 1
        t[(h + W - 1) % cap, 0] = TOMB  # a tombstone at the window's last slot is still the reusable slot
        _check(L, t, [past, absent], [8, 9], W)
        t[(h + 300) % cap, 0] = TOMB
        _check(L, t, [past, absent], [8, 9], W)


# ---- end to end: long clusters through both evaluation paths against the oracle ---------------------------------------------------

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


@pytest.mark.parametrize("path", ["pipeline", "fused"])
@pytest.mark.parametrize("rounds", [3, 40])
def test_long_clusters_match_oracle(R, rounds, path):
    """One cluster of keys sharing a home near the table's end (it wraps), `rounds` probe rounds long; every other key short-lived.
    After a sweep the survivors sit behind tombstones; then survivors, re-created keys and new keys arrive in random order."""
    import gubernator_b200 as G
    cap = 1024
    n = rounds * R + 2
    rng = random.Random(rounds)
    keys = np.array(sorted({_key_with_home(rng, cap - 3, cap) for _ in range(n + 40)})[:n + 40], dtype=np.uint64)
    assert len(keys) == n + 40
    nrng = np.random.default_rng(rounds)
    nrng.shuffle(keys)
    tab, pool = E.EmuTable(cap, fused=(path == "fused")), O.Pool(now_ms=T0)

    def batch(ks, now, duration):
        r = np.zeros(len(ks), dtype=G.REQ_DTYPE)
        r["key_xxh64"] = ks; r["key_fnv1"] = (ks * np.uint64(0x9E3779B97F4A7C15)) | np.uint64(0x100)
        r["hits"] = 1; r["limit"] = 10; r["duration"] = duration; r["created_at"] = now
        r["algorithm"] = (ks & np.uint64(1)).astype(np.uint32); r["behavior"] = G.native.REQ_IS_OWNER
        return r
    first = batch(keys[:n], T0, np.where(np.arange(n) % 2 == 0, 1000, 100000))
    _cmp(tab.submit(first, make_clock(T0), O.HRESP_DTYPE), pool.submit_hashed(first), "fill")
    now = T0 + 5000
    pool.set_now(now)
    assert tab.sweep(now) == (n + 1) // 2
    again = batch(keys, now, 100000)
    nrng.shuffle(again)
    _cmp(tab.submit(again, make_clock(now), O.HRESP_DTYPE), pool.submit_hashed(again), "after the sweep")
    again2 = batch(keys[::-1].copy(), now + 1, 100000)  # every key resident now: hits all along the cluster
    pool.set_now(now + 1)
    _cmp(tab.submit(again2, make_clock(now + 1), O.HRESP_DTYPE), pool.submit_hashed(again2), "all resident")
    _check_state(G, tab, pool)
