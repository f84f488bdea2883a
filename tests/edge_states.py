"""Bucket states that only a Store or a Loader can install, and request plans aimed at every evaluation route.  Test data only.

Requests alone never build these states: a leaky Remaining that is NaN (with a payload), +-Inf, -0.0, subnormal, >= 2^52 or above
Burst; an UpdatedAt far ahead of the clock or at INT64_MIN; an ExpireAt at either end of int64; a token Remaining outside [0, Limit].
gub_add_items, the Store's Get on the key-string path and the ring's Store path install whatever the plugin returns, and the
reference evaluates such items with algorithms.go like any other.

items()          ITEM_DTYPE records (gubernator_b200.native), one per lattice point, keys not yet assigned
oracle_item(r)   the same record as an oracle CacheItem, copied bit for bit (signalling NaNs arrive unchanged)
buckets()        the slot images of the items as the kernels open them (bucket_math.cuh's Bucket)
pairs()          (slot image, request, target rank) triples drawn around the buckets, for the element-wise bucket_math checks
plans(r)         request plans for one item: lists of REQ_DTYPE field dicts, one key per (item, plan) pair
"""
import ctypes as C

import numpy as np

import oracle_py as O
from gubernator_b200.native import ITEM_DTYPE
from workloads import T0

NOW = T0 + 777
LIMIT, DURATION = 100, 60_000
RATE = DURATION // LIMIT  # ms per token of the base leaky item
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


def wrap(v):
    """Go's int64 wrap-around."""
    return (int(v) + (1 << 63)) % (1 << 64) - (1 << 63)


def fbits(x):
    return int(np.array([x], dtype=np.float64).view(np.uint64)[0])


# leaky Remaining as IEEE-754 bits
NAN_BITS = [0x7FF8000000000001, 0xFFF80000DEADBEEF, 0x7FFC00000000ABCD, 0x7FF0000000000001, 0xFFF4000000000123]  # quiet +/-, quiet, signalling +/-
LEAKY_REMAINING = [fbits(x) for x in (0.0, -0.0, 5e-324, 0.5, 0.9999999999999999, 1.0, LIMIT - 0.5, float(LIMIT), LIMIT + 0.5,
                                      2.0 ** 52 - 0.5, 2.0 ** 52, 2.0 ** 53 + 2, 2.0 ** 63, -2.0 ** 63, 1e300, -1e300, np.inf, -np.inf,
                                      -2.5, 57.7)] + NAN_BITS
LEAKY_BURST = [0, 1, LIMIT, 3 * LIMIT, I64_MAX, -5]
LEAKY_STAMP = [NOW, NOW - 5 * RATE, NOW + (1 << 62), I64_MIN]
RATE_PAIRS = [(0, LIMIT), (DURATION, 0), (0, 0), (-DURATION, LIMIT)]  # (duration, limit): rate 0, +Inf, NaN, negative
TOKEN_LIMITS = [0, 1, LIMIT, -1, I64_MAX]
EXPIRE_AT = [NOW - 1, NOW, NOW + 1, I64_MIN, I64_MAX]
INVALID_AT = [NOW - 1000, NOW + 1000]
HITS = [I64_MIN, -1, 0, 1, 2, LIMIT, I64_MAX]
UNIFORM_RUNS = [2, 32, 33, 255, 256, 257, 1024, 1025, 7300]


def _item(algorithm, limit=LIMIT, duration=DURATION, stamp=NOW, expire_at=NOW + DURATION, invalid_at=0, remaining=0, status=0,
          rem_bits=0, burst=0):
    r = np.zeros(1, dtype=ITEM_DTYPE)
    r["algorithm"], r["limit"], r["duration"], r["stamp"] = algorithm, limit, duration, stamp
    r["expire_at"], r["invalid_at"] = expire_at, invalid_at
    if algorithm == 1:
        r["remaining_f"].view(np.uint64)[0] = rem_bits
        r["burst"] = burst
    else:
        r["remaining"], r["status"] = remaining, status
    return r[0]


def items():
    out = []
    for rb in LEAKY_REMAINING:
        out.append(_item(1, rem_bits=rb, burst=LIMIT))
        out.append(_item(1, rem_bits=rb, burst=LIMIT, stamp=NOW - 5 * RATE))  # a request at NOW leaks 5 into it
    for b in LEAKY_BURST:
        out.append(_item(1, rem_bits=fbits(50.0), burst=b))
    for s in LEAKY_STAMP:
        out.append(_item(1, rem_bits=fbits(50.0), burst=LIMIT, stamp=s))
    for d, lim in RATE_PAIRS:
        for rb in (fbits(50.0), NAN_BITS[1]):
            out.append(_item(1, limit=lim, duration=d, rem_bits=rb, burst=LIMIT))
    for lim in TOKEN_LIMITS:
        for rem in (I64_MIN, -1, 0, 1, wrap(lim - 1), lim, wrap(lim + 1), I64_MAX):
            for st in (O.UNDER_LIMIT, O.OVER_LIMIT):
                out.append(_item(0, limit=lim, remaining=rem, status=st))
    for e in EXPIRE_AT:
        out.append(_item(0, remaining=40, expire_at=e))
        out.append(_item(1, rem_bits=fbits(40.5), burst=LIMIT, expire_at=e))
    for inv in INVALID_AT:
        out.append(_item(0, remaining=40, invalid_at=inv))
        out.append(_item(1, rem_bits=fbits(40.5), burst=LIMIT, invalid_at=inv))
    return np.array(out, dtype=ITEM_DTYPE)


def oracle_item(r):
    """r (an ITEM_DTYPE record) as an oracle CacheItem, as gub_add_items installs it; remaining_f is copied bit for bit."""
    it = O.Item()
    leaky = int(r["algorithm"]) == 1
    it.algorithm = int(r["algorithm"]); it.value_kind = 2 if leaky else 1
    it.expire_at = int(r["expire_at"]); it.invalid_at = int(r["invalid_at"])
    it.status = 0 if leaky else int(r["status"]); it.limit = int(r["limit"]); it.duration = int(r["duration"])
    it.remaining_i = 0 if leaky else int(r["remaining"])
    if leaky:
        u = C.c_uint64(int(np.float64(r["remaining_f"]).view(np.uint64)))
        C.memmove(C.addressof(it) + O.Item.remaining_f.offset, C.addressof(u), 8)
    it.stamp = int(r["stamp"]); it.burst = int(r["burst"]) if leaky else 0
    return it


def item_of_oracle(it, kx, kf):
    """An oracle CacheItem as gub_get_items / gub_scan report it (token buckets carry no burst or float Remaining, leaky ones no
    status or int Remaining); remaining_f is copied bit for bit."""
    r = np.zeros(1, dtype=ITEM_DTYPE)
    leaky = it.value_kind == 2
    r["key_xxh64"], r["key_fnv1"] = kx, kf
    r["algorithm"] = 1 if leaky else 0
    r["status"] = 0 if leaky else it.status
    r["limit"], r["duration"], r["stamp"], r["expire_at"], r["invalid_at"] = it.limit, it.duration, it.stamp, it.expire_at, it.invalid_at
    r["remaining"] = 0 if leaky else it.remaining_i
    if leaky:
        r["remaining_f"].view(np.uint64)[0] = oracle_rem_bits(it)
        r["burst"] = it.burst
    return r[0]


def keyed_scan(scan, held):
    """gub_scan records and the oracle's cache (pool.each()) keyed alike: XXH64 as the table remaps it, FNV-1 without its low byte."""
    s = {(int(x["key_xxh64"]), int(x["key_fnv1"])): x for x in scan}
    h = {(x if x >= 2 else x + 2, (f >> 8) << 8): it for (x, f), it in held.items()}
    return s, h


def oracle_rem_bits(it):
    """IEEE-754 bits of an oracle CacheItem's remaining_f, read without a Python float in between."""
    u = C.c_uint64(0)
    C.memmove(C.addressof(u), C.addressof(it) + O.Item.remaining_f.offset, 8)
    return u.value


def buckets(bucket_dtype):
    """The slot images (tests/_host_math.BUCKET_DTYPE) of items() as gub_add_items installs them, opened at NOW: an InvalidAt is
    F_INVALID_AT, and one already past also F_STALE (what the kernels' apply_invalid_at marks when they open the slot)."""
    its = items()
    b = np.zeros(len(its), dtype=bucket_dtype)
    leaky = its["algorithm"] == 1
    inv = its["invalid_at"]
    b["flags"] = 4 | np.where(leaky, 1, 0) | np.where(~leaky & (its["status"] == O.OVER_LIMIT), 2, 0) | np.where(inv != 0, 8, 0) | \
        np.where((inv != 0) & (inv < NOW), 16, 0)
    b["limit"], b["duration"], b["stamp"], b["expire"] = its["limit"], its["duration"], its["stamp"], its["expire_at"]
    b["rem"] = np.where(leaky, its["remaining_f"].view(np.uint64), its["remaining"].view(np.uint64))
    b["burst"] = np.where(leaky, its["burst"], 0)
    return b


def pairs(rng, n, bucket_dtype, req_dtype):
    """n (slot image, request, target rank, index into items()) tuples: a lattice bucket and a request drawn around it (its
    own parameters or edge ones, either algorithm or an invalid one, every behaviour the algorithms branch on, created_at relative
    to the stamp)."""
    bk = buckets(bucket_dtype)
    idx = rng.integers(0, len(bk), n)
    b = bk[idx]
    leaky = (b["flags"] & 1) != 0
    s = b["stamp"].view(np.uint64)
    created = np.stack([np.full(n, NOW, dtype=np.uint64)] + [s + np.uint64(d) for d in (0, RATE, 1000 * RATE, I64_MAX)], axis=1).view(np.int64)
    rq = np.zeros(n, dtype=req_dtype)
    rq["key_xxh64"], rq["key_fnv1"] = np.arange(n, dtype=np.uint64) + np.uint64(1000), (np.arange(n, dtype=np.uint64) << np.uint64(8)) | np.uint64(7)
    u = rng.random(n)
    rq["algorithm"] = np.where(u < 0.8, leaky, np.where(u < 0.95, ~leaky, 3)).astype(np.uint32)
    rq["hits"] = rng.choice(np.array(HITS + [LIMIT - 1, 50, 3], dtype=np.int64), n)
    rq["limit"] = np.where(rng.random(n) < 0.7, b["limit"], rng.choice(np.array(TOKEN_LIMITS, dtype=np.int64), n))
    rq["duration"] = np.where(rng.random(n) < 0.6, b["duration"], rng.choice(np.array([0, 1, 2, 3, 5, 6, DURATION, -DURATION], dtype=np.int64), n))
    rq["burst"] = np.choose(rng.integers(0, 4, n), [np.zeros(n, dtype=np.int64), b["burst"], np.full(n, 7, dtype=np.int64),
                                                     np.full(n, I64_MAX, dtype=np.int64)])
    rq["behavior"] = rng.choice(np.array([0, O.RESET_REMAINING, O.DRAIN_OVER_LIMIT, O.DURATION_IS_GREGORIAN,
                                          O.DURATION_IS_GREGORIAN | O.DRAIN_OVER_LIMIT], dtype=np.uint32), n) | \
        np.where(rng.random(n) < 0.8, O.REQ_IS_OWNER, 0).astype(np.uint32)
    rq["created_at"] = created[np.arange(n), rng.integers(0, created.shape[1], n)]
    targets = rng.choice(np.array([0, 1, 2, 5, 33, 257, 1025], dtype=np.uint32), n)
    return b, rq, targets, idx


def _created(r):
    """created_at values relative to the item's UpdatedAt / CreatedAt: leak 0, 1, many, and an elapsed time that wraps."""
    s = int(r["stamp"])
    return [NOW, s, wrap(s + RATE), wrap(s + 1000 * RATE), wrap(s + I64_MAX)]


def plans(r):
    """Request plans for one loaded item: single requests (answered in k_rank), uniform runs (k_eval's closed forms; the longer
    ones cross k_group's 256-request blocks), runs longer than MIXED_CHUNK whose segments cross the chunk boundary (the k_finish
    fold), a chunk of one-request segments (the serial walk), RESET_REMAINING / DRAIN_OVER_LIMIT / Gregorian durations 0-6, the
    other algorithm, and created_at placed relative to the item's stamp."""
    algo = int(r["algorithm"])
    base = dict(hits=1, limit=int(r["limit"]), duration=int(r["duration"]), burst=int(r["burst"]) if algo == 1 else 0,
                created_at=NOW, algorithm=algo, behavior=O.REQ_IS_OWNER)

    def q(**kw):
        d = dict(base)
        d.update(kw)
        return d

    out = [[q(hits=h)] for h in HITS]
    out += [[q()] * m for m in UNIFORM_RUNS]
    out.append([q(hits=2, behavior=O.REQ_IS_OWNER | O.DRAIN_OVER_LIMIT)] * 33)
    out.append([q(behavior=O.REQ_IS_OWNER | O.RESET_REMAINING)] * 3)
    out.append([q(algorithm=1 - algo)] * 3 + [q()] * 2)
    out.append([q(algorithm=3)])
    out.append([q(limit=LIMIT, duration=DURATION, burst=0)] * 40)
    for d in range(7):
        out.append([q(duration=d, behavior=O.REQ_IS_OWNER | O.DURATION_IS_GREGORIAN)] * 5)
    for c in _created(r):
        out.append([q(created_at=c)])
        out.append([q(created_at=c)] * 33)
    # segments crossing the 1024-member chunk boundary: folded by k_finish
    out.append([q()] * 700 + [q(hits=2)] * 400 + [q(hits=0)] * 300 + [q(created_at=wrap(NOW + 7 * RATE))] * 100)
    # more than MIXED_SEGS one-request segments in a chunk: applied one at a time
    out.append([q(hits=h) for h in np.resize([0, 1, 2], 1100).tolist()])
    return out


def requests(plan, kx, kf, req_dtype):
    out = np.zeros(len(plan), dtype=req_dtype)
    out["key_xxh64"], out["key_fnv1"] = kx, kf
    for f in ("hits", "limit", "duration", "burst", "created_at", "algorithm", "behavior"):
        out[f] = [p[f] for p in plan]
    return out


def lattice(req_dtype, keep=None):
    """(items with their keys, one request array per (item, plan) pair).  keep(item index, plan index, plan) -> bool selects pairs
    (None: all of them); every kept pair has a key of its own, loaded with the item."""
    from workloads import key_hashes
    pairs_, reqs = [], []
    for i, r in enumerate(items()):
        for j, p in enumerate(plans(r)):
            if keep is None or keep(i, j, p):
                pairs_.append((i, p))
    kx, kf = key_hashes(np.arange(len(pairs_)), name="edge")
    its = items()[[i for i, _ in pairs_]]
    its["key_xxh64"], its["key_fnv1"] = kx, kf
    for n, (_, p) in enumerate(pairs_):
        reqs.append(requests(p, kx[n], kf[n], req_dtype))
    return its, reqs
