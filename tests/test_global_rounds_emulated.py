"""The GLOBAL sync tick's rounds on the CPU emulation of the kernels (tests/global_rounds_emu_harness.cpp): the histogram of the drained
hit records over the top 16 bits of XXH64 (k_gq_hist), the rounds every shard derives from all shards' histograms (gq_plan_rounds),
and the counting sort that puts one shard's records in round order (k_gq_partition, gq_round_span), checked against a NumPy
restatement and against the properties the tick relies on: every record travels in exactly one round, no round carries more than
`cap` records of one source, and a key's records from every source travel in the same round unless crafted keys overfill a bin."""
import numpy as np
import pytest

import _global_rounds_emu as G
import oracle_py as O

BINS = 1 << 16


def _recs(keys):
    r = np.zeros(len(keys), dtype=O.HREQ_DTYPE)
    r["key_xxh64"] = np.asarray(keys, dtype=np.uint64)
    r["key_fnv1"] = np.asarray(keys, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    r["hits"] = np.arange(len(keys)) + 1
    return r


def _keys(rng, n):
    """n distinct random nonzero keys (a drained queue holds each key once)."""
    k = np.unique(rng.integers(1, 2**64, size=n + 16, dtype=np.uint64))
    return rng.permutation(k)[:n]


def _bin(keys):
    return (np.asarray(keys, dtype=np.uint64) >> np.uint64(48)).astype(np.int64)


def np_plan(hists, cap):
    """gq_plan_rounds restated: consecutive bins packed while every source stays within cap; an over-full bin split by position."""
    H = np.stack(hists).astype(np.int64)
    most = H.max(axis=0)
    rounds, lo, sums, open_ = [], 0, np.zeros(len(hists), dtype=np.int64), False
    for b in np.nonzero(most)[0]:
        b = int(b)
        if most[b] > cap:
            if open_:
                rounds.append((lo, b, 0))
            rounds += [(b, b + 1, k) for k in range(-(-int(most[b]) // cap))]
            lo, sums[:], open_ = b + 1, 0, False
            continue
        if np.any(sums + H[:, b] > cap):
            if open_:
                rounds.append((lo, b, 0))
            lo, sums[:], open_ = b, 0, False
        sums += H[:, b]
        open_ = True
    if open_:
        rounds.append((lo, BINS, 0))
    return np.array(rounds or [(0, BINS, 0)], dtype=np.int64).reshape(-1, 3)


def _round_of(keys, offs, counts, part):
    """key -> the round whose span of the partitioned array holds it."""
    where = {int(k): i for i, k in enumerate(part["key_xxh64"])}
    starts = np.asarray(offs)
    out = {}
    for k in keys:
        pos = where[int(k)]
        i = int(np.searchsorted(starts + np.asarray(counts), pos, side="right"))
        assert starts[i] <= pos < starts[i] + counts[i]
        out[int(k)] = i
    return out


def _check_rounds(rounds):
    """Rounds cover increasing, non-overlapping bin ranges; the slices of a split bin are consecutive and start at 0."""
    for (lo, hi, sl), (lo2, hi2, sl2) in zip(rounds[:-1], rounds[1:]):
        if (lo2, hi2) == (lo, hi):
            assert hi == lo + 1 and sl2 == sl + 1
        else:
            assert hi <= lo2 and sl2 == 0
    assert rounds[0][2] == 0


def test_bins_is_top_16_bits():
    assert G.bins() == BINS


@pytest.mark.parametrize("n", [0, 1, 777, 20000])
def test_hist_matches_numpy(n):
    rng = np.random.default_rng(n)
    keys = _keys(rng, n)
    assert np.array_equal(G.hist(_recs(keys)), np.bincount(_bin(keys), minlength=BINS).astype(np.uint32))


@pytest.mark.parametrize("world,cap,sizes", [
    (1, 4096, [3000]),                   # everything fits: one round, as the single-round tick
    (1, 4096, [0]),                      # empty window: one empty round
    (1, 4096, [3 * 4096]),
    (2, 4096, [4 * 4096, 100]),
    (4, 512, [2048, 0, 512, 1500]),
    (8, 64, [640, 64, 0, 1, 300, 1000, 64, 65]),
])
def test_plan_matches_numpy(world, cap, sizes):
    rng = np.random.default_rng(world * 1000 + cap)
    hists = [G.hist(_recs(_keys(rng, n))) for n in sizes]
    got = G.plan(hists, cap)
    assert np.array_equal(got, np_plan(hists, cap))
    _check_rounds(got.tolist())
    if max(sizes) <= cap:
        assert len(got) == 1
    else:
        # every source's records fit in the rounds, and the packing leaves little room unused
        assert len(got) >= -(-max(sizes) // cap)
        assert len(got) <= 2 * -(-max(sizes) // cap) + 2


def _shards(rng, world, sizes, shared):
    """Per source: `sizes[s]` distinct keys, drawn from one pool of `shared` keys (so sources share many keys) plus keys of their own."""
    pool = _keys(rng, shared)
    out = []
    for n in sizes:
        k = np.unique(np.concatenate([rng.choice(pool, size=min(n // 2, shared), replace=False), _keys(rng, n)]))
        out.append(rng.permutation(k)[:n])
    return out


def _run(keys_per_source, cap):
    recs = [_recs(k) for k in keys_per_source]
    hists = [G.hist(r) for r in recs]
    rounds = G.plan(hists, cap)
    parts = [G.partition(r, h, cap, rounds) for r, h in zip(recs, hists)]
    return recs, rounds, parts


def _check_cover(recs, rounds, parts, cap):
    for r, (part, offs, counts) in zip(recs, parts):
        # every record exactly once, in the round order: spans are contiguous and cover the array
        assert sorted(part["key_xxh64"].tolist()) == sorted(r["key_xxh64"].tolist())
        assert np.array_equal(np.sort(part, order="key_xxh64"), np.sort(r, order="key_xxh64"))
        assert int(counts.sum()) == len(r)
        assert np.array_equal(offs, np.concatenate([[0], np.cumsum(counts)[:-1]]))
        assert counts.max() <= cap
        for (lo, hi, _), o, c in zip(rounds, offs, counts):
            b = _bin(part["key_xxh64"][o:o + c])
            assert np.all((b >= lo) & (b < hi))


@pytest.mark.parametrize("world,cap,scale", [(1, 4096, 3), (2, 1024, 4), (4, 512, 2.5), (8, 256, 1)])
def test_partition_and_key_consistency(world, cap, scale):
    rng = np.random.default_rng(world + cap)
    sizes = [int(scale * cap) if s % 3 != 2 else int(0.3 * cap) for s in range(world)]
    keys = _shards(rng, world, sizes, shared=2 * cap)
    recs, rounds, parts = _run(keys, cap)
    _check_cover(recs, rounds, parts, cap)
    assert not np.any(rounds[:, 2])  # random keys never overfill a bin
    maps = [_round_of(k, offs, counts, part) for k, (part, offs, counts) in zip(keys, parts)]
    seen = {}
    shared = 0
    for m in maps:
        for k, i in m.items():
            if k in seen:
                assert seen[k] == i, "a key's records from two sources travel in different rounds"
                shared += 1
            seen[k] = i
    assert shared > 0 or world == 1


def test_overfull_bin_is_split_and_nothing_dropped():
    """Keys crafted to share their top 16 bits: the bin takes ceil(most / cap) rounds, split by position; no record is lost."""
    rng = np.random.default_rng(9)
    cap = 512
    top = np.uint64(0xABCD) << np.uint64(48)
    crafted = np.unique(rng.integers(1, 2**48, size=3000, dtype=np.uint64)) | top
    keys = [np.concatenate([crafted[:int(2.5 * cap)], _keys(rng, 3 * cap)]),
            np.concatenate([crafted[:int(1.2 * cap)], _keys(rng, 700)]),
            _keys(rng, 100)]
    keys = [rng.permutation(np.unique(k)) for k in keys]
    recs, rounds, parts = _run(keys, cap)
    assert np.array_equal(rounds, np_plan([G.hist(r) for r in recs], cap))
    split = rounds[(rounds[:, 0] == 0xABCD) & (rounds[:, 1] == 0xABCD + 1)]
    assert split[:, 2].tolist() == [0, 1, 2]
    _check_cover(recs, rounds, parts, cap)
    # the crafted bin's rounds carry exactly its records: source 0 fills cap, cap, the rest; source 1 cap, the rest, nothing
    idx = np.nonzero((rounds[:, 0] == 0xABCD) & (rounds[:, 1] == 0xABCD + 1))[0]
    assert parts[0][2][idx].tolist() == [cap, cap, int(2.5 * cap) - 2 * cap]
    assert parts[1][2][idx].tolist() == [cap, int(1.2 * cap) - cap, 0]
    assert parts[2][2][idx].tolist() == [0, 0, 0]
    # keys outside the crafted bin stay key-consistent
    maps = [_round_of(k, offs, counts, part) for k, (part, offs, counts) in zip(keys, parts)]
    normal = set(maps[0]) & set(maps[1]) - set(int(k) for k in crafted)
    assert all(maps[0][k] == maps[1][k] for k in normal)
