"""What a Store plugin costs on the key-string path: µs per 65 536-request batch for
  (a) gub_submit_keys_async                                  (no Store),
  (b) gub_submit_keys_store_async with get = NULL            (a write-behind store: the pre- and post-pass, the change log over PCIe),
  (c) gub_submit_keys_store_async with a Get that finds nothing (adds the miss list, its host synchronisation and the callback),
on bench.py's end-to-end traffic: Zipf 1.1 over --keys resident keys, 16-byte keys "bench_k%09d", TOKEN / LEAKY by id parity, depth-4
pipelining from pinned host memory.  The arms run in alternating blocks; each block is timed on the host clock and ends in a device
synchronise.  Prints one JSON line (with the card's name and power limit, read in the same run) and a markdown table.

  python scripts/store_bench.py [--keys 1000000] [--steps 200] [--rounds 5] [--pool 8]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

BATCH = 65536
DEPTH = 4


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", type=int, default=1_000_000, help="resident keys")
    ap.add_argument("--steps", type=int, default=200, help="batches per block")
    ap.add_argument("--rounds", type=int, default=5, help="blocks per arm, alternating")
    ap.add_argument("--pool", type=int, default=8, help="distinct pre-generated batches cycled through")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("store_bench.py needs a CUDA device")
    import gubernator_b200 as g
    import oracle_py as O
    from workloads import T0, bench_key_bytes, bench_requests, zipf_ids
    native = g.native
    C = native.C

    rng = np.random.default_rng(1)
    tab = g.Table(max(1 << 20, 1 << int(np.ceil(np.log2(2 * a.keys)))))
    for lo in range(0, a.keys, BATCH):  # every key resident before timing
        ids = np.arange(lo, min(a.keys, lo + BATCH), dtype=np.int64)
        tab.submit(bench_requests(ids, T0, dtype=g.REQ_DTYPE), native.clock_fill(T0))

    params = np.zeros(2, dtype=native.PARAMS_DTYPE)
    params["limit"] = 100; params["duration"] = 60000; params["algorithm"] = [0, 1]; params["behavior"] = O.REQ_IS_OWNER
    ppin = native.PinnedArray(2, native.PARAMS_DTYPE); ppin.array[:] = params
    packed = []
    for k in range(a.pool):
        ids = zipf_ids(rng, BATCH, a.keys, 1.1)
        keys_u8 = np.ascontiguousarray(bench_key_bytes(ids)).reshape(-1)
        o_at, b_at, tot = C.c_size_t(), C.c_size_t(), C.c_size_t()
        native.lib().gub_keys_layout(BATCH, len(keys_u8), C.byref(o_at), C.byref(b_at), C.byref(tot))
        pin = native.PinnedArray(tot.value, np.uint8)
        kr = pin.array[:BATCH * 16].view(native.KREQ_DTYPE)
        kr["hits"] = 1; kr["params"] = (ids & 1).astype(np.uint32); kr["created_delta"] = 0
        pin.array[o_at.value:o_at.value + 4 * (BATCH + 1)].view(np.uint32)[:] = np.arange(BATCH + 1, dtype=np.uint32) * 16
        pin.array[b_at.value:b_at.value + len(keys_u8)] = keys_u8
        packed.append((pin, tot.value))
    outs = [native.PinnedArray(BATCH, g.RESP_DTYPE) for _ in range(DEPTH)]
    chs = [native.PinnedArray(BATCH, native.STORE_REC_DTYPE) for _ in range(DEPTH)]
    ncs = [native.PinnedArray(1, np.uint32) for _ in range(DEPTH)]
    clocks = [native.clock_fill(T0 + 1 + s) for s in range(64)]

    def finds_nothing(misses):
        return 0

    arms = {
        "a_keys_async": lambda pb, k, b: tab.submit_keys_async(packed[pb][0].ptr, packed[pb][1], BATCH, ppin.ptr, 2, T0, clocks[b % 64], outs[k].ptr),
        "b_store_get_null": lambda pb, k, b: tab.submit_keys_store_async(packed[pb][0].ptr, packed[pb][1], BATCH, ppin.ptr, 2, T0, clocks[b % 64], None,
                                                                       outs[k].ptr, chs[k].ptr, ncs[k].ptr),
        "c_store_get_finds_nothing": lambda pb, k, b: tab.submit_keys_store_async(packed[pb][0].ptr, packed[pb][1], BATCH, ppin.ptr, 2, T0, clocks[b % 64],
                                                                                finds_nothing, outs[k].ptr, chs[k].ptr, ncs[k].ptr),
    }
    step = [0]
    stats = {name: {"us": [], "records": []} for name in arms}

    def block(name, steps):
        submit = arms[name]
        tickets = [None] * DEPTH
        recs = 0
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for s in range(steps):
            k = s % DEPTH
            if tickets[k] is not None:
                tab.wait(tickets[k])
                recs += int(ncs[k].array[0]) if name != "a_keys_async" else 0
            tickets[k] = submit(step[0] % a.pool, k, step[0])
            step[0] += 1
        for k in range(DEPTH):
            if tickets[k] is not None:
                tab.wait(tickets[k])
                recs += int(ncs[k].array[0]) if name != "a_keys_async" else 0
        torch.cuda.synchronize()
        return 1e6 * (time.perf_counter() - t0) / steps, recs / steps

    for name in arms:  # warm-up: first launches, scratch allocation
        block(name, 16)
    for r in range(a.rounds):
        for name in arms:
            us, rec = block(name, a.steps)
            stats[name]["us"].append(us); stats[name]["records"].append(rec)

    res = {"card": card(), "keys": a.keys, "batch": BATCH, "depth": DEPTH, "steps_per_block": a.steps, "rounds": a.rounds,
           "record_bytes": native.STORE_REC_DTYPE.itemsize, "arms": {}}
    for name, st in stats.items():
        res["arms"][name] = {"us_per_batch_median": float(np.median(st["us"])), "us_per_batch_min": float(np.min(st["us"])),
                             "us_per_batch_max": float(np.max(st["us"])), "records_per_batch": float(np.mean(st["records"])),
                             "record_bytes_per_batch": float(np.mean(st["records"])) * native.STORE_REC_DTYPE.itemsize}
    print(json.dumps(res))
    print(f"\n{res['card']}; {a.keys} resident keys, {BATCH}-request batches, depth {DEPTH}, {a.rounds} alternating blocks of {a.steps} batches\n")
    print("| arm | µs per batch (median, min–max) | records per batch | record bytes per batch |")
    print("|---|---|---|---|")
    for name, v in res["arms"].items():
        print(f"| {name} | {v['us_per_batch_median']:.1f} ({v['us_per_batch_min']:.1f}–{v['us_per_batch_max']:.1f}) | {v['records_per_batch']:.0f} | "
              f"{v['record_bytes_per_batch'] / 1e6:.2f} MB |")


if __name__ == "__main__":
    main()
