"""Time of one GLOBAL sync tick (gub_global_tick_local_all) against the number of distinct GLOBAL keys in the window.  W in {1, 2, 4}
shards on device 0, and one shard per device when there are several; a window of 1/2, 1, 2 and 4 x cap distinct GLOBAL keys per shard
(the same ids on every shard, so every owner gets the hits of W - 1 sources; the ring's mailbox capacity cap = 65 536, the queues'
capacity 1 << 18).  The window is filled by untimed steps; the tick is timed with a host clock around the call, which ends in a
synchronise of every shard's stream.  Configurations are alternated within one run, `--reps` times each.  Prints a header line with
the GPU name and power limit, then one JSON line per configuration."""
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

CAP, GCAP = 65536, 1 << 18


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return [line.strip() for line in out.strip().splitlines()]
    except Exception as e:  # the timing itself does not depend on it
        return [f"nvidia-smi unavailable: {e}"]


def window(lr, ids, now):
    """Steps of at most CAP requests per shard until every shard has sent every id once (GLOBAL, token bucket, Hits = 1)."""
    import oracle_py as O
    from workloads import key_hashes
    for lo in range(0, len(ids), CAP):
        part = ids[lo:lo + CAP]
        b = np.zeros(len(part), dtype=O.HREQ_DTYPE)
        b["key_xxh64"], b["key_fnv1"] = key_hashes(part, name="tick")
        b["hits"] = 1; b["limit"] = 1 << 30; b["duration"] = 3600000; b["created_at"] = now
        b["behavior"] = np.uint32(O.GLOBAL | O.REQ_IS_OWNER)
        lr.step([b] * lr.W, now)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--worlds", default="1,2,4")
    ap.add_argument("--mults", default="0.5,1,2,4")
    args = ap.parse_args()
    import torch
    from local_ring import LocalRing
    from workloads import T0
    print(json.dumps({"gpus": gpu_info(), "device_count": torch.cuda.device_count()}), flush=True)
    shapes = [(int(w), False) for w in args.worlds.split(",")]
    if torch.cuda.device_count() > 1:
        shapes += [(w, True) for w in (2, 4) if w <= torch.cuda.device_count()]
    rings = {s: LocalRing(s[0], capacity=1 << 21, cap=CAP, global_capacity=GCAP, spread_devices=s[1]) for s in shapes}
    mults = [float(m) for m in args.mults.split(",")]
    times = {(s, m): [] for s in shapes for m in mults}
    sent = {}
    now = T0
    for rep in range(args.reps + 1):  # the first pass warms up and is not recorded
        for s in shapes:
            for m in mults:
                lr = rings[s]
                window(lr, np.arange(1, int(m * CAP) + 1), now)
                t0 = time.perf_counter()
                lr.tick(now)
                dt = time.perf_counter() - t0
                if rep:
                    times[(s, m)].append(dt * 1e3)
                sent[(s, m)] = max(x["hits_sent"] for x in lr.last_tick)
                assert all(t.counters()["gq_dropped"] == 0 for t in lr.tabs)
                now += 1
    for s in shapes:
        for m in mults:
            t = np.array(times[(s, m)])
            print(json.dumps({"world": s[0], "devices": "one per shard" if s[1] else "one", "keys_per_shard": int(m * CAP), "cap": CAP,
                              "hits_sent_max": sent[(s, m)], "min_rounds": max(1, -(-sent[(s, m)] // CAP)),
                              "tick_ms_median": round(float(np.median(t)), 3), "tick_ms_min": round(float(t.min()), 3),
                              "tick_ms_max": round(float(t.max()), 3), "reps": len(t)}), flush=True)


if __name__ == "__main__":
    main()
