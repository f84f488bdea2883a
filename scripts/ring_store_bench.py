"""Ring steps with and without a Store plugin, W in {1, 2, 4} shards in one process on ONE GPU (device 0).  ring_keys_bench.py's traffic:
Zipf 1.1 over `--keys` ids, 16-byte bench_k%09d keys, 65 536 requests per shard per step.  Three arms, alternated in blocks within one
run, each on its own ring fed the same step sequence:
  (a) plain: gub_p2p_step_keys_local_all;
  (b) store, get = NULL: gub_p2p_step_keys_store_local_all with a write-behind store (no miss list, change logs only);
  (c) store, empty get: the same with a Get callback that finds nothing (every owner's miss list is compacted, handed to the
      callback, and the call blocks until every routing is done).
Host clock around every block of steps, ending in a synchronise of the device.  Reports microseconds per step and change-log records
per step (all owners).  The last step's responses must be byte-identical across the arms.  Prints one JSON line per world size and a
header line with the GPU name and power limit."""
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

N = 65536


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return [line.strip() for line in out.strip().splitlines()]
    except Exception as e:  # the timing itself does not depend on it
        return [f"nvidia-smi unavailable: {e}"]


def run_world(W, args):
    import torch
    import gubernator_b200 as g
    from local_ring import LocalRing
    from workloads import T0, bench_key_bytes, zipf_ids

    rings = {arm: LocalRing(W, capacity=args.capacity, cap=N, spread_devices=False) for arm in "abc"}
    dev = torch.device("cuda", 0)
    table = np.zeros(2, dtype=g.native.PARAMS_DTYPE)
    table["limit"] = 100; table["duration"] = 60000; table["algorithm"] = [0, 1]; table["behavior"] = g.native.REQ_IS_OWNER
    rng = np.random.default_rng(2024 + W)
    batches = []  # [k][r]: packed key batches on the device (host generation stays out of the timed loop)
    for k in range(args.distinct):
        per = []
        for r in range(W):
            ids = zipf_ids(rng, N, args.keys, 1.1)
            packed = g.native.pack_keys([bytes(x) for x in bench_key_bytes(ids)], 1, (ids & 1).astype(np.uint32), 0)
            per.append((torch.from_numpy(packed).to(dev), len(packed)))
        batches.append(per)
    outs = {arm: [torch.zeros((N, 32), dtype=torch.uint8, device=dev) for _ in range(W)] for arm in "abc"}
    changes = {arm: [g.native.PinnedArray(W * N, g.native.STORE_REC_DTYPE) for _ in range(W)] for arm in "bc"}
    n_changes = {arm: [g.native.PinnedArray(1, np.uint32) for _ in range(W)] for arm in "bc"}
    records = {arm: 0 for arm in "bc"}
    ns = [N] * W

    def empty_get(misses):
        return 0

    def step(arm, k, now):
        lr, b = rings[arm], batches[k % args.distinct]
        clk = g.clock_fill(now)
        streams = [s.cuda_stream for s in lr.streams]
        o = [x.data_ptr() for x in outs[arm]]
        ptrs, sizes = [x[0].data_ptr() for x in b], [x[1] for x in b]
        if arm == "a":
            g.native.p2p_step_keys_local_all(lr.p2ps, ptrs, sizes, ns, table, T0, clk, o, streams)
        else:
            g.native.p2p_step_keys_store_local_all(lr.p2ps, ptrs, sizes, ns, table, T0, clk, None if arm == "b" else empty_get, o,
                                                   [c.ptr for c in changes[arm]], [c.ptr for c in n_changes[arm]], streams)

    def sync():
        torch.cuda.synchronize(dev)

    now = T0
    for _ in range(args.warmup):
        for arm in "abc":
            step(arm, 0, now)
        now += 1
    sync()
    spent = {arm: 0.0 for arm in "abc"}
    done = 0
    k = 1
    while done < args.steps:
        blk = min(args.block, args.steps - done)
        for arm in "abc":
            t0 = time.perf_counter()
            for j in range(blk):
                step(arm, k + j, now + j)
            sync()
            spent[arm] += time.perf_counter() - t0
            if arm != "a":  # the change logs of the block's last step
                records[arm] += sum(int(c.array[0]) for c in n_changes[arm])
        k += blk; now += blk; done += blk
    for lr in rings.values():
        lr.sync()
    last = {arm: [outs[arm][r].cpu().numpy().tobytes() for r in range(W)] for arm in "abc"}
    same = last["a"] == last["b"] == last["c"]
    blocks = (args.steps + args.block - 1) // args.block
    res = {"world": W, "requests_per_shard_step": N, "steps": args.steps, "identical_last_responses": same}
    for arm, name in (("a", "plain"), ("b", "store_no_get"), ("c", "store_empty_get")):
        us = spent[arm] / args.steps * 1e6
        res[name] = {"us_per_step": round(us, 1), "decisions_per_s": round(W * N / (us * 1e-6))}
        if arm != "a":
            res[name]["records_per_step"] = round(records[arm] / blocks)
    for lr in rings.values():
        for p in lr.p2ps:
            p.close()
        for t in lr.tabs:
            t.close()
    return res, same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", default="1,2,4")
    ap.add_argument("--steps", type=int, default=500)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--block", type=int, default=50, help="steps per arm before switching to the next arm")
    ap.add_argument("--distinct", type=int, default=4, help="pre-generated batches per shard, cycled")
    ap.add_argument("--keys", type=int, default=10_000_000)
    ap.add_argument("--capacity", type=int, default=1 << 20, help="table slots per shard")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("ring_store_bench: no GPU")
    print(json.dumps({"gpu": gpu_info(), "cuda_devices": torch.cuda.device_count()}), flush=True)
    ok = True
    for W in [int(w) for w in args.worlds.split(",")]:
        res, same = run_world(W, args)
        print(json.dumps(res), flush=True)
        ok &= same
    if not ok:
        sys.exit("ring_store_bench: the arms' last responses differ")


if __name__ == "__main__":
    main()
