"""Ring steps fed with key strings vs records, W in {1, 2, 4, 8} shards in one process (all on device 0 with one GPU, one per device
otherwise).  Bench-like traffic: Zipf 1.1 over `--keys` ids, 16-byte bench_k%09d keys, 65 536 requests per shard per step.  Three
arms, alternated in blocks within one run, each on its own ring fed the same step sequence:
  (a) records: 64-byte pre-hashed records in HBM + gub_p2p_step_local_all;
  (b) keys:    packed key strings in HBM + gub_p2p_step_keys_local_all (k_p2p_route_keys: hash, expand and route in one kernel);
  (c) two-kernel: gub_hash_keys_device writes the hashes into records that already hold the rest (hits, parameters, created_at),
      then gub_p2p_step_local_all.
Host clock around every block of steps, ending in a synchronise of every device.  The last step's responses must be byte-identical
across the arms.  Prints one JSON line per world size and a header line with the GPU name and power limit."""
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
    from workloads import T0, bench_key_bytes, bench_key_hashes, zipf_ids

    ndev = torch.cuda.device_count()
    rings = {arm: LocalRing(W, capacity=args.capacity, cap=N, spread_devices=ndev > 1) for arm in "abc"}
    devs = rings["a"].devs
    table = np.zeros(2, dtype=g.native.PARAMS_DTYPE)
    table["limit"] = 100; table["duration"] = 60000; table["algorithm"] = [0, 1]; table["behavior"] = g.native.REQ_IS_OWNER
    rng = np.random.default_rng(2024 + W)
    # args.distinct pre-generated batches per shard, cycled (host generation stays out of the timed loop)
    batches = []  # [k][r] = dict of device tensors
    for k in range(args.distinct):
        per = []
        for r in range(W):
            dev = torch.device("cuda", devs[r])
            ids = zipf_ids(rng, N, args.keys, 1.1)
            kb = bench_key_bytes(ids)                                     # [N, 16]
            xx, fv = bench_key_hashes(ids)
            rec = np.zeros(N, dtype=g.REQ_DTYPE)
            rec["hits"] = 1; rec["limit"] = 100; rec["duration"] = 60000; rec["created_at"] = T0
            rec["algorithm"] = ids & 1; rec["behavior"] = g.native.REQ_IS_OWNER
            tmpl = rec.copy()                                             # (c): everything but the hashes
            rec["key_xxh64"], rec["key_fnv1"] = xx, fv
            packed = g.native.pack_keys([bytes(x) for x in kb], 1, (ids & 1).astype(np.uint32), 0)
            offs64 = np.arange(N + 1, dtype=np.uint64) * 16
            per.append(dict(
                rec=torch.from_numpy(rec.view(np.uint8).reshape(N, 64).copy()).to(dev),
                packed=torch.from_numpy(packed).to(dev), packed_bytes=len(packed),
                crec=torch.from_numpy(tmpl.view(np.uint8).reshape(N, 64).copy()).to(dev),
                kbytes=torch.from_numpy(np.ascontiguousarray(kb).reshape(-1)).to(dev),
                offs=torch.from_numpy(offs64).to(dev)))
        batches.append(per)
    outs = {arm: [torch.zeros((N, 32), dtype=torch.uint8, device=torch.device("cuda", devs[r])) for r in range(W)] for arm in "abc"}
    ns = [N] * W

    def step(arm, k, now):
        lr, b = rings[arm], batches[k % args.distinct]
        clk = g.clock_fill(now)
        streams = [s.cuda_stream for s in lr.streams]
        o = [x.data_ptr() for x in outs[arm]]
        if arm == "a":
            g.native.p2p_step_local_all(lr.p2ps, [x["rec"].data_ptr() for x in b], ns, clk, o, streams)
        elif arm == "b":
            g.native.p2p_step_keys_local_all(lr.p2ps, [x["packed"].data_ptr() for x in b], [x["packed_bytes"] for x in b], ns, table, T0, clk, o, streams)
        else:
            for r in range(W):  # the records hold everything but the hashes (the routing only reads them)
                x = b[r]
                lr.tabs[r].hash_keys_device(x["kbytes"].data_ptr(), x["offs"].data_ptr(), N, None, None, x["crec"].data_ptr(), streams[r])
            g.native.p2p_step_local_all(lr.p2ps, [x["crec"].data_ptr() for x in b], ns, clk, o, streams)

    def sync():
        for d in set(devs):
            torch.cuda.synchronize(d)

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
        k += blk; now += blk; done += blk
    for lr in rings.values():
        lr.sync()
    last = {arm: [outs[arm][r].cpu().numpy().tobytes() for r in range(W)] for arm in "abc"}
    same = last["a"] == last["b"] == last["c"]
    res = {"world": W, "devices": sorted(set(devs)), "requests_per_shard_step": N, "steps": args.steps, "identical_last_responses": same}
    for arm, name in (("a", "records"), ("b", "keys_fused"), ("c", "hash_then_records")):
        us = spent[arm] / args.steps * 1e6
        res[name] = {"us_per_step": round(us, 1), "decisions_per_s": round(W * N / (us * 1e-6))}
    res["keys_fused_vs_two_kernel"] = round(res["hash_then_records"]["us_per_step"] / res["keys_fused"]["us_per_step"], 3)
    for lr in rings.values():
        for p in lr.p2ps:
            p.close()
        for t in lr.tabs:
            t.close()
    return res, same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", default="1,2,4,8")
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--block", type=int, default=50, help="steps per arm before switching to the next arm")
    ap.add_argument("--distinct", type=int, default=4, help="pre-generated batches per shard, cycled")
    ap.add_argument("--keys", type=int, default=10_000_000)
    ap.add_argument("--capacity", type=int, default=1 << 20, help="table slots per shard")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("ring_keys_bench: no GPU")
    print(json.dumps({"gpu": gpu_info(), "cuda_devices": torch.cuda.device_count()}), flush=True)
    ok = True
    for W in [int(w) for w in args.worlds.split(",")]:
        res, same = run_world(W, args)
        print(json.dumps(res), flush=True)
        ok &= same
    if not ok:
        sys.exit("ring_keys_bench: the arms' last responses differ")


if __name__ == "__main__":
    main()
