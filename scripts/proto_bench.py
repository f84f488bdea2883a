"""What decoding and encoding the protobuf wire format on the device costs: µs per 65 536-item call for
  (a) gub_submit_keys_async      packed key strings + 16-byte request records in, 32-byte gub_resp records out (bench.py's e2e leg),
  (b) gub_submit_proto_async     GetRateLimitsReq wire bytes in, GetRateLimitsResp wire bytes out, RPCs of 1000 items,
  (c) the same                   RPCs of 100 items,
on bench.py's end-to-end traffic: Zipf 1.1 over --keys resident keys, keys "bench_k%09d" (Name "bench", UniqueKey "k%09d"), hits 1,
limit 100, duration 60 000, TOKEN / LEAKY by id parity; depth-4 pipelining from pinned host memory.  The arms run in alternating blocks;
each block is timed on the host clock and ends in a device synchronise.  The host-side packing is done before timing (the wire bytes
stand for what a gRPC server hands over).  Prints one JSON line (with the card's name and power limit, read in the same run) and a
markdown table.

  python scripts/proto_bench.py [--keys 1000000] [--steps 200] [--rounds 5] [--pool 8]
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


def wire_item(i):
    """RateLimitReq{name "bench", unique_key "k%09d", hits 1, limit 100, duration 60000, algorithm i & 1} as proto.Marshal writes it."""
    return (b"\x0a\x05bench\x12\x0ak%09d\x18\x01\x20\x64\x28\xe0\xd4\x03" % i) + (b"\x30\x01" if i & 1 else b"")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keys", type=int, default=1_000_000, help="resident keys")
    ap.add_argument("--steps", type=int, default=200, help="calls per block")
    ap.add_argument("--rounds", type=int, default=5, help="blocks per arm, alternating")
    ap.add_argument("--pool", type=int, default=8, help="distinct pre-generated calls cycled through")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("proto_bench.py needs a CUDA device")
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
    keys_in, proto_in = [], {1000: [], 100: []}
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
        keys_in.append((pin, tot.value))
        items = [b"\x0a" + bytes([len(w)]) + w for w in map(wire_item, ids.tolist())]
        for per in proto_in:
            msgs = [b"".join(items[lo:lo + per]) for lo in range(0, BATCH, per)]
            buf, bound = native.pack_proto(msgs, T0)
            pp = native.PinnedArray(len(buf), np.uint8)
            pp.array[:] = buf
            proto_in[per].append((pp, len(buf), len(msgs), bound))
    bound = max(p[3] for v in proto_in.values() for p in v)
    n_max = max(p[2] for v in proto_in.values() for p in v)
    outs = [native.PinnedArray(BATCH, g.RESP_DTYPE) for _ in range(DEPTH)]
    pouts = [native.PinnedArray(bound, np.uint8) for _ in range(DEPTH)]
    poffs = [native.PinnedArray(n_max + 1, np.uint64) for _ in range(DEPTH)]
    psts = [native.PinnedArray(n_max, np.uint32) for _ in range(DEPTH)]
    clocks = [native.clock_fill(T0 + 1 + s) for s in range(64)]

    def proto_arm(per):
        def submit(pb, k, b):
            pp, nbytes, n, bd = proto_in[per][pb]
            return tab.submit_proto_async(pp.ptr, nbytes, n, clocks[b % 64], pouts[k].ptr, bound, poffs[k].ptr, psts[k].ptr)
        return submit

    arms = {
        "a_keys_async": lambda pb, k, b: tab.submit_keys_async(keys_in[pb][0].ptr, keys_in[pb][1], BATCH, ppin.ptr, 2, T0, clocks[b % 64],
                                                               outs[k].ptr),
        "b_proto_rpc1000": proto_arm(1000),
        "c_proto_rpc100": proto_arm(100),
    }
    step = [0]
    stats = {name: {"us": [], "d2h": []} for name in arms}

    def d2h(name, k, pb):
        if name == "a_keys_async":
            return BATCH * g.RESP_DTYPE.itemsize
        n = proto_in[1000 if "1000" in name else 100][pb][2]
        assert (psts[k].array[:n] == native.PROTO_OK).all()
        return int(poffs[k].array[n]) + 12 * n  # response bytes + one uint64 offset and one uint32 status per RPC

    def block(name, steps):
        submit = arms[name]
        tickets, pbs = [None] * DEPTH, [0] * DEPTH
        out_bytes = 0
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for s in range(steps):
            k = s % DEPTH
            if tickets[k] is not None:
                tab.wait(tickets[k])
                out_bytes += d2h(name, k, pbs[k])
            pbs[k] = step[0] % a.pool
            tickets[k] = submit(pbs[k], k, step[0])
            step[0] += 1
        for k in range(DEPTH):
            if tickets[k] is not None:
                tab.wait(tickets[k])
                out_bytes += d2h(name, k, pbs[k])
        torch.cuda.synchronize()
        return 1e6 * (time.perf_counter() - t0) / steps, out_bytes / steps

    for name in arms:  # warm-up: first launches, scratch allocation
        block(name, 16)
    for r in range(a.rounds):
        for name in arms:
            us, ob = block(name, a.steps)
            stats[name]["us"].append(us); stats[name]["d2h"].append(ob)

    h2d = {"a_keys_async": np.mean([p[1] for p in keys_in]), "b_proto_rpc1000": np.mean([p[1] for p in proto_in[1000]]),
           "c_proto_rpc100": np.mean([p[1] for p in proto_in[100]])}
    res = {"card": card(), "keys": a.keys, "items_per_call": BATCH, "depth": DEPTH, "steps_per_block": a.steps, "rounds": a.rounds,
           "timer": "host clock per block of calls, ending in a device synchronise", "arms": {}}
    for name, st in stats.items():
        us = float(np.median(st["us"]))
        res["arms"][name] = {"us_per_call_median": us, "us_per_call_min": float(np.min(st["us"])), "us_per_call_max": float(np.max(st["us"])),
                             "decisions_per_s": BATCH / us * 1e6, "h2d_bytes_per_item": float(h2d[name]) / BATCH,
                             "d2h_bytes_per_item": float(np.mean(st["d2h"])) / BATCH}
    print(json.dumps(res))
    print(f"\n{res['card']}; {a.keys} resident keys, {BATCH}-item calls, depth {DEPTH}, {a.rounds} alternating blocks of {a.steps} calls\n")
    print("| arm | µs per call (median, min–max) | decisions/s | H2D B/item | D2H B/item |")
    print("|---|---|---|---|---|")
    for name, v in res["arms"].items():
        print(f"| {name} | {v['us_per_call_median']:.1f} ({v['us_per_call_min']:.1f}–{v['us_per_call_max']:.1f}) | "
              f"{v['decisions_per_s'] / 1e9:.3f} G | {v['h2d_bytes_per_item']:.1f} | {v['d2h_bytes_per_item']:.1f} |")


if __name__ == "__main__":
    main()
