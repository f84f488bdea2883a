"""GetRateLimits wire bytes on the ring vs key strings on the ring, W in {1, 2, 4} shards in one process on ONE device, 65 536 items per
shard per step (cap = 65 536).  Traffic of scripts/proto_bench.py: Zipf 1.1 over --keys ids, keys "bench_k%09d" (Name "bench", UniqueKey
"k%09d"), hits 1, limit 100, duration 60 000, TOKEN / LEAKY by id parity.  Three arms, each on its own ring fed the same step sequence
(same items in the same order, same clocks), alternated in blocks within one run:
  (a) keys:      packed key strings in HBM + gub_p2p_step_keys_local_all, 32-byte gub_resp records out (device memory);
  (b) rpc100:    gub_p2p_step_proto_local_all, each shard's items as GetRateLimitsReq messages of 100 items in page-locked host memory,
                 GetRateLimitsResp bytes out into page-locked host memory;
  (c) rpc1000:   the same with messages of 1000 items.
The wire arms alternate two output sets by call parity (a call returns once the call two back is encoded).  Host clock around every
block of calls, ending in a synchronise of the device.  After timing, the last step's responses of (a), encoded as proto.Marshal writes
them, must equal the bytes of (b) and (c).  Prints a header line with the GPU name and power limit, then one JSON line per world size.

  python scripts/ring_proto_bench.py [--worlds 1,2,4] [--steps 200] [--block 20] [--keys 1000000]
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

N = 65536
ARMS = ("keys", "rpc100", "rpc1000")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout
        return [line.strip() for line in out.strip().splitlines()]
    except Exception as e:  # the timing itself does not depend on it
        return [f"nvidia-smi unavailable: {e}"]


def wire_item(i):
    """RateLimitReq{name "bench", unique_key "k%09d", hits 1, limit 100, duration 60000, algorithm i & 1} as proto.Marshal writes it."""
    return (b"\x0a\x05bench\x12\x0ak%09d\x18\x01\x20\x64\x28\xe0\xd4\x03" % i) + (b"\x30\x01" if i & 1 else b"")


def run_world(W, args):
    import torch
    import gubernator_b200 as g
    import _proto_wire as PW
    from local_ring import LocalRing
    from workloads import T0, bench_key_bytes, zipf_ids
    native = g.native

    rings = {arm: LocalRing(W, capacity=args.capacity, cap=N) for arm in ARMS}
    table = np.zeros(2, dtype=native.PARAMS_DTYPE)
    table["limit"] = 100; table["duration"] = 60000; table["algorithm"] = [0, 1]; table["behavior"] = native.REQ_IS_OWNER
    rng = np.random.default_rng(2024 + W)
    batches = []  # [k][r]: the keys arm's device buffer and the wire arms' page-locked buffers
    for k in range(args.distinct):
        per = []
        for r in range(W):
            ids = zipf_ids(rng, N, args.keys, 1.1)
            packed = native.pack_keys([bytes(x) for x in bench_key_bytes(ids)], 1, (ids & 1).astype(np.uint32), 0)
            items = [b"\x0a" + bytes([len(w)]) + w for w in map(wire_item, ids.tolist())]
            x = dict(packed=torch.from_numpy(packed).to("cuda"), packed_bytes=len(packed))
            for arm, rpc in (("rpc100", 100), ("rpc1000", 1000)):
                msgs = [b"".join(items[lo:lo + rpc]) for lo in range(0, N, rpc)]
                buf, bound = native.pack_proto(msgs, T0)
                pin = native.PinnedArray(len(buf), np.uint8)
                pin.array[:] = buf
                x[arm] = (pin, len(msgs), bound)
            per.append(x)
        batches.append(per)
    outs = [torch.zeros((N, 32), dtype=torch.uint8, device="cuda") for _ in range(W)]
    wire_out = {}  # arm -> [parity][r] = (out, off, status)
    for arm in ("rpc100", "rpc1000"):
        bound = max(b[r][arm][2] for b in batches for r in range(W))
        n_msgs = max(b[r][arm][1] for b in batches for r in range(W))
        wire_out[arm] = [[(native.PinnedArray(bound, np.uint8), native.PinnedArray(n_msgs + 1, np.uint64), native.PinnedArray(n_msgs, np.uint32))
                          for _ in range(W)] for _ in range(2)]
    ns = [N] * W
    calls = {arm: 0 for arm in ARMS}

    def step(arm, k, now):
        lr, b = rings[arm], batches[k % args.distinct]
        clk = g.clock_fill(now)
        streams = [s.cuda_stream for s in lr.streams]
        if arm == "keys":
            native.p2p_step_keys_local_all(lr.p2ps, [x["packed"].data_ptr() for x in b], [x["packed_bytes"] for x in b], ns, table, T0, clk,
                                           [o.data_ptr() for o in outs], streams)
            return
        o = wire_out[arm][calls[arm] & 1]
        calls[arm] += 1
        native.p2p_step_proto_local_all(lr.p2ps, [x[arm][0].ptr for x in b], [len(x[arm][0].array) for x in b], [x[arm][1] for x in b], clk,
                                        [o[r][0].ptr for r in range(W)], [len(o[r][0].array) for r in range(W)], [o[r][1].ptr for r in range(W)],
                                        [o[r][2].ptr for r in range(W)], streams)

    now = T0
    for _ in range(args.warmup):
        for arm in ARMS:
            step(arm, 0, now)
        now += 1
    torch.cuda.synchronize()
    spent = {arm: [] for arm in ARMS}
    done, k = 0, 1
    while done < args.steps:
        blk = min(args.block, args.steps - done)
        for arm in ARMS:
            t0 = time.perf_counter()
            for j in range(blk):
                step(arm, k + j, now + j)
            torch.cuda.synchronize()
            spent[arm].append((time.perf_counter() - t0) / blk)
        k += blk; now += blk; done += blk
    for lr in rings.values():
        lr.sync()
    # the last step: (a)'s records, encoded per RPC, against the bytes of (b) and (c)
    last = [outs[r].cpu().numpy().reshape(-1).view(native.RESP_DTYPE) for r in range(W)]
    assert all((x["err_code"] == 0).all() for x in last)
    enc = [[PW.encode_resp(int(v["status"]), int(v["limit"]), int(v["remaining"]), int(v["reset_time"])) for v in x] for x in last]
    same = True
    for arm, rpc in (("rpc100", 100), ("rpc1000", 1000)):
        o = wire_out[arm][(calls[arm] - 1) & 1]
        for r in range(W):
            n = batches[(k - 1) % args.distinct][r][arm][1]
            out, off, st = o[r][0].array, o[r][1].array, o[r][2].array
            same &= bool((st[:n] == native.PROTO_OK).all())
            same &= all(out[int(off[m]):int(off[m + 1])].tobytes() == b"".join(enc[r][m * rpc:(m + 1) * rpc]) for m in range(n))
    res = {"world": W, "device": 0, "items_per_shard_step": N, "steps": args.steps, "block": args.block, "resident_keys": args.keys,
           "timer": "host clock per block of calls, ending in a device synchronise", "identical_last_responses": same}
    for arm in ARMS:
        us = float(np.median(spent[arm])) * 1e6
        res[arm] = {"us_per_call_median": round(us, 1), "us_per_call_min": round(min(spent[arm]) * 1e6, 1),
                    "us_per_call_max": round(max(spent[arm]) * 1e6, 1), "decisions_per_s": round(W * N / (us * 1e-6))}
    for arm in ("rpc100", "rpc1000"):
        for par in wire_out[arm]:
            for t in par:
                for a in t:
                    a.free()
    for b in batches:
        for x in b:
            for arm in ("rpc100", "rpc1000"):
                x[arm][0].free()
    for lr in rings.values():
        for p in lr.p2ps:
            p.close()
        for t in lr.tabs:
            t.close()
    return res, same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", default="1,2,4")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--block", type=int, default=20, help="calls per arm before switching to the next arm")
    ap.add_argument("--distinct", type=int, default=3, help="pre-generated calls per shard, cycled")
    ap.add_argument("--keys", type=int, default=1_000_000)
    ap.add_argument("--capacity", type=int, default=1 << 21, help="table slots per shard")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("ring_proto_bench: no GPU")
    print(json.dumps({"gpu": gpu_info(), "cuda_devices": torch.cuda.device_count()}), flush=True)
    ok = True
    for W in [int(w) for w in args.worlds.split(",")]:
        res, same = run_world(W, args)
        print(json.dumps(res), flush=True)
        ok &= same
    if not ok:
        sys.exit("ring_proto_bench: the wire arms' last responses differ from the key-string arm's")


if __name__ == "__main__":
    main()
