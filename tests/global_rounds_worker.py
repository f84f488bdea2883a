"""torchrun worker of tests/test_gpu_global_rounds.py: one process per GPU, GLOBAL behaviour behind the C ABI with NCCL (gub_p2p_step,
gub_global_tick), windows of more GLOBAL keys than the mailbox capacity so that every tick runs several rounds.  Every rank replays the
whole cluster in the oracle-side model and checks its own responses and its final table against it."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.environ["GUB_ROOT"]
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import oracle_py as O  # noqa: E402
import gubernator_b200 as g  # noqa: E402
from gubernator_b200.sharded import shard_addresses  # noqa: E402
from global_model import OracleCluster  # noqa: E402
from workloads import T0, key_hashes  # noqa: E402

CAP, GCAP = 4096, 16384
local = int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
rank, W = dist.get_rank(), dist.get_world_size()
dev = torch.device("cuda", local)
tab = g.Table(1 << 17, device=local)
ring = g.Ring(0, 512)
for a in shard_addresses(W):
    ring.add(a)
p2p = g.native.P2P(tab, ring, rank, CAP)
handles = [None] * W
dist.all_gather_object(handles, p2p.export())
p2p.connect(handles)
p2p.enable_global(GCAP)
uid = [g.native.nccl_unique_id() if rank == 0 else None]
dist.broadcast_object_list(uid, src=0)
p2p.nccl_init(uid[0])
dist.barrier()


def batch(ids, src, window, now):
    b = np.zeros(len(ids), dtype=O.HREQ_DTYPE)
    xx, fv = key_hashes(ids, name="rounds")
    b["key_xxh64"], b["key_fnv1"] = xx, fv
    b["limit"] = 20 + ((ids + 3 * src + window) % 7) * 10
    b["duration"] = 30000 + (ids % 3) * 30000
    b["algorithm"] = (ids >> 1) & 1
    b["hits"] = np.where(ids % 11 == 0, 0, 1 + (ids % 3))
    b["created_at"] = now
    b["behavior"] = np.where(ids % 5 != 0, O.GLOBAL, 0).astype(np.uint32) | np.uint32(O.REQ_IS_OWNER)
    if window == 1:
        b["behavior"] |= np.where((ids % 5 != 0) & (ids % 13 == 0), O.RESET_REMAINING, 0).astype(np.uint32)
    return b


model = OracleCluster(W, T0)
rng = np.random.default_rng(31337)  # the same stream on every rank: everybody generates everybody's batches
st = torch.cuda.current_stream().cuda_stream
now = T0
sent = []
for window in range(2):
    for step in range(5):
        batches = [batch(rng.choice(np.arange(1, 20000), CAP, replace=False), r, window, now + step) for r in range(W)]
        mine = batches[rank]
        buf = torch.from_numpy(mine.view(np.uint8).reshape(CAP, 64).copy()).to(dev)
        out = torch.zeros((CAP, 32), dtype=torch.uint8, device=dev)
        p2p.step(buf.data_ptr(), CAP, g.clock_fill(now + step), out.data_ptr(), st)
        torch.cuda.synchronize()
        got = out.cpu().numpy().reshape(-1).view(O.HRESP_DTYPE)
        want = model.step(batches, now + step)[rank]
        if not np.array_equal(got, want):
            bad = np.nonzero(got != want)[0]
            raise AssertionError(f"rank {rank} window {window} step {step}: {len(bad)} responses differ; first {bad[0]}: {got[bad[0]]} vs {want[bad[0]]}")
    now += 5
    res = p2p.tick(g.clock_fill(now), now, st)
    torch.cuda.synchronize()
    model.tick(now)
    sent.append(res["hits_sent"])
    now += 400
p2p.status()
assert tab.counters()["gq_dropped"] == 0
allsent = [None] * W
dist.all_gather_object(allsent, sent)
assert max(max(s) for s in allsent) > CAP, allsent  # several rounds ran
items = model.pools[rank].each()
dev_items = {(int(s["key_xxh64"]), int(s["key_fnv1"]) >> 8): s for s in tab.scan()}
assert len(dev_items) == len(items)
for (kx, kf), it in items.items():
    s = dev_items[(kx, kf >> 8)]
    assert int(s["limit"]) == it.limit and int(s["expire_at"]) == it.expire_at and int(s["stamp"]) == it.stamp
    if it.value_kind == 2:
        assert np.float64(s["remaining_f"]).view(np.uint64) == np.float64(it.remaining_f).view(np.uint64)
    else:
        assert int(s["remaining"]) == it.remaining_i and int(s["status"]) == it.status
dist.barrier()
print(f"rank {rank} ok")
dist.destroy_process_group()
