"""Key-space sharding across the GPUs of one box: the intra-box replacement for the reference's peer forwarding
(gubernator.go:257-283 -> peer_client.go:284 runBatch -> GetPeerRateLimits, gubernator.go:462).

One process per GPU.  Per step every rank
  1. routes its ingest batch by owner — owner(key) is the reference's ReplicatedConsistentHash.Get over the addresses
     "gpu:0".."gpu:N-1" (replicated_hash.go:104-119) — as a stable partition, so per-key order inside the batch survives,
  2. exchanges the per-owner counts, then the 64-byte request records (all-to-all, variable splits; NCCL over NVLink on GPUs),
  3. evaluates the records it owns: the batch it sees is the concatenation over source ranks (rank order) of their
     owner-sorted records, a deterministic order that tests reproduce with one oracle per shard,
  4. sends the 32-byte responses back along the same splits and restores request order.

The device work (route / evaluate / unroute) is supplied by a backend; GpuBackend drives the CUDA library.  The
exchange logic itself is backend-agnostic so that tests/test_sharded_gloo.py can run it on CPU with gloo.
"""
import numpy as np


def shard_addresses(n):
    return [f"gpu:{r}" for r in range(n)]


class ShardedStep:
    """global_sync=True adds the reference's GLOBAL behaviour (global.go, gubernator.go:395-459): GLOBAL requests are
    answered by whichever shard ingests them (from its replica), their hits are queued and, at every tick(), summed per
    key, sent to the owner, applied there with DRAIN_OVER_LIMIT, and the owner's resulting state is broadcast to every
    other shard, which overwrites its replica.  tick() is the reference's GlobalSyncWait timer made explicit."""

    def __init__(self, backend, dist, world, global_sync=False):
        self.be, self.dist, self.world, self.global_sync = backend, dist, world, global_sync
        self.steps = 0

    def step(self, reqs, n, clk, out):
        """reqs/out: backend buffers holding n request / response records.  Returns the number of records evaluated here."""
        be, dist, W = self.be, self.dist, self.world
        self.steps += 1
        if self.global_sync:
            routed, perm, counts = be.route_global(reqs, n, self.steps)  # also queues the hits of GLOBAL requests owned elsewhere
        else:
            routed, perm, counts = be.route(reqs, n)             # counts: integer tensor [W] on the backend's device
        recv_counts = be.empty_like(counts)
        dist.all_to_all_single(recv_counts, counts)
        send_l, recv_l = be.two_lists(counts, recv_counts)       # the one host sync of the step: split sizes of the variable all-to-all
        m = sum(recv_l)
        inbox = be.req_buffer(m)
        dist.all_to_all_single(inbox[:m], routed[:n], output_split_sizes=recv_l, input_split_sizes=send_l)
        resp = be.evaluate(inbox, m, clk)
        if self.global_sync:
            be.queue_updates(inbox, m, self.steps)               # GLOBAL requests just evaluated as owner (gubernator.go:604-606)
        back = be.resp_buffer(n)
        dist.all_to_all_single(back[:n], resp[:m], output_split_sizes=send_l, input_split_sizes=recv_l)
        be.unroute(back, perm, n, out)
        return m


    def tick(self, clk, now_ms):
        """One GLOBAL sync: sendHits (global.go:144-190) then broadcastPeers (global.go:234-283).  Collective: every rank
        must call it.  Returns (hit records sent, update items received).  The window's hits travel in one all-to-all (a
        single round); the ring's gub_global_tick is the one that splits a window larger than its mailboxes into rounds."""
        be, dist, W = self.be, self.dist, self.world
        self.steps += 1
        # 1. aggregated hits -> owners (GetPeerRateLimits on the owner: DRAIN_OVER_LIMIT, IsOwner = true)
        hits, k = be.drain_hits()
        routed, perm, counts = be.route(hits, k)
        recv_counts = be.empty_like(counts)
        dist.all_to_all_single(recv_counts, counts)
        send_l, recv_l = be.two_lists(counts, recv_counts)
        m = sum(recv_l)
        inbox = be.req_buffer(m)
        dist.all_to_all_single(inbox[:m], routed[:k], output_split_sizes=recv_l, input_split_sizes=send_l)
        be.evaluate(inbox, m, clk)                               # responses are dropped, like sendHits drops them
        be.queue_updates(inbox, m, self.steps)
        # 2. owners read back the state of every key touched by GLOBAL traffic (Hits = 0) and broadcast it
        items, ki = be.make_updates(clk)
        mine = be.int_tensor([ki])
        all_counts = be.int_tensor([0] * W)
        dist.all_gather_into_tensor(all_counts, mine)
        cl = [int(x) for x in all_counts.tolist()]
        pad = max(max(cl), 1)
        gathered = be.item_buffer(pad * W)
        dist.all_gather_into_tensor(gathered[:pad * W], be.pad_items(items, ki, pad))
        got = 0
        for r in range(W):
            if r != be.rank and cl[r]:                           # "Exclude ourselves from the update" (global.go:263-265)
                be.add_items(gathered[r * pad:r * pad + cl[r]], cl[r], now_ms)
                got += cl[r]
        return k, got


class LocalExchange:
    """In-process stand-in for torch.distributed: W shards as W threads in one process (the reference's own test fixture
    does the same with N daemons, cluster/cluster.go:151).  Only the collectives ShardedStep uses."""

    def __init__(self, world):
        import threading
        self.world = world
        self.bar = threading.Barrier(world)
        self.box = [None] * world

    def handle(self, rank):
        return _LocalHandle(self, rank)


class _LocalHandle:
    def __init__(self, ex, rank):
        self.ex, self.rank = ex, rank

    def all_to_all_single(self, out, inp, output_split_sizes=None, input_split_sizes=None):
        ex, W, r = self.ex, self.ex.world, self.rank
        if input_split_sizes is None:
            per = inp.shape[0] // W
            input_split_sizes = [per] * W
            output_split_sizes = [out.shape[0] // W] * W
        offs = [0]
        for c in input_split_sizes:
            offs.append(offs[-1] + c)
        ex.box[r] = (inp, offs)
        ex.bar.wait()
        o = 0
        for src in range(W):
            sin, soffs = ex.box[src]
            a, b = soffs[r], soffs[r + 1]
            assert b - a == output_split_sizes[src]
            if b > a:
                out[o:o + (b - a)].copy_(sin[a:b])
            o += b - a
        _sync(out)
        ex.bar.wait()

    def all_gather_into_tensor(self, out, inp):
        ex, W, r = self.ex, self.ex.world, self.rank
        ex.box[r] = inp
        ex.bar.wait()
        n = inp.shape[0]
        for src in range(W):
            out[src * n:(src + 1) * n].copy_(ex.box[src])
        _sync(out)
        ex.bar.wait()

    def barrier(self):
        self.ex.bar.wait()


def _sync(t):
    if t.is_cuda:
        import torch
        torch.cuda.current_stream().synchronize()


class GpuBackend:
    """torch CUDA tensors as buffers (torch is only the allocator and the NCCL plumbing); kernels from the C ABI."""

    def __init__(self, table, ring, world, device, cap, rank=0, global_capacity=0):
        import torch
        from . import native
        self.torch, self.tab, self.ring, self.W, self.dev, self.rank = torch, table, ring, world, device, rank
        self.hits_q = self.updates_q = None
        if global_capacity:
            dev_index = device.index if device.index is not None else 0
            self.hits_q = native.GlobalQueue(dev_index, global_capacity, keep_latest=False)
            self.updates_q = native.GlobalQueue(dev_index, global_capacity, keep_latest=True)
            self.owner = torch.empty(cap, dtype=torch.uint8, device=device)
            self.gbuf = torch.empty((global_capacity, 64), dtype=torch.uint8, device=device)
            self.gresp = torch.empty((global_capacity, 32), dtype=torch.uint8, device=device)
            self.gitems = torch.empty((global_capacity, native.ITEM_DTYPE.itemsize), dtype=torch.uint8, device=device)
            self.gcount = torch.zeros(1, dtype=torch.int32, device=device)
            self.gcap = global_capacity
        self.cap = cap
        self.routed = torch.empty((cap, 64), dtype=torch.uint8, device=device)
        self.perm = torch.empty(cap, dtype=torch.int32, device=device)
        self.counts16 = torch.zeros(16, dtype=torch.int32, device=device)
        self.in_cap = 0
        self.inbox = self.inbox_resp = None
        self.back = torch.empty((cap, 32), dtype=torch.uint8, device=device)

    def _stream(self):
        return self.torch.cuda.current_stream().cuda_stream

    def route(self, reqs, n):
        self.tab.route_device(self.ring, reqs.data_ptr(), n, self.routed.data_ptr(), self.perm.data_ptr(), self.counts16.data_ptr(), self._stream())
        return self.routed, self.perm, self.counts16[:self.W].clone()

    def empty_like(self, t):
        return self.torch.empty_like(t)

    def two_lists(self, a, b):
        both = self.torch.stack([a, b]).tolist()  # one device->host copy instead of two
        return [int(x) for x in both[0]], [int(x) for x in both[1]]

    def req_buffer(self, m):
        if m > self.in_cap or self.inbox is None:
            self.in_cap = int(m * 1.25) + 4096
            self.inbox = self.torch.empty((self.in_cap, 64), dtype=self.torch.uint8, device=self.dev)
            self.inbox_resp = self.torch.empty((self.in_cap, 32), dtype=self.torch.uint8, device=self.dev)
        return self.inbox

    def resp_buffer(self, n):
        return self.back

    def evaluate(self, inbox, m, clk):
        self.tab.submit_device(inbox.data_ptr(), m, clk, self.inbox_resp.data_ptr(), self._stream())
        return self.inbox_resp

    def unroute(self, back, perm, n, out):
        self.tab.unroute_device(back.data_ptr(), perm.data_ptr(), n, out.data_ptr(), self._stream())

    # ---- GLOBAL behaviour
    def route_global(self, reqs, n, step):
        st = self._stream()
        self.tab.route_global_device(self.ring, self.rank, reqs.data_ptr(), n, self.routed.data_ptr(), self.perm.data_ptr(),
                                     self.counts16.data_ptr(), self.owner.data_ptr(), st)
        # a non-owner queues the hits of its GLOBAL requests (gubernator.go:402-404), keeping the first request per key
        self.hits_q.accumulate_device(reqs.data_ptr(), n, self.owner.data_ptr(), self.rank, step << 32, st)
        return self.routed, self.perm, self.counts16[:self.W].clone()

    def queue_updates(self, inbox, m, step):
        self.updates_q.accumulate_device(inbox.data_ptr(), m, None, self.rank, step << 32, self._stream())

    def drain_hits(self):
        self.hits_q.drain_device(self.gbuf.data_ptr(), self.gcap, self.gcount.data_ptr(), False, self._stream())
        return self.gbuf, min(int(self.gcount.item()), self.gcap)

    def make_updates(self, clk):
        st = self._stream()
        self.updates_q.drain_device(self.gbuf.data_ptr(), self.gcap, self.gcount.data_ptr(), True, st)
        k = min(int(self.gcount.item()), self.gcap)
        if k:
            self.tab.submit_device(self.gbuf.data_ptr(), k, clk, self.gresp.data_ptr(), st)
        self.tab.make_updates_device(self.gbuf.data_ptr(), self.gresp.data_ptr(), k, self.gitems.data_ptr(), self.gcount.data_ptr(), st)
        return self.gitems, int(self.gcount.item())

    def int_tensor(self, values):
        return self.torch.tensor(values, dtype=self.torch.int32, device=self.dev)

    def item_buffer(self, n):
        return self.torch.empty((n, self.gitems.shape[1]), dtype=self.torch.uint8, device=self.dev)

    def pad_items(self, items, k, pad):
        if k == pad:
            return items[:pad]
        buf = self.torch.zeros((pad, items.shape[1]), dtype=self.torch.uint8, device=self.dev)
        buf[:k].copy_(items[:k])
        return buf

    def add_items(self, items, n, now_ms):
        items = items.contiguous()
        self.tab.add_items_device(items.data_ptr(), n, now_ms, self._stream())
        self.torch.cuda.current_stream().synchronize()  # `items` may be a temporary


class P2PStep:
    """Same contract as ShardedStep.step, but the records travel by NVLink stores issued from the routing kernels themselves
    (gub_p2p_step): no NCCL collective and no exchange of split sizes."""

    def __init__(self, table, ring, world, rank, cap=65536):
        from . import native
        self.ring, self.world, self.rank = ring, world, rank
        self.p2p = native.P2P(table, ring, rank, cap)

    def connect(self, dist):
        """One process per GPU: swap cudaIpc handles through torch.distributed."""
        handles = [None] * self.world
        dist.all_gather_object(handles, self.p2p.export())
        self.p2p.connect(handles)
        dist.barrier()

    def connect_local(self, steppers):
        self.p2p.connect_local([s.p2p for s in steppers])

    def step(self, reqs, n, clk, out, stream=None, ingest_stream=None):
        """ingest_stream: the stream `reqs` was produced on; when given, routing runs there and overlaps the evaluation of
        the previous step, which runs on `stream` (where `out` becomes valid)."""
        import torch
        st = stream if stream is not None else torch.cuda.current_stream().cuda_stream
        self.p2p.step(reqs.data_ptr(), n, clk, out.data_ptr(), st, ingest_stream)
        return n
