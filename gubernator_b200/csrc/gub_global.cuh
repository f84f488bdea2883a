// gub_global.cuh — device side of GLOBAL behaviour (global.go:30-283, gubernator.go:395-459 of mailgun/gubernator v2.4.0).
//
// The reference keeps, per peer, two maps fed by channels:
//   hits    (runAsyncHits, global.go:91-141)   key -> the FIRST queued request, with Hits summed over the window and
//           RESET_REMAINING OR-ed in; flushed to the owning peers every GlobalSyncWait,
//   updates (runBroadcasts, global.go:193-231) key -> the LATEST request seen by the owner; on flush the owner re-reads the
//           state with Hits = 0 (global.go:243-245) and broadcasts it; peers overwrite their replica (UpdatePeerGlobals).
// Here both maps are one device structure, a `gq`: an open-addressed table of 64-byte gub_req records keyed by the
// request's XXH64, filled by two small kernels per batch (claim: insert / sum hits / order by sequence; fill: the winning
// request writes its parameters) and drained into a dense array of request records at each sync tick, which sends the hit
// records to their owners in key-consistent rounds (k_gq_hist, gq_plan_rounds, k_gq_partition below).
#pragma once
#if !defined(GUB_EMULATE)  // tests/kernel_emu_harness.cpp compiles this header for the CPU (see gub_kernels.cuh)
#include <cuda_runtime.h>
#endif
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "../../include/gubernator_b200.h"

namespace gub {

enum : uint32_t { GQ_KEEP_FIRST = 0, GQ_KEEP_LAST = 1 };

struct Gq {
  gub_req* slots;                 // capacity records; key_xxh64 == 0 <=> empty (keys are remapped off 0)
  unsigned long long* seq;        // capacity: sequence number of the request whose parameters the slot keeps
  uint32_t capacity_mask;
  uint32_t mode;
  unsigned long long* count;      // live entries
  unsigned long long* dropped;    // optional: requests not queued because the table was full within one sync window (counted, not silent)
};

// Which requests of a batch feed the queue:
//   hits queue    : GLOBAL set, this shard is NOT the owner, Hits != 0   (gubernator.go:402-404, global.go:74-78)
//   updates queue : GLOBAL set (only requests evaluated as owner still carry it), Hits != 0 (gubernator.go:604-606, global.go:80-84)
// `owner` is optional (nullptr for the updates queue): owner[i] != self selects non-owned keys.
__device__ __forceinline__ bool gq_selects(const gub_req& r, const uint8_t* owner, uint32_t i, uint32_t self, bool want_non_owner) {
  if (!(r.behavior & GUB_BEHAVIOR_GLOBAL) || r.hits == 0) return false;
  if (r.key_xxh64 == 0) return false;  // 0 marks an empty queue slot; a key hashing to exactly 0 (p = 2^-64) is simply never synchronised
  if (!owner) return !want_non_owner;
  return want_non_owner ? (owner[i] != self) : (owner[i] == self);
}

// Pass 1: insert the key, add Hits, OR RESET_REMAINING, and let the earliest (KEEP_FIRST) or latest (KEEP_LAST) sequence win.
// Returns the slot (0xFFFFFFFF: not queued).  s = the request's sequence number (> 0).
__device__ __forceinline__ uint32_t gq_claim_one(const Gq& q, unsigned long long key, int64_t hits, uint32_t behavior, unsigned long long s) {
  uint32_t pos = (uint32_t)(key ^ (key >> 31)) & q.capacity_mask;
  for (uint32_t probe = 0; probe <= q.capacity_mask; probe++) {
    unsigned long long* kp = reinterpret_cast<unsigned long long*>(&q.slots[pos].key_xxh64);
    const unsigned long long old = atomicCAS(kp, 0ull, key);
    if (old == 0ull) atomicAdd(q.count, 1ull);
    if (old == 0ull || old == key) {
      atomicAdd(reinterpret_cast<unsigned long long*>(&q.slots[pos].hits), (unsigned long long)hits);  // global.go:109 (wrapping, like Go)
      // only the hits aggregation ORs RESET_REMAINING in (global.go:105-108); the update map just keeps the latest request (global.go:201)
      if (q.mode == GQ_KEEP_FIRST && (behavior & GUB_BEHAVIOR_RESET_REMAINING)) atomicOr(&q.slots[pos].behavior, (unsigned)GUB_BEHAVIOR_RESET_REMAINING);
      if (q.mode == GQ_KEEP_LAST) atomicMax(&q.seq[pos], s);
      else atomicMax(&q.seq[pos], ~s);  // earliest wins: store ~s and take the max, so an empty (0) slot loses to anything
      return pos;
    }
    pos = (pos + 1) & q.capacity_mask;
  }
  if (q.dropped) atomicAdd(q.dropped, 1ull);  // the reference's maps are unbounded (global.go:99,201): size the queue for the hot set
  return 0xFFFFFFFFu;
}

// Pass 2: the request whose sequence won writes the parameters the entry keeps (everything but Hits and the OR-ed flag).
__device__ __forceinline__ void gq_fill_one(const Gq& q, const gub_req* rp, uint32_t pos, unsigned long long s) {
  const unsigned long long want = (q.mode == GQ_KEEP_LAST) ? s : ~s;
  if (q.seq[pos] != want) return;
  const gub_req r = *rp;
  gub_req* e = &q.slots[pos];
  e->key_fnv1 = r.key_fnv1; e->limit = r.limit; e->duration = r.duration; e->burst = r.burst; e->created_at = r.created_at;
  e->algorithm = r.algorithm;
  if (q.mode == GQ_KEEP_LAST) e->behavior = r.behavior;  // the latest request as it is
  else atomicOr(&e->behavior, r.behavior);               // the first request's bits; pass 1 may have OR-ed RESET_REMAINING in
}

__global__ void k_gq_claim(Gq q, const gub_req* reqs, uint32_t n, const uint32_t* n_dev, const uint8_t* owner, uint32_t self, uint32_t want_non_owner,
                           unsigned long long seq_base, uint32_t* slot_of /* [n] out: slot index or 0xFFFFFFFF */) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (n_dev) n = min(n, *n_dev);
  if (i >= n) return;
  const ulonglong2* p = reinterpret_cast<const ulonglong2*>(reqs + i);
  const ulonglong2 a = __ldg(p), b = __ldg(p + 1), d = __ldg(p + 3);
  gub_req r;
  r.key_xxh64 = a.x; r.hits = (int64_t)b.x; r.behavior = (uint32_t)(d.y >> 32);
  slot_of[i] = 0xFFFFFFFFu;
  if (!gq_selects(r, owner, i, self, want_non_owner != 0)) return;
  slot_of[i] = gq_claim_one(q, r.key_xxh64, r.hits, r.behavior, seq_base + i + 1);
}

__global__ void k_gq_fill(Gq q, const gub_req* reqs, uint32_t n, const uint32_t* n_dev, unsigned long long seq_base, const uint32_t* slot_of) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (n_dev) n = min(n, *n_dev);
  if (i >= n) return;
  const uint32_t pos = slot_of[i];
  if (pos == 0xFFFFFFFFu) return;
  gq_fill_one(q, reqs + i, pos, seq_base + i + 1);
}

// The same two passes over the W mailbox segments a shard has just evaluated (fused routing): segment s holds
// (flag[s] & 0xFFFFFFFF) records; order = (segment, position) = the order they were evaluated in.
struct GqSegs {
  const gub_req* reqs[16];
  const unsigned long long* flag[16];
  uint32_t nseg, cap;
};
__global__ void k_gq_claim_segs(Gq q, GqSegs G, unsigned long long seq_base, uint32_t* slot_of /* [nseg * cap] */) {
  const uint32_t total = G.nseg * G.cap;
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < total; v += gridDim.x * blockDim.x) {
    const uint32_t s = v / G.cap, j = v % G.cap;
    if (j >= (uint32_t)(*G.flag[s] & 0xFFFFFFFFull)) continue;
    const ulonglong2* p = reinterpret_cast<const ulonglong2*>(G.reqs[s] + j);
    const ulonglong2 a = __ldcg(p), b = __ldcg(p + 1), d = __ldcg(p + 3);
    gub_req r;
    r.key_xxh64 = a.x; r.hits = (int64_t)b.x; r.behavior = (uint32_t)(d.y >> 32);
    slot_of[v] = gq_selects(r, nullptr, 0, 0, false) ? gq_claim_one(q, r.key_xxh64, r.hits, r.behavior, seq_base + v + 1) : 0xFFFFFFFFu;
  }
}
__global__ void k_gq_fill_segs(Gq q, GqSegs G, unsigned long long seq_base, const uint32_t* slot_of) {
  const uint32_t total = G.nseg * G.cap;
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < total; v += gridDim.x * blockDim.x) {
    const uint32_t s = v / G.cap, j = v % G.cap;
    if (j >= (uint32_t)(*G.flag[s] & 0xFFFFFFFFull)) continue;
    const uint32_t pos = slot_of[v];
    if (pos != 0xFFFFFFFFu) gq_fill_one(q, G.reqs[s] + j, pos, seq_base + v + 1);
  }
}

// Drain: every live entry becomes one request record in `out` (dense, arbitrary order); the table is cleared.
//   hits queue    -> requests for the owner: Hits = the window's sum; GetPeerRateLimits adds DRAIN_OVER_LIMIT to GLOBAL
//                    requests (gubernator.go:510-512) and evaluates them as owner.
//   updates queue -> status queries: Hits = 0, evaluated with IsOwner = false (global.go:238-245).
__global__ void k_gq_drain(Gq q, gub_req* out, uint32_t out_cap, uint32_t* out_count, uint32_t as_status_query) {
  for (uint32_t pos = blockIdx.x * blockDim.x + threadIdx.x; pos <= q.capacity_mask; pos += gridDim.x * blockDim.x) {
    gub_req e = q.slots[pos];
    if (e.key_xxh64 == 0) continue;
    const uint32_t k = atomicAdd(out_count, 1u);
    if (k < out_cap) {
      if (as_status_query) { e.hits = 0; e.behavior &= ~(uint32_t)GUB_REQ_IS_OWNER; }
      else e.behavior |= (uint32_t)(GUB_BEHAVIOR_DRAIN_OVER_LIMIT | GUB_REQ_IS_OWNER);
      out[k] = e;
    } else if (q.dropped) {
      atomicAdd(q.dropped, 1ull);  // an output smaller than the queue (gub_gq_drain_device); the sync tick drains into the queue's capacity
    }
    gub_req z = {};
    q.slots[pos] = z;
    q.seq[pos] = 0ull;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *q.count = 0ull;
}

// ---- A sync tick's hit records in rounds ----------------------------------------------------------------------------------------
// A tick sends every drained hit record to its owner through the ring's mailboxes, which take at most `cap` records per source and
// step.  A window of more keys travels in rounds, one mailbox epoch each.  The rounds are key-consistent: the hash space is cut
// into GQ_BINS bins by the top 16 bits of key_xxh64, and consecutive bins are packed into rounds such that no source has more than
// `cap` records in one round.  Every source's record of a key therefore travels in the same round, and the owner applies them in
// source-rank order, exactly as a single-round tick (and OracleCluster.tick of tests/global_model.py) does.  The packing is a
// function of every shard's histogram alone, so every shard computes the same rounds.
// A bin that holds more than `cap` records of one source (only crafted keys sharing their top 16 bits of XXH64 do that) is split by
// position over consecutive rounds: nothing is dropped, but for those keys the order between sources is the round order.  The
// reference defines no order between its peers' sendHits either.
enum : uint32_t { GQ_BIN_BITS = 16, GQ_BINS = 1u << GQ_BIN_BITS };

__device__ __forceinline__ uint32_t gq_bin(unsigned long long key) { return (uint32_t)(key >> (64 - GQ_BIN_BITS)); }

// hist[bin] += records of that bin (hist zeroed by the caller).
__global__ void k_gq_hist(const gub_req* recs, uint32_t n, const uint32_t* n_dev, uint32_t* hist) {
  if (n_dev) n = min(n, *n_dev);
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    atomicAdd(&hist[gq_bin(__ldg(reinterpret_cast<const unsigned long long*>(&recs[i].key_xxh64)))], 1u);
}

// Counting sort by bin: cursor[bin] = the first output index of that bin (the exclusive prefix sum of k_gq_hist), advanced here.
// The order inside a bin is arbitrary; one source's records of one round are distinct keys, so it does not matter.
__global__ void k_gq_partition(const gub_req* recs, uint32_t n, const uint32_t* n_dev, uint32_t* cursor, gub_req* out) {
  if (n_dev) n = min(n, *n_dev);
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const ulonglong2* p = reinterpret_cast<const ulonglong2*>(recs + i);
    const ulonglong2 a = __ldg(p), b = __ldg(p + 1), c = __ldg(p + 2), d = __ldg(p + 3);
    ulonglong2* o = reinterpret_cast<ulonglong2*>(out + atomicAdd(&cursor[gq_bin(a.x)], 1u));
    o[0] = a; o[1] = b; o[2] = c; o[3] = d;
  }
}

// One round: the bins [lo, hi); for a split bin (hi = lo + 1) slice k carries records k*cap ... k*cap + cap - 1 of every source.
struct GqRound { uint32_t lo, hi, slice; };

// Host side, identical on every shard.  hist[s] = source s's GQ_BINS counts.  Empty bins join a neighbouring round; an empty window
// is one (empty) round, like the single-round tick.
inline void gq_plan_rounds(const uint32_t* const* hist, uint32_t nsrc, uint32_t cap, std::vector<GqRound>& out) {
  out.clear();
  std::vector<uint64_t> sum(nsrc, 0);
  uint32_t lo = 0;
  bool open = false;
  auto close = [&](uint32_t hi) {
    if (open) out.push_back(GqRound{lo, hi, 0});
    std::fill(sum.begin(), sum.end(), 0);
    open = false;
    lo = hi;
  };
  for (uint32_t b = 0; b < GQ_BINS; b++) {
    uint32_t most = 0;
    for (uint32_t s = 0; s < nsrc; s++) most = std::max(most, hist[s][b]);
    if (most == 0) continue;
    if (most > cap) {  // over-full bin: split by position
      close(b);
      for (uint32_t k = 0; k < (most + cap - 1) / cap; k++) out.push_back(GqRound{b, b + 1, k});
      lo = b + 1;
      continue;
    }
    bool fits = true;
    for (uint32_t s = 0; s < nsrc; s++) fits = fits && sum[s] + hist[s][b] <= cap;
    if (!fits) close(b);
    for (uint32_t s = 0; s < nsrc; s++) sum[s] += hist[s][b];
    open = true;
  }
  close(GQ_BINS);
  if (out.empty()) out.push_back(GqRound{0, GQ_BINS, 0});
}

// This source's records of round R in the partitioned array: start = the exclusive prefix sum of its histogram (GQ_BINS + 1).
inline void gq_round_span(const GqRound& R, const uint32_t* start, uint32_t cap, uint32_t* off, uint32_t* n) {
  const uint32_t total = start[R.hi] - start[R.lo];
  const uint64_t skip = std::min<uint64_t>((uint64_t)R.slice * cap, total);
  *off = start[R.lo] + (uint32_t)skip;
  *n = (uint32_t)std::min<uint64_t>(cap, total - skip);
}

// UpdatePeerGlobal records (peers.proto:52-72) from the owner's status queries: the CacheItem a peer will install
// (gubernator.go:427-451): ExpireAt = status.ResetTime; token {Status, Limit, Duration, Remaining, CreatedAt = now};
// leaky {Remaining = float64(status.Remaining), Limit, Duration, Burst = status.Limit, UpdatedAt = now}.
// `now` is filled in by the receiver (gub_add_items_device takes it), so the record carries stamp = 0 here.
__global__ void k_make_updates(const gub_req* queries, const gub_resp* resps, uint32_t n, const uint32_t* n_dev, gub_item* out, uint32_t* out_count) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (n_dev) n = min(n, *n_dev);
  if (i >= n) return;
  const gub_req r = queries[i];
  const gub_resp s = resps[i];
  if (s.err_code != 0 || r.algorithm > 1u) return;  // "while retrieving rate limit status": logged and skipped (global.go:246-249)
  const uint32_t k = atomicAdd(out_count, 1u);
  gub_item it;
  it.key_xxh64 = r.key_xxh64; it.key_fnv1 = r.key_fnv1; it.algorithm = (int32_t)r.algorithm; it.status = (int32_t)s.status;
  it.limit = s.limit; it.duration = r.duration; it.remaining = s.remaining; it.remaining_f = (double)s.remaining;
  it.stamp = 0; it.burst = s.limit; it.expire_at = s.reset_time; it.invalid_at = 0;
  out[k] = it;
}

}  // namespace gub
