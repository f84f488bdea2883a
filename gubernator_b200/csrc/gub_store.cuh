// gub_store.cuh — sm_90a kernels of the Store plugin on the key-string path (gub_submit_keys_store_async, include/gubernator_b200.h).
//
// The host layer (csrc/host_v1.cpp submit_with_store) honours Config.Store (config.go:95) around a batch with a host-side dedup and
// two gub_get_items round trips.  Here the same rule runs on the device, as a pre-pass and a post-pass around the unchanged batch
// kernels (k_group / k_rank / k_eval / k_finish of gub_kernels.cuh):
//   k_store_keys     per-key dedup over the full 120-bit fingerprint: an epoch-tagged open-addressing scratch (StoreKey) collects every
//                    key's first and last request and whether a TOKEN_BUCKET request of it carries RESET_REMAINING.  (The batch
//                    kernels' group entries cannot serve: two keys may share one.)
//   k_store_before   one thread per key, the thread of its first request: looks the key up as k_get_items does (absent, expired at
//                    now_ms or past its InvalidAt = a miss; a key the table lacks is also looked for among the previous batch's parked
//                    inserts, which the next k_group places), keeps `existed` and the algorithm found, and files a miss record at index
//                    `first`;
//   k_store_loaded   the host's verdict for the items Store.Get returned (host layer: existed when ExpireAt >= now_ms);
//   k_store_after    one thread per key, again at its first request: reads the state the batch left (the table, else this batch's
//                    parked inserts) and the response of the key's last request, decides REMOVE / CHANGE and files the record at index
//                    `first`;
//   k_store_compact  ordered compaction of the records filed at their `first` index: the order is the index order, no sort, and the
//                    output may be host memory (the caller's page-locked buffers).
// A record at index i is filed only by thread i (the key's work runs at its first request, not its last, for that reason), so each block
// counts what it filed and the compaction finds a block's output offset by summing the counts of the blocks before it.
// On a ring (gub_p2p_step_keys_store_local_all) the same passes run per owner over its mailbox segments (StoreRing: the *_ring kernels),
// and k_store_orig gives every source an inverse map of its routing so that an owner can name each request by (source, source index).
#pragma once
#include "gub_kernels.cuh"

namespace gub {

constexpr int STORE_THREADS = 256;

// One key of the batch.  Every word carries the batch's epoch in its high half, so a word left by an earlier batch loses every
// atomicMax against this batch's values and an entry needs no clearing between batches (only at the epoch's wrap).
//   claim = epoch << 32 | index of the request that claimed the entry (the entry's key is that request's key)
//   first = epoch << 32 | (0xFFFFFFFF - index): atomicMax keeps the smallest index
//   last  = epoch << 32 | index
//   reset = epoch << 32 | 1 when a TOKEN_BUCKET request of the key carries RESET_REMAINING
struct StoreKey { unsigned long long claim, first, last, reset; };
constexpr uint32_t S_EXISTED = 1u;
struct StoreState { uint32_t existed, algorithm; };  // a key's item at batch start: S_EXISTED, and the algorithm of the item that existed

struct StoreArgs {
  const gub_req* reqs;
  const gub_resp* out;
  uint32_t n, epoch;
  StoreKey* keys;
  uint32_t key_mask;       // entries - 1 (a power of two >= 2 x max_batch)
  uint32_t* kent;          // [n] entry of request i's key
  StoreState* bstate;      // [n] at a key's first request
  uint8_t* sel;            // [n] 1 = a record was filed at index i of `sparse`
  gub_store_rec* sparse;   // [n]
  uint32_t* blk;           // [blocks] records filed per block
  const Slot* table;
  uint64_t capacity;
  const OvfItem* ovf;      // parked inserts (see OvfItem)
  const uint32_t* ovf_count;
  InvIndex inv;
  int64_t now_ms;
  uint32_t want_misses;    // k_store_before files miss records (a store with a Get)
};

__device__ __forceinline__ uint32_t skey_first(const StoreKey& k) { return 0xFFFFFFFFu - (uint32_t)k.first; }

// LRUCache.GetItem's verdict as k_get_items gives it (lrucache.go:111-128, cache.go:43-57), on the table or, for a key the table lacks,
// on the parked inserts.  b / inv_at: the item found.
__device__ __forceinline__ bool store_lookup(const StoreArgs& S, uint64_t key, uint64_t tag, Bucket& b, int64_t& inv_at) {
  Cursor cur;
  cursor_open(cur, S.table, S.capacity, key, tag);
  b = cur.b;
  bool found = cur.found;
  if (!found) {
    const uint32_t m = min(__ldcg(S.ovf_count), (uint32_t)OVF_CAP);
#pragma unroll 1
    for (uint32_t k = 0; k < m; k++) {
      if (S.ovf[k].key != key || S.ovf[k].tag != tag) continue;
      const OvfItem it = S.ovf[k];
      b.flags = it.flags; b.limit = (int64_t)it.w[0]; b.duration = (int64_t)it.w[1]; b.rem = it.w[2]; b.stamp = (int64_t)it.w[3];
      b.burst = (int64_t)it.w[4]; b.expire = (int64_t)it.w[5];
      found = true;  // (the last parking of the key is its final state)
    }
  }
  inv_at = (found && (b.flags & F_INVALID_AT)) ? inv_lookup(S.inv, key, tag) : 0;
  return found && (b.flags & F_LIVE) && !(b.expire < S.now_ms) && !(inv_at != 0 && inv_at < S.now_ms);
}

// The gub_item of a slot image, as gub_get_items reports it (from_dev of gub_api.cu); the caller sets the key fields.
__device__ __forceinline__ void store_item(const Bucket& b, int64_t inv_at, gub_item& it) {
  const bool leaky = (b.flags & F_LEAKY) != 0;
  it.algorithm = leaky ? GUB_LEAKY_BUCKET : GUB_TOKEN_BUCKET;
  it.status = (b.flags & F_OVER) ? GUB_OVER_LIMIT : GUB_UNDER_LIMIT;
  it.limit = b.limit; it.duration = b.duration;
  it.remaining = leaky ? 0 : (int64_t)b.rem;
  it.remaining_f = leaky ? bits2f(b.rem) : 0.0;
  it.stamp = b.stamp; it.burst = b.burst; it.expire_at = b.expire; it.invalid_at = inv_at;
}

__device__ __forceinline__ void store_rec_init(gub_store_rec& r, uint32_t first, uint32_t last, uint32_t flags, const gub_req& rq) {
  r.first = first; r.last = last; r.flags = flags; r.first_shard = 0; r.last_shard = 0;
  r.item.key_xxh64 = rq.key_xxh64; r.item.key_fnv1 = rq.key_fnv1;
  r.item.algorithm = 0; r.item.status = 0; r.item.limit = 0; r.item.duration = 0; r.item.remaining = 0; r.item.remaining_f = 0.0;
  r.item.stamp = 0; r.item.burst = 0; r.item.expire_at = 0; r.item.invalid_at = 0;
}

// Block-wide: records this block filed (every thread of the block must call it).
__device__ __forceinline__ void store_block_count(bool filed, uint32_t* blk) {
  __shared__ uint32_t s_cnt;
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  const uint32_t w = (uint32_t)__popc(__ballot_sync(0xFFFFFFFFu, filed));
  if ((threadIdx.x & 31) == 0 && w) atomicAdd(&s_cnt, w);
  __syncthreads();
  if (threadIdx.x == 0) blk[blockIdx.x] = s_cnt;
}

// ---- where the requests of a pass live ---------------------------------------------------------------------------------------
// The kernels below are written once over an input.  StoreDense: a single table's batch (StoreArgs::reqs / out; a record names its
// requests by batch index).  StoreRing: an owner's pass over its mailbox segments (gub_p2p_step_keys_store_local_all): pass request
// g is record g - off[s] of source s's segment, its response sits in source s's response mailbox, and a record names a request by
// (source shard, index in that source's ingest batch), read from the source's inverse map.  StoreArgs::n is then the launch size
// (world x cap) and the pass size is seg_off[world], written by k_seg_wait.
struct StoreDense {
  const StoreArgs& S;
  __device__ __forceinline__ uint32_t n() const { return S.n; }
  __device__ __forceinline__ bool live(uint32_t) const { return true; }
  __device__ __forceinline__ gub_req req(uint32_t i) const { return S.reqs[i]; }
  __device__ __forceinline__ const gub_req* at(uint32_t i) const { return S.reqs + i; }
  __device__ __forceinline__ uint64_t ld(const uint64_t* p) const { return *p; }
  __device__ __forceinline__ uint32_t behavior(uint32_t i) const { return S.reqs[i].behavior; }
  __device__ __forceinline__ uint32_t err_code(uint32_t i) const { return S.out[i].err_code; }
  __device__ __forceinline__ void name(gub_store_rec&) const {}
};

// The segments of an owner's pass (device pointers of this step's parity; `orig` and `perm` are the sources' memory, read over peer access).
struct StoreSegs {
  uint32_t nseg;
  const uint32_t* seg_off;            // [nseg + 1] prefix sums of the segments (k_seg_wait)
  const gub_req* req[MAX_SHARDS];     // source s's segment of our request mailbox
  const gub_resp* out[MAX_SHARDS];    // our part of source s's response mailbox
  const uint32_t* orig[MAX_SHARDS];   // source s's inverse map, our row: orig[s][pos] = index in s's ingest batch (k_store_orig)
  const uint32_t* perm[MAX_SHARDS];   // source s's routing permutation: perm[s][i] = owner << 24 | pos (k_store_loaded_ring)
};
// The segment table in shared memory: a dynamic index into the kernel parameters would copy them to local memory.
struct StoreSegShared { const gub_req* req[MAX_SHARDS]; const gub_resp* out[MAX_SHARDS]; const uint32_t* orig[MAX_SHARDS]; const uint32_t* perm[MAX_SHARDS]; uint32_t off[MAX_SHARDS + 1]; uint32_t nseg; };

// Block-wide (a barrier): fills the shared segment table.
__device__ __forceinline__ const StoreSegShared* store_segs_open(const StoreSegs& G) {
  __shared__ StoreSegShared s_seg;
#pragma unroll
  for (int k = 0; k < MAX_SHARDS; k++) {
    if (threadIdx.x == (uint32_t)k && (uint32_t)k < G.nseg) { s_seg.req[k] = G.req[k]; s_seg.out[k] = G.out[k]; s_seg.orig[k] = G.orig[k]; s_seg.perm[k] = G.perm[k]; }
  }
  if (threadIdx.x <= G.nseg) s_seg.off[threadIdx.x] = __ldcg(G.seg_off + threadIdx.x);
  if (threadIdx.x == 0) s_seg.nseg = G.nseg;
  __syncthreads();
  return &s_seg;
}

struct StoreRing {
  const StoreArgs& S;
  const StoreSegShared* T;
  __device__ __forceinline__ uint32_t seg_of(uint32_t g) const { uint32_t s = 0; while (s + 1 < T->nseg && g >= T->off[s + 1]) s++; return s; }
  __device__ __forceinline__ const gub_req* at(uint32_t g) const { const uint32_t s = seg_of(g); return T->req[s] + (g - T->off[s]); }
  __device__ __forceinline__ uint32_t n() const { return min(T->off[T->nseg], S.n); }
  __device__ __forceinline__ bool live(uint32_t i) const { return i < n(); }
  // records other GPUs stored into this GPU's memory: L2 is the point of coherence
  __device__ __forceinline__ gub_req req(uint32_t i) const { return load_req_cg(at(i)); }
  __device__ __forceinline__ uint64_t ld(const uint64_t* p) const { return __ldcg(p); }
  __device__ __forceinline__ uint32_t behavior(uint32_t i) const { return __ldcg(&at(i)->behavior); }
  __device__ __forceinline__ uint32_t err_code(uint32_t i) const {
    const uint32_t s = seg_of(i);
    return __ldcg(&T->out[s][i - T->off[s]].err_code);
  }
  // pass indices -> (source shard, index in the source's ingest batch)
  __device__ __forceinline__ void name(gub_store_rec& r) const {
    const uint32_t sf = seg_of(r.first), sl = seg_of(r.last);
    r.first_shard = (uint16_t)sf; r.first = __ldcg(T->orig[sf] + (r.first - T->off[sf]));
    r.last_shard = (uint16_t)sl; r.last = __ldcg(T->orig[sl] + (r.last - T->off[sl]));
  }
};

template <typename In>
__device__ __forceinline__ void store_keys(const StoreArgs& S, const In& in) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= in.n()) return;
  const gub_req rq = in.req(i);
  const uint64_t key = remap_key(rq.key_xxh64), tag = rq.key_fnv1 >> 8;
  const unsigned long long ep = (unsigned long long)S.epoch << 32;
  uint32_t pos = (uint32_t)(key ^ (key >> 31)) & S.key_mask;
#pragma unroll 1
  for (;;) {  // the scratch has 2 x max_batch entries: a free one is always found
    unsigned long long c = __ldcg(&S.keys[pos].claim);
    if ((c >> 32) != (unsigned long long)S.epoch) {
      const unsigned long long old = atomicCAS(&S.keys[pos].claim, c, ep | i);
      if (old == c) break;
      c = old;
    }
    if ((c >> 32) == (unsigned long long)S.epoch) {
      const gub_req* o = in.at((uint32_t)c);
      if (remap_key(in.ld(&o->key_xxh64)) == key && (in.ld(&o->key_fnv1) >> 8) == tag) break;
    }
    pos = (pos + 1) & S.key_mask;
  }
  S.kent[i] = pos;
  atomicMax(&S.keys[pos].first, ep | (0xFFFFFFFFu - i));
  atomicMax(&S.keys[pos].last, ep | i);
  if (rq.algorithm == GUB_TOKEN_BUCKET && (rq.behavior & GUB_BEHAVIOR_RESET_REMAINING)) atomicMax(&S.keys[pos].reset, ep | 1u);
}

template <typename In>
__device__ __forceinline__ void store_before(const StoreArgs& S, const In& in) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool filed = false;
  if (i < S.n) {
    if (in.live(i)) {
      const StoreKey k = S.keys[S.kent[i]];
      if (skey_first(k) == i) {
        const gub_req rq = in.req(i);
        Bucket b;
        int64_t inv_at;
        const bool found = store_lookup(S, remap_key(rq.key_xxh64), rq.key_fnv1 >> 8, b, inv_at);
        S.bstate[i] = StoreState{found ? S_EXISTED : 0u, (b.flags & F_LEAKY) ? (uint32_t)GUB_LEAKY_BUCKET : (uint32_t)GUB_TOKEN_BUCKET};
        if (!found && S.want_misses) {
          gub_store_rec r;
          store_rec_init(r, i, (uint32_t)k.last, 0u, rq);
          in.name(r);
          S.sparse[i] = r;
          filed = true;
        }
      }
    }
    S.sel[i] = filed ? 1 : 0;
  }
  store_block_count(filed, S.blk);
}

template <typename In>
__device__ __forceinline__ void store_after(const StoreArgs& S, const In& in) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool filed = false;
  if (i < S.n) {
    if (in.live(i)) {
      const StoreKey k = S.keys[S.kent[i]];
      if (skey_first(k) == i) {
        const gub_req rq = in.req(i);
        const uint32_t last = (uint32_t)k.last;
        Bucket b;
        int64_t inv_at;
        const bool live = store_lookup(S, remap_key(rq.key_xxh64), rq.key_fnv1 >> 8, b, inv_at);
        const StoreState bs = S.bstate[i];
        // Store.Remove (algorithms.go:78-83, 91-100, 308-315): the item that existed was deleted
        const bool switched = (int32_t)bs.algorithm != (int32_t)rq.algorithm && rq.algorithm <= 1u;
        const bool reset = k.reset == (((unsigned long long)S.epoch << 32) | 1ull);
        // Store.OnChange (algorithms.go:149, 252): owner requests only
        const bool change = live && in.err_code(last) == 0 && (in.behavior(last) & GUB_REQ_IS_OWNER);
        const uint32_t flags = ((bs.existed & S_EXISTED) && (switched || reset) ? (uint32_t)GUB_STORE_REMOVE : 0u) | (change ? (uint32_t)GUB_STORE_CHANGE : 0u);
        if (flags) {
          gub_store_rec r;
          store_rec_init(r, i, last, flags, rq);
          if (change) {
            store_item(b, inv_at, r.item);
            r.item.key_xxh64 = rq.key_xxh64; r.item.key_fnv1 = rq.key_fnv1;
          }
          in.name(r);
          S.sparse[i] = r;
          filed = true;
        }
      }
    }
    S.sel[i] = filed ? 1 : 0;
  }
  store_block_count(filed, S.blk);
}

// Single table (gub_submit_keys_store_async).
__global__ void __launch_bounds__(STORE_THREADS) k_store_keys(const StoreArgs S) { store_keys(S, StoreDense{S}); }
__global__ void __launch_bounds__(STORE_THREADS) k_store_before(const StoreArgs S) { store_before(S, StoreDense{S}); }
__global__ void __launch_bounds__(STORE_THREADS) k_store_after(const StoreArgs S) { store_after(S, StoreDense{S}); }

// loaded[k] = (first, existed, algorithm, -) for the items Store.Get returned
__global__ void __launch_bounds__(STORE_THREADS) k_store_loaded(const uint4* loaded, uint32_t m, StoreState* bstate) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= m) return;
  const uint4 l = loaded[k];
  bstate[l.x] = StoreState{l.y, l.z};
}

// An owner's pass over its mailbox segments (gub_p2p_step_keys_store_local_all); S.n = world x cap, the grid's size.
__global__ void __launch_bounds__(STORE_THREADS) k_store_keys_ring(const StoreArgs S, const StoreSegs G) { store_keys(S, StoreRing{S, store_segs_open(G)}); }
__global__ void __launch_bounds__(STORE_THREADS) k_store_before_ring(const StoreArgs S, const StoreSegs G) { store_before(S, StoreRing{S, store_segs_open(G)}); }
__global__ void __launch_bounds__(STORE_THREADS) k_store_after_ring(const StoreArgs S, const StoreSegs G) { store_after(S, StoreRing{S, store_segs_open(G)}); }

// loaded[k] = (first, existed, algorithm, first_shard) for the items Store.Get returned: the record names the key's first request by
// source, so the pass index is found through that source's routing permutation (pass index = seg_off[s] + its mailbox position).
__global__ void __launch_bounds__(STORE_THREADS) k_store_loaded_ring(const uint4* loaded, uint32_t m, StoreState* bstate, const StoreSegs G) {
  const StoreSegShared* T = store_segs_open(G);
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= m) return;
  const uint4 l = loaded[k];
  const uint32_t g = T->off[l.w] + (__ldcg(T->perm[l.w] + l.x) & 0xFFFFFFu);
  bstate[g] = StoreState{l.y, l.z};
}

// Source side of a ring Store step, after its routing: orig[o * cap + pos] = i for every perm[i] = o << 24 | pos, so that owner o can
// name the request it finds at position pos of our segment.
__global__ void __launch_bounds__(256) k_store_orig(const uint32_t* perm, uint32_t n, uint32_t cap, uint32_t* orig) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t pk = __ldg(perm + i);
  orig[(size_t)(pk >> 24) * cap + (pk & 0xFFFFFFu)] = i;
}

// gub_store_rec's layout in 32-bit words and above.
struct StoreRecWords { uint32_t first, last, flags, shards; gub_item item; };
static_assert(sizeof(StoreRecWords) == sizeof(gub_store_rec), "gub_store_rec layout");

// out[0 .. *out_count) = the filed records in index order.  Same grid as the pass that filed them.
__global__ void __launch_bounds__(STORE_THREADS) k_store_compact(const uint8_t* sel, const gub_store_rec* sparse, const uint32_t* blk, uint32_t n,
                                                                 gub_store_rec* out, uint32_t* out_count) {
  __shared__ uint32_t s_part[STORE_THREADS / 32], s_wcnt[STORE_THREADS / 32];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t part = 0;
  for (uint32_t b = threadIdx.x; b < blockIdx.x; b += blockDim.x) part += __ldg(blk + b);
  part = __reduce_add_sync(0xFFFFFFFFu, part);
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool p = i < n && __ldg(sel + i) != 0;
  const uint32_t bal = __ballot_sync(0xFFFFFFFFu, p);
  if (lane == 0) { s_part[warp] = part; s_wcnt[warp] = (uint32_t)__popc(bal); }
  __syncthreads();
  uint32_t base = 0, before = 0, total = 0;
  for (uint32_t w = 0; w < (uint32_t)(STORE_THREADS / 32); w++) {
    base += s_part[w];
    if (w < warp) before += s_wcnt[w];
    total += s_wcnt[w];
  }
  if (p) {  // copied as whole 32-bit words (first_shard / last_shard are the two halves of one): 16-bit moves would cost more instructions
    const StoreRecWords* src = reinterpret_cast<const StoreRecWords*>(sparse) + i;
    reinterpret_cast<StoreRecWords*>(out)[base + before + (uint32_t)__popc(bal & ((1u << lane) - 1u))] = *src;
  }
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) *out_count = base + total;
}

}  // namespace gub
