// gub_kernels.cuh — sm_90a kernels of the rate-limit evaluation path.
//
// Replaces, for a whole batch at a time, WorkerPool.GetRateLimit -> Worker.handleGetRateLimit -> LRUCache.GetItem ->
// tokenBucket/leakyBucket (workers.go:261-324, lrucache.go:111, algorithms.go:37-493 of mailgun/gubernator v2.4.0).
//
// Data layout in HBM
//   table    : capacity x 64-byte slots, open addressing with linear probing from home = mulhi(key, capacity):
//              w0 key (XXH64, remapped off the two sentinels)   w1 tag(FNV-1 >> 8) << 8 | flags
//              w2 limit  w3 duration  w4 remaining (int64 | float64 bits)  w5 stamp  w6 burst  w7 expire_at
//   requests : n x 64 B gub_req (AoS, what the Go shim fills), responses: n x 32 B gub_resp
//
// The reference applies same-key requests strictly in index order (gubernator.go:203) and the updates do not commute,
// so what every request needs is (a) how many requests of the batch share its key and (b) its RANK among them in index
// order.  With those, a run of identical requests needs no ordering structure at all: every member evaluates
// run_to_rank(bucket, request, rank) by itself (closed forms make that O(1)), and the member holding the last rank
// writes the bucket back.  Only runs whose requests differ are materialised in rank order and walked segment by segment.
//
//   k_group  (256 consecutive requests per block) shared-memory grouping with index-ordered local ranks; one thread per
//            distinct (block, key) "fragment" joins the batch-wide group entry (count += members), sets the block's bit
//            in the group's presence bitmap and stores the fragment size.  Prefetches every request's home slot into L2.
//   k_rank   members of repeated keys get rank = (sum of earlier blocks' fragment sizes) + local rank and compare their
//            request with the group's representative; any difference marks the group non-uniform.  Keys seen once — most keys —
//            are evaluated right here (probe, apply_one, write-back, response) and the rank-0 member of a repeated key parks the
//            slot as found in a snapshot.
//   k_eval   every member of a uniform run evaluates run_to_rank(snapshot, request, rank) and answers; the last rank writes
//            the slot back.  Members of non-uniform runs only file themselves: order[base + rank] = index.
//   k_finish one block per non-uniform group: split the ordered run into segments of identical requests, plan each with
//            plan_run() on one thread, evaluate/scatter with all threads (serial walk when there are too many segments).
// The four kernels are chained with programmatic dependent launch (consecutive batches overlap: the small, high-occupancy kernels of
// batch b+1 start while the tail of batch b drains — this pipeline's throughput advantage over the single persistent kernel of
// gub_batch.cuh); block requests are partitioned by algorithm so that a warp runs one bucket algorithm's code path.
#pragma once
#if !defined(GUB_EMULATE)  // tests/kernel_emu_harness.cpp compiles this header for the CPU on top of tests/cuda_emu.h
#include <cuda_runtime.h>
#endif
#include <stdint.h>

#include "bucket_math.cuh"

namespace gub {

constexpr uint64_t KEY_EMPTY = 0ull;
constexpr uint64_t KEY_TOMB = 1ull;
constexpr int MAX_PROBE = 512;       // window [home, home + MAX_PROBE): inserts never leave it, so lookups may stop there
constexpr int GROUP_THREADS = 256;   // requests per block in k_group / k_rank (a "fragment" is one key's members in one block)
constexpr int GROUP_SLOTS = 512;     // shared-memory table entries per block (load factor <= 0.5)
constexpr int MIXED_THREADS = 256;
constexpr int MAX_PIECES = 16;
constexpr int MAX_SHARDS = 16;       // GPUs of one ring (= most mailbox segments a batch is made of)

struct __align__(64) Slot { uint64_t w[8]; };

struct __align__(32) AuxEntry {
  unsigned long long word;  // [63:48] epoch  [47:24] key tag  [23:0] member count
  uint32_t rep;             // index of one member (the claimer's first): the request every other member is compared with
  uint32_t flags;           // AUX_NONUNIFORM
  uint32_t gbase;           // non-uniform groups: start of the group's region in `order`
  uint32_t _pad[3];
};
constexpr uint32_t AUX_NONUNIFORM = 1u;
__host__ __device__ inline uint32_t aux_count(unsigned long long w) { return (uint32_t)(w & 0xFFFFFFull); }
__host__ __device__ inline uint32_t aux_epoch(unsigned long long w) { return (uint32_t)(w >> 48); }
__host__ __device__ inline uint32_t aux_tag(unsigned long long w) { return (uint32_t)((w >> 24) & 0xFFFFFFull); }

struct BatchCtr { uint32_t n_mixed, order_bump, next_mixed, _pad1; };

// Items whose insert found the probe window full are parked here and placed — evicting the entry of the window that expires first,
// like the reference's LRU would have evicted (lrucache.go:98,138-149) — before the next batch reads the table.
constexpr int OVF_CAP = 1024;
struct OvfItem { uint64_t key, tag; uint64_t w[6]; uint32_t flags, _pad; };  // 72 bytes
struct InvEntry { unsigned long long key, tag; long long invalid_at, _pad; };
struct InvIndex { InvEntry* e; uint32_t mask; };

enum { C_OVER = 0, C_HIT, C_MISS, C_INSERTS, C_FULL, C_REQUESTS, C_BATCHES, C_DUP_GROUPS, C_MIXED_GROUPS, C_SERIAL, C_EVICT_UNEXPIRED, C_SWEPT, C_GQ_DROPPED,
       C_COUNT };

struct BatchArgs {
  Slot* table;
  uint64_t capacity;
  const gub_req* reqs;
  gub_resp* out;
  uint32_t n;              // requests in this launch (grid size); with n_dev: the most this launch may hold
  const uint32_t* n_dev;   // optional: the batch size lives on the device (fused routing: known only after the gather kernel);
  uint32_t n_off;          //           this launch then covers requests [n_off, min(*n_dev, n_off + n)) of the batch
  uint32_t epoch;          // 1..65535
  AuxEntry* aux;
  uint32_t aux_mask;       // entries - 1 (power of two)
  uint32_t* presence;      // [entries * pres_words] bit b set <=> block b holds a fragment of the group; all zero between batches
  uint8_t* fragsize;       // [entries * max_blocks] fragment size - 1, valid where the presence bit is set
  uint32_t pres_words, max_blocks;
  uint32_t* ent;           // [n] group entry of request i
  uint32_t* meta;          // [n] (shared-memory slot of the fragment << 16) | local rank
  uint32_t* rank;          // [n] rank within the group (repeated keys only)
  ulonglong2* commit;      // [entries * 6] repeated keys: the slot as the run's rank-0 member found it (snapshot for its siblings)
  uint32_t* order;         // [max_batch] rank-ordered member indices of non-uniform groups
  uint32_t* mixed_ent;     // [max_batch / 2] entries of non-uniform groups
  BatchCtr* ctr;           // [2], indexed by epoch parity
  unsigned long long* counters;  // [C_COUNT]
  OvfItem* ovf;            // [OVF_CAP] parked inserts
  uint32_t* ovf_count;
  InvIndex inv;            // CacheItem.InvalidAt side index
  // Ring mode (gub_p2p): the batch is the concatenation, in source order, of `nseg` mailbox segments filled by the ring's shards over
  // NVLink; request g of the batch is seg_reqs[s][g - seg_off[s]] and its response goes to seg_out[s][g - seg_off[s]] (the source's
  // response mailbox: peer memory).  seg_off (device, nseg + 1 prefix sums) is written by k_seg_wait once every source's flag has
  // arrived; n_dev points at seg_off[nseg].  nseg == 0: one dense array (reqs / out).
  uint32_t nseg;
  const uint32_t* seg_off;
  const gub_req* seg_reqs[MAX_SHARDS];
  gub_resp* seg_out[MAX_SHARDS];
  unsigned long long* ktrace;  // optional (diagnostic, gub_set_trace): [4 kernels][KT_BLOCKS][KT_MARKS] latest %globaltimer at which a warp / a thread in a role passed a mark
  // Early hand-off (single table, see k_group): *chain_done = epoch of the last batch whose k_finish block 0 has left (it stores the
  // epoch last); early_ok = this batch's grouping scratch is not the previous batch's (two scratch sets) and epoch > 1.  chain_done may be null.
  uint32_t* chain_done;
  uint32_t early_ok;
  uint32_t* mixed_hint;    // optional, host-mapped: k_eval copies the batch's count of non-uniform groups here (sizes later k_finish grids)
  gub_clock clk;
};
constexpr int KT_MARKS = 8, KT_BLOCKS = 1024;
enum { KT_ENTRY = 0, KT_WAITED, KT_M2, KT_M3, KT_M4, KT_M5, KT_WORK_DONE, KT_EXIT };

__device__ __forceinline__ uint64_t remap_key(uint64_t k) { return k < 2 ? k + 2 : k; }

// Number of requests this launch evaluates (see BatchArgs::n_dev).
__device__ __forceinline__ uint32_t batch_n(const BatchArgs& A) {
  if (!A.n_dev) return A.n;
  const uint32_t total = __ldcg(A.n_dev);
  return total > A.n_off ? min(total - A.n_off, A.n) : 0u;
}

// Programmatic dependent launch (sm_90+): every batch kernel is launched with programmatic stream serialization, so its
// blocks may become resident while the previous kernel is still running.  pdl_wait() blocks until every earlier grid of
// the stream has completed and its writes are visible; only work that depends on nothing earlier may precede it.
// pdl_release() then lets the NEXT kernel start launching (after our wait, so that kernel may read anything that was
// complete before this one started, e.g. the request records).
#if defined(GUB_EMULATE)
__device__ __forceinline__ void pdl_wait() {}
__device__ __forceinline__ void pdl_release() {}
__device__ __forceinline__ void prefetch_l2(const void*) {}
#else
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_release() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
#endif


// Diagnostic time stamps (see BatchArgs::ktrace).  `dep`: a value the stamp must wait for (a load's result).  all = every calling thread
// stamps (marks inside divergent role code), else lane 0 of each warp.
#if defined(GUB_EMULATE)
#define KT(A, kernel, mark, dep, all) do { } while (0)
#else
__device__ __forceinline__ void kt_stamp(unsigned long long* ktrace, int kernel, int mark, uint32_t dep, bool all) {
  if (ktrace && (all || (threadIdx.x & 31) == 0) && blockIdx.x < 1024u) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t) : "r"(dep) : "memory");
    atomicMax(&ktrace[((size_t)kernel * 1024u + blockIdx.x) * 8u + (uint32_t)mark], t);
  }
}
#define KT(A, kernel, mark, dep, all) kt_stamp((A).ktrace, kernel, mark, (uint32_t)(dep), all)
#endif

// system-scope release / acquire on flags other GPUs (or the host) poll; gpu-scope ones on words only this device's kernels use
#if defined(GUB_EMULATE)
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) { *p = v; }
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) { return *p; }
__device__ __forceinline__ void st_release_gpu(uint32_t* p, uint32_t v) { *p = v; }
__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* p) { return *p; }
__device__ __forceinline__ void __nanosleep(unsigned) { emu::spin_yield(); }
#else
__device__ __forceinline__ void st_release_gpu(uint32_t* p, uint32_t v) { asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
#endif

// ---- slot access ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void slot_load(const Slot* s, ulonglong2& a, ulonglong2& b, ulonglong2& c, ulonglong2& d) {
  const ulonglong2* p = reinterpret_cast<const ulonglong2*>(s);
  a = __ldcg(p); b = __ldcg(p + 1); c = __ldcg(p + 2); d = __ldcg(p + 3);  // 4 x 128-bit, L2-only (no reuse in L1)
}
__device__ __forceinline__ void bucket_from(Bucket& bk, const ulonglong2& a, const ulonglong2& b, const ulonglong2& c, const ulonglong2& d) {
  bk.key = a.x; bk.tag = a.y >> 8; bk.flags = (uint32_t)(a.y & 0xFF);
  bk.limit = (int64_t)b.x; bk.duration = (int64_t)b.y; bk.rem = c.x; bk.stamp = (int64_t)c.y;
  bk.burst = (int64_t)d.x; bk.expire = (int64_t)d.y;
}

struct Cursor {  // one key's slot while requests are applied to it
  Bucket b, old;
  int64_t slot;      // slot index when found, else first free slot in the probe window (or -1)
  uint64_t home;
  bool found;
};

// CacheItem.InvalidAt (cache.go:40,47) is only ever set by Store / Loader plugins, so it does not get a word of the 64-byte
// slot: slots that have one carry F_INVALID_AT and the value sits in a small side index (open addressing by key, a few probes;
// a full neighbourhood overwrites its home entry: the item then merely falls back to ExpireAt).
constexpr int INV_PROBES = 16;
__device__ __forceinline__ int64_t inv_lookup(const InvIndex& I, uint64_t key, uint64_t tag) {
  uint32_t pos = (uint32_t)(key ^ (key >> 33)) & I.mask;
  for (int p = 0; p < INV_PROBES; p++) {
    const unsigned long long k = __ldcg(&I.e[pos].key);
    if (k == key && __ldcg(&I.e[pos].tag) == tag) return (int64_t)__ldcg(&I.e[pos].invalid_at);
    if (k == 0ull) break;
    pos = (pos + 1) & I.mask;
  }
  return 0;
}
__device__ __forceinline__ void inv_store(const InvIndex& I, uint64_t key, uint64_t tag, int64_t invalid_at) {
  const uint32_t home = (uint32_t)(key ^ (key >> 33)) & I.mask;
  uint32_t pos = home;
  for (int p = 0; p < INV_PROBES; p++) {
    const unsigned long long old = atomicCAS(&I.e[pos].key, 0ull, (unsigned long long)key);
    if (old == 0ull || (old == key && I.e[pos].tag == tag) || old == key) { I.e[pos].tag = tag; I.e[pos].invalid_at = invalid_at; return; }
    pos = (pos + 1) & I.mask;
  }
  I.e[home].key = key; I.e[home].tag = tag; I.e[home].invalid_at = invalid_at;
}
// IsExpired's first clause: an item past its InvalidAt counts as expired.  The bucket is marked F_STALE; the first request that
// reaches the cache (apply_one, past the algorithm check) removes it and reports a miss, one with a rejected algorithm leaves it.
__device__ __forceinline__ void apply_invalid_at(const InvIndex& I, Bucket& b, bool found, int64_t now_ms) {
  if (found && (b.flags & F_INVALID_AT)) {
    const int64_t inv = inv_lookup(I, b.key, b.tag);
    if (inv != 0 && inv < now_ms) b.flags |= F_STALE;
  }
}

// Slots past home whose (w0, w1) pairs one probe round loads at once.  A lookup walks slots home, home + 1, ... (mod capacity) and
// stops at the key, at the first EMPTY or after MAX_PROBE slots; at load factor 0.5 a quarter of the lookups need more than the home
// slot and the longest lookup of a 22 k-key batch about 25 slots (DESIGN.md, "The table probe in rounds").  Loading one slot after the
// other made that a chain of dependent round trips that the whole batch waits for; a round puts PROBE_ROUND independent 16-byte loads
// in flight instead.  4, not 8: rounds of 8 made k_rank spill.
constexpr int PROBE_ROUND = 4;

// Looks `key` up.  On a hit the slot is loaded into cur.b.  On a miss cur.b is an empty (not live) bucket and cur.slot
// is the first reusable slot (tombstone or empty) seen, if any.
// (The home slot's four words arrive in a..d: callers that know the key early issue that load ahead of other work.)
__device__ __forceinline__ void cursor_open_preloaded(Cursor& cur, const Slot* table, uint64_t cap, uint64_t key, uint64_t tag, ulonglong2 a, ulonglong2 b,
                                                      ulonglong2 c, ulonglong2 d) {
  uint64_t idx = __umul64hi(key, cap);
  cur.home = idx; cur.found = false; cur.slot = -1;
  bool hit = a.x == key && (a.y >> 8) == tag;
  if (!hit && a.x == KEY_EMPTY) cur.slot = (int64_t)idx;
  if (!hit && a.x != KEY_EMPTY) {
    if (a.x == KEY_TOMB) cur.slot = (int64_t)idx;
    bool done = false;
#pragma unroll 1
    for (int p = 1; p < MAX_PROBE && !done; p += PROBE_ROUND) {
      // every index wraps by itself: a table may be smaller than one round (the slots past the window are loaded, never examined)
      ulonglong2 w[PROBE_ROUND];
      uint64_t j = idx;
#pragma unroll
      for (int r = 0; r < PROBE_ROUND; r++) {
        j = (j + 1 == cap) ? 0 : j + 1;
        w[r] = __ldcg(reinterpret_cast<const ulonglong2*>(table + j));
      }
      // the same rules as for the home slot, in probe order
#pragma unroll
      for (int r = 0; r < PROBE_ROUND; r++) {
        if (p + r >= MAX_PROBE) { done = true; break; }
        idx = (idx + 1 == cap) ? 0 : idx + 1;
        if (w[r].x == key && (w[r].y >> 8) == tag) { a = w[r]; hit = true; done = true; break; }
        if (w[r].x == KEY_EMPTY) { if (cur.slot < 0) cur.slot = (int64_t)idx; done = true; break; }
        if (w[r].x == KEY_TOMB && cur.slot < 0) cur.slot = (int64_t)idx;
      }
    }
    if (hit) {  // the rest of the slot: its first sector came with the pair, so this mostly hits L2
      const ulonglong2* s = reinterpret_cast<const ulonglong2*>(table + idx);
      b = __ldcg(s + 1); c = __ldcg(s + 2); d = __ldcg(s + 3);
    }
  }
  if (hit) {
    bucket_from(cur.b, a, b, c, d);
    cur.old = cur.b; cur.slot = (int64_t)idx; cur.found = true;
    return;
  }
  cur.b.key = key; cur.b.tag = tag; cur.b.flags = 0; cur.b.limit = 0; cur.b.duration = 0; cur.b.rem = 0; cur.b.stamp = 0;
  cur.b.burst = 0; cur.b.expire = 0;
  cur.old = cur.b;
}
__device__ __forceinline__ void cursor_open(Cursor& cur, const Slot* table, uint64_t cap, uint64_t key, uint64_t tag) {
  ulonglong2 a, b, c, d;
  slot_load(table + __umul64hi(key, cap), a, b, c, d);
  cursor_open_preloaded(cur, table, cap, key, tag, a, b, c, d);
}

// Writes cur.b back.  Returns false when a new key needed a slot and the probe window had none (table full).
__device__ __forceinline__ bool cursor_close(Cursor& cur, Slot* table, uint64_t cap, uint32_t& inserts) {
  const Bucket& b = cur.b;
  const uint32_t flags = b.flags & ~(uint32_t)F_STALE;  // (a mark of this batch, not slot state)
  const uint64_t w1 = (b.tag << 8) | (uint64_t)(flags & 0xFF);
  if (cur.found) {
    ulonglong2* p = reinterpret_cast<ulonglong2*>(table + cur.slot);
    if (flags != (cur.old.flags & ~(uint32_t)F_STALE)) __stcg(p, make_ulonglong2(b.key, w1));
    if (b.limit != cur.old.limit || b.duration != cur.old.duration) __stcg(p + 1, make_ulonglong2((uint64_t)b.limit, (uint64_t)b.duration));
    if (b.rem != cur.old.rem || b.stamp != cur.old.stamp) __stcg(p + 2, make_ulonglong2(b.rem, (uint64_t)b.stamp));
    if (b.burst != cur.old.burst || b.expire != cur.old.expire) __stcg(p + 3, make_ulonglong2((uint64_t)b.burst, (uint64_t)b.expire));
    return true;
  }
  if (!(b.flags & F_LIVE)) return true;  // nothing was created
  // claim a slot inside the probe window, starting at the first reusable one seen
  if (cur.slot < 0) return false;
  uint64_t idx = (uint64_t)cur.slot;
  uint64_t dist = idx >= cur.home ? idx - cur.home : idx + cap - cur.home;
#pragma unroll 1
  for (; dist < (uint64_t)MAX_PROBE; dist++) {
    unsigned long long* w0 = reinterpret_cast<unsigned long long*>(&table[idx].w[0]);
    unsigned long long seen = __ldcg(w0);
    if (seen == KEY_EMPTY || seen == KEY_TOMB) {
      if (atomicCAS(w0, seen, (unsigned long long)b.key) == seen) {
        ulonglong2* p = reinterpret_cast<ulonglong2*>(table + idx);
        // w0 is already the key; writing the pair again stores the same value
        __stcg(p, make_ulonglong2(b.key, w1));
        __stcg(p + 1, make_ulonglong2((uint64_t)b.limit, (uint64_t)b.duration));
        __stcg(p + 2, make_ulonglong2(b.rem, (uint64_t)b.stamp));
        __stcg(p + 3, make_ulonglong2((uint64_t)b.burst, (uint64_t)b.expire));
        cur.slot = (int64_t)idx; cur.found = true; cur.old = cur.b;
        inserts++;
        return true;
      }
    }
    idx = (idx + 1 == cap) ? 0 : idx + 1;
  }
  return false;
}

// A repeated key's final state, parked in scratch by the run's last rank: its siblings read the slot during k_eval, so the
// table itself is only written by k_finish.  `who` = request index of the writer (its response reports a full table).
__device__ __forceinline__ void snap_store(ulonglong2* sp, const Cursor& c, uint32_t who) {
  __stcg(sp + 0, make_ulonglong2(c.b.key, c.b.tag));
  __stcg(sp + 1, make_ulonglong2((uint64_t)c.b.limit, (uint64_t)c.b.duration));
  __stcg(sp + 2, make_ulonglong2(c.b.rem, (uint64_t)c.b.stamp));
  __stcg(sp + 3, make_ulonglong2((uint64_t)c.b.burst, (uint64_t)c.b.expire));
  __stcg(sp + 4, make_ulonglong2((uint64_t)c.b.flags | ((uint64_t)(c.found ? 1u : 0u) << 32), (uint64_t)c.slot));
  __stcg(sp + 5, make_ulonglong2(c.home, (uint64_t)who));
}
__device__ __forceinline__ uint32_t snap_unpack(const ulonglong2& a, const ulonglong2& b, const ulonglong2& d, const ulonglong2& e, const ulonglong2& f,
                                                const ulonglong2& g, Cursor& c);
__device__ __forceinline__ uint32_t snap_load(const ulonglong2* sp, Cursor& c) {
  const ulonglong2 a = __ldcg(sp + 0), b = __ldcg(sp + 1), d = __ldcg(sp + 2), e = __ldcg(sp + 3), f = __ldcg(sp + 4), g = __ldcg(sp + 5);
  return snap_unpack(a, b, d, e, f, g, c);
}
__device__ __forceinline__ uint32_t snap_unpack(const ulonglong2& a, const ulonglong2& b, const ulonglong2& d, const ulonglong2& e, const ulonglong2& f,
                                                const ulonglong2& g, Cursor& c) {
  c.b.key = a.x; c.b.tag = a.y; c.b.limit = (int64_t)b.x; c.b.duration = (int64_t)b.y; c.b.rem = d.x; c.b.stamp = (int64_t)d.y;
  c.b.burst = (int64_t)e.x; c.b.expire = (int64_t)e.y; c.b.flags = (uint32_t)(f.x & 0xFFFFFFFFull); c.found = (f.x >> 32) != 0;
  c.slot = (int64_t)f.y; c.home = g.x; c.old = c.b;
  return (uint32_t)g.y;
}

struct Tally { uint32_t over, hit, miss, inserts, full; };

// Writes a key's final state.  A new key whose probe window has no free slot is parked (see OvfItem).
__device__ __forceinline__ void close_or_park(Cursor& cur, Slot* table, uint64_t cap, OvfItem* ovf, uint32_t* ovf_count, Tally& t) {
  if (cursor_close(cur, table, cap, t.inserts)) return;
  const uint32_t k = atomicAdd(ovf_count, 1u);
  if (k < (uint32_t)OVF_CAP) {
    OvfItem it;
    it.key = cur.b.key; it.tag = cur.b.tag; it.flags = cur.b.flags; it._pad = 0;
    it.w[0] = (uint64_t)cur.b.limit; it.w[1] = (uint64_t)cur.b.duration; it.w[2] = cur.b.rem; it.w[3] = (uint64_t)cur.b.stamp;
    it.w[4] = (uint64_t)cur.b.burst; it.w[5] = (uint64_t)cur.b.expire;
    ovf[k] = it;
  } else {
    t.full++;  // more than OVF_CAP keys without a slot in one batch: the state of this one is dropped (counted)
  }
}

// One warp places the parked items, evicting when the window is still full.  Runs when nothing reads the table.
__device__ __noinline__ void drain_parked(Slot* table, uint64_t capacity, OvfItem* ovf, uint32_t* ovf_count, int64_t now_ms, unsigned long long* counters,
                                          uint32_t* inserts) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t n = min(__ldcg(ovf_count), (uint32_t)OVF_CAP);
#pragma unroll 1
  for (uint32_t k = 0; k < n; k++) {
    const OvfItem it = ovf[k];
    const uint64_t home = __umul64hi(it.key, capacity);
    // every lane inspects 16 slots of the window: best = the key itself, else free, else removed / expired, else the smallest ExpireAt
    uint64_t best_rank = ~0ull, best_idx = 0;
#pragma unroll 1
    for (uint32_t p = lane; p < (uint32_t)MAX_PROBE; p += 32) {
      const uint64_t idx = (home + p) % capacity;  // (a table smaller than the window wraps more than once)
      const ulonglong2 a = __ldcg(reinterpret_cast<const ulonglong2*>(table + idx));
      const int64_t exp = (int64_t)__ldcg(&table[idx].w[7]);
      uint64_t rank;
      if (a.x == it.key && (a.y >> 8) == it.tag) rank = 0;
      else if (a.x <= KEY_TOMB) rank = 1;
      else if (!(a.y & F_LIVE) || exp < now_ms) rank = 2;
      else rank = 3 + ((uint64_t)exp ^ 0x8000000000000000ull) / 4;  // live: earliest ExpireAt first
      rank = (rank << 9) | (uint64_t)p;                               // ties: nearest to home
      if (rank < best_rank) { best_rank = rank; best_idx = idx; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const uint64_t r2 = __shfl_sync(0xFFFFFFFFu, (unsigned long long)best_rank, lane ^ o), i2 = __shfl_sync(0xFFFFFFFFu, (unsigned long long)best_idx, lane ^ o);
      if (r2 < best_rank) { best_rank = r2; best_idx = i2; }
    }
    if (lane == 0) {
      if ((best_rank >> 9) >= 3) atomicAdd(counters + C_EVICT_UNEXPIRED, 1ull);
      if ((best_rank >> 9) >= 1) (*inserts)++;
      ulonglong2* p = reinterpret_cast<ulonglong2*>(table + best_idx);
      __stcg(p, make_ulonglong2(it.key, (it.tag << 8) | (uint64_t)(it.flags & 0xFF)));
      __stcg(p + 1, make_ulonglong2(it.w[0], it.w[1]));
      __stcg(p + 2, make_ulonglong2(it.w[2], it.w[3]));
      __stcg(p + 3, make_ulonglong2(it.w[4], it.w[5]));
    }
    __syncwarp();
  }
  if (lane == 0 && n) *ovf_count = 0;
}

__device__ __forceinline__ gub_req load_req(const gub_req* p) {
  const ulonglong2* q = reinterpret_cast<const ulonglong2*>(p);
  ulonglong2 a = __ldg(q), b = __ldg(q + 1), c = __ldg(q + 2), d = __ldg(q + 3);
  gub_req r;
  r.key_xxh64 = a.x; r.key_fnv1 = a.y; r.hits = (int64_t)b.x; r.limit = (int64_t)b.y; r.duration = (int64_t)c.x;
  r.burst = (int64_t)c.y; r.created_at = (int64_t)d.x; r.algorithm = (uint32_t)(d.y & 0xFFFFFFFFull); r.behavior = (uint32_t)(d.y >> 32);
  return r;
}
__device__ __forceinline__ void store_resp(gub_resp* p, const gub_resp& r) {
  ulonglong2* q = reinterpret_cast<ulonglong2*>(p);
  __stcs(q, make_ulonglong2((uint64_t)r.status | ((uint64_t)r.err_code << 32), (uint64_t)r.limit));
  __stcs(q + 1, make_ulonglong2((uint64_t)r.remaining, (uint64_t)r.reset_time));
}

__device__ __forceinline__ gub_req load_req_cg(const gub_req* p) {  // records other GPUs stored into this GPU's memory: L2 is the point of coherence
  const ulonglong2* q = reinterpret_cast<const ulonglong2*>(p);
  ulonglong2 a = __ldcg(q), b = __ldcg(q + 1), c = __ldcg(q + 2), d = __ldcg(q + 3);
  gub_req r;
  r.key_xxh64 = a.x; r.key_fnv1 = a.y; r.hits = (int64_t)b.x; r.limit = (int64_t)b.y; r.duration = (int64_t)c.x;
  r.burst = (int64_t)c.y; r.created_at = (int64_t)d.x; r.algorithm = (uint32_t)(d.y & 0xFFFFFFFFull); r.behavior = (uint32_t)(d.y >> 32);
  return r;
}

// Where request i of this launch lives and where its response goes.  SEG = false: the dense arrays of BatchArgs.  SEG = true (ring
// mode): the batch is a concatenation of mailbox segments; the segment table sits in shared memory (io_open).
struct SegShared { const gub_req* req[MAX_SHARDS]; gub_resp* out[MAX_SHARDS]; uint32_t off[MAX_SHARDS + 1]; uint32_t nseg; };
template <bool SEG>
struct Io {
  const BatchArgs& A;
  const SegShared* S;
  __device__ __forceinline__ uint32_t seg_of(uint32_t g) const { uint32_t s = 0; while (s + 1 < S->nseg && g >= S->off[s + 1]) s++; return s; }
  __device__ __forceinline__ const gub_req* req(uint32_t i) const {
    if constexpr (!SEG) { return A.reqs + i; }
    else { const uint32_t g = A.n_off + i, s = seg_of(g); return S->req[s] + (g - S->off[s]); }
  }
  __device__ __forceinline__ gub_resp* resp(uint32_t i) const {
    if constexpr (!SEG) { return A.out + i; }
    else { const uint32_t g = A.n_off + i, s = seg_of(g); return S->out[s] + (g - S->off[s]); }
  }
  __device__ __forceinline__ gub_req load(uint32_t i) const {
    if constexpr (!SEG) return load_req(A.reqs + i); else return load_req_cg(req(i));
  }
  __device__ __forceinline__ uint64_t key(uint32_t i) const {
    if constexpr (!SEG) return __ldg(&A.reqs[i].key_xxh64); else return __ldcg(&req(i)->key_xxh64);
  }
  __device__ __forceinline__ uint32_t algorithm(uint32_t i) const {
    if constexpr (!SEG) return __ldg(&A.reqs[i].algorithm); else return __ldcg(&req(i)->algorithm);
  }
};
// Block-wide (SEG: fills the shared segment table and contains a barrier; seg_off must be final, i.e. k_seg_wait has completed).
template <bool SEG>
__device__ __forceinline__ Io<SEG> io_open(const BatchArgs& A) {
  if constexpr (SEG) {
    __shared__ SegShared s_seg;
#pragma unroll
    for (int k = 0; k < MAX_SHARDS; k++) {  // static indices: a dynamic index into the kernel parameters would copy them to local memory
      if (threadIdx.x == (uint32_t)k && (uint32_t)k < A.nseg) { s_seg.req[k] = A.seg_reqs[k]; s_seg.out[k] = A.seg_out[k]; }
    }
    if (threadIdx.x <= A.nseg) s_seg.off[threadIdx.x] = __ldcg(A.seg_off + threadIdx.x);
    if (threadIdx.x == 0) s_seg.nseg = A.nseg;
    __syncthreads();
    return Io<SEG>{A, &s_seg};
  } else {
    return Io<SEG>{A, nullptr};
  }
}

// Counter deltas are summed per block in shared memory first: a grid-wide atomicAdd per warp on five fixed addresses
// serialises in L2 and costs more than the probes themselves.
__device__ __forceinline__ void tally_flush_block(const Tally& t, unsigned long long* counters) {
  __shared__ uint32_t s_tally[5];
  if (threadIdx.x < 5) s_tally[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t over = __reduce_add_sync(0xFFFFFFFFu, t.over), hit = __reduce_add_sync(0xFFFFFFFFu, t.hit),
                 miss = __reduce_add_sync(0xFFFFFFFFu, t.miss), ins = __reduce_add_sync(0xFFFFFFFFu, t.inserts),
                 full = __reduce_add_sync(0xFFFFFFFFu, t.full);
  if ((threadIdx.x & 31) == 0) {
    if (over) atomicAdd(&s_tally[0], over);
    if (hit) atomicAdd(&s_tally[1], hit);
    if (miss) atomicAdd(&s_tally[2], miss);
    if (ins) atomicAdd(&s_tally[3], ins);
    if (full) atomicAdd(&s_tally[4], full);
  }
  __syncthreads();
  if (threadIdx.x < 5 && s_tally[threadIdx.x]) {
    const int slot[5] = {C_OVER, C_HIT, C_MISS, C_INSERTS, C_FULL};
    atomicAdd(counters + slot[threadIdx.x], (unsigned long long)s_tally[threadIdx.x]);
  }
}

// cursor_open + the InvalidAt clause of IsExpired (cache.go:47), and the write-back with parking, in terms of BatchArgs
__device__ __forceinline__ void open_slot(const BatchArgs& A, Cursor& cur, uint64_t key, uint64_t tag) {
  cursor_open(cur, A.table, A.capacity, key, tag);
  apply_invalid_at(A.inv, cur.b, cur.found, A.clk.now_ms);
}
__device__ __forceinline__ void close_slot(const BatchArgs& A, Cursor& cur, Tally& t) { close_or_park(cur, A.table, A.capacity, A.ovf, A.ovf_count, t); }

// ---- kernel 1: group the batch by key, rank members inside each block --------------------------------------------
// Joins `c` members to the batch-wide group of `key`; returns the entry position.  *claimed = this call created the entry.
__device__ __forceinline__ uint32_t aux_home(const BatchArgs& A, uint64_t key) { return (uint32_t)(key ^ (key >> 29)) & A.aux_mask; }

// `first` = the home entry's word as read earlier (prefetched while the block-local grouping ran).
__device__ __forceinline__ uint32_t aux_join(const BatchArgs& A, uint64_t key, uint32_t c, unsigned long long first, bool* claimed) {
  const uint32_t tag = (uint32_t)(key >> 40);  // 24 bits, disjoint from the position bits below
  uint32_t pos = aux_home(A, key);
  const unsigned long long fresh = ((unsigned long long)A.epoch << 48) | ((unsigned long long)tag << 24) | (unsigned long long)c;
  *claimed = false;
  bool have_first = true;
#pragma unroll 1
  for (;;) {
    unsigned long long cur = have_first ? first : __ldcg(&A.aux[pos].word);
    have_first = false;
    if (aux_epoch(cur) != A.epoch) {  // stale entry from an earlier batch == empty
      const unsigned long long old = atomicCAS(&A.aux[pos].word, cur, fresh);
      if (old == cur) { *claimed = true; break; }
      cur = old;  // somebody else just claimed it for this batch: fall through and compare tags
    }
    if (aux_epoch(cur) == A.epoch && aux_tag(cur) == tag) {
      atomicAdd(&A.aux[pos].word, (unsigned long long)c);
      break;
    }
    pos = (pos + 1) & A.aux_mask;
  }
  return pos;
}

// Group entries are matched on 24 bits of the key plus the entry position, so two different keys can share one (about 2^-42 per
// pair of keys in a batch).  That is harmless across blocks: the merged group is found non-uniform in k_rank and k_finish walks it
// key by key.  Inside ONE block, though, a group entry has room for one fragment only (one presence bit, one size byte, local
// ranks starting at 0), so fragments of a block that landed in the same entry are folded into one here: their members are
// re-ranked together in index order, pointed at the first fragment's shared-memory slot (k_rank keeps the fragment's base rank
// there) and the combined size is stored.  One thread does it; it runs once in ~10^7 blocks.
__device__ void merge_colliding_fragments(const BatchArgs& A, const uint32_t* s_pos, bool valid, uint32_t& sp, uint32_t& local) {
  __shared__ uint16_t s_tsp[GROUP_THREADS], s_tlocal[GROUP_THREADS];
  s_tsp[threadIdx.x] = valid ? (uint16_t)sp : (uint16_t)0xFFFFu;
  s_tlocal[threadIdx.x] = (uint16_t)0xFFFFu;  // 0xFFFF: keep the rank computed above
  __syncthreads();
  if (threadIdx.x == 0) {
    for (uint32_t t = 0; t < (uint32_t)GROUP_THREADS; t++) {
      const uint32_t spt = s_tsp[t];
      if (spt == 0xFFFFu || s_tlocal[t] != 0xFFFFu) continue;  // no request, or already folded into an earlier fragment
      const uint32_t pos = s_pos[spt];
      bool shared = false;
      for (uint32_t u = t + 1; u < (uint32_t)GROUP_THREADS && !shared; u++) shared = s_tsp[u] != 0xFFFFu && s_tsp[u] != spt && s_pos[s_tsp[u]] == pos;
      if (!shared) continue;
      uint32_t cnt = 0;
      for (uint32_t u = t; u < (uint32_t)GROUP_THREADS; u++) {
        if (s_tsp[u] != 0xFFFFu && s_pos[s_tsp[u]] == pos) { s_tlocal[u] = (uint16_t)cnt++; s_tsp[u] = (uint16_t)spt; }
      }
      A.fragsize[(size_t)pos * A.max_blocks + blockIdx.x] = (uint8_t)(cnt - 1);
    }
  }
  __syncthreads();
  if (valid && s_tlocal[threadIdx.x] != 0xFFFFu) { local = s_tlocal[threadIdx.x]; sp = s_tsp[threadIdx.x]; }
}

// What k_group does right after its wait.  Inserts a previous batch could not place (probe window full) are placed now, with eviction:
// the previous batch is complete and this batch's k_rank has not passed its wait (it waits for this grid), so nothing can observe a
// half-moved entry.
__device__ __forceinline__ void group_waited(const BatchArgs& A) {
  KT(A, 0, KT_WAITED, 0, false);
  if (blockIdx.x == 0 && threadIdx.x < 32 && __ldcg(A.ovf_count)) {
    uint32_t ins = 0;
    drain_parked(A.table, A.capacity, A.ovf, A.ovf_count, A.clk.now_ms, A.counters, &ins);
    if (threadIdx.x == 0 && ins) atomicAdd(A.counters + C_INSERTS, (unsigned long long)ins);
  }
}

// Early hand-off (single table): apart from that drain k_group does not touch the table, and it writes only the grouping scratch of its
// epoch's parity, which the batch before it does not use, so its body need not wait for that batch.  It does read the request records, which PDL guarantees only
// after the wait.  A block therefore looks at *chain_done first:
//  - it is not the previous epoch: k_finish of the previous batch has not finished, so this launch started as ITS programmatic
//    dependent.  A plain kernel in between would have waited for that k_finish to complete, and a memory operation breaks the
//    programmatic edge altogether, so nothing ran between the two submissions: the records were complete before the previous batch's
//    chain began (its k_rank waited for its k_group, which waited for everything earlier).  The block triggers its dependents, does its
//    whole body, and waits before it exits, so this grid's completion (what k_rank waits for) still implies the previous batch's.
//  - it is the previous epoch, or early_ok is off (first batch, one scratch set, ring mode): wait first, as before.
// Not detected: a caller kernel launched programmatically between two submissions that triggers its dependents before its last write of
// the records.  Blocks decide independently; either choice is correct for a block.
template <bool SEG>
__global__ void __launch_bounds__(GROUP_THREADS) k_group(const BatchArgs A) {
  __shared__ uint32_t s_early;
  __shared__ unsigned long long s_key[GROUP_SLOTS];
  __shared__ uint32_t s_cnt[GROUP_SLOTS];  // members of the key in this block
  __shared__ uint32_t s_pos[GROUP_SLOTS];  // batch-wide entry position
  __shared__ uint32_t s_conflict;          // two fragments of this block joined the same group entry (see merge_colliding_fragments)
  // [key slot][warp]: members of the key among the warp's lanes (<= 32).  Every warp counts its members per key (match.any); after one
  // barrier a member's index-ordered local rank is the sum over earlier warps + its rank inside the warp (one barrier instead of eight
  // warp turns with a barrier each).
  __shared__ __align__(16) uint8_t s_wcnt[GROUP_SLOTS][GROUP_THREADS / 32];
  static_assert(sizeof(s_wcnt) == GROUP_THREADS * sizeof(uint4), "one 16-byte store per thread clears it");
  for (uint32_t k = threadIdx.x; k < GROUP_SLOTS; k += GROUP_THREADS) { s_key[k] = 0ull; s_cnt[k] = 0u; }
  if (threadIdx.x == 0) s_conflict = 0u;
  reinterpret_cast<uint4*>(&s_wcnt[0][0])[threadIdx.x] = make_uint4(0u, 0u, 0u, 0u);
  KT(A, 0, KT_ENTRY, 0, false);
  if (threadIdx.x == 0) s_early = (!SEG && A.early_ok && ld_acquire_gpu(A.chain_done) != A.epoch - 1u) ? 1u : 0u;
  __syncthreads();
  const bool early = s_early != 0;
  if (early) {
    pdl_release();
  } else {
    pdl_wait();
    pdl_release();
    group_waited(A);
  }
  const Io<SEG> io = io_open<SEG>(A);
  __syncthreads();
  const uint32_t i = blockIdx.x * GROUP_THREADS + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t n = batch_n(A);  // an earlier kernel may have written it: after the wait, or (early) complete like the records
  if (blockIdx.x * GROUP_THREADS >= n) {  // whole block beyond the batch (uniform: no barrier is skipped by part of a block)
    if (early) { pdl_wait(); group_waited(A); }
    return;
  }
  const bool valid = i < n;
  uint32_t sp = 0xFFFFu;  // shared-memory slot of my key (0xFFFF: no request)
  uint64_t key = 0;
  unsigned long long first = 0;
  if (valid) {
    key = remap_key(io.key(i));  // never 0
    first = __ldcg(&A.aux[aux_home(A, key)].word);  // consumed much later, by the fragment's first member only
    prefetch_l2(A.table + __umul64hi(key, A.capacity));  // the slot k_rank / k_eval will probe
    sp = (uint32_t)((key * 0x9E3779B97F4A7C15ull) >> 55);  // top 9 bits -> GROUP_SLOTS
#pragma unroll 1
    for (;;) {
      const unsigned long long old = atomicCAS(&s_key[sp], 0ull, (unsigned long long)key);
      if (old == 0ull || old == key) break;
      sp = (sp + 1) & (GROUP_SLOTS - 1);
    }
  }
  KT(A, 0, KT_M2, sp, false);  // keys loaded and entered into the block's table
  __syncthreads();
  uint32_t local = 0;
  {
    constexpr int NW = GROUP_THREADS / 32;
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, sp);
    const uint32_t leader = __ffs(peers) - 1;
    if (valid && lane == leader) s_wcnt[sp][warp] = (uint8_t)__popc(peers);
    __syncthreads();
    if (valid) {
      uint32_t before = 0, total = 0;
#pragma unroll
      for (int w = 0; w < NW; w++) { const uint32_t c = s_wcnt[sp][w]; total += c; before += ((uint32_t)w < warp) ? c : 0u; }
      local = before + __popc(peers & ((1u << lane) - 1u));
      if (local == 0) s_cnt[sp] = total;
    }
    __syncthreads();
    KT(A, 0, KT_M3, local, false);  // local ranks known
  }
  // the first member of each fragment joins the batch-wide group
  if (valid && local == 0) {
    const uint32_t c = s_cnt[sp];
    bool claimed;
    const uint32_t pos = aux_join(A, key, c, first, &claimed);
    if (claimed) { A.aux[pos].rep = i; A.aux[pos].flags = 0; }
    const uint32_t bit = 1u << (blockIdx.x & 31);
    const uint32_t was = atomicOr(&A.presence[(size_t)pos * A.pres_words + (blockIdx.x >> 5)], bit);
    A.fragsize[(size_t)pos * A.max_blocks + blockIdx.x] = (uint8_t)(c - 1);
    s_pos[sp] = pos;
    if (was & bit) s_conflict = 1u;  // the bitmap is clean between batches: another fragment of this block is in this entry already
    KT(A, 0, KT_M4, was, true);  // a fragment has joined its group
  }
  KT(A, 0, KT_WORK_DONE, 0, false);
  __syncthreads();
  if (s_conflict) merge_colliding_fragments(A, s_pos, valid, sp, local);  // block-uniform, next to never taken
  if (valid) {
    A.ent[i] = s_pos[sp];
    A.meta[i] = (sp << 16) | local;
  }
  if (early) {
    pdl_wait();
    group_waited(A);
  }
  KT(A, 0, KT_EXIT, 0, false);
}

// ---- kernel 2: singletons are evaluated; members of repeated keys get their rank and check uniformity ------------
// Requests that can make an identical run irregular for ever (no subtract regime, no fixed point) are sent down the
// segment path, whose cost is linear in the run length: negative hits keep adding, RESET_REMAINING on a token bucket
// alternates delete/create, and float64 remaining beyond 2^52 loses integer steps.
__device__ __forceinline__ bool req_regular(const gub_req& r) {
  if (r.hits < 0) return false;
  if (r.algorithm == GUB_TOKEN_BUCKET && (r.behavior & GUB_BEHAVIOR_RESET_REMAINING)) return false;
  if (r.algorithm == GUB_LEAKY_BUCKET && (r.limit >= (1ll << 52) || r.burst >= (1ll << 52))) return false;
  return true;
}

// sum over present blocks b' < b of (fragsize[b'] + 1): the rank of block b's first member of this group.
// All loads are issued before any is consumed (a hot key has a fragment in every block: 8 bitmap words + 16 x 16 B of sizes
// for a 64 k batch), so the cost is two L2 round trips rather than one per word.
__device__ __forceinline__ uint32_t masked_sum32(const uint4& lo, const uint4& hi, uint32_t bits) {
  const uint32_t v[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
  uint32_t acc = __popc(bits);
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const uint32_t m4 = (bits >> (4 * k)) & 0xFu;
    const uint32_t mask = ((m4 * 0x00204081u) & 0x01010101u) * 0xFFu;  // bit j of m4 -> byte j all ones
    acc = __dp4a(v[k] & mask, 0x01010101u, acc);
  }
  return acc;
}

__device__ __forceinline__ uint32_t fragment_base(const BatchArgs& A, uint32_t pos, uint32_t b) {
  const uint32_t* pres = A.presence + (size_t)pos * A.pres_words;
  const uint8_t* row = A.fragsize + (size_t)pos * A.max_blocks;
  const uint32_t last = b >> 5, keep = (1u << (b & 31)) - 1u;
  uint32_t base = 0;
  if (A.pres_words == 8) {  // max_batch = 65536
    const uint4 p0 = __ldcg(reinterpret_cast<const uint4*>(pres)), p1 = __ldcg(reinterpret_cast<const uint4*>(pres) + 1);
    uint32_t bits[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
    uint32_t any = 0;
#pragma unroll
    for (int w = 0; w < 8; w++) { bits[w] = ((uint32_t)w < last) ? bits[w] : ((uint32_t)w == last ? (bits[w] & keep) : 0u); any += __popc(bits[w]); }
    if (any == 0) return 0;
    if (any <= 2) {  // the common case: a couple of earlier fragments
#pragma unroll
      for (int w = 0; w < 8; w++) {
        uint32_t x = bits[w];
        while (x) { const uint32_t k = __ffs(x) - 1; x &= x - 1; base += (uint32_t)row[w * 32 + k] + 1u; }
      }
      return base;
    }
    uint4 lo[8], hi[8];
#pragma unroll
    for (int w = 0; w < 8; w++) {
      if (bits[w]) { lo[w] = __ldcg(reinterpret_cast<const uint4*>(row + w * 32)); hi[w] = __ldcg(reinterpret_cast<const uint4*>(row + w * 32 + 16)); }
    }
#pragma unroll
    for (int w = 0; w < 8; w++) if (bits[w]) base += masked_sum32(lo[w], hi[w], bits[w]);
    return base;
  }
  // other batch sizes (rings evaluate up to 262 144 requests = 1024 blocks per launch): four bitmap words per round trip
  // (pres_words is a multiple of 4: gub_create)
  const uint32_t nq = (last >> 2) + 1;
#pragma unroll 1
  for (uint32_t q = 0; q < nq; q++) {
    const uint4 pv = __ldcg(reinterpret_cast<const uint4*>(pres) + q);
    uint32_t bits[4] = {pv.x, pv.y, pv.z, pv.w};
    uint4 lo[4], hi[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const uint32_t w = q * 4 + (uint32_t)k;
      bits[k] = w < last ? bits[k] : (w == last ? (bits[k] & keep) : 0u);
      if (bits[k]) { lo[k] = __ldcg(reinterpret_cast<const uint4*>(row + w * 32)); hi[k] = __ldcg(reinterpret_cast<const uint4*>(row + w * 32 + 16)); }
    }
#pragma unroll
    for (int k = 0; k < 4; k++) if (bits[k]) base += masked_sum32(lo[k], hi[k], bits[k]);
  }
  return base;
}

// Which request each thread of a 256-thread block evaluates: the block's token-bucket requests first, then its leaky-bucket
// ones (stable), so that all but one warp run a single algorithm's code path instead of both.  Only reads the 4-byte
// algorithm field, so it can run in the prologue ahead of pdl_wait().
template <bool SEG>
__device__ __forceinline__ uint32_t partition_by_algorithm(const Io<SEG>& io, uint32_t n) {
  __shared__ uint16_t s_perm[GROUP_THREADS];
  __shared__ uint32_t s_cnt3[GROUP_THREADS / 32][3];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t i = blockIdx.x * GROUP_THREADS + tid;
  uint32_t cls = 2;
  if (i < n) { const uint32_t a = io.algorithm(i); cls = a < 2u ? a : 2u; }
  const uint32_t b0 = __ballot_sync(0xFFFFFFFFu, cls == 0), b1 = __ballot_sync(0xFFFFFFFFu, cls == 1), b2 = ~(b0 | b1);
  if (lane == 0) { s_cnt3[warp][0] = __popc(b0); s_cnt3[warp][1] = __popc(b1); s_cnt3[warp][2] = __popc(b2); }
  __syncthreads();
  uint32_t tot0 = 0, tot1 = 0, before = 0;
#pragma unroll
  for (int w = 0; w < GROUP_THREADS / 32; w++) {
    tot0 += s_cnt3[w][0]; tot1 += s_cnt3[w][1];
    if ((uint32_t)w < warp) before += s_cnt3[w][cls];
  }
  const uint32_t mine = cls == 0 ? b0 : (cls == 1 ? b1 : b2);
  const uint32_t dest = (cls == 0 ? 0u : (cls == 1 ? tot0 : tot0 + tot1)) + before + __popc(mine & ((1u << lane) - 1u));
  s_perm[dest] = (uint16_t)tid;
  __syncthreads();
  return blockIdx.x * GROUP_THREADS + s_perm[tid];
}


// (Register budget: 2 resident blocks per SM, ~128 registers.  Capping at 80 / 64 registers for 3 / 4 blocks makes the kernels spill.)
template <bool SEG>
__global__ void __launch_bounds__(GROUP_THREADS, 2) k_rank(const BatchArgs A) {
  __shared__ uint32_t s_base[GROUP_SLOTS];
  const Io<SEG> io = io_open<SEG>(A);  // (ring mode: the segment table was final before k_group started)
  const uint32_t n = batch_n(A);  // written at least two kernels ago: safe ahead of the wait, like the records
  // A launch is sized for the most the batch can hold (ring mode: what all sources could send); blocks beyond the batch leave at once —
  // before the wait, so that they do not keep the register file from the blocks that have work (two resident blocks per SM).  Block 0
  // always stays: a grid whose blocks all skipped the wait would complete before its predecessor and break the chain of waits.
  if (blockIdx.x != 0 && blockIdx.x * GROUP_THREADS >= n) return;
  const uint32_t i = partition_by_algorithm(io, n);
  Tally t = {0, 0, 0, 0, 0};
  const bool valid = i < n;
  gub_req rq;
  if (valid) rq = io.load(i);  // the records were complete before k_group started: safe ahead of the wait
  KT(A, 1, KT_ENTRY, (uint32_t)rq.hits, false);  // (request in registers)
  pdl_wait();
  pdl_release();
  KT(A, 1, KT_WAITED, 0, false);
  if (blockIdx.x == 0 && threadIdx.x == 0) {  // reset the other parity's allocator for the next batch (nobody is using it now)
    BatchCtr* nxt = A.ctr + ((A.epoch + 1) & 1);
    nxt->n_mixed = 0; nxt->order_bump = 0; nxt->next_mixed = 0;
    atomicAdd(A.counters + C_REQUESTS, (unsigned long long)n);
    atomicAdd(A.counters + C_BATCHES, 1ull);
  }
  uint32_t pos = 0, cnt = 0, sp = 0, local = 0;
  if (valid) {
    pos = A.ent[i];
    const uint32_t m = A.meta[i];
    const ulonglong2 e = __ldcg(reinterpret_cast<const ulonglong2*>(&A.aux[pos]));
    const uint64_t key = remap_key(rq.key_xxh64);
    sp = m >> 16; local = m & 0xFFFFu;
    cnt = aux_count(e.x);
    KT(A, 1, KT_M2, cnt, true);  // group entry read
    const uint32_t rep = (uint32_t)(e.y & 0xFFFFFFFFull);
    if (cnt > 1) {
      // uniformity does not need the rank: start the representative's load before anything that waits
      bool mixed = !req_regular(rq);
      gub_req rr;
      const bool cmp = !mixed && i != rep;
      if (cmp) rr = io.load(rep);
      if (local == 0) {
        const uint32_t base = fragment_base(A, pos, blockIdx.x);
        s_base[sp] = base;
        KT(A, 1, KT_M3, base, true);  // a fragment's base rank
        if (base == 0) {  // rank 0 of the run: look the key up once for everybody
          Cursor cur;
          open_slot(A, cur, key, rq.key_fnv1 >> 8);
          snap_store(A.commit + (size_t)pos * 6, cur, i);
          KT(A, 1, KT_M4, (uint32_t)cur.b.flags, true);  // a run's snapshot stored
        }
      }
      if (cmp) mixed = !req_same(rq, rr);
      if (mixed) {
        const uint32_t old = atomicOr(&A.aux[pos].flags, AUX_NONUNIFORM);
        if (!(old & AUX_NONUNIFORM)) {  // first to notice: reserve the group's region of `order` and list the group
          BatchCtr* ctr = A.ctr + (A.epoch & 1);
          A.aux[pos].gbase = atomicAdd(&ctr->order_bump, cnt);
          A.mixed_ent[atomicAdd(&ctr->n_mixed, 1u)] = pos;
        }
      }
    } else if (cnt == 1) {  // a key seen once — most keys: evaluated right here (its slot was prefetched into L2 by k_group)
      A.presence[(size_t)pos * A.pres_words + (blockIdx.x >> 5)] = 0;  // hand the bitmap back clean (this block's bit is the only one)
      Cursor cur;
      open_slot(A, cur, key, rq.key_fnv1 >> 8);
      Delta d = {0, 0, 0};
      const gub_resp r = apply_one(cur.b, rq, A.clk, d);
      close_slot(A, cur, t);
      t.over += d.over; t.hit += d.hit; t.miss += d.miss;
      store_resp(io.resp(i), r);
      KT(A, 1, KT_M5, r.status, true);  // a key seen once answered
    }
  }
  KT(A, 1, KT_WORK_DONE, 0, false);
  __syncthreads();
  if (valid && cnt > 1) A.rank[i] = s_base[sp] + local;
  tally_flush_block(t, A.counters);
  KT(A, 1, KT_EXIT, 0, false);
}

// ---- kernel 3: every request of a uniform run evaluates its own rank ------------------------------------------------
template <bool SEG>
__global__ void __launch_bounds__(GROUP_THREADS, 2) k_eval(const BatchArgs A) {
  const Io<SEG> io = io_open<SEG>(A);
  const uint32_t n = batch_n(A);
  if (blockIdx.x != 0 && blockIdx.x * GROUP_THREADS >= n) return;  // (see k_rank)
  const uint32_t i = partition_by_algorithm(io, n);
  Tally t = {0, 0, 0, 0, 0};
  uint32_t dup = 0;
  gub_req rq;
  if (i < n) rq = io.load(i);  // safe ahead of the wait (see k_rank)
  KT(A, 2, KT_ENTRY, (uint32_t)rq.hits, false);
  pdl_wait();
  pdl_release();
  KT(A, 2, KT_WAITED, 0, false);
  if (A.mixed_hint && blockIdx.x == 0 && threadIdx.x == 0) *(volatile uint32_t*)A.mixed_hint = __ldcg(&A.ctr[A.epoch & 1].n_mixed);  // final: k_rank is complete
  if (i < n) {
    const uint32_t pos = A.ent[i];
    const uint32_t rank = A.rank[i];             // garbage for keys seen once: not used
    const AuxEntry* e = &A.aux[pos];
    const ulonglong2 ev = __ldcg(reinterpret_cast<const ulonglong2*>(e));
    const uint32_t cnt = aux_count(ev.x);
    KT(A, 2, KT_M2, cnt, true);  // group entry read
    const bool mixed = cnt > 1 && ((uint32_t)(ev.y >> 32) & AUX_NONUNIFORM) != 0;
    if (cnt > 1 && rank == 0) {  // hand the presence bitmap back clean
      uint32_t* pres = A.presence + (size_t)pos * A.pres_words;
      for (uint32_t w = 0; w < A.pres_words; w++) pres[w] = 0;
    }
    if (mixed) {
      A.order[__ldcg(&e->gbase) + rank] = i;
    } else if (cnt > 1) {
      Cursor cur;
      snap_load(A.commit + (size_t)pos * 6, cur);  // the slot as k_rank found it (the last rank may already be writing the table)
      Delta d = {0, 0, 0};
      const gub_resp r = run_to_rank(cur.b, rq, rank, A.clk, d);
      if (rank == cnt - 1) {  // I hold the run's final state and its total counter deltas
        t.over += d.over; t.hit += d.hit; t.miss += d.miss;
        close_slot(A, cur, t);
        dup = 1;
      }
      store_resp(io.resp(i), r);
      KT(A, 2, KT_M3, r.status, true);  // a member of a uniform run answered
    }
  }
  KT(A, 2, KT_WORK_DONE, 0, false);
  dup = __reduce_add_sync(0xFFFFFFFFu, dup);
  if ((threadIdx.x & 31) == 0 && dup) atomicAdd(A.counters + C_DUP_GROUPS, (unsigned long long)dup);
  tally_flush_block(t, A.counters);
  KT(A, 2, KT_EXIT, 0, false);
}

// ---- kernel 4: runs whose requests differ ---------------------------------------------------------------------------
// A group whose requests differ is a sequence of SEGMENTS (runs of identical requests).  It is taken in chunks of MIXED_CHUNK
// members (rank order: `order`): the block finds the chunk's segment starts in parallel and stages each segment's request in shared
// memory; thread 0 then FOLDS the segments in order — one closed-form run_to_rank() per segment, keeping the bucket state ENTERING
// each — and every member evaluates run_to_rank(entering state, request, rank within the segment) by itself.  A chunk that is
// mostly one-request runs (more than MIXED_SEGS segments), or a segment whose request can never settle, is applied one request
// at a time by thread 0.  The slot is opened once and written once for the whole group (thread 0 carries the cursor).
constexpr uint32_t MIXED_CHUNK = 1024, MIXED_SEGS = 256;
struct MixedShared {
  uint32_t nseg;
  uint32_t seg[MIXED_SEGS + 1];     // first member (offset in the chunk) of every segment, ascending; seg[nseg] = members in the chunk
  uint32_t raw[MIXED_SEGS];         // the starts as found (any order)
  uint8_t kind[MIXED_SEGS];         // 1: applied one by one by the folding thread
  gub_req shape[MIXED_SEGS];        // the segment's request
  Bucket state[MIXED_SEGS];         // bucket entering the segment
};

__device__ __forceinline__ Bucket bucket_from_lane(const Bucket& b, uint32_t src) {
  Bucket r;
  r.key = __shfl_sync(0xFFFFFFFFu, (unsigned long long)b.key, src); r.tag = __shfl_sync(0xFFFFFFFFu, (unsigned long long)b.tag, src);
  r.limit = (int64_t)__shfl_sync(0xFFFFFFFFu, (unsigned long long)b.limit, src); r.duration = (int64_t)__shfl_sync(0xFFFFFFFFu, (unsigned long long)b.duration, src);
  r.rem = __shfl_sync(0xFFFFFFFFu, (unsigned long long)b.rem, src); r.stamp = (int64_t)__shfl_sync(0xFFFFFFFFu, (unsigned long long)b.stamp, src);
  r.burst = (int64_t)__shfl_sync(0xFFFFFFFFu, (unsigned long long)b.burst, src); r.expire = (int64_t)__shfl_sync(0xFFFFFFFFu, (unsigned long long)b.expire, src);
  r.flags = __shfl_sync(0xFFFFFFFFu, b.flags, src);
  return r;
}

// Applies one segment to b: a closed form for the whole segment (the state entering it is kept for the members), else request by
// request with the responses stored right away.
template <bool SEG>
__device__ __forceinline__ void fold_segment(const BatchArgs& A, const Io<SEG>& io, MixedShared& S, const uint32_t* ord, uint32_t sgi, Bucket& b, Delta& d) {
  const uint32_t lo = S.seg[sgi], hi = S.seg[sgi + 1];
  gub_req rq = S.shape[sgi];
  const bool closed_form = req_regular(rq);
  S.kind[sgi] = closed_form ? 0 : 1;
  if (closed_form) {
    S.state[sgi] = b;
    run_to_rank(b, rq, hi - lo - 1, A.clk, d);
    return;
  }
#pragma unroll 1
  for (uint32_t k = lo; k < hi; k++) {
    if (k > lo) rq = io.load(ord[k]);
    store_resp(io.resp(ord[k]), apply_one(b, rq, A.clk, d));
  }
}

// The fold of one chunk, by warp 0.  A hot key whose requests differ (clients asking for different `hits`) is a long sequence of
// segments, and applying them is inherently sequential — but most segments of such a key leave the bucket where it was (over the
// limit: a fixed point).  So the warp SPECULATES: the segments are dealt to the lanes in contiguous ranges and every lane folds its
// range starting from the state E entering the first range not yet final.  Lanes up to and including the first one whose range
// moves the state (exit != E) started from the right state, so their results are exact; that lane's exit becomes the new E and the
// lanes behind it fold again.  One pass when nothing moves (the usual case for a key that is over its limit), at worst one pass per
// lane (the cost of the sequential fold).  Chunks whose segments do not all carry the chunk's first key (two keys sharing a group
// entry) and chunks with too many segments are folded by lane 0 alone, request by request where it has to be.
template <bool SEG>
__device__ void fold_chunk(const BatchArgs& A, const Io<SEG>& io, MixedShared& S, const uint32_t* ord, uint32_t cnt, bool planned, Cursor& cur,
                                        bool& open, uint64_t& ck, uint64_t& ct, Tally& t) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t nseg = planned ? S.nseg : 0u;
  bool one_key = planned;
  if (planned) {
    bool other = false;
    for (uint32_t q = lane; q < nseg; q += 32) other |= S.shape[q].key_xxh64 != S.shape[0].key_xxh64 || S.shape[q].key_fnv1 != S.shape[0].key_fnv1;
    one_key = !__any_sync(0xFFFFFFFFu, other);
  }
  if (!one_key) {  // lane 0 alone, keeping the slot of the current key in registers
    if (lane == 0) {
      const uint32_t steps = planned ? nseg : 1u;
#pragma unroll 1
      for (uint32_t sgi = 0; sgi < steps; sgi++) {
        const uint32_t lo = planned ? S.seg[sgi] : 0u, hi = planned ? S.seg[sgi + 1] : cnt;
        gub_req rq = planned ? S.shape[sgi] : io.load(ord[0]);
        const bool closed_form = planned && req_regular(rq);
        if (planned) S.kind[sgi] = closed_form ? 0 : 1;
#pragma unroll 1
        for (uint32_t k = lo; k < hi; k++) {  // closed form: one pass for the whole segment; else one pass per request
          if (!closed_form && k > lo) rq = io.load(ord[k]);
          const uint64_t key = remap_key(rq.key_xxh64), tag = rq.key_fnv1 >> 8;
          if (!open || key != ck || tag != ct) {  // (the key only changes when two keys share a group entry)
            if (open) close_slot(A, cur, t);
            open_slot(A, cur, key, tag);
            open = true; ck = key; ct = tag;
          }
          Delta d = {0, 0, 0};
          if (closed_form) {
            S.state[sgi] = cur.b;
            run_to_rank(cur.b, rq, hi - lo - 1, A.clk, d);
            t.over += d.over; t.hit += d.hit; t.miss += d.miss;
            break;
          }
          const gub_resp r = apply_one(cur.b, rq, A.clk, d);
          t.over += d.over; t.hit += d.hit; t.miss += d.miss;
          store_resp(io.resp(ord[k]), r);
        }
      }
      if (!planned) atomicAdd(A.counters + C_SERIAL, 1ull);
    }
    return;
  }
  if (lane == 0) {
    const uint64_t key = remap_key(S.shape[0].key_xxh64), tag = S.shape[0].key_fnv1 >> 8;
    if (!open || key != ck || tag != ct) {
      if (open) close_slot(A, cur, t);
      open_slot(A, cur, key, tag);
      open = true; ck = key; ct = tag;
    }
  }
  Bucket E = bucket_from_lane(cur.b, 0);
  const uint32_t per = (nseg + 31u) / 32u;
  const uint32_t s0 = min(lane * per, nseg), s1 = min(s0 + per, nseg);
  uint32_t first = 0;  // lanes below `first` are final
#pragma unroll 1
  for (;;) {
    Bucket b = E;
    Delta d = {0, 0, 0};
    if (lane >= first) {
#pragma unroll 1
      for (uint32_t sgi = s0; sgi < s1; sgi++) fold_segment(A, io, S, ord, sgi, b, d);
    }
    const uint32_t moved = __ballot_sync(0xFFFFFFFFu, lane >= first && !bucket_equal(b, E));
    const uint32_t J = moved ? (uint32_t)__ffs((int)moved) - 1u : 32u;  // lanes first..J started from the state that really enters their range
    if (lane >= first && lane <= J) { t.over += d.over; t.hit += d.hit; t.miss += d.miss; }
    if (J >= 32u) break;       // nothing moved: E is also the state leaving the chunk
    E = bucket_from_lane(b, J);
    first = J + 1u;
    if (first >= 32u) break;   // lane 31 was exact
  }
  if (lane == 0) cur.b = E;
}

template <bool SEG>
__device__ void mixed_group(const BatchArgs& A, const Io<SEG>& io, uint32_t pos, MixedShared& S, Tally& t) {
  const uint32_t tid = threadIdx.x;
  const uint32_t total = aux_count(__ldcg(&A.aux[pos].word));
  const uint32_t* ord_all = A.order + __ldcg(&A.aux[pos].gbase);
  Cursor cur;
  bool open = false;
  uint64_t ck = 0, ct = 0;
#pragma unroll 1
  for (uint32_t c0 = 0; c0 < total; c0 += MIXED_CHUNK) {
    const uint32_t* ord = ord_all + c0;
    const uint32_t cnt = min(MIXED_CHUNK, total - c0);
    __syncthreads();
    if (tid == 0) S.nseg = 0;
    __syncthreads();
    // segment starts: ranks whose request differs from the previous member's.  Every member loads its own request once; the previous
    // member's comes from the lane below (lane 0 loads it itself), so a chunk costs two dependent round trips per 256 members.
#pragma unroll 1
    for (uint32_t k0 = 0; k0 < cnt; k0 += MIXED_THREADS) {
      const uint32_t k = k0 + tid;
      const bool live = k < cnt;
      const uint32_t lane = tid & 31;
      gub_req a, b;
      if (live) a = io.load(ord[k]);
      if (live && lane == 0 && k > 0) b = io.load(ord[k - 1]);
      gub_req up;  // the request of the lane below
      up.key_xxh64 = __shfl_up_sync(0xFFFFFFFFu, (unsigned long long)a.key_xxh64, 1); up.key_fnv1 = __shfl_up_sync(0xFFFFFFFFu, (unsigned long long)a.key_fnv1, 1);
      up.hits = (int64_t)__shfl_up_sync(0xFFFFFFFFu, (unsigned long long)a.hits, 1); up.limit = (int64_t)__shfl_up_sync(0xFFFFFFFFu, (unsigned long long)a.limit, 1);
      up.duration = (int64_t)__shfl_up_sync(0xFFFFFFFFu, (unsigned long long)a.duration, 1); up.burst = (int64_t)__shfl_up_sync(0xFFFFFFFFu, (unsigned long long)a.burst, 1);
      up.created_at = (int64_t)__shfl_up_sync(0xFFFFFFFFu, (unsigned long long)a.created_at, 1);
      up.algorithm = __shfl_up_sync(0xFFFFFFFFu, a.algorithm, 1); up.behavior = __shfl_up_sync(0xFFFFFFFFu, a.behavior, 1);
      if (live) {
        const bool boundary = k == 0 || !req_same(a, lane == 0 ? b : up);
        if (boundary) { const uint32_t q = atomicAdd(&S.nseg, 1u); if (q < MIXED_SEGS) S.raw[q] = k; }
      }
    }
    __syncthreads();
    const uint32_t nseg = S.nseg;
    const bool planned = nseg <= MIXED_SEGS;
    if (planned) {  // rank sort of the starts, and the segments' requests into shared memory
      for (uint32_t q = tid; q < nseg; q += MIXED_THREADS) {
        const uint32_t v = S.raw[q];
        uint32_t r = 0;
        for (uint32_t j = 0; j < nseg; j++) r += S.raw[j] < v ? 1u : 0u;
        S.seg[r] = v;
        S.shape[r] = io.load(ord[v]);
      }
      if (tid == 0) S.seg[nseg] = cnt;
    }
    __syncthreads();
    if (tid < 32) fold_chunk(A, io, S, ord, cnt, planned, cur, open, ck, ct, t);  // warp 0 (thread 0 carries the group's cursor)
    __syncthreads();
    if (planned) {  // every member of a closed-form segment answers for itself
      for (uint32_t k = tid; k < cnt; k += MIXED_THREADS) {
        uint32_t lo = 0, hi = nseg;
        while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (S.seg[mid] <= k) lo = mid; else hi = mid; }
        if (S.kind[lo]) continue;
        Bucket b = S.state[lo];
        Delta d = {0, 0, 0};
        store_resp(io.resp(ord[k]), run_to_rank(b, S.shape[lo], k - S.seg[lo], A.clk, d));
      }
    }
  }
  if (tid == 0 && open) close_slot(A, cur, t);
}

// Non-uniform groups, one block each (grid-stride).  A launch with nothing to finish — the usual case — returns at once.
// Single table: it triggers its dependents at entry, so that the next batch's k_group can start beside this batch's tail.  That k_group
// launches only once every k_finish block has been resident, and a k_finish block (128 registers x 256 threads) fits on an SM only beside
// one k_eval block, so blocks that will find no group leave before the wait and hand their place on: the number of non-uniform groups was
// written by k_rank, which completed before k_eval passed its wait, i.e. two kernels ago (safe ahead of the wait, like batch_n in
// k_rank).  A stale read would only leave more of the queue to the blocks that stay.  Block 0 always waits (a grid whose blocks all
// skipped the wait would complete before its predecessor and break the chain of waits) and, last, stores the epoch into *chain_done: until
// then the next batch's k_group knows this grid has not finished (see k_group).
template <bool SEG>
#if !defined(GUB_FINISH_MIN_BLOCKS)
#define GUB_FINISH_MIN_BLOCKS 2  // 128 registers (the segment fold spills a little): an empty k_finish block must fit next to a k_eval / k_rank block
#endif
__global__ void __launch_bounds__(MIXED_THREADS, GUB_FINISH_MIN_BLOCKS) k_finish(const BatchArgs A) {
  __shared__ MixedShared S;
  Tally t = {0, 0, 0, 0, 0};
  KT(A, 3, KT_ENTRY, 0, false);
  if constexpr (!SEG) {
    pdl_release();
    if (blockIdx.x != 0) {
      __shared__ uint32_t s_idle;
      if (threadIdx.x == 0) s_idle = blockIdx.x >= __ldcg(&A.ctr[A.epoch & 1].n_mixed) ? 1u : 0u;
      __syncthreads();
      if (s_idle) return;
    }
  }
  pdl_wait();
  if constexpr (SEG) pdl_release();
  KT(A, 3, KT_WAITED, 0, false);
  const BatchCtr ctr = A.ctr[A.epoch & 1];
  if (ctr.n_mixed != 0) {
    const Io<SEG> io = io_open<SEG>(A);
    // groups differ a lot in size (a hot key's group has thousands of members): blocks pull the next one when they are done
    __shared__ uint32_t s_next;
    for (;;) {
      if (threadIdx.x == 0) s_next = atomicAdd(&A.ctr[A.epoch & 1].next_mixed, 1u);
      __syncthreads();
      const uint32_t g = s_next;
      if (g >= ctr.n_mixed) break;
      mixed_group(A, io, A.mixed_ent[g], S, t);
      __syncthreads();
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
      atomicAdd(A.counters + C_DUP_GROUPS, (unsigned long long)ctr.n_mixed);
      atomicAdd(A.counters + C_MIXED_GROUPS, (unsigned long long)ctr.n_mixed);
    }
    tally_flush_block(t, A.counters);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0 && A.chain_done) st_release_gpu(A.chain_done, A.epoch);
}

// ---- key hashing on the device: client.go:39-41 HashKey + workers.go:153 XXH64 + replicated_hash.go:108 FNV-1 ----------
// One thread per key; keys are packed back to back (key i = bytes[offsets[i] .. offsets[i+1])).  The step right before the
// path (SURVEY section 8f-2): a shim can ship raw key bytes instead of hashing on the CPU.
__device__ __forceinline__ uint64_t rotl64(uint64_t v, int s) { return (v << s) | (v >> (64 - s)); }
__device__ __forceinline__ uint64_t load_u64_le(const uint8_t* p) {
  uint64_t v = 0;
#pragma unroll
  for (int k = 0; k < 8; k++) v |= (uint64_t)p[k] << (8 * k);
  return v;
}
__device__ __forceinline__ uint64_t xxh_lane(uint64_t acc, uint64_t w) { return rotl64(acc + w * 0xC2B2AE3D27D4EB4Full, 31) * 0x9E3779B185EBCA87ull; }

__device__ __forceinline__ void hash_key_bytes(const uint8_t* p, uint32_t len, uint64_t* xxh, uint64_t* fnv) {
  constexpr uint64_t P1 = 0x9E3779B185EBCA87ull, P2 = 0xC2B2AE3D27D4EB4Full, P3 = 0x165667B19E3779F9ull, P4 = 0x85EBCA77C2B2AE63ull,
                     P5 = 0x27D4EB2F165667C5ull;
  uint64_t f = 0xCBF29CE484222325ull;
  for (uint32_t k = 0; k < len; k++) f = (f * 0x100000001B3ull) ^ p[k];
  const uint8_t* q = p;
  const uint8_t* const end = p + len;
  uint64_t h;
  if (len >= 32) {
    uint64_t v1 = P1 + P2, v2 = P2, v3 = 0, v4 = 0 - P1;
    for (; end - q >= 32; q += 32) {
      v1 = xxh_lane(v1, load_u64_le(q)); v2 = xxh_lane(v2, load_u64_le(q + 8));
      v3 = xxh_lane(v3, load_u64_le(q + 16)); v4 = xxh_lane(v4, load_u64_le(q + 24));
    }
    h = rotl64(v1, 1) + rotl64(v2, 7) + rotl64(v3, 12) + rotl64(v4, 18);
    h = (h ^ xxh_lane(0, v1)) * P1 + P4; h = (h ^ xxh_lane(0, v2)) * P1 + P4;
    h = (h ^ xxh_lane(0, v3)) * P1 + P4; h = (h ^ xxh_lane(0, v4)) * P1 + P4;
  } else {
    h = P5;
  }
  h += len;
  for (; end - q >= 8; q += 8) h = rotl64(h ^ xxh_lane(0, load_u64_le(q)), 27) * P1 + P4;
  if (end - q >= 4) {
    const uint64_t w = (uint64_t)q[0] | ((uint64_t)q[1] << 8) | ((uint64_t)q[2] << 16) | ((uint64_t)q[3] << 24);
    h = rotl64(h ^ (w * P1), 23) * P2 + P3;
    q += 4;
  }
  for (; q < end; q++) h = rotl64(h ^ (*q * P5), 11) * P1;
  h = (h ^ (h >> 33)) * P2;
  h = (h ^ (h >> 29)) * P3;
  h ^= h >> 32;
  *xxh = h; *fnv = f;
}

__global__ void __launch_bounds__(256) k_hash_keys(const uint8_t* bytes, const uint64_t* offsets, uint32_t n, uint64_t* xxh_out, uint64_t* fnv_out,
                                                   gub_req* reqs_out /* optional: fill key_xxh64 / key_fnv1 of request i */) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t h, f;
  hash_key_bytes(bytes + offsets[i], (uint32_t)(offsets[i + 1] - offsets[i]), &h, &f);
  if (xxh_out) xxh_out[i] = h;
  if (fnv_out) fnv_out[i] = f;
  if (reqs_out) { reqs_out[i].key_xxh64 = h; reqs_out[i].key_fnv1 = f; }
}

// ---- compact requests -> gub_req records (see gub_creq in the header) --------------------------------------------------
__device__ __forceinline__ void expand_words(ulonglong2 q0, ulonglong2 q1, bool known, ulonglong2 a, ulonglong2 b, int64_t created_base,
                                             ulonglong2& w0, ulonglong2& w1, ulonglong2& w2, ulonglong2& w3) {
  if (!known) { q0 = make_ulonglong2(0, 0); q1 = make_ulonglong2(0, 0xFFFFFFFFull); }  // unknown parameter set -> invalid algorithm (in-band error)
  const int32_t delta = (int32_t)(uint32_t)(b.y >> 32);
  w0 = a;                                                                   // key_xxh64, key_fnv1
  w1 = make_ulonglong2(b.x, q0.x);                                          // hits, limit
  w2 = make_ulonglong2(q0.y, q1.x);                                         // duration, burst
  w3 = make_ulonglong2((uint64_t)wadd(created_base, (int64_t)delta), q1.y); // created_at, algorithm | behavior << 32
}
__device__ __forceinline__ void expand_one(const gub_creq* creqs, uint32_t i, ulonglong2 q0, ulonglong2 q1, bool known, ulonglong2 a, ulonglong2 b,
                                           int64_t created_base, gub_req* out) {
  ulonglong2* o = reinterpret_cast<ulonglong2*>(out + i);
  expand_words(q0, q1, known, a, b, created_base, o[0], o[1], o[2], o[3]);
}

__global__ void __launch_bounds__(256) k_expand(const gub_creq* creqs, uint32_t n, const gub_params* params, uint32_t n_params, int64_t created_base,
                                                gub_req* out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const ulonglong2* p = reinterpret_cast<const ulonglong2*>(creqs + i);
  const ulonglong2 a = __ldcs(p), b = __ldcs(p + 1);  // streamed once
  const uint32_t pi = (uint32_t)(b.y & 0xFFFFFFFFull);
  ulonglong2 q0 = make_ulonglong2(0, 0), q1 = q0;
  if (pi < n_params) {
    const ulonglong2* pp = reinterpret_cast<const ulonglong2*>(params + pi);
    q0 = __ldg(pp); q1 = __ldg(pp + 1);
  }
  expand_one(creqs, i, q0, q1, pi < n_params, a, b, created_base, out);
}

// Same, with the parameter table passed by value in the kernel arguments.  A deployment has a handful of limit
// configurations, and a separate small host-to-device copy per batch stalls the copy stream far longer than its size
// suggests, so tables of up to
// INLINE_PARAMS sets travel with the launch instead.
constexpr uint32_t INLINE_PARAMS = 32;
struct InlineParams { ulonglong2 q[INLINE_PARAMS][2]; };
__global__ void __launch_bounds__(256) k_expand_inline(const gub_creq* creqs, uint32_t n, const InlineParams P, uint32_t n_params, int64_t created_base,
                                                       gub_req* out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const ulonglong2* p = reinterpret_cast<const ulonglong2*>(creqs + i);
  const ulonglong2 a = __ldcs(p), b = __ldcs(p + 1);
  const uint32_t pi = (uint32_t)(b.y & 0xFFFFFFFFull);
  const bool known = pi < n_params;
  const uint32_t k = known ? pi : 0u;
  expand_one(creqs, i, P.q[k][0], P.q[k][1], known, a, b, created_base, out);
}

// ---- key strings -> gub_req records: HashKey (client.go:39-41) + XXH64 (workers.go:153) + FNV-1 (replicated_hash.go:108) on the
// device, fused with the expansion of the per-limit parameters.  One packed buffer per batch: [gub_kreq x n][uint32 offsets x (n+1)]
// [key bytes], key i = bytes[offsets[i] .. offsets[i+1]).
// kreq_decode: one request of such a batch -> its gub_req record as four 16-byte words (the layout of expand_one).  kr = the request's
// gub_kreq (hits | params, created_delta); key = its len key bytes; params_far != nullptr: the table lives in device memory, else in P.
__device__ __forceinline__ void kreq_decode(const ulonglong2 kr, const uint8_t* key, uint32_t len, const InlineParams& P, uint32_t n_params,
                                            const gub_params* params_far, int64_t created_base, ulonglong2& w0, ulonglong2& w1, ulonglong2& w2,
                                            ulonglong2& w3) {
  uint64_t xxh, fnv;
  hash_key_bytes(key, len, &xxh, &fnv);
  const uint32_t pi = (uint32_t)(kr.y & 0xFFFFFFFFull);
  const bool known = pi < n_params;
  ulonglong2 q0 = make_ulonglong2(0, 0), q1 = q0;
  if (known) {
    if (params_far) { const ulonglong2* pp = reinterpret_cast<const ulonglong2*>(params_far + pi); q0 = __ldg(pp); q1 = __ldg(pp + 1); }
    else { q0 = P.q[pi][0]; q1 = P.q[pi][1]; }
  }
  expand_words(q0, q1, known, make_ulonglong2(xxh, fnv), kr, created_base, w0, w1, w2, w3);
}

__global__ void __launch_bounds__(256) k_hash_expand(const uint8_t* packed, uint32_t n, const InlineParams P, uint32_t n_params, const gub_params* params_far,
                                                     int64_t created_base, gub_req* out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const ulonglong2 kr = __ldcs(reinterpret_cast<const ulonglong2*>(packed) + i);  // hits | params, created_delta
  const uint32_t* offsets = reinterpret_cast<const uint32_t*>(packed + (size_t)n * 16);
  const uint8_t* bytes = packed + (size_t)n * 16 + ((size_t)n + 1) * 4;
  const uint32_t lo = __ldg(offsets + i), hi = __ldg(offsets + i + 1);
  ulonglong2* o = reinterpret_cast<ulonglong2*>(out + i);
  kreq_decode(kr, bytes + lo, hi - lo, P, n_params, params_far, created_base, o[0], o[1], o[2], o[3]);
}

// ---- maintenance kernels -------------------------------------------------------------------------------------
// Upsert whole items: WorkerPool.AddCacheItem / Load / UpdatePeerGlobals.  Keys are unique within one launch.
struct DevItem { uint64_t key, tag; uint64_t w[6]; uint32_t flags; uint32_t _pad; int64_t invalid_at; };

__global__ void k_add_items(Slot* table, uint64_t cap, const DevItem* items, uint32_t n, unsigned long long* counters, uint32_t* failed, InvIndex inv) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const DevItem it = items[i];
  Cursor cur;
  cursor_open(cur, table, cap, it.key, it.tag);
  cur.b.key = it.key; cur.b.tag = it.tag; cur.b.flags = it.flags | (it.invalid_at != 0 ? F_INVALID_AT : 0u);
  if (it.invalid_at != 0) inv_store(inv, it.key, it.tag, it.invalid_at);
  cur.b.limit = (int64_t)it.w[0]; cur.b.duration = (int64_t)it.w[1]; cur.b.rem = it.w[2]; cur.b.stamp = (int64_t)it.w[3];
  cur.b.burst = (int64_t)it.w[4]; cur.b.expire = (int64_t)it.w[5];
  uint32_t ins = 0;
  if (!cursor_close(cur, table, cap, ins)) atomicAdd(failed, 1u);
  if (ins) atomicAdd(counters + C_INSERTS, (unsigned long long)ins);
}

// UpdatePeerGlobals (gubernator.go:425-459): install the owners' UpdatePeerGlobal items (public gub_item records, as built by
// k_make_updates) as this shard's replicas: token {Status, Limit, Duration, Remaining, CreatedAt = now}, leaky {Remaining =
// float64(status.Remaining), Limit, Duration, Burst = Limit, UpdatedAt = now}, ExpireAt = the status' ResetTime.
__global__ void k_add_items_pub(Slot* table, uint64_t cap, const gub_item* items, uint32_t n, int64_t now_ms, unsigned long long* counters, InvIndex inv) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const gub_item it = items[i];
  if (it.algorithm != GUB_TOKEN_BUCKET && it.algorithm != GUB_LEAKY_BUCKET) return;
  Cursor cur;
  const uint64_t key = remap_key(it.key_xxh64), tag = it.key_fnv1 >> 8;
  cursor_open(cur, table, cap, key, tag);
  const bool leaky = it.algorithm == GUB_LEAKY_BUCKET;
  cur.b.key = key; cur.b.tag = tag;
  cur.b.flags = F_LIVE | (leaky ? F_LEAKY : 0u) | ((!leaky && it.status == GUB_OVER_LIMIT) ? F_OVER : 0u) | (it.invalid_at != 0 ? F_INVALID_AT : 0u);
  if (it.invalid_at != 0) inv_store(inv, key, tag, it.invalid_at);
  cur.b.limit = it.limit; cur.b.duration = it.duration;
  cur.b.rem = leaky ? f2bits(it.remaining_f) : (uint64_t)it.remaining;
  cur.b.stamp = now_ms; cur.b.burst = leaky ? it.burst : 0; cur.b.expire = it.expire_at;
  uint32_t ins = 0;
  if (!cursor_close(cur, table, cap, ins)) atomicAdd(counters + C_FULL, 1ull);
  if (ins) atomicAdd(counters + C_INSERTS, (unsigned long long)ins);
}


__global__ void k_get_items(const Slot* table, uint64_t cap, const uint64_t* keys, const uint64_t* fnv, uint32_t n, int64_t now_ms,
                            DevItem* out, uint8_t* found, InvIndex inv) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Cursor cur;
  cursor_open(cur, table, cap, remap_key(keys[i]), fnv[i] >> 8);
  const int64_t inv_at = (cur.found && (cur.b.flags & F_INVALID_AT)) ? inv_lookup(inv, cur.b.key, cur.b.tag) : 0;
  const bool ok = cur.found && (cur.b.flags & F_LIVE) && !(cur.b.expire < now_ms) && !(inv_at != 0 && inv_at < now_ms);  // lrucache.go:111-128, cache.go:43-57
  found[i] = ok ? 1 : 0;
  DevItem o;
  o.key = keys[i]; o.tag = cur.b.tag; o.flags = cur.b.flags; o._pad = 0; o.invalid_at = inv_at;
  o.w[0] = (uint64_t)cur.b.limit; o.w[1] = (uint64_t)cur.b.duration; o.w[2] = cur.b.rem; o.w[3] = (uint64_t)cur.b.stamp;
  o.w[4] = (uint64_t)cur.b.burst; o.w[5] = (uint64_t)cur.b.expire;
  out[i] = o;
}

// Cache.Each: every live item (expired ones included until something removes them, like the reference's map walk).
__global__ void k_scan(const Slot* table, uint64_t cap, DevItem* out, unsigned long long out_cap, unsigned long long* n_out, InvIndex inv) {
  for (uint64_t s = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < cap; s += (uint64_t)gridDim.x * blockDim.x) {
    const ulonglong2 a = __ldcs(reinterpret_cast<const ulonglong2*>(table + s));
    if (a.x > KEY_TOMB && (a.y & F_LIVE)) {
      const unsigned long long k = atomicAdd(n_out, 1ull);
      if (k < out_cap) {
        ulonglong2 a2, b, c, d;
        slot_load(table + s, a2, b, c, d);
        DevItem o;
        o.key = a.x; o.tag = a.y >> 8; o.flags = (uint32_t)(a.y & 0xFF); o._pad = 0;
        o.invalid_at = (o.flags & F_INVALID_AT) ? inv_lookup(inv, o.key, o.tag) : 0;
        o.w[0] = b.x; o.w[1] = b.y; o.w[2] = c.x; o.w[3] = c.y; o.w[4] = d.x; o.w[5] = d.y;
        out[k] = o;
      }
    }
  }
}

// Frees slots whose item is gone (removed, or ExpireAt < now): the batch path only ever marks them not-live.
// (slots [lo, hi): gub_sweep takes the whole table; the library's incremental sweep a slice at a time, between batches.)
__global__ void k_sweep(Slot* table, uint64_t lo, uint64_t hi, int64_t now_ms, unsigned long long* removed) {
  unsigned long long mine = 0;
  for (uint64_t s = lo + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; s < hi; s += (uint64_t)gridDim.x * blockDim.x) {
    const ulonglong2 a = __ldcs(reinterpret_cast<const ulonglong2*>(table + s));
    if (a.x > KEY_TOMB) {
      bool dead = !(a.y & F_LIVE);
      if (!dead) dead = (int64_t)__ldcs(&table[s].w[7]) < now_ms;
      if (dead) { table[s].w[0] = KEY_TOMB; mine++; }
    }
  }
  if (mine) atomicAdd(removed, mine);
}

// Roofline denominator for this path ("HBM random access", SURVEY 8d): every thread reads one pseudo-random 64-byte slot with
// the four 128-bit loads the batch kernels use and writes the same 64 bytes back (`zero` is 0 at run time, unknown at compile
// time, so the stores stay).  The table's contents are unchanged.  Must not run concurrently with a batch.
__global__ void __launch_bounds__(256) k_random_rmw(Slot* table, uint64_t cap, uint64_t n, uint64_t seed, uint64_t zero) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t h = (i + seed) * 0x9E3779B97F4A7C15ull;
    h ^= h >> 32; h *= 0xD6E8FEB86659FD93ull; h ^= h >> 29;
    Slot* s = table + __umul64hi(h, cap);
    ulonglong2 a, b, c, d;
    slot_load(s, a, b, c, d);
    ulonglong2* q = reinterpret_cast<ulonglong2*>(s);
    a.x ^= zero; b.x ^= zero; c.x ^= zero; d.x ^= zero;
    q[0] = a; q[1] = b; q[2] = c; q[3] = d;
  }
}

// ---- multi-GPU routing ----------------------------------------------------------------------------------------
// Owner of a key = first ring point >= FNV-1(key), wrapping (replicated_hash.go:104-119).  Stable partition of the
// batch by owner: per-tile counts -> exclusive scan over (owner, tile) -> ordered scatter.
constexpr int ROUTE_TILE = 1024;  // requests per block

__device__ __forceinline__ uint32_t ring_owner(const uint64_t* pts, const int32_t* peers, uint32_t npts, uint64_t h) {
  uint32_t lo = 0, hi = npts;
  while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (pts[mid] >= h) hi = mid; else lo = mid + 1; }
  if (lo == npts) lo = 0;
  return (uint32_t)peers[lo];
}

// `self` >= 0 turns on GLOBAL handling (gubernator.go:257-269): a GLOBAL request this shard does not own is not forwarded
// but answered from the local replica, so its destination is `self` (bit 7 of dest[] marks it for the scatter to rewrite
// its behaviour bits).  true_owner (optional) always receives the ring owner.
__global__ void __launch_bounds__(256) k_route_count(const gub_req* reqs, uint32_t n, const uint64_t* pts, const int32_t* peers, uint32_t npts,
                                                     uint32_t nshards, uint8_t* owner, uint32_t* tile_counts /* [nshards][ntiles] */, uint32_t ntiles,
                                                     int32_t self, uint8_t* true_owner) {
  __shared__ uint32_t cnt[MAX_SHARDS];
  if (threadIdx.x < MAX_SHARDS) cnt[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t base = blockIdx.x * ROUTE_TILE;
  for (uint32_t k = threadIdx.x; k < ROUTE_TILE; k += blockDim.x) {
    const uint32_t i = base + k;
    if (i < n) {
      uint32_t o = ring_owner(pts, peers, npts, __ldg(&reqs[i].key_fnv1));
      if (true_owner) true_owner[i] = (uint8_t)o;
      uint32_t mark = 0;
      if (self >= 0 && o != (uint32_t)self && (__ldg(&reqs[i].behavior) & GUB_BEHAVIOR_GLOBAL)) { o = (uint32_t)self; mark = 0x80u; }
      owner[i] = (uint8_t)(o | mark);
      atomicAdd(&cnt[o], 1u);
    }
  }
  __syncthreads();
  if (threadIdx.x < nshards) tile_counts[threadIdx.x * ntiles + blockIdx.x] = cnt[threadIdx.x];
}

// one block: exclusive scan of tile_counts in (owner-major, tile-minor) order; also totals per owner
__global__ void __launch_bounds__(1024) k_route_scan(uint32_t* tile_counts, uint32_t total, uint32_t nshards, uint32_t ntiles, uint32_t* counts) {
  __shared__ uint32_t warp_sums[32];
  __shared__ uint32_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (uint32_t base = 0; base < total; base += blockDim.x) {
    const uint32_t k = base + threadIdx.x;
    const uint32_t v = k < total ? tile_counts[k] : 0;
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { uint32_t u = __shfl_up_sync(0xFFFFFFFFu, incl, o); if ((threadIdx.x & 31) >= (uint32_t)o) incl += u; }
    if ((threadIdx.x & 31) == 31) warp_sums[threadIdx.x >> 5] = incl;
    __syncthreads();
    uint32_t off = carry;
    for (uint32_t w = 0; w < (threadIdx.x >> 5); w++) off += warp_sums[w];
    if (k < total) tile_counts[k] = off + incl - v;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) carry = off + incl;
    __syncthreads();
  }
  // totals: owner g covers tile_counts[g*ntiles .. (g+1)*ntiles)
  if (threadIdx.x < nshards) {
    const uint32_t start = tile_counts[threadIdx.x * ntiles];
    const uint32_t end = (threadIdx.x + 1 < nshards) ? tile_counts[(threadIdx.x + 1) * ntiles] : carry;
    counts[threadIdx.x] = end - start;
  }
}

__global__ void __launch_bounds__(256) k_route_scatter(const gub_req* reqs, uint32_t n, const uint8_t* owner, const uint32_t* tile_offsets,
                                                       uint32_t ntiles, uint32_t nshards, gub_req* out_reqs, uint32_t* perm) {
  // ranks inside the tile are computed warp by warp in index order so the partition is stable
  __shared__ uint32_t run[MAX_SHARDS];
  if (threadIdx.x < MAX_SHARDS) run[threadIdx.x] = (threadIdx.x < nshards) ? tile_offsets[threadIdx.x * ntiles + blockIdx.x] : 0;
  __syncthreads();
  const uint32_t base = blockIdx.x * ROUTE_TILE;
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (uint32_t chunk = 0; chunk < ROUTE_TILE; chunk += blockDim.x) {
    // within a chunk of blockDim.x consecutive requests, warps take turns in order
    for (uint32_t w = 0; w < nwarps; w++) {
      if (w == warp) {
        const uint32_t i = base + chunk + threadIdx.x;
        const bool valid = i < n;
        const uint32_t oraw = valid ? owner[i] : 0xFFu;
        const uint32_t o = valid ? (oraw & 0x7Fu) : 0xFFu;
        const uint32_t peers_mask = __match_any_sync(0xFFFFFFFFu, o);
        const uint32_t rank = __popc(peers_mask & ((1u << lane) - 1u));
        const uint32_t leader = __ffs(peers_mask) - 1;
        uint32_t start = 0;
        if (valid && lane == leader) { start = run[o]; run[o] = start + __popc(peers_mask); }
        start = __shfl_sync(0xFFFFFFFFu, start, leader);
        if (valid) {
          const uint32_t dst = start + rank;
          const ulonglong2* src = reinterpret_cast<const ulonglong2*>(reqs + i);
          ulonglong2* d2 = reinterpret_cast<ulonglong2*>(out_reqs + dst);
          ulonglong2 last = __ldg(src + 3);
          if (oraw & 0x80u) {  // GLOBAL on a non-owner: clone with NO_BATCHING set, GLOBAL cleared, IsOwner = false (gubernator.go:408-411)
            uint32_t beh = (uint32_t)(last.y >> 32);
            beh = (beh | (uint32_t)GUB_BEHAVIOR_NO_BATCHING) & ~(uint32_t)(GUB_BEHAVIOR_GLOBAL | GUB_REQ_IS_OWNER);
            last.y = (last.y & 0xFFFFFFFFull) | ((unsigned long long)beh << 32);
          }
          d2[0] = __ldg(src); d2[1] = __ldg(src + 1); d2[2] = __ldg(src + 2); d2[3] = last;
          perm[dst] = i;
        }
      }
      __syncthreads();
    }
  }
}

__global__ void k_unroute(const gub_resp* in, const uint32_t* perm, uint32_t n, gub_resp* out) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const ulonglong2* s = reinterpret_cast<const ulonglong2*>(in + j);
  ulonglong2* d = reinterpret_cast<ulonglong2*>(out + perm[j]);
  d[0] = s[0]; d[1] = s[1];
}

}  // namespace gub
