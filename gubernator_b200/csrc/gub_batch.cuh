// gub_batch.cuh — the rate-limit evaluation path as ONE persistent kernel per batch (sm_90a).
//
// Replaces, for a whole batch at a time, WorkerPool.GetRateLimit -> Worker.handleGetRateLimit -> LRUCache.GetItem ->
// tokenBucket/leakyBucket (workers.go:261-324, lrucache.go:111, algorithms.go:37-493 of mailgun/gubernator v2.4.0) with the
// results of applying the batch's requests one after another in index order (gubernator.go:203) under a frozen clock.
//
// One CTA per SM, 512 threads, one request per thread.  A CTA owns one TILE of consecutive requests per round:
//
//   phase 1  the tile's request records are staged into shared memory with one bulk-async copy (TMA, cp.async.bulk +
//            mbarrier); the tile is grouped by key in a shared-memory table with index-ordered local ranks (per-warp counts,
//            one barrier); the first member of each (tile, key) FRAGMENT joins the batch-wide group entry (64-bit CAS on the
//            key, count += members, fragments += 1), sets the tile's bit in the group's presence bitmap and stores the
//            fragment size; every key's home slot is prefetched into L2.
//   ---- one grid-wide barrier: every fragment of the batch is registered ----
//   phase 2  fragments read their group entry (total members, fragments); a fragment of a key that also occurs in other tiles
//            gets its base rank = sum of the earlier tiles' fragment sizes.  The table is probed WARP-COOPERATIVELY: four
//            lanes per fragment, one 16-byte load each = one coalesced 64-byte slot per quad, tag compare broadcast inside
//            the quad, linear probing until every quad of the warp is done; the slot lands in a shared-memory snapshot.
//            Every request then evaluates run_to_rank(snapshot, request, base + local rank) by itself (closed forms make that
//            O(1)) and stores its 32-byte response.  Nobody writes a slot other tiles may still read: a key confined to one
//            tile is written back by its last member; for a key spread over tiles every fragment checks in on the group
//            entry (atomicAdd) after reading, and the LAST fragment to arrive writes the final state (or, when the group's
//            requests differ, redoes the group in order, segment by segment) and hands the entry back clean.
//
// The request tile is read from HBM exactly once; there is one launch per batch instead of four; the only grid-wide
// synchronisation is the one barrier (plus one per extra round when a batch exceeds (SMs) x 512 requests: 132 x 512 on an H100 SXM).
#pragma once
#if !defined(GUB_EMULATE)
#include <cuda_runtime.h>
#endif
#include <stdint.h>

#include "gub_kernels.cuh"

namespace gub {

constexpr int FB_THREADS = 512;      // threads per CTA = most requests per tile
constexpr int FB_WARPS = FB_THREADS / 32;
constexpr int FB_HT = 1024;          // tile-local key table (load factor <= 0.5)
constexpr int FB_PRES_WORDS = 8;     // presence bitmap: one bit per tile of a round (grid <= 256)
constexpr int FB_MAX_GRID = FB_PRES_WORDS * 32;
constexpr int FB_ROW = FB_MAX_GRID;  // fragment-size row (uint16) per group entry
constexpr int FB_MAX_SEGS = MAX_SHARDS;
constexpr uint32_t FB_AUX_ENTRIES = 1u << 17;  // batch-wide group table (a round of 132 tiles holds <= 67 584 keys; of 256, the grid's limit, 131 072)
constexpr uint32_t G_NONUNIFORM = 1u;
constexpr int FB_OVF_CAP = OVF_CAP;  // items whose insert found the probe window full; placed (with eviction) at the next batch

// Batch-wide group entry.  All zero between batches: whoever finishes a group hands the entry back clean.
struct __align__(32) GEntry {
  unsigned long long key;   // remapped XXH64 (0 = free), claimed with atomicCAS
  unsigned long long cnt;   // [63:32] fragments  [31:0] members
  uint32_t rep;             // round-local index of one member: every fragment's first member is compared with it
  uint32_t flags;           // G_NONUNIFORM
  uint32_t arrived;         // fragments that have read the slot and answered
  uint32_t _pad;
};

struct FSeg {                           // one run of request records, evaluated in order after the previous segment
  const gub_req* reqs;
  gub_resp* out;                        // response j of the segment -> out[j] (may be peer memory)
  const unsigned long long* flag;       // optional: (epoch << 32 | count), published by the producer of the segment
  const uint32_t* n_dev;                // optional: count on the device
  uint32_t n;                           // count when neither is given
  uint32_t _pad;
};

struct FCtl {
  uint32_t bar_cnt, bar_gen;            // grid barrier
  uint32_t chain_done;                  // four-kernel pipeline: epoch of the last batch whose k_finish has finished (BatchArgs::chain_done)
  uint32_t done_ctr;                    // CTAs that have stored all their responses (multi-GPU: the last one publishes the flags)
  uint32_t error;                       // a flag wait timed out (a peer died)
  uint32_t ovf_count;                   // pending items in `ovf`
  unsigned long long sweep_cursor;      // next slot of the incremental expiry sweep
};

struct FArgs {
  Slot* table;
  uint64_t capacity;
  FSeg seg[FB_MAX_SEGS];
  uint32_t nseg;
  uint32_t flag_epoch;                  // epoch the segments' flags must show
  GEntry* aux;
  uint32_t* presence;                   // [FB_AUX_ENTRIES][FB_PRES_WORDS]
  unsigned long long* fragrow;          // [FB_AUX_ENTRIES][FB_ROW] per tile: [63:32] rank of the fragment's first member within the group (written by the
                                        // group's scanner) [31:16] offset of the fragment's members in the tile's list [15:0] fragment size
  uint16_t* members;                    // [FB_MAX_GRID * FB_THREADS] per tile: the members of each of its fragments, contiguous, in index order
  FCtl* ctl;
  OvfItem* ovf;                         // [FB_OVF_CAP]
  unsigned long long* counters;
  // multi-GPU: when every response of this launch has been stored, resp_flag[k] (k < n_resp_flags) receives flag_epoch << 32
  unsigned long long* resp_flag[FB_MAX_SEGS];
  uint32_t n_resp_flags;
  uint32_t sweep_chunk;                 // slots each CTA sweeps per round (0 = off)
  InvIndex inv;                         // CacheItem.InvalidAt side index (see gub_kernels.cuh)
  unsigned long long* trace;            // optional [gridDim.x][FB_TRACE_MARKS]: %globaltimer of every CTA at the phase boundaries (diagnostic)
  gub_clock clk;
};
constexpr int FB_TRACE_MARKS = 12;

// What the rarely taken, out-of-line parts of the kernel need of FArgs, kept in shared memory (a non-inlined function taking the
// kernel's parameter struct by reference would force a 1 KB local copy of it).  Same member names as FArgs.
struct FCtx {
  Slot* table;
  uint64_t capacity;
  GEntry* aux;
  uint32_t* presence;
  unsigned long long* fragrow;
  uint16_t* members;
  FCtl* ctl;
  OvfItem* ovf;
  unsigned long long* counters;
  unsigned long long* trace;
  InvIndex inv;
  uint32_t nseg, sweep_chunk, n_resp_flags, _pad;
  gub_clock clk;
};

// ---- PTX: bulk-async copy (TMA) + mbarrier, acquire/release, grid barrier ---------------------------------------------
#if defined(GUB_EMULATE)
struct MBar { uint64_t w; };
__device__ __forceinline__ void mbar_init(MBar*) {}
__device__ __forceinline__ void tile_load(void* dst, const void* src, uint32_t bytes, MBar*) { std::memcpy(dst, src, bytes); }
__device__ __forceinline__ void mbar_wait(MBar*, uint32_t) {}
__device__ __forceinline__ void spin_pause() { emu::spin_yield(); }
__device__ __forceinline__ uint32_t ld_relaxed_gpu(const uint32_t* p) { return *p; }
__device__ __forceinline__ void st_relaxed_gpu(uint32_t* p, uint32_t v) { *p = v; }
__device__ __forceinline__ uint32_t atomic_add_release_gpu(uint32_t* p, uint32_t v) { const uint32_t o = *p; *p = o + v; return o; }
__device__ __forceinline__ void fence_acquire_gpu() {}
__device__ __forceinline__ uint32_t atomic_add_acq_rel_gpu(uint32_t* p, uint32_t v) { const uint32_t o = *p; *p = o + v; return o; }
#else
struct __align__(8) MBar { uint64_t w; };
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(MBar* b) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_addr(b)) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// One thread: arm the barrier with the byte count and start the copy; the bytes land in shared memory through the async proxy.
__device__ __forceinline__ void tile_load(void* dst, const void* src, uint32_t bytes, MBar* b) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(b)), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_addr(dst)), "l"(src), "r"(bytes),
               "r"(smem_addr(b))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(MBar* b, uint32_t parity) {
  uint32_t ok = 0;
  while (!ok) {
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(ok)
                 : "r"(smem_addr(b)), "r"(parity)
                 : "memory");
  }
}
__device__ __forceinline__ void spin_pause() {}
__device__ __forceinline__ uint32_t ld_relaxed_gpu(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_gpu(uint32_t* p, uint32_t v) { asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ uint32_t atomic_add_release_gpu(uint32_t* p, uint32_t v) {
  uint32_t o;
  asm volatile("atom.add.release.gpu.global.u32 %0, [%1], %2;" : "=r"(o) : "l"(p), "r"(v) : "memory");
  return o;
}
__device__ __forceinline__ void fence_acquire_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
__device__ __forceinline__ uint32_t atomic_add_acq_rel_gpu(uint32_t* p, uint32_t v) {
  uint32_t o;
  asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], %2;" : "=r"(o) : "l"(p), "r"(v) : "memory");
  return o;
}
#endif

#if defined(GUB_EMULATE)
__device__ __forceinline__ void trace_mark(const FCtx&, int) {}
#else
__device__ __forceinline__ void trace_mark(const FCtx& A, int k) {
  if (A.trace && threadIdx.x == 0) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    A.trace[(size_t)blockIdx.x * FB_TRACE_MARKS + k] = t;
  }
}
#endif

// Every CTA of the grid is resident (one per SM, cooperative launch), so a counter + generation barrier is safe.  The
// generation is read before arriving: it cannot advance until this CTA has arrived.
__device__ __forceinline__ void grid_barrier(FCtl* ctl) {
  __syncthreads();
  if (threadIdx.x == 0) {
    const uint32_t gen = ld_acquire_gpu(&ctl->bar_gen);
    if (atomic_add_acq_rel_gpu(&ctl->bar_cnt, 1u) == gridDim.x - 1) {  // release: everything this CTA wrote (cumulative over the barrier above)
      ctl->bar_cnt = 0;
      st_release_gpu(&ctl->bar_gen, gen + 1);
    } else {
      // bounded (seconds): a CTA that never arrives (a fault, a grid that is not co-resident) must not hang the device
      uint32_t it = 0;
      while (ld_acquire_gpu(&ctl->bar_gen) == gen && ++it < (1u << 26)) spin_pause();
      if (it >= (1u << 26)) atomicExch(&ctl->error, 2u);
    }
  }
  __syncthreads();
}

// ---- shared memory of one CTA --------------------------------------------------------------------------------------
// Scratch of one team (a warp, or the whole CTA) evaluating a non-uniform group: the tiles holding its members, the starts of
// its runs of identical requests (segments) and the bucket state entering each segment.
template <int TILES, int SEGS>
struct MixScratch {
  uint32_t nseg, ntile;
  uint32_t cum[TILES + 1];       // members in the tiles before slot j
  uint16_t tile[TILES], off[TILES];
  uint32_t seg[SEGS + 1];        // first member (rank within the group) of every segment, ascending; seg[nseg] = members
  uint8_t kind[SEGS];            // 1: the segment's requests were applied one by one by the planner (no closed form)
  Bucket state[SEGS];            // bucket entering the segment
};
constexpr int MIX_WARP_TILES = 32, MIX_WARP_SEGS = 12, MIX_CTA_SEGS = 96;
constexpr uint32_t MIX_WARP_MAX = 32;  // groups of up to this many members are taken by one warp each, larger ones by the CTA
using MixWarp = MixScratch<MIX_WARP_TILES, MIX_WARP_SEGS>;
using MixCta = MixScratch<FB_MAX_GRID, MIX_CTA_SEGS>;

struct TileInfo { uint32_t seg, off, n; };

struct __align__(128) FSmem {
  gub_req req[FB_THREADS];               // the tile (TMA destination); later: scratch of the CTA-wide evaluation of large non-uniform groups
  ulonglong2 snap[FB_THREADS][4];        // per fragment: the slot as found; later: per-warp scratch of the evaluation of small non-uniform groups
  unsigned long long key[FB_HT];         // tile-local key table
  uint8_t wcnt[FB_HT][FB_WARPS];         // [key slot][warp]: members of the key among the warp's lanes
  long long fslot[FB_THREADS];           // per fragment: slot index when found, else first reusable slot of the window (or -1)
  uint32_t fpos[FB_THREADS];             // per fragment: batch-wide group entry
  uint32_t fbase[FB_THREADS];            // per fragment: rank of its first member within the group
  uint32_t ftotal[FB_THREADS];           // per fragment: members of the whole group
  uint16_t fnfrag[FB_THREADS];           // per fragment: fragments of the whole group
  uint16_t flead[FB_THREADS];            // per fragment: its first member (thread / tile-local request index)
  uint16_t fcnt[FB_THREADS];             // per fragment: members in this tile
  uint16_t f_of_sp[FB_HT];               // key slot -> fragment
  uint16_t sp[FB_THREADS];               // per request: key slot
  uint16_t local[FB_THREADS];            // per request: rank within the fragment
  uint16_t fin[FB_THREADS];              // fragments whose group this CTA finishes
  uint32_t fdone[FB_THREADS];            // per fragment: members that have answered
  uint8_t fready[FB_THREADS];            // per fragment: its first member has published the slot snapshot and the base rank
  uint8_t ffound[FB_THREADS];            // per fragment: key is in the table
  uint8_t fmixed[FB_THREADS];            // per fragment: its members differ (or can never settle): the group takes the segment walk
  FCtx cx;
  uint16_t foff[FB_THREADS];             // per fragment: offset of its members in the tile's member list
  uint32_t moff, wq, last, parity;
  TileInfo ti;                           // this CTA's tile of the current round
  // the batch's segments
  const gub_req* seg_reqs[FB_MAX_SEGS];
  gub_resp* seg_out[FB_MAX_SEGS];
  uint32_t seg_cnt[FB_MAX_SEGS];
  uint32_t seg_tile0[FB_MAX_SEGS + 1];
  uint32_t ts, ntiles, total;
  uint32_t nfrag, nfin;
  uint32_t tally[8];
  MBar mbar;
};

__device__ __forceinline__ TileInfo tile_info(const FSmem& S, uint32_t nseg, uint32_t tl) {
  TileInfo ti;
  uint32_t s = 0;
  while (s + 1 < nseg && tl >= S.seg_tile0[s + 1]) s++;
  ti.seg = s;
  ti.off = (tl - S.seg_tile0[s]) * S.ts;
  ti.n = min(S.ts, S.seg_cnt[s] - ti.off);
  return ti;
}
// Round-local request index i = tile-in-round * FB_THREADS + position in the tile.
__device__ __forceinline__ const gub_req* req_at(const FSmem& S, uint32_t nseg, uint32_t round, uint32_t i) {
  const TileInfo ti = tile_info(S, nseg, round * gridDim.x + i / FB_THREADS);
  return S.seg_reqs[ti.seg] + ti.off + (i % FB_THREADS);
}
__device__ __forceinline__ gub_resp* resp_at(const FSmem& S, uint32_t nseg, uint32_t round, uint32_t i) {
  const TileInfo ti = tile_info(S, nseg, round * gridDim.x + i / FB_THREADS);
  return S.seg_out[ti.seg] + ti.off + (i % FB_THREADS);
}

__device__ __forceinline__ gub_req smem_req(const gub_req* p) {
  const ulonglong2* q = reinterpret_cast<const ulonglong2*>(p);
  const ulonglong2 a = q[0], b = q[1], c = q[2], d = q[3];
  gub_req r;
  r.key_xxh64 = a.x; r.key_fnv1 = a.y; r.hits = (int64_t)b.x; r.limit = (int64_t)b.y; r.duration = (int64_t)c.x;
  r.burst = (int64_t)c.y; r.created_at = (int64_t)d.x; r.algorithm = (uint32_t)(d.y & 0xFFFFFFFFull); r.behavior = (uint32_t)(d.y >> 32);
  return r;
}
__device__ __forceinline__ gub_req global_req(const gub_req* p) {  // written earlier in this launch's lifetime by other devices / kernels: L2
  const ulonglong2* q = reinterpret_cast<const ulonglong2*>(p);
  const ulonglong2 a = __ldcg(q), b = __ldcg(q + 1), c = __ldcg(q + 2), d = __ldcg(q + 3);
  gub_req r;
  r.key_xxh64 = a.x; r.key_fnv1 = a.y; r.hits = (int64_t)b.x; r.limit = (int64_t)b.y; r.duration = (int64_t)c.x;
  r.burst = (int64_t)c.y; r.created_at = (int64_t)d.x; r.algorithm = (uint32_t)(d.y & 0xFFFFFFFFull); r.behavior = (uint32_t)(d.y >> 32);
  return r;
}

// ---- the batch-wide group table ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t gentry_join(const FCtx& A, uint64_t key, bool look_first, bool* claimed) {
  uint32_t pos = (uint32_t)((key * 0x9E3779B97F4A7C15ull) >> 40) & (FB_AUX_ENTRIES - 1);
  *claimed = false;
#pragma unroll 1
  for (;;) {
    // a key with several members in this tile is probably in many tiles: 132 CTAs doing a CAS on one address serialise in L2,
    // so look first (reads of one address do not) and only CAS what looks free
    unsigned long long old = look_first ? __ldcg(&A.aux[pos].key) : 0ull;
    if (old == 0ull) {
      old = atomicCAS(&A.aux[pos].key, 0ull, (unsigned long long)key);
      if (old == 0ull) { *claimed = true; break; }
    }
    if (old == key) break;
    pos = (pos + 1) & (FB_AUX_ENTRIES - 1);
  }
  return pos;
}
__device__ __forceinline__ void gentry_clear(GEntry* e) {
  ulonglong2* p = reinterpret_cast<ulonglong2*>(e);
  __stcg(p, make_ulonglong2(0ull, 0ull));
  __stcg(p + 1, make_ulonglong2(0ull, 0ull));
}

// Sum of the fragment sizes of the tiles before `tt` that hold members of group `pos`.
// ---- base ranks: one scan per group, not one per fragment ----------------------------------------------------------------------
// A fragment's members rank base + 0, base + 1, ... within the group, base = members in the tiles before it.  Every fragment
// summing the row itself costs O(fragments^2) loads per group (a hot key has a fragment in every tile).  Instead ONE fragment of
// each group — picked by key hash among the tiles the group occupies, so the duty spreads evenly over the CTAs — scans the row
// once, warp-cooperatively (64 tiles per step, coalesced), and stores every fragment's base (+ 1: non-zero = published) next to its
// size; the other fragments poll their own row entry: one word is both the flag and the data, so no fence is involved.
__device__ __forceinline__ uint32_t kth_set_bit(const uint32_t bits[FB_PRES_WORDS], uint32_t k) {  // position of the k-th (0-based) set bit
  uint32_t w = 0;
#pragma unroll 1
  for (; w < (uint32_t)FB_PRES_WORDS - 1; w++) { const uint32_t c = __popc(bits[w]); if (k < c) break; k -= c; }
  uint32_t x = bits[w];
  for (; k > 0; k--) x &= x - 1;
  return w * 32 + (uint32_t)(__ffs(x) - 1);
}

__device__ __forceinline__ void scan_group_row(const FCtx& A, uint32_t pos, const uint32_t bits[FB_PRES_WORDS]) {  // whole warp
  const uint32_t lane = threadIdx.x & 31;
  unsigned long long* row = A.fragrow + (size_t)pos * FB_ROW;
  uint32_t carry = 0;
#pragma unroll 1
  for (uint32_t c = 0; c < (uint32_t)FB_PRES_WORDS / 2; c++) {  // 64 tiles per step: lane -> tiles 64c + 2 lane, + 1
    const uint32_t w0 = bits[2 * c], w1 = bits[2 * c + 1];
    if (!(w0 | w1)) continue;
    const uint32_t pair = lane < 16 ? (w0 >> (2 * lane)) & 3u : (w1 >> (2 * (lane - 16))) & 3u;
    ulonglong2 e = make_ulonglong2(0ull, 0ull);
    if (pair) e = __ldcg(reinterpret_cast<const ulonglong2*>(row + 64 * c + 2 * lane));
    const uint32_t v0 = (pair & 1u) ? (uint32_t)(e.x & 0xFFFFull) : 0u, v1 = (pair & 2u) ? (uint32_t)(e.y & 0xFFFFull) : 0u;
    uint32_t incl = v0 + v1;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, incl, o); if (lane >= (uint32_t)o) incl += u; }
    const uint32_t excl = carry + incl - (v0 + v1);
    uint32_t* hi = reinterpret_cast<uint32_t*>(row + 64 * c + 2 * lane);
    if (pair & 1u) st_relaxed_gpu(hi + 1, excl + 1u);        // base + 1: non-zero = published (the finisher of the group zeroes it again)
    if (pair & 2u) st_relaxed_gpu(hi + 3, excl + v0 + 1u);
    carry += __shfl_sync(0xFFFFFFFFu, incl, 31);
  }
}

__device__ __forceinline__ void cursor_from_snapshot(const FCtx& A, const FSmem& S, uint32_t f, uint64_t key, uint64_t tag, Cursor& c) {
  c.home = __umul64hi(key, A.capacity);
  c.found = S.ffound[f] != 0;
  c.slot = S.fslot[f];
  if (c.found) {
    bucket_from(c.b, S.snap[f][0], S.snap[f][1], S.snap[f][2], S.snap[f][3]);
  } else {
    c.b.key = key; c.b.tag = tag; c.b.flags = 0; c.b.limit = 0; c.b.duration = 0; c.b.rem = 0; c.b.stamp = 0; c.b.burst = 0; c.b.expire = 0;
  }
  c.old = c.b;
}

// Writes a key's final state; a new key whose probe window has no free slot is parked (gub_kernels.cuh: close_or_park).
template <class Ctx>
__device__ __forceinline__ void close_or_park(const Ctx& A, Cursor& cur, Tally& t) {
  close_or_park(cur, A.table, A.capacity, A.ovf, &A.ctl->ovf_count, t);
}

// ---- groups whose requests differ ---------------------------------------------------------------------------------------------
// A group's members, in index order, are its fragments in tile order; tile t keeps the members of each of its fragments
// contiguous in members[t * 512 + off ..] (off and size are in the group's fragrow[t]).  The group is a sequence of SEGMENTS
// (runs of identical requests).  A team — one warp for groups of up to 32 members, the whole CTA for larger ones — finds the
// segment starts in parallel (each member compares its request with its predecessor's), one thread then folds the segments in
// order (closed forms: O(1) per segment) keeping the bucket state ENTERING each, writes the final state back, and every member
// evaluates run_to_rank(entering state, request, rank within the segment) by itself.  More segments than the scratch holds
// (or segments whose requests can never settle) are applied one request at a time by the folding thread.
template <int NT> struct TeamOps;
template <> struct TeamOps<32> {
  static __device__ __forceinline__ uint32_t tid() { return threadIdx.x & 31u; }
  static __device__ __forceinline__ void sync() { __syncwarp(); }
};
template <> struct TeamOps<FB_THREADS> {
  static __device__ __forceinline__ uint32_t tid() { return threadIdx.x; }
  static __device__ __forceinline__ void sync() { __syncthreads(); }
};

template <class SC>
__device__ __forceinline__ uint32_t member_at(const FCtx& A, const SC& sc, uint32_t k) {  // round-local index of the group's k-th member
  uint32_t lo = 0, hi = sc.ntile;
  while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (sc.cum[mid] <= k) lo = mid; else hi = mid; }
  const uint32_t t = sc.tile[lo];
  return t * FB_THREADS + (uint32_t)__ldcg(A.members + t * FB_THREADS + sc.off[lo] + (k - sc.cum[lo]));
}

template <int NT, class SC>
__device__ __noinline__ void mixed_group(const FCtx& A, FSmem& S, SC& sc, uint32_t pos, uint32_t total, const uint32_t* bits /* FB_PRES_WORDS */,
                                        uint32_t round, Tally& t) {
  using T = TeamOps<NT>;
  const uint32_t tid = T::tid();
  constexpr uint32_t TILES = sizeof(sc.tile) / sizeof(sc.tile[0]), SEGS = sizeof(sc.kind);
  // 1. the tiles that hold members, in order, with their member counts
  if (tid == 0) { sc.nseg = 0; sc.ntile = 0; }
  T::sync();
  const unsigned long long* row = A.fragrow + (size_t)pos * FB_ROW;
  for (uint32_t b = tid; b < (uint32_t)FB_MAX_GRID; b += NT) {
    if (!((bits[b >> 5] >> (b & 31)) & 1u)) continue;
    uint32_t slot = __popc(bits[b >> 5] & ((1u << (b & 31)) - 1u));
    for (uint32_t w = 0; w < (b >> 5); w++) slot += __popc(bits[w]);
    if (slot < TILES) {
      const uint32_t r = (uint32_t)(__ldcg(row + b) & 0xFFFFFFFFull);
      sc.tile[slot] = (uint16_t)b; sc.off[slot] = (uint16_t)(r >> 16); sc.cum[slot + 1] = r & 0xFFFFu;
    }
    atomicAdd(&sc.ntile, 1u);
  }
  T::sync();
  if (tid == 0) {
    sc.cum[0] = 0;
    const uint32_t nt = min(sc.ntile, TILES);
    sc.ntile = nt;
    for (uint32_t j = 0; j < nt; j++) sc.cum[j + 1] += sc.cum[j];
  }
  T::sync();
  // 2. segment starts: members whose request differs from their predecessor's
  for (uint32_t k = tid; k < total; k += NT) {
    bool boundary = k == 0;
    if (!boundary) {
      const gub_req a = global_req(req_at(S, A.nseg, round, member_at(A, sc, k))), b = global_req(req_at(S, A.nseg, round, member_at(A, sc, k - 1)));
      boundary = !req_same(a, b);
    }
    if (boundary) { const uint32_t q = atomicAdd(&sc.nseg, 1u); if (q < SEGS) sc.seg[q] = k; }
  }
  T::sync();
  const uint32_t nseg = sc.nseg;
  // 3. one thread folds the segments in order
  if (tid == 0) {
    Cursor cur;
    bool open = false;
    uint64_t ck = 0, ct = 0;
    if (nseg <= SEGS) {
      for (uint32_t a = 1; a < nseg; a++) {  // the starts arrived in any order
        const uint32_t v = sc.seg[a];
        int b = (int)a - 1;
        while (b >= 0 && sc.seg[b] > v) { sc.seg[b + 1] = sc.seg[b]; b--; }
        sc.seg[b + 1] = v;
      }
      sc.seg[nseg] = total;
    }
    const uint32_t steps = nseg <= SEGS ? nseg : 1u;
#pragma unroll 1
    for (uint32_t sgi = 0; sgi < steps; sgi++) {
      const uint32_t lo = nseg <= SEGS ? sc.seg[sgi] : 0u, hi = nseg <= SEGS ? sc.seg[sgi + 1] : total;
      gub_req rq = global_req(req_at(S, A.nseg, round, member_at(A, sc, lo)));
      const bool closed_form = nseg <= SEGS && req_regular(rq);
      if (nseg <= SEGS) sc.kind[sgi] = closed_form ? 0 : 1;
#pragma unroll 1
      for (uint32_t k = lo; k < hi; k++) {  // closed form: one pass for the whole segment; else one pass per request
        uint32_t i_k = 0;
        if (!closed_form) { i_k = member_at(A, sc, k); if (k > lo) rq = global_req(req_at(S, A.nseg, round, i_k)); }
        const uint64_t key = remap_key(rq.key_xxh64), tag = rq.key_fnv1 >> 8;
        if (!open || key != ck || tag != ct) {  // (the key only changes when two keys share their XXH64)
          if (open) close_or_park(A, cur, t);
          cursor_open(cur, A.table, A.capacity, key, tag);
          apply_invalid_at(A.inv, cur.b, cur.found, A.clk.now_ms);
          open = true; ck = key; ct = tag;
        }
        Delta d = {0, 0, 0};
        if (closed_form) {
          sc.state[sgi] = cur.b;
          run_to_rank(cur.b, rq, hi - lo - 1, A.clk, d);
          t.over += d.over; t.hit += d.hit; t.miss += d.miss;
          break;
        }
        const gub_resp r = apply_one(cur.b, rq, A.clk, d);
        t.over += d.over; t.hit += d.hit; t.miss += d.miss;
        store_resp(resp_at(S, A.nseg, round, i_k), r);
      }
    }
    if (nseg > SEGS) atomicAdd(A.counters + C_SERIAL, 1ull);
    if (open) close_or_park(A, cur, t);
  }
  T::sync();
  // 4. every member of a closed-form segment answers for itself
  if (nseg <= SEGS) {
    for (uint32_t k = tid; k < total; k += NT) {
      uint32_t lo = 0, hi = nseg;
      while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (sc.seg[mid] <= k) lo = mid; else hi = mid; }
      if (sc.kind[lo]) continue;
      const uint32_t i_k = member_at(A, sc, k);
      const gub_req rq = global_req(req_at(S, A.nseg, round, i_k));
      Bucket b = sc.state[lo];
      Delta d = {0, 0, 0};
      store_resp(resp_at(S, A.nseg, round, i_k), run_to_rank(b, rq, k - sc.seg[lo], A.clk, d));
    }
  }
  T::sync();
}

// The tiles of a group that is being finished: its presence bitmap, or just this tile.
__device__ __forceinline__ void group_bits(const FCtx& A, uint32_t pos, bool spread, uint32_t bits[FB_PRES_WORDS]) {
#pragma unroll
  for (int w = 0; w < FB_PRES_WORDS; w++) bits[w] = 0;
  if (spread) {
    const uint4* pres = reinterpret_cast<const uint4*>(A.presence + (size_t)pos * FB_PRES_WORDS);
    const uint4 p0 = __ldcg(pres), p1 = __ldcg(pres + 1);
    bits[0] = p0.x; bits[1] = p0.y; bits[2] = p0.z; bits[3] = p0.w; bits[4] = p1.x; bits[5] = p1.y; bits[6] = p1.z; bits[7] = p1.w;
  } else {
    bits[blockIdx.x >> 5] = 1u << (blockIdx.x & 31);
  }
}
__device__ __forceinline__ void group_release(const FCtx& A, uint32_t pos) {  // hands the entry, its bitmap and the published bases back clean
  uint4* pz = reinterpret_cast<uint4*>(A.presence + (size_t)pos * FB_PRES_WORDS);
  const uint4 p0 = __ldcg(pz), p1 = __ldcg(pz + 1);
  const uint32_t bits[FB_PRES_WORDS] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
  uint32_t* row = reinterpret_cast<uint32_t*>(A.fragrow + (size_t)pos * FB_ROW);
#pragma unroll 1
  for (uint32_t w = 0; w < (uint32_t)FB_PRES_WORDS; w++)
    for (uint32_t x = bits[w]; x; x &= x - 1) st_relaxed_gpu(row + 2 * (w * 32 + (uint32_t)__ffs(x) - 1) + 1, 0u);
  __stcg(pz, make_uint4(0u, 0u, 0u, 0u)); __stcg(pz + 1, make_uint4(0u, 0u, 0u, 0u));
  gentry_clear(&A.aux[pos]);
}

// All non-uniform groups this CTA finishes (S.fin, entries 0xFFFF are done): small ones are dealt to the warps, large ones
// take the whole CTA one after another.
__device__ __noinline__ void finish_mixed_groups(FSmem& S, uint32_t nfin, uint32_t round, Tally& t, uint32_t& dup, uint32_t& mixed_groups) {
  const FCtx& A = S.cx;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) S.wq = 0;
  __syncthreads();
  static_assert(sizeof(MixWarp) * FB_WARPS <= sizeof(S.snap), "per-warp scratch lives in the snapshot area");
  static_assert(sizeof(MixCta) <= sizeof(S.req), "CTA scratch lives in the tile area");
  MixWarp& wsc = reinterpret_cast<MixWarp*>(&S.snap[0][0])[warp];
  for (;;) {
    uint32_t k = 0;
    if (lane == 0) k = atomicAdd(&S.wq, 1u);
    k = __shfl_sync(0xFFFFFFFFu, k, 0);
    if (k >= nfin) break;
    const uint32_t ff = S.fin[k];
    if (ff == 0xFFFFu || S.ftotal[ff] > MIX_WARP_MAX) continue;
    const uint32_t pos = S.fpos[ff];
    const bool spread = S.fnfrag[ff] > 1;
    uint32_t bits[FB_PRES_WORDS];
    group_bits(A, pos, spread, bits);
    mixed_group<32>(A, S, wsc, pos, S.ftotal[ff], bits, round, t);
    if (lane == 0) { dup++; mixed_groups++; if (spread) group_release(A, pos); }
  }
  __syncthreads();
  MixCta& csc = *reinterpret_cast<MixCta*>(&S.req[0]);
#pragma unroll 1
  for (uint32_t k = 0; k < nfin; k++) {
    const uint32_t ff = S.fin[k];
    if (ff == 0xFFFFu || S.ftotal[ff] <= MIX_WARP_MAX) continue;
    const uint32_t pos = S.fpos[ff];
    const bool spread = S.fnfrag[ff] > 1;
    uint32_t bits[FB_PRES_WORDS];
    group_bits(A, pos, spread, bits);
    mixed_group<FB_THREADS>(A, S, csc, pos, S.ftotal[ff], bits, round, t);
    if (tid == 0) { dup++; mixed_groups++; if (spread) group_release(A, pos); }
  }
  __syncthreads();
}

// ---- maintenance inside the batch kernel (both run before the grid barrier, when nothing reads the table) -------------------
// Items parked by close_or_park(): one warp places them (gub_kernels.cuh: drain_parked).
__device__ __forceinline__ void drain_overflow(const FCtx& A, Tally& t) {
  drain_parked(A.table, A.capacity, A.ovf, &A.ctl->ovf_count, A.clk.now_ms, A.counters, &t.inserts);
}

// Incremental expiry sweep: every CTA frees the removed / expired entries of a few slots per round (tombstones; a tombstone
// run that ends at an empty slot becomes empty again), so that a long-running service does not fill its probe windows with
// dead keys.  The reference frees them lazily on access (lrucache.go:115) and by LRU eviction (lrucache.go:138).
__device__ __noinline__ void sweep_slice(const FCtx& A, uint32_t* swept) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t start = (__ldcg(&A.ctl->sweep_cursor) + (uint64_t)blockIdx.x * A.sweep_chunk) % A.capacity;
#pragma unroll 1
  for (uint32_t c0 = 0; c0 < A.sweep_chunk; c0 += 32) {
    const uint32_t k = c0 + lane;
    const bool in = k < A.sweep_chunk;
    const uint64_t idx = (start + k) % A.capacity;
    uint32_t cls = 2;  // 0 empty, 1 tombstone (or about to be), 2 live
    if (in) {
      const ulonglong2 a = __ldcs(reinterpret_cast<const ulonglong2*>(A.table + idx));
      if (a.x == KEY_EMPTY) cls = 0;
      else if (a.x == KEY_TOMB) cls = 1;
      else if (!(a.y & F_LIVE) || (int64_t)__ldcs(&A.table[idx].w[7]) < A.clk.now_ms) { cls = 1; A.table[idx].w[0] = KEY_TOMB; (*swept)++; }
    }
    // the slot after the warp's 32: decides whether a trailing tombstone run may become empty
    uint64_t nxt = start + c0 + 32; nxt %= A.capacity;
    const unsigned long long after = __ldcs(&A.table[nxt].w[0]);
    const uint64_t E = (uint64_t)__ballot_sync(0xFFFFFFFFu, in && cls == 0) | ((after == KEY_EMPTY && c0 + 32 <= A.sweep_chunk) ? (1ull << 32) : 0ull);
    const uint64_t T = (uint64_t)__ballot_sync(0xFFFFFFFFu, in && cls == 1);
    if (in && cls == 1) {
      const uint64_t notT = ~T >> lane;                 // first slot at or above mine that is not a tombstone
      const uint32_t m = lane + (uint32_t)__ffsll((long long)notT) - 1;
      if (m <= 32 && ((E >> m) & 1ull)) A.table[idx].w[0] = KEY_EMPTY;
    }
  }
}

// ---- the kernel -----------------------------------------------------------------------------------------------------------
#if defined(GUB_EMULATE)
#define GUB_DYN_SMEM() (emu::dyn_smem())
#else
extern __shared__ __align__(128) unsigned char gub_dyn_smem[];
#define GUB_DYN_SMEM() (gub_dyn_smem)
#endif

__device__ __forceinline__ uint32_t segment_count(const FArgs& A, uint32_t s) {
  const FSeg& g = A.seg[s];
  if (g.flag) {
    for (uint32_t it = 0; it < 20000000u; it++) {
      const unsigned long long v = ld_acquire_sys(g.flag);
      if ((uint32_t)(v >> 32) == A.flag_epoch) return (uint32_t)(v & 0xFFFFFFFFull);
      __nanosleep(100);
    }
    atomicExch(&A.ctl->error, 1u);  // a peer died: its segment counts as empty; the host reads the flag after the step
    return 0;
  }
  if (g.n_dev) return min(__ldcg(g.n_dev), g.n);
  return g.n;
}

// Folds a phase's counter deltas into the CTA's shared-memory tally.
__device__ __forceinline__ void tally_to_smem(FSmem& S, const Tally& t, uint32_t dup, uint32_t mixed_groups, uint32_t swept) {
  const uint32_t v[8] = {t.over, t.hit, t.miss, t.inserts, t.full, dup, mixed_groups, swept};
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const uint32_t s = __reduce_add_sync(0xFFFFFFFFu, v[k]);
    if ((threadIdx.x & 31) == 0 && s) atomicAdd(&S.tally[k], s);
  }
}

// ---- phase 1 of a round: stage the tile, group it by key, register the fragments (see the header of this file) ----------------
__device__ __noinline__ void batch_phase1(FSmem& S, uint32_t round) {
  const FCtx& A = S.cx;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t ntiles = S.ntiles;
  Tally t = {0, 0, 0, 0, 0};
  uint32_t swept = 0;
  // =============================== phase 1: stage, group, register ===============================
  const uint32_t tl = round * gridDim.x + blockIdx.x;
  TileInfo ti = {0, 0, 0};
  if (tl < ntiles) ti = tile_info(S, A.nseg, tl);
  const uint32_t n_t = ti.n;
  if (tid == 0) S.ti = ti;
  if (tid == 0 && n_t) tile_load(&S.req[0], S.seg_reqs[ti.seg] + ti.off, n_t * (uint32_t)sizeof(gub_req), &S.mbar);
  {
    ulonglong2* kz = reinterpret_cast<ulonglong2*>(&S.key[0]);  // 8 KB
    kz[tid] = make_ulonglong2(0ull, 0ull);
    ulonglong2* wz = reinterpret_cast<ulonglong2*>(&S.wcnt[0][0]);  // 16 KB
    wz[tid] = make_ulonglong2(0ull, 0ull);
    wz[tid + FB_THREADS] = make_ulonglong2(0ull, 0ull);
    S.fmixed[tid] = 0; S.fready[tid] = 0; S.fdone[tid] = 0;
  }
  if (tid == 0) S.moff = 0;
  __syncthreads();
  if (round == 0) trace_mark(A, 1);
  if (n_t) mbar_wait(&S.mbar, S.parity);
  if (round == 0) trace_mark(A, 2);
  const bool valid = tid < n_t;
  uint64_t key = 0;
  uint32_t sp = 0xFFFFu;
  if (valid) {
    key = remap_key(S.req[tid].key_xxh64);
    const uint64_t home = __umul64hi(key, A.capacity);
    prefetch_l2(A.table + home);
    prefetch_l2(A.table + (home + 1 == A.capacity ? 0 : home + 1));
    sp = (uint32_t)((key * 0x9E3779B97F4A7C15ull) >> 54);  // top 10 bits -> FB_HT
#pragma unroll 1
    for (;;) {
      const unsigned long long old = atomicCAS(&S.key[sp], 0ull, (unsigned long long)key);
      if (old == 0ull || old == key) break;
      sp = (sp + 1) & (FB_HT - 1);
    }
  }
  __syncthreads();
  // index-ordered rank inside the tile: members in earlier warps + earlier lanes of my warp
  const uint32_t peers = __match_any_sync(0xFFFFFFFFu, valid ? sp : (0x10000u | lane));
  if (valid && lane == (uint32_t)(__ffs(peers) - 1)) S.wcnt[sp][warp] = (uint8_t)__popc(peers);
  __syncthreads();
  uint32_t local = 0;
  if (valid) {
    const uint4 wc = *reinterpret_cast<const uint4*>(&S.wcnt[sp][0]);
    const uint32_t wv[4] = {wc.x, wc.y, wc.z, wc.w};
    uint32_t before = 0, total = 0;
#pragma unroll
    for (int w = 0; w < FB_WARPS; w++) {
      const uint32_t c = (wv[w >> 2] >> (8 * (w & 3))) & 0xFFu;
      total += c;
      before += ((uint32_t)w < warp) ? c : 0u;
    }
    local = before + __popc(peers & ((1u << lane) - 1u));
    S.sp[tid] = (uint16_t)sp; S.local[tid] = (uint16_t)local;
    if (local == 0) {  // the fragment's first member registers it
      const uint32_t f = atomicAdd(&S.nfrag, 1u);
      S.f_of_sp[sp] = (uint16_t)f; S.flead[f] = (uint16_t)tid; S.fcnt[f] = (uint16_t)total;
      bool claimed;
      const uint32_t pos = gentry_join(A, key, total > 1, &claimed);
      atomicAdd(&A.aux[pos].cnt, (1ull << 32) | (unsigned long long)total);
      if (claimed) A.aux[pos].rep = blockIdx.x * FB_THREADS + tid;
      atomicOr(&A.presence[(size_t)pos * FB_PRES_WORDS + (blockIdx.x >> 5)], 1u << (blockIdx.x & 31));
      const uint32_t foff = atomicAdd(&S.moff, total);  // this fragment's place in the tile's member list
      S.foff[f] = (uint16_t)foff;
      A.fragrow[(size_t)pos * FB_ROW + blockIdx.x] = (foff << 16) | total;
      S.fpos[f] = pos;
    }
  }
  // maintenance: nothing reads the table before the barrier
  if (blockIdx.x == 0 && warp == 0 && __ldcg(&A.ctl->ovf_count)) drain_overflow(S.cx, t);
  if (A.sweep_chunk && warp == FB_WARPS - 1 && !__ldcg(&A.ctl->ovf_count)) sweep_slice(S.cx, &swept);  // (a pending placement may pick a slot the sweep is freeing)

  tally_to_smem(S, t, 0, 0, swept);
}

// ---- phase 2 of a round: probe, evaluate, finish ---------------------------------------------------------------------------------
__device__ __noinline__ void batch_phase2(FSmem& S, uint32_t round) {
  const FCtx& A = S.cx;
  const uint32_t tid = threadIdx.x;
  const TileInfo ti = S.ti;
  const bool valid = tid < ti.n;
  const uint32_t sp = S.sp[tid], local = S.local[tid];
  const uint64_t key = valid ? remap_key(S.req[tid].key_xxh64) : 0;
  Tally t = {0, 0, 0, 0, 0};
  uint32_t dup = 0, mixed_groups = 0;
  // =============================== phase 2: probe, evaluate, finish ===============================
  // No block-wide barrier from here to the end of the evaluation: every warp runs on its own.  A fragment's first member
  // (its leader) reads the group entry, computes the base rank, probes the table and publishes the slot for its siblings
  // through shared memory (flag per fragment; siblings sit in the same or a later warp).  Every member answers for itself.
  // The member that completes a fragment (shared-memory counter) checks the fragment in on the group entry; the last
  // fragment to arrive finishes the group.
  if (A.sweep_chunk && blockIdx.x == 0 && tid == 0) A.ctl->sweep_cursor = (A.ctl->sweep_cursor + (uint64_t)gridDim.x * A.sweep_chunk) % A.capacity;
  uint32_t f = 0, lead = 0, cnt = 0, nfrag = 1, total = 1, base = 0, lpos = 0;
  gub_req rq;
  Cursor cur;
  bool have_cur = false, is_scanner = false;
  uint32_t pbits[FB_PRES_WORDS];
#pragma unroll
  for (int w = 0; w < FB_PRES_WORDS; w++) pbits[w] = 0;
  if (valid) {
    rq = smem_req(&S.req[tid]);
    f = S.f_of_sp[sp]; lead = S.flead[f]; cnt = S.fcnt[f];
    if (tid == lead) {
      lpos = S.fpos[f];
      // the group entry, its presence bitmap, and the probe: all issued before any is consumed
      const ulonglong2 e0 = __ldcg(reinterpret_cast<const ulonglong2*>(&A.aux[lpos]));
      const uint32_t e_rep = __ldcg(&A.aux[lpos].rep);
      const uint4* pres = reinterpret_cast<const uint4*>(A.presence + (size_t)lpos * FB_PRES_WORDS);
      const uint4 p0 = __ldcg(pres), p1 = __ldcg(pres + 1);
      cursor_open(cur, A.table, A.capacity, key, rq.key_fnv1 >> 8);
      apply_invalid_at(A.inv, cur.b, cur.found, A.clk.now_ms);
      have_cur = true;
      total = (uint32_t)(e0.y & 0xFFFFFFFFull); nfrag = (uint32_t)(e0.y >> 32);
      if (nfrag > 1) {
        pbits[0] = p0.x; pbits[1] = p0.y; pbits[2] = p0.z; pbits[3] = p0.w; pbits[4] = p1.x; pbits[5] = p1.y; pbits[6] = p1.z; pbits[7] = p1.w;
        is_scanner = kth_set_bit(pbits, (uint32_t)(key >> 17) % nfrag) == blockIdx.x;
        if (e_rep != blockIdx.x * FB_THREADS + tid) {  // uniformity across tiles: every fragment's first member == the representative
          const gub_req rr = global_req(req_at(S, A.nseg, round, e_rep));
          if (!req_same(rq, rr)) atomicOr(&A.aux[lpos].flags, G_NONUNIFORM);
        }
      } else {  // the key lives in this tile only: hand the entry and the bitmap word back now
        A.presence[(size_t)lpos * FB_PRES_WORDS + (blockIdx.x >> 5)] = 0;
        gentry_clear(&A.aux[lpos]);
      }
    }
  }
  // the groups this warp scans (see scan_group_row)
  for (uint32_t m = __ballot_sync(0xFFFFFFFFu, is_scanner); m; m &= m - 1) {
    const uint32_t src = __ffs(m) - 1;
    uint32_t bits[FB_PRES_WORDS];
#pragma unroll
    for (int w = 0; w < FB_PRES_WORDS; w++) bits[w] = __shfl_sync(0xFFFFFFFFu, pbits[w], src);
    const uint32_t spos = __shfl_sync(0xFFFFFFFFu, lpos, src);
    scan_group_row(A, spos, bits);
  }
  if (valid && tid == lead) {
    if (nfrag > 1) {  // the group's scanner (maybe a lane of this very warp, above) publishes base + 1 in our row entry
      const uint32_t* hi = reinterpret_cast<const uint32_t*>(A.fragrow + (size_t)lpos * FB_ROW + blockIdx.x) + 1;
      uint32_t v = ld_relaxed_gpu(hi), it = 0;
      while (v == 0 && ++it < (1u << 26)) { spin_pause(); v = ld_relaxed_gpu(hi); }
      base = v - 1u;
    }
    S.fbase[f] = base; S.ftotal[f] = total; S.fnfrag[f] = (uint16_t)nfrag;
    if (cnt > 1 || nfrag > 1) {  // somebody else (a sibling, or whoever finishes the group from this CTA) needs the slot as found
      const Bucket& b = cur.b;
      S.snap[f][0] = make_ulonglong2(b.key, (b.tag << 8) | (uint64_t)(b.flags & 0xFF));
      S.snap[f][1] = make_ulonglong2((uint64_t)b.limit, (uint64_t)b.duration);
      S.snap[f][2] = make_ulonglong2(b.rem, (uint64_t)b.stamp);
      S.snap[f][3] = make_ulonglong2((uint64_t)b.burst, (uint64_t)b.expire);
      S.fslot[f] = cur.slot; S.ffound[f] = cur.found ? 1 : 0;
      __threadfence_block();
      *reinterpret_cast<volatile uint8_t*>(&S.fready[f]) = 1;
    }
  }
  __syncwarp();  // a leader and its siblings in this warp: published before anybody below waits
  if (round == 0) trace_mark(A, 5);
  if (valid) {
    if (!have_cur) {
      while (*reinterpret_cast<volatile uint8_t*>(&S.fready[f]) == 0) spin_pause();
      __threadfence_block();
      cursor_from_snapshot(A, S, f, key, rq.key_fnv1 >> 8, cur);
      base = S.fbase[f]; total = S.ftotal[f]; nfrag = S.fnfrag[f];
    }
    // uniformity inside the fragment: every member == the fragment's first, and can settle
    bool irregular = false;
    if (total > 1) {
      irregular = !req_regular(rq);
      if (tid != lead && !irregular) irregular = !req_same(rq, smem_req(&S.req[lead]));
      if (irregular) *reinterpret_cast<volatile uint8_t*>(&S.fmixed[f]) = 1;
      A.members[blockIdx.x * FB_THREADS + S.foff[f] + local] = (uint16_t)tid;  // the group's member list, should it need one
    }
    Delta d = {0, 0, 0};
    if (!irregular) store_resp(S.seg_out[ti.seg] + ti.off + tid, run_to_rank(cur.b, rq, base + local, A.clk, d));
    // the member that completes the fragment speaks for it
    bool completer = true;
    if (cnt > 1) { __threadfence_block(); completer = atomicAdd(&S.fdone[f], 1u) + 1u == cnt; }
    if (completer) {
      const bool mixedf = cnt > 1 ? *reinterpret_cast<volatile uint8_t*>(&S.fmixed[f]) != 0 : irregular;
      const uint32_t pos = S.fpos[f];
      uint32_t fin_kind = 0;  // 1: finish a uniform group from the snapshot, 2: a group whose requests differ
      if (nfrag == 1) {
        if (mixedf) fin_kind = 2;
        else if (cnt == 1) {  // a key seen once: its state is in my registers
          t.over += d.over; t.hit += d.hit; t.miss += d.miss;
          close_or_park(A, cur, t);
        } else fin_kind = 1;
      } else {
        if (mixedf) atomicOr(&A.aux[pos].flags, G_NONUNIFORM);
        if (A.n_resp_flags) __threadfence_system();  // responses in peer memory: system scope
        // release: this CTA's slot reads and response stores precede the check-in (cumulative over the shared-memory counter above)
        if (atomic_add_release_gpu(&A.aux[pos].arrived, 1u) == nfrag - 1) {  // every other fragment has read the slot and answered: finish the group
          fence_acquire_gpu();
          fin_kind = (__ldcg(&A.aux[pos].flags) & G_NONUNIFORM) ? 2u : 1u;
        }
      }
      if (fin_kind) S.fin[atomicAdd(&S.nfin, 1u)] = (uint16_t)(f | (fin_kind == 2 ? 0x8000u : 0u));
    }
  }
  if (round == 0) trace_mark(A, 7);
  tally_to_smem(S, t, dup, mixed_groups, 0);
}

// ---- end of a round: groups this CTA finishes ---------------------------------------------------------------------------------------
__device__ __noinline__ void batch_finish(FSmem& S, uint32_t round) {
  const FCtx& A = S.cx;
  const uint32_t tid = threadIdx.x;
  Tally t = {0, 0, 0, 0, 0};
  uint32_t dup = 0, mixed_groups = 0;
  __syncthreads();
  if (round == 0) trace_mark(A, 8);
  // (a) repeated keys whose requests are all the same: one thread each evaluates the run's last rank from the slot as found
  //     and writes the final state; (b) groups whose requests differ (rare): the teams of this CTA evaluate them
  {
    const uint32_t nfin = S.nfin;
    bool mixed_here = false;
    for (uint32_t k = tid; k < nfin; k += FB_THREADS) {
      const uint32_t e = S.fin[k], ff = e & 0x7FFFu;
      if (e & 0x8000u) { S.fin[k] = (uint16_t)ff; mixed_here = true; continue; }
      S.fin[k] = 0xFFFFu;
      const gub_req lr = smem_req(&S.req[S.flead[ff]]);
      Cursor c2;
      cursor_from_snapshot(A, S, ff, remap_key(lr.key_xxh64), lr.key_fnv1 >> 8, c2);
      Delta d2 = {0, 0, 0};
      run_to_rank(c2.b, lr, S.ftotal[ff] - 1, A.clk, d2);
      t.over += d2.over; t.hit += d2.hit; t.miss += d2.miss;
      close_or_park(A, c2, t);
      dup++;
      if (S.fnfrag[ff] > 1) group_release(S.cx, S.fpos[ff]);
    }
    if (round == 0) trace_mark(A, 9);
    if (__syncthreads_or(mixed_here)) finish_mixed_groups(S, nfin, round, t, dup, mixed_groups);
  }
  tally_to_smem(S, t, dup, mixed_groups, 0);
}

__global__ void __launch_bounds__(FB_THREADS, 1) k_batch(const FArgs A) {
  FSmem& S = *reinterpret_cast<FSmem*>(GUB_DYN_SMEM());
  const uint32_t tid = threadIdx.x;
  if (tid == 0) {
    mbar_init(&S.mbar); S.nfrag = 0; S.nfin = 0; S.parity = 0;
    S.cx.table = A.table; S.cx.capacity = A.capacity; S.cx.fragrow = A.fragrow; S.cx.members = A.members; S.cx.presence = A.presence; S.cx.aux = A.aux; S.cx.ctl = A.ctl;
    S.cx.ovf = A.ovf; S.cx.counters = A.counters; S.cx.trace = A.trace; S.cx.inv = A.inv; S.cx.nseg = A.nseg; S.cx.sweep_chunk = A.sweep_chunk; S.cx.n_resp_flags = A.n_resp_flags;
    S.cx.clk = A.clk;
  }
  if (tid < 8) S.tally[tid] = 0;
  __syncthreads();
  trace_mark(S.cx, 0);
  pdl_wait();     // everything earlier in the stream (the producer of the records, the previous batch) is complete and visible
  pdl_release();
  if (tid < A.nseg) {
    S.seg_cnt[tid] = segment_count(A, tid);
    S.seg_reqs[tid] = A.seg[tid].reqs;
    S.seg_out[tid] = A.seg[tid].out;
  }
  __syncthreads();
  if (tid == 0) {
    uint32_t total = 0;
    for (uint32_t s = 0; s < A.nseg; s++) total += S.seg_cnt[s];
    // tile size: spread the batch over the grid (segments end with a partial tile each)
    const uint32_t usable = gridDim.x > A.nseg ? gridDim.x - A.nseg : 1u;
    uint32_t ts = (total + usable - 1) / usable;
    ts = (ts + 31u) & ~31u;
    if (ts < 32u) ts = 32u;
    if (ts > (uint32_t)FB_THREADS) ts = FB_THREADS;
    uint32_t tiles = 0;
    for (uint32_t s = 0; s < A.nseg; s++) { S.seg_tile0[s] = tiles; tiles += (S.seg_cnt[s] + ts - 1) / ts; }
    S.seg_tile0[A.nseg] = tiles;
    S.ts = ts; S.ntiles = tiles; S.total = total;
  }
  __syncthreads();
  const uint32_t ntiles = S.ntiles;
  const uint32_t rounds = (ntiles + gridDim.x - 1) / gridDim.x;
  if (blockIdx.x == 0 && tid == 0) {
    atomicAdd(A.counters + C_REQUESTS, (unsigned long long)S.total);
    atomicAdd(A.counters + C_BATCHES, 1ull);
  }

#pragma unroll 1
  for (uint32_t round = 0; round < max(rounds, 1u); round++) {
    batch_phase1(S, round);
    if (round == 0) trace_mark(S.cx, 3);
    grid_barrier(A.ctl);
    if (round == 0) trace_mark(S.cx, 4);
    batch_phase2(S, round);
    batch_finish(S, round);
    __syncthreads();
    if (tid == 0) { S.nfrag = 0; S.nfin = 0; if (S.ti.n) S.parity ^= 1u; }
    if (round + 1 < rounds) grid_barrier(A.ctl);  // the next round's groups start from a clean group table and the updated slots
  }

  trace_mark(S.cx, 10);
  // ---- counters: summed per CTA first ----
  __syncthreads();
  if (tid < 8 && S.tally[tid]) {
    const int slot[8] = {C_OVER, C_HIT, C_MISS, C_INSERTS, C_FULL, C_DUP_GROUPS, C_MIXED_GROUPS, C_SWEPT};
    atomicAdd(A.counters + slot[tid], (unsigned long long)S.tally[tid]);
  }
  trace_mark(S.cx, 11);
  // ---- multi-GPU: the last CTA to finish tells every source that its responses are in place ----
  if (A.n_resp_flags) {
    __threadfence_system();
    __syncthreads();
    if (tid == 0) S.last = atomicAdd(&A.ctl->done_ctr, 1u) == gridDim.x - 1 ? 1u : 0u;
    __syncthreads();
    if (S.last) {
      if (tid < A.n_resp_flags) {
        __threadfence_system();
        st_release_sys(A.resp_flag[tid], (unsigned long long)A.flag_epoch << 32);
      }
      if (tid == 0) A.ctl->done_ctr = 0;
    }
  }
}

// Places parked items ahead of a maintenance call that reads the table (scan, get, add).
__global__ void k_drain_overflow(const FArgs A) {
  Tally t = {0, 0, 0, 0, 0};
  __shared__ FCtx cx;
  if (threadIdx.x == 0) {
    cx.table = A.table; cx.capacity = A.capacity; cx.fragrow = A.fragrow; cx.members = A.members; cx.presence = A.presence; cx.aux = A.aux; cx.ctl = A.ctl; cx.ovf = A.ovf; cx.counters = A.counters;
    cx.nseg = A.nseg; cx.sweep_chunk = 0; cx.clk = A.clk;
  }
  __syncthreads();
  if (__ldcg(&A.ctl->ovf_count)) drain_overflow(cx, t);
  if (threadIdx.x == 0 && t.inserts) atomicAdd(A.counters + C_INSERTS, (unsigned long long)t.inserts);
}

}  // namespace gub
