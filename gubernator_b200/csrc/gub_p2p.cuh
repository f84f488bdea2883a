// gub_p2p.cuh — request routing between the GPUs of one box over NVLink peer memory, fused into the routing kernels.
//
// Replaces the reference's peer forwarding (gubernator.go:257-283 -> peer_client.go:284 runBatch -> GetPeerRateLimits,
// gubernator.go:462) inside one NVSwitch domain.  Instead of "partition locally, then three NCCL all-to-alls and a
// host round trip for the split sizes", the kernel that partitions a batch by owning shard stores every 64-byte
// request record straight into the owner's mailbox (a peer-mapped buffer) and publishes the per-owner counts with a
// release store; the owner acquires those flags (k_seg_wait) and evaluates the W mailbox segments IN PLACE with the batch kernels in
// ring mode (source-rank order, then source index order: the deterministic order the tests reproduce), which store every 32-byte
// response straight into the source's response mailbox; k_seg_publish then tells the sources, whose k_p2p_collect puts the
// responses back in request order.
//
// Per rank, one peer-visible allocation (exported with cudaIpcGetMemHandle, or shared by pointer inside one process):
//   req_mb  [2][W][cap] gub_req    written by sources     resp_mb [2][W][cap] gub_resp   written by owners
//   req_flag[2][W] u64 (epoch << 32 | count)              resp_flag[2][W] u64 (epoch)
// indexed by step parity so that step e+1 may start filling while a slow peer still drains step e.
#pragma once
#if !defined(GUB_EMULATE)  // tests/kernel_emu_harness.cpp compiles this header for the CPU (see gub_kernels.cuh)
#include <cuda_runtime.h>
#endif
#include <stdint.h>

#include "gub_kernels.cuh"

namespace gub {

struct P2PView {        // one rank's mailbox block as seen from a given process
  gub_req* req_mb;
  gub_resp* resp_mb;
  unsigned long long* req_flag;
  unsigned long long* resp_flag;
};

struct P2PArgs {
  P2PView peers[MAX_SHARDS];  // peers[r] = rank r's block (peers[rank] is our own)
  uint32_t world, rank, cap, epoch;
  uint32_t* done_ctr;         // (unused: kept for layout compatibility of the kernel arguments)
  uint32_t* error;            // set when a spin timed out
};

__device__ __forceinline__ size_t mb_index(const P2PArgs& P, uint32_t src, uint32_t p) {
  return ((size_t)(P.epoch & 1u) * P.world + src) * P.cap + p;
}
// Spins until flag's epoch field equals `epoch`; gives up after 2 x 10^7 polls (seconds: a peer died): sets *error so the host can tell.
__device__ __forceinline__ unsigned long long wait_flag(const unsigned long long* flag, uint32_t epoch, uint32_t* error) {
  for (uint32_t it = 0; it < 20000000u; it++) {
    const unsigned long long v = ld_acquire_sys(flag);
    if ((uint32_t)(v >> 32) == epoch) return v;
    __nanosleep(100);
  }
  atomicExch(error, 1u);
  return ((unsigned long long)epoch << 32);  // count 0
}

// ---- routing in one launch -------------------------------------------------------------------------------------------------
// k_p2p_route = owner lookup + stable partition + NVLink stores + flag publication, one CTA per tile of 512 requests, no grid
// barrier: tiles are taken in ticket order, every tile publishes its per-owner counts (epoch-tagged, so nothing is ever cleared)
// and waits only for the tiles before it (which hold earlier tickets, so they are resident or done: forward progress without
// co-residency of the grid — this kernel runs next to the cooperative batch kernel of the previous step).
constexpr int RT_THREADS = 512;
constexpr int RT_WARPS = RT_THREADS / 32;

struct RouteArgs {
  P2PArgs P;
  const gub_req* reqs;
  uint32_t n;                      // requests (or the most there can be, with n_dev)
  const uint32_t* n_dev;           // optional: the count lives on the device
  const uint64_t* pts;             // ring points, ascending
  const int32_t* pt_peer;          // shard of every point
  const uint16_t* lut;             // [65536] first point whose hash is >= (bucket << 48)
  uint32_t npts;
  int32_t self_global;             // >= 0: GLOBAL requests this shard does not own stay here (gubernator.go:257-269)
  uint8_t* true_owner;             // optional [n]: the ring owner of every request (input of the GLOBAL hits queue)
  unsigned long long* tile_agg;    // [tiles][MAX_SHARDS] (epoch << 32 | count)
  uint32_t* counts;                // [MAX_SHARDS] out: records sent to every owner (the un-route needs the segment starts)
  uint32_t* perm;                  // [n] out: perm[dense position] = original index
  uint32_t* ticket;                // [2]: tile ticket, tiles done
};

__device__ __forceinline__ uint32_t ring_owner_lut(const RouteArgs& R, uint64_t h) {
  uint32_t idx = __ldg(R.lut + (h >> 48));
  while (idx < R.npts && __ldg(R.pts + idx) < h) idx++;
  if (idx >= R.npts) idx = 0;
  return (uint32_t)__ldg(R.pt_peer + idx);
}

// The parts of a routing CTA that do not depend on where its records come from (k_p2p_route: 64-byte records; k_p2p_route_keys:
// key strings hashed and expanded on the spot).
struct RouteSmem {
  uint32_t tile, last;
  uint32_t cnt[MAX_SHARDS], off[MAX_SHARDS];
  uint16_t w[MAX_SHARDS][RT_WARPS];
};

// Takes the CTA's tile ticket and clears the per-owner counts; returns the tile.
__device__ __forceinline__ uint32_t route_tile_begin(const RouteArgs& R, RouteSmem& S) {
  const uint32_t tid = threadIdx.x;
  if (tid == 0) S.tile = atomicAdd(&R.ticket[0], 1u);
  if (tid < MAX_SHARDS) S.cnt[tid] = 0;
  for (uint32_t k = tid; k < (uint32_t)(MAX_SHARDS * RT_WARPS); k += RT_THREADS) (&S.w[0][0])[k] = 0;
  __syncthreads();
  return S.tile;
}

// Owner of request i by its FNV-1 hash (replicated_hash.go:104-119), recorded for the GLOBAL hits queue; a GLOBAL request this shard
// does not own is rewritten in r3 and stays here.
__device__ __forceinline__ uint32_t route_owner(const RouteArgs& R, uint32_t i, uint64_t fnv, ulonglong2& r3) {
  uint32_t o = ring_owner_lut(R, fnv);
  if (R.true_owner) R.true_owner[i] = (uint8_t)o;
  if (R.self_global >= 0 && o != (uint32_t)R.self_global && ((uint32_t)(r3.y >> 32) & GUB_BEHAVIOR_GLOBAL)) {
    // GLOBAL on a non-owner: answered here from the replica, as a clone with NO_BATCHING set, GLOBAL cleared, IsOwner = false (gubernator.go:408-411)
    o = (uint32_t)R.self_global;
    uint32_t beh = (uint32_t)(r3.y >> 32);
    beh = (beh | (uint32_t)GUB_BEHAVIOR_NO_BATCHING) & ~(uint32_t)(GUB_BEHAVIOR_GLOBAL | GUB_REQ_IS_OWNER);
    r3.y = (r3.y & 0xFFFFFFFFull) | ((unsigned long long)beh << 32);
  }
  return o;
}

// Stable partition of the tile by owner (per-warp counts per owner give the rank inside the tile), tile publication, NVLink stores
// into the owners' mailboxes, perm, and — in the last tile to finish — the totals and the epoch-tagged flag release.
__device__ __forceinline__ void route_tile_end(const RouteArgs& R, RouteSmem& S, uint32_t t, uint32_t ntiles, uint32_t i, bool valid, uint32_t o,
                                               const ulonglong2& r0, const ulonglong2& r1, const ulonglong2& r2, const ulonglong2& r3) {
  const P2PArgs& P = R.P;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t mates = __match_any_sync(0xFFFFFFFFu, valid ? o : (0x100u | lane));
  if (valid && lane == (uint32_t)(__ffs(mates) - 1)) { S.w[o][warp] = (uint16_t)__popc(mates); atomicAdd(&S.cnt[o], (uint32_t)__popc(mates)); }
  __syncthreads();
  // publish this tile's counts, then sum the tiles before it (warp o handles owner o)
  if (t < ntiles && tid < P.world) __stcg(&R.tile_agg[(size_t)t * MAX_SHARDS + tid], ((unsigned long long)P.epoch << 32) | (unsigned long long)S.cnt[tid]);
  if (warp < P.world && t < ntiles) {
    uint32_t sum = 0;
    for (uint32_t tp = lane; tp < t; tp += 32) {
      const unsigned long long* a = &R.tile_agg[(size_t)tp * MAX_SHARDS + warp];
      unsigned long long v = ld_acquire_sys(a);
      for (uint32_t it = 0; (uint32_t)(v >> 32) != P.epoch && it < 20000000u; it++) { __nanosleep(40); v = ld_acquire_sys(a); }
      if ((uint32_t)(v >> 32) != P.epoch) atomicExch(P.error, 3u);
      sum += (uint32_t)(v & 0xFFFFFFFFull);
    }
    sum = __reduce_add_sync(0xFFFFFFFFu, sum);
    if (lane == 0) S.off[warp] = sum;
  }
  __syncthreads();
  if (valid) {
    uint32_t before = 0;
#pragma unroll
    for (int w = 0; w < RT_WARPS; w++) before += ((uint32_t)w < warp) ? (uint32_t)S.w[o][w] : 0u;
    const uint32_t pos = S.off[o] + before + __popc(mates & ((1u << lane) - 1u));  // position within (me -> owner o)'s mailbox segment
    ulonglong2* dst = reinterpret_cast<ulonglong2*>(P.peers[o].req_mb + mb_index(P, P.rank, pos));  // NVLink store
    dst[0] = r0; dst[1] = r1; dst[2] = r2; dst[3] = r3;
    // the way back: responses of owner o come back in its response mailbox at `pos`; (o, pos) packed for the un-route
    R.perm[i] = (o << 24) | pos;
  }
  // the last tile knows the totals
  if (t + 1 == ntiles && tid < P.world) R.counts[tid] = S.off[tid] + S.cnt[tid];
  if (ntiles == 0 && t == 0 && tid < P.world) R.counts[tid] = 0;
  __threadfence_system();
  __syncthreads();
  if (tid == 0) S.last = atomicAdd(&R.ticket[1], 1u) == gridDim.x - 1 ? 1u : 0u;
  __syncthreads();
  if (S.last) {  // every tile has been stored: tell every owner how many records it got from us
    __threadfence_system();
    if (tid < P.world)
      st_release_sys(&P.peers[tid].req_flag[(size_t)(P.epoch & 1u) * P.world + P.rank], ((unsigned long long)P.epoch << 32) | (unsigned long long)__ldcg(&R.counts[tid]));
    if (tid == 0) { R.ticket[0] = 0; R.ticket[1] = 0; }
  }
}

__global__ void __launch_bounds__(RT_THREADS) k_p2p_route(const RouteArgs R) {
  __shared__ RouteSmem S;
  const uint32_t t = route_tile_begin(R, S);
  const uint32_t n = R.n_dev ? min(__ldcg(R.n_dev), R.n) : R.n;
  const uint32_t ntiles = (n + RT_THREADS - 1) / RT_THREADS;
  const uint32_t i = t * RT_THREADS + threadIdx.x;
  const bool valid = i < n;
  uint32_t o = 0xFFu;
  ulonglong2 r0, r1, r2, r3;
  if (valid) {
    const ulonglong2* src = reinterpret_cast<const ulonglong2*>(R.reqs + i);
    r0 = __ldg(src); r1 = __ldg(src + 1); r2 = __ldg(src + 2); r3 = __ldg(src + 3);
    o = route_owner(R, i, r0.y, r3);
  }
  route_tile_end(R, S, t, ntiles, i, valid, o, r0, r1, r2, r3);
}

// ---- routing straight from key strings --------------------------------------------------------------------------------------
// k_p2p_route_keys = k_hash_expand + k_p2p_route in one launch: every thread hashes its key (XXH64 + FNV-1), expands its parameter set
// into the 64-byte record and routes it exactly like k_p2p_route (same owner lookup by FNV-1, same stable partition, same mailbox
// layout), so that a step may mix shards that ingest key strings with shards that ingest records.  The packed buffer
// ([gub_kreq x n][uint32 offsets x (n + 1)][key bytes], gub_keys_layout) is device memory the host cannot check, so the key bounds
// are clamped here: hi = min(offsets[i + 1], key_bytes), lo = min(offsets[i], hi); a malformed entry is hashed as that (possibly
// empty) key and nothing outside the buffer is read.  The host checks that the buffer holds the records and offsets.
struct KeysRouteArgs {
  RouteArgs R;                     // R.reqs is unused
  const uint8_t* packed;
  uint64_t key_bytes;              // bytes after the offsets (packed_bytes - bytes_at)
  InlineParams Pi;                 // the parameter table when n_params <= INLINE_PARAMS ...
  const gub_params* params_far;    // ... else here (device memory)
  uint32_t n_params;
  int64_t created_base;
  gub_req* expanded;               // optional [n]: the expanded records by original index (input of the GLOBAL hits queue)
};

__global__ void __launch_bounds__(RT_THREADS) k_p2p_route_keys(const KeysRouteArgs K) {
  __shared__ RouteSmem S;
  const RouteArgs& R = K.R;
  const uint32_t t = route_tile_begin(R, S);
  const uint32_t n = R.n;
  const uint32_t ntiles = (n + RT_THREADS - 1) / RT_THREADS;
  const uint32_t i = t * RT_THREADS + threadIdx.x;
  const bool valid = i < n;
  uint32_t o = 0xFFu;
  ulonglong2 r0, r1, r2, r3;
  if (valid) {
    const ulonglong2 kr = __ldcs(reinterpret_cast<const ulonglong2*>(K.packed) + i);  // hits | params, created_delta
    const uint32_t* offsets = reinterpret_cast<const uint32_t*>(K.packed + (size_t)n * 16);
    const uint8_t* bytes = K.packed + (size_t)n * 16 + ((size_t)n + 1) * 4;
    const uint64_t hi = min((uint64_t)__ldg(offsets + i + 1), K.key_bytes);
    const uint64_t lo = min((uint64_t)__ldg(offsets + i), hi);
    kreq_decode(kr, bytes + lo, (uint32_t)(hi - lo), K.Pi, K.n_params, K.params_far, K.created_base, r0, r1, r2, r3);
    if (K.expanded) {
      ulonglong2* e = reinterpret_cast<ulonglong2*>(K.expanded + i);
      e[0] = r0; e[1] = r1; e[2] = r2; e[3] = r3;
    }
    o = route_owner(R, i, r0.y, r3);
  }
  route_tile_end(R, S, t, ntiles, i, valid, o, r0, r1, r2, r3);
}

// Source side: wait for every owner's response flag, then out[i] = resp_mb[owner(i)][pos(i)] (perm as written by k_p2p_route).
// An owner whose flag never comes (it died) costs its requests an in-band error instead of stale mailbox contents.
__global__ void __launch_bounds__(256) k_p2p_collect(const P2PArgs P, const uint32_t* perm, uint32_t n, const uint32_t* n_dev, gub_resp* out) {
  __shared__ uint32_t ok[MAX_SHARDS];
  if (threadIdx.x < P.world) {
    const unsigned long long* f = &P.peers[P.rank].resp_flag[(size_t)(P.epoch & 1u) * P.world + threadIdx.x];
    uint32_t good = 0;
    for (uint32_t it = 0; it < 20000000u; it++) {
      if ((uint32_t)(ld_acquire_sys(f) >> 32) == P.epoch) { good = 1; break; }
      __nanosleep(100);
    }
    if (!good) atomicExch(P.error, 1u);
    ok[threadIdx.x] = good;
  }
  __syncthreads();
  if (n_dev) n = min(n, __ldcg(n_dev));
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t pk = perm[i], o = pk >> 24, pos = pk & 0xFFFFFFu;
    ulonglong2* dst = reinterpret_cast<ulonglong2*>(out + i);
    if (ok[o]) {
      const ulonglong2* src = reinterpret_cast<const ulonglong2*>(P.peers[P.rank].resp_mb + mb_index(P, o, pos));
      dst[0] = __ldcg(src); dst[1] = __ldcg(src + 1);
    } else {
      dst[0] = make_ulonglong2((unsigned long long)GUB_ERR_PEER_TIMEOUT << 32, 0ull); dst[1] = make_ulonglong2(0ull, 0ull);
    }
  }
}

// ---- the owner side of a step on the four-kernel pipeline ------------------------------------------------------------------
// k_seg_wait: one warp waits for every source's flag (count of records it stored into our mailbox for this epoch) and writes the
// prefix sums the batch kernels index the mailbox segments with (BatchArgs::seg_off; seg_off[world] = requests of the step).  A
// tiny kernel of its own, so that no SM is held by spinning CTAs while the peers are still routing: the batch kernels that follow
// find everything in place.  A source that never shows up (bounded wait) counts as empty and raises the ring's error flag.
__global__ void __launch_bounds__(32) k_seg_wait(const P2PArgs P, uint32_t* seg_off) {
  __shared__ uint32_t cnt[MAX_SHARDS];
  if (threadIdx.x < P.world) {
    const unsigned long long v = wait_flag(&P.peers[P.rank].req_flag[(size_t)(P.epoch & 1u) * P.world + threadIdx.x], P.epoch, P.error);
    cnt[threadIdx.x] = min((uint32_t)(v & 0xFFFFFFFFull), P.cap);
  }
  __syncwarp();
  if (threadIdx.x == 0) {
    uint32_t a = 0;
    for (uint32_t s = 0; s < P.world; s++) { seg_off[s] = a; a += cnt[s]; }
    seg_off[P.world] = a;
  }
}
// k_seg_publish: every response of the step has been stored into the sources' response mailboxes by the batch kernels before this
// one starts (stream order; griddepcontrol.wait when launched programmatically): tell every source.
__global__ void __launch_bounds__(32) k_seg_publish(const P2PArgs P) {
  pdl_wait();
  if (threadIdx.x < P.world) {
    __threadfence_system();
    st_release_sys(&P.peers[threadIdx.x].resp_flag[(size_t)(P.epoch & 1u) * P.world + P.rank], (unsigned long long)P.epoch << 32);
  }
}

}  // namespace gub
