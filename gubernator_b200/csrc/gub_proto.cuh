// gub_proto.cuh — sm_90a kernels of the wire-format entry (gub_submit_proto_async, include/gubernator_b200.h): GetRateLimitsReq
// messages in, GetRateLimitsResp messages out, with what the host layer does per item (V1Instance.GetRateLimits, gubernator.go:183-295,
// csrc/host_v1.cpp prepare_call / finish_call) on the device.
//
// One call carries n_msgs messages, one per RPC ([int64 created_at x n][uint32 offsets x (n + 1)][message bytes], gub_proto_layout).
//   k_proto_scan(0)    slot bases: message m owns min(L_m / 2, 1000) item slots (every top-level field takes at least 2 bytes, and a
//                      message of more than 1000 items is not evaluated), so the item scratch is sized by the input alone;
//   k_proto_decode     one block per message, staged in shared memory when it fits (PROTO_SMEM), else read in place.  Thread 0 walks
//                      the top-level fields (a chain of dependent length hops) and lists the items; then every thread decodes up to 4
//                      items: the fields by protobuf-go's rules, the checks of gubernator.go:208-220, the key Name + "_" + UniqueKey
//                      copied to scratch and hashed (hash_key_bytes), and the gub_req built at the item's slot.  A malformed item makes
//                      the whole message MALFORMED; a block scan ranks the evaluable items in item order;
//   k_proto_scan(1)    batch bases: message order, then item order (the aggregator's order); the total goes to a mapped host word;
//   k_proto_compact    the evaluable items' records into the dense batch the unchanged pipeline (launch_batch) evaluates;
//   k_proto_encode     one block per message: every item's RateLimitResp as Go's proto.Marshal writes it, into a device staging area
//                      at PROTO_OUT_FACTOR x the message's input offset (the bound needs no other message's size);
//   k_proto_scan(2)    output offsets and statuses, straight into the caller's page-locked out_off / msg_status;
//   k_proto_copy_out   each message's bytes from staging into the caller's page-locked out_bytes, 16 bytes per store where aligned.
// On the ring (gub_p2p_step_proto_local_all) every shard runs the same kernels on its own RPCs; ring steps of cap items of the dense
// batch take the place of launch_batch, and the collects fill `resp`.
#pragma once
#include "gub_kernels.cuh"

namespace gub {

constexpr uint32_t PROTO_THREADS = 256;
constexpr uint32_t PROTO_ITEMS_PER_THREAD = 4;     // PROTO_THREADS x 4 >= PROTO_MAX_ITEMS
constexpr uint32_t PROTO_MAX_ITEMS = 1000;         // maxBatchSize, gubernator.go:40
constexpr uint32_t PROTO_SMEM = 160 * 1024;       // messages up to this size are decoded from (dynamic) shared memory
constexpr uint32_t PROTO_GROUP_DEPTH = 100;        // nested groups in unknown fields (protobuf-go allows 10 000: see DESIGN.md)
constexpr uint32_t PROTO_SCAN_THREADS = 1024;
constexpr uint64_t PROTO_OUT_FACTOR = 24;          // output bytes <= 24 x input bytes, per message (DESIGN.md derives it)
constexpr uint32_t PROTO_ERR = 0x80000000u;        // ProtoItem::rank: not evaluated, low byte = the GUB_ERR_* code
constexpr uint64_t PW_MAX_FIELD = (1u << 29) - 1;  // protowire.MaxValidNumber (message level)
constexpr uint64_t PW_MAX_TAG = 0x7FFFFFFFu;       // protowire.ConsumeTag's limit (inside groups)

enum { PROTO_OK = 0, PROTO_TOO_LARGE = 1, PROTO_MALFORMED = 2 };  // = GUB_PROTO_*

struct ProtoItem {
  uint32_t key_at;   // key scratch offset (= the item's offset in the call's message bytes)
  uint32_t key_len;
  int32_t algorithm; // as decoded (error text)
  uint32_t rank;     // evaluable: rank among the message's evaluable items; else PROTO_ERR | code
};

struct ProtoArgs {
  const int64_t* created;    // [n_msgs] default created_at per message
  const uint32_t* offs;      // [n_msgs + 1], offs[0] = 0
  const uint8_t* bytes;      // message bytes
  uint32_t n_msgs;
  uint32_t smem;             // k_proto_decode's dynamic shared memory: messages up to this size are staged
  uint32_t force_global;     // Behaviors.ForceGlobal (gubernator.go:232-234): every evaluable item also gets GLOBAL
  uint32_t* slot_base;       // [n_msgs + 1]
  uint32_t* batch_base;      // [n_msgs + 1]
  uint32_t *mcount, *meval, *mstatus, *msize;  // [n_msgs]: items listed, items evaluated, status, output bytes
  unsigned long long* moff;  // [n_msgs + 1]
  ProtoItem* items;          // [slots]
  gub_req* sreq;             // [slots]
  uint8_t* keys;             // [message bytes]
  uint8_t* stage;            // [PROTO_OUT_FACTOR x message bytes]
  gub_req* reqs;             // dense batch
  const gub_resp* resp;      // its responses
  uint32_t* n_eval;          // mapped host word
  uint8_t* out;              // device views of the caller's page-locked buffers
  unsigned long long* out_off;
  uint32_t* out_status;
};

// ---- protobuf wire format, by protobuf-go's rules (encoding/protowire, internal/impl) ----------------------------------------------
// ConsumeVarint: at most 10 bytes, the 10th < 2 (an 11th byte or bits past 64 are an overflow).
__device__ __forceinline__ bool pw_varint(const uint8_t* b, uint32_t& p, uint32_t e, uint64_t& v) {
  v = 0;
  for (uint32_t k = 0; k < 10; k++) {
    if (p >= e) return false;
    const uint64_t c = b[p++];
    if (k == 9) { if (c >= 2) return false; v |= c << 63; return true; }
    v |= (c & 0x7Fu) << (7 * k);
    if (c < 0x80) return true;
  }
  return false;
}

__device__ __forceinline__ bool pw_tag(const uint8_t* b, uint32_t& p, uint32_t e, uint64_t max_num, uint32_t& num, uint32_t& wt) {
  uint64_t v;
  if (!pw_varint(b, p, e, v)) return false;
  if ((v >> 3) < 1 || (v >> 3) > max_num) return false;
  num = (uint32_t)(v >> 3); wt = (uint32_t)(v & 7u);
  return true;
}

// An unknown field's value (ConsumeFieldValue): groups nest up to PROTO_GROUP_DEPTH and must close with their own field number; a
// stray end-group and wire types 6 and 7 are malformed.
__device__ __noinline__ bool pw_skip(const uint8_t* b, uint32_t& p, uint32_t e, uint32_t num, uint32_t wt) {
  uint32_t open[PROTO_GROUP_DEPTH];
  uint32_t depth = 0;
  for (;;) {
    if (wt == 0) {
      uint64_t v;
      if (!pw_varint(b, p, e, v)) return false;
    } else if (wt == 1 || wt == 5) {
      const uint32_t w = wt == 1 ? 8u : 4u;
      if (e - p < w) return false;
      p += w;
    } else if (wt == 2) {
      uint64_t l;
      if (!pw_varint(b, p, e, l) || l > e - p) return false;
      p += (uint32_t)l;
    } else if (wt == 3) {
      if (depth == PROTO_GROUP_DEPTH) return false;
      open[depth++] = num;
    } else if (wt == 4) {
      if (depth == 0 || open[depth - 1] != num) return false;
      depth--;
    } else {
      return false;
    }
    if (depth == 0) return true;
    if (!pw_tag(b, p, e, PW_MAX_TAG, num, wt)) return false;
  }
}

// utf8.Valid: no overlong forms, no surrogates, nothing above U+10FFFF.
__device__ __forceinline__ bool pw_utf8(const uint8_t* b, uint32_t p, uint32_t e) {
  while (p < e) {
    const uint32_t c = b[p];
    if (c < 0x80) { p++; continue; }
    uint32_t n, lo = 0x80, hi = 0xBF;
    if (c >= 0xC2 && c <= 0xDF) n = 1;
    else if (c == 0xE0) { n = 2; lo = 0xA0; }
    else if ((c >= 0xE1 && c <= 0xEC) || c == 0xEE || c == 0xEF) n = 2;
    else if (c == 0xED) { n = 2; hi = 0x9F; }
    else if (c == 0xF0) { n = 3; lo = 0x90; }
    else if (c >= 0xF1 && c <= 0xF3) n = 3;
    else if (c == 0xF4) { n = 3; hi = 0x8F; }
    else return false;
    if (e - p - 1 < n) return false;
    const uint32_t c1 = b[p + 1];
    if (c1 < lo || c1 > hi) return false;
    for (uint32_t k = 2; k <= n; k++) if ((b[p + k] & 0xC0u) != 0x80u) return false;
    p += n + 1;
  }
  return true;
}

// A length-delimited value at p: [*s, p) after the call.
__device__ __forceinline__ bool pw_bytes(const uint8_t* b, uint32_t& p, uint32_t e, uint32_t& s) {
  uint64_t l;
  if (!pw_varint(b, p, e, l) || l > e - p) return false;
  s = p;
  p += (uint32_t)l;
  return true;
}

// One entry of RateLimitReq.metadata (map<string, string>, field 9): key 1 and value 2 are proto3 strings; anything else is skipped.
__device__ __forceinline__ bool pw_map_entry(const uint8_t* b, uint32_t p, uint32_t e) {
  while (p < e) {
    uint32_t num, wt, s;
    if (!pw_tag(b, p, e, PW_MAX_FIELD, num, wt)) return false;
    if ((num == 1 || num == 2) && wt == 2) {
      if (!pw_bytes(b, p, e, s) || !pw_utf8(b, s, p)) return false;
    } else if (!pw_skip(b, p, e, num, wt)) {
      return false;
    }
  }
  return true;
}

struct ProtoFields {
  uint32_t name_at, name_len, uk_at, uk_len;
  int64_t hits, limit, duration, burst, created_at;
  int32_t algorithm, behavior;
  bool has_created;
};

// RateLimitReq (gubernator.proto:137-183) in [p, e).  Scalars: last one wins; a known field with another wire type is unknown.
__device__ __forceinline__ bool pw_item(const uint8_t* b, uint32_t p, uint32_t e, ProtoFields& f) {
  f.name_at = f.name_len = f.uk_at = f.uk_len = 0;
  f.hits = f.limit = f.duration = f.burst = f.created_at = 0;
  f.algorithm = f.behavior = 0;
  f.has_created = false;
  while (p < e) {
    uint32_t num, wt, s;
    if (!pw_tag(b, p, e, PW_MAX_FIELD, num, wt)) return false;
    if ((num == 1 || num == 2 || num == 9) && wt == 2) {
      if (!pw_bytes(b, p, e, s)) return false;
      if (num == 9) {
        if (!pw_map_entry(b, s, p)) return false;
      } else {
        if (!pw_utf8(b, s, p)) return false;
        if (num == 1) { f.name_at = s; f.name_len = p - s; } else { f.uk_at = s; f.uk_len = p - s; }
      }
    } else if (wt == 0 && num >= 3 && num <= 10 && num != 9) {
      uint64_t v;
      if (!pw_varint(b, p, e, v)) return false;
      switch (num) {
        case 3: f.hits = (int64_t)v; break;
        case 4: f.limit = (int64_t)v; break;
        case 5: f.duration = (int64_t)v; break;
        case 6: f.algorithm = (int32_t)(uint32_t)v; break;  // open enum: int32 of the varint
        case 7: f.behavior = (int32_t)(uint32_t)v; break;
        case 8: f.burst = (int64_t)v; break;
        default: f.created_at = (int64_t)v; f.has_created = true; break;  // 10, optional
      }
    } else if (!pw_skip(b, p, e, num, wt)) {
      return false;
    }
  }
  return true;
}

template <typename T>
__device__ __forceinline__ T proto_block_scan(T v, T* sm, T& total) {  // exclusive; every thread of the block calls it
  const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  T x = v;
  for (uint32_t d = 1; d < 32; d <<= 1) { const T y = __shfl_up_sync(0xFFFFFFFFu, x, d); if (lane >= d) x += y; }
  if (lane == 31) sm[w] = x;
  __syncthreads();
  if (w == 0) {
    T s = lane < nw ? sm[lane] : (T)0;
    for (uint32_t d = 1; d < 32; d <<= 1) { const T y = __shfl_up_sync(0xFFFFFFFFu, s, d); if (lane >= d) s += y; }
    if (lane < nw) sm[lane] = s;
  }
  __syncthreads();
  total = sm[nw - 1];
  const T r = (w ? sm[w - 1] : (T)0) + x - v;
  __syncthreads();
  return r;
}

// mode 0: slot bases; 1: batch bases and the evaluable count; 2: output offsets and statuses.  One block.
__global__ void __launch_bounds__(PROTO_SCAN_THREADS) k_proto_scan(ProtoArgs A, uint32_t mode) {
  __shared__ unsigned long long s_scan[32];
  const uint32_t n = A.n_msgs, per = (n + PROTO_SCAN_THREADS - 1) / PROTO_SCAN_THREADS;
  const uint32_t lo = min(n, threadIdx.x * per), hi = min(n, lo + per);
  auto val = [&](uint32_t m) -> unsigned long long {
    if (mode == 0) return min((A.offs[m + 1] - A.offs[m]) / 2u, PROTO_MAX_ITEMS);
    return mode == 1 ? A.meval[m] : A.msize[m];
  };
  unsigned long long s = 0, total;
  for (uint32_t m = lo; m < hi; m++) s += val(m);
  unsigned long long base = proto_block_scan<unsigned long long>(s, s_scan, total);
  auto put = [&](uint32_t m, unsigned long long at) {
    if (mode == 0) A.slot_base[m] = (uint32_t)at;
    else if (mode == 1) A.batch_base[m] = (uint32_t)at;
    else { A.moff[m] = at; A.out_off[m] = at; if (m < n) A.out_status[m] = A.mstatus[m]; }
  };
  for (uint32_t m = lo; m < hi; m++) { put(m, base); base += val(m); }
  if (threadIdx.x == 0) {
    put(n, total);
    if (mode == 1) *(volatile uint32_t*)A.n_eval = (uint32_t)total;
  }
}

__global__ void __launch_bounds__(PROTO_THREADS) k_proto_decode(ProtoArgs A) {
#ifdef GUB_EMULATE
  __shared__ __align__(16) uint8_t s_msg[PROTO_SMEM];
#else
  extern __shared__ __align__(16) uint8_t s_msg[];
#endif
  __shared__ uint32_t s_start[PROTO_MAX_ITEMS], s_len[PROTO_MAX_ITEMS];
  __shared__ uint32_t s_cnt, s_bad, s_scan[32];
  const uint32_t m = blockIdx.x;
  const uint32_t lo = A.offs[m], L = A.offs[m + 1] - lo;
  const uint8_t* g = A.bytes + lo;
  const bool staged = L <= A.smem;
  if (staged) for (uint32_t k = threadIdx.x; k < L; k += blockDim.x) s_msg[k] = g[k];
  __syncthreads();
  const uint8_t* b = staged ? s_msg : g;
  if (threadIdx.x == 0) {  // GetRateLimitsReq: field 1 = the items; past the 1000th an item is only checked
    uint32_t p = 0, cnt = 0, bad = 0;
    while (p < L) {
      uint32_t num, wt, s;
      if (!pw_tag(b, p, L, PW_MAX_FIELD, num, wt)) { bad = 1; break; }
      if (num == 1 && wt == 2) {
        if (!pw_bytes(b, p, L, s)) { bad = 1; break; }
        if (cnt < PROTO_MAX_ITEMS) { s_start[cnt] = s; s_len[cnt] = p - s; }
        else { ProtoFields f; if (!pw_item(b, s, p, f)) { bad = 1; break; } }
        cnt++;
      } else if (!pw_skip(b, p, L, num, wt)) { bad = 1; break; }
    }
    s_cnt = cnt; s_bad = bad;
  }
  __syncthreads();
  const uint32_t cnt = s_cnt, nd = min(cnt, PROTO_MAX_ITEMS), slot0 = A.slot_base[m];
  int bad = s_bad != 0;
  uint32_t evalmask = 0, nev = 0;
  for (uint32_t k = 0; k < PROTO_ITEMS_PER_THREAD && !bad; k++) {
    const uint32_t j = threadIdx.x * PROTO_ITEMS_PER_THREAD + k;
    if (j >= nd) break;
    ProtoFields f;
    if (!pw_item(b, s_start[j], s_start[j] + s_len[j], f)) { bad = 1; break; }
    ProtoItem it;
    it.key_at = lo + s_start[j]; it.key_len = 0; it.algorithm = f.algorithm; it.rank = 0;
    if (f.uk_len == 0) {         // gubernator.go:208-212, checked before the namespace
      it.rank = PROTO_ERR | GUB_ERR_UNIQUE_KEY_EMPTY;
    } else if (f.name_len == 0) {  // :213-217
      it.rank = PROTO_ERR | GUB_ERR_NAMESPACE_EMPTY;
    } else {                       // client.go:39-41; the key fits in the item's own bytes
      uint8_t* key = A.keys + it.key_at;
      for (uint32_t q = 0; q < f.name_len; q++) key[q] = b[f.name_at + q];
      key[f.name_len] = '_';
      for (uint32_t q = 0; q < f.uk_len; q++) key[f.name_len + 1 + q] = b[f.uk_at + q];
      it.key_len = f.name_len + 1 + f.uk_len;
      gub_req r;
      hash_key_bytes(key, it.key_len, &r.key_xxh64, &r.key_fnv1);
      r.hits = f.hits; r.limit = f.limit; r.duration = f.duration; r.burst = f.burst;
      r.created_at = (f.has_created && f.created_at != 0) ? f.created_at : A.created[m];  // :218-220
      r.algorithm = (uint32_t)f.algorithm;
      r.behavior = ((uint32_t)f.behavior & 0xFFu) | GUB_REQ_IS_OWNER | (A.force_global ? (uint32_t)GUB_BEHAVIOR_GLOBAL : 0u);  // the
      // ring's routing clears IS_OWNER where another shard owns the key
      A.sreq[slot0 + j] = r;
      evalmask |= 1u << k;
      nev++;
    }
    A.items[slot0 + j] = it;
  }
  bad = __syncthreads_or(bad);
  const bool ok = !bad && cnt <= PROTO_MAX_ITEMS;
  uint32_t total;
  uint32_t rank = proto_block_scan<uint32_t>(ok ? nev : 0u, s_scan, total);
  if (ok) {
    for (uint32_t k = 0; k < PROTO_ITEMS_PER_THREAD; k++)
      if (evalmask & (1u << k)) A.items[slot0 + threadIdx.x * PROTO_ITEMS_PER_THREAD + k].rank = rank++;
  }
  if (threadIdx.x == 0) {
    A.mstatus[m] = bad ? PROTO_MALFORMED : (ok ? PROTO_OK : PROTO_TOO_LARGE);
    A.mcount[m] = ok ? nd : 0u;
    A.meval[m] = ok ? total : 0u;
  }
}

__global__ void __launch_bounds__(PROTO_THREADS) k_proto_compact(ProtoArgs A) {
  const uint32_t m = blockIdx.x, cnt = A.mcount[m], slot0 = A.slot_base[m], bb = A.batch_base[m];
  for (uint32_t j = threadIdx.x; j < cnt; j += blockDim.x) {
    const uint32_t rank = A.items[slot0 + j].rank;
    if (!(rank & PROTO_ERR)) A.reqs[bb + rank] = A.sreq[slot0 + j];
  }
}

// ---- GetRateLimitsResp ------------------------------------------------------------------------------------------------------------
struct ProtoEmit {  // d == nullptr: count only
  uint8_t* d;
  uint32_t n;
  __device__ __forceinline__ void c(uint32_t x) { if (d) d[n] = (uint8_t)x; n++; }
  __device__ __forceinline__ void s(const char* z) { while (*z) c((uint8_t)*z++); }
  __device__ __forceinline__ void v(uint64_t x) { while (x >= 0x80) { c((uint32_t)(x & 0x7F) | 0x80u); x >>= 7; } c((uint32_t)x); }
  __device__ __forceinline__ void i32(int32_t x) {  // %d
    char t[12];
    int k = 0;
    uint32_t u = x < 0 ? 0u - (uint32_t)x : (uint32_t)x;
    do { t[k++] = (char)('0' + u % 10); u /= 10; } while (u);
    if (x < 0) c('-');
    while (k) c((uint8_t)t[--k]);
  }
};

// RateLimitResp.Error: gub_format_error's text (csrc/host_v1.cpp), without its 255-byte limit.
__device__ __noinline__ void proto_error_text(ProtoEmit& o, uint32_t code, const uint8_t* key, uint32_t key_len, int32_t algorithm) {
  if (code == GUB_ERR_UNIQUE_KEY_EMPTY) { o.s("field 'unique_key' cannot be empty"); return; }
  if (code == GUB_ERR_NAMESPACE_EMPTY) { o.s("field 'namespace' cannot be empty"); return; }
  if (code == GUB_ERR_PEER_TIMEOUT) {  // gubernator.go:374 wrapping the deadline error of a peer call that timed out (ring steps only)
    o.s("Error while fetching rate limit '");
    for (uint32_t q = 0; q < key_len; q++) o.c(key[q]);
    o.s("' from peer: context deadline exceeded");
    return;
  }
  if (code < GUB_ERR_INVALID_ALGORITHM || code > GUB_ERR_TABLE_FULL) return;
  o.s("Error while apply rate limit for '");
  for (uint32_t q = 0; q < key_len; q++) o.c(key[q]);
  o.s("': during workerPool.GetRateLimit: ");
  if (code == GUB_ERR_INVALID_ALGORITHM) { o.s("Invalid rate limit algorithm '"); o.i32(algorithm); o.c('\''); return; }
  if (code == GUB_ERR_TABLE_FULL) { o.s("rate limit table is full"); return; }
  o.s(algorithm == GUB_LEAKY_BUCKET ? "Error in leakyBucket" : "Error in tokenBucket");
  if (code == GUB_ERR_GREGORIAN_WEEKS) o.s(": `Duration = GregorianWeeks` not yet supported; consider making a PR!`");
  else o.s(": behavior DURATION_IS_GREGORIAN is set; but `Duration` is not a valid gregorian interval");
}

// One element of GetRateLimitsResp.responses: 0x0A, length, then the fields in number order with zero values omitted.
__device__ __forceinline__ uint32_t proto_emit_resp(uint8_t* dst, const ProtoItem& it, const gub_resp* r, const uint8_t* keys) {
  const uint32_t code = (it.rank & PROTO_ERR) ? (it.rank & 0xFFu) : r->err_code;
  ProtoEmit o{dst, 0}, sz{nullptr, 0};
  uint32_t text = 0;
  if (code == 0) {
    if (r->status) { sz.c(0x08); sz.v((uint64_t)(int64_t)(int32_t)r->status); }
    if (r->limit) { sz.c(0x10); sz.v((uint64_t)r->limit); }
    if (r->remaining) { sz.c(0x18); sz.v((uint64_t)r->remaining); }
    if (r->reset_time) { sz.c(0x20); sz.v((uint64_t)r->reset_time); }
  } else {
    ProtoEmit t{nullptr, 0};
    proto_error_text(t, code, keys + it.key_at, it.key_len, it.algorithm);
    text = t.n;
    if (text) { sz.c(0x2A); sz.v(text); sz.n += text; }
  }
  o.c(0x0A);
  o.v(sz.n);
  if (!dst) return o.n + sz.n;  // dst == nullptr: the size only
  if (code == 0) {
    if (r->status) { o.c(0x08); o.v((uint64_t)(int64_t)(int32_t)r->status); }
    if (r->limit) { o.c(0x10); o.v((uint64_t)r->limit); }
    if (r->remaining) { o.c(0x18); o.v((uint64_t)r->remaining); }
    if (r->reset_time) { o.c(0x20); o.v((uint64_t)r->reset_time); }
  } else if (text) {
    o.c(0x2A);
    o.v(text);
    proto_error_text(o, code, keys + it.key_at, it.key_len, it.algorithm);
  }
  return o.n;
}

__global__ void __launch_bounds__(PROTO_THREADS) k_proto_encode(ProtoArgs A) {
  __shared__ uint32_t s_scan[32];
  const uint32_t m = blockIdx.x, cnt = A.mcount[m], slot0 = A.slot_base[m], bb = A.batch_base[m];
  uint32_t mine = 0;
  for (uint32_t k = 0; k < PROTO_ITEMS_PER_THREAD; k++) {
    const uint32_t j = threadIdx.x * PROTO_ITEMS_PER_THREAD + k;
    if (j >= cnt) break;
    const ProtoItem it = A.items[slot0 + j];
    mine += proto_emit_resp(nullptr, it, (it.rank & PROTO_ERR) ? nullptr : &A.resp[bb + it.rank], A.keys);
  }
  uint32_t total;
  uint32_t at = proto_block_scan<uint32_t>(mine, s_scan, total);
  uint8_t* dst = A.stage + PROTO_OUT_FACTOR * A.offs[m];
  for (uint32_t k = 0; k < PROTO_ITEMS_PER_THREAD; k++) {
    const uint32_t j = threadIdx.x * PROTO_ITEMS_PER_THREAD + k;
    if (j >= cnt) break;
    const ProtoItem it = A.items[slot0 + j];
    at += proto_emit_resp(dst + at, it, (it.rank & PROTO_ERR) ? nullptr : &A.resp[bb + it.rank], A.keys);
  }
  if (threadIdx.x == 0) A.msize[m] = total;
}

__global__ void __launch_bounds__(PROTO_THREADS) k_proto_copy_out(ProtoArgs A) {
  const uint32_t m = blockIdx.x, len = A.msize[m];
  if (len == 0) return;
  const uint8_t* src = A.stage + PROTO_OUT_FACTOR * A.offs[m];
  uint8_t* dst = A.out + A.moff[m];
  const uint32_t head = min(len, (uint32_t)((16u - ((uintptr_t)dst & 15u)) & 15u));
  const uint32_t body = (len - head) / 16u, tail = head + body * 16u;
  for (uint32_t k = threadIdx.x; k < head; k += blockDim.x) dst[k] = src[k];
  for (uint32_t q = threadIdx.x; q < body; q += blockDim.x) {
    const uint8_t* s = src + head + 16u * q;
    uint32_t w[4];
    for (int x = 0; x < 4; x++)
      w[x] = (uint32_t)s[4 * x] | ((uint32_t)s[4 * x + 1] << 8) | ((uint32_t)s[4 * x + 2] << 16) | ((uint32_t)s[4 * x + 3] << 24);
    *reinterpret_cast<uint4*>(dst + head + 16u * q) = make_uint4(w[0], w[1], w[2], w[3]);
  }
  for (uint32_t k = tail + threadIdx.x; k < len; k += blockDim.x) dst[k] = src[k];
}

// ---- host side: the checks and sizes of one call, from the caller's offsets (host memory) ------------------------------------------
struct ProtoPlan {
  size_t offsets_at, bytes_at, msg_bytes, slots;
  uint32_t smem;  // the largest message, rounded up to 16 bytes, up to PROTO_SMEM
};
// nullptr = the call is well formed; else the reason.
inline const char* proto_plan(const uint8_t* packed, size_t packed_bytes, size_t n_msgs, size_t out_cap, ProtoPlan& P) {
  P.offsets_at = n_msgs * 8;
  P.bytes_at = P.offsets_at + (n_msgs + 1) * 4;
  P.msg_bytes = 0; P.slots = 0; P.smem = 0;
  if (packed_bytes < P.bytes_at) return "packed buffer too small for its offsets";
  const uint8_t* ob = packed + P.offsets_at;
  uint32_t prev;
  std::memcpy(&prev, ob, 4);
  if (prev != 0) return "offsets[0] must be 0";
  for (size_t m = 1; m <= n_msgs; m++) {
    uint32_t o;
    std::memcpy(&o, ob + 4 * m, 4);
    if (o < prev) return "offsets must not decrease";
    P.slots += std::min<uint32_t>((o - prev) / 2u, PROTO_MAX_ITEMS);
    if (o - prev <= PROTO_SMEM) P.smem = std::max<uint32_t>(P.smem, (o - prev + 15u) & ~15u);
    prev = o;
  }
  P.msg_bytes = prev;
  if (P.msg_bytes > packed_bytes - P.bytes_at) return "offsets run past the end of the packed buffer";
  if (P.msg_bytes > 0x7FFFFFFFull) return "more than 2^31 - 1 message bytes";
  if (out_cap < PROTO_OUT_FACTOR * P.msg_bytes) return "out_cap is below the bound gub_proto_layout gives for these messages";
  return nullptr;
}

}  // namespace gub
