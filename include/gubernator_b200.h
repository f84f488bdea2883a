/*
 * gubernator_b200.h — C ABI of the H100-native (sm_90a) rate-limit evaluation path.
 *
 * This is the drop-in boundary for mailgun/gubernator v2.4.0's WorkerPool (the only thing `gubernator.go` calls on
 * the hot path).  Every entry point names the reference interface it replaces (file:line under the reference repo).
 * The reference-side cgo binding is shown in INTEGRATION.md and go/workerpool_b200.go.
 *
 * Model.  A `gub_table` is one GPU's shard of the key space: a device-resident open-addressed hash table of 64-byte
 * bucket-state slots (TokenBucketItem / LeakyBucketItem + CacheItem.ExpireAt, store.go:29-43, cache.go:29-41),
 * replacing the per-worker LRUCache (lrucache.go:32) of every Worker in the pool (workers.go:54-61).  One
 * `gub_submit*` call evaluates a whole batch of pre-hashed requests on the GPU with exactly the results the
 * reference produces when it applies the same requests one after another in index order (the order of the loop at
 * gubernator.go:203) under a frozen clock `now_ms`.
 *
 * Strings never cross this ABI on the fast path: a request carries XXH64(Name+"_"+UniqueKey, seed 0) — the hash
 * workers.go:153 already computes per request — and the FNV-1 64 hash replicated_hash.go:108 computes for peer
 * routing.  Together they form the 120-bit key fingerprint stored in the slot (see DESIGN.md for the residual
 * collision probability).  gub_hash_keys() computes both from packed key bytes.
 *
 * Threading: all calls on one gub_table are serialised internally (a mutex), mirroring "each worker owns its cache"
 * (workers.go:19-25); use one long call per batch, never one per request.  Ownership: the caller owns every buffer it
 * passes for the duration of the call only; the library owns all device memory.  Errors: 0 = ok, negative = failure
 * with text in gub_last_error(); per-request errors come back in-band in gub_resp.err_code exactly as the reference
 * returns them in RateLimitResp.Error (gubernator.go:210,215,255), the shim maps codes to the reference strings.
 */
#ifndef GUBERNATOR_B200_H
#define GUBERNATOR_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GUB_ABI_VERSION 2

/* Algorithm, Status, Behavior: gubernator.proto:56-135 */
enum { GUB_TOKEN_BUCKET = 0, GUB_LEAKY_BUCKET = 1 };
enum { GUB_UNDER_LIMIT = 0, GUB_OVER_LIMIT = 1 };
enum {
  GUB_BEHAVIOR_NO_BATCHING = 1,
  GUB_BEHAVIOR_GLOBAL = 2,
  GUB_BEHAVIOR_DURATION_IS_GREGORIAN = 4,
  GUB_BEHAVIOR_RESET_REMAINING = 8,
  GUB_BEHAVIOR_MULTI_REGION = 16,
  GUB_BEHAVIOR_DRAIN_OVER_LIMIT = 32,
  /* RateLimitReqState.IsOwner (gubernator.go:56): gates metricOverLimitCounter only (algorithms.go:164,184,242) */
  GUB_REQ_IS_OWNER = 0x100
};

/* gub_resp.err_code: in-band per-request errors */
enum {
  GUB_OK = 0,
  GUB_ERR_UNIQUE_KEY_EMPTY = 1,   /* gubernator.go:208-211 (raised by the host layer, never by the device) */
  GUB_ERR_NAMESPACE_EMPTY = 2,    /* gubernator.go:213-216 (host layer) */
  GUB_ERR_INVALID_ALGORITHM = 3,  /* workers.go:318 */
  GUB_ERR_GREGORIAN_WEEKS = 4,    /* interval.go:93,134 */
  GUB_ERR_GREGORIAN_INVALID = 5,  /* interval.go:107,147 */
  GUB_ERR_TABLE_FULL = 6,         /* no longer produced by the batch path (a full probe window evicts, like lrucache.go:98); gub_add_items only */
  GUB_ERR_PEER_TIMEOUT = 7        /* the owning shard did not answer within the bounded wait (peer_client.go:169-189 returns the RPC error in-band) */
};

/* One RateLimitReq (gubernator.proto:137-183) after HashKey() (client.go:39-41) and hashing.  64 bytes. */
typedef struct {
  uint64_t key_xxh64;  /* XXH64(Name + "_" + UniqueKey, seed 0)      workers.go:153-155 */
  uint64_t key_fnv1;   /* FNV-1 64 of the same string                replicated_hash.go:108 */
  int64_t hits;
  int64_t limit;
  int64_t duration;    /* ms, or a Gregorian interval id 0..5 when DURATION_IS_GREGORIAN */
  int64_t burst;
  int64_t created_at;  /* epoch ms; must already be defaulted (gubernator.go:218-220) */
  uint32_t algorithm;
  uint32_t behavior;   /* Behavior bits | GUB_REQ_IS_OWNER */
} gub_req;

/* One RateLimitResp (gubernator.proto:190-203).  32 bytes.  All other fields are zero when err_code != 0. */
typedef struct {
  uint32_t status;
  uint32_t err_code;
  int64_t limit;
  int64_t remaining;
  int64_t reset_time;
} gub_resp;

/* The frozen clock of one batch.  now_ms is what clock.Now()/MillisecondNow() return for every request of the batch
 * (lrucache.go:106-108, algorithms.go:128,219,339-344,442); the Gregorian tables are GregorianExpiration(now, d) and
 * GregorianDuration(now, d) for d = 0..5 (interval.go:84-148), computed on the host by gub_clock_fill(). */
typedef struct {
  int64_t now_ms;
  int64_t greg_expire[6];
  int64_t greg_duration[6];
} gub_clock;

/* One CacheItem with its bucket value flattened (cache.go:29-41, store.go:29-43). */
typedef struct {
  uint64_t key_xxh64;
  uint64_t key_fnv1;     /* on output only the top 56 bits are meaningful (low 8 bits read back as zero) */
  int32_t algorithm;     /* GUB_TOKEN_BUCKET | GUB_LEAKY_BUCKET: also the dynamic type of CacheItem.Value */
  int32_t status;        /* TokenBucketItem.Status */
  int64_t limit;
  int64_t duration;
  int64_t remaining;     /* TokenBucketItem.Remaining */
  double remaining_f;    /* LeakyBucketItem.Remaining */
  int64_t stamp;         /* TokenBucketItem.CreatedAt | LeakyBucketItem.UpdatedAt */
  int64_t burst;         /* LeakyBucketItem.Burst */
  int64_t expire_at;     /* CacheItem.ExpireAt */
  int64_t invalid_at;    /* CacheItem.InvalidAt (cache.go:40): 0 = none; set by Store / Loader plugins only; an item past it is a miss (cache.go:47) */
} gub_item;

/* Mirrors metricOverLimitCounter (gubernator.go:74), metricCacheAccess hit/miss (lrucache.go:52) + table stats */
typedef struct {
  uint64_t over_limit;
  uint64_t cache_hit;
  uint64_t cache_miss;
  uint64_t inserts;        /* slots claimed for new keys */
  uint64_t table_full;     /* requests answered GUB_ERR_TABLE_FULL */
  uint64_t requests;       /* decisions evaluated */
  uint64_t batches;
  uint64_t dup_groups;     /* keys that occurred more than once within a batch */
  uint64_t mixed_groups;   /* of those, keys whose requests differed within the batch (segment path) */
  uint64_t serial_fallbacks; /* chunks (<= 512 requests) of such groups that were mostly one-request runs: applied one by one */
  uint64_t unexpired_evictions; /* live entries displaced because a probe window was full: metricCacheUnexpiredEvictions (lrucache.go:138-149) */
  uint64_t swept;          /* removed / expired entries freed by the incremental sweep inside the batch kernel */
  uint64_t gq_dropped;     /* GLOBAL requests not queued because a gub_gq was full within one sync window (queue overflow only:
                              a sync tick carries every queued key) */
} gub_counters;

typedef struct {
  uint64_t capacity_slots; /* table size in 64-byte slots (>= 2x expected live keys); replaces Config.CacheSize (config.go:86) */
  uint32_t max_batch;      /* largest batch evaluated by one launch sequence; larger submits are chunked in order. 0 = 65536.
                              Up to 65 536 the table keeps two sets of grouping scratch (80.5 MiB more at 65 536) so that
                              consecutive batches on one stream overlap (see gub_submit_device). */
  int32_t device;          /* CUDA device ordinal */
} gub_config;

typedef struct gub_table gub_table;

/* ---- lifecycle: NewWorkerPool (workers.go:125) / WorkerPool.Close (workers.go:157) ------------------------- */
int gub_create(const gub_config* cfg, gub_table** out);
void gub_destroy(gub_table* t);
const char* gub_last_error(void);
int gub_abi_version(void);

/* ---- the hot path: WorkerPool.GetRateLimit (workers.go:261-324) for a whole batch -------------------------- */
/* Host buffers: copies requests H2D, evaluates, copies responses D2H, returns when `out` is filled. */
int gub_submit(gub_table* t, const gub_req* reqs, size_t n, const gub_clock* clk, gub_resp* out);
/* Device buffers (already resident in this GPU's HBM); enqueued on `stream` (a cudaStream_t), returns immediately.
 * When two submissions follow each other on one stream with nothing in between, the second one's grouping kernel reads its
 * requests while the first one is still evaluated (programmatic dependent launch).  A kernel the caller puts in between is
 * detected on the device and makes the second submission wait for it; the one case that is not detected is a caller kernel
 * launched with programmatic stream serialization that triggers its dependents (griddepcontrol.launch_dependents) before its
 * last write of the requests.  Plain kernels, copies and event waits in between are safe. */
int gub_submit_device(gub_table* t, const gub_req* d_reqs, size_t n, const gub_clock* clk, gub_resp* d_out, void* stream);
/* Same, when the batch size is only known on the device: *d_n (<= n_cap) requests; launches are sized for n_cap. */
int gub_submit_device_n(gub_table* t, const gub_req* d_reqs, size_t n_cap, const uint32_t* d_n, const gub_clock* clk, gub_resp* d_out, void* stream);
/* Pipelined host path: up to gub_pipeline_depth() submissions may be in flight; each uses library-owned pinned
 * staging.  gub_submit_async returns a ticket; gub_wait(ticket) blocks until that batch's responses are in `out`. */
int gub_pipeline_depth(gub_table* t);
int gub_submit_async(gub_table* t, const gub_req* reqs, size_t n, const gub_clock* clk, gub_resp* out, int* ticket);
int gub_wait(gub_table* t, int ticket);

/* ---- compact requests: the host link is the bottleneck of the host-to-host path (64 B per request over PCIe), and most
 * of a RateLimitReq is per-limit configuration that repeats across a batch.  A compact batch carries 32-byte records
 * plus one small table of the distinct (limit, duration, burst, algorithm, behavior) tuples; a kernel expands it to
 * gub_req records on the device and the normal path runs.  Results are identical to submitting the expanded batch.
 * Tables of up to 32 sets travel inside the kernel launch (read during the call: `params` may be reused right after it
 * returns; `reqs` and `out` must stay valid until gub_wait); larger tables are copied to the device separately (then `params` must
 * stay valid until gub_wait as well), which costs the pipeline far more than their size suggests: keep tables small. */
typedef struct {
  uint64_t key_xxh64;
  uint64_t key_fnv1;
  int64_t hits;
  uint32_t params;        /* index into the batch's gub_params table */
  int32_t created_delta;  /* created_at = created_base + created_delta (ms) */
} gub_creq;               /* 32 bytes */
typedef struct {
  int64_t limit, duration, burst;
  uint32_t algorithm;
  uint32_t behavior;      /* Behavior bits | GUB_REQ_IS_OWNER */
} gub_params;             /* 32 bytes */
int gub_submit_compact_async(gub_table* t, const gub_creq* reqs, size_t n, const gub_params* params, size_t n_params,
                             int64_t created_base, const gub_clock* clk, gub_resp* out, int* ticket);
int gub_submit_compact(gub_table* t, const gub_creq* reqs, size_t n, const gub_params* params, size_t n_params,
                       int64_t created_base, const gub_clock* clk, gub_resp* out);

/* ---- key strings: the step right before the path (client.go:39-41 HashKey, workers.go:153 XXH64, replicated_hash.go:108 FNV-1)
 * runs on the device too.  The host ships the raw key bytes ("Name_UniqueKey") and one 16-byte record per request; a kernel hashes
 * the keys and builds the gub_req records (parameter table as for the compact path), then the normal path runs.  Results are
 * identical to hashing on the host and submitting the full records. */
typedef struct {
  int64_t hits;
  uint32_t params;        /* index into the batch's gub_params table */
  int32_t created_delta;  /* created_at = created_base + created_delta (ms) */
} gub_kreq;               /* 16 bytes */
/* One buffer per batch: [gub_kreq x n][uint32 offsets x (n + 1)][key bytes]; key i = bytes[offsets[i] .. offsets[i+1]). */
int gub_keys_layout(size_t n, size_t key_bytes, size_t* offsets_at, size_t* bytes_at, size_t* total);
int gub_submit_keys_async(gub_table* t, const void* packed, size_t packed_bytes, size_t n, const gub_params* params, size_t n_params,
                          int64_t created_base, const gub_clock* clk, gub_resp* out, int* ticket);

/* ---- the Store plugin (config.go:95: Store.Get on a cache miss, Store.OnChange after an owner's update, Store.Remove when an item is
 * deleted; algorithms.go:45-51, 78-100, 149-153, 252-254, 274-315, 382-384, 488-490) on the key-string path, one batch at a time.
 * The device computes the batch's miss list before evaluating it and its change log after; the host calls the store.  The rule is
 * the host layer's (gubernator_b200_host.h gub_store), at batch granularity, per distinct key:
 *   Get       once per key that misses (absent, expired at now_ms, or past its InvalidAt), with the key's first request;
 *             what it returns is installed before the batch is evaluated (as gub_add_items installs it);
 *   Remove    when the item that existed at batch start was deleted: a TOKEN_BUCKET request with RESET_REMAINING anywhere among the
 *             key's requests, or an algorithm switch by its first request (a loaded item existed when its ExpireAt >= now_ms);
 *   OnChange  once, with the item as the batch left it, when the key is live afterwards and its last request has err_code 0 and
 *             carries GUB_REQ_IS_OWNER. */
enum { GUB_STORE_FOUND = 1, GUB_STORE_REMOVE = 2, GUB_STORE_CHANGE = 4 };
typedef struct {
  uint32_t first;   /* batch index of the key's first request (the request Store.Get receives) */
  uint32_t last;    /* batch index of the key's last request  (the request Store.OnChange receives) */
  uint32_t flags;   /* GUB_STORE_FOUND (Get: item filled by the callback) | GUB_STORE_REMOVE | GUB_STORE_CHANGE */
  uint16_t first_shard, last_shard;  /* rings: the shard whose ingest batch `first` / `last` index; 0 on a single table */
  gub_item item;    /* key_xxh64 / key_fnv1 always set by the library; the rest per flags */
} gub_store_rec;    /* 104 bytes */

/* Store.Get for the batch's misses, called once per batch, on the calling thread (which holds the table's lock: the callback must not
 * call into the library for this table), only when there is at least one miss.
 * Fill misses[k].item and set GUB_STORE_FOUND for the keys the store has.  Non-zero = fail the submission: nothing is evaluated. */
typedef int (*gub_store_get_fn)(void* user, gub_store_rec* misses, size_t n);

/* gub_submit_keys_async (same batch format, same responses on the same table state, except where Store.Get returned an item) plus the
 * Store's calls.  After gub_wait(ticket), changes[0 .. *n_changes) holds one record per key with GUB_STORE_REMOVE and/or
 * GUB_STORE_CHANGE set, ordered by `first`; call Remove, then OnChange, for each record in turn (the host layer's order).
 * `changes` (room for n records) and `n_changes` must be page-locked (gub_host_alloc): the device writes the records there directly,
 * so they cross PCIe once, 104 bytes each.
 * get == NULL (a write-behind store that never reads): fully asynchronous, like gub_submit_keys_async.
 * get != NULL: BLOCKS until this batch's miss list is known, which is after every earlier submission on this table has finished
 * evaluating: the pipelining of consecutive batches is lost.
 * Refused (with text in gub_last_error()): n > max_batch (a key split over two chunks would get two records), a table created under
 * GUB_PATH=fused, and `changes` / `n_changes` outside page-locked host memory.  Rings driven from one process: see
 * gub_p2p_step_keys_store_local_all. */
int gub_submit_keys_store_async(gub_table* t, const void* packed, size_t packed_bytes, size_t n, const gub_params* params,
                                size_t n_params, int64_t created_base, const gub_clock* clk,
                                gub_store_get_fn get, void* user,
                                gub_resp* out, gub_store_rec* changes, uint32_t* n_changes, int* ticket);

/* ---- wire bytes: V1Instance.GetRateLimits (gubernator.go:183-295) on one node, from the protobuf bytes of whole GetRateLimitsReq
 * messages (one per RPC) to the bytes of their GetRateLimitsResp.  The device decodes every message as protobuf-go does (field numbers of
 * gubernator.proto; unknown fields, the metadata map and known fields with another wire type skipped; open enums; created_at with
 * presence), checks each item as gubernator.go:208-220 does (empty unique_key, then empty name: answered in-band, not evaluated;
 * created_at absent or 0 = the message's default; behavior & 0xFF | GUB_REQ_IS_OWNER), hashes Name + "_" + UniqueKey, evaluates the
 * call's items as one batch (message order, then item order: the host layer's aggregator) and writes each message's response as Go's
 * proto.Marshal would: one 0x0A-framed RateLimitResp per item, zero fields omitted, the error text of gub_format_error in full.
 * One buffer per call: [int64 created_at x n_msgs][uint32 offsets x (n_msgs + 1)][message bytes]; message m = bytes[offsets[m] ..
 * offsets[m + 1]), offsets[0] = 0, at most 2^31 - 1 message bytes.  created_at[m] is the default of message m (gubernator.go:195 takes
 * one epochMillis(clock.Now()) per RPC).  gub_proto_layout also returns out_bound, a safe upper bound on the output bytes. */
enum { GUB_PROTO_OK = 0, GUB_PROTO_TOO_LARGE = 1 /* more than 1000 items: codes.OutOfRange (gubernator.go:189-193) */,
       GUB_PROTO_MALFORMED = 2 /* what grpc-go's unmarshal rejects */ };
int gub_proto_layout(size_t n_msgs, size_t msg_bytes, size_t* offsets_at, size_t* bytes_at, size_t* total, size_t* out_bound);
/* After gub_wait(ticket): msg_status[m] per message, and message m's response = out_bytes[out_off[m] .. out_off[m + 1]) (empty unless
 * GUB_PROTO_OK; nothing of a TOO_LARGE or MALFORMED message is evaluated, and the other messages are unaffected).
 * out_bytes (out_cap >= out_bound for the call's message bytes), out_off (n_msgs + 1) and msg_status (n_msgs) must be page-locked
 * (gub_host_alloc): the device writes them directly.  The offsets are checked on the host.  Pipelined like gub_submit_keys_async (up to
 * gub_pipeline_depth() calls in flight, library-owned staging), except that the call returns only once its messages are decoded: the
 * evaluation is sized by the number of items the device found. */
int gub_submit_proto_async(gub_table* t, const void* packed, size_t packed_bytes, size_t n_msgs, const gub_clock* clk, void* out_bytes,
                           size_t out_cap, uint64_t* out_off, uint32_t* msg_status, int* ticket);

/* Page-locked host memory for request/response buffers: with these the H2D/D2H copies of gub_submit_async are truly
 * asynchronous (a Go shim allocates its batch arenas here once).  Any other host memory works too, just slower. */
void* gub_host_alloc(size_t bytes);
void gub_host_free(void* p);

/* Gregorian tables for a batch clock: GregorianDuration / GregorianExpiration (interval.go:84-148), UTC. */
int gub_clock_fill(int64_t now_ms, gub_clock* out);

/* ---- WorkerPool.AddCacheItem (workers.go:537), WorkerPool.Load (workers.go:329), UpdatePeerGlobals
 *      (gubernator.go:425-459): upsert whole items.  Duplicate keys within one call: last one wins. ------------ */
int gub_add_items(gub_table* t, const gub_item* items, size_t n);
/* WorkerPool.GetCacheItem (workers.go:583) -> LRUCache.GetItem (lrucache.go:111): expired entries are misses. */
int gub_get_items(gub_table* t, const uint64_t* key_xxh64, const uint64_t* key_fnv1, size_t n, int64_t now_ms,
                  gub_item* out, uint8_t* found);
/* WorkerPool.Store (workers.go:451) -> Cache.Each (lrucache.go:76): every stored item, in no particular order.
 * Writes at most `cap` items; *n_out receives the total number stored. */
int gub_scan(gub_table* t, gub_item* out, size_t cap, size_t* n_out);
/* Cache.Size (lrucache.go:159) */
int gub_size(gub_table* t, size_t* n_out);
/* Reclaims slots whose item has expired (ExpireAt < now_ms) or was removed; the reference does this lazily on access
 * (lrucache.go:115) and by LRU eviction (lrucache.go:98,138).  *removed may be NULL. */
int gub_sweep(gub_table* t, int64_t now_ms, size_t* removed);
int gub_get_counters(gub_table* t, gub_counters* out);

/* Incremental expiry sweep inside the batch kernel: every CTA frees the removed / expired entries of `slots_per_cta` table slots
 * per batch (tombstones; tombstone runs that end at an empty slot become empty again), so that a long-running service does not
 * fill its probe windows with dead keys (the reference frees lazily on access, lrucache.go:115, and by eviction, :138).
 * Default: the whole table once every ~65536 batches.  0 = off. */
int gub_set_sweep(gub_table* t, uint32_t slots_per_cta);
/* Diagnostic: per-CTA timestamps at the phase boundaries of the batch kernel, for the last launch (12 marks: entry, tile issued,
 * tile landed, phase 1 done, grid barrier passed, probe done, entries read, evaluated, checked in, uniform groups finished,
 * non-uniform groups finished, counters flushed): us since the first CTA entered; max and mean over CTAs. */
int gub_set_trace(gub_table* t, int on);
int gub_get_trace(gub_table* t, double* max_us /* 12 */, double* mean_us /* 12 */);
int gub_get_trace_raw(gub_table* t, uint64_t* out /* 256 CTAs x 12 marks, ns; 0 = CTA not launched */);
/* The same for the four-kernel pipeline (also switched by gub_set_trace): out[(kernel * 1024 + block) * 8 + mark] = the latest
 * %globaltimer (ns) at which a warp of the block — for marks 2..5 inside role code: a thread in that role — passed the mark since the
 * last reset, 0 = never.  kernel: 0 k_group, 1 k_rank, 2 k_eval, 3 k_finish; marks: 0 entry (request loaded), 1 after
 * griddepcontrol.wait, 6 work done (before the block's last barrier), 7 exit; 2..5 per kernel (gub_kernels.cuh). */
int gub_get_ktrace(gub_table* t, uint64_t* out /* 4 x 1024 x 8 */, int reset);

/* Diagnostic: random 64-byte read-modify-write rate of the device over the table's own slots (contents unchanged), in GB/s
 * moved (64 B read + 64 B written per access): the "HBM random access" ceiling bench.py reports the path against. */
int gub_probe_random_access(gub_table* t, uint64_t accesses, double* gbs);
/* Optional per-kernel device timing of the batch path (CUDA events around k_group / k_rank / k_eval / k_finish), the
 * measurement counterpart of the reference's metricFuncTimeDuration summaries (gubernator.go:65-73).  Off by default. */
int gub_set_profiling(gub_table* t, int on);
int gub_get_profile(gub_table* t, double kernel_ms[4], uint64_t* launches, int reset);

/* ---- key hashing: client.go:39-41 HashKey + workers.go:153 + replicated_hash.go:108 -------------------------
 * keys are packed back to back in `bytes`; key i is bytes[offsets[i] .. offsets[i+1]).  Host implementation. */
int gub_hash_keys(const char* bytes, const uint64_t* offsets, size_t n, uint64_t* xxh64_out, uint64_t* fnv1_out);
/* The same on the device (all pointers device pointers on the table's GPU, enqueued on `stream`): outputs may be NULL;
 * d_reqs_out, when given, receives the two hashes in request i's key_xxh64 / key_fnv1 fields. */
int gub_hash_keys_device(gub_table* t, const char* d_bytes, const uint64_t* d_offsets, size_t n, uint64_t* d_xxh64_out,
                         uint64_t* d_fnv1_out, gub_req* d_reqs_out, void* stream);
uint64_t gub_xxh64(const void* data, size_t len, uint64_t seed);
uint64_t gub_fnv1_64(const void* data, size_t len);
uint64_t gub_fnv1a_64(const void* data, size_t len);

/* ---- ReplicatedConsistentHash (replicated_hash.go:36-119): which shard (GPU / peer) owns a key -------------- */
typedef struct gub_ring gub_ring;
gub_ring* gub_ring_create(int hash_kind /* 0 fnv1 (replicated_hash.go:33), 1 fnv1a (config.go:429) */, int replicas /* 0 = 512 */);
void gub_ring_destroy(gub_ring* r);
int gub_ring_add(gub_ring* r, const char* grpc_address);                 /* Add, replicated_hash.go:78-91 */
int gub_ring_size(const gub_ring* r);                                    /* Size, :94 */
int gub_ring_get(const gub_ring* r, const char* key, size_t len);        /* Get, :104-119; -1 when empty */
int gub_ring_get_by_hash(const gub_ring* r, uint64_t key_hash);
size_t gub_ring_points(const gub_ring* r, uint64_t* hashes, int32_t* peers, size_t cap);

/* ---- multi-GPU routing (replaces the peer forwarding of gubernator.go:257-283 / peer_client.go:284 inside one
 *      NVSwitch domain).  All pointers are device pointers on the table's GPU; work is enqueued on `stream`.
 *  gub_route_device: stable partition of a batch by owning shard: out_reqs holds the requests grouped by owner
 *      (owner 0 first), each group in original index order; perm[j] = original index of out_reqs[j];
 *      counts[g] = number of requests owned by shard g (device array of n_shards uint32).
 *  gub_unroute_device: resp_out[perm[j]] = resp_in[j]. */
int gub_route_device(gub_table* t, const gub_ring* ring, const gub_req* d_reqs, size_t n, gub_req* d_out_reqs,
                     uint32_t* d_perm, uint32_t* d_counts, void* stream);
int gub_unroute_device(gub_table* t, const gub_resp* d_resp_in, const uint32_t* d_perm, size_t n, gub_resp* d_resp_out,
                       void* stream);

/* ---- GLOBAL behaviour (global.go:30-283, gubernator.go:395-459): per-shard queues on the device -------------------
 * A gub_gq accumulates GLOBAL requests between sync ticks, keyed by the request's XXH64:
 *   mode 0 (hits queue,    runAsyncHits  global.go:91):  keeps the FIRST request per key, Hits summed, RESET_REMAINING OR-ed;
 *   mode 1 (update queue,  runBroadcasts global.go:193): keeps the LATEST request per key.
 * All pointers are device pointers on the queue's GPU; work is enqueued on `stream`. */
typedef struct gub_gq gub_gq;
int gub_gq_create(int device, uint32_t capacity, int keep_latest, gub_gq** out);
void gub_gq_destroy(gub_gq* q);
/* Feeds the queue from one batch.  d_owner: per-request owning shard (uint8, e.g. from gub_route_device's scratch via
 * gub_route_owner_device) or NULL.  With d_owner: select GLOBAL requests with Hits != 0 whose owner != self (a non-owner
 * queues its hits, gubernator.go:402-404).  Without: select every GLOBAL request with Hits != 0 (what an owner has just
 * evaluated still carries GLOBAL, gubernator.go:604-606).  `seq_base` orders requests across calls (first / latest). */
int gub_gq_accumulate_device(gub_gq* q, const gub_req* d_reqs, size_t n, const uint8_t* d_owner, uint32_t self,
                             uint64_t seq_base, void* stream);
/* Requests that were not queued because the queue was full within one window (the reference's maps are unbounded: size for the hot set). */
int gub_gq_dropped(gub_gq* q, uint64_t* dropped);
/* Drains the queue into request records and clears it: as_status_query = 0 -> hit requests for the owner (Hits = window
 * sum, DRAIN_OVER_LIMIT | IS_OWNER set, gubernator.go:510-512); 1 -> Hits = 0 status queries, IsOwner = false
 * (global.go:238-245).  *d_count (device uint32) receives the number of records (<= cap are written). */
int gub_gq_drain_device(gub_gq* q, gub_req* d_out, size_t cap, uint32_t* d_count, int as_status_query, void* stream);
/* Owner side of broadcastPeers (global.go:234-258): status-query requests + their responses -> UpdatePeerGlobal items. */
int gub_make_updates_device(gub_table* t, const gub_req* d_queries, const gub_resp* d_resps, size_t n, gub_item* d_items,
                            uint32_t* d_count, void* stream);
/* Peer side: UpdatePeerGlobals (gubernator.go:425-459) for a device-resident array of items; CreatedAt/UpdatedAt = now_ms. */
int gub_add_items_device(gub_table* t, const gub_item* d_items, size_t n, int64_t now_ms, void* stream);
/* Owning shard of every request of a batch (uint8 per request), by the ring (replicated_hash.go:104-119). */
int gub_route_owner_device(gub_table* t, const gub_ring* ring, const gub_req* d_reqs, size_t n, uint8_t* d_owner, void* stream);
/* gub_route_device variant for GLOBAL traffic: GLOBAL requests this shard does not own stay here and are evaluated
 * against the local replica with GLOBAL cleared, NO_BATCHING set and IsOwner = false (gubernator.go:259-269,408-411). */
int gub_route_global_device(gub_table* t, const gub_ring* ring, uint32_t self, const gub_req* d_reqs, size_t n, gub_req* d_out_reqs,
                            uint32_t* d_perm, uint32_t* d_counts, uint8_t* d_owner_out, void* stream);

/* ---- the ring of GPUs inside one box: fused routing over NVLink peer memory, GLOBAL sync with NCCL -----------------------------
 * (replaces gubernator.go:257-283 peer forwarding + peer_client.go:284 batching + global.go inside one NVSwitch domain)
 * One gub_p2p per shard (GPU): one process per GPU (gub_p2p_export / gub_p2p_connect swap cudaIpc handles), or all shards in
 * one process like the reference daemon (gub_p2p_connect_local enables peer access between the devices).
 * gub_p2p_step:
 *   k_p2p_route   partitions the ingest batch by owning shard (replicated_hash.go:104-119, stable: per-key order survives) and
 *                 stores every 64-byte record straight into the owner's mailbox; the last tile publishes the per-owner counts;
 *   on the owner  k_seg_wait (one warp waits for the W flags, bounded) -> the four batch kernels in ring mode: they read the W mailbox
 *                 segments in place (segment order = source rank, then source index) and store every 32-byte response straight into
 *                 the source's response mailbox -> k_seg_publish (response flags).  (GUB_PATH=fused: one launch of the persistent
 *                 kernel k_batch instead.)  gub_p2p_create sizes the table's batch scratch for min(world x cap, 262 144) requests
 *                 per pass;
 *   k_p2p_collect the source waits for the owners' flags and puts the responses back in request order.
 * Collective: every shard of the ring must call gub_p2p_step the same number of times.  n <= cap. */
typedef struct gub_p2p gub_p2p;
#define GUB_P2P_HANDLE_BYTES 64
int gub_p2p_create(gub_table* t, const gub_ring* ring /* one address per shard; must outlive the p2p */, uint32_t rank, uint32_t cap, gub_p2p** out);
void gub_p2p_destroy(gub_p2p* p);
int gub_p2p_export(gub_p2p* p, void* handle_out /* GUB_P2P_HANDLE_BYTES: a cudaIpcMemHandle_t */);
int gub_p2p_connect(gub_p2p* p, const void* handles /* world x GUB_P2P_HANDLE_BYTES, rank order; own entry ignored */);
int gub_p2p_connect_local(gub_p2p* p, gub_p2p* const* peers /* world pointers, same process; devices may differ */);
int gub_p2p_step(gub_p2p* p, const gub_req* d_reqs, size_t n, const gub_clock* clk, gub_resp* d_out, void* stream);
/* Same step on two streams: the routing kernel (partition + NVLink stores into the owners' mailboxes) runs on
 * `ingest_stream`, the stream d_reqs was produced on; evaluation, response return and collect run on `stream`,
 * where d_out becomes valid (GUB_RING_STREAMS=3, experimental: evaluation and collect on streams of the ring's own, `stream` only
 * waits for the collect).  Routing touches no bucket state, so the routing of step e+1 overlaps the evaluation of step
 * e (the reference overlaps forwarding and evaluation the same way: peer_client.go:284 runs in its own goroutine). */
int gub_p2p_step_streams(gub_p2p* p, const gub_req* d_reqs, size_t n, const gub_clock* clk, gub_resp* d_out, void* ingest_stream,
                         void* stream);
/* One step of every shard of this process, driven by ONE host thread (the reference daemon is one process, daemon.go:73): all
 * routings are enqueued, then all evaluations, then all collects.  streams[r] = the stream of shard r (on its device). */
int gub_p2p_step_local_all(gub_p2p* const* ps, uint32_t world, const gub_req* const* d_reqs, const size_t* n, const gub_clock* clk,
                           gub_resp* const* d_out, void* const* streams);
/* The ring fed with key strings: the step's ingest is a packed batch in the layout of gub_keys_layout ([gub_kreq x n][uint32 offsets
 * x (n + 1)][key bytes]) in device memory on the shard's GPU, and `params` a host array as for gub_submit_keys_async.  One kernel,
 * k_p2p_route_keys, hashes every key (XXH64 + FNV-1), expands its parameter set and created_at = created_base + created_delta
 * (an unknown parameter index answers GUB_ERR_INVALID_ALGORITHM in-band) and routes the record exactly as gub_p2p_step would route
 * the host-hashed one: same owner (by FNV-1, whatever the ring's hash_kind), same mailbox layout.  The rest of the step, GLOBAL
 * handling and the tick are unchanged; stream semantics are those of gub_p2p_step_streams (pass the same stream twice for one stream).
 * Offsets are not checked on the host (they live on the device); the kernel clamps them to the buffer: with key_bytes = packed_bytes -
 * bytes_at, key i = bytes[lo .. hi) with hi = min(offsets[i + 1], key_bytes) and lo = min(offsets[i], hi), so a malformed entry is
 * hashed as that (possibly empty) key and nothing outside the buffer is read.  packed_bytes must cover the records and offsets.
 * More than 32 parameter sets are copied on the ingest stream into a device buffer of the gub_p2p (one per step parity); the buffer
 * grows when a larger table arrives, which is the only allocation a step makes (and synchronises the device once).
 * Mixing: the mailbox format is the same for both kinds of ingest, so in one step some shards may ingest key strings while others
 * ingest records (gub_p2p_step_keys on some, gub_p2p_step on others; gub_p2p_step_mixed_local_all in one process).  The collective
 * rule is unchanged: every shard steps once per step, whichever entry it uses. */
int gub_p2p_step_keys(gub_p2p* p, const void* d_packed, size_t packed_bytes, size_t n, const gub_params* params, size_t n_params,
                      int64_t created_base, const gub_clock* clk, gub_resp* d_out, void* ingest_stream, void* stream);
/* gub_p2p_step_local_all with key strings: shard r ingests d_packed[r] (packed_bytes[r], n[r] requests); one parameter table. */
int gub_p2p_step_keys_local_all(gub_p2p* const* ps, uint32_t world, const void* const* d_packed, const size_t* packed_bytes, const size_t* n,
                                const gub_params* params, size_t n_params, int64_t created_base, const gub_clock* clk,
                                gub_resp* const* d_out, void* const* streams);
/* Both in one step of the shards of this process: shard r ingests key strings when d_packed[r] != NULL, else the records d_reqs[r]. */
int gub_p2p_step_mixed_local_all(gub_p2p* const* ps, uint32_t world, const gub_req* const* d_reqs, const void* const* d_packed,
                                 const size_t* packed_bytes, const size_t* n, const gub_params* params, size_t n_params,
                                 int64_t created_base, const gub_clock* clk, gub_resp* const* d_out, void* const* streams);
/* gub_p2p_step_keys_local_all with a Store plugin (see gub_submit_keys_store_async for the rule and gub_store_rec).  The step, its
 * responses and the tables are those of gub_p2p_step_keys_local_all on the same input, except where Store.Get returned an item.  Every
 * owner applies the single-table rule, per distinct key, to its pass: what it evaluates in the step, in source-rank order, then
 * source-index order.  A record names its requests by source: `first` indexes shard first_shard's ingest batch (d_packed[first_shard]),
 * `last` shard last_shard's.
 *   get       called once per owner that has misses, in rank order, on the calling thread, with that owner's misses ordered by pass
 *             index; every call completes before any owner installs or evaluates anything.  With a get the call BLOCKS until every
 *             shard's routing of this step is done; get == NULL: as asynchronous as gub_p2p_step_keys_local_all.  A non-zero return
 *             fails the call (the owners after it are not asked): no table is changed on any shard and d_out is undefined, but the
 *             ring stays in step (every owner publishes its response flags without evaluating, every shard's epoch advances) and the
 *             next step works normally.  The library keeps its own copy of each miss's request names (first, last, first_shard,
 *             last_shard) and keys: what the callback writes there is ignored.
 *             A table that cannot take the items Get returned fails the call the same way (nothing is evaluated, the ring stays in
 *             step), but it is detected only after every owner has installed: each owner's table keeps the items it placed and the
 *             parked inserts that were placed before them, as gub_add_items would have left it.
 *   changes[r] / n_changes[r]   owner r's change log: page-locked (gub_host_alloc), room for world x cap records; valid once
 *             streams[r] has completed the step.  Ordered by pass index; call Remove, then OnChange, for each record in turn.
 * Refused (with text in gub_last_error()): GUB_PATH=fused; a ring with GLOBAL enabled (the owner-side application of a tick's hits
 * would call Store.OnChange and needs a change log of its own); shards not connected with gub_p2p_connect_local; world x cap larger
 * than an owner's pass (the table's max_batch after gub_p2p_create: one pass per step keeps one record per key); change logs outside
 * page-locked memory.
 * Memory, allocated by the first Store step: on every shard the table's Store scratch (as gub_submit_keys_store_async allocates it:
 * 117 B x max_batch + 32 B x next_pow2(2 x max_batch) on the device, 200 B x max_batch page-locked) and an inverse map of its
 * routing, 2 x world x cap x 4 B on the device, which the owners read over peer access. */
int gub_p2p_step_keys_store_local_all(gub_p2p* const* ps, uint32_t world, const void* const* d_packed, const size_t* packed_bytes,
                                      const size_t* n, const gub_params* params, size_t n_params, int64_t created_base,
                                      const gub_clock* clk, gub_store_get_fn get, void* user, gub_resp* const* d_out,
                                      gub_store_rec* const* changes, uint32_t* const* n_changes, void* const* streams);
/* gub_submit_proto_async on the ring of this process: shard r takes the GetRateLimitsReq messages of packed[r] (host memory in the
 * layout of gub_proto_layout; any split of the RPCs over the shards is valid) and writes their responses to its own page-locked
 * out_bytes[r] (out_cap[r] >= out_bound) / out_off[r] (n_msgs[r] + 1) / msg_status[r] (n_msgs[r]), valid once streams[r] has completed
 * the call (no tickets: the ring's convention).  Per item the rules of gub_submit_proto_async apply unchanged (decoding, the checks of
 * gubernator.go:208-220, created_at per message, behavior & 0xFF | GUB_REQ_IS_OWNER, TOO_LARGE and MALFORMED messages evaluate nothing).
 *   force_global   Behaviors.ForceGlobal (gubernator.go:232-234): every item that passes the checks also gets GUB_BEHAVIOR_GLOBAL.
 *   evaluation     n_r = the evaluable items of shard r (message order, then item order), S = max_r ceil(n_r / cap): the call performs
 *                  S steps, and in step k shard r ingests its items [k x cap, min(n_r, (k + 1) x cap)) as the records of exactly the step
 *                  gub_p2p_step_local_all would perform.  For each key, items apply in (step, source rank, source index) order; with a
 *                  contiguous split and every n_r <= cap that is message order, and the bytes equal those of gub_submit_proto_async on one
 *                  table for the concatenated messages.  S = 0: no step, no epoch advances, the responses are still written.
 *   GLOBAL rings   as for record steps: a GLOBAL item another shard owns is answered from the replica and its hits are queued.
 *   timeouts       an item whose owner never answered (GUB_ERR_PEER_TIMEOUT) gets the error text of gubernator.go:374, "Error while
 *                  fetching rate limit '<key>' from peer: context deadline exceeded".
 * Blocks until every shard's messages are decoded (the steps are sized by the items the devices found) and, on each shard, until the
 * call two back is encoded: two sets of library-owned scratch per shard alternate by call parity, so consecutive calls need no
 * synchronisation by the caller and a call's decode overlaps the previous call's steps.  The sets grow with the input (allocating
 * synchronises the device).  Refused (text in gub_last_error()) before anything is copied or enqueued on any shard, so no epoch advances:
 * offsets that fail the checks of gub_submit_proto_async, out_cap below the bound, outputs outside page-locked memory, a shard that fails
 * the checks of gub_p2p_step_local_all, more than 2^31 - 1 messages on a shard; a failed allocation fails the call before any shard routes. */
int gub_p2p_step_proto_local_all(gub_p2p* const* ps, uint32_t world, const void* const* packed, const size_t* packed_bytes, const size_t* n_msgs,
                                 int force_global, const gub_clock* clk, void* const* out_bytes, const size_t* out_cap, uint64_t* const* out_off,
                                 uint32_t* const* msg_status, void* const* streams);
/* Device-side waits are bounded (a dead peer must not hang the GPU); a wait that gave up marks the step: *error_out != 0 and the
 * call fails with text in gub_last_error().  Requests whose owner never answered carry GUB_ERR_PEER_TIMEOUT in-band.  Costs a
 * device synchronisation: poll at your own cadence. */
int gub_p2p_status(gub_p2p* p, int* error_out);

/* GLOBAL behaviour (global.go, gubernator.go:395-459) for the ring.  After gub_p2p_enable_global, a step answers GLOBAL
 * requests this shard does not own from the local replica (GLOBAL cleared, NO_BATCHING set, IsOwner = false) and queues their
 * hits; GLOBAL requests evaluated as owner are queued for the broadcast.  gub_global_tick is the reference's GlobalSyncWait
 * timer made explicit: hits go to their owners (applied with DRAIN_OVER_LIMIT), owners re-read the touched keys with Hits = 0,
 * and an NCCL all-gather delivers the UpdatePeerGlobal items to every other shard, which overwrites its replica.
 * capacity = most distinct GLOBAL keys per sync window, rounded up to a power of two Q; every tick carries all the keys the queues
 * accepted.  Device memory per shard: the two queues, (64 + 32 + 88) B x Q of tick staging, a 256 KiB histogram, world x 256 KiB
 * for the histogram exchange and 88 B x min(Q, mailbox capacity) x world for the item all-gather. */
int gub_p2p_enable_global(gub_p2p* p, uint32_t capacity /* most distinct GLOBAL keys per sync window */);
int gub_nccl_unique_id(void* out128 /* 128 bytes: ncclUniqueId, to be handed to every shard by the host application */);
int gub_p2p_nccl_init(gub_p2p* p, const void* id128);                     /* one process per GPU; collective */
int gub_p2p_nccl_init_local(gub_p2p* const* ps, uint32_t world);           /* all shards in this process */
/* A window of more hit records than the mailboxes take (the capacity given to gub_p2p_create, per source) travels in rounds, one
 * mailbox epoch each.  The rounds are key-consistent: every source's record of a key travels in the same round, so an owner applies
 * them in source-rank order, as a single-round tick does.  Every shard's histogram of its records over the top 16 bits of XXH64
 * reaches every shard (one added host synchronisation per tick), and all shards derive the same rounds from it.  Keys crafted to
 * share their top 16 bits beyond that capacity are split over consecutive rounds: none is dropped, but for those keys the order
 * between sources is the round order. */
int gub_global_tick(gub_p2p* p, const gub_clock* clk, int64_t now_ms, void* stream, uint64_t* stats /* optional, 4 values */);
/* All shards in this process, driven by ONE host thread (gub_global_tick itself expects one calling thread per local shard). */
int gub_global_tick_local_all(gub_p2p* const* ps, uint32_t world, const gub_clock* clk, int64_t now_ms, void* const* streams,
                              uint64_t* stats /* optional, world x 4 */);

#ifdef __cplusplus
}
#endif
#endif /* GUBERNATOR_B200_H */
