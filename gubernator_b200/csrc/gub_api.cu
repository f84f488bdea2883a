// gub_api.cu — the C ABI (include/gubernator_b200.h) over the kernels in gub_kernels.cuh.
//
// This is the layer that sits where gubernator's WorkerPool sits (workers.go:54-61): gub_create = NewWorkerPool,
// gub_submit* = GetRateLimit for a whole batch, gub_add_items = AddCacheItem/Load, gub_scan = Store, gub_destroy = Close.
// There is no CPU fallback: every entry point that evaluates requests launches CUDA kernels or fails.
#include <cuda_runtime.h>

#include <dlfcn.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <condition_variable>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/gubernator_b200.h"
#include "gub_kernels.cuh"
#include "gub_batch.cuh"
#include "gub_global.cuh"
#include "gub_p2p.cuh"
#include "gub_store.cuh"
#include "gub_proto.cuh"

extern "C" uint64_t gub_ring_version_(const gub_ring* r);

namespace {

thread_local std::string g_err;
int fail(const std::string& msg) { g_err = msg; return -1; }

#define CK(call)                                                                                         \
  do {                                                                                                   \
    cudaError_t e__ = (call);                                                                            \
    if (e__ != cudaSuccess) {                                                                            \
      return fail(std::string(#call) + ": " + cudaGetErrorString(e__) + " (" __FILE__ ":" + std::to_string(__LINE__) + ")"); \
    }                                                                                                    \
  } while (0)

constexpr int PIPE_DEPTH = 4;
constexpr uint32_t FINISH_GRID_NO_MIXED = 8;  // k_finish blocks when batches have no non-uniform group (launch_chunk)

struct PipeSlot {
  gub_req* d_req = nullptr;
  gub_resp* d_resp = nullptr;
  gub_creq* d_creq = nullptr;       // compact submissions: what arrives over PCIe
  uint8_t* d_packed = nullptr;      // key-string submissions: [gub_kreq x n][offsets x (n+1)][key bytes]
  size_t packed_cap = 0;
  gub_params* d_params = nullptr;
  size_t cap = 0, params_cap = 0;
  cudaEvent_t in_done = nullptr, out_done = nullptr;
  bool busy = false;
  // wire-format submissions (gub_submit_proto_async): scratch sized by the call's input, grown on demand
  struct Proto {
    uint32_t *slot_base = nullptr, *batch_base = nullptr, *mcount = nullptr, *meval = nullptr, *mstatus = nullptr, *msize = nullptr;
    unsigned long long* moff = nullptr;
    gub::ProtoItem* items = nullptr;
    gub_req* sreq = nullptr;
    uint8_t *keys = nullptr, *stage = nullptr;
    size_t msgs_cap = 0, slots_cap = 0, bytes_cap = 0;
    uint32_t* h_neval = nullptr;      // mapped: the call's evaluable item count, written by k_proto_scan
    cudaEvent_t decoded = nullptr;
  } proto;
};

uint32_t next_pow2(uint64_t v) { uint64_t p = 1; while (p < v) p <<= 1; return (uint32_t)p; }

}  // namespace

struct gub_table {
  int device = 0;
  std::mutex mu;
  gub::Slot* table = nullptr;
  uint64_t capacity = 0;
  uint32_t max_batch = 0;
  // per-batch scratch of the four-kernel pipeline (gub_kernels.cuh).  What k_group writes comes in two sets, picked by epoch parity, so
  // that the next batch's k_group can run while the current batch still reads its set; a ring shard's table has set 0 only.
  struct Scratch {
    gub::AuxEntry* aux[2] = {};
    uint32_t *ent[2] = {}, *meta[2] = {}, *presence[2] = {};
    uint8_t* fragsize[2] = {};
    uint32_t *rank = nullptr, *order = nullptr, *mixed_ent = nullptr;
    ulonglong2* commit = nullptr;
    gub::BatchCtr* ctr = nullptr;
    uint32_t epoch = 0;
  } scr;
  uint32_t aux_entries = 0, pres_words = 0, max_blocks = 0;
  // the fused batch kernel (gub_batch.cuh): one scratch set, one cooperative launch per batch
  // Which kernels evaluate a single table's batches (gub_submit*): the four-kernel pipeline (default: consecutive batches
  // overlap) or the single persistent kernel (GUB_PATH=fused: one launch per batch, no overlap between
  // batches).  Rings (gub_p2p_*) always evaluate out of the mailboxes with the persistent kernel.
  bool fused = false;
  bool coop = true;                   // cooperative launch (co-residency of the grid guaranteed by the driver)
  int num_sms = 0;                    // the device's SM count (capped at FB_MAX_GRID): grid sizes of the persistent and grid-stride kernels
  uint32_t sweep_chunk = 0;           // slots every CTA sweeps per batch (incremental expiry sweep), 0 = off
  // the four-kernel pipeline's incremental sweep: every SWEEP_EVERY batches one slice of the table is swept between two batches
  // (k_sweep on the batch's stream: nothing else touches the table then); the whole table once every ~65 536 batches
  uint32_t since_sweep = 0;
  uint64_t sweep_cursor = 0;
  gub::GEntry* gaux = nullptr;
  uint32_t* gpres = nullptr;
  unsigned long long* gfrag = nullptr;
  uint16_t* gmembers = nullptr;
  gub::FCtl* ctl = nullptr;
  gub::OvfItem* ovf = nullptr;
  gub::InvIndex inv{};                // CacheItem.InvalidAt side index
  unsigned long long* trace = nullptr; // per-CTA phase timestamps of the last k_batch launch (gub_set_trace)
  unsigned long long* ktrace = nullptr; // pipeline kernels: [4][KT_BLOCKS][KT_MARKS] latest time stamps (gub_set_trace / gub_get_ktrace)
  unsigned long long* counters = nullptr;
  // ordering between streams that touch the shared scratch
  cudaEvent_t last_done = nullptr;
  cudaStream_t last_stream = nullptr; // stream of the most recent table-touching work
  bool last_pending = false;          // work was enqueued on last_stream after (or without) the last event record
  // host path
  cudaStream_t s_h2d = nullptr, s_compute = nullptr, s_d2h = nullptr;
  cudaStream_t s_proto = nullptr;     // decoding of wire-format calls: touches no table, so it does not wait for earlier evaluations
  cudaEvent_t compute_done[PIPE_DEPTH] = {};
  PipeSlot pipe[PIPE_DEPTH];
  int next_slot = 0;
  // maintenance scratch
  unsigned long long* d_scalar = nullptr;
  // route
  uint64_t* d_ring_pts = nullptr; int32_t* d_ring_peers = nullptr; uint16_t* d_ring_lut = nullptr; uint32_t ring_npts = 0; const gub_ring* ring_cached = nullptr; uint64_t ring_version = 0;
  uint8_t* d_owner = nullptr; uint32_t* d_tile_counts = nullptr;
  size_t owner_cap = 0, tiles_cap = 0;
  // optional per-kernel timing (bench.py's roofline leg): events bracket every kernel of the batch path
  bool pdl = true;                    // programmatic dependent launch between the batch kernels (GUB_PDL=0 disables)
  // GUB_PIPE_TRACE=<file>: stage timestamps of the first host-to-host submissions (diagnostic)
  std::string trace_path;
  cudaEvent_t trace_base = nullptr;
  std::vector<cudaEvent_t> trace_ev;  // 6 per traced submission
  bool prof = false;
  uint32_t* h_mixed_hint = nullptr;   // host-mapped word: non-uniform groups of the last batch k_eval saw (BatchArgs::mixed_hint)
  uint32_t* d_mixed_hint = nullptr;
  std::vector<cudaEvent_t> prof_ev;   // 5 events per pending chunk
  size_t prof_pending = 0;            // chunks recorded and not yet accumulated
  double prof_ms[4] = {0, 0, 0, 0};
  uint64_t prof_launches = 0;
  // the Store plugin's pre- and post-pass (gub_store.cuh, gub_submit_keys_store_async), allocated on first use, sized for max_batch
  struct StoreScratch {
    gub::StoreKey* keys = nullptr;
    uint32_t key_entries = 0, epoch = 0;
    uint32_t *kent = nullptr, *blk = nullptr, *d_failed = nullptr;
    gub::StoreState* bstate = nullptr;
    uint8_t* sel = nullptr;
    gub_store_rec* sparse = nullptr;
    // page-locked, read by the device in place: the miss list the Get callback receives, its count, the verdicts and items to install
    gub_store_rec* h_miss = nullptr;
    uint32_t* h_count = nullptr;
    uint4* h_loaded = nullptr;
    gub::DevItem* h_items = nullptr;
    cudaEvent_t misses_done = nullptr;
  } store;
};

namespace {

// Folds finished per-kernel event triples into the running totals.  force: wait for everything pending.
int prof_flush(gub_table* t, bool force) {
  if (!force && t->prof_pending < 1024) return 0;
  for (size_t c = 0; c < t->prof_pending; c++) {
    cudaEvent_t* pe = &t->prof_ev[c * 5];
    CK(cudaEventSynchronize(pe[4]));
    for (int k = 0; k < 4; k++) { float ms = 0; CK(cudaEventElapsedTime(&ms, pe[k], pe[k + 1])); t->prof_ms[k] += ms; }
    t->prof_launches++;
  }
  t->prof_pending = 0;
  return 0;
}

constexpr size_t TRACE_MAX = 400;  // submissions
inline bool tracing(gub_table* t) { return t->trace_base && t->trace_ev.size() < TRACE_MAX * 6; }
int trace_mark(gub_table* t, cudaStream_t st) {
  cudaEvent_t e;
  CK(cudaEventCreate(&e));
  CK(cudaEventRecord(e, st));
  t->trace_ev.push_back(e);
  return 0;
}
void trace_dump(gub_table* t) {
  if (!t->trace_base || t->trace_ev.empty()) return;
  cudaDeviceSynchronize();
  if (FILE* f = std::fopen(t->trace_path.c_str(), "w")) {
    std::fprintf(f, "# us since table creation: h2d_start h2d_done compute_start compute_done d2h_start d2h_done\n");
    for (size_t i = 0; i + 6 <= t->trace_ev.size(); i += 6) {
      for (int k = 0; k < 6; k++) { float ms = 0; cudaEventElapsedTime(&ms, t->trace_base, t->trace_ev[i + k]); std::fprintf(f, "%.1f%c", ms * 1e3, k == 5 ? '\n' : ' '); }
    }
    std::fclose(f);
  }
  for (auto e : t->trace_ev) cudaEventDestroy(e);
  t->trace_ev.clear();
  cudaEventDestroy(t->trace_base);
  t->trace_base = nullptr;  // one dump per table
}

// Launches one batch kernel, with programmatic stream serialization when enabled (the kernels call griddepcontrol.wait
// before touching anything an earlier kernel produced; without the attribute that instruction is a no-op).
template <typename K>
cudaError_t launch_k(gub_table* t, K kernel, uint32_t grid, uint32_t block, cudaStream_t st, const gub::BatchArgs& A, bool plain = false) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(block); cfg.dynamicSmemBytes = 0; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  // With per-kernel profiling on, an event record sits between consecutive kernels: they are launched plainly then (full stream
  // order; griddepcontrol.* are no-ops without the attribute) rather than as programmatic dependents of "the previous kernel".
  // `plain`: the stream's previous operation is not a kernel of this chain (the memsets at the epoch wrap): full stream order.
  cfg.attrs = attr; cfg.numAttrs = (t->pdl && !t->prof && !plain) ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, A);
}

void fused_base_args(gub_table* t, const gub_clock* clk, gub::FArgs& A) {
  std::memset(&A, 0, sizeof A);
  A.table = t->table; A.capacity = t->capacity; A.aux = t->gaux; A.presence = t->gpres; A.fragrow = t->gfrag; A.members = t->gmembers;
  A.ctl = t->ctl; A.ovf = t->ovf; A.counters = t->counters; A.sweep_chunk = t->sweep_chunk; A.trace = t->trace; A.inv = t->inv; A.clk = *clk;
}

// One launch of k_batch over the segments in A (A.seg / A.nseg / flags filled by the caller).  `total_hint` = number of requests
// when the host knows it (sizes the grid for small batches), 0 = only the device knows: one CTA per SM.
int launch_fused(gub_table* t, const gub::FArgs& A, uint64_t total_hint, cudaStream_t st) {
  uint32_t grid = (uint32_t)t->num_sms;
  if (total_hint) grid = (uint32_t)std::min<uint64_t>(grid, std::max<uint64_t>(1, (total_hint + 127) / 128 + A.nseg));
  cudaEvent_t* pe = nullptr;
  if (t->prof) {
    if (prof_flush(t, false)) return -1;
    if (t->prof_ev.size() < (t->prof_pending + 1) * 5) {
      for (int k = 0; k < 5; k++) { cudaEvent_t e; CK(cudaEventCreate(&e)); t->prof_ev.push_back(e); }
    }
    pe = &t->prof_ev[t->prof_pending * 5];
    t->prof_pending++;
    CK(cudaEventRecord(pe[0], st));
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(gub::FB_THREADS); cfg.dynamicSmemBytes = sizeof(gub::FSmem); cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (t->coop) { attr[na].id = cudaLaunchAttributeCooperative; attr[na].val.cooperative = 1; na++; }
  if (t->pdl) { attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization; attr[na].val.programmaticStreamSerializationAllowed = 1; na++; }
  cfg.attrs = attr; cfg.numAttrs = na;
  cudaError_t e = cudaLaunchKernelEx(&cfg, gub::k_batch, A);
  if (e != cudaSuccess && t->coop && t->pdl) {  // the two attributes do not combine on this driver: keep the co-residency guarantee
    cudaGetLastError();
    t->pdl = false;
    cfg.numAttrs = 1;
    e = cudaLaunchKernelEx(&cfg, gub::k_batch, A);
  }
  if (e != cudaSuccess) return fail(std::string("k_batch launch: ") + cudaGetErrorString(e));
  if (pe) { for (int k = 1; k < 5; k++) CK(cudaEventRecord(pe[k], st)); }
  return 0;
}

// Ring mode: the batch is the concatenation of mailbox segments (see BatchArgs::nseg).
struct SegDesc {
  uint32_t nseg = 0;
  const uint32_t* seg_off = nullptr;
  const gub_req* reqs[gub::MAX_SHARDS] = {};
  gub_resp* out[gub::MAX_SHARDS] = {};
};

// One batch (<= max_batch requests) through the four-kernel pipeline, chained with programmatic dependent launch.
int launch_chunk(gub_table* t, const gub_req* d_reqs, uint32_t n, const gub_clock* clk, gub_resp* d_out, cudaStream_t st,
                 const uint32_t* n_dev = nullptr, uint32_t n_off = 0, const SegDesc* seg = nullptr) {
  gub_table::Scratch& sc = t->scr;
  bool wrapped = false;
  if (sc.epoch >= 65535u) {  // 16-bit epoch tags wrapped: clear the grouping tables so stale tags cannot alias
    wrapped = true;
    for (gub::AuxEntry* aux : sc.aux) if (aux) CK(cudaMemsetAsync(aux, 0, (size_t)t->aux_entries * sizeof(gub::AuxEntry), st));
    // 65535 -> 1 keeps the parity: the batch after the wrap reuses ctr[1], which k_rank (it only resets the OTHER parity) left
    // holding batch 65535's allocators.  Clear both.
    CK(cudaMemsetAsync(sc.ctr, 0, 2 * sizeof(gub::BatchCtr), st));
    sc.epoch = 0;
  }
  sc.epoch++;
  gub::BatchArgs A;
  std::memset(&A, 0, sizeof A);
  if (seg) {
    A.nseg = seg->nseg; A.seg_off = seg->seg_off;
    for (uint32_t k = 0; k < seg->nseg; k++) { A.seg_reqs[k] = seg->reqs[k]; A.seg_out[k] = seg->out[k]; }
  }
  A.table = t->table; A.capacity = t->capacity; A.reqs = d_reqs; A.out = d_out; A.n = n; A.n_dev = n_dev; A.n_off = n_off; A.epoch = sc.epoch;
  const bool two_sets = sc.aux[1] != nullptr;
  const uint32_t par = two_sets ? (sc.epoch & 1u) : 0u;
  A.aux = sc.aux[par]; A.aux_mask = t->aux_entries - 1; A.presence = sc.presence[par]; A.fragsize = sc.fragsize[par];
  A.pres_words = t->pres_words; A.max_blocks = t->max_blocks; A.ent = sc.ent[par]; A.meta = sc.meta[par]; A.rank = sc.rank;
  A.commit = sc.commit; A.order = sc.order; A.mixed_ent = sc.mixed_ent; A.ctr = sc.ctr;
  A.counters = t->counters; A.ovf = t->ovf; A.ovf_count = &t->ctl->ovf_count; A.inv = t->inv;
  A.ktrace = t->ktrace;
  A.chain_done = &t->ctl->chain_done;
  A.early_ok = (two_sets && sc.epoch > 1u) ? 1u : 0u;  // (epoch 1: the first batch since the scratch was made or wrapped)
  A.mixed_hint = seg ? nullptr : t->d_mixed_hint;
  A.clk = *clk;
  const uint32_t blocks = (n + 255) / 256;
  cudaEvent_t* pe = nullptr;
  if (t->prof) {
    if (prof_flush(t, false)) return -1;
    if (t->prof_ev.size() < (t->prof_pending + 1) * 5) {
      for (int k = 0; k < 5; k++) { cudaEvent_t e; CK(cudaEventCreate(&e)); t->prof_ev.push_back(e); }
    }
    pe = &t->prof_ev[t->prof_pending * 5];
    t->prof_pending++;
    CK(cudaEventRecord(pe[0], st));
  }
  // k_finish: one block per SM, except on a single table with two scratch sets when the last batch k_eval has seen had no non-uniform
  // group (the bench workload: every repeated key a uniform run).  Then the next batch's k_group, which launches only once every
  // k_finish block has been resident, should not wait for 132 of them: a k_finish block (128 registers x 256 threads) fits on an SM only
  // beside ONE k_eval block, and 65 536 requests are 256 k_eval blocks on 132 SMs x 2, so 8 fit at once.  The count read here may be a
  // few batches old; the grid size changes how fast the non-uniform groups are worked off, never the results.
  const bool few_mixed = !seg && two_sets && t->h_mixed_hint && *(volatile const uint32_t*)t->h_mixed_hint == 0;
  const uint32_t fin_blocks = std::min<uint32_t>(few_mixed ? FINISH_GRID_NO_MIXED : (uint32_t)t->num_sms, std::max<uint32_t>(1u, n / 2));
  if (seg) {
    CK(launch_k(t, gub::k_group<true>, blocks, gub::GROUP_THREADS, st, A, wrapped));
    if (pe) CK(cudaEventRecord(pe[1], st));
    CK(launch_k(t, gub::k_rank<true>, blocks, gub::GROUP_THREADS, st, A));
    if (pe) CK(cudaEventRecord(pe[2], st));
    CK(launch_k(t, gub::k_eval<true>, blocks, gub::GROUP_THREADS, st, A));
    if (pe) CK(cudaEventRecord(pe[3], st));
    CK(launch_k(t, gub::k_finish<true>, fin_blocks, gub::MIXED_THREADS, st, A));
  } else {
    CK(launch_k(t, gub::k_group<false>, blocks, gub::GROUP_THREADS, st, A, wrapped));
    if (pe) CK(cudaEventRecord(pe[1], st));
    CK(launch_k(t, gub::k_rank<false>, blocks, gub::GROUP_THREADS, st, A));
    if (pe) CK(cudaEventRecord(pe[2], st));
    CK(launch_k(t, gub::k_eval<false>, blocks, gub::GROUP_THREADS, st, A));
    if (pe) CK(cudaEventRecord(pe[3], st));
    // non-uniform groups, one block each (grid-stride; normally none: the blocks return at once)
    CK(launch_k(t, gub::k_finish<false>, fin_blocks, gub::MIXED_THREADS, st, A));
  }
  if (pe) CK(cudaEventRecord(pe[4], st));
  CK(cudaGetLastError());
  return 0;
}

// The pipeline's share of the capacity policy (lrucache.go:115 frees expired items lazily on access; a table slot whose key never
// comes back would stay occupied for ever): every SWEEP_EVERY batches, 1/64 of the table is swept on the batch's stream, after the
// batch — removed / expired entries become tombstones, which inserts reuse.  (The persistent kernel sweeps a few slots per batch
// itself.)  Off with gub_set_sweep(t, 0) / GUB_SWEEP=0.
constexpr uint32_t SWEEP_EVERY = 1024;
int maybe_sweep(gub_table* t, const gub_clock* clk, cudaStream_t st) {
  if (!t->sweep_chunk || ++t->since_sweep < SWEEP_EVERY) return 0;
  t->since_sweep = 0;
  const uint64_t slice = (t->capacity + 63) / 64;
  const uint64_t lo = t->sweep_cursor, hi = std::min<uint64_t>(t->capacity, lo + slice);
  t->sweep_cursor = hi >= t->capacity ? 0 : hi;
  gub::k_sweep<<<t->num_sms * 4, 256, 0, st>>>(t->table, lo, hi, clk->now_ms, t->counters + gub::C_SWEPT);
  CK(cudaGetLastError());
  return 0;
}

// Table-touching work from different caller streams must be ordered.  The common case (same stream as last time) costs
// nothing; only a change of stream records an event on the old stream and makes the new one wait for it.
int order_after_last(gub_table* t, cudaStream_t st) {
  if (t->last_pending && t->last_stream != st) {
    CK(cudaEventRecord(t->last_done, t->last_stream));
    CK(cudaStreamWaitEvent(st, t->last_done, 0));
    t->last_pending = false;
  }
  return 0;
}

// n_dev != nullptr: the real batch size is *n_dev (<= n) on the device; launches are sized for n and trim themselves.
int launch_batch(gub_table* t, const gub_req* d_reqs, size_t n, const gub_clock* clk, gub_resp* d_out, cudaStream_t st,
                 const uint32_t* n_dev = nullptr) {
  if (order_after_last(t, st)) return -1;
  if (t->fused) {  // any size in one launch: the kernel takes the batch in rounds of one tile per CTA
    if (n > 0xFFFFFFFFull) return fail("batch too large");
    gub::FArgs A;
    fused_base_args(t, clk, A);
    A.seg[0].reqs = d_reqs; A.seg[0].out = d_out; A.seg[0].n = (uint32_t)n; A.seg[0].n_dev = n_dev;
    A.nseg = 1;
    if (((uintptr_t)d_reqs & 15u) || ((uintptr_t)d_out & 15u)) return fail("request / response buffers must be 16-byte aligned");
    if (launch_fused(t, A, n_dev ? 0 : n, st)) return -1;
    t->last_stream = st; t->last_pending = true;
    return 0;
  }
  for (size_t off = 0; off < n; off += t->max_batch) {
    const uint32_t m = (uint32_t)std::min<size_t>(t->max_batch, n - off);
    if (launch_chunk(t, d_reqs + off, m, clk, d_out + off, st, n_dev, (uint32_t)off)) return -1;
  }
  if (maybe_sweep(t, clk, st)) return -1;
  t->last_stream = st; t->last_pending = true;
  return 0;
}

void free_slot(PipeSlot& s) {
  if (s.d_req) cudaFree(s.d_req);
  if (s.d_resp) cudaFree(s.d_resp);
  if (s.d_creq) cudaFree(s.d_creq);
  if (s.d_packed) cudaFree(s.d_packed);
  if (s.d_params) cudaFree(s.d_params);
  if (s.in_done) cudaEventDestroy(s.in_done);
  if (s.out_done) cudaEventDestroy(s.out_done);
  auto& pr = s.proto;
  void* dev[] = {pr.slot_base, pr.batch_base, pr.mcount, pr.meval, pr.mstatus, pr.msize, pr.moff, pr.items, pr.sreq, pr.keys, pr.stage};
  for (void* p : dev) if (p) cudaFree(p);
  if (pr.h_neval) cudaFreeHost(pr.h_neval);
  if (pr.decoded) cudaEventDestroy(pr.decoded);
  s = PipeSlot();
}

int ensure_slot(PipeSlot& s, size_t n) {
  if (s.cap >= n) return 0;
  if (s.d_req) cudaFree(s.d_req);
  if (s.d_resp) cudaFree(s.d_resp);
  if (s.d_creq) cudaFree(s.d_creq);
  s.d_req = nullptr; s.d_resp = nullptr; s.d_creq = nullptr; s.cap = 0;
  CK(cudaMalloc(&s.d_req, n * sizeof(gub_req)));
  CK(cudaMalloc(&s.d_resp, n * sizeof(gub_resp)));
  s.cap = n;
  return 0;
}

gub::DevItem to_dev(const gub_item& it) {
  gub::DevItem d;
  std::memset(&d, 0, sizeof d);
  d.key = it.key_xxh64 < 2 ? it.key_xxh64 + 2 : it.key_xxh64;
  d.tag = it.key_fnv1 >> 8;
  const bool leaky = it.algorithm == GUB_LEAKY_BUCKET;
  d.flags = gub::F_LIVE | (leaky ? gub::F_LEAKY : 0u) | ((!leaky && it.status == GUB_OVER_LIMIT) ? gub::F_OVER : 0u);
  d.w[0] = (uint64_t)it.limit; d.w[1] = (uint64_t)it.duration;
  if (leaky) std::memcpy(&d.w[2], &it.remaining_f, 8); else d.w[2] = (uint64_t)it.remaining;
  d.w[3] = (uint64_t)it.stamp; d.w[4] = leaky ? (uint64_t)it.burst : 0; d.w[5] = (uint64_t)it.expire_at;
  d.invalid_at = it.invalid_at;
  return d;
}
gub_item from_dev(const gub::DevItem& d) {
  gub_item it;
  std::memset(&it, 0, sizeof it);
  it.key_xxh64 = d.key; it.key_fnv1 = d.tag << 8;
  const bool leaky = (d.flags & gub::F_LEAKY) != 0;
  it.algorithm = leaky ? GUB_LEAKY_BUCKET : GUB_TOKEN_BUCKET;
  it.status = (d.flags & gub::F_OVER) ? GUB_OVER_LIMIT : GUB_UNDER_LIMIT;
  it.limit = (int64_t)d.w[0]; it.duration = (int64_t)d.w[1];
  if (leaky) std::memcpy(&it.remaining_f, &d.w[2], 8); else it.remaining = (int64_t)d.w[2];
  it.stamp = (int64_t)d.w[3]; it.burst = (int64_t)d.w[4]; it.expire_at = (int64_t)d.w[5];
  it.invalid_at = d.invalid_at;
  return it;
}

void free_scratch(gub_table::Scratch& sc) {
  for (int s = 0; s < 2; s++) {
    void* set[] = {sc.aux[s], sc.ent[s], sc.meta[s], sc.presence[s], sc.fragsize[s]};
    for (void* p : set) if (p) cudaFree(p);
  }
  void* rest[] = {sc.rank, sc.order, sc.mixed_ent, sc.commit, sc.ctr};
  for (void* p : rest) if (p) cudaFree(p);
  sc = gub_table::Scratch();
}

// Per-batch scratch of the four-kernel pipeline for batches of up to B requests (replaces what was there: the device must be idle).
// sets = 2: a second set of what k_group writes (aux, presence, fragsize, ent, meta; 80.5 MiB more at B = 65 536), which lets the next
// batch's k_group overlap the current batch (launch_chunk).
int alloc_scratch(gub_table* t, uint32_t B, int sets) {
  auto& sc = t->scr;
  free_scratch(sc);
  B = std::max<uint32_t>(1024u, std::min<uint32_t>(B, 262144u));
  B = (B + 255u) & ~255u;
  t->max_batch = B;
  t->aux_entries = next_pow2((uint64_t)B * 4);
  t->max_blocks = (B / gub::GROUP_THREADS + 127u) & ~127u;  // fragment-size row per group entry; a multiple of 128 blocks = 4 presence words (16-byte loads)
  t->pres_words = t->max_blocks / 32;
  struct { void** p; size_t bytes; } want[] = {
      {(void**)&sc.aux[0], (size_t)t->aux_entries * sizeof(gub::AuxEntry)},
      {(void**)&sc.presence[0], (size_t)t->aux_entries * t->pres_words * 4},
      {(void**)&sc.fragsize[0], (size_t)t->aux_entries * t->max_blocks},
      {(void**)&sc.ent[0], (size_t)B * 4}, {(void**)&sc.meta[0], (size_t)B * 4},
      {(void**)&sc.aux[1], sets > 1 ? (size_t)t->aux_entries * sizeof(gub::AuxEntry) : 0},
      {(void**)&sc.presence[1], sets > 1 ? (size_t)t->aux_entries * t->pres_words * 4 : 0},
      {(void**)&sc.fragsize[1], sets > 1 ? (size_t)t->aux_entries * t->max_blocks : 0},
      {(void**)&sc.ent[1], sets > 1 ? (size_t)B * 4 : 0}, {(void**)&sc.meta[1], sets > 1 ? (size_t)B * 4 : 0},
      {(void**)&sc.commit, (size_t)t->aux_entries * 6 * sizeof(ulonglong2)},
      {(void**)&sc.rank, (size_t)B * 4}, {(void**)&sc.order, (size_t)B * 4},
      {(void**)&sc.mixed_ent, ((size_t)B / 2 + 1) * 4}, {(void**)&sc.ctr, 2 * sizeof(gub::BatchCtr)},
  };
  for (auto& w : want) {
    if (!w.bytes) continue;
    cudaError_t e = cudaMalloc(w.p, w.bytes);
    if (e != cudaSuccess) return fail(std::string("cudaMalloc(batch scratch): ") + cudaGetErrorString(e));
    CK(cudaMemset(*w.p, 0, w.bytes));
  }
  return 0;
}

}  // namespace

extern "C" {

const char* gub_last_error(void) { return g_err.c_str(); }
int gub_abi_version(void) { return GUB_ABI_VERSION; }

void gub_destroy(gub_table* t) {
  if (!t) return;
  cudaSetDevice(t->device);
  cudaDeviceSynchronize();
  trace_dump(t);
  void* ptrs[] = {t->table, t->counters, t->d_scalar, t->d_ring_pts, t->d_ring_peers, t->d_ring_lut, t->d_owner, t->d_tile_counts,
                  t->gaux, t->gpres, t->gfrag, t->gmembers, t->ctl, t->ovf, t->trace, t->ktrace, t->inv.e};
  for (void* p : ptrs) if (p) cudaFree(p);
  free_scratch(t->scr);
  for (auto& s : t->pipe) free_slot(s);
  for (auto& e : t->compute_done) if (e) cudaEventDestroy(e);
  for (auto& e : t->prof_ev) cudaEventDestroy(e);
  {
    auto& ss = t->store;
    void* dev[] = {ss.keys, ss.kent, ss.blk, ss.d_failed, ss.bstate, ss.sel, ss.sparse};
    for (void* p : dev) if (p) cudaFree(p);
    void* host[] = {ss.h_miss, ss.h_count, ss.h_loaded, ss.h_items};
    for (void* p : host) if (p) cudaFreeHost(p);
    if (ss.misses_done) cudaEventDestroy(ss.misses_done);
  }
  if (t->h_mixed_hint) cudaFreeHost(t->h_mixed_hint);
  if (t->last_done) cudaEventDestroy(t->last_done);
  if (t->s_h2d) cudaStreamDestroy(t->s_h2d);
  if (t->s_compute) cudaStreamDestroy(t->s_compute);
  if (t->s_d2h) cudaStreamDestroy(t->s_d2h);
  if (t->s_proto) cudaStreamDestroy(t->s_proto);
  delete t;
}

int gub_create(const gub_config* cfg, gub_table** out) {
  if (!cfg || !out) return fail("gub_create: null argument");
  *out = nullptr;
  if (cfg->capacity_slots < 64) return fail("gub_create: capacity_slots must be >= 64");
  int ndev = 0;
  CK(cudaGetDeviceCount(&ndev));
  if (cfg->device < 0 || cfg->device >= ndev) return fail("gub_create: no such CUDA device");
  CK(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9 || prop.minor != 0) return fail("gub_create: this library is built for sm_90a (H100) only");
  gub_table* t = new gub_table();
  t->device = cfg->device;
  if (const char* e = getenv("GUB_PDL")) t->pdl = std::atoi(e) != 0;
  t->capacity = cfg->capacity_slots;
  t->max_batch = cfg->max_batch ? cfg->max_batch : 65536u;
  if (t->max_batch < 1024) t->max_batch = 1024;
  if (t->max_batch > 262144u) t->max_batch = 262144u;
  t->max_batch = (t->max_batch + 255u) & ~255u;
#define ALLOC(ptr, bytes)                                                    \
  do {                                                                       \
    cudaError_t e__ = cudaMalloc((void**)&(ptr), (bytes));                   \
    if (e__ != cudaSuccess) {                                                \
      fail(std::string("cudaMalloc(" #ptr "): ") + cudaGetErrorString(e__)); \
      gub_destroy(t);                                                        \
      return -1;                                                             \
    }                                                                        \
    cudaMemset((ptr), 0, (bytes));                                           \
  } while (0)
  ALLOC(t->table, t->capacity * sizeof(gub::Slot));
  // two scratch sets up to 65 536 requests per batch (80.5 MiB more); beyond that the second set would cost 4 x as much per 4 x requests
  if (alloc_scratch(t, t->max_batch, t->max_batch <= 65536u ? 2 : 1)) { gub_destroy(t); return -1; }
  t->num_sms = std::min<int>(prop.multiProcessorCount, gub::FB_MAX_GRID);
  if (const char* e = getenv("GUB_PATH")) t->fused = std::string(e) == "fused";
  if (const char* e = getenv("GUB_COOP")) t->coop = std::atoi(e) != 0;
  ALLOC(t->gaux, (size_t)gub::FB_AUX_ENTRIES * sizeof(gub::GEntry));
  ALLOC(t->gpres, (size_t)gub::FB_AUX_ENTRIES * gub::FB_PRES_WORDS * 4);
  ALLOC(t->gfrag, (size_t)gub::FB_AUX_ENTRIES * gub::FB_ROW * 8);
  ALLOC(t->gmembers, (size_t)gub::FB_MAX_GRID * gub::FB_THREADS * 2);
  ALLOC(t->ctl, sizeof(gub::FCtl));
  ALLOC(t->ovf, (size_t)gub::FB_OVF_CAP * sizeof(gub::OvfItem));
  ALLOC(t->inv.e, (size_t)65536 * sizeof(gub::InvEntry));
  {
    cudaError_t e = cudaHostAlloc((void**)&t->h_mixed_hint, sizeof(uint32_t), cudaHostAllocMapped);
    if (e == cudaSuccess) { *t->h_mixed_hint = 0; e = cudaHostGetDevicePointer((void**)&t->d_mixed_hint, t->h_mixed_hint, 0); }
    if (e != cudaSuccess) { fail(std::string("cudaHostAlloc(mixed_hint): ") + cudaGetErrorString(e)); gub_destroy(t); return -1; }
  }
  t->inv.mask = 65535;
  {
    // incremental expiry sweep: the whole table once every ~65536 batches (GUB_SWEEP=<slots per CTA per batch>, 0 = off)
    uint64_t chunk = (t->capacity + (uint64_t)t->num_sms * 65536 - 1) / ((uint64_t)t->num_sms * 65536);
    if (const char* e = getenv("GUB_SWEEP")) chunk = (uint64_t)std::atoll(e);
    t->sweep_chunk = (uint32_t)std::min<uint64_t>(chunk, 1024);
    cudaError_t e2 = cudaFuncSetAttribute(gub::k_batch, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(gub::FSmem));
    if (e2 != cudaSuccess) { fail(std::string("cudaFuncSetAttribute(k_batch): ") + cudaGetErrorString(e2)); gub_destroy(t); return -1; }
  }
  ALLOC(t->counters, gub::C_COUNT * sizeof(unsigned long long));
  ALLOC(t->d_scalar, 4 * sizeof(unsigned long long));
#undef ALLOC
  CK(cudaStreamCreateWithFlags(&t->s_h2d, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&t->s_compute, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&t->s_d2h, cudaStreamNonBlocking));
  CK(cudaEventCreateWithFlags(&t->last_done, cudaEventDisableTiming));
  for (int i = 0; i < PIPE_DEPTH; i++) {
    CK(cudaEventCreateWithFlags(&t->pipe[i].in_done, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&t->pipe[i].out_done, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&t->compute_done[i], cudaEventDisableTiming));
  }
  if (const char* e = getenv("GUB_PIPE_TRACE")) {
    t->trace_path = e;
    CK(cudaEventCreate(&t->trace_base));
    CK(cudaEventRecord(t->trace_base, t->s_h2d));
  }
  CK(cudaDeviceSynchronize());
  *out = t;
  return 0;
}

int gub_submit_device(gub_table* t, const gub_req* d_reqs, size_t n, const gub_clock* clk, gub_resp* d_out, void* stream) {
  if (!t || !clk || (n && (!d_reqs || !d_out))) return fail("gub_submit_device: null argument");
  if (n == 0) return 0;
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  return launch_batch(t, d_reqs, n, clk, d_out, (cudaStream_t)stream);
}

int gub_submit_device_n(gub_table* t, const gub_req* d_reqs, size_t n_cap, const uint32_t* d_n, const gub_clock* clk, gub_resp* d_out, void* stream) {
  if (!t || !clk || !d_n || (n_cap && (!d_reqs || !d_out))) return fail("gub_submit_device_n: null argument");
  if (n_cap == 0) return 0;
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  return launch_batch(t, d_reqs, n_cap, clk, d_out, (cudaStream_t)stream, d_n);
}

int gub_pipeline_depth(gub_table*) { return PIPE_DEPTH; }

int gub_submit_async(gub_table* t, const gub_req* reqs, size_t n, const gub_clock* clk, gub_resp* out, int* ticket) {
  if (!t || !clk || !ticket || (n && (!reqs || !out))) return fail("gub_submit_async: null argument");
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  const int si = t->next_slot;
  t->next_slot = (t->next_slot + 1) % PIPE_DEPTH;
  PipeSlot& s = t->pipe[si];
  if (s.busy) { CK(cudaEventSynchronize(s.out_done)); s.busy = false; }
  *ticket = si;
  if (n == 0) { CK(cudaEventRecord(s.out_done, t->s_d2h)); s.busy = true; return 0; }
  if (ensure_slot(s, n)) return -1;
  CK(cudaMemcpyAsync(s.d_req, reqs, n * sizeof(gub_req), cudaMemcpyHostToDevice, t->s_h2d));
  CK(cudaEventRecord(s.in_done, t->s_h2d));
  CK(cudaStreamWaitEvent(t->s_compute, s.in_done, 0));
  if (launch_batch(t, s.d_req, n, clk, s.d_resp, t->s_compute)) return -1;
  CK(cudaEventRecord(t->compute_done[si], t->s_compute));
  CK(cudaStreamWaitEvent(t->s_d2h, t->compute_done[si], 0));
  CK(cudaMemcpyAsync(out, s.d_resp, n * sizeof(gub_resp), cudaMemcpyDeviceToHost, t->s_d2h));
  CK(cudaEventRecord(s.out_done, t->s_d2h));
  s.busy = true;
  return 0;
}

int gub_submit_compact_async(gub_table* t, const gub_creq* reqs, size_t n, const gub_params* params, size_t n_params, int64_t created_base,
                             const gub_clock* clk, gub_resp* out, int* ticket) {
  if (!t || !clk || !ticket || (n && (!reqs || !out || !params))) return fail("gub_submit_compact_async: null argument");
  if (n > 0xFFFFFFFFull || n_params > 0xFFFFFFFFull) return fail("gub_submit_compact_async: too large");
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  const int si = t->next_slot;
  t->next_slot = (t->next_slot + 1) % PIPE_DEPTH;
  PipeSlot& s = t->pipe[si];
  if (s.busy) { CK(cudaEventSynchronize(s.out_done)); s.busy = false; }
  *ticket = si;
  if (n == 0) { CK(cudaEventRecord(s.out_done, t->s_d2h)); s.busy = true; return 0; }
  if (ensure_slot(s, n)) return -1;
  if (!s.d_creq) CK(cudaMalloc(&s.d_creq, s.cap * sizeof(gub_creq)));
  const bool inl = n_params <= gub::INLINE_PARAMS;  // the table travels in the kernel arguments: no second copy
  if (!inl && (s.params_cap < n_params || !s.d_params)) {
    if (s.d_params) cudaFree(s.d_params);
    s.d_params = nullptr;
    s.params_cap = std::max<size_t>(n_params, 1024);
    CK(cudaMalloc(&s.d_params, s.params_cap * sizeof(gub_params)));
  }
  const bool tr = tracing(t);
  if (tr && trace_mark(t, t->s_h2d)) return -1;
  CK(cudaMemcpyAsync(s.d_creq, reqs, n * sizeof(gub_creq), cudaMemcpyHostToDevice, t->s_h2d));
  if (!inl) CK(cudaMemcpyAsync(s.d_params, params, n_params * sizeof(gub_params), cudaMemcpyHostToDevice, t->s_h2d));
  CK(cudaEventRecord(s.in_done, t->s_h2d));
  if (tr && trace_mark(t, t->s_h2d)) return -1;
  CK(cudaStreamWaitEvent(t->s_compute, s.in_done, 0));
  if (tr && trace_mark(t, t->s_compute)) return -1;
  // The expansion runs on the compute stream: a kernel behind a copy on the copy stream costs an engine switch per batch that
  // stalls the ingest stage under PCIe load.
  if (inl) {
    gub::InlineParams P;
    static_assert(sizeof(gub_params) == 32, "gub_params is two 16-byte words");
    std::memset(&P, 0, sizeof P);
    std::memcpy(&P, params, n_params * sizeof(gub_params));
    gub::k_expand_inline<<<(unsigned)((n + 255) / 256), 256, 0, t->s_compute>>>(s.d_creq, (uint32_t)n, P, (uint32_t)n_params, created_base, s.d_req);
  } else {
    gub::k_expand<<<(unsigned)((n + 255) / 256), 256, 0, t->s_compute>>>(s.d_creq, (uint32_t)n, s.d_params, (uint32_t)n_params, created_base, s.d_req);
  }
  if (launch_batch(t, s.d_req, n, clk, s.d_resp, t->s_compute)) return -1;
  CK(cudaEventRecord(t->compute_done[si], t->s_compute));
  if (tr && trace_mark(t, t->s_compute)) return -1;
  CK(cudaStreamWaitEvent(t->s_d2h, t->compute_done[si], 0));
  if (tr && trace_mark(t, t->s_d2h)) return -1;
  CK(cudaMemcpyAsync(out, s.d_resp, n * sizeof(gub_resp), cudaMemcpyDeviceToHost, t->s_d2h));
  CK(cudaEventRecord(s.out_done, t->s_d2h));
  if (tr && trace_mark(t, t->s_d2h)) return -1;
  if (tr && t->trace_ev.size() >= TRACE_MAX * 6) trace_dump(t);
  s.busy = true;
  return 0;
}

/* Key strings in, responses out: the host ships raw key bytes and 16-byte request records; hashing (XXH64 + FNV-1), the
 * expansion of the per-limit parameters and the evaluation all run on the device.  `packed` = [gub_kreq x n][uint32 offsets x
 * (n + 1)][key bytes] in one buffer (one host-to-device copy per batch: small separate copies cost the copy stream far more than
 * their size); gub_keys_layout() gives the offsets of the three parts. */
int gub_keys_layout(size_t n, size_t key_bytes, size_t* offsets_at, size_t* bytes_at, size_t* total) {
  if (!offsets_at || !bytes_at || !total) return fail("gub_keys_layout: null argument");
  *offsets_at = n * sizeof(gub_kreq);
  *bytes_at = *offsets_at + (n + 1) * 4;
  *total = (*bytes_at + key_bytes + 15) & ~(size_t)15;
  return 0;
}

}  // extern "C"

extern "C" {
namespace {
int drain_pending(gub_table* t, cudaStream_t st = 0);  // (defined with gub_add_items)
}  // namespace
}  // extern "C"

namespace {

// A Store plugin's part in one submission (gub_submit_keys_store_async): the Get callback and where the change log goes (device views
// of the caller's page-locked buffers).
struct StoreCall {
  gub_store_get_fn get;
  void* user;
  gub_store_rec* changes;
  uint32_t* n_changes;
};

int store_ensure(gub_table* t) {
  auto& ss = t->store;
  if (ss.keys) return 0;
  const size_t B = t->max_batch;
  ss.key_entries = next_pow2((uint64_t)B * 2);
  struct { void** p; size_t bytes; } dev[] = {
      {(void**)&ss.keys, (size_t)ss.key_entries * sizeof(gub::StoreKey)}, {(void**)&ss.kent, B * 4},
      {(void**)&ss.blk, (B / gub::STORE_THREADS + 1) * 4}, {(void**)&ss.d_failed, 4}, {(void**)&ss.bstate, B * sizeof(gub::StoreState)},
      {(void**)&ss.sel, B}, {(void**)&ss.sparse, B * sizeof(gub_store_rec)}};
  for (auto& d : dev) {
    CK(cudaMalloc(d.p, d.bytes));
    CK(cudaMemset(*d.p, 0, d.bytes));
  }
  struct { void** p; size_t bytes; } host[] = {{(void**)&ss.h_miss, B * sizeof(gub_store_rec)}, {(void**)&ss.h_count, 64},
                                               {(void**)&ss.h_loaded, B * sizeof(uint4)}, {(void**)&ss.h_items, B * sizeof(gub::DevItem)}};
  for (auto& h : host) CK(cudaHostAlloc(h.p, h.bytes, cudaHostAllocMapped));
  CK(cudaEventCreateWithFlags(&ss.misses_done, cudaEventDisableTiming));
  return 0;
}

template <typename T>
int device_view(T* host_ptr, T** dev_ptr) {
  CK(cudaHostGetDevicePointer((void**)dev_ptr, host_ptr, 0));
  return 0;
}

// What every Store pass shares: the scratch (allocated on first use), the dedup epoch, the table and the clock.  The caller sets
// S.reqs / S.n (and S.out before the post-pass).
int store_args(gub_table* t, const gub_clock* clk, bool want_misses, gub::StoreArgs& S, cudaStream_t st) {
  if (store_ensure(t)) return -1;
  if (order_after_last(t, st)) return -1;  // the lookups read the table
  auto& ss = t->store;
  if (ss.epoch >= 0xFFFFFFFFu) {  // the epoch tags of the dedup scratch wrapped: stale entries must not alias
    CK(cudaMemsetAsync(ss.keys, 0, (size_t)ss.key_entries * sizeof(gub::StoreKey), st));
    ss.epoch = 0;
  }
  ss.epoch++;
  std::memset(&S, 0, sizeof S);
  S.epoch = ss.epoch; S.keys = ss.keys; S.key_mask = ss.key_entries - 1; S.kent = ss.kent; S.bstate = ss.bstate;
  S.sel = ss.sel; S.sparse = ss.sparse; S.blk = ss.blk; S.table = t->table; S.capacity = t->capacity; S.ovf = t->ovf;
  S.ovf_count = &t->ctl->ovf_count; S.inv = t->inv; S.now_ms = clk->now_ms; S.want_misses = want_misses ? 1u : 0u;
  return 0;
}

// The miss records k_store_before filed (a grid of `blocks`), compacted into the library's page-locked miss list.
int store_misses(gub_table* t, unsigned blocks, uint32_t n, cudaStream_t st) {
  auto& ss = t->store;
  gub_store_rec* d_miss;
  uint32_t* d_count;
  if (device_view(ss.h_miss, &d_miss) || device_view(ss.h_count, &d_count)) return -1;
  gub::k_store_compact<<<blocks, gub::STORE_THREADS, 0, st>>>(ss.sel, ss.sparse, ss.blk, n, d_miss, d_count);
  CK(cudaGetLastError());
  CK(cudaEventRecord(ss.misses_done, st));
  return 0;
}

// Store.Get on the miss list (complete: store_misses' event has been waited for), then the host's verdict for what it returned:
// *nl loaded records (h_loaded), of which *ni items to install (h_items).
int store_get(gub_table* t, gub_store_get_fn get, void* user, const gub_clock* clk, const char* what, uint32_t* nl_out, uint32_t* ni_out) {
  auto& ss = t->store;
  *nl_out = 0; *ni_out = 0;
  const uint32_t m = *(volatile uint32_t*)ss.h_count;
  if (m == 0) return 0;
  // the callback may write the whole record; the keys and the request names (which the device indexes with) are the library's
  std::vector<gub_store_rec> named((size_t)m);
  std::memcpy(named.data(), ss.h_miss, (size_t)m * sizeof(gub_store_rec));
  const int rc = get(user, ss.h_miss, m);
  if (rc != 0) return fail(std::string(what) + ": the store's get callback failed (" + std::to_string(rc) + "); nothing was evaluated");
  uint32_t nl = 0, ni = 0;
  for (uint32_t k = 0; k < m; k++) {
    gub_store_rec& r = ss.h_miss[k];
    if (!(r.flags & GUB_STORE_FOUND)) continue;
    r.first = named[k].first; r.last = named[k].last; r.first_shard = named[k].first_shard; r.last_shard = named[k].last_shard;
    r.item.key_xxh64 = named[k].item.key_xxh64; r.item.key_fnv1 = named[k].item.key_fnv1;
    // the host layer's rule for a loaded item: it existed when it had not expired; the algorithm is the one the store returned.  The
    // record's first_shard (0 on a single table) lets a ring owner find the pass index again (k_store_loaded_ring).
    ss.h_loaded[nl++] = make_uint4(r.first, r.item.expire_at >= clk->now_ms ? gub::S_EXISTED : 0u, (uint32_t)r.item.algorithm, (uint32_t)r.first_shard);
    if (r.item.algorithm == GUB_TOKEN_BUCKET || r.item.algorithm == GUB_LEAKY_BUCKET) ss.h_items[ni++] = to_dev(r.item);  // as gub_add_items
  }
  *nl_out = nl; *ni_out = ni;
  return 0;
}

// What store_get returned, installed before the pass: what gub_add_items does (place the parked inserts, then upsert the items), then the
// verdicts.  segs: a ring owner's pass (the loaded records name their requests by source).
int store_install(gub_table* t, uint32_t nl, uint32_t ni, const gub::StoreSegs* segs, cudaStream_t st) {
  auto& ss = t->store;
  if (nl == 0) return 0;
  uint4* d_loaded;
  gub::DevItem* d_items;
  if (device_view(ss.h_loaded, &d_loaded) || device_view(ss.h_items, &d_items)) return -1;
  if (ni) {
    if (drain_pending(t, st)) return -1;
    CK(cudaMemsetAsync(ss.d_failed, 0, 4, st));
    gub::k_add_items<<<(ni + 255) / 256, 256, 0, st>>>(t->table, t->capacity, d_items, ni, t->counters, ss.d_failed, t->inv);
  }
  const unsigned blocks = (nl + gub::STORE_THREADS - 1) / gub::STORE_THREADS;
  if (segs) gub::k_store_loaded_ring<<<blocks, gub::STORE_THREADS, 0, st>>>(d_loaded, nl, ss.bstate, *segs);
  else gub::k_store_loaded<<<blocks, gub::STORE_THREADS, 0, st>>>(d_loaded, nl, ss.bstate);
  CK(cudaGetLastError());
  return 0;
}

// After store_install with ni > 0: fails when the table had no room for some of the items.
int store_install_check(gub_table* t, const char* what, cudaStream_t st) {
  uint32_t failed = 0;
  CK(cudaMemcpyAsync(&failed, t->store.d_failed, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (failed) return fail(std::string(what) + ": table full for " + std::to_string(failed) + " items the store returned");
  return 0;
}

// Before the batch (host layer: gub_get_items, Store.Get, gub_add_items): the per-key dedup, the lookup of every key at its first
// request and, with a Get callback, the miss list, the call and the installation of what the store returned.
int store_before(gub_table* t, const gub_req* d_req, uint32_t n, const gub_clock* clk, const StoreCall& sc, gub::StoreArgs& S, cudaStream_t st) {
  if (store_args(t, clk, sc.get != nullptr, S, st)) return -1;
  S.reqs = d_req; S.n = n;
  const unsigned blocks = (n + gub::STORE_THREADS - 1) / gub::STORE_THREADS;
  gub::k_store_keys<<<blocks, gub::STORE_THREADS, 0, st>>>(S);
  gub::k_store_before<<<blocks, gub::STORE_THREADS, 0, st>>>(S);
  CK(cudaGetLastError());
  t->last_stream = st; t->last_pending = true;
  if (!sc.get) return 0;
  if (store_misses(t, blocks, n, st)) return -1;
  CK(cudaEventSynchronize(t->store.misses_done));
  const char* what = "gub_submit_keys_store_async";
  uint32_t nl, ni;
  if (store_get(t, sc.get, sc.user, clk, what, &nl, &ni)) return -1;
  if (store_install(t, nl, ni, nullptr, st)) return -1;
  if (ni && store_install_check(t, what, st)) return -1;
  return 0;
}

// After the batch (host layer: the second gub_get_items, Store.Remove / Store.OnChange): the records, straight into the caller's buffers.
int store_after(gub_table* t, const gub_resp* d_out, const StoreCall& sc, gub::StoreArgs& S, cudaStream_t st) {
  S.out = d_out;
  const unsigned blocks = (S.n + gub::STORE_THREADS - 1) / gub::STORE_THREADS;
  gub::k_store_after<<<blocks, gub::STORE_THREADS, 0, st>>>(S);
  gub::k_store_compact<<<blocks, gub::STORE_THREADS, 0, st>>>(S.sel, S.sparse, S.blk, S.n, sc.changes, sc.n_changes);
  CK(cudaGetLastError());
  t->last_stream = st; t->last_pending = true;
  return 0;
}

// gub_submit_keys_async, and with `sc` the Store's pre- and post-pass around the batch.
int submit_keys(gub_table* t, const void* packed, size_t packed_bytes, size_t n, const gub_params* params, size_t n_params,
                int64_t created_base, const gub_clock* clk, gub_resp* out, int* ticket, const StoreCall* sc) {
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  const int si = t->next_slot;
  t->next_slot = (t->next_slot + 1) % PIPE_DEPTH;
  PipeSlot& s = t->pipe[si];
  if (s.busy) { CK(cudaEventSynchronize(s.out_done)); s.busy = false; }
  *ticket = si;
  if (n == 0) { CK(cudaEventRecord(s.out_done, t->s_d2h)); s.busy = true; return 0; }
  if (ensure_slot(s, n)) return -1;
  if (s.packed_cap < packed_bytes) {
    if (s.d_packed) cudaFree(s.d_packed);
    s.d_packed = nullptr;
    s.packed_cap = std::max<size_t>(packed_bytes + packed_bytes / 4, (size_t)1 << 20);
    CK(cudaMalloc(&s.d_packed, s.packed_cap));
  }
  const bool inl = n_params <= gub::INLINE_PARAMS;
  if (!inl && (s.params_cap < n_params || !s.d_params)) {
    if (s.d_params) cudaFree(s.d_params);
    s.d_params = nullptr;
    s.params_cap = std::max<size_t>(n_params, 1024);
    CK(cudaMalloc(&s.d_params, s.params_cap * sizeof(gub_params)));
  }
  CK(cudaMemcpyAsync(s.d_packed, packed, packed_bytes, cudaMemcpyHostToDevice, t->s_h2d));
  if (!inl) CK(cudaMemcpyAsync(s.d_params, params, n_params * sizeof(gub_params), cudaMemcpyHostToDevice, t->s_h2d));
  CK(cudaEventRecord(s.in_done, t->s_h2d));
  CK(cudaStreamWaitEvent(t->s_compute, s.in_done, 0));
  gub::InlineParams P;
  std::memset(&P, 0, sizeof P);
  if (inl) std::memcpy(&P, params, n_params * sizeof(gub_params));
  gub::k_hash_expand<<<(unsigned)((n + 255) / 256), 256, 0, t->s_compute>>>(s.d_packed, (uint32_t)n, P, (uint32_t)n_params, inl ? nullptr : s.d_params, created_base, s.d_req);
  gub::StoreArgs S;
  if (sc && store_before(t, s.d_req, (uint32_t)n, clk, *sc, S, t->s_compute)) return -1;
  if (launch_batch(t, s.d_req, n, clk, s.d_resp, t->s_compute)) return -1;
  if (sc && store_after(t, s.d_resp, *sc, S, t->s_compute)) return -1;
  CK(cudaEventRecord(t->compute_done[si], t->s_compute));
  CK(cudaStreamWaitEvent(t->s_d2h, t->compute_done[si], 0));
  CK(cudaMemcpyAsync(out, s.d_resp, n * sizeof(gub_resp), cudaMemcpyDeviceToHost, t->s_d2h));
  CK(cudaEventRecord(s.out_done, t->s_d2h));
  s.busy = true;
  return 0;
}

// The device address of page-locked host memory, or null when `p` is not page-locked.
template <typename T>
T* pinned_view(const T* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  return a.type == cudaMemoryTypeHost ? static_cast<T*>(a.devicePointer) : nullptr;
}

}  // namespace

extern "C" {

int gub_submit_keys_async(gub_table* t, const void* packed, size_t packed_bytes, size_t n, const gub_params* params, size_t n_params, int64_t created_base,
                          const gub_clock* clk, gub_resp* out, int* ticket) {
  if (!t || !clk || !ticket || (n && (!packed || !out || !params))) return fail("gub_submit_keys_async: null argument");
  if (n > 0x7FFFFFFFull || n_params > 0xFFFFFFFFull) return fail("gub_submit_keys_async: too large");
  if (n && packed_bytes < n * sizeof(gub_kreq) + (n + 1) * 4) return fail("gub_submit_keys_async: packed buffer too small");
  return submit_keys(t, packed, packed_bytes, n, params, n_params, created_base, clk, out, ticket, nullptr);
}

int gub_submit_keys_store_async(gub_table* t, const void* packed, size_t packed_bytes, size_t n, const gub_params* params, size_t n_params,
                                int64_t created_base, const gub_clock* clk, gub_store_get_fn get, void* user, gub_resp* out,
                                gub_store_rec* changes, uint32_t* n_changes, int* ticket) {
  static_assert(sizeof(gub_store_rec) == 104, "gub_store_rec is 16 bytes + a gub_item");
  if (!t || !clk || !ticket || !changes || !n_changes || (n && (!packed || !out || !params))) return fail("gub_submit_keys_store_async: null argument");
  if (n > t->max_batch) return fail("gub_submit_keys_store_async: n = " + std::to_string(n) + " exceeds max_batch = " + std::to_string(t->max_batch) +
                                    " (a key split over two chunks would get two records)");
  if (n_params > 0xFFFFFFFFull) return fail("gub_submit_keys_store_async: too large");
  if (n && packed_bytes < n * sizeof(gub_kreq) + (n + 1) * 4) return fail("gub_submit_keys_store_async: packed buffer too small");
  if (t->fused) return fail("gub_submit_keys_store_async: not available on a table created under GUB_PATH=fused");
  CK(cudaSetDevice(t->device));
  StoreCall sc;
  sc.get = get; sc.user = user; sc.changes = pinned_view(changes); sc.n_changes = pinned_view(n_changes);
  if (!sc.changes || !sc.n_changes) return fail("gub_submit_keys_store_async: changes and n_changes must be page-locked host memory (gub_host_alloc)");
  if (n == 0) *n_changes = 0;
  return submit_keys(t, packed, packed_bytes, n, params, n_params, created_base, clk, out, ticket, &sc);
}

int gub_proto_layout(size_t n_msgs, size_t msg_bytes, size_t* offsets_at, size_t* bytes_at, size_t* total, size_t* out_bound) {
  if (!offsets_at || !bytes_at || !total || !out_bound) return fail("gub_proto_layout: null argument");
  *offsets_at = n_msgs * 8;
  *bytes_at = *offsets_at + (n_msgs + 1) * 4;
  *total = (*bytes_at + msg_bytes + 15) & ~(size_t)15;
  *out_bound = (size_t)gub::PROTO_OUT_FACTOR * msg_bytes;
  return 0;
}

}  // extern "C"

namespace {
int proto_ensure(PipeSlot& s, const gub::ProtoPlan& P, size_t n_msgs) {
  auto& pr = s.proto;
  if (!pr.decoded) {
    CK(cudaEventCreateWithFlags(&pr.decoded, cudaEventDisableTiming));
    CK(cudaHostAlloc((void**)&pr.h_neval, 64, cudaHostAllocMapped));
  }
  if (pr.msgs_cap < n_msgs + 1) {
    const size_t c = std::max<size_t>(n_msgs + 1, 1024);
    uint32_t** u32s[] = {&pr.slot_base, &pr.batch_base, &pr.mcount, &pr.meval, &pr.mstatus, &pr.msize};
    for (uint32_t** a : u32s) { if (*a) cudaFree(*a); *a = nullptr; CK(cudaMalloc(a, c * 4)); }
    if (pr.moff) cudaFree(pr.moff);
    pr.moff = nullptr;
    CK(cudaMalloc(&pr.moff, c * 8));
    pr.msgs_cap = c;
  }
  if (pr.slots_cap < P.slots || !pr.items) {
    const size_t c = std::max<size_t>(P.slots + P.slots / 4, 1024);
    if (pr.items) cudaFree(pr.items);
    if (pr.sreq) cudaFree(pr.sreq);
    pr.items = nullptr; pr.sreq = nullptr;
    CK(cudaMalloc(&pr.items, c * sizeof(gub::ProtoItem)));
    CK(cudaMalloc(&pr.sreq, c * sizeof(gub_req)));
    pr.slots_cap = c;
  }
  if (pr.bytes_cap < P.msg_bytes || !pr.keys) {
    const size_t c = std::max<size_t>(P.msg_bytes + P.msg_bytes / 4, (size_t)1 << 16);
    if (pr.keys) cudaFree(pr.keys);
    if (pr.stage) cudaFree(pr.stage);
    pr.keys = nullptr; pr.stage = nullptr;
    CK(cudaMalloc(&pr.keys, c));
    CK(cudaMalloc(&pr.stage, c * gub::PROTO_OUT_FACTOR));
    pr.bytes_cap = c;
  }
  return 0;
}

// The decode half of a wire-bytes call on `st`, after the copy of the packed buffer into s.d_packed: slot bases, decoding, batch bases
// (the evaluable count to the mapped word) and the compaction into s.d_req; then the `decoded` event.  A.out*, A.force_global: the caller's.
int proto_decode(PipeSlot& s, const gub::ProtoPlan& P, size_t n_msgs, gub::ProtoArgs& A, cudaStream_t st) {
  auto& pr = s.proto;
  A.created = reinterpret_cast<const int64_t*>(s.d_packed);
  A.offs = reinterpret_cast<const uint32_t*>(s.d_packed + P.offsets_at);
  A.bytes = s.d_packed + P.bytes_at;
  A.n_msgs = (uint32_t)n_msgs;
  A.smem = P.smem;
  A.slot_base = pr.slot_base; A.batch_base = pr.batch_base; A.mcount = pr.mcount; A.meval = pr.meval; A.mstatus = pr.mstatus;
  A.msize = pr.msize; A.moff = pr.moff; A.items = pr.items; A.sreq = pr.sreq; A.keys = pr.keys; A.stage = pr.stage;
  A.reqs = s.d_req; A.resp = s.d_resp;
  if (device_view(pr.h_neval, &A.n_eval)) return -1;
  const unsigned grid = (unsigned)n_msgs;
  gub::k_proto_scan<<<1, gub::PROTO_SCAN_THREADS, 0, st>>>(A, 0u);
  gub::k_proto_decode<<<grid, gub::PROTO_THREADS, P.smem, st>>>(A);
  gub::k_proto_scan<<<1, gub::PROTO_SCAN_THREADS, 0, st>>>(A, 1u);
  gub::k_proto_compact<<<grid, gub::PROTO_THREADS, 0, st>>>(A);
  CK(cudaGetLastError());
  CK(cudaEventRecord(pr.decoded, st));
  return 0;
}

// The encode half on `st`, once the responses of the dense batch are in A.resp: every message's bytes, offsets and status into the
// caller's page-locked buffers.
int proto_encode(const gub::ProtoArgs& A, cudaStream_t st) {
  const unsigned grid = A.n_msgs;
  gub::k_proto_encode<<<grid, gub::PROTO_THREADS, 0, st>>>(A);
  gub::k_proto_scan<<<1, gub::PROTO_SCAN_THREADS, 0, st>>>(A, 2u);
  gub::k_proto_copy_out<<<grid, gub::PROTO_THREADS, 0, st>>>(A);
  CK(cudaGetLastError());
  return 0;
}
}  // namespace

extern "C" {

/* Wire bytes in, wire bytes out (see the header).  Decoding runs on s_proto, which waits only for this call's copy; the host then waits
 * for the decoded item count (a mapped word), so that the evaluation is sized for the items there are, and enqueues the evaluation and
 * the encoding on the compute stream. */
int gub_submit_proto_async(gub_table* t, const void* packed, size_t packed_bytes, size_t n_msgs, const gub_clock* clk, void* out_bytes,
                           size_t out_cap, uint64_t* out_off, uint32_t* msg_status, int* ticket) {
  const std::string what = "gub_submit_proto_async";
  if (!t || !clk || !ticket || !out_off || (n_msgs && (!packed || !out_bytes || !msg_status))) return fail(what + ": null argument");
  if (n_msgs > 0x7FFFFFFFull) return fail(what + ": too many messages");
  gub::ProtoPlan P;
  if (n_msgs) {
    if (const char* why = gub::proto_plan(static_cast<const uint8_t*>(packed), packed_bytes, n_msgs, out_cap, P)) return fail(what + ": " + why);
  }
  CK(cudaSetDevice(t->device));
  uint8_t* d_out = n_msgs ? pinned_view(static_cast<uint8_t*>(out_bytes)) : nullptr;
  unsigned long long* d_off = pinned_view(reinterpret_cast<unsigned long long*>(out_off));
  uint32_t* d_status = n_msgs ? pinned_view(msg_status) : nullptr;
  if (!d_off || (n_msgs && (!d_out || !d_status)))
    return fail(what + ": out_bytes, out_off and msg_status must be page-locked host memory (gub_host_alloc)");
  std::lock_guard<std::mutex> lk(t->mu);
  const int si = t->next_slot;
  t->next_slot = (t->next_slot + 1) % PIPE_DEPTH;
  PipeSlot& s = t->pipe[si];
  if (s.busy) { CK(cudaEventSynchronize(s.out_done)); s.busy = false; }
  *ticket = si;
  if (n_msgs == 0) { out_off[0] = 0; CK(cudaEventRecord(s.out_done, t->s_compute)); s.busy = true; return 0; }
  if (!t->s_proto) {
    CK(cudaStreamCreateWithFlags(&t->s_proto, cudaStreamNonBlocking));
    CK(cudaFuncSetAttribute(gub::k_proto_decode, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gub::PROTO_SMEM));
  }
  if (ensure_slot(s, std::max<size_t>(P.slots, 1)) || proto_ensure(s, P, n_msgs)) return -1;
  if (s.packed_cap < packed_bytes) {
    if (s.d_packed) cudaFree(s.d_packed);
    s.d_packed = nullptr;
    s.packed_cap = std::max<size_t>(packed_bytes + packed_bytes / 4, (size_t)1 << 20);
    CK(cudaMalloc(&s.d_packed, s.packed_cap));
  }
  auto& pr = s.proto;
  CK(cudaMemcpyAsync(s.d_packed, packed, P.bytes_at + P.msg_bytes, cudaMemcpyHostToDevice, t->s_h2d));
  CK(cudaEventRecord(s.in_done, t->s_h2d));
  CK(cudaStreamWaitEvent(t->s_proto, s.in_done, 0));
  gub::ProtoArgs A;
  std::memset(&A, 0, sizeof A);
  A.out = d_out; A.out_off = d_off; A.out_status = d_status;
  if (proto_decode(s, P, n_msgs, A, t->s_proto)) return -1;
  CK(cudaEventSynchronize(pr.decoded));
  const uint32_t n_eval = *(volatile uint32_t*)pr.h_neval;
  CK(cudaStreamWaitEvent(t->s_compute, pr.decoded, 0));
  if (n_eval && launch_batch(t, s.d_req, n_eval, clk, s.d_resp, t->s_compute)) return -1;
  if (proto_encode(A, t->s_compute)) return -1;
  CK(cudaEventRecord(s.out_done, t->s_compute));
  s.busy = true;
  return 0;
}

int gub_wait(gub_table* t, int ticket) {
  if (!t || ticket < 0 || ticket >= PIPE_DEPTH) return fail("gub_wait: bad ticket");
  cudaEvent_t ev;
  {
    std::lock_guard<std::mutex> lk(t->mu);
    if (!t->pipe[ticket].busy) return 0;
    ev = t->pipe[ticket].out_done;
  }
  CK(cudaSetDevice(t->device));
  CK(cudaEventSynchronize(ev));
  std::lock_guard<std::mutex> lk(t->mu);
  t->pipe[ticket].busy = false;
  return 0;
}

int gub_submit_compact(gub_table* t, const gub_creq* reqs, size_t n, const gub_params* params, size_t n_params, int64_t created_base,
                       const gub_clock* clk, gub_resp* out) {
  int ticket = -1;
  if (gub_submit_compact_async(t, reqs, n, params, n_params, created_base, clk, out, &ticket)) return -1;
  return gub_wait(t, ticket);
}

int gub_submit(gub_table* t, const gub_req* reqs, size_t n, const gub_clock* clk, gub_resp* out) {
  int ticket = -1;
  if (gub_submit_async(t, reqs, n, clk, out, &ticket)) return -1;
  return gub_wait(t, ticket);
}

void* gub_host_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) { g_err = "cudaHostAlloc failed"; return nullptr; }
  return p;
}
void gub_host_free(void* p) { if (p) cudaFreeHost(p); }

namespace {
// Items parked by a batch whose probe window was full are placed before anything else reads or writes the table.
int drain_pending(gub_table* t, cudaStream_t st) {
  gub_clock clk;
  std::memset(&clk, 0, sizeof clk);
  clk.now_ms = INT64_MIN;  // nothing counts as expired here: only free, removed and then the earliest-expiring entries give way
  gub::FArgs A;
  fused_base_args(t, &clk, A);
  gub::k_drain_overflow<<<1, 32, 0, st>>>(A);
  CK(cudaGetLastError());
  return 0;
}
}  // namespace

int gub_add_items(gub_table* t, const gub_item* items, size_t n) {
  if (!t || (n && !items)) return fail("gub_add_items: null argument");
  if (n == 0) return 0;
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  // last one wins for duplicate keys (sequential AddCacheItem calls would overwrite in order)
  std::vector<gub::DevItem> dev;
  dev.reserve(n);
  std::unordered_map<uint64_t, size_t> seen;
  seen.reserve(n * 2);
  for (size_t i = 0; i < n; i++) {
    if (items[i].algorithm != GUB_TOKEN_BUCKET && items[i].algorithm != GUB_LEAKY_BUCKET) continue;  // Value would be nil (gubernator.go:434-451)
    gub::DevItem d = to_dev(items[i]);
    const uint64_t h = d.key ^ (d.tag * 0x9E3779B97F4A7C15ULL);
    auto it = seen.find(h);
    if (it != seen.end() && dev[it->second].key == d.key && dev[it->second].tag == d.tag) dev[it->second] = d;
    else { seen[h] = dev.size(); dev.push_back(d); }
  }
  if (dev.empty()) return 0;
  CK(cudaDeviceSynchronize());
  if (drain_pending(t)) return -1;
  gub::DevItem* d_items = nullptr;
  CK(cudaMalloc(&d_items, dev.size() * sizeof(gub::DevItem)));
  cudaError_t e = cudaMemcpy(d_items, dev.data(), dev.size() * sizeof(gub::DevItem), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemset(t->d_scalar, 0, 8);
  uint32_t failed = 0;
  if (e == cudaSuccess) {
    gub::k_add_items<<<(unsigned)((dev.size() + 255) / 256), 256>>>(t->table, t->capacity, d_items, (uint32_t)dev.size(), t->counters,
                                                                    reinterpret_cast<uint32_t*>(t->d_scalar), t->inv);
    e = cudaDeviceSynchronize();
  }
  if (e == cudaSuccess) e = cudaMemcpy(&failed, t->d_scalar, 4, cudaMemcpyDeviceToHost);
  cudaFree(d_items);
  if (e != cudaSuccess) return fail(std::string("gub_add_items: ") + cudaGetErrorString(e));
  if (failed) return fail("gub_add_items: table full for " + std::to_string(failed) + " items");
  return 0;
}

int gub_get_items(gub_table* t, const uint64_t* kx, const uint64_t* kf, size_t n, int64_t now_ms, gub_item* out, uint8_t* found) {
  if (!t || (n && (!kx || !kf || !out || !found))) return fail("gub_get_items: null argument");
  if (n == 0) return 0;
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  CK(cudaDeviceSynchronize());
  if (drain_pending(t)) return -1;
  uint64_t *d_kx = nullptr, *d_kf = nullptr; gub::DevItem* d_out = nullptr; uint8_t* d_found = nullptr;
  std::vector<gub::DevItem> host(n);
  cudaError_t e = cudaMalloc(&d_kx, n * 8);
  if (e == cudaSuccess) e = cudaMalloc(&d_kf, n * 8);
  if (e == cudaSuccess) e = cudaMalloc(&d_out, n * sizeof(gub::DevItem));
  if (e == cudaSuccess) e = cudaMalloc(&d_found, n);
  if (e == cudaSuccess) e = cudaMemcpy(d_kx, kx, n * 8, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(d_kf, kf, n * 8, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) {
    gub::k_get_items<<<(unsigned)((n + 255) / 256), 256>>>(t->table, t->capacity, d_kx, d_kf, (uint32_t)n, now_ms, d_out, d_found, t->inv);
    e = cudaDeviceSynchronize();
  }
  if (e == cudaSuccess) e = cudaMemcpy(host.data(), d_out, n * sizeof(gub::DevItem), cudaMemcpyDeviceToHost);
  if (e == cudaSuccess) e = cudaMemcpy(found, d_found, n, cudaMemcpyDeviceToHost);
  cudaFree(d_kx); cudaFree(d_kf); cudaFree(d_out); cudaFree(d_found);
  if (e != cudaSuccess) return fail(std::string("gub_get_items: ") + cudaGetErrorString(e));
  for (size_t i = 0; i < n; i++) { out[i] = from_dev(host[i]); out[i].key_xxh64 = kx[i]; out[i].key_fnv1 = kf[i]; }
  return 0;
}

int gub_scan(gub_table* t, gub_item* out, size_t cap, size_t* n_out) {
  if (!t || !n_out || (cap && !out)) return fail("gub_scan: null argument");
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  CK(cudaDeviceSynchronize());
  if (drain_pending(t)) return -1;
  gub::DevItem* d_out = nullptr;
  if (cap) CK(cudaMalloc(&d_out, cap * sizeof(gub::DevItem)));
  unsigned long long total = 0;
  cudaError_t e = cudaMemset(t->d_scalar, 0, 8);
  if (e == cudaSuccess) {
    gub::k_scan<<<t->num_sms * 8, 256>>>(t->table, t->capacity, d_out, (unsigned long long)cap, t->d_scalar, t->inv);
    e = cudaDeviceSynchronize();
  }
  if (e == cudaSuccess) e = cudaMemcpy(&total, t->d_scalar, 8, cudaMemcpyDeviceToHost);
  std::vector<gub::DevItem> host(std::min<size_t>(cap, (size_t)total));
  if (e == cudaSuccess && !host.empty()) e = cudaMemcpy(host.data(), d_out, host.size() * sizeof(gub::DevItem), cudaMemcpyDeviceToHost);
  if (d_out) cudaFree(d_out);
  if (e != cudaSuccess) return fail(std::string("gub_scan: ") + cudaGetErrorString(e));
  for (size_t i = 0; i < host.size(); i++) out[i] = from_dev(host[i]);
  *n_out = (size_t)total;
  return 0;
}

int gub_size(gub_table* t, size_t* n_out) { return gub_scan(t, nullptr, 0, n_out); }

int gub_sweep(gub_table* t, int64_t now_ms, size_t* removed) {
  if (!t) return fail("gub_sweep: null argument");
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  CK(cudaDeviceSynchronize());
  CK(cudaMemset(t->d_scalar, 0, 8));
  gub::k_sweep<<<t->num_sms * 8, 256>>>(t->table, (uint64_t)0, t->capacity, now_ms, t->d_scalar);
  CK(cudaDeviceSynchronize());
  unsigned long long r = 0;
  CK(cudaMemcpy(&r, t->d_scalar, 8, cudaMemcpyDeviceToHost));
  if (removed) *removed = (size_t)r;
  return 0;
}

int gub_get_counters(gub_table* t, gub_counters* out) {
  if (!t || !out) return fail("gub_get_counters: null argument");
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  CK(cudaDeviceSynchronize());
  unsigned long long c[gub::C_COUNT];
  CK(cudaMemcpy(c, t->counters, sizeof c, cudaMemcpyDeviceToHost));
  out->over_limit = c[gub::C_OVER]; out->cache_hit = c[gub::C_HIT]; out->cache_miss = c[gub::C_MISS];
  out->inserts = c[gub::C_INSERTS]; out->table_full = c[gub::C_FULL]; out->requests = c[gub::C_REQUESTS];
  out->batches = c[gub::C_BATCHES]; out->dup_groups = c[gub::C_DUP_GROUPS]; out->mixed_groups = c[gub::C_MIXED_GROUPS];
  out->serial_fallbacks = c[gub::C_SERIAL];
  out->unexpired_evictions = c[gub::C_EVICT_UNEXPIRED]; out->swept = c[gub::C_SWEPT]; out->gq_dropped = c[gub::C_GQ_DROPPED];
  return 0;
}

int gub_hash_keys_device(gub_table* t, const char* d_bytes, const uint64_t* d_offsets, size_t n, uint64_t* d_xxh64_out, uint64_t* d_fnv1_out,
                         gub_req* d_reqs_out, void* stream) {
  if (!t || (n && (!d_bytes || !d_offsets))) return fail("gub_hash_keys_device: null argument");
  if (n == 0) return 0;
  CK(cudaSetDevice(t->device));
  gub::k_hash_keys<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const uint8_t*>(d_bytes), d_offsets, (uint32_t)n,
                                                                                 d_xxh64_out, d_fnv1_out, d_reqs_out);
  CK(cudaGetLastError());
  return 0;
}

/* Incremental expiry sweep inside the batch kernel: every CTA frees the removed / expired entries of `slots_per_cta` slots per batch
 * (0 = off).  The default visits the whole table once every ~65536 batches. */
int gub_set_sweep(gub_table* t, uint32_t slots_per_cta) {
  if (!t) return fail("gub_set_sweep: null argument");
  std::lock_guard<std::mutex> lk(t->mu);
  t->sweep_chunk = std::min<uint32_t>(slots_per_cta, 1024u);
  return 0;
}

/* Diagnostic: per-CTA %globaltimer stamps at the phase boundaries of k_batch.  gub_get_trace reports, for the LAST launch, the
 * time (us since the earliest CTA entered the kernel) at which the last CTA passed each of the 12 marks, and the mean over CTAs. */
int gub_set_trace(gub_table* t, int on) {
  if (!t) return fail("gub_set_trace: null argument");
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  CK(cudaDeviceSynchronize());
  if (on && !t->trace) {
    CK(cudaMalloc(&t->trace, (size_t)gub::FB_MAX_GRID * gub::FB_TRACE_MARKS * 8));
    CK(cudaMemset(t->trace, 0, (size_t)gub::FB_MAX_GRID * gub::FB_TRACE_MARKS * 8));
    CK(cudaMalloc(&t->ktrace, (size_t)4 * gub::KT_BLOCKS * gub::KT_MARKS * 8));
    CK(cudaMemset(t->ktrace, 0, (size_t)4 * gub::KT_BLOCKS * gub::KT_MARKS * 8));
  } else if (!on && t->trace) {
    cudaFree(t->trace);
    t->trace = nullptr;
    if (t->ktrace) cudaFree(t->ktrace);
    t->ktrace = nullptr;
  }
  return 0;
}

/* Diagnostic: the pipeline kernels' time stamps since the last reset: out[(kernel * 1024 + block) * 8 + mark] = latest %globaltimer
 * (ns) at which a warp of the block — or, for the role marks, a thread in that role — passed the mark; 0 = never.  kernel:
 * 0 k_group, 1 k_rank, 2 k_eval, 3 k_finish. */
int gub_get_ktrace(gub_table* t, uint64_t* out /* 4 x 1024 x 8 */, int reset) {
  if (!t || !out) return fail("gub_get_ktrace: null argument");
  std::lock_guard<std::mutex> lk(t->mu);
  if (!t->ktrace) return fail("gub_get_ktrace: tracing is off");
  CK(cudaSetDevice(t->device));
  CK(cudaDeviceSynchronize());
  const size_t bytes = (size_t)4 * gub::KT_BLOCKS * gub::KT_MARKS * 8;
  CK(cudaMemcpy(out, t->ktrace, bytes, cudaMemcpyDeviceToHost));
  if (reset) CK(cudaMemset(t->ktrace, 0, bytes));
  return 0;
}
int gub_get_trace(gub_table* t, double* max_us /* 12 */, double* mean_us /* 12 */) {
  if (!t || !max_us || !mean_us) return fail("gub_get_trace: null argument");
  std::lock_guard<std::mutex> lk(t->mu);
  if (!t->trace) return fail("gub_get_trace: tracing is off");
  CK(cudaSetDevice(t->device));
  CK(cudaDeviceSynchronize());
  std::vector<unsigned long long> h((size_t)gub::FB_MAX_GRID * gub::FB_TRACE_MARKS);
  CK(cudaMemcpy(h.data(), t->trace, h.size() * 8, cudaMemcpyDeviceToHost));
  unsigned long long t0 = ~0ull;
  int ctas = 0;
  for (int b = 0; b < gub::FB_MAX_GRID; b++) if (h[(size_t)b * gub::FB_TRACE_MARKS]) { t0 = std::min(t0, h[(size_t)b * gub::FB_TRACE_MARKS]); ctas++; }
  for (int k = 0; k < gub::FB_TRACE_MARKS; k++) {
    double mx = 0, sum = 0;
    for (int b = 0; b < gub::FB_MAX_GRID; b++) {
      const unsigned long long v = h[(size_t)b * gub::FB_TRACE_MARKS + k];
      if (!h[(size_t)b * gub::FB_TRACE_MARKS] || v < t0) continue;
      const double us = (double)(v - t0) * 1e-3;
      mx = std::max(mx, us); sum += us;
    }
    max_us[k] = mx; mean_us[k] = ctas ? sum / ctas : 0;
  }
  return 0;
}

/* Raw stamps of the last launch: out[cta * 12 + mark] in ns (0 = CTA not launched). */
int gub_get_trace_raw(gub_table* t, uint64_t* out /* 256 x 12 */) {
  if (!t || !out) return fail("gub_get_trace_raw: null argument");
  std::lock_guard<std::mutex> lk(t->mu);
  if (!t->trace) return fail("gub_get_trace_raw: tracing is off");
  CK(cudaSetDevice(t->device));
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(out, t->trace, (size_t)gub::FB_MAX_GRID * gub::FB_TRACE_MARKS * 8, cudaMemcpyDeviceToHost));
  return 0;
}

int gub_set_profiling(gub_table* t, int on) {
  if (!t) return fail("gub_set_profiling: null argument");
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  if (prof_flush(t, true)) return -1;
  t->prof = on != 0;
  return 0;
}

int gub_get_profile(gub_table* t, double kernel_ms[4], uint64_t* launches, int reset) {
  if (!t || !kernel_ms || !launches) return fail("gub_get_profile: null argument");
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  if (prof_flush(t, true)) return -1;
  for (int k = 0; k < 4; k++) kernel_ms[k] = t->prof_ms[k];
  *launches = t->prof_launches;
  if (reset) { for (int k = 0; k < 4; k++) t->prof_ms[k] = 0; t->prof_launches = 0; }
  return 0;
}

// Measures the random 64-byte read-modify-write rate of this device over the table itself (contents unchanged): the
// "HBM random access" ceiling the batch path is compared with.  accesses are spread over all slots; returns GB/s moved
// (64 B read + 64 B written per access) in *gbs.
int gub_probe_random_access(gub_table* t, uint64_t accesses, double* gbs) {
  if (!t || !gbs || accesses == 0) return fail("gub_probe_random_access: bad argument");
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  CK(cudaDeviceSynchronize());
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  const uint64_t zero = (uint64_t)(getenv("GUB_PROBE_NONZERO") != nullptr);  // always 0 in practice; opaque to the compiler
  gub::k_random_rmw<<<t->num_sms * 16, 256>>>(t->table, t->capacity, accesses / 8 + 1, 1, zero);  // warm-up
  CK(cudaEventRecord(e0, 0));
  gub::k_random_rmw<<<t->num_sms * 16, 256>>>(t->table, t->capacity, accesses, 12345, zero);
  CK(cudaEventRecord(e1, 0));
  CK(cudaEventSynchronize(e1));
  float ms = 0;
  CK(cudaEventElapsedTime(&ms, e0, e1));
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  CK(cudaGetLastError());
  *gbs = ms > 0 ? (double)accesses * 128.0 / (ms * 1e-3) * 1e-9 : 0.0;
  return 0;
}

// ---- multi-GPU routing ----------------------------------------------------------------------------------------
static int ensure_ring(gub_table* t, const gub_ring* ring) {
  const uint64_t ver = gub_ring_version_(ring);
  if (t->ring_cached == ring && t->ring_version == ver && t->d_ring_pts) return 0;
  const size_t npts = gub_ring_points(ring, nullptr, nullptr, 0);
  if (npts == 0) return fail("gub_route_device: ring is empty");
  if (gub_ring_size(ring) > gub::MAX_SHARDS) return fail("gub_route_device: at most 16 shards");
  std::vector<uint64_t> hs(npts); std::vector<int32_t> ps(npts);
  gub_ring_points(ring, hs.data(), ps.data(), npts);
  CK(cudaDeviceSynchronize());
  if (t->d_ring_pts) cudaFree(t->d_ring_pts);
  if (t->d_ring_peers) cudaFree(t->d_ring_peers);
  t->d_ring_pts = nullptr; t->d_ring_peers = nullptr;
  CK(cudaMalloc(&t->d_ring_pts, npts * 8));
  CK(cudaMalloc(&t->d_ring_peers, npts * 4));
  CK(cudaMemcpy(t->d_ring_pts, hs.data(), npts * 8, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(t->d_ring_peers, ps.data(), npts * 4, cudaMemcpyHostToDevice));
  {  // direct-mapped entry into the sorted points by the hash's top 16 bits: first point >= (bucket << 48)
    if (npts > 0xFFFFu) return fail("gub_route_device: ring has too many points");
    std::vector<uint16_t> lut(65536);
    size_t k = 0;
    for (uint32_t b = 0; b < 65536; b++) {
      const uint64_t lo = (uint64_t)b << 48;
      while (k < npts && hs[k] < lo) k++;
      lut[b] = (uint16_t)k;
    }
    if (t->d_ring_lut) cudaFree(t->d_ring_lut);
    t->d_ring_lut = nullptr;
    CK(cudaMalloc(&t->d_ring_lut, 65536 * 2));
    CK(cudaMemcpy(t->d_ring_lut, lut.data(), 65536 * 2, cudaMemcpyHostToDevice));
  }
  t->ring_npts = (uint32_t)npts; t->ring_cached = ring; t->ring_version = ver;
  return 0;
}

static int route_impl(gub_table* t, const gub_ring* ring, int32_t self, const gub_req* d_reqs, size_t n, gub_req* d_out_reqs, uint32_t* d_perm,
                      uint32_t* d_counts, uint8_t* d_true_owner, void* stream) {
  if (!t || !ring || !d_counts || (n && (!d_reqs || !d_out_reqs || !d_perm))) return fail("gub_route_device: null argument");
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  if (ensure_ring(t, ring)) return -1;
  const uint32_t nshards = (uint32_t)gub_ring_size(ring);
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) { CK(cudaMemsetAsync(d_counts, 0, nshards * 4, st)); return 0; }
  if (n > 0x7FFFFFFFull) return fail("gub_route_device: batch too large");
  const uint32_t ntiles = (uint32_t)((n + gub::ROUTE_TILE - 1) / gub::ROUTE_TILE);
  if (!t->d_owner || t->owner_cap < n) { if (t->d_owner) { CK(cudaDeviceSynchronize()); cudaFree(t->d_owner); } CK(cudaMalloc(&t->d_owner, n)); t->owner_cap = n; }
  const size_t tc = (size_t)ntiles * gub::MAX_SHARDS;
  if (!t->d_tile_counts || t->tiles_cap < tc) { if (t->d_tile_counts) { CK(cudaDeviceSynchronize()); cudaFree(t->d_tile_counts); } CK(cudaMalloc(&t->d_tile_counts, tc * 4)); t->tiles_cap = tc; }
  gub::k_route_count<<<ntiles, 256, 0, st>>>(d_reqs, (uint32_t)n, t->d_ring_pts, t->d_ring_peers, t->ring_npts, nshards, t->d_owner,
                                            t->d_tile_counts, ntiles, self, d_true_owner);
  gub::k_route_scan<<<1, 1024, 0, st>>>(t->d_tile_counts, nshards * ntiles, nshards, ntiles, d_counts);
  gub::k_route_scatter<<<ntiles, 256, 0, st>>>(d_reqs, (uint32_t)n, t->d_owner, t->d_tile_counts, ntiles, nshards, d_out_reqs, d_perm);
  CK(cudaGetLastError());
  return 0;
}

int gub_route_device(gub_table* t, const gub_ring* ring, const gub_req* d_reqs, size_t n, gub_req* d_out_reqs, uint32_t* d_perm,
                     uint32_t* d_counts, void* stream) {
  return route_impl(t, ring, -1, d_reqs, n, d_out_reqs, d_perm, d_counts, nullptr, stream);
}

int gub_route_global_device(gub_table* t, const gub_ring* ring, uint32_t self, const gub_req* d_reqs, size_t n, gub_req* d_out_reqs,
                            uint32_t* d_perm, uint32_t* d_counts, uint8_t* d_owner_out, void* stream) {
  if (ring && self >= (uint32_t)gub_ring_size(ring)) return fail("gub_route_global_device: self is not a shard of the ring");
  return route_impl(t, ring, (int32_t)self, d_reqs, n, d_out_reqs, d_perm, d_counts, d_owner_out, stream);
}

__global__ void k_owner_only(const gub_req* reqs, uint32_t n, const uint64_t* pts, const int32_t* peers, uint32_t npts, uint8_t* owner) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) owner[i] = (uint8_t)gub::ring_owner(pts, peers, npts, __ldg(&reqs[i].key_fnv1));
}

int gub_route_owner_device(gub_table* t, const gub_ring* ring, const gub_req* d_reqs, size_t n, uint8_t* d_owner, void* stream) {
  if (!t || !ring || (n && (!d_reqs || !d_owner))) return fail("gub_route_owner_device: null argument");
  if (n == 0) return 0;
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  if (ensure_ring(t, ring)) return -1;
  k_owner_only<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(d_reqs, (uint32_t)n, t->d_ring_pts, t->d_ring_peers, t->ring_npts, d_owner);
  CK(cudaGetLastError());
  return 0;
}

// ---- GLOBAL behaviour: device queues ---------------------------------------------------------------------------
}  // extern "C"

struct gub_gq {
  int device = 0;
  int num_sms = 0;                    // grid of the drain kernel
  gub::Gq q{};
  uint32_t* slot_of = nullptr;
  size_t slot_cap = 0;
};

namespace {
int gq_reserve(gub_gq* g, size_t n, cudaStream_t st) {
  if (g->slot_cap >= n) return 0;
  CK(cudaStreamSynchronize(st));
  if (g->slot_of) cudaFree(g->slot_of);
  g->slot_of = nullptr;
  CK(cudaMalloc(&g->slot_of, n * 4));
  g->slot_cap = n;
  return 0;
}
// n_dev (optional): the batch size lives on the device (<= n)
int gq_accumulate(gub_gq* g, const gub_req* d_reqs, size_t n, const uint32_t* n_dev, const uint8_t* d_owner, uint32_t self, uint64_t seq_base, cudaStream_t st) {
  if (n == 0) return 0;
  if (gq_reserve(g, n, st)) return -1;
  const unsigned blocks = (unsigned)((n + 255) / 256);
  gub::k_gq_claim<<<blocks, 256, 0, st>>>(g->q, d_reqs, (uint32_t)n, n_dev, d_owner, self, d_owner ? 1u : 0u, (unsigned long long)seq_base, g->slot_of);
  gub::k_gq_fill<<<blocks, 256, 0, st>>>(g->q, d_reqs, (uint32_t)n, n_dev, (unsigned long long)seq_base, g->slot_of);
  CK(cudaGetLastError());
  return 0;
}
}  // namespace

extern "C" {

int gub_gq_create(int device, uint32_t capacity, int keep_latest, gub_gq** out) {
  if (!out || capacity < 64) return fail("gub_gq_create: bad argument");
  CK(cudaSetDevice(device));
  gub_gq* g = new gub_gq();
  g->device = device;
  cudaError_t e = cudaDeviceGetAttribute(&g->num_sms, cudaDevAttrMultiProcessorCount, device);
  const uint32_t cap = next_pow2(capacity);
  g->q.capacity_mask = cap - 1;
  g->q.mode = keep_latest ? gub::GQ_KEEP_LAST : gub::GQ_KEEP_FIRST;
  if (e == cudaSuccess) e = cudaMalloc(&g->q.slots, (size_t)cap * sizeof(gub_req));
  if (e == cudaSuccess) e = cudaMalloc(&g->q.seq, (size_t)cap * 8);
  if (e == cudaSuccess) e = cudaMalloc(&g->q.count, 16);
  if (e == cudaSuccess) e = cudaMemset(g->q.count, 0, 16);
  if (e == cudaSuccess) g->q.dropped = g->q.count + 1;
  if (e == cudaSuccess) e = cudaMemset(g->q.slots, 0, (size_t)cap * sizeof(gub_req));
  if (e == cudaSuccess) e = cudaMemset(g->q.seq, 0, (size_t)cap * 8);
  if (e == cudaSuccess) e = cudaMemset(g->q.count, 0, 8);
  if (e != cudaSuccess) { gub_gq_destroy(g); return fail(std::string("gub_gq_create: ") + cudaGetErrorString(e)); }
  *out = g;
  return 0;
}

void gub_gq_destroy(gub_gq* g) {
  if (!g) return;
  cudaSetDevice(g->device);
  cudaDeviceSynchronize();
  if (g->q.slots) cudaFree(g->q.slots);
  if (g->q.seq) cudaFree(g->q.seq);
  if (g->q.count) cudaFree(g->q.count);
  if (g->slot_of) cudaFree(g->slot_of);
  delete g;
}

int gub_gq_accumulate_device(gub_gq* g, const gub_req* d_reqs, size_t n, const uint8_t* d_owner, uint32_t self, uint64_t seq_base, void* stream) {
  if (!g || (n && !d_reqs)) return fail("gub_gq_accumulate_device: null argument");
  if (n == 0) return 0;
  CK(cudaSetDevice(g->device));
  return gq_accumulate(g, d_reqs, n, nullptr, d_owner, self, seq_base, (cudaStream_t)stream);
}

int gub_gq_dropped(gub_gq* g, uint64_t* dropped) {
  if (!g || !dropped) return fail("gub_gq_dropped: null argument");
  CK(cudaSetDevice(g->device));
  unsigned long long v = 0;
  CK(cudaMemcpy(&v, g->q.dropped, 8, cudaMemcpyDeviceToHost));
  *dropped = v;
  return 0;
}

int gub_gq_drain_device(gub_gq* g, gub_req* d_out, size_t cap, uint32_t* d_count, int as_status_query, void* stream) {
  if (!g || !d_count || (cap && !d_out)) return fail("gub_gq_drain_device: null argument");
  CK(cudaSetDevice(g->device));
  cudaStream_t st = (cudaStream_t)stream;
  CK(cudaMemsetAsync(d_count, 0, 4, st));
  gub::k_gq_drain<<<g->num_sms, 256, 0, st>>>(g->q, d_out, (uint32_t)std::min<size_t>(cap, 0xFFFFFFFFu), d_count, as_status_query ? 1u : 0u);
  CK(cudaGetLastError());
  return 0;
}

int gub_make_updates_device(gub_table* t, const gub_req* d_queries, const gub_resp* d_resps, size_t n, gub_item* d_items, uint32_t* d_count,
                            void* stream) {
  if (!t || !d_count || (n && (!d_queries || !d_resps || !d_items))) return fail("gub_make_updates_device: null argument");
  CK(cudaSetDevice(t->device));
  cudaStream_t st = (cudaStream_t)stream;
  CK(cudaMemsetAsync(d_count, 0, 4, st));
  if (n == 0) return 0;
  gub::k_make_updates<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_queries, d_resps, (uint32_t)n, nullptr, d_items, d_count);
  CK(cudaGetLastError());
  return 0;
}

int gub_add_items_device(gub_table* t, const gub_item* d_items, size_t n, int64_t now_ms, void* stream) {
  if (!t || (n && !d_items)) return fail("gub_add_items_device: null argument");
  if (n == 0) return 0;
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  cudaStream_t st = (cudaStream_t)stream;
  if (order_after_last(t, st)) return -1;
  gub::k_add_items_pub<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(t->table, t->capacity, d_items, (uint32_t)n, now_ms, t->counters, t->inv);
  CK(cudaGetLastError());
  t->last_stream = st; t->last_pending = true;
  return 0;
}

int gub_unroute_device(gub_table* t, const gub_resp* d_resp_in, const uint32_t* d_perm, size_t n, gub_resp* d_resp_out, void* stream) {
  if (!t || (n && (!d_resp_in || !d_perm || !d_resp_out))) return fail("gub_unroute_device: null argument");
  if (n == 0) return 0;
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  gub::k_unroute<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(d_resp_in, d_perm, (uint32_t)n, d_resp_out);
  CK(cudaGetLastError());
  return 0;
}


// ---- fused routing over peer memory -----------------------------------------------------------------------------
}  // extern "C"

extern "C" void gub_nccl_comm_destroy_(void* comm);
struct gub_p2p;
namespace {
int gq_accumulate_segments(gub_p2p* p, const gub::P2PArgs& A, cudaStream_t st);
}

struct gub_p2p {
  gub_table* t = nullptr;
  const gub_ring* ring = nullptr;
  uint32_t world = 0, rank = 0, cap = 0, epoch = 0;
  void* block = nullptr;           // our peer-visible allocation
  size_t block_bytes = 0;
  gub::P2PView views[gub::MAX_SHARDS];
  void* opened[gub::MAX_SHARDS] = {};
  bool connected = false;
  uint32_t* error = nullptr;       // device flag: a bounded wait gave up (a peer died)
  uint32_t* ticket = nullptr;      // [2] tile ticket / tiles done of the routing kernel
  // gub_p2p_step_streams: evaluation and collect run on streams of our own, so that neither the caller's stream nor the next step's
  // evaluation ever queues behind a wait for the slowest peer
  cudaStream_t s_eval = nullptr, s_collect = nullptr;
  cudaEvent_t ev_fork = nullptr;   // scratch event for one-off stream-to-stream ordering
  cudaStream_t last_ingest = nullptr;
  bool own_streams_used = false;
  uint32_t* seg_off = nullptr;     // [MAX_SHARDS + 1] prefix sums of this step's mailbox segments (k_seg_wait -> the batch kernels)
  // Routing scratch, preallocated (nothing is allocated or freed inside a step) and double-buffered by step parity: with a
  // separate ingest stream the routing of step e+1 runs while step e is still being evaluated and collected.
  struct Route {
    unsigned long long* tile_agg = nullptr;  // [(cap / RT_THREADS + 1) * MAX_SHARDS]
    uint32_t* counts = nullptr;    // [MAX_SHARDS]
    uint32_t* perm = nullptr;      // [cap]
    uint8_t* true_owner = nullptr; // [cap] (GLOBAL mode)
    gub_req* expanded = nullptr;   // [cap] (GLOBAL mode) key-string steps: the expanded records, read by the hits queue
    gub_params* params = nullptr;  // key-string steps with more than INLINE_PARAMS parameter sets: the table, grown on demand
    size_t params_cap = 0;
    cudaEvent_t routed = nullptr;     // this parity's routing has been issued (ingest stream)
    cudaEvent_t step_done = nullptr;  // this parity's collect has completed (evaluation stream)
    bool step_done_valid = false;
  } rt[2];
  // GLOBAL behaviour (gub_p2p_enable_global): device queues + tick buffers
  gub_gq *hits_q = nullptr, *updates_q = nullptr;
  uint32_t gq_recs = 0;            // next_pow2(capacity): the queues' size, and the most records / items one tick handles
  uint32_t gcap = 0;               // min(gq_recs, cap): the items one NCCL all-gather slice carries per rank
  // g_reqs: the hit records in round order, then the status queries; g_items: the drained hit records (before partitioning), then
  // the UpdatePeerGlobal items
  gub_req *g_reqs = nullptr; gub_resp* g_resps = nullptr; gub_item *g_items = nullptr, *g_gather = nullptr;
  uint32_t* g_count = nullptr;     // [4] device counters (hits drained, queries drained, items made, spare)
  uint32_t* g_counts_all = nullptr;  // [MAX_SHARDS] device: items per rank
  uint32_t* g_hist = nullptr;      // [GQ_BINS] device: this tick's hit records per bin, then the partition's cursors
  uint32_t* g_hist_all = nullptr;  // [world x GQ_BINS] device: every rank's histogram (NCCL all-gather)
  uint32_t* h_hist = nullptr;      // pinned [world x GQ_BINS]: row r = rank r's histogram (local group: only our own row is filled)
  uint32_t* h_start = nullptr;     // pinned [GQ_BINS + 1]: exclusive prefix sum of our histogram
  std::vector<gub::GqRound> rounds;  // the tick's rounds, identical on every shard
  uint32_t round_n = 0;            // hit records this shard sends in the round in flight
  uint64_t seq = 0;
  // all shards in one process (gub_p2p_connect_local): peers by pointer + a host-side rendezvous for the GLOBAL tick
  struct LocalGroup { std::mutex mu; std::condition_variable cv; uint32_t arrived = 0, gen = 0; } own_group;
  LocalGroup* group = nullptr;
  gub_p2p* local_peers[gub::MAX_SHARDS] = {};
  cudaEvent_t phase_ev = nullptr;  // single-thread drivers: 'this shard's phase has been enqueued and completed' (see local_phase_sync)
  uint32_t* h_counts = nullptr;    // pinned: {hits drained, queries drained, items made, spare} of the tick in flight
  void* nccl = nullptr;            // ncclComm_t
  uint64_t tick_bytes = 0;         // bytes all-gathered by the last tick
  // Store steps (gub_p2p_step_keys_store_local_all), allocated by the first one: [2][world][cap] inverse map of this shard's routing by
  // step parity (k_store_orig), read by the owners over peer access
  uint32_t* store_orig = nullptr;
  // Wire-bytes steps (gub_p2p_step_proto_local_all), allocated and grown by the calls: two sets by call parity, each holding the
  // packed copy, the decode scratch and the dense batch with its responses.  A set is reused once the call two back has been encoded.
  PipeSlot proto_set[2];
  uint32_t proto_calls = 0;
  cudaStream_t s_proto = nullptr;  // decoding: waits only for its own call's copy, so it overlaps the previous call's steps
};

namespace {
size_t p2p_req_bytes(uint32_t W, uint32_t cap) { return (size_t)2 * W * cap * sizeof(gub_req); }
size_t p2p_resp_bytes(uint32_t W, uint32_t cap) { return (size_t)2 * W * cap * sizeof(gub_resp); }
gub::P2PView p2p_view(void* base, uint32_t W, uint32_t cap) {
  gub::P2PView v;
  char* b = static_cast<char*>(base);
  v.req_mb = reinterpret_cast<gub_req*>(b);
  v.resp_mb = reinterpret_cast<gub_resp*>(b + p2p_req_bytes(W, cap));
  v.req_flag = reinterpret_cast<unsigned long long*>(b + p2p_req_bytes(W, cap) + p2p_resp_bytes(W, cap));
  v.resp_flag = v.req_flag + 2 * W;
  return v;
}

// A bounded device-side wait gave up during an earlier step (a peer died or hung): surfaced here, at the next call, without
// adding a host round trip to the step itself.  The flag is host-mapped... it is device memory; reading it costs a sync, so
// callers poll it with gub_p2p_status() at their own cadence.
}  // namespace

extern "C" {

void gub_p2p_destroy(gub_p2p* p) {
  if (!p) return;
  cudaSetDevice(p->t->device);
  cudaDeviceSynchronize();
  for (uint32_t r = 0; r < p->world; r++) if (p->opened[r]) cudaIpcCloseMemHandle(p->opened[r]);
  void* ptrs[] = {p->block, p->error, p->ticket, p->seg_off, p->g_reqs, p->g_resps, p->g_items, p->g_gather, p->g_count, p->g_counts_all,
                  p->g_hist, p->g_hist_all, p->store_orig};
  for (void* q : ptrs) if (q) cudaFree(q);
  if (p->h_counts) cudaFreeHost(p->h_counts);
  if (p->h_hist) cudaFreeHost(p->h_hist);
  if (p->h_start) cudaFreeHost(p->h_start);
  if (p->phase_ev) cudaEventDestroy(p->phase_ev);
  if (p->ev_fork) cudaEventDestroy(p->ev_fork);
  if (p->s_eval) cudaStreamDestroy(p->s_eval);
  if (p->s_collect) cudaStreamDestroy(p->s_collect);
  for (auto& r : p->rt) {
    void* rp[] = {r.tile_agg, r.counts, r.perm, r.true_owner, r.expanded, r.params};
    for (void* q : rp) if (q) cudaFree(q);
    if (r.routed) cudaEventDestroy(r.routed);
    if (r.step_done) cudaEventDestroy(r.step_done);
  }
  for (auto& s : p->proto_set) free_slot(s);
  if (p->s_proto) cudaStreamDestroy(p->s_proto);
  if (p->hits_q) gub_gq_destroy(p->hits_q);
  if (p->updates_q) gub_gq_destroy(p->updates_q);
  gub_nccl_comm_destroy_(p->nccl);
  delete p;
}

int gub_p2p_create(gub_table* t, const gub_ring* ring, uint32_t rank, uint32_t cap, gub_p2p** out) {
  const uint32_t world = ring ? (uint32_t)gub_ring_size(ring) : 0;
  if (!t || !out || world == 0 || world > (uint32_t)gub::MAX_SHARDS || rank >= world || cap == 0 || cap >= (1u << 24))
    return fail("gub_p2p_create: bad argument");
  CK(cudaSetDevice(t->device));
  {
    std::lock_guard<std::mutex> lk(t->mu);
    if (ensure_ring(t, ring)) return -1;  // upload the ring now: a step never allocates or synchronises the device
  }
  if (!t->fused) {
    // An owner evaluates what all `world` sources send it in a step: up to world x cap records, normally about cap.  Size the
    // pipeline's scratch so that a step is one pass where it can be (<= 262 144 requests per pass; more passes beyond that).
    const uint32_t want = (uint32_t)std::min<uint64_t>((uint64_t)world * cap, 262144u);
    std::lock_guard<std::mutex> lk(t->mu);
    if (t->max_batch < want) {
      CK(cudaDeviceSynchronize());
      if (alloc_scratch(t, want, 1)) return -1;  // a ring shard's batches wait for their k_seg_wait: one set
    }
  }
  gub_p2p* p = new gub_p2p();
  p->t = t; p->ring = ring; p->world = world; p->rank = rank; p->cap = cap;
  p->block_bytes = p2p_req_bytes(world, cap) + p2p_resp_bytes(world, cap) + (size_t)4 * world * 8;
  cudaError_t e = cudaMalloc(&p->block, p->block_bytes);
  if (e == cudaSuccess) e = cudaMemset(p->block, 0, p->block_bytes);
  if (e == cudaSuccess) e = cudaMalloc(&p->error, 4);
  if (e == cudaSuccess) e = cudaMemset(p->error, 0, 4);
  if (e == cudaSuccess) e = cudaMalloc(&p->ticket, 8);
  if (e == cudaSuccess) e = cudaMemset(p->ticket, 0, 8);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&p->s_eval, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&p->s_collect, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&p->ev_fork, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaMalloc(&p->seg_off, (gub::MAX_SHARDS + 1) * 4);
  if (e == cudaSuccess) e = cudaMemset(p->seg_off, 0, (gub::MAX_SHARDS + 1) * 4);
  const size_t agg = ((size_t)cap / gub::RT_THREADS + 1) * gub::MAX_SHARDS;
  for (auto& r : p->rt) {
    if (e == cudaSuccess) e = cudaMalloc(&r.tile_agg, agg * 8);
    if (e == cudaSuccess) e = cudaMemset(r.tile_agg, 0, agg * 8);
    if (e == cudaSuccess) e = cudaMalloc(&r.counts, gub::MAX_SHARDS * 4);
    if (e == cudaSuccess) e = cudaMemset(r.counts, 0, gub::MAX_SHARDS * 4);
    if (e == cudaSuccess) e = cudaMalloc(&r.perm, (size_t)cap * 4);
    if (e == cudaSuccess) e = cudaMalloc(&r.true_owner, (size_t)cap);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&r.routed, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&r.step_done, cudaEventDisableTiming);
  }
  if (e != cudaSuccess) { gub_p2p_destroy(p); return fail(std::string("gub_p2p_create: ") + cudaGetErrorString(e)); }
  for (uint32_t r = 0; r < world; r++) p->views[r] = p2p_view(p->block, world, cap);  // until connected: everything loops back
  CK(cudaDeviceSynchronize());
  *out = p;
  return 0;
}

int gub_p2p_export(gub_p2p* p, void* handle_out) {
  if (!p || !handle_out) return fail("gub_p2p_export: null argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == GUB_P2P_HANDLE_BYTES, "handle size");
  CK(cudaSetDevice(p->t->device));
  cudaIpcMemHandle_t h;
  CK(cudaIpcGetMemHandle(&h, p->block));
  std::memcpy(handle_out, &h, sizeof h);
  return 0;
}

int gub_p2p_connect(gub_p2p* p, const void* handles) {
  if (!p || !handles) return fail("gub_p2p_connect: null argument");
  CK(cudaSetDevice(p->t->device));
  for (uint32_t r = 0; r < p->world; r++) {
    if (r == p->rank) { p->views[r] = p2p_view(p->block, p->world, p->cap); continue; }
    cudaIpcMemHandle_t h;
    std::memcpy(&h, static_cast<const char*>(handles) + (size_t)r * GUB_P2P_HANDLE_BYTES, sizeof h);
    void* base = nullptr;
    CK(cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess));
    p->opened[r] = base;
    p->views[r] = p2p_view(base, p->world, p->cap);
  }
  p->connected = true;
  return 0;
}

// All shards in this process (the reference daemon is one process: daemon.go:73): the mailboxes are shared by pointer, and
// shards on different devices get peer access to each other's memory enabled here.
int gub_p2p_connect_local(gub_p2p* p, gub_p2p* const* peers) {
  if (!p || !peers) return fail("gub_p2p_connect_local: null argument");
  CK(cudaSetDevice(p->t->device));
  for (uint32_t r = 0; r < p->world; r++) {
    if (!peers[r] || peers[r]->world != p->world || peers[r]->cap != p->cap) return fail("gub_p2p_connect_local: mismatched peer");
    const int dev = peers[r]->t->device;
    if (dev != p->t->device) {
      int can = 0;
      CK(cudaDeviceCanAccessPeer(&can, p->t->device, dev));
      if (!can) return fail("gub_p2p_connect_local: device " + std::to_string(p->t->device) + " cannot access device " + std::to_string(dev));
      cudaError_t e = cudaDeviceEnablePeerAccess(dev, 0);
      if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
      else if (e != cudaSuccess) return fail(std::string("cudaDeviceEnablePeerAccess: ") + cudaGetErrorString(e));
    }
    p->views[r] = p2p_view(peers[r]->block, p->world, p->cap);
    p->local_peers[r] = peers[r];
  }
  p->group = &peers[0]->own_group;
  p->connected = true;
  return 0;
}

int gub_p2p_status(gub_p2p* p, int* error_out) {
  if (!p || !error_out) return fail("gub_p2p_status: null argument");
  CK(cudaSetDevice(p->t->device));
  uint32_t e1 = 0, e2 = 0;
  CK(cudaMemcpy(&e1, p->error, 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(&e2, &p->t->ctl->error, 4, cudaMemcpyDeviceToHost));
  *error_out = (int)(e1 | e2);
  if (e1 | e2) return fail("gub_p2p: a bounded device-side wait gave up (peer flag / grid barrier): a shard of the ring is not answering");
  return 0;
}

}  // extern "C"

namespace {

void p2p_args(gub_p2p* p, gub::P2PArgs& A) {
  for (uint32_t r = 0; r < p->world; r++) A.peers[r] = p->views[r];
  A.world = p->world; A.rank = p->rank; A.cap = p->cap; A.epoch = p->epoch; A.done_ctr = nullptr; A.error = p->error;
}

// The three launches of a step.  d_n (optional): the ingest batch's size lives on the device (<= n).  self_global >= 0: GLOBAL
// requests this shard does not own are answered here (and their true owners recorded for the hits queue).
int p2p_route(gub_p2p* p, gub_p2p::Route* rt, const gub::P2PArgs& A, const gub_req* d_reqs, uint32_t n, const uint32_t* d_n, int self_global, cudaStream_t si) {
  gub_table* t = p->t;
  gub::RouteArgs R;
  R.P = A; R.reqs = d_reqs; R.n = n; R.n_dev = d_n; R.pts = t->d_ring_pts; R.pt_peer = t->d_ring_peers; R.lut = t->d_ring_lut; R.npts = t->ring_npts;
  R.self_global = self_global; R.true_owner = self_global >= 0 ? rt->true_owner : nullptr; R.tile_agg = rt->tile_agg; R.counts = rt->counts; R.perm = rt->perm;
  R.ticket = p->ticket;
  const uint32_t tiles = std::max<uint32_t>(1u, (n + gub::RT_THREADS - 1) / gub::RT_THREADS);
  gub::k_p2p_route<<<tiles, gub::RT_THREADS, 0, si>>>(R);
  CK(cudaGetLastError());
  return 0;
}

// What phase 1 of a step routes: 64-byte records, or a packed key-string batch (gub_keys_layout) with its parameter table (host memory).
struct Ingest {
  bool keys = false;
  const gub_req* reqs = nullptr;
  const uint8_t* packed = nullptr;
  size_t packed_bytes = 0;
  const gub_params* params = nullptr;
  size_t n_params = 0;
  int64_t created_base = 0;
};

// p2p_route for a key-string batch: one launch of k_p2p_route_keys.  A parameter table of more than INLINE_PARAMS sets is copied
// on the ingest stream into this parity's table buffer (grown by p2p_phase_route).  GLOBAL mode: the expanded records also go to
// this parity's scratch for the hits queue.
int p2p_route_keys(gub_p2p* p, gub_p2p::Route* rt, const gub::P2PArgs& A, const Ingest& in, uint32_t n, int self_global, cudaStream_t si) {
  gub_table* t = p->t;
  gub::KeysRouteArgs K;
  std::memset(&K, 0, sizeof K);
  gub::RouteArgs& R = K.R;
  R.P = A; R.reqs = nullptr; R.n = n; R.n_dev = nullptr; R.pts = t->d_ring_pts; R.pt_peer = t->d_ring_peers; R.lut = t->d_ring_lut; R.npts = t->ring_npts;
  R.self_global = self_global; R.true_owner = self_global >= 0 ? rt->true_owner : nullptr; R.tile_agg = rt->tile_agg; R.counts = rt->counts; R.perm = rt->perm;
  R.ticket = p->ticket;
  const size_t bytes_at = (size_t)n * sizeof(gub_kreq) + ((size_t)n + 1) * 4;
  K.packed = in.packed;
  K.key_bytes = n ? in.packed_bytes - bytes_at : 0;
  K.n_params = (uint32_t)in.n_params;
  K.created_base = in.created_base;
  K.expanded = self_global >= 0 ? rt->expanded : nullptr;
  if (in.n_params <= gub::INLINE_PARAMS) {
    if (in.n_params) std::memcpy(&K.Pi, in.params, in.n_params * sizeof(gub_params));
  } else {
    CK(cudaMemcpyAsync(rt->params, in.params, in.n_params * sizeof(gub_params), cudaMemcpyHostToDevice, si));
    K.params_far = rt->params;
  }
  const uint32_t tiles = std::max<uint32_t>(1u, (n + gub::RT_THREADS - 1) / gub::RT_THREADS);
  gub::k_p2p_route_keys<<<tiles, gub::RT_THREADS, 0, si>>>(K);
  CK(cudaGetLastError());
  return 0;
}

// The mailbox segments of this step as the batch kernels in ring mode read them.
SegDesc p2p_segs(gub_p2p* p, const gub::P2PArgs& A) {
  const uint32_t par = p->epoch & 1u;
  SegDesc sd;
  sd.nseg = p->world; sd.seg_off = p->seg_off;
  for (uint32_t s = 0; s < p->world; s++) {
    sd.reqs[s] = A.peers[p->rank].req_mb + ((size_t)par * p->world + s) * p->cap;   // what source s stored into our mailbox
    sd.out[s] = A.peers[s].resp_mb + ((size_t)par * p->world + p->rank) * p->cap;   // NVLink stores into source s's response mailbox
  }
  return sd;
}

// The pieces of the owner side on the four-kernel pipeline: k_seg_wait (one warp waits for the sources' flags and writes the segment
// offsets), the batch kernels in ring mode over as many passes as world x cap takes (responses stored straight into the sources'
// response mailboxes), k_seg_publish (response flags).
int p2p_seg_wait(gub_p2p* p, const gub::P2PArgs& A, cudaStream_t st) {
  gub::k_seg_wait<<<1, 32, 0, st>>>(A, p->seg_off);
  CK(cudaGetLastError());
  return 0;
}
int p2p_eval_passes(gub_p2p* p, const gub::P2PArgs& A, const gub_clock* clk, cudaStream_t st) {
  gub_table* t = p->t;
  const SegDesc sd = p2p_segs(p, A);
  const uint64_t total = (uint64_t)p->world * p->cap;
  for (uint64_t off = 0; off < total; off += t->max_batch) {
    const uint32_t m = (uint32_t)std::min<uint64_t>(t->max_batch, total - off);
    if (launch_chunk(t, nullptr, m, clk, nullptr, st, p->seg_off + p->world, (uint32_t)off, &sd)) return -1;
  }
  return 0;
}
int p2p_publish_flags(gub_p2p* p, const gub::P2PArgs& A, cudaStream_t st) {
  gub_table* t = p->t;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(1); cfg.blockDim = dim3(32); cfg.dynamicSmemBytes = 0; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = (t->pdl && !t->prof) ? 1 : 0;
  CK(cudaLaunchKernelEx(&cfg, gub::k_seg_publish, A));
  return 0;
}
int p2p_publish(gub_p2p* p, const gub::P2PArgs& A, const gub_clock* clk, cudaStream_t st) {
  if (p2p_publish_flags(p, A, st)) return -1;
  return maybe_sweep(p->t, clk, st);
}

// The owner side of a step.  Default: the four-kernel pipeline reading the mailbox segments in place (p2p_seg_wait, p2p_eval_passes,
// p2p_publish).  GUB_PATH=fused: one launch of the persistent kernel instead.
int p2p_evaluate(gub_p2p* p, const gub::P2PArgs& A, const gub_clock* clk, cudaStream_t st) {
  gub_table* t = p->t;
  if (!t->fused) {
    if (p2p_seg_wait(p, A, st)) return -1;
    // GLOBAL requests evaluated here as owner go to the updates queue (gubernator.go:604-606, global.go:80-84).  The queue kernels
    // read the request mailboxes, so they run BEFORE the response flags go out: once a source has its answers it may route the
    // step after next into the same mailbox half.
    if (p->updates_q && gq_accumulate_segments(p, A, st)) return -1;
    if (p2p_eval_passes(p, A, clk, st)) return -1;
    return p2p_publish(p, A, clk, st);
  }
  gub::FArgs F;
  fused_base_args(t, clk, F);
  const uint32_t par = p->epoch & 1u;
  for (uint32_t s = 0; s < p->world; s++) {
    F.seg[s].reqs = A.peers[p->rank].req_mb + ((size_t)par * p->world + s) * p->cap;         // what source s stored into our mailbox
    F.seg[s].flag = &A.peers[p->rank].req_flag[(size_t)par * p->world + s];
    F.seg[s].out = A.peers[s].resp_mb + ((size_t)par * p->world + p->rank) * p->cap;         // NVLink stores into source s's response mailbox
    F.seg[s].n = p->cap;
    F.resp_flag[s] = &A.peers[s].resp_flag[(size_t)par * p->world + p->rank];
  }
  F.nseg = p->world; F.n_resp_flags = p->world; F.flag_epoch = p->epoch;
  return launch_fused(t, F, 0, st);
}

}  // namespace

extern "C" {

}  // extern "C"

namespace {

int p2p_step_check(gub_p2p* p, const void* d_in, size_t n, const gub_clock* clk, gub_resp* d_out, const char* what = "gub_p2p_step") {
  if (!p || !clk || (n && (!d_in || !d_out))) return fail(std::string(what) + ": null argument");
  if (n > p->cap) return fail(std::string(what) + ": n exceeds the mailbox capacity");
  if (p->t->ring_cached != p->ring || p->t->ring_version != gub_ring_version_(p->ring)) return fail(std::string(what) + ": the table's ring changed since gub_p2p_create");
  return 0;
}

// The checks of p2p_step_check plus those of a key-string batch (the offsets themselves are device memory: the kernel clamps them).
int p2p_step_keys_check(gub_p2p* p, const void* d_packed, size_t packed_bytes, size_t n, const gub_params* params, size_t n_params, const gub_clock* clk,
                        gub_resp* d_out, const char* what) {
  if (p2p_step_check(p, d_packed, n, clk, d_out, what)) return -1;
  if (n_params && !params) return fail(std::string(what) + ": null argument");
  if (n_params > 0xFFFFFFFFull) return fail(std::string(what) + ": too many parameter sets");
  if (n && packed_bytes < n * sizeof(gub_kreq) + (n + 1) * 4) return fail(std::string(what) + ": packed buffer smaller than its records and offsets");
  return 0;
}

// Phase 1 of a step, on the ingest stream: partition by owner and store the records into the owners' mailboxes.  This parity's
// scratch and mailbox halves were last used two steps ago; that step's collect (on the evaluation stream) must have finished,
// which also means every peer has drained what we sent it then.
int p2p_phase_route(gub_p2p* p, const Ingest& in, size_t n, cudaStream_t si, cudaStream_t st) {
  gub_table* t = p->t;
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  const bool two = si != st;
  if (in.keys && in.n_params > gub::INLINE_PARAMS) {  // grow the next parity's parameter table before the step counts as started
    gub_p2p::Route* nx = &p->rt[(p->epoch + 1) & 1u];
    if (nx->params_cap < in.n_params) {
      if (nx->params) CK(cudaFree(nx->params));
      nx->params = nullptr; nx->params_cap = 0;
      CK(cudaMalloc(&nx->params, in.n_params * sizeof(gub_params)));
      nx->params_cap = in.n_params;
    }
  }
  p->epoch++;
  gub_p2p::Route* rt = &p->rt[p->epoch & 1u];
  gub::P2PArgs A;
  p2p_args(p, A);
  if (two && rt->step_done_valid) CK(cudaStreamWaitEvent(si, rt->step_done, 0));
  const int self_global = p->hits_q ? (int)p->rank : -1;
  if (in.keys) {
    if (p2p_route_keys(p, rt, A, in, (uint32_t)n, self_global, si)) return -1;
  } else {
    if (p2p_route(p, rt, A, in.reqs, (uint32_t)n, nullptr, self_global, si)) return -1;
  }
  if (p->hits_q && n) {  // a non-owner queues the hits of its GLOBAL requests (gubernator.go:402-404, global.go:74-78)
    if (gq_accumulate(p->hits_q, in.keys ? rt->expanded : in.reqs, n, nullptr, rt->true_owner, p->rank, p->seq, si)) return -1;
  }
  if (two) CK(cudaEventRecord(rt->routed, si));
  return 0;
}

// Phase 2, on the evaluation stream: the batch kernel synchronises with every source (ourselves included) through the mailbox
// flags, evaluates straight out of the mailboxes and stores the responses into the sources' response mailboxes.
int p2p_phase_evaluate(gub_p2p* p, const gub_clock* clk, cudaStream_t st) {
  gub_table* t = p->t;
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  gub::P2PArgs A;
  p2p_args(p, A);
  if (order_after_last(t, st)) return -1;
  if (p2p_evaluate(p, A, clk, st)) return -1;
  t->last_stream = st; t->last_pending = true;
  if (p->updates_q && t->fused) {  // GLOBAL requests just evaluated as owner (gubernator.go:604-606, global.go:80-84); the pipeline path queues them itself
    if (gq_accumulate_segments(p, A, st)) return -1;
  }
  return 0;
}

// Phase 3: wait for the owners' flags, responses back in request order.
int p2p_phase_collect(gub_p2p* p, size_t n, gub_resp* d_out, cudaStream_t si, cudaStream_t st) {
  gub_table* t = p->t;
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  const bool two = si != st;
  gub_p2p::Route* rt = &p->rt[p->epoch & 1u];
  gub::P2PArgs A;
  p2p_args(p, A);
  if (two) CK(cudaStreamWaitEvent(st, rt->routed, 0));  // the collect reads this parity's permutation
  gub::k_p2p_collect<<<std::max<unsigned>(1u, std::min<unsigned>((unsigned)t->num_sms, (unsigned)((n + 255) / 256))), 256, 0, st>>>(A, rt->perm, (uint32_t)n, nullptr, d_out);
  if (two) { CK(cudaEventRecord(rt->step_done, st)); rt->step_done_valid = true; }
  CK(cudaGetLastError());
  p->seq += (uint64_t)1 << 32;
  return 0;
}

int p2p_step_streams(gub_p2p* p, const Ingest& in, size_t n, const gub_clock* clk, gub_resp* d_out, void* ingest_stream, void* stream);

}  // namespace

extern "C" {

int gub_p2p_step_streams(gub_p2p* p, const gub_req* d_reqs, size_t n, const gub_clock* clk, gub_resp* d_out, void* ingest_stream, void* stream) {
  if (p2p_step_check(p, d_reqs, n, clk, d_out)) return -1;
  Ingest in;
  in.reqs = d_reqs;
  return p2p_step_streams(p, in, n, clk, d_out, ingest_stream, stream);
}

}  // extern "C"

namespace {

int p2p_step_streams(gub_p2p* p, const Ingest& in, size_t n, const gub_clock* clk, gub_resp* d_out, void* ingest_stream, void* stream) {
  cudaStream_t st = (cudaStream_t)stream, si = (cudaStream_t)ingest_stream;
  // Default: routing on the ingest stream, evaluation and collect on `stream`.  GUB_RING_STREAMS=3 (experimental) moves the evaluation
  // and the collect — which waits for the slowest owner — onto streams of the ring's own, so that step e+1 is evaluated while step e's
  // answers travel; that variant has been seen to stall under the per-kernel profiling events.
  static const int own_streams = [] { const char* e = getenv("GUB_RING_STREAMS"); return e ? std::atoi(e) : 2; }();
  if (si != st && own_streams < 3) {
    if (p2p_phase_route(p, in, n, si, st)) return -1;
    if (p2p_phase_evaluate(p, clk, st)) return -1;
    return p2p_phase_collect(p, n, d_out, si, st);
  }
  if (si == st) {  // one stream: the three phases in stream order
    if (p2p_phase_route(p, in, n, si, st)) return -1;
    if (p2p_phase_evaluate(p, clk, st)) return -1;
    return p2p_phase_collect(p, n, d_out, si, st);
  }
  // Two caller streams: routing on the ingest stream; the owner-side evaluation on our own evaluation stream (it synchronises with
  // the peers through the mailbox flags, not through the caller's streams); the collect — which waits for the slowest owner — on our
  // collect stream; `stream` then waits for the collect only.  Step e+1 is routed and evaluated while step e's answers travel.
  if (p2p_phase_route(p, in, n, si, p->s_collect)) return -1;
  if (p2p_phase_evaluate(p, clk, p->s_eval)) return -1;
  CK(cudaEventRecord(p->ev_fork, st));                 // d_out is ours to write once everything queued on `stream` so far is done
  CK(cudaStreamWaitEvent(p->s_collect, p->ev_fork, 0));
  if (p2p_phase_collect(p, n, d_out, si, p->s_collect)) return -1;
  CK(cudaStreamWaitEvent(st, p->rt[p->epoch & 1u].step_done, 0));
  p->last_ingest = si; p->own_streams_used = true;
  return 0;
}

Ingest keys_ingest(const void* d_packed, size_t packed_bytes, const gub_params* params, size_t n_params, int64_t created_base) {
  Ingest in;
  in.keys = true; in.packed = static_cast<const uint8_t*>(d_packed); in.packed_bytes = packed_bytes;
  in.params = params; in.n_params = n_params; in.created_base = created_base;
  return in;
}

}  // namespace

extern "C" {

/* Key strings in (gub_keys_layout, on the shard's device), responses out: k_p2p_route_keys hashes, expands and routes in one launch,
 * then the step goes on exactly as gub_p2p_step_streams. */
int gub_p2p_step_keys(gub_p2p* p, const void* d_packed, size_t packed_bytes, size_t n, const gub_params* params, size_t n_params, int64_t created_base,
                      const gub_clock* clk, gub_resp* d_out, void* ingest_stream, void* stream) {
  if (p2p_step_keys_check(p, d_packed, packed_bytes, n, params, n_params, clk, d_out, "gub_p2p_step_keys")) return -1;
  return p2p_step_streams(p, keys_ingest(d_packed, packed_bytes, params, n_params, created_base), n, clk, d_out, ingest_stream, stream);
}

}  // extern "C"

namespace {
// Between the phases of the single-thread drivers: every shard's stream waits for the phase just enqueued on every other shard's
// stream.  The kernels of the next phase then find their mailbox flags already published and never spin: on a device shared by
// several shards a spinning kernel could keep another shard's (cooperative, all-SM) batch kernel from ever becoming resident.
int local_phase_sync(gub_p2p* const* ps, uint32_t world, void* const* streams) {
  if (world < 2) return 0;
  for (uint32_t r = 0; r < world; r++) {
    CK(cudaSetDevice(ps[r]->t->device));
    if (!ps[r]->phase_ev) CK(cudaEventCreateWithFlags(&ps[r]->phase_ev, cudaEventDisableTiming));
    CK(cudaEventRecord(ps[r]->phase_ev, (cudaStream_t)streams[r]));
  }
  for (uint32_t r = 0; r < world; r++) {
    CK(cudaSetDevice(ps[r]->t->device));
    for (uint32_t q = 0; q < world; q++) if (q != r) CK(cudaStreamWaitEvent((cudaStream_t)streams[r], ps[q]->phase_ev, 0));
  }
  return 0;
}

// The phases of every shard in order: all routings, then all evaluations, then all collects (arguments checked by the caller).
int p2p_local_all(gub_p2p* const* ps, uint32_t world, const Ingest* in, const size_t* n, const gub_clock* clk, gub_resp* const* d_out,
                  void* const* streams) {
  for (uint32_t r = 0; r < world; r++) if (p2p_phase_route(ps[r], in[r], n[r], (cudaStream_t)streams[r], (cudaStream_t)streams[r])) return -1;
  if (local_phase_sync(ps, world, streams)) return -1;
  for (uint32_t r = 0; r < world; r++) if (p2p_phase_evaluate(ps[r], clk, (cudaStream_t)streams[r])) return -1;
  if (local_phase_sync(ps, world, streams)) return -1;
  for (uint32_t r = 0; r < world; r++) if (p2p_phase_collect(ps[r], n[r], d_out[r], (cudaStream_t)streams[r], (cudaStream_t)streams[r])) return -1;
  return 0;
}
}  // namespace

extern "C" {

/* One step of every shard of this process, driven by ONE host thread (the shape of the reference daemon: one process): the
 * phases are enqueued shard by shard — all routings, then all evaluations, then all collects — so that no shard's kernels wait
 * for work the host has not enqueued yet (on ONE device that would deadlock: the batch kernel occupies every SM). */
int gub_p2p_step_local_all(gub_p2p* const* ps, uint32_t world, const gub_req* const* d_reqs, const size_t* n, const gub_clock* clk,
                           gub_resp* const* d_out, void* const* streams) {
  if (!ps || !d_reqs || !n || !d_out || !streams || world == 0) return fail("gub_p2p_step_local_all: bad argument");
  for (uint32_t r = 0; r < world; r++) if (p2p_step_check(ps[r], d_reqs[r], n[r], clk, d_out[r])) return -1;
  std::vector<Ingest> in(world);
  for (uint32_t r = 0; r < world; r++) in[r].reqs = d_reqs[r];
  return p2p_local_all(ps, world, in.data(), n, clk, d_out, streams);
}

/* gub_p2p_step_local_all with key strings: shard r ingests the packed batch d_packed[r] (n[r] requests, on its device); one parameter
 * table for all shards. */
int gub_p2p_step_keys_local_all(gub_p2p* const* ps, uint32_t world, const void* const* d_packed, const size_t* packed_bytes, const size_t* n,
                                const gub_params* params, size_t n_params, int64_t created_base, const gub_clock* clk, gub_resp* const* d_out,
                                void* const* streams) {
  return gub_p2p_step_mixed_local_all(ps, world, nullptr, d_packed, packed_bytes, n, params, n_params, created_base, clk, d_out, streams);
}

/* Both kinds of ingest in one step: shard r ingests key strings when d_packed[r] != NULL, else the records d_reqs[r]. */
int gub_p2p_step_mixed_local_all(gub_p2p* const* ps, uint32_t world, const gub_req* const* d_reqs, const void* const* d_packed, const size_t* packed_bytes,
                                 const size_t* n, const gub_params* params, size_t n_params, int64_t created_base, const gub_clock* clk,
                                 gub_resp* const* d_out, void* const* streams) {
  const char* what = d_reqs ? "gub_p2p_step_mixed_local_all" : "gub_p2p_step_keys_local_all";
  if (!ps || !d_packed || !packed_bytes || !n || !d_out || !streams || world == 0) return fail(std::string(what) + ": bad argument");
  std::vector<Ingest> in(world);
  for (uint32_t r = 0; r < world; r++) {
    if (d_packed[r] || !d_reqs) {
      if (p2p_step_keys_check(ps[r], d_packed[r], packed_bytes[r], n[r], params, n_params, clk, d_out[r], what)) return -1;
      in[r] = keys_ingest(d_packed[r], packed_bytes[r], params, n_params, created_base);
    } else {
      if (p2p_step_check(ps[r], d_reqs[r], n[r], clk, d_out[r], what)) return -1;
      in[r].reqs = d_reqs[r];
    }
  }
  return p2p_local_all(ps, world, in.data(), n, clk, d_out, streams);
}

int gub_p2p_step(gub_p2p* p, const gub_req* d_reqs, size_t n, const gub_clock* clk, gub_resp* d_out, void* stream) {
  return gub_p2p_step_streams(p, d_reqs, n, clk, d_out, stream, stream);
}

}  // extern "C"

namespace {

// A Store plugin's part in a ring step: the Get callback and every owner's change log (device views of the caller's page-locked buffers).
struct RingStore {
  gub_store_get_fn get = nullptr;
  void* user = nullptr;
  std::vector<gub_store_rec*> changes;
  std::vector<uint32_t*> n_changes;
};

// Owner p's pass as the Store kernels read it: its mailbox segments, and every source's inverse map and routing permutation of this
// step's parity (the sources' memory: peer access).
gub::StoreSegs store_segs(gub_p2p* p, const gub::P2PArgs& A) {
  const uint32_t par = p->epoch & 1u;
  const SegDesc sd = p2p_segs(p, A);
  gub::StoreSegs G;
  std::memset(&G, 0, sizeof G);
  G.nseg = p->world; G.seg_off = p->seg_off;
  for (uint32_t s = 0; s < p->world; s++) {
    const gub_p2p* src = p->local_peers[s];
    G.req[s] = sd.reqs[s]; G.out[s] = sd.out[s];
    G.orig[s] = src->store_orig + ((size_t)par * p->world + p->rank) * p->cap;
    G.perm[s] = src->rt[par].perm;
  }
  return G;
}

// p2p_local_all with the Store's pre- and post-pass on every owner (arguments checked by the caller):
//   1. every routing, each followed by its inverse map (k_store_orig);   2. local_phase_sync;
//   3. per owner: k_seg_wait, the pre-pass and, with a Get, the miss list compacted into the table's page-locked buffer;
//   4. with a Get: wait for every miss list, call Get per owner in rank order, then install what it returned on every owner;
//   5. per owner: the ring-mode passes, the post-pass straight into changes[r], k_seg_publish.  The post-pass reads the request
//      mailbox, so it runs before the response flags go out (a source that has its answers may route step e + 2 into that half);
//   6. local_phase_sync;   7. every collect.
// A failing Get (or a table that cannot take the items the store returned) fails the call, but every owner still publishes its flags
// (without evaluating) and every source collects, so that the ring stays in step.
int p2p_local_all_store(gub_p2p* const* ps, uint32_t world, const Ingest* in, const size_t* n, const gub_clock* clk, const RingStore& rs,
                        gub_resp* const* d_out, void* const* streams) {
  const char* what = "gub_p2p_step_keys_store_local_all";
  const uint32_t pass = world * ps[0]->cap;  // launch size of the Store kernels; the pass itself is seg_off[world] <= pass
  const unsigned blocks = (pass + gub::STORE_THREADS - 1) / gub::STORE_THREADS;
  for (uint32_t r = 0; r < world; r++) {
    gub_p2p* p = ps[r];
    const cudaStream_t st = (cudaStream_t)streams[r];
    if (p2p_phase_route(p, in[r], n[r], st, st)) return -1;
    std::lock_guard<std::mutex> lk(p->t->mu);
    CK(cudaSetDevice(p->t->device));
    if (n[r]) {
      gub::k_store_orig<<<(unsigned)((n[r] + 255) / 256), 256, 0, st>>>(p->rt[p->epoch & 1u].perm, (uint32_t)n[r], p->cap,
                                                                         p->store_orig + (size_t)(p->epoch & 1u) * world * p->cap);
      CK(cudaGetLastError());
    }
  }
  if (local_phase_sync(ps, world, streams)) return -1;
  std::vector<gub::StoreArgs> S(world);
  std::vector<gub::StoreSegs> G(world);
  for (uint32_t r = 0; r < world; r++) {
    gub_p2p* p = ps[r];
    gub_table* t = p->t;
    const cudaStream_t st = (cudaStream_t)streams[r];
    std::lock_guard<std::mutex> lk(t->mu);
    CK(cudaSetDevice(t->device));
    gub::P2PArgs A;
    p2p_args(p, A);
    if (order_after_last(t, st)) return -1;
    if (p2p_seg_wait(p, A, st)) return -1;
    if (store_args(t, clk, rs.get != nullptr, S[r], st)) return -1;
    S[r].n = pass;
    G[r] = store_segs(p, A);
    gub::k_store_keys_ring<<<blocks, gub::STORE_THREADS, 0, st>>>(S[r], G[r]);
    gub::k_store_before_ring<<<blocks, gub::STORE_THREADS, 0, st>>>(S[r], G[r]);
    CK(cudaGetLastError());
    t->last_stream = st; t->last_pending = true;
    if (rs.get && store_misses(t, blocks, pass, st)) return -1;
  }
  bool failed = false;
  if (rs.get) {
    std::vector<uint32_t> nl(world, 0), ni(world, 0);
    for (uint32_t r = 0; r < world; r++) {
      CK(cudaSetDevice(ps[r]->t->device));
      CK(cudaEventSynchronize(ps[r]->t->store.misses_done));
    }
    for (uint32_t r = 0; r < world && !failed; r++) {
      std::lock_guard<std::mutex> lk(ps[r]->t->mu);
      failed = store_get(ps[r]->t, rs.get, rs.user, clk, what, &nl[r], &ni[r]) != 0;
    }
    for (uint32_t r = 0; r < world && !failed; r++) {
      std::lock_guard<std::mutex> lk(ps[r]->t->mu);
      CK(cudaSetDevice(ps[r]->t->device));
      failed = store_install(ps[r]->t, nl[r], ni[r], &G[r], (cudaStream_t)streams[r]) != 0;
    }
    for (uint32_t r = 0; r < world && !failed; r++) {
      if (!ni[r]) continue;
      std::lock_guard<std::mutex> lk(ps[r]->t->mu);
      CK(cudaSetDevice(ps[r]->t->device));
      failed = store_install_check(ps[r]->t, what, (cudaStream_t)streams[r]) != 0;
    }
  }
  const std::string err = failed ? g_err : std::string();
  for (uint32_t r = 0; r < world; r++) {
    gub_p2p* p = ps[r];
    gub_table* t = p->t;
    const cudaStream_t st = (cudaStream_t)streams[r];
    std::lock_guard<std::mutex> lk(t->mu);
    CK(cudaSetDevice(t->device));
    gub::P2PArgs A;
    p2p_args(p, A);
    if (failed) {
      if (p2p_publish_flags(p, A, st)) return -1;
      continue;
    }
    if (p2p_eval_passes(p, A, clk, st)) return -1;
    gub::k_store_after_ring<<<blocks, gub::STORE_THREADS, 0, st>>>(S[r], G[r]);
    gub::k_store_compact<<<blocks, gub::STORE_THREADS, 0, st>>>(t->store.sel, t->store.sparse, t->store.blk, pass, rs.changes[r], rs.n_changes[r]);
    CK(cudaGetLastError());
    if (p2p_publish(p, A, clk, st)) return -1;
    t->last_stream = st; t->last_pending = true;
  }
  if (local_phase_sync(ps, world, streams)) return -1;
  for (uint32_t r = 0; r < world; r++) if (p2p_phase_collect(ps[r], n[r], d_out[r], (cudaStream_t)streams[r], (cudaStream_t)streams[r])) return -1;
  if (failed) return fail(err);
  return 0;
}

}  // namespace

extern "C" {

int gub_p2p_step_keys_store_local_all(gub_p2p* const* ps, uint32_t world, const void* const* d_packed, const size_t* packed_bytes,
                                      const size_t* n, const gub_params* params, size_t n_params, int64_t created_base,
                                      const gub_clock* clk, gub_store_get_fn get, void* user, gub_resp* const* d_out,
                                      gub_store_rec* const* changes, uint32_t* const* n_changes, void* const* streams) {
  const std::string what = "gub_p2p_step_keys_store_local_all";
  if (!ps || !d_packed || !packed_bytes || !n || !d_out || !changes || !n_changes || !streams || world == 0) return fail(what + ": bad argument");
  std::vector<Ingest> in(world);
  RingStore rs;
  rs.get = get; rs.user = user;
  for (uint32_t r = 0; r < world; r++) {
    gub_p2p* p = ps[r];
    if (p2p_step_keys_check(p, d_packed[r], packed_bytes[r], n[r], params, n_params, clk, d_out[r], what.c_str())) return -1;
    if (p->world != world || p->rank != r) return fail(what + ": ps[" + std::to_string(r) + "] is not rank " + std::to_string(r) + " of a ring of " + std::to_string(world));
    if (p->t->fused) return fail(what + ": not available on tables created under GUB_PATH=fused");
    if (p->hits_q || p->updates_q) return fail(what + ": not available on a ring with GLOBAL enabled (the owner-side application of a tick's hits has no change log)");
    bool local = p->group != nullptr;
    for (uint32_t s = 0; s < world; s++) local = local && p->local_peers[s] == ps[s];
    if (!local) return fail(what + ": the shards must be connected with gub_p2p_connect_local");
    if ((uint64_t)world * p->cap > p->t->max_batch)
      return fail(what + ": world x cap = " + std::to_string((uint64_t)world * p->cap) + " exceeds an owner's pass of " + std::to_string(p->t->max_batch) +
                  " requests (a key split over two passes would get two records)");
    CK(cudaSetDevice(p->t->device));
    if (!changes[r] || !n_changes[r]) return fail(what + ": null argument");
    rs.changes.push_back(pinned_view(changes[r]));
    rs.n_changes.push_back(pinned_view(n_changes[r]));
    if (!rs.changes.back() || !rs.n_changes.back()) return fail(what + ": changes and n_changes must be page-locked host memory (gub_host_alloc)");
    in[r] = keys_ingest(d_packed[r], packed_bytes[r], params, n_params, created_base);
  }
  for (uint32_t r = 0; r < world; r++) {  // the first Store step allocates (and synchronises the device) before anything is enqueued
    gub_p2p* p = ps[r];
    std::lock_guard<std::mutex> lk(p->t->mu);
    CK(cudaSetDevice(p->t->device));
    if (store_ensure(p->t)) return -1;
    if (!p->store_orig) {
      const size_t bytes = (size_t)2 * world * p->cap * 4;
      CK(cudaMalloc(&p->store_orig, bytes));
      CK(cudaMemset(p->store_orig, 0, bytes));
    }
  }
  return p2p_local_all_store(ps, world, in.data(), n, clk, rs, d_out, streams);
}

}  // extern "C"

namespace {
// One shard's part in a wire-bytes call: its plan, its decode set and the arguments its kernels share.
struct ProtoShard {
  gub::ProtoPlan P{};
  gub::ProtoArgs A{};
  PipeSlot* set = nullptr;
  size_t n_msgs = 0;
  uint32_t n_eval = 0;
};
}  // namespace

extern "C" {

/* Wire bytes on the ring (see the header).  1. every check on every shard; 2. per shard: wait for the call two back on this parity's
 * set, grow it; 3. per shard on its decode stream: copy, decode, compact; 4. the host waits for every decoded count; 5. S ring steps
 * through p2p_local_all, step k ingesting [k x cap, (k + 1) x cap) of each dense batch; 6. per shard on streams[r]: encode. */
int gub_p2p_step_proto_local_all(gub_p2p* const* ps, uint32_t world, const void* const* packed, const size_t* packed_bytes, const size_t* n_msgs,
                                 int force_global, const gub_clock* clk, void* const* out_bytes, const size_t* out_cap, uint64_t* const* out_off,
                                 uint32_t* const* msg_status, void* const* streams) {
  const std::string what = "gub_p2p_step_proto_local_all";
  if (!ps || !packed || !packed_bytes || !n_msgs || !out_bytes || !out_cap || !out_off || !msg_status || !streams || world == 0)
    return fail(what + ": bad argument");
  std::vector<ProtoShard> sh(world);
  for (uint32_t r = 0; r < world; r++) {  // 1. nothing is allocated, copied or enqueued before every shard has passed
    gub_p2p* p = ps[r];
    ProtoShard& h = sh[r];
    const std::string at = what + ": shard " + std::to_string(r) + ": ";
    if (p2p_step_check(p, nullptr, 0, clk, nullptr, what.c_str())) return -1;
    h.n_msgs = n_msgs[r];
    if (!out_off[r] || (h.n_msgs && (!packed[r] || !out_bytes[r] || !msg_status[r]))) return fail(at + "null argument");
    if (h.n_msgs > 0x7FFFFFFFull) return fail(at + "too many messages");
    if (h.n_msgs) {
      if (const char* why = gub::proto_plan(static_cast<const uint8_t*>(packed[r]), packed_bytes[r], h.n_msgs, out_cap[r], h.P)) return fail(at + why);
    }
    CK(cudaSetDevice(p->t->device));
    std::memset(&h.A, 0, sizeof h.A);
    h.A.out = h.n_msgs ? pinned_view(static_cast<uint8_t*>(out_bytes[r])) : nullptr;
    h.A.out_off = pinned_view(reinterpret_cast<unsigned long long*>(out_off[r]));
    h.A.out_status = h.n_msgs ? pinned_view(msg_status[r]) : nullptr;
    if (!h.A.out_off || (h.n_msgs && (!h.A.out || !h.A.out_status)))
      return fail(at + "out_bytes, out_off and msg_status must be page-locked host memory (gub_host_alloc)");
    h.A.force_global = force_global ? 1u : 0u;
  }
  for (uint32_t r = 0; r < world; r++) {  // 2. a failed allocation fails the call before any shard routes
    gub_p2p* p = ps[r];
    ProtoShard& h = sh[r];
    if (!h.n_msgs) continue;
    CK(cudaSetDevice(p->t->device));
    PipeSlot& s = p->proto_set[p->proto_calls & 1u];
    if (s.busy) { CK(cudaEventSynchronize(s.out_done)); s.busy = false; }
    if (!p->s_proto) {
      CK(cudaStreamCreateWithFlags(&p->s_proto, cudaStreamNonBlocking));
      CK(cudaFuncSetAttribute(gub::k_proto_decode, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gub::PROTO_SMEM));
    }
    if (!s.out_done) CK(cudaEventCreateWithFlags(&s.out_done, cudaEventDisableTiming));
    if (ensure_slot(s, std::max<size_t>(h.P.slots, 1)) || proto_ensure(s, h.P, h.n_msgs)) return -1;
    const size_t need = h.P.bytes_at + h.P.msg_bytes;
    if (s.packed_cap < need) {
      if (s.d_packed) cudaFree(s.d_packed);
      s.d_packed = nullptr; s.packed_cap = 0;
      const size_t c = std::max<size_t>(need + need / 4, (size_t)1 << 20);
      CK(cudaMalloc(&s.d_packed, c));
      s.packed_cap = c;
    }
    h.set = &s;
  }
  for (uint32_t r = 0; r < world; r++) {  // 3. the decode of every shard
    gub_p2p* p = ps[r];
    ProtoShard& h = sh[r];
    if (!h.n_msgs) continue;
    CK(cudaSetDevice(p->t->device));
    CK(cudaMemcpyAsync(h.set->d_packed, packed[r], h.P.bytes_at + h.P.msg_bytes, cudaMemcpyHostToDevice, p->s_proto));
    if (proto_decode(*h.set, h.P, h.n_msgs, h.A, p->s_proto)) return -1;
  }
  size_t S = 0;
  for (uint32_t r = 0; r < world; r++) {  // 4. every shard's evaluable count
    gub_p2p* p = ps[r];
    ProtoShard& h = sh[r];
    if (!h.n_msgs) continue;
    CK(cudaSetDevice(p->t->device));
    CK(cudaEventSynchronize(h.set->proto.decoded));
    h.n_eval = *(volatile uint32_t*)h.set->proto.h_neval;
    S = std::max<size_t>(S, ((size_t)h.n_eval + p->cap - 1) / p->cap);
    CK(cudaStreamWaitEvent((cudaStream_t)streams[r], h.set->proto.decoded, 0));
  }
  std::vector<Ingest> in(world);
  std::vector<size_t> n(world);
  std::vector<gub_resp*> d_out(world);
  for (size_t k = 0; k < S; k++) {  // 5. the ring steps: exactly gub_p2p_step_local_all's on each chunk of the dense batches
    for (uint32_t r = 0; r < world; r++) {
      const size_t lo = k * ps[r]->cap;
      n[r] = sh[r].n_eval > lo ? std::min<size_t>(ps[r]->cap, sh[r].n_eval - lo) : 0;
      in[r].reqs = n[r] ? sh[r].set->d_req + lo : nullptr;
      d_out[r] = n[r] ? sh[r].set->d_resp + lo : nullptr;
    }
    if (p2p_local_all(ps, world, in.data(), n.data(), clk, d_out.data(), streams)) return -1;
  }
  for (uint32_t r = 0; r < world; r++) {  // 6. every shard's responses, on its stream
    gub_p2p* p = ps[r];
    ProtoShard& h = sh[r];
    p->proto_calls++;
    if (!h.n_msgs) { out_off[r][0] = 0; continue; }
    CK(cudaSetDevice(p->t->device));
    if (proto_encode(h.A, (cudaStream_t)streams[r])) return -1;
    CK(cudaEventRecord(h.set->out_done, (cudaStream_t)streams[r]));
    h.set->busy = true;
  }
  return 0;
}

}  // extern "C"


// ---- GLOBAL behaviour behind the C ABI: queues fed by the step, and the sync tick (global.go:91-283) with NCCL -----------------
namespace {

int gq_accumulate_segments(gub_p2p* p, const gub::P2PArgs& A, cudaStream_t st) {
  gub_gq* g = p->updates_q;
  const size_t total = (size_t)p->world * p->cap;
  if (gq_reserve(g, total, st)) return -1;
  gub::GqSegs G;
  const uint32_t par = p->epoch & 1u;
  for (uint32_t s = 0; s < p->world; s++) {
    G.reqs[s] = A.peers[p->rank].req_mb + ((size_t)par * p->world + s) * p->cap;
    G.flag[s] = &A.peers[p->rank].req_flag[(size_t)par * p->world + s];
  }
  G.nseg = p->world; G.cap = p->cap;
  gub::k_gq_claim_segs<<<p->t->num_sms, 256, 0, st>>>(g->q, G, (unsigned long long)p->seq, g->slot_of);
  gub::k_gq_fill_segs<<<p->t->num_sms, 256, 0, st>>>(g->q, G, (unsigned long long)p->seq, g->slot_of);
  CK(cudaGetLastError());
  return 0;
}

// NCCL is loaded at run time (libnccl.so.2, the one torch bundles when the host process is Python): a single-GPU deployment
// needs no NCCL at all.  Minimal prototypes of nccl.h (2.27): ncclResult_t is an int enum, ncclComm_t an opaque pointer.
struct Id128 { char b[128]; };
struct NcclApi {
  void* h = nullptr;
  int (*GetUniqueId)(void*) = nullptr;
  int (*CommInitRank)(void**, int, /* ncclUniqueId by value: 128 bytes */ Id128, int) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  bool ok = false;
};
NcclApi g_nccl;
std::mutex g_nccl_mu;

int nccl_load() {
  std::lock_guard<std::mutex> lk(g_nccl_mu);
  if (g_nccl.ok) return 0;
  const char* names[] = {getenv("GUB_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
  for (const char* nm : names) {
    if (!nm) continue;
    g_nccl.h = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
    if (g_nccl.h) break;
  }
  if (!g_nccl.h) return fail("NCCL not found (dlopen libnccl.so.2): GLOBAL sync across GPUs needs it");
#define SYM(field, name)                                                              \
  *reinterpret_cast<void**>(&g_nccl.field) = dlsym(g_nccl.h, name);                   \
  if (!g_nccl.field) return fail(std::string("NCCL symbol missing: ") + name)
  SYM(GetUniqueId, "ncclGetUniqueId");
  SYM(CommInitRank, "ncclCommInitRank");
  SYM(CommDestroy, "ncclCommDestroy");
  SYM(AllGather, "ncclAllGather");
  SYM(GroupStart, "ncclGroupStart");
  SYM(GroupEnd, "ncclGroupEnd");
  SYM(GetErrorString, "ncclGetErrorString");
#undef SYM
  g_nccl.ok = true;
  return 0;
}
#define NCK(call)                                                                                                  \
  do {                                                                                                             \
    int r__ = (call);                                                                                              \
    if (r__ != 0) return fail(std::string(#call) + ": " + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r__) : "nccl error")); \
  } while (0)
}  // namespace

extern "C" {

void gub_nccl_comm_destroy_(void* comm) {
  if (comm && g_nccl.ok) g_nccl.CommDestroy(comm);
}

/* ncclGetUniqueId: 128 bytes the host application hands to every rank (its own channel: the Go daemon's peer discovery, torch.distributed, a file) */
int gub_nccl_unique_id(void* out128) {
  if (!out128) return fail("gub_nccl_unique_id: null argument");
  if (nccl_load()) return -1;
  NCK(g_nccl.GetUniqueId(out128));
  return 0;
}

/* One communicator per shard (rank = the shard's index in the ring).  Collective across the ring's processes. */
int gub_p2p_nccl_init(gub_p2p* p, const void* id128) {
  if (!p || !id128) return fail("gub_p2p_nccl_init: null argument");
  if (nccl_load()) return -1;
  CK(cudaSetDevice(p->t->device));
  Id128 id;
  std::memcpy(&id, id128, sizeof id);
  NCK(g_nccl.CommInitRank(&p->nccl, (int)p->world, id, (int)p->rank));
  return 0;
}

/* All shards in one process: the communicators are created inside one NCCL group. */
int gub_p2p_nccl_init_local(gub_p2p* const* ps, uint32_t world) {
  if (!ps || world == 0) return fail("gub_p2p_nccl_init_local: bad argument");
  if (nccl_load()) return -1;
  Id128 id;
  NCK(g_nccl.GetUniqueId(&id));
  NCK(g_nccl.GroupStart());
  for (uint32_t r = 0; r < world; r++) {
    CK(cudaSetDevice(ps[r]->t->device));
    NCK(g_nccl.CommInitRank(&ps[r]->nccl, (int)world, id, (int)ps[r]->rank));
  }
  NCK(g_nccl.GroupEnd());
  return 0;
}

/* Turns GLOBAL handling on for this shard's steps: GLOBAL requests it does not own are answered from the local replica
 * (gubernator.go:257-269,408-411) and their hits queued (global.go:74-111); GLOBAL requests it evaluates as owner are queued for
 * the broadcast (global.go:80-84,201).  capacity = most distinct GLOBAL keys per sync window, rounded up to a power of two Q; a tick
 * carries all of them (in rounds when they exceed the mailbox capacity), and only requests that find the queue full are counted in
 * gq_dropped.  Device memory per shard: the two queues, (64 + 32 + 88) B x Q of tick staging, a 256 KiB histogram, world x 256 KiB
 * for the histogram exchange and 88 B x min(Q, cap) x world for the item all-gather; (world + 1) x 256 KiB of pinned host memory. */
int gub_p2p_enable_global(gub_p2p* p, uint32_t capacity) {
  if (!p || capacity < 64) return fail("gub_p2p_enable_global: bad argument");
  if (p->hits_q) return 0;
  CK(cudaSetDevice(p->t->device));
  if (gub_gq_create(p->t->device, capacity, 0, &p->hits_q)) return -1;
  if (gub_gq_create(p->t->device, capacity, 1, &p->updates_q)) return -1;
  p->hits_q->q.dropped = p->t->counters + gub::C_GQ_DROPPED;
  p->updates_q->q.dropped = p->t->counters + gub::C_GQ_DROPPED;
  p->gq_recs = next_pow2(capacity);
  p->gcap = std::min<uint32_t>(p->gq_recs, p->cap);
  static_assert(sizeof(gub_item) >= sizeof(gub_req), "g_items also holds the drained hit records");
  CK(cudaMalloc(&p->g_reqs, (size_t)p->gq_recs * sizeof(gub_req)));
  CK(cudaMalloc(&p->g_resps, (size_t)p->gq_recs * sizeof(gub_resp)));
  CK(cudaMalloc(&p->g_items, (size_t)p->gq_recs * sizeof(gub_item)));
  CK(cudaMalloc(&p->g_gather, (size_t)p->gcap * p->world * sizeof(gub_item)));
  CK(cudaMalloc(&p->g_count, 16));
  CK(cudaMemset(p->g_count, 0, 16));
  CK(cudaMalloc(&p->g_counts_all, gub::MAX_SHARDS * 4));
  CK(cudaMalloc(&p->g_hist, (size_t)gub::GQ_BINS * 4));
  CK(cudaMalloc(&p->g_hist_all, (size_t)gub::GQ_BINS * 4 * p->world));
  for (auto& r : p->rt) CK(cudaMalloc(&r.expanded, (size_t)p->cap * sizeof(gub_req)));
  CK(cudaHostAlloc(&p->h_counts, 16, cudaHostAllocDefault));
  std::memset(p->h_counts, 0, 16);
  CK(cudaHostAlloc(&p->h_hist, (size_t)gub::GQ_BINS * 4 * p->world, cudaHostAllocDefault));
  std::memset(p->h_hist, 0, (size_t)gub::GQ_BINS * 4 * p->world);
  CK(cudaHostAlloc(&p->h_start, ((size_t)gub::GQ_BINS + 1) * 4, cudaHostAllocDefault));
  std::memset(p->h_start, 0, ((size_t)gub::GQ_BINS + 1) * 4);
  if (gq_reserve(p->updates_q, (size_t)p->world * p->cap, 0)) return -1;
  if (gq_reserve(p->hits_q, p->cap, 0)) return -1;
  return 0;
}

/* One GLOBAL sync: sendHits (global.go:144-190), then broadcastPeers (global.go:234-283): the owners' UpdatePeerGlobal items reach
 * every other shard, which installs them (UpdatePeerGlobals, gubernator.go:425-459).  Transport of the broadcast: an NCCL
 * all-gather when the shard has a communicator (one process per GPU); direct peer reads when all shards live in this process
 * (gub_p2p_connect_local), where the calling threads — one per shard — rendezvous on the host.  Collective: every shard of the
 * ring calls it the same number of times, interleaved the same way with its steps.  now_ms = MillisecondNow() of the receivers
 * (CreatedAt / UpdatedAt of the installed items).
 * The window's hit records travel in key-consistent rounds of at most `cap` records per source, one mailbox epoch each (see
 * gub_global.cuh): every shard's histogram of its records over the hash space reaches every shard (read in place inside one
 * process, all-gathered by NCCL across processes), and every shard derives the same rounds from them.  Two host round trips: the
 * histograms, then the per-shard item counts (a tick runs every GlobalSyncWait = 500 ms, not per batch).
 * stats (optional, 4 x uint64): hit records sent to owners, update items broadcast by this shard, items installed here, bytes moved. */
}  // extern "C"

namespace {

// A tick in enqueue-only pieces (the drivers synchronise between them), so that one host thread can drive all the shards of a
// process piece by piece (see gub_p2p_step_local_all).
// The drained hit records wait in g_items until k_gq_partition has put them in round order; the items come later.
gub_req* hit_stage(gub_p2p* p) { return reinterpret_cast<gub_req*>(p->g_items); }

// The window's aggregated hits, drained and counted per bin.  Our histogram lands in our row of h_hist; with `gather` (NCCL) every
// rank's histogram lands in h_hist.
int tick_drain_hits(gub_p2p* p, bool gather, cudaStream_t st) {
  gub_table* t = p->t;
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  if (p->own_streams_used) {  // the steps' queue updates and evaluations ran on other streams: the tick comes after all of them
    cudaStream_t others[3] = {p->last_ingest, p->s_eval, p->s_collect};
    for (cudaStream_t o : others) {
      if (o == st) continue;
      CK(cudaEventRecord(p->ev_fork, o));
      CK(cudaStreamWaitEvent(st, p->ev_fork, 0));
    }
  }
  const size_t row = (size_t)gub::GQ_BINS * 4;
  CK(cudaMemsetAsync(p->g_count, 0, 16, st));
  CK(cudaMemsetAsync(p->g_hist, 0, row, st));
  gub::k_gq_drain<<<t->num_sms, 256, 0, st>>>(p->hits_q->q, hit_stage(p), p->gq_recs, p->g_count + 0, 0u);
  gub::k_gq_hist<<<t->num_sms, 256, 0, st>>>(hit_stage(p), p->gq_recs, p->g_count + 0, p->g_hist);
  CK(cudaGetLastError());
  if (gather) {
    NCK(g_nccl.AllGather(p->g_hist, p->g_hist_all, gub::GQ_BINS, /* ncclUint32 */ 3, p->nccl, st));
    CK(cudaMemcpyAsync(p->h_hist, p->g_hist_all, row * p->world, cudaMemcpyDeviceToHost, st));
  } else {
    CK(cudaMemcpyAsync(p->h_hist + (size_t)p->rank * gub::GQ_BINS, p->g_hist, row, cudaMemcpyDeviceToHost, st));
  }
  return 0;
}

// Our drained records in round order (g_reqs), by a counting sort over the bins; `own` = our histogram (host).
int tick_partition(gub_p2p* p, const uint32_t* own, cudaStream_t st) {
  gub_table* t = p->t;
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  p->h_start[0] = 0;
  for (uint32_t b = 0; b < gub::GQ_BINS; b++) p->h_start[b + 1] = p->h_start[b] + own[b];
  // the histogram has reached the host (and the NCCL all-gather): its device buffer becomes the partition's cursors
  CK(cudaMemcpyAsync(p->g_hist, p->h_start, (size_t)gub::GQ_BINS * 4, cudaMemcpyHostToDevice, st));
  gub::k_gq_partition<<<t->num_sms, 256, 0, st>>>(hit_stage(p), p->gq_recs, p->g_count + 0, p->g_hist, p->g_reqs);
  CK(cudaGetLastError());
  return 0;
}

// Round i, routed: our records of that round -> their owners' mailboxes (plain routing: these records go to the owner).
int tick_round_route(gub_p2p* p, size_t i, cudaStream_t st) {
  gub_table* t = p->t;
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  uint32_t off = 0;
  gub::gq_round_span(p->rounds[i], p->h_start, p->cap, &off, &p->round_n);
  p->epoch++;
  gub_p2p::Route* rt = &p->rt[p->epoch & 1u];
  if (rt->step_done_valid) CK(cudaStreamWaitEvent(st, rt->step_done, 0));
  gub::P2PArgs A;
  p2p_args(p, A);
  return p2p_route(p, rt, A, p->g_reqs + off, p->round_n, nullptr, -1, st);
}
// Owners apply the round's hits with DRAIN_OVER_LIMIT as owner (gubernator.go:510-512).
int tick_phase_b(gub_p2p* p, const gub_clock* clk, cudaStream_t st) {
  gub_table* t = p->t;
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  gub::P2PArgs A;
  p2p_args(p, A);
  if (order_after_last(t, st)) return -1;
  if (p2p_evaluate(p, A, clk, st)) return -1;
  t->last_stream = st; t->last_pending = true;
  if (t->fused && gq_accumulate_segments(p, A, st)) return -1;
  CK(cudaGetLastError());
  return 0;
}
// The owners' answers to our hit records are dropped (sendHits ignores them), but the flags are consumed: epochs stay aligned.
// (Enqueued after EVERY shard's evaluation of the round: on a device shared by several shards a collect spinning ahead of another
// shard's batch kernel would keep that cooperative kernel from ever becoming resident.)
int tick_round_collect(gub_p2p* p, cudaStream_t st) {
  gub_table* t = p->t;
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  gub_p2p::Route* rt = &p->rt[p->epoch & 1u];
  gub::P2PArgs A;
  p2p_args(p, A);
  gub::k_p2p_collect<<<64, 256, 0, st>>>(A, rt->perm, p->round_n, nullptr, p->g_resps);
  CK(cudaEventRecord(rt->step_done, st)); rt->step_done_valid = true;
  CK(cudaGetLastError());
  p->seq += (uint64_t)1 << 32;
  return 0;
}
// Owners re-read every key touched by GLOBAL traffic with Hits = 0 (global.go:243-245) and build the UpdatePeerGlobal items.
int tick_updates(gub_p2p* p, const gub_clock* clk, cudaStream_t st) {
  gub_table* t = p->t;
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  const uint32_t Q = p->gq_recs;
  gub::k_gq_drain<<<t->num_sms, 256, 0, st>>>(p->updates_q->q, p->g_reqs, Q, p->g_count + 1, 1u);
  if (launch_batch(t, p->g_reqs, Q, clk, p->g_resps, st, p->g_count + 1)) return -1;  // (either kernel path; chunked; the count lives on the device)
  gub::k_make_updates<<<(Q + 255) / 256, 256, 0, st>>>(p->g_reqs, p->g_resps, Q, p->g_count + 1, p->g_items, p->g_count + 2);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(p->h_counts, p->g_count, 16, cudaMemcpyDeviceToHost, st));
  return 0;
}

void group_barrier(gub_p2p::LocalGroup* g, uint32_t world) {
  std::unique_lock<std::mutex> lk(g->mu);
  const uint32_t my = g->gen;
  if (++g->arrived == world) { g->arrived = 0; g->gen++; g->cv.notify_all(); }
  else g->cv.wait(lk, [&] { return g->gen != my; });
}

// local_phase_sync for one thread per shard: our stream waits for the piece every other shard has just enqueued.  Reaches both
// barriers whatever happens, so that a failing shard does not leave its peers waiting.
int group_phase_sync(gub_p2p* p, cudaStream_t st) {
  bool ok = cudaSetDevice(p->t->device) == cudaSuccess;
  if (ok && !p->phase_ev) ok = cudaEventCreateWithFlags(&p->phase_ev, cudaEventDisableTiming) == cudaSuccess;
  if (ok) ok = cudaEventRecord(p->phase_ev, st) == cudaSuccess;
  group_barrier(p->group, p->world);
  for (uint32_t q = 0; q < p->world; q++) {
    if (ok && q != p->rank) ok = p->local_peers[q]->phase_ev && cudaStreamWaitEvent(st, p->local_peers[q]->phase_ev, 0) == cudaSuccess;
  }
  group_barrier(p->group, p->world);  // nobody records its event again before every peer has waited on it
  return ok ? 0 : fail("gub_global_tick: ordering the shards' streams failed");
}

// The rounds of one shard, driven by its own thread (with `group`: the shards of this process rendezvous between the pieces).
// rc != 0: an earlier piece failed; nothing more is enqueued, but the rendezvous still happen.
int tick_rounds(gub_p2p* p, const gub_clock* clk, cudaStream_t st, bool group, int rc) {
  for (size_t i = 0; i < p->rounds.size(); i++) {
    if (!rc) rc = tick_round_route(p, i, st);
    if (group && group_phase_sync(p, st)) rc = -1;
    if (!rc) rc = tick_phase_b(p, clk, st);
    if (group && group_phase_sync(p, st)) rc = -1;
    if (!rc) rc = tick_round_collect(p, st);
  }
  return rc;
}

// Installs the items every other shard of this process has made (their g_items, read in place: same device or peer memory).
int tick_install_local(gub_p2p* p, int64_t now_ms, cudaStream_t st, uint64_t* installed) {
  gub_table* t = p->t;
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  p->tick_bytes = 0;
  for (uint32_t r = 0; r < p->world; r++) {
    if (r == p->rank) continue;  // "Exclude ourselves from the update" (global.go:263-265)
    const gub_p2p* q = p->local_peers[r];
    const uint32_t k = std::min(q->h_counts[2], q->gq_recs);
    if (!k) continue;
    gub::k_add_items_pub<<<(k + 255) / 256, 256, 0, st>>>(t->table, t->capacity, q->g_items, k, now_ms, t->counters, t->inv);
    *installed += k;
    p->tick_bytes += (uint64_t)k * sizeof(gub_item);
  }
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(st));  // the peers may overwrite their items at their next tick
  return 0;
}

int tick_install_nccl(gub_p2p* p, int64_t now_ms, cudaStream_t st, uint64_t* installed) {
  gub_table* t = p->t;
  std::lock_guard<std::mutex> lk(t->mu);
  CK(cudaSetDevice(t->device));
  // all-gather: counts first (the host needs them to size the item gathers), then the items in slices of gcap per rank, each padded
  // to the largest count of its slice (g_gather stays gcap x world items)
  std::vector<uint32_t> all(p->world, 0);
  NCK(g_nccl.AllGather(p->g_count + 2, p->g_counts_all, 1, /* ncclUint32 */ 3, p->nccl, st));
  CK(cudaMemcpyAsync(all.data(), p->g_counts_all, p->world * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  auto slice = [&](uint32_t r, uint32_t base) { const uint32_t k = std::min(all[r], p->gq_recs); return k > base ? std::min(k - base, p->gcap) : 0u; };
  p->tick_bytes = 0;
  for (uint32_t base = 0;; base += p->gcap) {
    uint32_t pad = 0;
    for (uint32_t r = 0; r < p->world; r++) pad = std::max(pad, slice(r, base));
    if (!pad) break;
    NCK(g_nccl.AllGather(p->g_items + base, p->g_gather, (size_t)pad * sizeof(gub_item), /* ncclUint8 */ 1, p->nccl, st));
    p->tick_bytes += (uint64_t)pad * sizeof(gub_item) * p->world;
    for (uint32_t r = 0; r < p->world; r++) {
      const uint32_t k = slice(r, base);
      if (r == p->rank || !k) continue;  // "Exclude ourselves from the update" (global.go:263-265)
      gub::k_add_items_pub<<<(k + 255) / 256, 256, 0, st>>>(t->table, t->capacity, p->g_gather + (size_t)r * pad, k, now_ms, t->counters, t->inv);
      *installed += k;
    }
    CK(cudaGetLastError());
  }
  return 0;
}

void tick_stats(gub_p2p* p, uint64_t installed, uint64_t* stats) {
  if (!stats) return;
  stats[0] = std::min(p->h_counts[0], p->gq_recs); stats[1] = std::min(p->h_counts[2], p->gq_recs); stats[2] = installed; stats[3] = p->tick_bytes;
}

}  // namespace

extern "C" {

int gub_global_tick(gub_p2p* p, const gub_clock* clk, int64_t now_ms, void* stream, uint64_t* stats) {
  if (!p || !clk) return fail("gub_global_tick: null argument");
  if (!p->hits_q) return fail("gub_global_tick: gub_p2p_enable_global has not been called");
  if (p->world > 1 && !p->nccl && !p->group) return fail("gub_global_tick: no NCCL communicator (gub_p2p_nccl_init) and the shards are not local to this process");
  cudaStream_t st = (cudaStream_t)stream;
  const bool nccl = p->world > 1 && p->nccl, group = p->world > 1 && !nccl;
  // From here on a shard of a local group reaches every rendezvous even when a piece fails, so that its peers do not wait forever.
  int rc = tick_drain_hits(p, nccl, st);
  if (!rc && (cudaSetDevice(p->t->device) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)) rc = fail("gub_global_tick: the hit histogram did not arrive");
  if (group) group_barrier(p->group, p->world);  // every shard's histogram is on the host
  std::vector<const uint32_t*> rows(p->world);
  for (uint32_t q = 0; q < p->world; q++) rows[q] = (group ? p->local_peers[q]->h_hist : p->h_hist) + (size_t)q * gub::GQ_BINS;
  gub::gq_plan_rounds(rows.data(), p->world, p->cap, p->rounds);
  if (!rc) rc = tick_partition(p, rows[p->rank], st);
  rc = tick_rounds(p, clk, st, group, rc);
  if (!rc) rc = tick_updates(p, clk, st);
  uint64_t installed = 0;
  if (nccl) {
    if (!rc) rc = tick_install_nccl(p, now_ms, st, &installed);
    if (!rc) CK(cudaStreamSynchronize(st));
  } else {
    if (!rc && cudaStreamSynchronize(st) != cudaSuccess) rc = fail("gub_global_tick: the tick failed on the device");  // my items and their count are final
    if (group) {
      group_barrier(p->group, p->world);  // ... and so are everybody else's
      if (!rc) rc = tick_install_local(p, now_ms, st, &installed);
      group_barrier(p->group, p->world);  // nobody still reads my items
    }
  }
  if (rc) return -1;
  tick_stats(p, installed, stats);
  return 0;
}

/* The same for a single host thread driving all the shards of this process (gub_p2p_connect_local): pieces run shard by shard. */
int gub_global_tick_local_all(gub_p2p* const* ps, uint32_t world, const gub_clock* clk, int64_t now_ms, void* const* streams, uint64_t* stats /* world x 4, optional */) {
  if (!ps || !clk || !streams || world == 0) return fail("gub_global_tick_local_all: bad argument");
  for (uint32_t r = 0; r < world; r++) {
    if (!ps[r] || !ps[r]->hits_q || ps[r]->world != world || (world > 1 && !ps[r]->group)) return fail("gub_global_tick_local_all: shards must be local, connected and GLOBAL-enabled");
  }
  for (uint32_t r = 0; r < world; r++) if (tick_drain_hits(ps[r], false, (cudaStream_t)streams[r])) return -1;
  for (uint32_t r = 0; r < world; r++) { CK(cudaSetDevice(ps[r]->t->device)); CK(cudaStreamSynchronize((cudaStream_t)streams[r])); }
  std::vector<const uint32_t*> rows(world);
  for (uint32_t q = 0; q < world; q++) rows[q] = ps[q]->h_hist + (size_t)q * gub::GQ_BINS;
  gub::gq_plan_rounds(rows.data(), world, ps[0]->cap, ps[0]->rounds);
  for (uint32_t r = 0; r < world; r++) {
    ps[r]->rounds = ps[0]->rounds;
    if (tick_partition(ps[r], rows[r], (cudaStream_t)streams[r])) return -1;
  }
  for (size_t i = 0; i < ps[0]->rounds.size(); i++) {
    for (uint32_t r = 0; r < world; r++) if (tick_round_route(ps[r], i, (cudaStream_t)streams[r])) return -1;
    if (local_phase_sync(ps, world, streams)) return -1;
    for (uint32_t r = 0; r < world; r++) if (tick_phase_b(ps[r], clk, (cudaStream_t)streams[r])) return -1;
    if (local_phase_sync(ps, world, streams)) return -1;
    for (uint32_t r = 0; r < world; r++) if (tick_round_collect(ps[r], (cudaStream_t)streams[r])) return -1;
  }
  for (uint32_t r = 0; r < world; r++) if (tick_updates(ps[r], clk, (cudaStream_t)streams[r])) return -1;
  for (uint32_t r = 0; r < world; r++) { CK(cudaSetDevice(ps[r]->t->device)); CK(cudaStreamSynchronize((cudaStream_t)streams[r])); }
  for (uint32_t r = 0; r < world; r++) {
    uint64_t installed = 0;
    if (world > 1 && tick_install_local(ps[r], now_ms, (cudaStream_t)streams[r], &installed)) return -1;
    tick_stats(ps[r], installed, stats ? stats + 4 * r : nullptr);
  }
  return 0;
}

}  // extern "C"
