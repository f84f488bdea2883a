// TEST-ONLY: the batch kernels of gubernator_b200/csrc/gub_kernels.cuh compiled for the CPU on top of tests/cuda_emu.h,
// driven the way gub_api.cu drives them (same scratch sizing, same launch sequence and grid sizes), so that the kernel source
// itself can be checked against the oracle where there is no GPU.  Built by tests/_kernel_emu.py with g++; never part of the
// product library, which has no CPU path.
#define GUB_EMULATE 1
#include "cuda_emu.h"

#include "../gubernator_b200/csrc/gub_kernels.cuh"
#include "../gubernator_b200/csrc/gub_batch.cuh"
#include "../gubernator_b200/csrc/gub_p2p.cuh"
#include "../gubernator_b200/csrc/gub_global.cuh"

#include <cstdlib>
#include <cstring>
#include <vector>

using namespace gub;

namespace {

uint32_t next_pow2(uint64_t v) { uint64_t p = 1; while (p < v) p <<= 1; return (uint32_t)p; }

template <class T> T* zalloc(size_t n) {
  void* p = nullptr;
  if (posix_memalign(&p, 64, std::max<size_t>(n * sizeof(T), 64))) std::abort();
  std::memset(p, 0, std::max<size_t>(n * sizeof(T), 64));
  return static_cast<T*>(p);
}

uint32_t g_finish_cap = 132;

struct EmuTable {  // what gub_create allocates (gub_api.cu), one scratch set
  Slot* table = nullptr;
  uint64_t capacity = 0;
  uint32_t max_batch = 0, aux_entries = 0, max_blocks = 0, pres_words = 0, epoch = 0;
  AuxEntry* aux = nullptr;
  uint32_t *presence = nullptr, *ent = nullptr, *meta = nullptr, *rank = nullptr, *order = nullptr, *mixed_ent = nullptr, *commit_ent = nullptr;
  uint8_t* fragsize = nullptr;
  ulonglong2* commit = nullptr;
  BatchCtr* ctr = nullptr;
  unsigned long long* counters = nullptr;
  // the fused batch kernel (gub_batch.cuh)
  GEntry* gaux = nullptr;
  uint32_t* gpres = nullptr;
  unsigned long long* gfrag = nullptr;
  uint16_t* gmembers = nullptr;
  FCtl* ctl = nullptr;
  OvfItem* ovf = nullptr;
  InvIndex inv{};
  uint32_t grid = 6, sweep_chunk = 0;
};

uint32_t g_fused = 0;  // emu_set_fused(1): the persistent kernel k_batch instead of the four-kernel pipeline (single tables and rings alike)

DevItem to_dev(const gub_item& it) {  // same mapping as gub_api.cu
  DevItem d;
  std::memset(&d, 0, sizeof d);
  d.key = it.key_xxh64 < 2 ? it.key_xxh64 + 2 : it.key_xxh64;
  d.tag = it.key_fnv1 >> 8;
  const bool leaky = it.algorithm == GUB_LEAKY_BUCKET;
  d.flags = F_LIVE | (leaky ? F_LEAKY : 0u) | ((!leaky && it.status == GUB_OVER_LIMIT) ? F_OVER : 0u);
  d.w[0] = (uint64_t)it.limit; d.w[1] = (uint64_t)it.duration;
  if (leaky) std::memcpy(&d.w[2], &it.remaining_f, 8); else d.w[2] = (uint64_t)it.remaining;
  d.w[3] = (uint64_t)it.stamp; d.w[4] = leaky ? (uint64_t)it.burst : 0; d.w[5] = (uint64_t)it.expire_at;
  d.invalid_at = it.invalid_at;
  return d;
}
gub_item from_dev(const DevItem& d) {
  gub_item it;
  std::memset(&it, 0, sizeof it);
  it.key_xxh64 = d.key; it.key_fnv1 = d.tag << 8;
  const bool leaky = (d.flags & F_LEAKY) != 0;
  it.algorithm = leaky ? GUB_LEAKY_BUCKET : GUB_TOKEN_BUCKET;
  it.status = (d.flags & F_OVER) ? GUB_OVER_LIMIT : GUB_UNDER_LIMIT;
  it.limit = (int64_t)d.w[0]; it.duration = (int64_t)d.w[1];
  if (leaky) std::memcpy(&it.remaining_f, &d.w[2], 8); else it.remaining = (int64_t)d.w[2];
  it.stamp = (int64_t)d.w[3]; it.burst = (int64_t)d.w[4]; it.expire_at = (int64_t)d.w[5];
  it.invalid_at = d.invalid_at;
  return it;
}
}  // namespace

extern "C" {

void* emu_create(uint64_t capacity_slots, uint32_t max_batch) {
  EmuTable* t = new EmuTable();
  t->capacity = capacity_slots;
  uint32_t B = max_batch ? max_batch : 65536u;
  if (B < 1024) B = 1024;
  B = (B + 255u) & ~255u;
  t->max_batch = B;
  t->aux_entries = next_pow2((uint64_t)B * 4);
  t->max_blocks = (B / GROUP_THREADS + 127u) & ~127u;
  t->pres_words = t->max_blocks / 32;
  t->table = zalloc<Slot>(capacity_slots);
  t->aux = zalloc<AuxEntry>(t->aux_entries);
  t->presence = zalloc<uint32_t>((size_t)t->aux_entries * t->pres_words);
  t->fragsize = zalloc<uint8_t>((size_t)t->aux_entries * t->max_blocks);
  t->commit = zalloc<ulonglong2>((size_t)t->aux_entries * 6);
  t->commit_ent = zalloc<uint32_t>((size_t)B / 2 + 1);
  t->ent = zalloc<uint32_t>(B); t->meta = zalloc<uint32_t>(B); t->rank = zalloc<uint32_t>(B); t->order = zalloc<uint32_t>(B);
  t->mixed_ent = zalloc<uint32_t>((size_t)B / 2 + 1);
  t->ctr = zalloc<BatchCtr>(2);
  t->counters = zalloc<unsigned long long>(C_COUNT);
  t->gaux = zalloc<GEntry>(FB_AUX_ENTRIES);
  t->gpres = zalloc<uint32_t>((size_t)FB_AUX_ENTRIES * FB_PRES_WORDS);
  t->gfrag = zalloc<unsigned long long>((size_t)FB_AUX_ENTRIES * FB_ROW);
  t->gmembers = zalloc<uint16_t>((size_t)FB_MAX_GRID * FB_THREADS);
  t->ctl = zalloc<FCtl>(1);
  t->ovf = zalloc<OvfItem>(FB_OVF_CAP);
  t->inv.e = zalloc<InvEntry>(65536); t->inv.mask = 65535;
  return t;
}

void emu_destroy(void* tv) {
  EmuTable* t = static_cast<EmuTable*>(tv);
  void* ptrs[] = {t->table, t->aux, t->presence, t->fragsize, t->commit, t->commit_ent, t->ent, t->meta, t->rank, t->order, t->mixed_ent, t->ctr, t->counters,
                  t->gaux, t->gpres, t->gfrag, t->gmembers, t->ctl, t->ovf};
  for (void* p : ptrs) std::free(p);
  delete t;
}

void emu_set_finish_cap(uint32_t blocks) { g_finish_cap = blocks ? blocks : 132u; }
// Test hook: jump to an arbitrary epoch.  A real sequence alternates parity, and k_rank resets the other parity's allocator for the
// next batch; a jump may keep the parity, so hand over clean allocators like the launcher does at the wrap.
void emu_set_epoch(void* tv, uint32_t epoch) {
  EmuTable* t = static_cast<EmuTable*>(tv);
  t->epoch = epoch;
  std::memset(t->ctr, 0, 2 * sizeof(BatchCtr));
}

void emu_set_fused(uint32_t on) { g_fused = on; }
void emu_set_grid(void* tv, uint32_t grid) { static_cast<EmuTable*>(tv)->grid = grid ? grid : 6u; }
void emu_set_sweep(void* tv, uint32_t chunk) { static_cast<EmuTable*>(tv)->sweep_chunk = chunk; }

static void fused_args(EmuTable* t, const gub_clock* clk, FArgs& A) {
  std::memset(&A, 0, sizeof A);
  A.table = t->table; A.capacity = t->capacity; A.aux = t->gaux; A.presence = t->gpres; A.fragrow = t->gfrag; A.members = t->gmembers;
  A.ctl = t->ctl; A.ovf = t->ovf; A.counters = t->counters; A.sweep_chunk = t->sweep_chunk; A.inv = t->inv; A.clk = *clk;
}

// launch_fused of gub_api.cu: one cooperative launch of k_batch over the batch's segments (here with a small grid: every emulated
// CTA costs 512 fibers; the kernel takes any grid size, more rounds make up for it).
static int submit_fused(EmuTable* t, const FSeg* segs, uint32_t nseg, uint32_t flag_epoch, const gub_clock* clk, unsigned long long* const* resp_flags = nullptr,
                        uint32_t n_resp_flags = 0) {
  FArgs A;
  fused_args(t, clk, A);
  for (uint32_t s = 0; s < nseg; s++) A.seg[s] = segs[s];
  A.nseg = nseg; A.flag_epoch = flag_epoch;
  for (uint32_t k = 0; k < n_resp_flags; k++) A.resp_flag[k] = resp_flags[k];
  A.n_resp_flags = n_resp_flags;
  emu::launch_coop(k_batch, t->grid, (unsigned)FB_THREADS, sizeof(FSmem), A);
  return 0;
}

// launch_batch / launch_chunk / launch_finish of gub_api.cu, minus streams.  n_dev != nullptr: the batch size is *n_dev (<= n), as in
// gub_submit_device_n.
struct EmuSegs {  // ring mode (SegDesc of gub_api.cu)
  uint32_t nseg = 0;
  const uint32_t* seg_off = nullptr;
  const gub_req* reqs[MAX_SHARDS] = {};
  gub_resp* out[MAX_SHARDS] = {};
};

// launch_chunk of gub_api.cu, minus streams
static void submit_chunk(EmuTable* t, const gub_req* reqs, uint32_t m, const uint32_t* n_dev, uint32_t n_off, const gub_clock* clk, gub_resp* out, const EmuSegs* seg) {
  if (t->epoch >= 65535u) { std::memset(t->aux, 0, (size_t)t->aux_entries * sizeof(AuxEntry)); std::memset(t->ctr, 0, 2 * sizeof(BatchCtr)); t->epoch = 0; }
  t->epoch++;
  BatchArgs A;
  std::memset(&A, 0, sizeof A);
  if (seg) {
    A.nseg = seg->nseg; A.seg_off = seg->seg_off;
    for (uint32_t k = 0; k < seg->nseg; k++) { A.seg_reqs[k] = seg->reqs[k]; A.seg_out[k] = seg->out[k]; }
  }
  A.table = t->table; A.capacity = t->capacity; A.reqs = reqs; A.out = out; A.n = m; A.n_dev = n_dev; A.n_off = n_off; A.epoch = t->epoch;
  A.aux = t->aux; A.aux_mask = t->aux_entries - 1; A.presence = t->presence; A.fragsize = t->fragsize;
  A.pres_words = t->pres_words; A.max_blocks = t->max_blocks; A.ent = t->ent; A.meta = t->meta; A.rank = t->rank;
  A.commit = t->commit; A.order = t->order; A.mixed_ent = t->mixed_ent; A.ctr = t->ctr;
  A.counters = t->counters; A.ovf = t->ovf; A.ovf_count = &t->ctl->ovf_count; A.inv = t->inv;
  A.clk = *clk;
  const uint32_t blocks = (m + 255) / 256;
  const uint32_t fin = std::min<uint32_t>(g_finish_cap, std::max<uint32_t>(1u, m / 2));  // gub_api.cu caps the grid at the SM count (132 on an H100 SXM)
  if (seg) {
    emu::launch(k_group<true>, blocks, GROUP_THREADS, A);
    emu::launch(k_rank<true>, blocks, GROUP_THREADS, A);
    emu::launch(k_eval<true>, blocks, GROUP_THREADS, A);
    emu::launch(k_finish<true>, fin, MIXED_THREADS, A);
  } else {
    emu::launch(k_group<false>, blocks, GROUP_THREADS, A);
    emu::launch(k_rank<false>, blocks, GROUP_THREADS, A);
    emu::launch(k_eval<false>, blocks, GROUP_THREADS, A);
    emu::launch(k_finish<false>, fin, MIXED_THREADS, A);
  }
}

// launch_batch of gub_api.cu.  n_dev != nullptr: the batch size is *n_dev (<= n), as in gub_submit_device_n.
static int submit_impl(EmuTable* t, const gub_req* reqs, size_t n, const uint32_t* n_dev, const gub_clock* clk, gub_resp* out) {
  if (g_fused) {
    FSeg sg;
    std::memset(&sg, 0, sizeof sg);
    sg.reqs = reqs; sg.out = out; sg.n = (uint32_t)n; sg.n_dev = n_dev;
    return submit_fused(t, &sg, 1, 0, clk);
  }
  for (size_t off = 0; off < n; off += t->max_batch) {
    const uint32_t m = (uint32_t)std::min<size_t>(t->max_batch, n - off);
    submit_chunk(t, reqs + off, m, n_dev, (uint32_t)off, clk, out + off, nullptr);
  }
  return 0;
}

int emu_submit(void* tv, const gub_req* reqs, size_t n, const gub_clock* clk, gub_resp* out) {
  return submit_impl(static_cast<EmuTable*>(tv), reqs, n, nullptr, clk, out);
}

int emu_submit_compact(void* tv, const gub_creq* creqs, size_t n, const gub_params* params, size_t n_params, int64_t created_base, const gub_clock* clk,
                       gub_resp* out) {
  std::vector<gub_req> reqs(std::max<size_t>(n, 1));
  if (n) {
    if (n_params <= INLINE_PARAMS) {
      InlineParams P;
      std::memset(&P, 0, sizeof P);
      std::memcpy(&P, params, n_params * sizeof(gub_params));
      emu::launch(k_expand_inline, (unsigned)((n + 255) / 256), 256u, creqs, (uint32_t)n, P, (uint32_t)n_params, created_base, reqs.data());
    } else {
      emu::launch(k_expand, (unsigned)((n + 255) / 256), 256u, creqs, (uint32_t)n, params, (uint32_t)n_params, created_base, reqs.data());
    }
  }
  return emu_submit(tv, reqs.data(), n, clk, out);
}

void emu_counters(void* tv, unsigned long long* out /* C_COUNT */) { std::memcpy(out, static_cast<EmuTable*>(tv)->counters, C_COUNT * sizeof(unsigned long long)); }
int emu_counter_count(void) { return C_COUNT; }

// Live items, as gub_scan reports them (k_scan + the DevItem -> gub_item mapping of gub_api.cu).
uint64_t emu_scan(void* tv, gub_item* out, uint64_t cap) {
  EmuTable* t = static_cast<EmuTable*>(tv);
  std::vector<DevItem> dev(std::max<uint64_t>(cap, 1));
  unsigned long long n = 0;
  emu::launch(k_scan, 4u, 256u, (const Slot*)t->table, t->capacity, dev.data(), (unsigned long long)cap, &n, t->inv);
  const uint64_t m = std::min<uint64_t>(n, cap);
  for (uint64_t i = 0; i < m; i++) out[i] = from_dev(dev[i]);
  return n;
}

// gub_add_items / gub_get_items of gub_api.cu (k_add_items / k_get_items and the gub_item <-> DevItem mapping); duplicate keys in
// one call are not merged here, callers pass distinct keys.
uint32_t emu_add_items(void* tv, const gub_item* items, uint32_t n) {
  EmuTable* t = static_cast<EmuTable*>(tv);
  std::vector<DevItem> dev;
  for (uint32_t i = 0; i < n; i++)
    if (items[i].algorithm == GUB_TOKEN_BUCKET || items[i].algorithm == GUB_LEAKY_BUCKET) dev.push_back(to_dev(items[i]));
  uint32_t failed = 0;
  if (!dev.empty())
    emu::launch(k_add_items, (unsigned)((dev.size() + 255) / 256), 256u, t->table, t->capacity, (const DevItem*)dev.data(), (uint32_t)dev.size(),
                t->counters, &failed, t->inv);
  return failed;
}
void emu_get_items(void* tv, const uint64_t* kx, const uint64_t* kf, uint32_t n, int64_t now_ms, gub_item* out, uint8_t* found) {
  EmuTable* t = static_cast<EmuTable*>(tv);
  std::vector<DevItem> host(std::max<uint32_t>(n, 1));
  if (n) emu::launch(k_get_items, (n + 255) / 256, 256u, (const Slot*)t->table, t->capacity, kx, kf, n, now_ms, host.data(), found, t->inv);
  for (uint32_t i = 0; i < n; i++) { out[i] = from_dev(host[i]); out[i].key_xxh64 = kx[i]; out[i].key_fnv1 = kf[i]; }
}

// gub_probe_random_access's kernel (the timing around it is host code): the table must come out unchanged.
void emu_random_rmw(void* tv, uint64_t accesses) {
  EmuTable* t = static_cast<EmuTable*>(tv);
  emu::launch(k_random_rmw, 4u, 256u, t->table, t->capacity, accesses, (uint64_t)12345, (uint64_t)0);
}

uint64_t emu_sweep(void* tv, int64_t now_ms) {
  EmuTable* t = static_cast<EmuTable*>(tv);
  unsigned long long removed = 0;
  emu::launch(k_sweep, 4u, 256u, t->table, (uint64_t)0, t->capacity, now_ms, &removed);
  return removed;
}
// maybe_sweep of gub_api.cu: one slice [lo, hi) of the table (the pipeline's incremental sweep, between batches)
uint64_t emu_sweep_range(void* tv, uint64_t lo, uint64_t hi, int64_t now_ms) {
  EmuTable* t = static_cast<EmuTable*>(tv);
  unsigned long long removed = 0;
  emu::launch(k_sweep, 4u, 256u, t->table, lo, std::min<uint64_t>(hi, t->capacity), now_ms, &removed);
  return removed;
}

// k_hash_keys: XXH64 + FNV-1 over packed keys.
void emu_hash_keys(const uint8_t* bytes, const uint64_t* offsets, uint32_t n, uint64_t* xxh_out, uint64_t* fnv_out) {
  if (n) emu::launch(k_hash_keys, (n + 255) / 256, 256u, bytes, offsets, n, xxh_out, fnv_out, (gub_req*)nullptr);
}

// gub_route_device: owner of every request by the ring + stable partition by owner (k_route_count / k_route_scan / k_route_scatter),
// and k_unroute for the way back.
void emu_route(const gub_req* reqs, uint32_t n, const uint64_t* pts, const int32_t* peers, uint32_t npts, uint32_t nshards, gub_req* out_reqs, uint32_t* perm,
               uint32_t* counts, uint8_t* owner) {
  if (!n) { std::memset(counts, 0, nshards * 4); return; }
  const uint32_t ntiles = (n + ROUTE_TILE - 1) / ROUTE_TILE;
  std::vector<uint32_t> tile_counts((size_t)nshards * ntiles + 1);
  emu::launch(k_route_count, ntiles, 256u, reqs, n, pts, peers, npts, nshards, owner, tile_counts.data(), ntiles, -1, (uint8_t*)nullptr);
  emu::launch(k_route_scan, 1u, 1024u, tile_counts.data(), nshards * ntiles, nshards, ntiles, counts);
  emu::launch(k_route_scatter, ntiles, 256u, reqs, n, (const uint8_t*)owner, (const uint32_t*)tile_counts.data(), ntiles, nshards, out_reqs, perm);
}
void emu_unroute(const gub_resp* in, const uint32_t* perm, uint32_t n, gub_resp* out) {
  if (n) emu::launch(k_unroute, (n + 255) / 256, 256u, in, perm, n, out);
}

// ---- GLOBAL queues (gub_gq_*): claim + fill per batch, drain at a tick -----------------------------------------------------------
struct EmuGq { Gq q; uint32_t capacity; };

void* emu_gq_create(uint32_t capacity, uint32_t keep_latest) {
  EmuGq* g = new EmuGq();
  g->capacity = next_pow2(capacity);
  g->q.slots = zalloc<gub_req>(g->capacity);
  g->q.seq = zalloc<unsigned long long>(g->capacity);
  g->q.count = zalloc<unsigned long long>(1);
  g->q.dropped = zalloc<unsigned long long>(1);
  g->q.capacity_mask = g->capacity - 1;
  g->q.mode = keep_latest ? GQ_KEEP_LAST : GQ_KEEP_FIRST;
  return g;
}
// owner == nullptr: the updates queue of an owner (every GLOBAL request with hits counts); else the hits queue of shard `self`
void emu_gq_accumulate(void* gv, const gub_req* reqs, uint32_t n, const uint8_t* owner, uint32_t self, unsigned long long seq_base) {
  EmuGq* g = static_cast<EmuGq*>(gv);
  if (!n) return;
  std::vector<uint32_t> slot_of(n);
  emu::launch(k_gq_claim, (n + 255) / 256, 256u, g->q, reqs, n, (const uint32_t*)nullptr, owner, self, owner ? 1u : 0u, seq_base, slot_of.data());
  emu::launch(k_gq_fill, (n + 255) / 256, 256u, g->q, reqs, n, (const uint32_t*)nullptr, seq_base, (const uint32_t*)slot_of.data());
}
uint32_t emu_gq_drain(void* gv, gub_req* out, uint32_t cap, uint32_t as_status_query) {
  EmuGq* g = static_cast<EmuGq*>(gv);
  uint32_t count = 0;
  emu::launch(k_gq_drain, 4u, 256u, g->q, out, cap, &count, as_status_query);
  return count;
}
uint32_t emu_make_updates(const gub_req* queries, const gub_resp* resps, uint32_t n, gub_item* out) {
  uint32_t count = 0;
  if (n) emu::launch(k_make_updates, (n + 255) / 256, 256u, queries, resps, n, (const uint32_t*)nullptr, out, &count);
  return count;
}

// UpdatePeerGlobals: install UpdatePeerGlobal items as replicas (k_add_items_pub: gub_add_items_device / the tick's install phase)
void emu_install_updates(void* tv, const gub_item* items, uint32_t n, int64_t now_ms) {
  EmuTable* t = static_cast<EmuTable*>(tv);
  if (n) emu::launch(k_add_items_pub, (n + 255) / 256, 256u, t->table, t->capacity, items, n, now_ms, t->counters, t->inv);
}

// ---- gub_p2p_step for W shards living in one process, phase by phase: every shard scatters, then every shard gathers,
// evaluates and returns responses, then every shard un-routes.  The flag waits of the real kernels find their flags already
// published, so the spin loops fall through; what is exercised is the mailbox indexing, the (source rank, source index) order at
// the owner, the device-side batch size and the way back.
struct EmuP2P {
  uint32_t world = 0, cap = 0, epoch = 0;
  std::vector<EmuTable*> tabs;
  std::vector<uint64_t> pts; std::vector<int32_t> peers; std::vector<uint16_t> lut;
  struct Rank {
    P2PView view;
    unsigned long long* tile_agg;
    uint32_t *error, *counts, *perm, *ticket, *seg_off;
    uint8_t* true_owner;
  };
  std::vector<Rank> ranks;
};

void* emu_p2p_create(uint32_t world, uint32_t cap, uint64_t capacity_slots, uint32_t max_batch, const uint64_t* pts, const int32_t* peers, uint32_t npts) {
  EmuP2P* p = new EmuP2P();
  p->world = world; p->cap = cap;
  p->pts.assign(pts, pts + npts); p->peers.assign(peers, peers + npts);
  p->lut.resize(65536);
  size_t k = 0;
  for (uint32_t b = 0; b < 65536; b++) {  // ensure_ring of gub_api.cu
    const uint64_t lo = (uint64_t)b << 48;
    while (k < npts && pts[k] < lo) k++;
    p->lut[b] = (uint16_t)k;
  }
  for (uint32_t r = 0; r < world; r++) {
    p->tabs.push_back(static_cast<EmuTable*>(emu_create(capacity_slots, max_batch)));
    EmuP2P::Rank k2;
    k2.view.req_mb = zalloc<gub_req>((size_t)2 * world * cap);
    k2.view.resp_mb = zalloc<gub_resp>((size_t)2 * world * cap);
    k2.view.req_flag = zalloc<unsigned long long>((size_t)2 * world);
    k2.view.resp_flag = zalloc<unsigned long long>((size_t)2 * world);
    k2.tile_agg = zalloc<unsigned long long>(((size_t)cap / RT_THREADS + 1) * MAX_SHARDS);
    k2.error = zalloc<uint32_t>(1); k2.counts = zalloc<uint32_t>(MAX_SHARDS); k2.perm = zalloc<uint32_t>(cap); k2.ticket = zalloc<uint32_t>(2);
    k2.true_owner = zalloc<uint8_t>(cap); k2.seg_off = zalloc<uint32_t>(MAX_SHARDS + 1);
    p->ranks.push_back(k2);
  }
  return p;
}

void* emu_p2p_table(void* pv, uint32_t rank) { return static_cast<EmuP2P*>(pv)->tabs[rank]; }

// gub_p2p_step_streams of gub_api.cu for W shards in one process, phase by phase: every shard routes (k_p2p_route), then every
// shard evaluates straight out of its mailboxes (k_batch over W flagged segments, responses into the sources' mailboxes), then
// every shard collects.  self_global != 0: GLOBAL requests a shard does not own stay with it (rewritten).
int emu_p2p_step(void* pv, const gub_req* const* reqs, const uint32_t* n, const gub_clock* clk, gub_resp* const* outs, uint32_t self_global,
                 uint8_t* const* true_owner_out) {
  EmuP2P* p = static_cast<EmuP2P*>(pv);
  p->epoch++;
  std::vector<P2PArgs> args(p->world);
  for (uint32_t r = 0; r < p->world; r++) {
    P2PArgs& A = args[r];
    for (uint32_t q = 0; q < p->world; q++) A.peers[q] = p->ranks[q].view;
    A.world = p->world; A.rank = r; A.cap = p->cap; A.epoch = p->epoch; A.done_ctr = nullptr; A.error = p->ranks[r].error;
  }
  for (uint32_t r = 0; r < p->world; r++) {  // phase 1
    EmuP2P::Rank& k = p->ranks[r];
    RouteArgs R;
    R.P = args[r]; R.reqs = reqs[r]; R.n = n[r]; R.n_dev = nullptr; R.pts = p->pts.data(); R.pt_peer = p->peers.data(); R.lut = p->lut.data();
    R.npts = (uint32_t)p->pts.size(); R.self_global = self_global ? (int32_t)r : -1; R.true_owner = self_global ? k.true_owner : nullptr;
    R.tile_agg = k.tile_agg; R.counts = k.counts; R.perm = k.perm; R.ticket = k.ticket;
    emu::launch(k_p2p_route, std::max<uint32_t>(1u, (n[r] + RT_THREADS - 1) / RT_THREADS), (unsigned)RT_THREADS, R);
    if (self_global && true_owner_out && n[r]) std::memcpy(true_owner_out[r], k.true_owner, n[r]);
  }
  const uint32_t par = p->epoch & 1u;
  for (uint32_t r = 0; r < p->world; r++) {  // phase 2
    if (!g_fused) {  // p2p_evaluate's default: k_seg_wait, the pipeline in ring mode (as many passes as world x cap takes), k_seg_publish
      EmuTable* t = p->tabs[r];
      EmuSegs sd;
      sd.nseg = p->world; sd.seg_off = p->ranks[r].seg_off;
      for (uint32_t s = 0; s < p->world; s++) {
        sd.reqs[s] = args[r].peers[r].req_mb + ((size_t)par * p->world + s) * p->cap;
        sd.out[s] = args[r].peers[s].resp_mb + ((size_t)par * p->world + r) * p->cap;
      }
      emu::launch(k_seg_wait, 1u, 32u, args[r], p->ranks[r].seg_off);
      const uint64_t total = (uint64_t)p->world * p->cap;
      for (uint64_t off = 0; off < total; off += t->max_batch) {
        const uint32_t m = (uint32_t)std::min<uint64_t>(t->max_batch, total - off);
        submit_chunk(t, nullptr, m, p->ranks[r].seg_off + p->world, (uint32_t)off, clk, nullptr, &sd);
      }
      emu::launch(k_seg_publish, 1u, 32u, args[r]);
      continue;
    }
    FSeg segs[MAX_SHARDS];
    unsigned long long* rflags[MAX_SHARDS];
    std::memset(segs, 0, sizeof segs);
    for (uint32_t s = 0; s < p->world; s++) {
      segs[s].reqs = args[r].peers[r].req_mb + ((size_t)par * p->world + s) * p->cap;
      segs[s].flag = &args[r].peers[r].req_flag[(size_t)par * p->world + s];
      segs[s].out = args[r].peers[s].resp_mb + ((size_t)par * p->world + r) * p->cap;
      segs[s].n = p->cap;
      rflags[s] = &args[r].peers[s].resp_flag[(size_t)par * p->world + r];
    }
    submit_fused(p->tabs[r], segs, p->world, p->epoch, clk, rflags, p->world);
  }
  int err = 0;
  for (uint32_t r = 0; r < p->world; r++) {  // phase 3
    EmuP2P::Rank& k = p->ranks[r];
    emu::launch(k_p2p_collect, 4u, 256u, args[r], (const uint32_t*)k.perm, n[r], (const uint32_t*)nullptr, outs[r]);
    err |= (int)*k.error | (int)p->tabs[r]->ctl->error;
  }
  return err;
}

}  // extern "C"
