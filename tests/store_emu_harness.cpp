// TEST-ONLY: the CPU emulation of the kernels (tests/kernel_emu_harness.cpp, included whole) plus the Store plugin's pre- and post-pass
// (gubernator_b200/csrc/gub_store.cuh), driven like store_before / launch_batch / store_after of gub_api.cu on the pipeline path.
// Built by tests/_store_emu.py with g++; never part of the product library.
#include "kernel_emu_harness.cpp"

#include "../gubernator_b200/csrc/gub_store.cuh"

#include <map>

namespace {

struct EmuStore {
  StoreKey* keys;
  uint32_t key_entries, epoch;
  uint32_t *kent, *blk, failed;
  StoreState* bstate;
  uint8_t* sel;
  gub_store_rec *sparse, *miss;
  uint32_t miss_count;
};
std::map<void*, EmuStore> g_store;

DevItem item_dev(const gub_item& it) {  // to_dev of gub_api.cu
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

}  // namespace

extern "C" {

void* emu_store_create(uint64_t capacity_slots, uint32_t max_batch) {
  EmuTable* t = static_cast<EmuTable*>(emu_create(capacity_slots, max_batch));
  EmuStore s;
  std::memset(&s, 0, sizeof s);
  s.key_entries = next_pow2((uint64_t)t->max_batch * 2);
  s.keys = zalloc<StoreKey>(s.key_entries);
  s.kent = zalloc<uint32_t>(t->max_batch);
  s.blk = zalloc<uint32_t>(t->max_batch / STORE_THREADS + 1);
  s.bstate = zalloc<StoreState>(t->max_batch);
  s.sel = zalloc<uint8_t>(t->max_batch);
  s.sparse = zalloc<gub_store_rec>(t->max_batch);
  s.miss = zalloc<gub_store_rec>(t->max_batch);
  g_store[t] = s;
  return t;
}

void emu_store_destroy(void* tv) {
  const EmuStore s = g_store[tv];
  void* ptrs[] = {s.keys, s.kent, s.blk, s.bstate, s.sel, s.sparse, s.miss};
  for (void* p : ptrs) std::free(p);
  g_store.erase(tv);
  emu_destroy(tv);
}

void emu_store_set_epoch(void* tv, uint32_t epoch) { g_store[tv].epoch = epoch; }
uint32_t emu_store_epoch(void* tv) { return g_store[tv].epoch; }
uint32_t emu_ovf_count(void* tv) { return static_cast<EmuTable*>(tv)->ctl->ovf_count; }

// One batch (n <= max_batch) with a Store: returns 0, or the callback's non-zero result (nothing evaluated), or -1 (table full for a
// loaded item).
int emu_store_submit(void* tv, const gub_req* reqs, size_t n, const gub_clock* clk, gub_store_get_fn get, void* user, gub_resp* out,
                     gub_store_rec* changes, uint32_t* n_changes) {
  EmuTable* t = static_cast<EmuTable*>(tv);
  EmuStore& ss = g_store[tv];
  if (n == 0) { *n_changes = 0; return 0; }
  if (ss.epoch >= 0xFFFFFFFFu) { std::memset(ss.keys, 0, (size_t)ss.key_entries * sizeof(StoreKey)); ss.epoch = 0; }
  ss.epoch++;
  StoreArgs S;
  std::memset(&S, 0, sizeof S);
  S.reqs = reqs; S.n = (uint32_t)n; S.epoch = ss.epoch; S.keys = ss.keys; S.key_mask = ss.key_entries - 1; S.kent = ss.kent; S.bstate = ss.bstate;
  S.sel = ss.sel; S.sparse = ss.sparse; S.blk = ss.blk; S.table = t->table; S.capacity = t->capacity; S.ovf = t->ovf;
  S.ovf_count = &t->ctl->ovf_count; S.inv = t->inv; S.now_ms = clk->now_ms; S.want_misses = get ? 1u : 0u;
  const unsigned blocks = (unsigned)((n + STORE_THREADS - 1) / STORE_THREADS);
  emu::launch(k_store_keys, blocks, (unsigned)STORE_THREADS, S);
  emu::launch(k_store_before, blocks, (unsigned)STORE_THREADS, S);
  if (get) {
    emu::launch(k_store_compact, blocks, (unsigned)STORE_THREADS, (const uint8_t*)ss.sel, (const gub_store_rec*)ss.sparse, (const uint32_t*)ss.blk,
                (uint32_t)n, ss.miss, &ss.miss_count);
    const uint32_t m = ss.miss_count;
    if (m) {
      std::vector<uint64_t> keys((size_t)m * 2);
      for (uint32_t k = 0; k < m; k++) { keys[2 * k] = ss.miss[k].item.key_xxh64; keys[2 * k + 1] = ss.miss[k].item.key_fnv1; }
      const int rc = get(user, ss.miss, m);
      if (rc) return rc;
      std::vector<uint4> loaded;
      std::vector<DevItem> items;
      for (uint32_t k = 0; k < m; k++) {
        gub_store_rec& r = ss.miss[k];
        if (!(r.flags & GUB_STORE_FOUND)) continue;
        r.item.key_xxh64 = keys[2 * k]; r.item.key_fnv1 = keys[2 * k + 1];
        loaded.push_back(make_uint4(r.first, r.item.expire_at >= clk->now_ms ? S_EXISTED : 0u, (uint32_t)r.item.algorithm, 0u));
        if (r.item.algorithm == GUB_TOKEN_BUCKET || r.item.algorithm == GUB_LEAKY_BUCKET) items.push_back(item_dev(r.item));
      }
      if (!items.empty()) {
        gub_clock dclk;
        std::memset(&dclk, 0, sizeof dclk);
        dclk.now_ms = INT64_MIN;  // drain_pending of gub_api.cu
        FArgs A;
        fused_args(t, &dclk, A);
        emu::launch(k_drain_overflow, 1u, 32u, A);
        ss.failed = 0;
        emu::launch(k_add_items, (unsigned)((items.size() + 255) / 256), 256u, t->table, t->capacity, (const DevItem*)items.data(),
                    (uint32_t)items.size(), t->counters, &ss.failed, t->inv);
      }
      if (!loaded.empty())
        emu::launch(k_store_loaded, (unsigned)((loaded.size() + STORE_THREADS - 1) / STORE_THREADS), (unsigned)STORE_THREADS, (const uint4*)loaded.data(),
                    (uint32_t)loaded.size(), ss.bstate);
      if (ss.failed) return -1;
    }
  }
  submit_impl(t, reqs, n, nullptr, clk, out);
  S.out = out;
  emu::launch(k_store_after, blocks, (unsigned)STORE_THREADS, S);
  emu::launch(k_store_compact, blocks, (unsigned)STORE_THREADS, (const uint8_t*)ss.sel, (const gub_store_rec*)ss.sparse, (const uint32_t*)ss.blk,
              (uint32_t)n, changes, n_changes);
  return 0;
}

}  // extern "C"
