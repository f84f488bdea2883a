// TEST-ONLY: the C ABI of include/gubernator_b200.h implemented over the CPU emulation of the kernels (tests/cuda_emu.h), linked with
// the REAL host layer (gubernator_b200/csrc/host_v1.cpp, host_util.cpp) into tests/libgub_emulated_test.so, so that the host logic —
// V1Instance.GetRateLimits validation and error strings, the RPC aggregator's threads, the Store plugin's call sequences — runs in
// the CPU suite against the same kernel source the GPU runs.  It is loaded only by tests/host_layer_emulated_cases.py (which
// points the Python binding at it explicitly); the product library has no CPU path and nothing in the package refers to this file.
//
// Emulated: table lifecycle, gub_submit*, items / scan / size / sweep / counters, pinned-memory helpers (plain malloc).  Everything
// that takes device pointers or peers is a stub that fails with "not emulated".
#include "kernel_emu_harness.cpp"

#include <mutex>
#include <string>
#include <unordered_map>

struct gub_table { EmuTable* e = nullptr; };

namespace {
std::mutex g_emu_mu;  // the fiber scheduler has one global state: one emulated launch at a time
thread_local std::string g_err;
int fail(const std::string& m) { g_err = m; return -1; }

}  // namespace

extern "C" {

const char* gub_last_error(void) { return g_err.c_str(); }
int gub_abi_version(void) { return GUB_ABI_VERSION; }

int gub_create(const gub_config* cfg, gub_table** out) {
  if (!cfg || !out) return fail("gub_create: null argument");
  *out = nullptr;
  if (cfg->capacity_slots < 64) return fail("gub_create: capacity_slots must be >= 64");
  uint32_t mb = cfg->max_batch ? cfg->max_batch : 65536u;
  if (mb > 262144u) mb = 262144u;
  gub_table* t = new gub_table();
  t->e = static_cast<EmuTable*>(emu_create(cfg->capacity_slots, mb));
  *out = t;
  return 0;
}
void gub_destroy(gub_table* t) {
  if (!t) return;
  emu_destroy(t->e);
  delete t;
}

int gub_submit(gub_table* t, const gub_req* reqs, size_t n, const gub_clock* clk, gub_resp* out) {
  if (!t || !clk || (n && (!reqs || !out))) return fail("gub_submit: null argument");
  std::lock_guard<std::mutex> lk(g_emu_mu);
  return submit_impl(t->e, reqs, n, nullptr, clk, out);
}
int gub_submit_compact(gub_table* t, const gub_creq* reqs, size_t n, const gub_params* params, size_t n_params, int64_t created_base, const gub_clock* clk,
                       gub_resp* out) {
  if (!t || !clk || (n && (!reqs || !out || !params))) return fail("gub_submit_compact: null argument");
  std::lock_guard<std::mutex> lk(g_emu_mu);
  return emu_submit_compact(t->e, reqs, n, params, n_params, created_base, clk, out);
}
// the pipelined entries complete at once: ticket 0, nothing to wait for
int gub_pipeline_depth(gub_table*) { return 1; }
int gub_submit_async(gub_table* t, const gub_req* reqs, size_t n, const gub_clock* clk, gub_resp* out, int* ticket) {
  if (ticket) *ticket = 0;
  return gub_submit(t, reqs, n, clk, out);
}
int gub_submit_compact_async(gub_table* t, const gub_creq* reqs, size_t n, const gub_params* params, size_t n_params, int64_t created_base,
                             const gub_clock* clk, gub_resp* out, int* ticket) {
  if (ticket) *ticket = 0;
  return gub_submit_compact(t, reqs, n, params, n_params, created_base, clk, out);
}
int gub_wait(gub_table*, int) { return 0; }
void* gub_host_alloc(size_t bytes) { return std::malloc(bytes ? bytes : 1); }
void gub_host_free(void* p) { std::free(p); }

int gub_add_items(gub_table* t, const gub_item* items, size_t n) {
  if (!t || (n && !items)) return fail("gub_add_items: null argument");
  if (n == 0) return 0;
  std::lock_guard<std::mutex> lk(g_emu_mu);
  std::vector<DevItem> dev;  // last one wins for duplicate keys, like gub_api.cu
  std::unordered_map<uint64_t, size_t> seen;
  for (size_t i = 0; i < n; i++) {
    if (items[i].algorithm != GUB_TOKEN_BUCKET && items[i].algorithm != GUB_LEAKY_BUCKET) continue;
    const DevItem d = to_dev(items[i]);
    const uint64_t h = d.key ^ (d.tag * 0x9E3779B97F4A7C15ULL);
    auto it = seen.find(h);
    if (it != seen.end() && dev[it->second].key == d.key && dev[it->second].tag == d.tag) dev[it->second] = d;
    else { seen[h] = dev.size(); dev.push_back(d); }
  }
  if (dev.empty()) return 0;
  uint32_t failed = 0;
  emu::launch(k_add_items, (unsigned)((dev.size() + 255) / 256), 256u, t->e->table, t->e->capacity, (const DevItem*)dev.data(), (uint32_t)dev.size(), t->e->counters,
              &failed, t->e->inv);
  if (failed) return fail("gub_add_items: table full for " + std::to_string(failed) + " items");
  return 0;
}

int gub_get_items(gub_table* t, const uint64_t* kx, const uint64_t* kf, size_t n, int64_t now_ms, gub_item* out, uint8_t* found) {
  if (!t || (n && (!kx || !kf || !out || !found))) return fail("gub_get_items: null argument");
  if (n == 0) return 0;
  std::lock_guard<std::mutex> lk(g_emu_mu);
  std::vector<DevItem> host(n);
  emu::launch(k_get_items, (unsigned)((n + 255) / 256), 256u, (const Slot*)t->e->table, t->e->capacity, kx, kf, (uint32_t)n, now_ms, host.data(), found, t->e->inv);
  for (size_t i = 0; i < n; i++) { out[i] = from_dev(host[i]); out[i].key_xxh64 = kx[i]; out[i].key_fnv1 = kf[i]; }
  return 0;
}

int gub_scan(gub_table* t, gub_item* out, size_t cap, size_t* n_out) {
  if (!t || !n_out || (cap && !out)) return fail("gub_scan: null argument");
  std::lock_guard<std::mutex> lk(g_emu_mu);
  std::vector<DevItem> dev(std::max<size_t>(cap, 1));
  unsigned long long total = 0;
  emu::launch(k_scan, 4u, 256u, (const Slot*)t->e->table, t->e->capacity, dev.data(), (unsigned long long)cap, &total, t->e->inv);
  for (size_t i = 0; i < std::min<size_t>(cap, (size_t)total); i++) out[i] = from_dev(dev[i]);
  *n_out = (size_t)total;
  return 0;
}
int gub_size(gub_table* t, size_t* n_out) { return gub_scan(t, nullptr, 0, n_out); }

int gub_sweep(gub_table* t, int64_t now_ms, size_t* removed) {
  if (!t) return fail("gub_sweep: null argument");
  std::lock_guard<std::mutex> lk(g_emu_mu);
  const uint64_t r = emu_sweep(t->e, now_ms);
  if (removed) *removed = (size_t)r;
  return 0;
}

int gub_get_counters(gub_table* t, gub_counters* out) {
  if (!t || !out) return fail("gub_get_counters: null argument");
  std::lock_guard<std::mutex> lk(g_emu_mu);
  const unsigned long long* c = t->e->counters;
  out->over_limit = c[C_OVER]; out->cache_hit = c[C_HIT]; out->cache_miss = c[C_MISS]; out->inserts = c[C_INSERTS]; out->table_full = c[C_FULL];
  out->requests = c[C_REQUESTS]; out->batches = c[C_BATCHES]; out->dup_groups = c[C_DUP_GROUPS]; out->mixed_groups = c[C_MIXED_GROUPS];
  out->serial_fallbacks = c[C_SERIAL]; out->unexpired_evictions = c[C_EVICT_UNEXPIRED]; out->swept = c[C_SWEPT]; out->gq_dropped = c[C_GQ_DROPPED];
  return 0;
}

int gub_probe_random_access(gub_table* t, uint64_t accesses, double* gbs) {
  if (!t || !gbs || accesses == 0) return fail("gub_probe_random_access: bad argument");
  std::lock_guard<std::mutex> lk(g_emu_mu);
  emu_random_rmw(t->e, accesses);
  *gbs = 1.0;
  return 0;
}

// The entry points that take device pointers or peers are stubs in tests/emu_abi_stubs.cpp (kept apart: their prototypes in the header
// do not match a stub's); they report through this.
int emu_abi_not_emulated(const char* name) { return fail(std::string(name) + ": not emulated (tests/emu_abi.cpp)"); }

}  // extern "C"
