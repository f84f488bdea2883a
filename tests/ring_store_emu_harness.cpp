// TEST-ONLY: the CPU emulation of the kernels with the Store passes (tests/store_emu_harness.cpp, included whole, which includes
// tests/kernel_emu_harness.cpp) plus a ring Store step: emu_ring_store_step drives the ring of kernel_emu_harness.cpp (EmuP2P) the way
// p2p_local_all_store of gub_api.cu drives it.  Phase 1 routes records (k_p2p_route): what reaches the owners' mailboxes is the same as
// with key strings, and the Store passes only read the mailboxes.  Built by tests/_ring_store_emu.py with g++; never part of the product
// library.
#include "store_emu_harness.cpp"

namespace {

std::map<void*, std::vector<uint32_t*>> g_orig;  // per EmuP2P: every rank's [2][world][cap] inverse map (k_store_orig)

EmuStore& store_of(EmuTable* t) {  // the Store scratch of a ring table (emu_store_create's, made on first use)
  auto it = g_store.find(t);
  if (it != g_store.end()) return it->second;
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
  return g_store[t] = s;
}

}  // namespace

extern "C" {

uint32_t emu_ring_ovf_count(void* pv, uint32_t rank) { return static_cast<EmuP2P*>(pv)->tabs[rank]->ctl->ovf_count; }
void emu_ring_store_set_epoch(void* pv, uint32_t rank, uint32_t epoch) { store_of(static_cast<EmuP2P*>(pv)->tabs[rank]).epoch = epoch; }
uint32_t emu_ring_store_epoch(void* pv, uint32_t rank) { return store_of(static_cast<EmuP2P*>(pv)->tabs[rank]).epoch; }

// One step of every shard with a Store (world x cap <= max_batch).  Returns 0, the first non-zero result of `get` (nothing evaluated,
// the ring kept in step), -1 (table full for a loaded item) or -2 (a mailbox flag wait timed out).
int emu_ring_store_step(void* pv, const gub_req* const* reqs, const uint32_t* n, const gub_clock* clk, gub_store_get_fn get, void* user,
                        gub_resp* const* outs, gub_store_rec* const* changes, uint32_t* n_changes) {
  EmuP2P* p = static_cast<EmuP2P*>(pv);
  const uint32_t W = p->world, cap = p->cap, pass = W * cap;
  std::vector<uint32_t*>& orig = g_orig[pv];
  if (orig.empty()) for (uint32_t r = 0; r < W; r++) orig.push_back(zalloc<uint32_t>((size_t)2 * W * cap));
  p->epoch++;
  const uint32_t par = p->epoch & 1u;
  std::vector<P2PArgs> args(W);
  for (uint32_t r = 0; r < W; r++) {
    P2PArgs& A = args[r];
    for (uint32_t q = 0; q < W; q++) A.peers[q] = p->ranks[q].view;
    A.world = W; A.rank = r; A.cap = cap; A.epoch = p->epoch; A.done_ctr = nullptr; A.error = p->ranks[r].error;
  }
  for (uint32_t r = 0; r < W; r++) {  // 1. routing, then the inverse map
    EmuP2P::Rank& k = p->ranks[r];
    RouteArgs R;
    R.P = args[r]; R.reqs = reqs[r]; R.n = n[r]; R.n_dev = nullptr; R.pts = p->pts.data(); R.pt_peer = p->peers.data(); R.lut = p->lut.data();
    R.npts = (uint32_t)p->pts.size(); R.self_global = -1; R.true_owner = nullptr;
    R.tile_agg = k.tile_agg; R.counts = k.counts; R.perm = k.perm; R.ticket = k.ticket;
    emu::launch(k_p2p_route, std::max<uint32_t>(1u, (n[r] + RT_THREADS - 1) / RT_THREADS), (unsigned)RT_THREADS, R);
    if (n[r]) emu::launch(k_store_orig, (n[r] + 255) / 256, 256u, (const uint32_t*)k.perm, n[r], cap, orig[r] + (size_t)par * W * cap);
  }
  const unsigned blocks = (pass + STORE_THREADS - 1) / STORE_THREADS;
  std::vector<StoreArgs> S(W);
  std::vector<StoreSegs> G(W);
  for (uint32_t r = 0; r < W; r++) {  // 3. k_seg_wait, the pre-pass, the miss list
    EmuTable* t = p->tabs[r];
    EmuStore& ss = store_of(t);
    emu::launch(k_seg_wait, 1u, 32u, args[r], p->ranks[r].seg_off);
    if (ss.epoch >= 0xFFFFFFFFu) { std::memset(ss.keys, 0, (size_t)ss.key_entries * sizeof(StoreKey)); ss.epoch = 0; }
    ss.epoch++;
    StoreArgs& s = S[r];
    std::memset(&s, 0, sizeof s);
    s.n = pass; s.epoch = ss.epoch; s.keys = ss.keys; s.key_mask = ss.key_entries - 1; s.kent = ss.kent; s.bstate = ss.bstate;
    s.sel = ss.sel; s.sparse = ss.sparse; s.blk = ss.blk; s.table = t->table; s.capacity = t->capacity; s.ovf = t->ovf;
    s.ovf_count = &t->ctl->ovf_count; s.inv = t->inv; s.now_ms = clk->now_ms; s.want_misses = get ? 1u : 0u;
    StoreSegs& g = G[r];
    std::memset(&g, 0, sizeof g);
    g.nseg = W; g.seg_off = p->ranks[r].seg_off;
    for (uint32_t q = 0; q < W; q++) {
      g.req[q] = args[r].peers[r].req_mb + ((size_t)par * W + q) * cap;
      g.out[q] = args[r].peers[q].resp_mb + ((size_t)par * W + r) * cap;
      g.orig[q] = orig[q] + ((size_t)par * W + r) * cap;
      g.perm[q] = p->ranks[q].perm;
    }
    emu::launch(k_store_keys_ring, blocks, (unsigned)STORE_THREADS, s, g);
    emu::launch(k_store_before_ring, blocks, (unsigned)STORE_THREADS, s, g);
    if (get) emu::launch(k_store_compact, blocks, (unsigned)STORE_THREADS, (const uint8_t*)ss.sel, (const gub_store_rec*)ss.sparse, (const uint32_t*)ss.blk,
                         pass, ss.miss, &ss.miss_count);
  }
  int rc = 0;
  if (get) {  // 4. every Get in rank order, then every installation
    std::vector<std::vector<uint4>> loaded(W);
    std::vector<std::vector<DevItem>> items(W);
    for (uint32_t r = 0; r < W && rc == 0; r++) {
      EmuStore& ss = store_of(p->tabs[r]);
      const uint32_t m = ss.miss_count;
      if (!m) continue;
      std::vector<gub_store_rec> named(ss.miss, ss.miss + m);  // store_get of gub_api.cu: the keys and request names are the library's
      rc = get(user, ss.miss, m);
      if (rc) break;
      for (uint32_t k = 0; k < m; k++) {
        gub_store_rec& rr = ss.miss[k];
        if (!(rr.flags & GUB_STORE_FOUND)) continue;
        rr.first = named[k].first; rr.last = named[k].last; rr.first_shard = named[k].first_shard; rr.last_shard = named[k].last_shard;
        rr.item.key_xxh64 = named[k].item.key_xxh64; rr.item.key_fnv1 = named[k].item.key_fnv1;
        loaded[r].push_back(make_uint4(rr.first, rr.item.expire_at >= clk->now_ms ? S_EXISTED : 0u, (uint32_t)rr.item.algorithm, (uint32_t)rr.first_shard));
        if (rr.item.algorithm == GUB_TOKEN_BUCKET || rr.item.algorithm == GUB_LEAKY_BUCKET) items[r].push_back(item_dev(rr.item));
      }
    }
    for (uint32_t r = 0; r < W && rc == 0; r++) {
      EmuTable* t = p->tabs[r];
      EmuStore& ss = store_of(t);
      if (!items[r].empty()) {
        gub_clock dclk;
        std::memset(&dclk, 0, sizeof dclk);
        dclk.now_ms = INT64_MIN;  // drain_pending of gub_api.cu
        FArgs A;
        fused_args(t, &dclk, A);
        emu::launch(k_drain_overflow, 1u, 32u, A);
        ss.failed = 0;
        emu::launch(k_add_items, (unsigned)((items[r].size() + 255) / 256), 256u, t->table, t->capacity, (const DevItem*)items[r].data(),
                    (uint32_t)items[r].size(), t->counters, &ss.failed, t->inv);
        if (ss.failed) rc = -1;
      }
      if (!loaded[r].empty())
        emu::launch(k_store_loaded_ring, (unsigned)((loaded[r].size() + STORE_THREADS - 1) / STORE_THREADS), (unsigned)STORE_THREADS,
                    (const uint4*)loaded[r].data(), (uint32_t)loaded[r].size(), ss.bstate, G[r]);
    }
  }
  for (uint32_t r = 0; r < W; r++) {  // 5. the passes, the post-pass, the flags
    if (rc == 0) {
      EmuTable* t = p->tabs[r];
      EmuStore& ss = store_of(t);
      EmuSegs sd;
      sd.nseg = W; sd.seg_off = p->ranks[r].seg_off;
      for (uint32_t q = 0; q < W; q++) { sd.reqs[q] = G[r].req[q]; sd.out[q] = const_cast<gub_resp*>(G[r].out[q]); }
      submit_chunk(t, nullptr, pass, p->ranks[r].seg_off + W, 0u, clk, nullptr, &sd);
      emu::launch(k_store_after_ring, blocks, (unsigned)STORE_THREADS, S[r], G[r]);
      emu::launch(k_store_compact, blocks, (unsigned)STORE_THREADS, (const uint8_t*)ss.sel, (const gub_store_rec*)ss.sparse, (const uint32_t*)ss.blk,
                  pass, changes[r], n_changes + r);
    }
    emu::launch(k_seg_publish, 1u, 32u, args[r]);
  }
  int err = 0;
  for (uint32_t r = 0; r < W; r++) {  // 7. collects
    EmuP2P::Rank& k = p->ranks[r];
    emu::launch(k_p2p_collect, 4u, 256u, args[r], (const uint32_t*)k.perm, n[r], (const uint32_t*)nullptr, outs[r]);
    err |= (int)*k.error | (int)p->tabs[r]->ctl->error;
  }
  return rc ? rc : (err ? -2 : 0);
}

}  // extern "C"
