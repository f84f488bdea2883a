// TEST-ONLY: the CPU emulation of the kernels (tests/kernel_emu_harness.cpp, included whole) plus the ring fed with key strings:
// emu_p2p_step_keys is emu_p2p_step with k_p2p_route_keys in phase 1 (p2p_route_keys of gub_api.cu).  Built by
// tests/_ring_keys_emu.py with g++; never part of the product library.
#include "kernel_emu_harness.cpp"

extern "C" {

// packed[r] = shard r's batch in the layout of gub_keys_layout, packed_bytes[r] its size in bytes; one parameter table for the step.
// self_global != 0: GLOBAL mode (true_owner_out / expanded_out, optional: every shard's ring owners and expanded records).
int emu_p2p_step_keys(void* pv, const uint8_t* const* packed, const uint64_t* packed_bytes, const uint32_t* n, const gub_params* params,
                      uint32_t n_params, int64_t created_base, const gub_clock* clk, gub_resp* const* outs, uint32_t self_global,
                      uint8_t* const* true_owner_out, gub_req* const* expanded_out) {
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
    std::vector<KeysRouteArgs> K(1);  // (on the heap: the inline parameter table makes it large)
    std::memset(K.data(), 0, sizeof(KeysRouteArgs));
    RouteArgs& R = K[0].R;
    R.P = args[r]; R.reqs = nullptr; R.n = n[r]; R.n_dev = nullptr; R.pts = p->pts.data(); R.pt_peer = p->peers.data(); R.lut = p->lut.data();
    R.npts = (uint32_t)p->pts.size(); R.self_global = self_global ? (int32_t)r : -1; R.true_owner = self_global ? k.true_owner : nullptr;
    R.tile_agg = k.tile_agg; R.counts = k.counts; R.perm = k.perm; R.ticket = k.ticket;
    K[0].packed = packed[r];
    K[0].key_bytes = n[r] ? packed_bytes[r] - ((uint64_t)n[r] * 16 + ((uint64_t)n[r] + 1) * 4) : 0;
    K[0].n_params = n_params; K[0].created_base = created_base;
    if (n_params <= INLINE_PARAMS) { if (n_params) std::memcpy(&K[0].Pi, params, n_params * sizeof(gub_params)); }
    else K[0].params_far = params;
    K[0].expanded = self_global && expanded_out ? expanded_out[r] : nullptr;
    emu::launch(k_p2p_route_keys, std::max<uint32_t>(1u, (n[r] + RT_THREADS - 1) / RT_THREADS), (unsigned)RT_THREADS, K[0]);
    if (self_global && true_owner_out && n[r]) std::memcpy(true_owner_out[r], k.true_owner, n[r]);
  }
  const uint32_t par = p->epoch & 1u;
  for (uint32_t r = 0; r < p->world; r++) {  // phase 2, as in emu_p2p_step
    if (!g_fused) {
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

// What phase 1 left behind on shard r: its request mailbox block (both parities, [2][W][cap]), perm [cap] and counts [W].
void emu_p2p_route_state(void* pv, uint32_t rank, gub_req* req_mb, uint32_t* perm, uint32_t* counts) {
  EmuP2P* p = static_cast<EmuP2P*>(pv);
  const EmuP2P::Rank& k = p->ranks[rank];
  std::memcpy(req_mb, k.view.req_mb, (size_t)2 * p->world * p->cap * sizeof(gub_req));
  std::memcpy(perm, k.perm, (size_t)p->cap * 4);
  std::memcpy(counts, k.counts, (size_t)p->world * 4);
}

}  // extern "C"
