// TEST-ONLY: the CPU emulation of the kernels (tests/kernel_emu_harness.cpp, included whole) driven like launch_chunk of gub_api.cu on a
// single table with two grouping scratch sets: the set is picked by epoch parity, k_finish stores the chain-done word and k_group may take
// its early path.  Built by tests/_handoff_emu.py with g++; never part of the product library.
#include "kernel_emu_harness.cpp"

#include <map>

namespace {

struct SecondSet { AuxEntry* aux; uint32_t *presence, *ent, *meta; uint8_t* fragsize; };
std::map<void*, SecondSet> g_second;

}  // namespace

extern "C" {

void* emu_handoff_create(uint64_t capacity_slots, uint32_t max_batch) {
  EmuTable* t = static_cast<EmuTable*>(emu_create(capacity_slots, max_batch));
  SecondSet s;
  s.aux = zalloc<AuxEntry>(t->aux_entries);
  s.presence = zalloc<uint32_t>((size_t)t->aux_entries * t->pres_words);
  s.fragsize = zalloc<uint8_t>((size_t)t->aux_entries * t->max_blocks);
  s.ent = zalloc<uint32_t>(t->max_batch);
  s.meta = zalloc<uint32_t>(t->max_batch);
  g_second[t] = s;
  return t;
}

void emu_handoff_destroy(void* tv) {
  const SecondSet s = g_second[tv];
  void* ptrs[] = {s.aux, s.presence, s.fragsize, s.ent, s.meta};
  for (void* p : ptrs) std::free(p);
  g_second.erase(tv);
  emu_destroy(tv);
}

uint32_t emu_handoff_chain_done(void* tv) { return static_cast<EmuTable*>(tv)->ctl->chain_done; }

// early = 0: the chain-done word as the previous k_finish left it, so every k_group block waits first (the emulator runs one launch after
// another).  early = 1: a stale word before every k_group, so every block takes the early path: grouping before the wait, drain after it.
// That is safe here because everything before the launch has completed, and it runs the early path's code on the batch's real data.
int emu_handoff_submit(void* tv, const gub_req* reqs, size_t n, const gub_clock* clk, gub_resp* out, uint32_t early) {
  EmuTable* t = static_cast<EmuTable*>(tv);
  const SecondSet& s2 = g_second[tv];
  for (size_t off = 0; off < n; off += t->max_batch) {
    const uint32_t m = (uint32_t)std::min<size_t>(t->max_batch, n - off);
    if (t->epoch >= 65535u) {
      std::memset(t->aux, 0, (size_t)t->aux_entries * sizeof(AuxEntry));
      std::memset(s2.aux, 0, (size_t)t->aux_entries * sizeof(AuxEntry));
      std::memset(t->ctr, 0, 2 * sizeof(BatchCtr));
      t->epoch = 0;
    }
    t->epoch++;
    const bool odd = (t->epoch & 1u) != 0;
    BatchArgs A;
    std::memset(&A, 0, sizeof A);
    A.table = t->table; A.capacity = t->capacity; A.reqs = reqs + off; A.out = out + off; A.n = m; A.n_dev = nullptr; A.n_off = (uint32_t)off;
    A.epoch = t->epoch;
    A.aux = odd ? s2.aux : t->aux; A.aux_mask = t->aux_entries - 1; A.presence = odd ? s2.presence : t->presence;
    A.fragsize = odd ? s2.fragsize : t->fragsize; A.pres_words = t->pres_words; A.max_blocks = t->max_blocks;
    A.ent = odd ? s2.ent : t->ent; A.meta = odd ? s2.meta : t->meta; A.rank = t->rank;
    A.commit = t->commit; A.order = t->order; A.mixed_ent = t->mixed_ent; A.ctr = t->ctr;
    A.counters = t->counters; A.ovf = t->ovf; A.ovf_count = &t->ctl->ovf_count; A.inv = t->inv;
    A.chain_done = &t->ctl->chain_done;
    A.early_ok = t->epoch > 1u ? 1u : 0u;
    A.clk = *clk;
    if (early) t->ctl->chain_done = 0xFFFFFFFFu;
    const uint32_t blocks = (m + 255) / 256;
    const uint32_t fin = std::min<uint32_t>(g_finish_cap, std::max<uint32_t>(1u, m / 2));
    emu::launch(k_group<false>, blocks, GROUP_THREADS, A);
    emu::launch(k_rank<false>, blocks, GROUP_THREADS, A);
    emu::launch(k_eval<false>, blocks, GROUP_THREADS, A);
    emu::launch(k_finish<false>, fin, MIXED_THREADS, A);
  }
  return 0;
}

}  // extern "C"
