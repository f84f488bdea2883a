// TEST-ONLY: cursor_open of gubernator_b200/csrc/gub_kernels.cuh compiled for the CPU on top of tests/cuda_emu.h and run over a given
// table image, one key after the other.  Built by tests/test_probe_rounds_emulated.py with g++; never part of the product library.
#define GUB_EMULATE 1
#include "cuda_emu.h"

#include "../gubernator_b200/csrc/gub_kernels.cuh"

using namespace gub;

extern "C" {

int emu_probe_round(void) { return PROBE_ROUND; }
int emu_max_probe(void) { return MAX_PROBE; }

// For key i: found[i], slot[i], home[i] and the bucket cursor_open produced, as b[i] = key, tag, flags, limit, duration, rem, stamp, burst,
// expire (cur.old must equal cur.b; old_ok[i] says whether it does).
void emu_probe(const Slot* table, uint64_t cap, const uint64_t* keys, const uint64_t* tags, uint32_t n, uint8_t* found, int64_t* slot, uint64_t* home,
               uint64_t* b, uint8_t* old_ok) {
  for (uint32_t i = 0; i < n; i++) {
    Cursor c;
    cursor_open(c, table, cap, keys[i], tags[i]);
    found[i] = c.found ? 1 : 0; slot[i] = c.slot; home[i] = c.home;
    const Bucket& k = c.b;
    const uint64_t w[9] = {k.key, k.tag, k.flags, (uint64_t)k.limit, (uint64_t)k.duration, k.rem, (uint64_t)k.stamp, (uint64_t)k.burst, (uint64_t)k.expire};
    for (int j = 0; j < 9; j++) b[9 * (size_t)i + j] = w[j];
    const Bucket& o = c.old;
    old_ok[i] = o.key == k.key && o.tag == k.tag && o.flags == k.flags && o.limit == k.limit && o.duration == k.duration && o.rem == k.rem &&
                o.stamp == k.stamp && o.burst == k.burst && o.expire == k.expire;
  }
}

}  // extern "C"
