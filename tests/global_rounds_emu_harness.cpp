// TEST-ONLY: the CPU emulation of the kernels (tests/kernel_emu_harness.cpp, included whole) plus the pieces of a GLOBAL sync tick
// that put the drained hit records into key-consistent rounds: k_gq_hist, gq_plan_rounds, k_gq_partition and gq_round_span of
// gub_global.cuh, called as tick_drain_hits / tick_partition / tick_round_route of gub_api.cu call them.  Built by
// tests/_global_rounds_emu.py with g++; never part of the product library.
#include "kernel_emu_harness.cpp"

extern "C" {

uint32_t emu_gq_bins() { return GQ_BINS; }

// hist[GQ_BINS] = the records of every bin (k_gq_hist over n records; the count also passes through n_dev, as in the tick).
void emu_gq_hist(const gub_req* recs, uint32_t n, uint32_t* hist) {
  std::memset(hist, 0, (size_t)GQ_BINS * 4);
  emu::launch(k_gq_hist, 4u, 256u, recs, n + 7, (const uint32_t*)&n, hist);
}

// The rounds of nsrc sources' histograms (hists: nsrc x GQ_BINS) as (lo, hi, slice) triples; returns how many (<= max_rounds written).
uint32_t emu_gq_plan(const uint32_t* hists, uint32_t nsrc, uint32_t cap, uint32_t* out, uint32_t max_rounds) {
  std::vector<const uint32_t*> rows(nsrc);
  for (uint32_t s = 0; s < nsrc; s++) rows[s] = hists + (size_t)s * GQ_BINS;
  std::vector<GqRound> rounds;
  gq_plan_rounds(rows.data(), nsrc, cap, rounds);
  for (size_t i = 0; i < rounds.size() && i < max_rounds; i++) {
    out[3 * i] = rounds[i].lo; out[3 * i + 1] = rounds[i].hi; out[3 * i + 2] = rounds[i].slice;
  }
  return (uint32_t)rounds.size();
}

// One source's records in round order (k_gq_partition with the exclusive prefix sum of `hist` as cursors), and the span
// (offset, count) of each of the given rounds in that array.
void emu_gq_partition(const gub_req* recs, uint32_t n, const uint32_t* hist, uint32_t cap, const uint32_t* rounds, uint32_t nrounds,
                      gub_req* out, uint32_t* offs, uint32_t* counts) {
  std::vector<uint32_t> start(GQ_BINS + 1, 0);
  for (uint32_t b = 0; b < GQ_BINS; b++) start[b + 1] = start[b] + hist[b];
  std::vector<uint32_t> cursor(start.begin(), start.end() - 1);
  emu::launch(k_gq_partition, 4u, 256u, recs, n + 7, (const uint32_t*)&n, cursor.data(), out);
  for (uint32_t i = 0; i < nrounds; i++) {
    const GqRound R{rounds[3 * i], rounds[3 * i + 1], rounds[3 * i + 2]};
    gq_round_span(R, start.data(), cap, &offs[i], &counts[i]);
  }
}

}  // extern "C"
