// TEST-ONLY host build of gubernator_b200/csrc/bucket_math.cuh (the exact header the CUDA kernels include), so the
// bucket state machines and the run planner can be checked against the oracle on a machine without a GPU.
// Built by tests/_host_math.py with g++; never part of the product library.
#include <cstring>
#include <unordered_map>
#include <vector>

#include "../gubernator_b200/csrc/bucket_math.cuh"

using namespace gub;

namespace {
struct K { uint64_t a, b; bool operator==(const K& o) const { return a == o.a && b == o.b; } };
struct KH { size_t operator()(const K& k) const { return (size_t)(k.a ^ (k.b * 0x9E3779B97F4A7C15ULL)); } };
struct Table { std::unordered_map<K, Bucket, KH> m; Delta d{0, 0, 0}; };
}  // namespace

extern "C" {

void* hm_table_new() { return new Table(); }
void hm_table_free(void* t) { delete (Table*)t; }

// Sequential index-order walk with apply_one() — the semantic every kernel path must reproduce.
void hm_apply_seq(void* tv, const gub_req* reqs, size_t n, const gub_clock* clk, gub_resp* out, uint64_t counters3[3]) {
  Table* t = (Table*)tv;
  for (size_t i = 0; i < n; i++) {
    K k{reqs[i].key_xxh64, reqs[i].key_fnv1};
    auto it = t->m.find(k);
    if (it == t->m.end()) {
      Bucket b;
      std::memset(&b, 0, sizeof b);
      it = t->m.emplace(k, b).first;
    }
    out[i] = apply_one(it->second, reqs[i], *clk, t->d);
  }
  counters3[0] = t->d.over; counters3[1] = t->d.hit; counters3[2] = t->d.miss;
}

// Applies `rq` m times to bucket *b: once serially (ground truth) and once through plan_run()+eval_piece(), falling
// back to apply_one() for ranks beyond the piece buffer like the kernels do.  Returns 0 when everything is identical
// (responses, final bucket, counter deltas), else a positive code.  *npieces_out reports the plan size.
int hm_plan_check(const Bucket* b0, const gub_req* rq, uint32_t m, const gub_clock* clk, uint32_t cap, uint32_t* npieces_out,
                  uint32_t* covered_out) {
  Bucket bs = *b0, bp = *b0;
  Delta ds{0, 0, 0}, dp{0, 0, 0};
  std::vector<gub_resp> want(m), got(m);
  for (uint32_t i = 0; i < m; i++) want[i] = apply_one(bs, *rq, *clk, ds);
  std::vector<Piece> pieces(cap);
  uint32_t np = 0;
  uint32_t covered = plan_run(bp, *rq, m, *clk, dp, pieces.data(), cap, &np);
  *npieces_out = np; *covered_out = covered;
  for (uint32_t r = 0; r < covered; r++) {
    uint32_t pi = 0;
    while (pi + 1 < np && pieces[pi + 1].start <= r) pi++;
    got[r] = eval_piece(pieces[pi], r);
  }
  for (uint32_t r = covered; r < m; r++) got[r] = apply_one(bp, *rq, *clk, dp);
  for (uint32_t r = 0; r < m; r++)
    if (std::memcmp(&want[r], &got[r], sizeof(gub_resp)) != 0) return 1000 + (int)(r < 1000000 ? r : 999999);
  if (!bucket_equal(bs, bp)) return 2;
  if (ds.over != dp.over || ds.hit != dp.hit || ds.miss != dp.miss) return 3;
  return 0;
}

// run_to_rank() for every rank (or a sample of ranks) of an m-long run against m sequential apply_one() calls.
int hm_rank_check(const Bucket* b0, const gub_req* rq, uint32_t m, const gub_clock* clk, uint32_t stride) {
  Bucket bs = *b0;
  Delta ds{0, 0, 0};
  std::vector<gub_resp> want(m);
  std::vector<Bucket> states(m);
  std::vector<Delta> deltas(m);
  for (uint32_t i = 0; i < m; i++) { want[i] = apply_one(bs, *rq, *clk, ds); states[i] = bs; deltas[i] = ds; }
  for (uint32_t r = 0; r < m; r += (r + 1 == m || r + stride < m) ? stride : (m - 1 - r)) {
    Bucket b = *b0;
    Delta d{0, 0, 0};
    gub_resp got = run_to_rank(b, *rq, r, *clk, d);
    if (std::memcmp(&want[r], &got, sizeof(gub_resp)) != 0) return 1000 + (int)(r < 1000000 ? r : 999999);
    if (!bucket_equal(states[r], b)) return 2;
    if (deltas[r].over != d.over || deltas[r].hit != d.hit || deltas[r].miss != d.miss) return 3;
    if (r + 1 == m) break;
  }
  return 0;
}

size_t hm_sizeof_bucket() { return sizeof(Bucket); }

// Element-wise entries over arrays; tests/bucket_math_dev.cu exports the same signatures over the device build of the header.
void hm_f2i(const double* x, int64_t* out, size_t n) {
  for (size_t i = 0; i < n; i++) out[i] = f2i(x[i]);
}
// b[i] <- apply_one(b[i], rq[i]); d[i] holds that one application's counter deltas
void hm_apply_one(Bucket* b, const gub_req* rq, const gub_clock* clk, size_t n, gub_resp* out, Delta* d) {
  for (size_t i = 0; i < n; i++) { d[i] = Delta{0, 0, 0}; out[i] = apply_one(b[i], rq[i], *clk, d[i]); }
}
// b[i] <- the state after rank target[i] of a run of identical requests rq[i]
void hm_run_to_rank(Bucket* b, const gub_req* rq, const uint32_t* target, const gub_clock* clk, size_t n, gub_resp* out, Delta* d) {
  for (size_t i = 0; i < n; i++) { d[i] = Delta{0, 0, 0}; out[i] = run_to_rank(b[i], rq[i], target[i], *clk, d[i]); }
}
}
