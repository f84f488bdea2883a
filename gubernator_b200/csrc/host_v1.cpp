// host_v1.cpp — C++ stand-in for the Go side of the boundary (include/gubernator_b200_host.h): the request loop of
// V1Instance.GetRateLimits (gubernator.go:183-295) re-expressed as "validate, hash, one device batch, map errors".
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <deque>
#include <mutex>
#include <thread>
#include <unordered_map>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/gubernator_b200_host.h"

struct gub_instance {
  gub_table* table = nullptr;
  int64_t frozen_now = -1;
  bool has_store = false;
  gub_store store{};
};

namespace {
int64_t wall_ms() {
  using namespace std::chrono;
  return duration_cast<milliseconds>(system_clock::now().time_since_epoch()).count();
}
const char* algo_scope(int32_t algorithm) { return algorithm == GUB_LEAKY_BUCKET ? "Error in leakyBucket" : "Error in tokenBucket"; }
}  // namespace

extern "C" {

void gub_format_error(int err_code, const char* key, int32_t algorithm, char* out, size_t cap) {
  // gubernator.go:252 wraps gubernator.go:600 wraps workers.go:304/313 wraps interval.go:93/107 (pkg/errors "a: b")
  static const char* pre = "Error while apply rate limit for '%s': during workerPool.GetRateLimit: ";
  char head[512];
  std::snprintf(head, sizeof head, pre, key);
  switch (err_code) {
    case GUB_ERR_UNIQUE_KEY_EMPTY: std::snprintf(out, cap, "field 'unique_key' cannot be empty"); break;
    case GUB_ERR_NAMESPACE_EMPTY: std::snprintf(out, cap, "field 'namespace' cannot be empty"); break;
    case GUB_ERR_INVALID_ALGORITHM: std::snprintf(out, cap, "%sInvalid rate limit algorithm '%d'", head, algorithm); break;
    case GUB_ERR_GREGORIAN_WEEKS:
      std::snprintf(out, cap, "%s%s: `Duration = GregorianWeeks` not yet supported; consider making a PR!`", head, algo_scope(algorithm));
      break;
    case GUB_ERR_GREGORIAN_INVALID:
      std::snprintf(out, cap, "%s%s: behavior DURATION_IS_GREGORIAN is set; but `Duration` is not a valid gregorian interval", head,
                    algo_scope(algorithm));
      break;
    case GUB_ERR_TABLE_FULL: std::snprintf(out, cap, "%srate limit table is full", head); break;
    case GUB_ERR_PEER_TIMEOUT:  // gubernator.go:374 wrapping the deadline error of a timed-out peer call
      std::snprintf(out, cap, "Error while fetching rate limit '%s' from peer: context deadline exceeded", key);
      break;
    default: if (cap) out[0] = 0;
  }
}

int gub_instance_create(gub_table* table, gub_instance** out) {
  if (!table || !out) return -1;
  *out = new gub_instance();
  (*out)->table = table;
  return 0;
}
void gub_instance_destroy(gub_instance* s) { delete s; }
void gub_instance_set_clock(gub_instance* s, int64_t frozen_now_ms) { s->frozen_now = frozen_now_ms; }
int64_t gub_instance_now(gub_instance* s) { return s->frozen_now >= 0 ? s->frozen_now : wall_ms(); }

}  // extern "C"

namespace {
// One GetRateLimits call, validated and hashed (gubernator.go:195-220): the requests that reach the device and where their
// answers go.
struct PreparedCall {
  std::vector<gub_req> batch;
  std::vector<size_t> where;      // batch position -> request index of the call
  std::vector<std::string> keys;  // for error text
};

void prepare_call(const gub_rate_limit_req* reqs, size_t n, gub_rate_limit_resp* out, int64_t now, PreparedCall& pc) {
  pc.batch.reserve(n); pc.where.reserve(n); pc.keys.reserve(n);
  for (size_t i = 0; i < n; i++) {
    gub_rate_limit_resp& o = out[i];
    std::memset(&o, 0, sizeof o);
    const char* name = reqs[i].name ? reqs[i].name : "";
    const char* uk = reqs[i].unique_key ? reqs[i].unique_key : "";
    if (!uk[0]) {  // :208-212, checked before the namespace
      o.err_code = GUB_ERR_UNIQUE_KEY_EMPTY;
      gub_format_error(o.err_code, "", 0, o.error, sizeof o.error);
      continue;
    }
    if (!name[0]) {  // :213-217
      o.err_code = GUB_ERR_NAMESPACE_EMPTY;
      gub_format_error(o.err_code, "", 0, o.error, sizeof o.error);
      continue;
    }
    std::string key = std::string(name) + "_" + uk;  // client.go:39-41
    gub_req r;
    r.key_xxh64 = gub_xxh64(key.data(), key.size(), 0);
    r.key_fnv1 = gub_fnv1_64(key.data(), key.size());
    r.hits = reqs[i].hits; r.limit = reqs[i].limit; r.duration = reqs[i].duration; r.burst = reqs[i].burst;
    r.created_at = reqs[i].created_at != 0 ? reqs[i].created_at : now;  // :218-220
    r.algorithm = (uint32_t)reqs[i].algorithm;
    r.behavior = ((uint32_t)reqs[i].behavior & 0xFFu) | GUB_REQ_IS_OWNER;  // one-node cluster: every key is ours (:247-250)
    pc.batch.push_back(r); pc.where.push_back(i); pc.keys.push_back(std::move(key));
  }
}

void finish_call(const PreparedCall& pc, const gub_rate_limit_req* reqs, const gub_resp* resp, gub_rate_limit_resp* out) {
  for (size_t j = 0; j < pc.batch.size(); j++) {
    gub_rate_limit_resp& o = out[pc.where[j]];
    o.err_code = (int32_t)resp[j].err_code;
    if (resp[j].err_code) {
      gub_format_error((int)resp[j].err_code, pc.keys[j].c_str(), reqs[pc.where[j]].algorithm, o.error, sizeof o.error);
    } else {
      o.status = (int32_t)resp[j].status; o.limit = resp[j].limit; o.remaining = resp[j].remaining; o.reset_time = resp[j].reset_time;
    }
  }
}
}  // namespace

namespace {
// Store plugin around one batch (see gub_store in the header).  Distinct keys in first-occurrence order.
struct StoreKeys {
  std::vector<size_t> first, last;  // batch positions of each distinct key's first / last request
  std::vector<uint64_t> kx, kf;
  std::vector<char> reset_token;    // some TOKEN_BUCKET request of the key carries RESET_REMAINING
};

void collect_keys(const PreparedCall& pc, StoreKeys& sk) {
  std::unordered_map<uint64_t, size_t> seen;
  for (size_t j = 0; j < pc.batch.size(); j++) {
    const gub_req& r = pc.batch[j];
    const uint64_t h = r.key_xxh64 ^ (r.key_fnv1 * 0x9E3779B97F4A7C15ULL);
    auto it = seen.find(h);
    size_t k;
    if (it == seen.end()) {
      k = sk.first.size();
      seen.emplace(h, k);
      sk.first.push_back(j); sk.last.push_back(j); sk.kx.push_back(r.key_xxh64); sk.kf.push_back(r.key_fnv1); sk.reset_token.push_back(0);
    } else {
      k = it->second;
      sk.last[k] = j;
    }
    if (r.algorithm == GUB_TOKEN_BUCKET && (r.behavior & GUB_BEHAVIOR_RESET_REMAINING)) sk.reset_token[k] = 1;
  }
}

int submit_with_store(gub_instance* s, const PreparedCall& pc, const gub_rate_limit_req* reqs, const gub_clock& clk, gub_resp* resp) {
  StoreKeys sk;
  collect_keys(pc, sk);
  const size_t nk = sk.first.size();
  std::vector<gub_item> before(nk), after(nk);
  std::vector<uint8_t> had(nk), has(nk);
  if (gub_get_items(s->table, sk.kx.data(), sk.kf.data(), nk, clk.now_ms, before.data(), had.data()) != 0) return -1;
  // cache miss -> Store.Get (algorithms.go:45-51); what it returns is added to the cache before the request runs
  std::vector<gub_item> loaded;
  for (size_t k = 0; k < nk; k++) {
    if (had[k] || !s->store.get) continue;
    const size_t j = sk.first[k];
    gub_item it;
    std::memset(&it, 0, sizeof it);
    if (s->store.get(s->store.user, &reqs[pc.where[j]], pc.keys[j].c_str(), &it)) {
      it.key_xxh64 = sk.kx[k]; it.key_fnv1 = sk.kf[k];
      loaded.push_back(it);
      before[k] = it; had[k] = 2;  // present, from the store
    }
  }
  if (!loaded.empty() && gub_add_items(s->table, loaded.data(), loaded.size()) != 0) return -1;
  if (gub_submit(s->table, pc.batch.data(), pc.batch.size(), &clk, resp) != 0) return -1;
  if (gub_get_items(s->table, sk.kx.data(), sk.kf.data(), nk, clk.now_ms, after.data(), has.data()) != 0) return -1;
  for (size_t k = 0; k < nk; k++) {
    const size_t jf = sk.first[k], jl = sk.last[k];
    // Store.Remove: the item that existed was deleted — RESET_REMAINING on a token bucket (algorithms.go:78-83) or the
    // client switched algorithms (algorithms.go:91-100, 308-315)
    const bool existed = had[k] != 0 && (had[k] == 2 ? before[k].expire_at >= clk.now_ms : true);
    if (existed && s->store.remove) {
      const bool switched = before[k].algorithm != (int32_t)pc.batch[jf].algorithm && pc.batch[jf].algorithm <= 1u;
      if (switched || sk.reset_token[k]) s->store.remove(s->store.user, pc.keys[jf].c_str());
    }
    // Store.OnChange: once per key, with the item as the batch left it (owner requests only: algorithms.go:149,252)
    if (has[k] && s->store.on_change && resp[jl].err_code == 0 && (pc.batch[jl].behavior & GUB_REQ_IS_OWNER))
      s->store.on_change(s->store.user, &reqs[pc.where[jl]], pc.keys[jl].c_str(), &after[k]);
  }
  return 0;
}
}  // namespace

extern "C" {

void gub_instance_set_store(gub_instance* s, const gub_store* store) {
  if (!s) return;
  s->has_store = store != nullptr;
  if (store) s->store = *store;
}

int gub_instance_get_rate_limits_unbounded(gub_instance* s, const gub_rate_limit_req* reqs, size_t n, gub_rate_limit_resp* out) {
  if (!s || (n && (!reqs || !out))) return -1;
  const int64_t now = gub_instance_now(s);  // gubernator.go:195: one timestamp per call
  PreparedCall pc;
  prepare_call(reqs, n, out, now, pc);
  if (pc.batch.empty()) return 0;
  gub_clock clk;
  gub_clock_fill(now, &clk);
  std::vector<gub_resp> resp(pc.batch.size());
  if (s->has_store) {
    if (submit_with_store(s, pc, reqs, clk, resp.data()) != 0) return -1;
  } else if (gub_submit(s->table, pc.batch.data(), pc.batch.size(), &clk, resp.data()) != 0) {
    return -1;
  }
  finish_call(pc, reqs, resp.data(), out);
  return 0;
}

int gub_instance_get_rate_limits(gub_instance* s, const gub_rate_limit_req* reqs, size_t n, gub_rate_limit_resp* out) {
  if (n > GUB_MAX_BATCH_SIZE) return GUB_E_TOO_LARGE;  // gubernator.go:189-193
  return gub_instance_get_rate_limits_unbounded(s, reqs, n, out);
}

int gub_instance_update_peer_global(gub_instance* s, const char* key, int32_t algorithm, int64_t duration, int32_t status, int64_t limit,
                                    int64_t remaining, int64_t reset_time) {
  if (!s || !key) return -1;
  const int64_t now = gub_instance_now(s);  // gubernator.go:427
  gub_item it;
  std::memset(&it, 0, sizeof it);
  const size_t len = std::strlen(key);
  it.key_xxh64 = gub_xxh64(key, len, 0);
  it.key_fnv1 = gub_fnv1_64(key, len);
  it.algorithm = algorithm; it.expire_at = reset_time;  // :429-433
  it.limit = limit; it.duration = duration; it.stamp = now;
  if (algorithm == GUB_LEAKY_BUCKET) { it.remaining_f = (double)remaining; it.burst = limit; }  // :435-442
  else { it.status = status; it.remaining = remaining; }                                       // :443-450
  return gub_add_items(s->table, &it, 1);
}

}  // extern "C"

// ---- RPC aggregator ---------------------------------------------------------------------------------------------
struct gub_aggregator {
  gub_instance* inst = nullptr;
  uint32_t max_batch = 65536, window_us = 500;
  struct Call {
    const gub_rate_limit_req* reqs; size_t n; gub_rate_limit_resp* out;
    PreparedCall pc;
    bool done = false; int rc = 0;
  };
  std::mutex mu;
  std::condition_variable cv_work, cv_done;
  std::deque<Call*> queue;
  size_t queued = 0;
  bool stop = false;
  uint64_t batches = 0, requests = 0;
  std::thread flusher;

  void run() {
    std::unique_lock<std::mutex> lk(mu);
    for (;;) {
      cv_work.wait(lk, [&] { return stop || !queue.empty(); });
      if (stop && queue.empty()) return;
      // BatchWait: give other callers `window_us` to join, unless the batch is already full (peer_client.go:296-330)
      const auto deadline = std::chrono::steady_clock::now() + std::chrono::microseconds(window_us);
      cv_work.wait_until(lk, deadline, [&] { return stop || queued >= max_batch; });
      std::vector<Call*> calls(queue.begin(), queue.end());
      queue.clear();
      queued = 0;
      lk.unlock();
      flush(calls);
      lk.lock();
      for (Call* c : calls) c->done = true;
      cv_done.notify_all();
    }
  }

  void flush(std::vector<Call*>& calls) {
    // arrival order, each call's requests in index order: sequential semantics across the coalesced calls
    std::vector<gub_req> batch;
    size_t total = 0;
    for (Call* c : calls) total += c->pc.batch.size();
    batch.reserve(total);
    for (Call* c : calls) batch.insert(batch.end(), c->pc.batch.begin(), c->pc.batch.end());
    int rc = 0;
    std::vector<gub_resp> resp(total);
    if (total) {
      gub_clock clk;
      gub_clock_fill(gub_instance_now(inst), &clk);
      if (inst->has_store) {
        // a Store plugin sees Get / OnChange / Remove per call (algorithms.go:45-51,149,252): the coalesced calls are evaluated one
        // after another, in arrival order, through the same path gub_instance_get_rate_limits takes (ADVICE r1)
        size_t o = 0;
        for (Call* c : calls) {
          if (!c->pc.batch.empty() && rc == 0) rc = submit_with_store(inst, c->pc, c->reqs, clk, resp.data() + o);
          o += c->pc.batch.size();
        }
      } else {
        rc = gub_submit(inst->table, batch.data(), total, &clk, resp.data());
      }
    }
    size_t off = 0;
    for (Call* c : calls) {
      c->rc = rc;
      if (rc == 0) finish_call(c->pc, c->reqs, resp.data() + off, c->out);
      off += c->pc.batch.size();
    }
    std::lock_guard<std::mutex> lk(mu);
    batches += total ? 1 : 0;
    requests += total;
  }
};

extern "C" {

int gub_aggregator_create(gub_instance* s, uint32_t max_batch, uint32_t window_us, gub_aggregator** out) {
  if (!s || !out) return -1;
  gub_aggregator* a = new gub_aggregator();
  a->inst = s;
  a->max_batch = max_batch ? max_batch : 65536;
  a->window_us = window_us;
  a->flusher = std::thread([a] { a->run(); });
  *out = a;
  return 0;
}

void gub_aggregator_destroy(gub_aggregator* a) {
  if (!a) return;
  {
    std::lock_guard<std::mutex> lk(a->mu);
    a->stop = true;
  }
  a->cv_work.notify_all();
  a->flusher.join();
  delete a;
}

int gub_aggregator_get_rate_limits(gub_aggregator* a, const gub_rate_limit_req* reqs, size_t n, gub_rate_limit_resp* out) {
  if (!a || (n && (!reqs || !out))) return -1;
  if (n > GUB_MAX_BATCH_SIZE) return GUB_E_TOO_LARGE;  // gubernator.go:189-193
  gub_aggregator::Call call;
  call.reqs = reqs; call.n = n; call.out = out;
  prepare_call(reqs, n, out, gub_instance_now(a->inst), call.pc);  // gubernator.go:195: the call's own timestamp
  std::unique_lock<std::mutex> lk(a->mu);
  a->queue.push_back(&call);
  a->queued += call.pc.batch.size();
  a->cv_work.notify_all();
  a->cv_done.wait(lk, [&] { return call.done; });
  return call.rc;
}

void gub_aggregator_stats(gub_aggregator* a, uint64_t* batches, uint64_t* requests) {
  std::lock_guard<std::mutex> lk(a->mu);
  if (batches) *batches = a->batches;
  if (requests) *requests = a->requests;
}

}  // extern "C"
