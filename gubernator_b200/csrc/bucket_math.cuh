// bucket_math.cuh — the rate-limit state machines on a register-resident image of one table slot.
//
// Pure functions, usable from device code (the kernels) and from host code (tests/host_math_harness.cpp checks them
// against the oracle on the CPU, where there is no GPU to run the kernels).  No memory traffic happens here: callers
// load a slot into a Bucket, apply one or many requests, and write the Bucket back.
//
// Semantics follow mailgun/gubernator v2.4.0 algorithms.go:37-493 with lrucache.go:111-128 / cache.go:43-57 folded in
// as "an expired bucket is not live".  Line references in comments are to that file unless stated otherwise.
#pragma once
#include <stdint.h>

#include "../../include/gubernator_b200.h"

#include <emmintrin.h>  // host-side CVTTSD2SI (the host compilation of this header is what tests run on CPU)

#if defined(__CUDACC__)
#define GUB_HD __host__ __device__ __forceinline__
#else
#define GUB_HD inline
#endif

namespace gub {

// ---- Go numeric semantics -----------------------------------------------------------------------------------
// int64 arithmetic wraps (Go spec); C++ signed overflow is undefined, so go through uint64.
GUB_HD int64_t wadd(int64_t a, int64_t b) { return (int64_t)((uint64_t)a + (uint64_t)b); }
GUB_HD int64_t wsub(int64_t a, int64_t b) { return (int64_t)((uint64_t)a - (uint64_t)b); }
GUB_HD int64_t wmul(int64_t a, int64_t b) { return (int64_t)((uint64_t)a * (uint64_t)b); }

// int64(float64) on amd64 Go is CVTTSD2SI: truncate toward zero; NaN and anything outside int64 give INT64_MIN.
// cvt.rzi.s64.f64 saturates instead (NaN -> 0, +big -> INT64_MAX), so patch those cases.
GUB_HD int64_t f2i(double f) {
#if defined(__CUDA_ARCH__)
  long long r = __double2ll_rz(f);
  if (!(f < 9223372036854775808.0)) r = (long long)0x8000000000000000ULL;  // NaN, +Inf, >= 2^63
  return (int64_t)r;
#else
  return (int64_t)_mm_cvttsd_si64(_mm_set_sd(f));
#endif
}
GUB_HD double i2f(int64_t i) { return (double)i; }  // CVTSI2SD / cvt.rn.f64.s64: round to nearest even
GUB_HD uint64_t f2bits(double f) {
#if defined(__CUDA_ARCH__)
  return (uint64_t)__double_as_longlong(f);
#else
  uint64_t u; __builtin_memcpy(&u, &f, 8); return u;
#endif
}
GUB_HD double bits2f(uint64_t u) {
#if defined(__CUDA_ARCH__)
  return __longlong_as_double((long long)u);
#else
  double f; __builtin_memcpy(&f, &u, 8); return f;
#endif
}

// ---- slot image ---------------------------------------------------------------------------------------------
enum : uint32_t {
  F_LEAKY = 1u,  // Value is *LeakyBucketItem (else *TokenBucketItem)
  F_OVER = 2u,   // TokenBucketItem.Status == OVER_LIMIT (sticky, :168)
  F_LIVE = 4u,   // the cache holds an item for this key
  F_INVALID_AT = 8u,  // CacheItem.InvalidAt != 0 (set by Store / Loader plugins only): the value lives in the table's side index
  F_STALE = 16u,      // InvalidAt < now, found when the slot was opened; never stored in the table (cursor_close drops it)
};

struct Bucket {
  uint64_t key;   // remapped XXH64
  uint64_t tag;   // FNV-1 >> 8
  int64_t limit, duration;
  uint64_t rem;   // token: int64 Remaining; leaky: IEEE-754 bits of float64 Remaining
  int64_t stamp;  // token CreatedAt / leaky UpdatedAt
  int64_t burst;  // leaky only
  int64_t expire; // CacheItem.ExpireAt
  uint32_t flags;
};

GUB_HD bool bucket_equal(const Bucket& a, const Bucket& b) {
  return a.flags == b.flags && a.limit == b.limit && a.duration == b.duration && a.rem == b.rem && a.stamp == b.stamp &&
         a.burst == b.burst && a.expire == b.expire;
}

struct Delta {  // counter increments produced by applying requests
  uint32_t over, hit, miss;
};

GUB_HD gub_resp mk_resp(uint32_t status, int64_t limit, int64_t remaining, int64_t reset) {
  gub_resp r;
  r.status = status; r.err_code = 0; r.limit = limit; r.remaining = remaining; r.reset_time = reset;
  return r;
}
GUB_HD gub_resp mk_err(uint32_t code) {
  gub_resp r;
  r.status = 0; r.err_code = code; r.limit = 0; r.remaining = 0; r.reset_time = 0;
  return r;
}

// interval.go:117-148 via the host-computed per-batch table
GUB_HD uint32_t greg_expiration(const gub_clock& clk, int64_t d, int64_t* out) {
  if (d == 3) return GUB_ERR_GREGORIAN_WEEKS;
  if (d < 0 || d > 5) return GUB_ERR_GREGORIAN_INVALID;
  *out = clk.greg_expire[d];
  return 0;
}
GUB_HD uint32_t greg_duration(const gub_clock& clk, int64_t d, int64_t* out) {
  if (d == 3) return GUB_ERR_GREGORIAN_WEEKS;
  if (d < 0 || d > 5) return GUB_ERR_GREGORIAN_INVALID;
  *out = clk.greg_duration[d];
  return 0;
}

GUB_HD bool req_same(const gub_req& a, const gub_req& b) {
  return a.key_xxh64 == b.key_xxh64 && a.key_fnv1 == b.key_fnv1 && a.hits == b.hits && a.limit == b.limit &&
         a.duration == b.duration && a.burst == b.burst && a.created_at == b.created_at && a.algorithm == b.algorithm &&
         a.behavior == b.behavior;
}

// ---- one request against one bucket -------------------------------------------------------------------------
GUB_HD gub_resp apply_one(Bucket& b, const gub_req& rq, const gub_clock& clk, Delta& d) {
  const uint32_t algo = rq.algorithm, beh = rq.behavior;
  if (algo > 1u) return mk_err(GUB_ERR_INVALID_ALGORITHM);  // workers.go:317-320: the cache is never touched
  const bool owner = (beh & GUB_REQ_IS_OWNER) != 0;
  const bool greg = (beh & GUB_BEHAVIOR_DURATION_IS_GREGORIAN) != 0;
  const bool reset = (beh & GUB_BEHAVIOR_RESET_REMAINING) != 0;
  const bool drain = (beh & GUB_BEHAVIOR_DRAIN_OVER_LIMIT) != 0;
  const int64_t hits = rq.hits, limit = rq.limit, created = rq.created_at;

  // GetItem: an entry past its InvalidAt or its ExpireAt is removed and reported as a miss (cache.go:43-57, lrucache.go:115-119;
  // strict '<').  Only here, after the algorithm check: a rejected request never reaches the cache (workers.go:317-320).
  if (b.flags & F_STALE) b.flags &= ~(F_LIVE | F_INVALID_AT | F_STALE);
  if ((b.flags & F_LIVE) && b.expire < clk.now_ms) b.flags &= ~F_LIVE;
  bool have = (b.flags & F_LIVE) != 0;
  if (have) d.hit++; else d.miss++;

  if (algo == GUB_TOKEN_BUCKET) {
    if (have) {
      if (reset) {  // :78-90 the item is deleted and Hits are ignored
        b.flags &= ~F_LIVE;
        return mk_resp(GUB_UNDER_LIMIT, limit, limit, 0);
      }
      if (b.flags & F_LEAKY) {  // :91-103 algorithm switch: remove, then start over
        b.flags &= ~F_LIVE;
        have = false;
      }
    }
    if (have) {
      int64_t rem = (int64_t)b.rem;
      if (b.limit != limit) {  // :106-113
        rem = wadd(rem, wsub(limit, b.limit));
        if (rem < 0) rem = 0;
        b.limit = limit;
      }
      uint32_t status = (b.flags & F_OVER) ? GUB_OVER_LIMIT : GUB_UNDER_LIMIT;  // :116 the stored, sticky status
      int64_t shown = rem, reset_time = b.expire;                               // :115-120
      if (b.duration != rq.duration) {                                          // :123-147
        int64_t expire = wadd(b.stamp, rq.duration);
        if (greg) {
          uint32_t e = greg_expiration(clk, rq.duration, &expire);
          if (e) { b.rem = (uint64_t)rem; return mk_err(e); }  // the limit delta above has already been stored
        }
        if (expire <= created) {  // :136-142 renew; the response keeps the pre-renewal Remaining
          expire = wadd(created, rq.duration);
          b.stamp = created;
          rem = b.limit;
        }
        b.expire = expire;
        b.duration = rq.duration;
        reset_time = expire;
      }
      if (hits != 0) {  // :157
        if (shown == 0 && hits > 0) {  // :162-170
          if (owner) d.over++;
          status = GUB_OVER_LIMIT;
          b.flags |= F_OVER;
        } else if (rem == hits) {  // :173-178
          rem = 0; shown = 0;
        } else if (hits > rem) {  // :182-194
          if (owner) d.over++;
          status = GUB_OVER_LIMIT;
          if (drain) { rem = 0; shown = 0; }
        } else {  // :196-198
          rem = wsub(rem, hits);
          shown = rem;
        }
      }
      b.rem = (uint64_t)rem;
      return mk_resp(status, limit, shown, reset_time);
    }
    // tokenBucketNewItem :206-257
    int64_t expire = wadd(created, rq.duration);
    int64_t rem = wsub(limit, hits);
    if (greg) {
      uint32_t e = greg_expiration(clk, rq.duration, &expire);
      if (e) return mk_err(e);
    }
    uint32_t status = GUB_UNDER_LIMIT;
    int64_t shown = rem;
    if (hits > limit) {  // :240-248
      if (owner) d.over++;
      status = GUB_OVER_LIMIT;
      shown = limit; rem = limit;
    }
    b.flags = F_LIVE;
    b.limit = limit; b.duration = rq.duration; b.rem = (uint64_t)rem; b.stamp = created; b.burst = 0; b.expire = expire;
    return mk_resp(status, limit, shown, expire);
  }

  // ---- leaky bucket :260-493
  const int64_t burst = rq.burst == 0 ? limit : rq.burst;  // :264-266
  if (have && !(b.flags & F_LEAKY)) {                      // :308-318
    b.flags &= ~F_LIVE;
    have = false;
  }
  if (have) {
    double rem = bits2f(b.rem);
    if (reset) rem = i2f(burst);  // :320-322
    if (b.burst != burst) {       // :325-330
      if (burst > f2i(rem)) rem = i2f(burst);
      b.burst = burst;
    }
    b.limit = limit;            // :332
    b.duration = rq.duration;   // :333
    int64_t duration = rq.duration;
    double rate = i2f(duration) / i2f(limit);  // :336
    if (greg) {                                // :338-354
      int64_t gd, ge;
      uint32_t e = greg_duration(clk, rq.duration, &gd);
      if (!e) e = greg_expiration(clk, rq.duration, &ge);
      if (e) { b.rem = f2bits(rem); return mk_err(e); }
      rate = i2f(gd) / i2f(limit);
      duration = wsub(ge, clk.now_ms);
    }
    if (hits != 0) b.expire = wadd(created, duration);  // :356-358
    const int64_t elapsed = wsub(created, b.stamp);     // :361
    const double leak = i2f(elapsed) / rate;            // :362
    if (f2i(leak) > 0) {                                // :364-367
      rem += leak;
      b.stamp = created;
    }
    if (f2i(rem) > b.burst) rem = i2f(b.burst);  // :369-371
    const int64_t rate_i = f2i(rate);
    int64_t shown = f2i(rem);
    uint32_t status = GUB_UNDER_LIMIT;
    int64_t reset_time = wadd(created, wmul(wsub(b.limit, shown), rate_i));  // :373-378
    if (shown == 0 && hits > 0) {                                             // :389-395
      if (owner) d.over++;
      status = GUB_OVER_LIMIT;
    } else if (shown == hits) {  // :398-403 (also fires for Hits == 0 with Remaining in [0,1): the fraction is dropped)
      rem = 0.0;
      shown = 0;
      reset_time = wadd(created, wmul(wsub(b.limit, 0), rate_i));
    } else if (hits > shown) {  // :407-420
      if (owner) d.over++;
      status = GUB_OVER_LIMIT;
      if (drain) { rem = 0.0; shown = 0; }
    } else if (hits != 0) {  // :423-430
      rem -= i2f(hits);
      shown = f2i(rem);
      reset_time = wadd(created, wmul(wsub(b.limit, shown), rate_i));
    }
    b.rem = f2bits(rem);
    return mk_resp(status, b.limit, shown, reset_time);
  }
  // leakyBucketNewItem :437-493
  int64_t duration = rq.duration;
  const double rate = i2f(duration) / i2f(limit);  // :440 the raw duration even under Gregorian
  if (greg) {
    int64_t ge;
    uint32_t e = greg_expiration(clk, rq.duration, &ge);
    if (e) return mk_err(e);
    duration = wsub(ge, clk.now_ms);  // :449
  }
  const int64_t rate_i = f2i(rate);
  double rem = i2f(wsub(burst, hits));
  int64_t shown = wsub(burst, hits);
  uint32_t status = GUB_UNDER_LIMIT;
  int64_t reset_time = wadd(created, wmul(wsub(limit, shown), rate_i));  // :461-466
  if (hits > burst) {                                                    // :469-477
    if (owner) d.over++;
    status = GUB_OVER_LIMIT;
    shown = 0;
    reset_time = wadd(created, wmul(limit, rate_i));
    rem = 0.0;
  }
  b.flags = F_LIVE | F_LEAKY;
  b.limit = limit; b.duration = duration; b.rem = f2bits(rem); b.stamp = created; b.burst = burst;
  b.expire = wadd(created, duration);  // :480
  return mk_resp(status, limit, shown, reset_time);
}

// ---- m identical requests against one bucket ----------------------------------------------------------------
// A hot key can occur thousands of times in one batch (Zipf traffic), usually with identical parameters.  Applying
// the same request repeatedly has only three regimes: a few irregular steps, a run of plain subtractions
// ("linear": Remaining -= Hits with nothing else changing), and a fixed point (state stops changing, so the response
// repeats).  plan_run() walks the m applications exactly — apply_one() for irregular steps, closed forms for the two
// regular regimes — and records the result as a short list of pieces from which any rank's response can be evaluated
// independently (eval_piece), so a thread block can fill in thousands of responses in parallel.

enum : uint32_t { P_EXPLICIT = 0, P_LINEAR = 1, P_FIXED = 2 };

struct Piece {
  uint32_t start;  // first rank covered (rank 0 = first application)
  uint32_t kind;
  gub_resp resp;   // EXPLICIT/FIXED: the response.  LINEAR: the response of the piece's first rank
  int64_t hits;    // LINEAR: Remaining decreases by this much per rank
  int64_t created; // LINEAR leaky: reset_time = created + (limit - remaining) * rate_i
  int64_t rate_i;
  uint32_t leaky;
  uint32_t _pad;
};

// Number of further applications of `rq` that are guaranteed to be plain subtractions, given the bucket state
// *after at least one application of the same request in this batch*.  0 when the regime does not apply.
GUB_HD uint64_t linear_steps(const Bucket& b, const gub_req& rq, const gub_clock& clk, int64_t* rate_i_out) {
  const uint32_t beh = rq.behavior;
  const int64_t h = rq.hits;
  *rate_i_out = 0;
  if (rq.algorithm > 1u || !(b.flags & F_LIVE) || h <= 0) return 0;
  if (beh & GUB_BEHAVIOR_RESET_REMAINING) return 0;
  if (b.expire < clk.now_ms) return 0;
  if (b.limit != rq.limit) return 0;
  if (rq.algorithm == GUB_TOKEN_BUCKET) {
    if ((b.flags & F_LEAKY) || b.duration != rq.duration) return 0;
    const int64_t R = (int64_t)b.rem;
    if (R <= h) return 0;
    return (uint64_t)((R - 1) / h);  // steps j = 0.. while R - j*h > h
  }
  if (!(b.flags & F_LEAKY)) return 0;
  const int64_t burst = rq.burst == 0 ? rq.limit : rq.burst;
  if (b.burst != burst || b.duration != rq.duration) return 0;
  int64_t duration = rq.duration;
  double rate = i2f(duration) / i2f(rq.limit);
  if (beh & GUB_BEHAVIOR_DURATION_IS_GREGORIAN) {
    int64_t gd, ge;
    if (greg_duration(clk, rq.duration, &gd) || greg_expiration(clk, rq.duration, &ge)) return 0;
    rate = i2f(gd) / i2f(rq.limit);
    duration = wsub(ge, clk.now_ms);
  }
  if (b.expire != wadd(rq.created_at, duration)) return 0;                 // :356-358 would move ExpireAt
  if (f2i(i2f(wsub(rq.created_at, b.stamp)) / rate) > 0) return 0;         // :364 would leak
  const double rem = bits2f(b.rem);
  if (!(rem > 0.0 && rem < 4503599627370496.0)) return 0;                  // exact integer steps need |rem| < 2^52
  const int64_t I = f2i(rem);
  if (I > b.burst || I <= h) return 0;                                     // :369 clamp, :398/:407 not plain
  *rate_i_out = f2i(rate);
  return (uint64_t)((I - 1) / h);
}

// Response of rank `rank` (>= p.start) inside piece p.
GUB_HD gub_resp eval_piece(const Piece& p, uint32_t rank) {
  if (p.kind != P_LINEAR) return p.resp;
  gub_resp r = p.resp;
  const int64_t j = (int64_t)(rank - p.start);
  r.remaining = wsub(p.resp.remaining, wmul(j, p.hits));
  if (p.leaky) r.reset_time = wadd(p.created, wmul(wsub(r.limit, r.remaining), p.rate_i));
  return r;
}

// Walks m applications of rq on b.  Pieces are appended to `pieces` (capacity cap); returns the number of ranks
// covered (== m unless the piece buffer filled up, in which case the caller continues from that rank, e.g. with
// apply_one()).  *npieces receives the number of pieces written.  Counter deltas are accumulated exactly.
GUB_HD uint32_t plan_run(Bucket& b, const gub_req& rq, uint32_t m, const gub_clock& clk, Delta& d, Piece* pieces,
                         uint32_t cap, uint32_t* npieces) {
  uint32_t rank = 0, np = 0;
  while (rank < m && np < cap) {
    const Bucket before = b;
    Delta d1 = {0, 0, 0};
    const gub_resp resp = apply_one(b, rq, clk, d1);
    d.over += d1.over; d.hit += d1.hit; d.miss += d1.miss;
    Piece& p = pieces[np++];
    p.start = rank; p.kind = P_EXPLICIT; p.resp = resp; p.hits = 0; p.created = 0; p.rate_i = 0; p.leaky = 0; p._pad = 0;
    rank++;
    if (rank == m) break;
    if (bucket_equal(before, b)) {
      // Fixed point: the same (state, request) pair recurs, so every later response and counter delta is the same.
      // (An invalid algorithm or an erroring request on a dead bucket also lands here.)
      p.kind = P_FIXED;
      const uint32_t left = m - rank;
      d.over += d1.over * left; d.hit += d1.hit * left; d.miss += d1.miss * left;
      rank = m;
      break;
    }
    int64_t rate_i;
    uint64_t q = linear_steps(b, rq, clk, &rate_i);
    if (q > (uint64_t)(m - rank)) q = (uint64_t)(m - rank);
    if (q > 0 && np < cap) {
      Piece& l = pieces[np++];
      const bool leaky = (b.flags & F_LEAKY) != 0;
      const int64_t cur = leaky ? f2i(bits2f(b.rem)) : (int64_t)b.rem;
      const int64_t first = cur - rq.hits;
      l.start = rank; l.kind = P_LINEAR; l.hits = rq.hits; l.created = rq.created_at; l.rate_i = rate_i; l.leaky = leaky; l._pad = 0;
      l.resp = mk_resp(leaky ? (uint32_t)GUB_UNDER_LIMIT : ((b.flags & F_OVER) ? (uint32_t)GUB_OVER_LIMIT : (uint32_t)GUB_UNDER_LIMIT),
                       rq.limit, first,
                       leaky ? wadd(rq.created_at, wmul(wsub(rq.limit, first), rate_i)) : b.expire);
      const int64_t total = (int64_t)q * rq.hits;  // <= Remaining: no overflow
      if (leaky) b.rem = f2bits(bits2f(b.rem) - i2f(total));  // exact: see linear_steps()
      else b.rem = (uint64_t)((int64_t)b.rem - total);
      d.hit += (uint32_t)q;
      rank += (uint32_t)q;
    }
  }
  *npieces = np;
  return rank;
}

// Response of the `target`-th (0-based) of a run of identical requests `rq` against bucket b, without materialising a
// plan: walks the same regimes as plan_run() and stops at `target`.  On return b is the state after rank `target` and
// d holds the counter deltas of ranks 0..target — so the caller holding the LAST rank of the run ends up with the run's
// final state and total deltas, while every other member of the run computes only its own response.  This lets every
// member of a hot key's run be evaluated by its own thread, in parallel, with no ordering structure beyond its rank.
GUB_HD gub_resp run_to_rank(Bucket& b, const gub_req& rq, uint32_t target, const gub_clock& clk, Delta& d) {
  uint32_t rank = 0;
  for (;;) {
    const Bucket before = b;
    Delta d1 = {0, 0, 0};
    const gub_resp resp = apply_one(b, rq, clk, d1);
    d.over += d1.over; d.hit += d1.hit; d.miss += d1.miss;
    if (rank == target) return resp;
    rank++;
    if (bucket_equal(before, b)) {  // fixed point: ranks rank..target repeat this response and these deltas
      const uint32_t left = target - rank + 1;
      d.over += d1.over * left; d.hit += d1.hit * left; d.miss += d1.miss * left;
      return resp;
    }
    int64_t rate_i;
    const uint64_t q = linear_steps(b, rq, clk, &rate_i);
    if (q > 0) {
      const uint64_t avail = (uint64_t)(target - rank) + 1;  // ranks rank..target
      const uint64_t steps = q < avail ? q : avail;
      const bool leaky = (b.flags & F_LEAKY) != 0;
      const int64_t total = (int64_t)steps * rq.hits;  // <= Remaining: no overflow
      int64_t shown;
      if (leaky) {
        const double rem = bits2f(b.rem) - i2f(total);  // exact: see linear_steps()
        b.rem = f2bits(rem);
        shown = f2i(rem);
      } else {
        shown = (int64_t)b.rem - total;
        b.rem = (uint64_t)shown;
      }
      d.hit += (uint32_t)steps;
      rank += (uint32_t)steps;
      if (steps == avail) {  // the target is the last of these plain subtractions
        return mk_resp(leaky ? (uint32_t)GUB_UNDER_LIMIT : ((b.flags & F_OVER) ? (uint32_t)GUB_OVER_LIMIT : (uint32_t)GUB_UNDER_LIMIT), rq.limit, shown,
                       leaky ? wadd(rq.created_at, wmul(wsub(rq.limit, shown), rate_i)) : b.expire);
      }
    }
  }
}

}  // namespace gub
