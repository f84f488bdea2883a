//go:build cgo

// Package gubernator: drop-in replacement for WorkerPool (workers.go:54-61) that evaluates rate limits on an H100
// through libgubernator_b200.so.  NOT COMPILED BY THIS REPOSITORY'S BUILD (it needs no Go toolchain);
// it is written against the reference's exact method set and kept small enough to review by eye.  The same C ABI is
// exercised by the C++ host layer (gubernator_b200/csrc/host_v1.cpp) and the Python tests.
//
// Wiring (one line in NewV1Instance, gubernator.go:129):
//
//	s.workerPool, err = NewB200WorkerPool(&conf)   // instead of NewWorkerPool(&conf)
//
// Build with CGO_ENABLED=1 (the reference Dockerfile sets 0, Dockerfile:22) and
// CGO_LDFLAGS="-L<repo>/gubernator_b200 -lgubernator_b200".
package gubernator

/*
#cgo CFLAGS: -I${SRCDIR}/../include
#cgo LDFLAGS: -lgubernator_b200
#include <stdlib.h>
#include "gubernator_b200.h"
extern int b200StoreGet(void* user, gub_store_rec* misses, size_t n);
*/
import "C"

import (
	"context"
	"runtime/cgo"
	"sync"
	"time"
	"unsafe"

	"github.com/OneOfOne/xxhash"
	"github.com/mailgun/holster/v4/clock"
	"github.com/pkg/errors"
	"github.com/segmentio/fasthash/fnv1"
)

// B200WorkerPool has the method set V1Instance uses on WorkerPool: GetRateLimit (gubernator.go:598, global.go:245),
// Load (:143), Store (:161), AddCacheItem (:452), GetCacheItem, Close (:169).
//
// Concurrency: callers only append to a channel; ONE goroutine (run) owns the pinned arenas, builds the batches, makes the cgo
// call and hands the responses out, so batches never overlap an arena and requests are evaluated in arrival order.
type B200WorkerPool struct {
	conf  *Config
	table *C.gub_table

	in   chan *pendingReq // requests waiting for the next device batch
	quit chan struct{}
	done sync.WaitGroup
	// pinned arenas (gub_host_alloc), owned by run(): the packed key-string batch ([gub_kreq][offsets][key bytes]) and the responses
	packed    unsafe.Pointer
	packedCap int
	resps     unsafe.Pointer
	// with a conf.Store: the change log the device writes (gub_submit_keys_store_async), pinned
	changes, nChanges unsafe.Pointer
	overLimit uint64 // last gub_counters.over_limit seen: the metric is fed from the device's own count
	// key strings by fingerprint, kept only when a Loader needs CacheItem.Key back (store.go:69-78)
	mu   sync.Mutex
	keys map[[2]uint64]string
}

type pendingReq struct {
	req   *RateLimitReq
	state RateLimitReqState
	done  chan pendingResp
}
type pendingResp struct {
	resp *RateLimitResp
	err  error
}

const (
	b200MaxBatch  = 65536                  // device batch; RPCs (<= 1000 items each, gubernator.go:40) are coalesced up to this
	b200BatchWait = 500 * time.Microsecond // same window as BehaviorConfig.BatchWait (config.go:128)
	b200KeyBytes  = 64                     // arena room per key string; longer keys grow the arena
)

func NewB200WorkerPool(conf *Config) (*B200WorkerPool, error) {
	cfg := C.gub_config{
		capacity_slots: C.uint64_t(2 * conf.CacheSize), // load factor <= 0.5; replaces CacheSize/Workers LRUs (workers.go:132)
		max_batch:      b200MaxBatch,
		device:         0,
	}
	p := &B200WorkerPool{conf: conf, in: make(chan *pendingReq, 4*b200MaxBatch), quit: make(chan struct{})}
	if rc := C.gub_create(&cfg, &p.table); rc != 0 {
		return nil, errors.Errorf("gub_create: %s", C.GoString(C.gub_last_error()))
	}
	p.packedCap = b200MaxBatch*(16+4+b200KeyBytes) + 64
	p.packed = C.gub_host_alloc(C.size_t(p.packedCap))
	p.resps = C.gub_host_alloc(C.size_t(b200MaxBatch * 32))
	if conf.Store != nil {
		p.changes = C.gub_host_alloc(C.size_t(b200MaxBatch * C.sizeof_gub_store_rec))
		p.nChanges = C.gub_host_alloc(4)
	}
	if conf.Loader != nil {
		p.keys = make(map[[2]uint64]string)
	}
	p.done.Add(1)
	go p.run()
	return p, nil
}

// GetRateLimit mirrors WorkerPool.GetRateLimit (workers.go:261-290): the caller blocks until its request has been
// evaluated.  Instead of a channel hop to a worker goroutine, the request joins the next device batch.
func (p *B200WorkerPool) GetRateLimit(ctx context.Context, r *RateLimitReq, st RateLimitReqState) (*RateLimitResp, error) {
	pr := &pendingReq{req: r, state: st, done: make(chan pendingResp, 1)}
	select {
	case p.in <- pr:
	case <-ctx.Done():
		return nil, ctx.Err()
	}
	select {
	case out := <-pr.done:
		return out.resp, out.err
	case <-ctx.Done():
		return nil, ctx.Err() // workers.go:278-288
	}
}

// run is the only goroutine that touches the arenas and the device batch path.
func (p *B200WorkerPool) run() {
	defer p.done.Done()
	batch := make([]*pendingReq, 0, b200MaxBatch)
	for {
		batch = batch[:0]
		select {
		case pr := <-p.in:
			batch = append(batch, pr)
		case <-p.quit:
			return
		}
		deadline := time.NewTimer(b200BatchWait)
	fill:
		for len(batch) < b200MaxBatch {
			select {
			case pr := <-p.in:
				batch = append(batch, pr)
			case <-deadline.C:
				break fill
			}
		}
		deadline.Stop()
		p.flush(batch)
	}
}

// flush evaluates one batch: key strings + 16-byte records into the pinned arena, one cgo call (hashing happens on the device:
// gub_submit_keys_async), every caller gets its response.  Called from run() only.
func (p *B200WorkerPool) flush(batch []*pendingReq) {
	n := len(batch)
	// the batch's distinct (limit, duration, burst, algorithm, behaviour) tuples: a deployment has a handful
	type cfgKey struct {
		limit, duration, burst int64
		algo, beh             uint32
	}
	sets := make(map[cfgKey]uint32, 8)
	params := make([]C.gub_params, 0, 8)
	keyBytes := 0
	keys := make([]string, n)
	for i, pr := range batch {
		keys[i] = pr.req.HashKey() // client.go:39-41
		keyBytes += len(keys[i])
	}
	var offAt, bytesAt, total C.size_t
	C.gub_keys_layout(C.size_t(n), C.size_t(keyBytes), &offAt, &bytesAt, &total)
	if int(total) > p.packedCap {
		C.gub_host_free(p.packed)
		p.packedCap = int(total) * 2
		p.packed = C.gub_host_alloc(C.size_t(p.packedCap))
	}
	kreqs := unsafe.Slice((*C.gub_kreq)(p.packed), n)
	offs := unsafe.Slice((*C.uint32_t)(unsafe.Add(p.packed, int(offAt))), n+1)
	blob := unsafe.Slice((*byte)(unsafe.Add(p.packed, int(bytesAt))), keyBytes)
	resps := unsafe.Slice((*C.gub_resp)(p.resps), b200MaxBatch)
	base := *batch[0].req.CreatedAt // defaulted by GetRateLimits (gubernator.go:218-220)
	for _, pr := range batch {
		if *pr.req.CreatedAt < base {
			base = *pr.req.CreatedAt
		}
	}
	at := 0
	for i, pr := range batch {
		r := pr.req
		beh := uint32(r.Behavior) & 0xff
		if pr.state.IsOwner {
			beh |= C.GUB_REQ_IS_OWNER
		}
		ck := cfgKey{r.Limit, r.Duration, r.Burst, uint32(r.Algorithm), beh}
		idx, ok := sets[ck]
		if !ok {
			idx = uint32(len(params))
			sets[ck] = idx
			params = append(params, C.gub_params{limit: C.int64_t(r.Limit), duration: C.int64_t(r.Duration), burst: C.int64_t(r.Burst),
				algorithm: C.uint32_t(r.Algorithm), behavior: C.uint32_t(beh)})
		}
		kreqs[i].hits = C.int64_t(r.Hits)
		kreqs[i].params = C.uint32_t(idx)
		kreqs[i].created_delta = C.int32_t(*r.CreatedAt - base)
		offs[i] = C.uint32_t(at)
		at += copy(blob[at:], keys[i])
		if r.Algorithm == Algorithm_LEAKY_BUCKET && r.Burst == 0 {
			r.Burst = r.Limit // the reference mutates the request (algorithms.go:264-266); keep that visible to callers
		}
	}
	offs[n] = C.uint32_t(at)
	if p.keys != nil { // a Loader wants CacheItem.Key back at Store(): remember the strings by fingerprint
		p.mu.Lock()
		for _, k := range keys {
			p.keys[[2]uint64{xxhash.ChecksumString64S(k, 0), fnv1.HashString64(k) >> 8}] = k
		}
		p.mu.Unlock()
	}
	var clk C.gub_clock
	C.gub_clock_fill(C.int64_t(clock.Now().UnixNano()/1000000), &clk)
	var ticket C.int
	var rc C.int
	if p.conf.Store == nil {
		rc = C.gub_submit_keys_async(p.table, p.packed, total, C.size_t(n), &params[0], C.size_t(len(params)), C.int64_t(base), &clk, &resps[0], &ticket)
	} else {
		// Store.Get runs inside the call (b200StoreGet, once per batch, for its misses); Remove / OnChange are replayed below
		h := cgo.NewHandle(&storeCall{p: p, batch: batch, keys: keys})
		rc = C.gub_submit_keys_store_async(p.table, p.packed, total, C.size_t(n), &params[0], C.size_t(len(params)), C.int64_t(base), &clk,
			C.gub_store_get_fn(C.b200StoreGet), unsafe.Pointer(&h), &resps[0], (*C.gub_store_rec)(p.changes), (*C.uint32_t)(p.nChanges), &ticket)
		h.Delete()
	}
	if rc == 0 {
		rc = C.gub_wait(p.table, ticket)
	}
	if rc == 0 && p.conf.Store != nil {
		// one record per key, ordered by its first request: Remove, then OnChange, as the reference calls them (algorithms.go)
		ctx := context.Background()
		for _, r := range unsafe.Slice((*C.gub_store_rec)(p.changes), int(*(*C.uint32_t)(p.nChanges))) {
			if r.flags&C.GUB_STORE_REMOVE != 0 {
				p.conf.Store.Remove(ctx, keys[r.first])
			}
			if r.flags&C.GUB_STORE_CHANGE != 0 {
				item := p.fromItem(&r.item)
				item.Key = keys[r.first]
				p.conf.Store.OnChange(ctx, batch[r.last].req, item)
			}
		}
	}
	for i, pr := range batch {
		if rc != 0 {
			pr.done <- pendingResp{nil, errors.New(C.GoString(C.gub_last_error()))}
			continue
		}
		o := &resps[i]
		if o.err_code != 0 {
			pr.done <- pendingResp{nil, b200Error(int(o.err_code), pr.req)}
			continue
		}
		pr.done <- pendingResp{&RateLimitResp{
			Status: Status(o.status), Limit: int64(o.limit), Remaining: int64(o.remaining), ResetTime: int64(o.reset_time),
		}, nil}
	}
	// metricOverLimitCounter (algorithms.go:164,184,242,252,...): the device counts exactly those events (owner only, not the
	// sticky-status reads); feed the metric from its counter instead of re-deriving it from the responses
	var c C.gub_counters
	if C.gub_get_counters(p.table, &c) == 0 {
		if d := uint64(c.over_limit) - p.overLimit; d > 0 {
			metricOverLimitCounter.Add(float64(d))
		}
		p.overLimit = uint64(c.over_limit)
	}
}

type storeCall struct {
	p     *B200WorkerPool
	batch []*pendingReq
	keys  []string
}

// b200StoreGet is the batch's Store.Get (algorithms.go:45-51): one call per key that missed, with the key's first request.
//
//export b200StoreGet
func b200StoreGet(user unsafe.Pointer, misses *C.gub_store_rec, n C.size_t) C.int {
	sc := (*(*cgo.Handle)(user)).Value().(*storeCall)
	ms := unsafe.Slice(misses, int(n))
	for i := range ms {
		m := &ms[i]
		item, ok := sc.p.conf.Store.Get(context.Background(), sc.batch[m.first].req)
		if !ok || item == nil {
			continue
		}
		it, known := toItem(sc.keys[m.first], item)
		if !known {
			it.algorithm = -1 // a Value the cache cannot hold: counted as existing, never installed
		}
		m.item = it
		m.flags |= C.GUB_STORE_FOUND
	}
	return 0
}

// b200Error rebuilds the error values handleGetRateLimit returns (workers.go:299-320); V1Instance wraps them further.
func b200Error(code int, r *RateLimitReq) error {
	scope := "Error in tokenBucket"
	if r.Algorithm == Algorithm_LEAKY_BUCKET {
		scope = "Error in leakyBucket"
	}
	switch code {
	case C.GUB_ERR_INVALID_ALGORITHM:
		return errors.Errorf("Invalid rate limit algorithm '%d'", r.Algorithm)
	case C.GUB_ERR_GREGORIAN_WEEKS:
		return errors.Wrap(errors.New("`Duration = GregorianWeeks` not yet supported; consider making a PR!`"), scope)
	case C.GUB_ERR_GREGORIAN_INVALID:
		return errors.Wrap(errors.New("behavior DURATION_IS_GREGORIAN is set; but `Duration` is not a valid gregorian interval"), scope)
	case C.GUB_ERR_PEER_TIMEOUT:
		return errors.New("the owning shard did not answer in time")
	}
	return errors.Errorf("device error %d", code)
}

func toItem(key string, item *CacheItem) (C.gub_item, bool) {
	var it C.gub_item
	it.key_xxh64 = C.uint64_t(xxhash.ChecksumString64S(key, 0))
	it.key_fnv1 = C.uint64_t(fnv1.HashString64(key))
	it.expire_at = C.int64_t(item.ExpireAt)
	it.invalid_at = C.int64_t(item.InvalidAt)
	switch v := item.Value.(type) {
	case *TokenBucketItem:
		it.algorithm = C.GUB_TOKEN_BUCKET
		it.status, it.limit, it.duration, it.remaining, it.stamp = C.int32_t(v.Status), C.int64_t(v.Limit), C.int64_t(v.Duration), C.int64_t(v.Remaining), C.int64_t(v.CreatedAt)
	case *LeakyBucketItem:
		it.algorithm = C.GUB_LEAKY_BUCKET
		it.limit, it.duration, it.remaining_f, it.stamp, it.burst = C.int64_t(v.Limit), C.int64_t(v.Duration), C.double(v.Remaining), C.int64_t(v.UpdatedAt), C.int64_t(v.Burst)
	default:
		return it, false
	}
	return it, true
}

func (p *B200WorkerPool) fromItem(it *C.gub_item) *CacheItem {
	item := &CacheItem{ExpireAt: int64(it.expire_at), InvalidAt: int64(it.invalid_at), Algorithm: Algorithm(it.algorithm)}
	if p.keys != nil {
		p.mu.Lock()
		item.Key = p.keys[[2]uint64{uint64(it.key_xxh64), uint64(it.key_fnv1) >> 8}]
		p.mu.Unlock()
	}
	if it.algorithm == C.GUB_LEAKY_BUCKET {
		item.Value = &LeakyBucketItem{Limit: int64(it.limit), Duration: int64(it.duration), Remaining: float64(it.remaining_f), UpdatedAt: int64(it.stamp), Burst: int64(it.burst)}
	} else {
		item.Value = &TokenBucketItem{Status: Status(it.status), Limit: int64(it.limit), Duration: int64(it.duration), Remaining: int64(it.remaining), CreatedAt: int64(it.stamp)}
	}
	return item
}

// AddCacheItem mirrors workers.go:537 (used by UpdatePeerGlobals, gubernator.go:452).
func (p *B200WorkerPool) AddCacheItem(ctx context.Context, key string, item *CacheItem) error {
	it, ok := toItem(key, item)
	if !ok {
		return nil
	}
	if p.keys != nil {
		p.mu.Lock()
		p.keys[[2]uint64{uint64(it.key_xxh64), uint64(it.key_fnv1) >> 8}] = key
		p.mu.Unlock()
	}
	if C.gub_add_items(p.table, &it, 1) != 0 {
		return errors.New(C.GoString(C.gub_last_error()))
	}
	return nil
}

// GetCacheItem mirrors workers.go:583.
func (p *B200WorkerPool) GetCacheItem(ctx context.Context, key string) (*CacheItem, bool, error) {
	kx := C.uint64_t(xxhash.ChecksumString64S(key, 0))
	kf := C.uint64_t(fnv1.HashString64(key))
	var it C.gub_item
	var found C.uint8_t
	if C.gub_get_items(p.table, &kx, &kf, 1, C.int64_t(MillisecondNow()), &it, &found) != 0 {
		return nil, false, errors.New(C.GoString(C.gub_last_error()))
	}
	if found == 0 {
		return nil, false, nil
	}
	item := p.fromItem(&it)
	item.Key = key
	return item, true, nil
}

// Load mirrors workers.go:329: stream Loader.Load() into the table in bulk.
func (p *B200WorkerPool) Load(ctx context.Context) error {
	ch, err := p.conf.Loader.Load()
	if err != nil {
		return errors.Wrap(err, "Error in loader.Load")
	}
	buf := make([]C.gub_item, 0, 65536)
	flush := func() error {
		if len(buf) == 0 {
			return nil
		}
		if C.gub_add_items(p.table, &buf[0], C.size_t(len(buf))) != 0 {
			return errors.New(C.GoString(C.gub_last_error()))
		}
		buf = buf[:0]
		return nil
	}
	for item := range ch {
		if it, ok := toItem(item.Key, item); ok {
			p.mu.Lock()
			p.keys[[2]uint64{uint64(it.key_xxh64), uint64(it.key_fnv1) >> 8}] = item.Key
			p.mu.Unlock()
			buf = append(buf, it)
			if len(buf) == cap(buf) {
				if err := flush(); err != nil {
					return err
				}
			}
		}
	}
	return flush()
}

// Store mirrors workers.go:451: scan the table and hand every item to Loader.Save().
func (p *B200WorkerPool) Store(ctx context.Context) error {
	var n C.size_t
	if C.gub_size(p.table, &n) != 0 {
		return errors.New(C.GoString(C.gub_last_error()))
	}
	items := make([]C.gub_item, int(n)+1)
	if C.gub_scan(p.table, &items[0], C.size_t(len(items)), &n) != 0 {
		return errors.New(C.GoString(C.gub_last_error()))
	}
	out := make(chan *CacheItem, 500)
	go func() {
		for i := 0; i < int(n) && i < len(items); i++ {
			out <- p.fromItem(&items[i])
		}
		close(out)
	}()
	return p.conf.Loader.Save(out)
}

// Close mirrors workers.go:157.
func (p *B200WorkerPool) Close() error {
	close(p.quit)
	p.done.Wait()
	C.gub_host_free(p.packed)
	C.gub_host_free(p.resps)
	C.gub_host_free(p.changes)
	C.gub_host_free(p.nChanges)
	C.gub_destroy(p.table)
	return nil
}
