// TEST-ONLY: the CPU emulation of the kernels (tests/kernel_emu_harness.cpp, included whole) plus the wire-format entry on the ring:
// emu_p2p_step_proto is gub_p2p_step_proto_local_all's sequence (gub_api.cu) on an emulated ring: every shard's decode, the S steps of
// emu_p2p_step on the chunks of the dense batches, every shard's encode.  Built by tests/_ring_proto_emu.py with g++; never part of the
// product library.
#include "kernel_emu_harness.cpp"
#include "../gubernator_b200/csrc/gub_proto.cuh"

namespace {
struct EmuProtoShard {
  ProtoPlan P{};
  ProtoArgs A{};
  std::vector<uint8_t> dpk;  // the device copy of the packed buffer
  gub_req* reqs = nullptr;   // the dense batch
  gub_resp* resp = nullptr;  // its responses
  uint32_t n_msgs = 0, n_eval = 0;
};

void free_shard(EmuProtoShard& h) {
  ProtoArgs& A = h.A;
  void* all[] = {A.slot_base, A.batch_base, A.mcount, A.meval, A.mstatus, A.msize, A.moff, A.items, A.sreq, A.keys, A.stage, h.reqs, h.resp};
  for (void* p : all) std::free(p);
}
}  // namespace

extern "C" {

// Shard r: packed[r] (packed_bytes[r], n_msgs[r] messages) in the layout of gub_proto_layout; out[r] (out_cap[r] bytes), out_off[r]
// (n_msgs[r] + 1) and status[r] (n_msgs[r]) its outputs.  self_global != 0: GLOBAL mode (as emu_p2p_step).  timeout[r] (optional, with
// n_timeout[r] entries): indices into shard r's dense batch whose response is replaced, after the steps, by what k_p2p_collect writes
// for an owner that never answered.  owners_out[r] (optional, GLOBAL mode): the ring owner of every item of shard r's dense batch, as
// the routing recorded it for the hits queue.  *steps_out = S.  Returns -1 when the host-side checks refuse the call (nothing has run), else the
// flag-wait error of the steps (0).
int emu_p2p_step_proto(void* pv, const uint8_t* const* packed, const uint64_t* packed_bytes, const uint32_t* n_msgs, uint32_t force_global,
                       const gub_clock* clk, uint8_t* const* out, const uint64_t* out_cap, unsigned long long* const* out_off,
                       uint32_t* const* status, uint32_t self_global, const uint32_t* const* timeout, const uint32_t* n_timeout,
                       uint8_t* const* owners_out, uint32_t* steps_out) {
  EmuP2P* p = static_cast<EmuP2P*>(pv);
  const uint32_t W = p->world;
  std::vector<EmuProtoShard> sh(W);
  for (uint32_t r = 0; r < W; r++) {  // the host-side checks of every shard first
    sh[r].n_msgs = n_msgs[r];
    if (n_msgs[r] && proto_plan(packed[r], packed_bytes[r], n_msgs[r], out_cap[r], sh[r].P)) return -1;
  }
  for (uint32_t r = 0; r < W; r++) {  // decode
    EmuProtoShard& h = sh[r];
    if (!h.n_msgs) continue;
    const ProtoPlan& P = h.P;
    const size_t slots = std::max<size_t>(P.slots, 1), msgs = (size_t)h.n_msgs + 1, bytes = std::max<size_t>(P.msg_bytes, 1);
    h.dpk.assign(packed[r], packed[r] + P.bytes_at + P.msg_bytes);
    ProtoArgs& A = h.A;
    std::memset(&A, 0, sizeof A);
    A.created = reinterpret_cast<const int64_t*>(h.dpk.data());
    A.offs = reinterpret_cast<const uint32_t*>(h.dpk.data() + P.offsets_at);
    A.bytes = h.dpk.data() + P.bytes_at;
    A.n_msgs = h.n_msgs;
    A.smem = P.smem;
    A.force_global = force_global;
    A.slot_base = zalloc<uint32_t>(msgs); A.batch_base = zalloc<uint32_t>(msgs); A.mcount = zalloc<uint32_t>(msgs);
    A.meval = zalloc<uint32_t>(msgs); A.mstatus = zalloc<uint32_t>(msgs); A.msize = zalloc<uint32_t>(msgs);
    A.moff = zalloc<unsigned long long>(msgs); A.items = zalloc<ProtoItem>(slots); A.sreq = zalloc<gub_req>(slots);
    A.keys = zalloc<uint8_t>(bytes); A.stage = zalloc<uint8_t>(bytes * PROTO_OUT_FACTOR);
    h.reqs = zalloc<gub_req>(slots); h.resp = zalloc<gub_resp>(slots);
    A.reqs = h.reqs; A.resp = h.resp; A.n_eval = &h.n_eval; A.out = out[r]; A.out_off = out_off[r]; A.out_status = status[r];
    emu::launch(k_proto_scan, 1u, PROTO_SCAN_THREADS, A, 0u);
    emu::launch(k_proto_decode, h.n_msgs, PROTO_THREADS, A);
    emu::launch(k_proto_scan, 1u, PROTO_SCAN_THREADS, A, 1u);
    emu::launch(k_proto_compact, h.n_msgs, PROTO_THREADS, A);
  }
  uint32_t S = 0;
  for (uint32_t r = 0; r < W; r++) S = std::max<uint32_t>(S, (sh[r].n_eval + p->cap - 1) / p->cap);
  int err = 0;
  std::vector<const gub_req*> reqs(W);
  std::vector<gub_resp*> outs(W);
  std::vector<uint32_t> n(W);
  std::vector<uint8_t*> owners(W);
  static uint8_t no_owner;
  static gub_req no_req;
  static gub_resp no_resp;
  for (uint32_t k = 0; k < S; k++) {  // the ring steps, chunk k of every dense batch
    for (uint32_t r = 0; r < W; r++) {
      const uint32_t lo = k * p->cap;
      n[r] = sh[r].n_eval > lo ? std::min<uint32_t>(p->cap, sh[r].n_eval - lo) : 0u;
      reqs[r] = n[r] ? sh[r].reqs + lo : &no_req;
      outs[r] = n[r] ? sh[r].resp + lo : &no_resp;
      owners[r] = owners_out && n[r] ? owners_out[r] + lo : &no_owner;
    }
    err |= emu_p2p_step(p, reqs.data(), n.data(), clk, outs.data(), self_global, owners_out ? owners.data() : nullptr);
  }
  for (uint32_t r = 0; r < W; r++) {  // encode
    EmuProtoShard& h = sh[r];
    if (!h.n_msgs) { out_off[r][0] = 0; continue; }
    for (uint32_t q = 0; timeout && timeout[r] && q < n_timeout[r]; q++) {
      gub_resp& x = h.resp[timeout[r][q]];
      std::memset(&x, 0, sizeof x);
      x.err_code = GUB_ERR_PEER_TIMEOUT;
    }
    emu::launch(k_proto_encode, h.n_msgs, PROTO_THREADS, h.A);
    emu::launch(k_proto_scan, 1u, PROTO_SCAN_THREADS, h.A, 2u);
    emu::launch(k_proto_copy_out, h.n_msgs, PROTO_THREADS, h.A);
    free_shard(h);
  }
  *steps_out = S;
  return err;
}

uint32_t emu_p2p_epoch(void* pv) { return static_cast<EmuP2P*>(pv)->epoch; }

}  // extern "C"
