// TEST-ONLY: the CPU emulation of the kernels (tests/kernel_emu_harness.cpp, included whole) plus the wire-format entry:
// emu_submit_proto is gub_submit_proto_async's sequence (gub_api.cu) on an emulated table, one call at a time.  Built by
// tests/_proto_emu.py with g++; never part of the product library.
#include "kernel_emu_harness.cpp"
#include "../gubernator_b200/csrc/gub_proto.cuh"

extern "C" {

// out: out_cap bytes; out_off: n_msgs + 1; status: n_msgs.  Returns 0, or -1 when the host-side checks refuse the call.
int emu_submit_proto(void* tv, const uint8_t* packed, uint64_t packed_bytes, uint32_t n_msgs, const gub_clock* clk, uint8_t* out,
                     uint64_t out_cap, unsigned long long* out_off, uint32_t* status) {
  EmuTable* t = static_cast<EmuTable*>(tv);
  ProtoPlan P;
  if (n_msgs == 0) { out_off[0] = 0; return 0; }
  if (proto_plan(packed, packed_bytes, n_msgs, out_cap, P)) return -1;
  const size_t slots = std::max<size_t>(P.slots, 1), msgs = (size_t)n_msgs + 1, bytes = std::max<size_t>(P.msg_bytes, 1);
  std::vector<uint8_t> dpk(packed, packed + P.bytes_at + P.msg_bytes);  // the device copy
  uint32_t n_eval = 0;
  ProtoArgs A;
  std::memset(&A, 0, sizeof A);
  A.created = reinterpret_cast<const int64_t*>(dpk.data());
  A.offs = reinterpret_cast<const uint32_t*>(dpk.data() + P.offsets_at);
  A.bytes = dpk.data() + P.bytes_at;
  A.n_msgs = n_msgs;
  A.smem = P.smem;
  A.slot_base = zalloc<uint32_t>(msgs); A.batch_base = zalloc<uint32_t>(msgs); A.mcount = zalloc<uint32_t>(msgs);
  A.meval = zalloc<uint32_t>(msgs); A.mstatus = zalloc<uint32_t>(msgs); A.msize = zalloc<uint32_t>(msgs);
  A.moff = zalloc<unsigned long long>(msgs); A.items = zalloc<ProtoItem>(slots); A.sreq = zalloc<gub_req>(slots);
  A.keys = zalloc<uint8_t>(bytes); A.stage = zalloc<uint8_t>(bytes * PROTO_OUT_FACTOR);
  gub_req* reqs = zalloc<gub_req>(slots);
  gub_resp* resp = zalloc<gub_resp>(slots);
  A.reqs = reqs; A.resp = resp; A.n_eval = &n_eval; A.out = out; A.out_off = out_off; A.out_status = status;
  emu::launch(k_proto_scan, 1u, PROTO_SCAN_THREADS, A, 0u);
  emu::launch(k_proto_decode, n_msgs, PROTO_THREADS, A);
  emu::launch(k_proto_scan, 1u, PROTO_SCAN_THREADS, A, 1u);
  emu::launch(k_proto_compact, n_msgs, PROTO_THREADS, A);
  if (n_eval) submit_impl(t, reqs, n_eval, nullptr, clk, resp);
  emu::launch(k_proto_encode, n_msgs, PROTO_THREADS, A);
  emu::launch(k_proto_scan, 1u, PROTO_SCAN_THREADS, A, 2u);
  emu::launch(k_proto_copy_out, n_msgs, PROTO_THREADS, A);
  void* all[] = {A.slot_base, A.batch_base, A.mcount, A.meval, A.mstatus, A.msize, A.moff, A.items, A.sreq, A.keys, A.stage, reqs, resp};
  for (void* p : all) std::free(p);
  return 0;
}

}  // extern "C"
