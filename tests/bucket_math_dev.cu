// TEST-ONLY device build of gubernator_b200/csrc/bucket_math.cuh, with the product library's nvcc flags (gubernator_b200/build.py
// NVCC_FLAGS: sm_90a, --fmad=false).  Its entries have the signatures of tests/host_math_harness.cpp's element-wise entries, so one
// test hands the same arrays to the host build and to this one and compares the outputs bit for bit.  Built by
// tests/_host_math.py build_dev() (called from build()); never part of the product library.
#include <cuda_runtime.h>

#include <cstring>

#include "../gubernator_b200/csrc/bucket_math.cuh"

using namespace gub;

namespace {

cudaError_t g_err = cudaSuccess;

__global__ void k_f2i(const double* x, int64_t* out, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = f2i(x[i]);
}
// Control: the bare saturating conversion, without f2i's patch for NaN and values >= 2^63.
__global__ void k_f2i_bare(const double* x, int64_t* out, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (int64_t)__double2ll_rz(x[i]);
}
// Probe: the bits add.f64 returns, for reporting what the device does with NaN operands.
__global__ void k_add(const uint64_t* a, const uint64_t* b, uint64_t* out, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = f2bits(bits2f(a[i]) + bits2f(b[i]));
}
__global__ void k_apply_one(Bucket* b, const gub_req* rq, gub_clock clk, size_t n, gub_resp* out, Delta* d) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Bucket bi = b[i];
  Delta di = {0, 0, 0};
  out[i] = apply_one(bi, rq[i], clk, di);
  b[i] = bi; d[i] = di;
}
__global__ void k_run_to_rank(Bucket* b, const gub_req* rq, const uint32_t* target, gub_clock clk, size_t n, gub_resp* out, Delta* d) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Bucket bi = b[i];
  Delta di = {0, 0, 0};
  out[i] = run_to_rank(bi, rq[i], target[i], clk, di);
  b[i] = bi; d[i] = di;
}

unsigned grid(size_t n) { return (unsigned)((n + 255) / 256); }

// Copies every (host pointer, bytes, copy back) buffer to the device, runs `launch` on the device pointers, copies the outputs back.
struct Buf { void* host; size_t bytes; bool out; void* dev; };
template <size_t N, class F> void run(Buf (&bufs)[N], F launch) {
  cudaError_t e = cudaSuccess;
  for (Buf& b : bufs) { b.dev = nullptr; if (e == cudaSuccess) e = cudaMalloc(&b.dev, b.bytes ? b.bytes : 1); }
  for (Buf& b : bufs) if (e == cudaSuccess && b.bytes) e = cudaMemcpy(b.dev, b.host, b.bytes, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) { launch(); e = cudaGetLastError(); }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  for (Buf& b : bufs) if (e == cudaSuccess && b.out && b.bytes) e = cudaMemcpy(b.host, b.dev, b.bytes, cudaMemcpyDeviceToHost);
  for (Buf& b : bufs) if (b.dev) cudaFree(b.dev);
  g_err = e;
}

}  // namespace

extern "C" {

// cudaError_t of the last call (0: it ran)
int bmd_error() { return (int)g_err; }

void hm_f2i(const double* x, int64_t* out, size_t n) {
  Buf b[] = {{(void*)x, n * 8, false}, {out, n * 8, true}};
  if (n) run(b, [&] { k_f2i<<<grid(n), 256>>>((const double*)b[0].dev, (int64_t*)b[1].dev, n); });
}
void bmd_f2i_bare(const double* x, int64_t* out, size_t n) {
  Buf b[] = {{(void*)x, n * 8, false}, {out, n * 8, true}};
  if (n) run(b, [&] { k_f2i_bare<<<grid(n), 256>>>((const double*)b[0].dev, (int64_t*)b[1].dev, n); });
}
void bmd_add(const uint64_t* x, const uint64_t* y, uint64_t* out, size_t n) {
  Buf b[] = {{(void*)x, n * 8, false}, {(void*)y, n * 8, false}, {out, n * 8, true}};
  if (n) run(b, [&] { k_add<<<grid(n), 256>>>((const uint64_t*)b[0].dev, (const uint64_t*)b[1].dev, (uint64_t*)b[2].dev, n); });
}
void hm_apply_one(Bucket* bk, const gub_req* rq, const gub_clock* clk, size_t n, gub_resp* out, Delta* d) {
  Buf b[] = {{bk, n * sizeof(Bucket), true}, {(void*)rq, n * sizeof(gub_req), false}, {out, n * sizeof(gub_resp), true}, {d, n * sizeof(Delta), true}};
  if (n) run(b, [&] { k_apply_one<<<grid(n), 256>>>((Bucket*)b[0].dev, (const gub_req*)b[1].dev, *clk, n, (gub_resp*)b[2].dev, (Delta*)b[3].dev); });
}
void hm_run_to_rank(Bucket* bk, const gub_req* rq, const uint32_t* target, const gub_clock* clk, size_t n, gub_resp* out, Delta* d) {
  Buf b[] = {{bk, n * sizeof(Bucket), true}, {(void*)rq, n * sizeof(gub_req), false}, {(void*)target, n * 4, false},
             {out, n * sizeof(gub_resp), true}, {d, n * sizeof(Delta), true}};
  if (n) run(b, [&] { k_run_to_rank<<<grid(n), 256>>>((Bucket*)b[0].dev, (const gub_req*)b[1].dev, (const uint32_t*)b[2].dev, *clk, n,
                                                      (gub_resp*)b[3].dev, (Delta*)b[4].dev); });
}
size_t hm_sizeof_bucket() { return sizeof(Bucket); }

}  // extern "C"
