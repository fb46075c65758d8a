// cuda_sim.hpp -- just enough of the CUDA runtime and device environment to run the product's
// kernels on the CPU, one simulated thread at a time.
//
// TEST INFRASTRUCTURE (tests/host/make_host_sim.py, tests/test_kernels_on_cpu_sim.py).  "Device"
// memory is host memory, every copy and launch is synchronous, a launch runs the kernel function
// once per (block, thread) with blockIdx / threadIdx set.  Threads of a block therefore never run
// concurrently: fine for these kernels (one pairing per thread; the only barriers are the lock-step
// ones of miller_cc.cuh, which order instruction fetch, not data).  Shared memory is one static
// buffer per host thread, sized like the largest opt-in allocation of an SM.
#pragma once
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

struct uint2 { uint32_t x, y; };
struct alignas(16) uint4 { uint32_t x, y, z, w; };
static inline uint2 make_uint2(uint32_t x, uint32_t y) { return uint2{x, y}; }
static inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return uint4{x, y, z, w}; }
struct dim3 { unsigned x = 1, y = 1, z = 1; dim3() {} dim3(unsigned a) : x(a) {} dim3(int a) : x((unsigned)a) {} dim3(size_t a) : x((unsigned)a) {} };

namespace cusim {
// per host thread: the engine drives each simulated device from its own thread
inline dim3& tid() { static thread_local dim3 v; return v; }
inline dim3& bid() { static thread_local dim3 v; return v; }
inline dim3& bdim() { static thread_local dim3 v; return v; }
inline dim3& gdim() { static thread_local dim3 v; return v; }
inline int& current_device() { static thread_local int d = 0; return d; }
// PBC_SIM_DEVICES=N makes the simulator report N devices (they share the host's memory)
inline int device_count() { const char* e = getenv("PBC_SIM_DEVICES"); int n = e ? atoi(e) : 1; return n > 0 ? n : 1; }
inline uint64_t& launches() { static uint64_t n = 0; return n; }
// optional cap on simulated threads per launch (0 = all): kernels whose padding threads keep
// computing (k_a_miller9's `live` pattern) would otherwise cost a full block per launch
inline size_t& live_threads() { static size_t n = 0; return n; }
// shared memory is poisoned at the start of every block and device allocations at birth, so a
// kernel that reads what it never wrote sees garbage here as it would on the GPU
inline void (*&poison_shared())() { static void (*f)() = nullptr; return f; }
template <class F>
inline void launch(dim3 grid, dim3 block, F&& body) {
  launches()++;
  gdim() = grid; bdim() = block;
  size_t done = 0;
  for (unsigned b = 0; b < grid.x; b++) {
    if (poison_shared()) poison_shared()();
    for (unsigned t = 0; t < block.x; t++) {
      if (live_threads() && done >= live_threads()) return;
      bid() = dim3(b); tid() = dim3(t);
      body();
      done++;
    }
  }
}
}  // namespace cusim
#define threadIdx (::cusim::tid())
#define blockIdx (::cusim::bid())
#define blockDim (::cusim::bdim())
#define gridDim (::cusim::gdim())

static inline void __syncthreads() {}
static inline void __syncwarp() {}
static inline uint32_t __funnelshift_r(uint32_t lo, uint32_t hi, uint32_t s) {
  return (uint32_t)((((uint64_t)hi << 32) | lo) >> (s & 31));
}
static inline uint32_t __byte_perm(uint32_t a, uint32_t b, uint32_t sel) {
  uint64_t v = ((uint64_t)b << 32) | a;
  uint32_t r = 0;
  for (int i = 0; i < 4; i++) r |= (uint32_t)((v >> (8 * ((sel >> (4 * i)) & 7))) & 0xff) << (8 * i);
  return r;
}

// ---- runtime API ----
typedef int cudaError_t;
typedef void* cudaStream_t;
typedef void* cudaEvent_t;
enum { cudaSuccess = 0 };
enum cudaMemcpyKind { cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice, cudaMemcpyDefault };
enum { cudaStreamNonBlocking = 1, cudaHostAllocPortable = 1, cudaFuncAttributeMaxDynamicSharedMemorySize = 8,
       cudaFuncAttributePreferredSharedMemoryCarveout = 9, cudaSharedmemCarveoutMaxShared = 100 };
static inline const char* cudaGetErrorString(cudaError_t) { return "simulated"; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int* d) { *d = ::cusim::current_device(); return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int d) { if (d < 0 || d >= ::cusim::device_count()) return 101; ::cusim::current_device() = d; return cudaSuccess; }
static inline cudaError_t cudaGetDeviceCount(int* n) { *n = ::cusim::device_count(); return cudaSuccess; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
template <class T> static inline cudaError_t cudaMalloc(T** p, size_t n) { *p = (T*)malloc(n ? n : 1); if (*p) memset((void*)*p, 0xCD, n); return *p ? 0 : 2; }
static inline cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
template <class T> static inline cudaError_t cudaHostAlloc(T** p, size_t n, unsigned) { *p = (T*)malloc(n ? n : 1); return *p ? 0 : 2; }
static inline cudaError_t cudaFreeHost(void* p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { memcpy(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { memcpy(d, s, n); return cudaSuccess; }
template <class S> static inline cudaError_t cudaMemcpyToSymbol(S& sym, const void* s, size_t n) { memcpy((void*)&sym, s, n); return cudaSuccess; }
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = (void*)1; return cudaSuccess; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = (void*)1; return cudaSuccess; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t) { return cudaSuccess; }
enum { cudaEventDisableTiming = 2 };
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { *e = (void*)1; return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned = 0) { return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = nullptr) { return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) { *ms = 0; return cudaSuccess; }
template <class K> static inline cudaError_t cudaFuncSetAttribute(K, int, int) { return cudaSuccess; }
enum { cudaDevAttrMultiProcessorCount = 16 };
// an H100 SXM's 132 multiprocessors; PBC_SIM_SMS=N reports N, so that a small batch spans several
// batch-inversion chains per thread (T = multiprocessors * 128 or 256 chains, engine.cu inv_threads)
static inline cudaError_t cudaDeviceGetAttribute(int* v, int, int) {
  const char* e = getenv("PBC_SIM_SMS");
  *v = e && atoi(e) > 0 ? atoi(e) : 132;
  return cudaSuccess;
}
