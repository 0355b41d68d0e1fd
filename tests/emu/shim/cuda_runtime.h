// tests/emu/shim/cuda_runtime.h -- TEST INFRASTRUCTURE, never part of the product.
//
// A host-side SIMT emulator: the product's CUDA sources (smplsim_b200/csrc/*.cuh, smplsim_capi.cu) are compiled UNCHANGED
// with g++ against this header (it shadows <cuda_runtime.h> through the include path), so the `-m "not gpu"` tests can run
// the very kernel source against the oracle on a machine without a GPU.  Every CUDA thread of a CTA is a ucontext
// coroutine; warp collectives (__shfl_sync, __ballot_sync, __syncwarp, ...) and __syncthreads are rendezvous points of the
// cooperative scheduler, so mis-synchronised code deadlocks here (reported) instead of silently racing.  Shared memory is
// one heap block per CTA.
// Nothing under smplsim_b200/ includes or links this.
#pragma once
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <ucontext.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <string>
#include <vector>

#define SMPLSIM_EMU 1
#define __device__
#define __host__
#define __global__
#define __forceinline__ inline __attribute__((always_inline))
#define __noinline__ __attribute__((noinline))
#define __launch_bounds__(...)
#define __shared__ static
#define __constant__ static
#ifndef __restrict__
#define __restrict__
#endif

struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct float4 { float x, y, z, w; };
struct float2 { float x, y; };
struct uint4 { unsigned x, y, z, w; };
struct int4 { int x, y, z, w; };
struct int2 { int x, y; };
static inline float4 make_float4(float x, float y, float z, float w) { float4 r = {x, y, z, w}; return r; }

typedef int cudaError_t;
typedef void* cudaStream_t;
#define cudaSuccess 0
enum { cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaDevAttrMaxSharedMemoryPerBlockOptin = 97, cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
static inline const char* cudaGetErrorString(cudaError_t) { return "emu"; }
static inline cudaError_t cudaSetDevice(int) { return 0; }
static inline cudaError_t cudaGetDevice(int* d) { *d = 0; return 0; }
static inline cudaError_t cudaGetLastError() { return 0; }
static inline cudaError_t cudaDeviceSynchronize() { return 0; }
static inline cudaError_t cudaMalloc(void* p, size_t n) { *(void**)p = calloc(1, n ? n : 1); return 0; }
static inline cudaError_t cudaFree(void* p) { free(p); return 0; }
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, int) { memcpy(d, s, n); return 0; }
static inline cudaError_t cudaMemset(void* d, int v, size_t n) { memset(d, v, n); return 0; }
static inline cudaError_t cudaDeviceGetAttribute(int* v, int, int) { *v = 232448; return 0; }
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, int, int) { return 0; }

namespace emu {
struct Thread {
  ucontext_t ctx;
  char* stack;
  int tid;
  bool done;
  int wait_kind;   // 0 runnable, 1 waiting at a warp rendezvous, 2 waiting at the CTA barrier
  unsigned gen;
  unsigned orcalls;
};
struct Warp {
  unsigned slot[32];
  int arrived;
  unsigned gen;
  int alive;
};
struct Cta {
  std::vector<Thread> th;
  std::vector<Warp> warp;
  int nthreads, cta_arrived, cta_alive;
  unsigned cta_gen;
  int or_acc[2];
  dim3 bidx, bdim, gdim;
  char* smem;
  std::function<void()> body;
  ucontext_t sched;
  int cur;
};
extern Cta* g_cta;
extern unsigned long long g_events;
inline Thread& cur() { return g_cta->th[g_cta->cur]; }
inline void yield() { Thread& t = cur(); swapcontext(&t.ctx, &g_cta->sched); }

// rendezvous of the calling thread's warp: deposit v, wait for all alive lanes, then `read` may look at every slot;
// a second rendezvous keeps the slots stable until every lane has read them
inline void warp_arrive() {
  Cta& c = *g_cta;
  Thread& t = cur();
  Warp& w = c.warp[t.tid >> 5];
  unsigned gen = w.gen;
  g_events++;
  if (++w.arrived >= w.alive) { w.arrived = 0; w.gen++; }
  else { t.wait_kind = 1; while (w.gen == gen) yield(); t.wait_kind = 0; }
}
template <class R> inline unsigned warp_collect(unsigned v, R read) {
  Cta& c = *g_cta;
  Thread& t = cur();
  Warp& w = c.warp[t.tid >> 5];
  w.slot[t.tid & 31] = v;
  warp_arrive();
  unsigned r = read(w);
  warp_arrive();
  return r;
}
inline void cta_barrier() {
  Cta& c = *g_cta;
  Thread& t = cur();
  unsigned gen = c.cta_gen;
  g_events++;
  if (++c.cta_arrived >= c.cta_alive) { c.cta_arrived = 0; c.cta_gen++; }
  else { t.wait_kind = 2; while (c.cta_gen == gen) yield(); t.wait_kind = 0; }
}
void launch(dim3 grid, dim3 block, size_t smem, const std::function<void()>& body);
}  // namespace emu

struct EmuIdx { unsigned x, y, z; };
static inline EmuIdx emu_tidx() { EmuIdx r = {(unsigned)emu::cur().tid, 0, 0}; return r; }
#define threadIdx (emu_tidx())
#define blockIdx (emu::g_cta->bidx)
#define blockDim (emu::g_cta->bdim)
#define gridDim (emu::g_cta->gdim)

#define EMU_FULL 0xffffffffu
static inline void emu_check_mask(unsigned m) {
  if (m != EMU_FULL) { fprintf(stderr, "emu: warp collective with a partial mask 0x%x (unsupported)\n", m); abort(); }
}
static inline void __syncwarp(unsigned m = EMU_FULL) { emu_check_mask(m); emu::warp_arrive(); }
static inline void __syncthreads() { emu::cta_barrier(); }
static inline int __syncthreads_or(int p) {
  emu::Cta& c = *emu::g_cta;
  int k = (int)(emu::cur().orcalls++ & 1u);
  c.or_acc[k] |= (p != 0);
  emu::cta_barrier();
  int r = c.or_acc[k];
  c.or_acc[k ^ 1] = 0;
  emu::cta_barrier();
  return r;
}
static inline unsigned emu_bits(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
static inline float emu_float(unsigned u) { float f; memcpy(&f, &u, 4); return f; }
static inline unsigned emu_shfl(unsigned m, unsigned v, int src) {
  emu_check_mask(m);
  return emu::warp_collect(v, [&](emu::Warp& w) { return w.slot[src & 31]; });
}
static inline float __shfl_sync(unsigned m, float v, int src) { return emu_float(emu_shfl(m, emu_bits(v), src)); }
static inline int __shfl_sync(unsigned m, int v, int src) { return (int)emu_shfl(m, (unsigned)v, src); }
static inline unsigned __shfl_sync(unsigned m, unsigned v, int src) { return emu_shfl(m, v, src); }
static inline float __shfl_xor_sync(unsigned m, float v, int x) { return __shfl_sync(m, v, (emu::cur().tid & 31) ^ x); }
static inline int __shfl_xor_sync(unsigned m, int v, int x) { return __shfl_sync(m, v, (emu::cur().tid & 31) ^ x); }
static inline unsigned __shfl_xor_sync(unsigned m, unsigned v, int x) { return __shfl_sync(m, v, (emu::cur().tid & 31) ^ x); }
static inline int __shfl_up_sync(unsigned m, int v, int d) { int l = emu::cur().tid & 31; int s = l - d; return __shfl_sync(m, v, s < 0 ? l : s); }
static inline float __shfl_up_sync(unsigned m, float v, int d) { int l = emu::cur().tid & 31; int s = l - d; return __shfl_sync(m, v, s < 0 ? l : s); }
static inline unsigned __ballot_sync(unsigned m, bool p) {
  emu_check_mask(m);
  int mytid = emu::cur().tid;
  (void)mytid;
  return emu::warp_collect(p ? 1u : 0u, [&](emu::Warp& w) {
    unsigned r = 0;
    int base = (emu::cur().tid >> 5) << 5;
    for (int i = 0; i < 32; i++) if (base + i < emu::g_cta->nthreads && !emu::g_cta->th[base + i].done && w.slot[i]) r |= 1u << i;
    return r;
  });
}
static inline bool __any_sync(unsigned m, bool p) { return __ballot_sync(m, p) != 0u; }
static inline bool __all_sync(unsigned m, bool p) { return __ballot_sync(m, !p) == 0u; }
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline int __popcll(unsigned long long v) { return __builtin_popcountll(v); }
static inline int __ffs(int v) { return __builtin_ffs(v); }
static inline int __clz(int v) { return v ? __builtin_clz((unsigned)v) : 32; }
static inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((unsigned long long)a * b) >> 32); }
#define __powf(a, b) powf(a, b)
static inline float __fdividef(float a, float b) { return a / b; }
static inline float __frcp_rn(float a) { return 1.0f / a; }
static inline float rsqrtf(float a) { return 1.0f / sqrtf(a); }
static inline int atomicAdd(int* p, int v) { int o = *p; *p = o + v; return o; }
static inline unsigned atomicOr(unsigned* p, unsigned v) { unsigned o = *p; *p = o | v; return o; }
template <class T> static inline T __ldg(const T* p) { return *p; }
static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }

// dynamic shared memory of the running CTA
#define EMU_SMEM_BASE ((float*)emu::g_cta->smem)
