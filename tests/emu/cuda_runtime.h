// TEST INFRASTRUCTURE ONLY — a tiny stand-in for the CUDA runtime and device language so that the
// queue / count protocols of taudem_b200/csrc/sweep_warp.cu can be executed on a CPU (tests/test_emu.py).
//
// Execution model: the blocks of a launch run one after the other; the threads of a block are fibers
// (ucontext) that a scheduler switches between at every "interesting" point — atomics, acquire loads,
// fences, warp collectives, __syncthreads — picking the next runnable fiber at random (seeded), so that
// different interleavings of the warps of a block are explored.  Memory is sequentially consistent: this
// checks protocol logic and arithmetic (bit-exact: plain IEEE float/double, no contraction), not the
// PTX memory model.  `__shared__` variables are function-local statics (one block at a time).
#pragma once
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <ucontext.h>

#include <algorithm>
#include <deque>
#include <functional>
#include <vector>

#define TD_EMU 1
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __launch_bounds__(...)
#define __shared__ static
#define __align__(n) __attribute__((aligned(n)))

struct dim3 { unsigned x = 1, y = 1, z = 1; dim3() {} dim3(unsigned a, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {} };
struct uint4 { unsigned x, y, z, w; };
struct uint2 { unsigned x, y; };
inline uint2 make_uint2(unsigned a, unsigned b) { return {a, b}; }
struct ushort4 { unsigned short x, y, z, w; };
struct uchar4 { unsigned char x, y, z, w; };
struct float4 { float x, y, z, w; };
struct short4 { short x, y, z, w; };
inline uint4 make_uint4(unsigned a, unsigned b, unsigned c, unsigned d) { return {a, b, c, d}; }
inline ushort4 make_ushort4(unsigned short a, unsigned short b, unsigned short c, unsigned short d) { return {a, b, c, d}; }
inline uchar4 make_uchar4(unsigned char a, unsigned char b, unsigned char c, unsigned char d) { return {a, b, c, d}; }
inline float4 make_float4(float a, float b, float c, float d) { return {a, b, c, d}; }
struct alignas(16) double2 { double x, y; };
inline double2 make_double2(double a, double b) { return {a, b}; }
inline short4 make_short4(short a, short b, short c, short d) { return {a, b, c, d}; }

// ---- host runtime
typedef int cudaError_t;
typedef void* cudaStream_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorMemoryAllocation = 2 };
enum cudaMemcpyKind { cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice };
enum { cudaDevAttrMultiProcessorCount = 16 };
inline cudaError_t cudaMalloc(void** p, size_t n) { *p = calloc(1, n ? n : 1); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
template <typename T> inline cudaError_t cudaMalloc(T** p, size_t n) { return cudaMalloc((void**)p, n); }
inline cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
inline cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t) { memset(p, v, n); return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t) { memmove(d, s, n); return cudaSuccess; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
inline cudaError_t cudaDeviceGetAttribute(int* v, int, int) { *v = 3; return cudaSuccess; }   // "3 SMs"
template <typename F> inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int* n, F, int, size_t) { *n = 2; return cudaSuccess; }
inline cudaError_t cudaMemset(void* p, int v, size_t n) { memset(p, v, n); return cudaSuccess; }
inline const char* cudaGetErrorString(cudaError_t) { return "emulated"; }
enum { cudaFuncAttributeMaxDynamicSharedMemorySize = 8, cudaIpcMemLazyEnablePeerAccess = 1 };
template <typename F> inline cudaError_t cudaFuncSetAttribute(F, int, int) { return cudaSuccess; }
struct cudaIpcMemHandle_t { char reserved[64]; };
inline cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t*, void*) { return 1; }       // no peers on the emulation
inline cudaError_t cudaIpcOpenMemHandle(void**, cudaIpcMemHandle_t, unsigned) { return 1; }
inline cudaError_t cudaIpcCloseMemHandle(void*) { return cudaSuccess; }

// ---- fibers
namespace emu {
// context of a fiber: on x86-64 just the saved stack pointer (callee-saved registers live on the fiber's stack; no signal
// mask system calls like swapcontext makes), elsewhere a ucontext
#if defined(__x86_64__)
struct Context { void* sp = nullptr; };
#else
struct Context { ucontext_t uc; };
#endif
struct Fiber {
  Context ctx;
  bool done = false;
  dim3 tid;
};
struct Block {
  std::vector<Fiber> f;
  Context sched;
  int cur = -1;
  int alive = 0;
  // warp collectives: one slot per participant mask (a *_sync with a partial mask involves only those lanes);
  // the lanes of a generation deposit their values, the last arrival publishes res[] / ballot[] of that parity
  struct Slot { unsigned mask = 0; unsigned long long val[32]; int arrived = 0; unsigned gen = 0; unsigned long long res[2][32]; unsigned ballot[2]; };
  struct Warp { std::deque<Slot> slots; unsigned alive = 0xffffffffu; };
  std::vector<Warp> warps;
  int bar_arrived = 0; unsigned bar_gen = 0;
};
extern thread_local Block* g_blk;      // one emulated device per host thread (the multi-strip tests run one thread per strip)
extern thread_local unsigned long long g_rng;
extern thread_local std::function<void()> g_body;
inline unsigned rnd() { g_rng = g_rng * 6364136223846793005ull + 1442695040888963407ull; return (unsigned)(g_rng >> 33); }
void yield();                       // back to the scheduler (random next fiber)
void run_block(dim3 grid, dim3 block, dim3 bid, const std::function<void()>& body);
}  // namespace emu

extern thread_local dim3 threadIdx, blockIdx, blockDim, gridDim;

template <typename F> inline void emu_launch(dim3 grid, dim3 block, F body) {
  for (unsigned by = 0; by < grid.y; ++by)
    for (unsigned bx = 0; bx < grid.x; ++bx) emu::run_block(grid, block, dim3(bx, by, 0), body);
}

// ---- device language
inline void __threadfence() { emu::yield(); }
inline void __threadfence_block() {}
inline void __threadfence_system() { emu::yield(); }
inline void __nanosleep(unsigned) { emu::yield(); }
template <typename T> inline T __ldcg(const T* p) { emu::yield(); return *p; }
template <typename T> inline T __ldg(const T* p) { return *p; }
inline int __popc(unsigned v) { return __builtin_popcount(v); }
inline int __ffs(unsigned v) { return __builtin_ffs((int)v); }
inline long long clock64() { return 0; }
inline long long __double_as_longlong(double d) { long long v; memcpy(&v, &d, 8); return v; }
inline double __longlong_as_double(long long v) { double d; memcpy(&d, &v, 8); return d; }
inline int __clz(int v) { return v ? __builtin_clz((unsigned)v) : 32; }
inline unsigned __byte_perm(unsigned x, unsigned y, unsigned sel) {     // PRMT, default mode: selector nibbles 0-3 = bytes of x, 4-7 = bytes of y
  const unsigned long long v = ((unsigned long long)y << 32) | x;
  unsigned r = 0;
  for (int i = 0; i < 4; ++i) r |= (unsigned)((v >> (8 * ((sel >> (4 * i)) & 7u))) & 0xffull) << (8 * i);
  return r;
}
inline unsigned __funnelshift_l(unsigned lo, unsigned hi, unsigned sh) { return (unsigned)((((unsigned long long)hi << 32) | lo) << (sh & 31) >> 32); }
inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned sh) { return (unsigned)((((unsigned long long)hi << 32) | lo) >> (sh & 31)); }
using std::max;
using std::min;
inline int min(int a, unsigned b) { return a < (int)b ? a : (int)b; }

#define EMU_ATOMIC(T)                                                                       \
  inline T atomicAdd(T* p, T v) { emu::yield(); T o = *p; *p = (T)(o + v); return o; }       \
  inline T atomicSub(T* p, T v) { emu::yield(); T o = *p; *p = (T)(o - v); return o; }       \
  inline T atomicOr(T* p, T v) { emu::yield(); T o = *p; *p = (T)(o | v); return o; }         \
  inline T atomicExch(T* p, T v) { emu::yield(); T o = *p; *p = v; return o; }               \
  inline T atomicCAS(T* p, T c, T v) { emu::yield(); T o = *p; if (o == c) *p = v; return o; }
EMU_ATOMIC(int)
EMU_ATOMIC(unsigned)
EMU_ATOMIC(unsigned long long)
#define atomicAdd_system atomicAdd
#define atomicCAS_system atomicCAS
#define atomicExch_system atomicExch

unsigned __activemask();
void __syncthreads();
int __syncthreads_or(int pred);
void __syncwarp(unsigned mask = 0xffffffffu);
unsigned __ballot_sync(unsigned mask, int pred);
unsigned long long emu_shfl(unsigned mask, unsigned long long v, int src_lane_or_delta, int mode);   // mode 0 = idx, 1 = up, 2 = xor
template <typename T> inline T __shfl_sync(unsigned mask, T v, int lane) {
  unsigned long long x = 0; memcpy(&x, &v, sizeof(T)); x = emu_shfl(mask, x, lane, 0); T r; memcpy(&r, &x, sizeof(T)); return r;
}
template <typename T> inline T __shfl_xor_sync(unsigned mask, T v, int lanemask) {
  unsigned long long x = 0; memcpy(&x, &v, sizeof(T)); x = emu_shfl(mask, x, lanemask, 2); T r; memcpy(&r, &x, sizeof(T)); return r;
}
template <typename T> inline T __shfl_up_sync(unsigned mask, T v, int delta) {
  unsigned long long x = 0; memcpy(&x, &v, sizeof(T)); x = emu_shfl(mask, x, delta, 1); T r; memcpy(&r, &x, sizeof(T)); return r;
}
