// Contributing-area evaluation sweep: tile dataflow with one WARP per tile visit (D8 and D-infinity).
//
// reference: aread8 main loop src/aread8.cpp:216-304, area() main loop src/areadinf.cpp:173-265 — a queue of cells
// whose dependency count is zero; evaluate (k-ordered float32 gather over the neighbours that drain into the cell),
// decrement the receivers, push those that reach zero.  The value of a cell does not depend on the schedule
// (SURVEY.md A.6), so the schedule here is the GPU's:
//
//  * the strip is cut into 32 x 32 tiles; tile ids wait in a device-side multi-producer / multi-consumer ticket queue;
//  * every warp of a grid of persistent CTAs is an independent worker: it pops a tile, stages the tile's dependency
//    counts, node words, areas (and angles) with a one-cell ring in its own slice of shared memory (cp.async, one round trip) and runs the wavefront
//    there — each lane follows one chain (evaluate, shared-memory atomic decrement of the receiver(s), go on when it
//    was the last arrival), second receivers of D-infinity cells go to a warp-local queue that idle lanes drain;
//    no CTA-wide barrier exists anywhere, a warp that holds a long chain delays nobody;
//  * what a visit costs is proportional to what it evaluates: only evaluated areas and changed count words are
//    written back (one fence), flow that leaves the tile is one global atomic per crossing, and the arrival that
//    zeroes a count activates the owning tile (per-tile state idle / queued / running / running + dirty, so that a
//    tile is never processed by two warps at once);
//  * the carry: of the tiles a visit made ready, the one its last crossing reached (a river leaving the tile) is claimed
//    by the same warp and visited next, without a trip through the ticket queue;
//  * the kernel ends when no tile is queued or running.
// Flow that crosses the strip boundary (one strip per GPU) is recorded in `halo` for the exchange rounds of the
// row-strip driver (src/aread8.cpp:282-297, linearpart::addBorders).  Every algebra crosses it: what a cell reads at a
// contributor in a halo row is the travelling value (exchanged or delivered like the area), an input grid's halo row (the
// caller loads it: decay multiplier, discharge, gridnet's mask and the D8 codes of that row) or, for ALG 9, the
// concentration (exchanged with the value rows, or delivered into the second half of the peer halo buffer).
#include <stddef.h>
#include <string.h>

#include <algorithm>

#include "ctx.h"
#include "dinf_common.cuh"
#include "kernels.h"
#include "rowfact.cuh"

namespace td {
namespace {

constexpr int TS = 32;                                // tile width (cells) = lanes of a warp
constexpr int TH = 32;                                // tile height: one row per lane (64-row D8 tiles were slower: 330 instead of 288 ms at 65536^2)
constexpr int RS = TS + 4;                            // ring row stride: cell lx of a tile row at lx + 4, its west neighbour at 3, its east neighbour at
                                                      // 36 = slot 0 of the next row (slots 0..2 of a row are otherwise unused): rows stay 16-byte aligned
constexpr int RH = TH + 2;                            // ring rows
constexpr int RN = RH * RS + 4;                       // ring array length (the east neighbour of the last ring row lives at RH * RS)
#ifndef TD_WSTK
#define TD_WSTK 128
#endif
constexpr int STKCAP = TD_WSTK;                       // fork stack entries per worker (D-infinity)
constexpr unsigned NODE_VALID = 0x8000u, NODE_CON = 0x1000u;
constexpr unsigned FULL = 0xffffffffu;
constexpr int EXP_NO_CARRY = 16;                      // TAUDEM_B200_EXP bit: every activation goes through the ticket queue (no carried tiles)
// The scheduler's words (WArgs::ctr, 8-byte words, one 128-byte line each).  The ticket queue is cut into up to MAXSH
// independent shards (tile t belongs to shard t & (nsh - 1), worker w pops from shard w & (nsh - 1)): one queue's head /
// tail / finished counters were the throughput limit of the whole sweep (three hot addresses, ~7 ns per atomic each).
#ifdef TD_EMU
constexpr int MAXSH = 8;     // the CPU emulation runs the CTAs one after the other: the first one alone must serve every shard
#else
constexpr int MAXSH = 64;
#endif
constexpr int C_TERM = 3 * MAXSH * 16, C_ACTIVE = (3 * MAXSH + 1) * 16, C_WORDS = (3 * MAXSH + 2) * 16;

// neighbour offsets as 2-bit fields (value + 1) indexed by the direction k = 1..8
constexpr unsigned pack_dir(bool row) {
  unsigned v = 0;
  for (int k = 1; k <= 8; ++k) v |= (unsigned)((row ? drow(k) : dcol(k)) + 1) << (2 * k);
  return v;
}
constexpr unsigned DROW_LUT = pack_dir(true), DCOL_LUT = pack_dir(false);
__device__ __forceinline__ int lut_drow(int k) { return (int)((DROW_LUT >> (2 * k)) & 3u) - 1; }
__device__ __forceinline__ int lut_dcol(int k) { return (int)((DCOL_LUT >> (2 * k)) & 3u) - 1; }

// one worker's shared memory: everything a visit touches while it runs the wavefront
template <bool DINF>
struct __align__(16) WarpMem {
  float area[RN];                         // areas of the tile and its ring (-1 = nodata / not final)
  float ang[DINF ? RN : 4];               // D-infinity: angles of the same cells
  unsigned short node[RN];                // node words of the same cells
  alignas(16) unsigned cnt[TS * TH / 4];  // dependency counts, four cells per word: 0..8 (0 = ready or evaluated by this visit), 0xFE = evaluated
                                          // by an earlier visit, 0xFF = not a node
  unsigned short stk[DINF ? STKCAP : 2];  // D-infinity: second receivers that became ready (what does not fit is found again by a rescan of the counts)
  unsigned short ext[DINF ? 256 : 128];   // flow that leaves the tile: source cell | (direction - 1) << 11  (<= 124 perimeter cells x receivers)
  unsigned evmask[TH];                    // per tile row: cells evaluated by this visit
  int sp, next, ovf, pad;                 // ovf (statistics only): a second receiver did not fit the fork stack in this visit
};
template <bool DINF> constexpr int workers_per_cta() { return DINF ? 16 : 26; }
static_assert(sizeof(WarpMem<false>) * workers_per_cta<false>() <= 227 * 1024 && sizeof(WarpMem<true>) * workers_per_cta<true>() + 1024 <= 227 * 1024,
              "the workers of a CTA must fit the shared memory of an SM");
static_assert(offsetof(WarpMem<true>, ang) % 16 == 0 && offsetof(WarpMem<true>, node) % 8 == 0 && offsetof(WarpMem<false>, node) % 8 == 0, "cp.async alignment");

// what a neighbouring strip exposes to this GPU (device pointers into the peer's memory)
struct PeerStrip {
  unsigned* cntw = nullptr; int* state = nullptr; int* tq = nullptr; unsigned long long* ctr = nullptr; float* halo_in = nullptr;
  unsigned qmask = 0; int ntx = 0, ny = 0, valid = 0, nsh = 1, qshift = 0;
};

struct WArgs {
  const unsigned short* node;
  unsigned* cntw;
  float* area;
  const float* w;
  const float* ang;
  Strip s;
  int usew, contcheck;
  float w_nodata;
  const double* theta;
  const double* dxc;
  int* halo;
  int ntx, nty, th;        // tiles of the strip, tile height
  const float* dm; float dm_nodata;   // ALG 3: the decay multiplier grid (strip layout) and its nodata; ALG 4-6: the mask grid (0 = outside) or NULL
  const float* dist;                  // ALG 4-6: cell-to-cell distances, [row][direction - 1] (float, like src/gridnet.cpp:190-200)
  SweepExtra x;                       // ALG 7-9: indicator grid / solubility, supply concentration, deposition and concentration outputs
  int* state;              // per tile: 0 idle, 1 queued, 2 running, 3 running + re-activated
  int* tq;                 // ring of tile ids + 1
  unsigned qmask;          // slots of one shard's ring - 1
  int nsh, qshift;         // queue shards (a power of two), log2 of a shard's ring size
  PropRow prop;            // D-infinity: the strip's prop() table (prop.uniform: every row has the same cell size dx0) — else per-row angles from `theta`
  double dx0;              // the cell size a cell's own area adds (src/areadinf.cpp:216)
  unsigned long long* ctr; // scheduler words (see MAXSH)
  unsigned long long* stat;// [0] carried visits, [1] cells, [2] wavefront iterations, [3] visits, [4..7] cycle statistics, [8] visits whose
                           // fork stack overflowed (more than STKCAP second receivers pending: the rescan of the counts finds the rest) (TAUDEM_B200_TIMING)
  int stats, exp;          // exp: TAUDEM_B200_EXP (EXP_NO_CARRY)
  // peer mode (one strip per GPU, the neighbours' buffers mapped over NVLink with CUDA IPC): no exchange rounds — a tile
  // delivers into the neighbour GPU exactly as it delivers into a neighbour tile.  Every GPU only WRITES remote memory
  // (the neighbour's halo-area buffer, counts, tile states, queue); everything it reads is its own.
  int peer;
  PeerStrip up, down;      // the strip above (rank - 1) / below (rank + 1)
  unsigned long long* G;   // strips that still have queued / running tiles + activations in flight between strips (lives on rank 0)
  const float* halo_in;    // areas of the neighbours' edge cells: [0, pitch) row above, [pitch, 2 pitch) row below; ALG 9: their
                           // concentrations in [2 pitch, 4 pitch) the same way
};

#ifdef TD_EMU
template <typename T> __device__ __forceinline__ T ldv(const T* p) { emu::yield(); return *((const volatile T*)p); }
#else
template <typename T> __device__ __forceinline__ T ldv(const T* p) { return *((const volatile T*)p); }
#endif
template <typename T> __device__ __forceinline__ void stv(T* p, T v) { *((volatile T*)p) = v; }

#ifndef TD_EMU
__device__ __forceinline__ void cp16(void* smem, const void* g) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem)), "l"(g) : "memory"); }
__device__ __forceinline__ void cp8(void* smem, const void* g) { asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(smem)), "l"(g) : "memory"); }
__device__ __forceinline__ void cp4(void* smem, const void* g) { asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem)), "l"(g) : "memory"); }
__device__ __forceinline__ void cp_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
#else
__device__ __forceinline__ void cp_check(const void* smem, const void* g, size_t n) { if ((size_t)smem % n || (size_t)g % n) { fprintf(stderr, "emu: misaligned %zu-byte cp.async\n", n); abort(); } }
__device__ __forceinline__ void cp16(void* smem, const void* g) { emu::yield(); cp_check(smem, g, 16); memcpy(smem, g, 16); }
__device__ __forceinline__ void cp8(void* smem, const void* g) { cp_check(smem, g, 8); memcpy(smem, g, 8); }
__device__ __forceinline__ void cp4(void* smem, const void* g) { cp_check(smem, g, 4); memcpy(smem, g, 4); }
__device__ __forceinline__ void cp_wait_all() {}
#endif

// ---- scheduler (one lane per worker)
// In peer mode a neighbour GPU operates on this strip's scheduler words and on the counts of its edge rows with
// system-scope atomics over NVLink; the owner then uses system scope on the same words (atomics of different scopes on one
// address are not guaranteed to be atomic with respect to each other).
#define W_ADD(ptr, v) (a.peer ? atomicAdd_system((ptr), (v)) : atomicAdd((ptr), (v)))
#define W_CAS(ptr, c, v) (a.peer ? atomicCAS_system((ptr), (c), (v)) : atomicCAS((ptr), (c), (v)))
#define W_EXCH(ptr, v) (a.peer ? atomicExch_system((ptr), (v)) : atomicExch((ptr), (v)))
// the words a neighbour GPU can touch: counts of the strip's first / last row, states of the tiles that hold them
#define W_ADD_IF(sys, ptr, v) ((sys) ? atomicAdd_system((ptr), (v)) : atomicAdd((ptr), (v)))
#define W_CAS_IF(sys, ptr, c, v) ((sys) ? atomicCAS_system((ptr), (c), (v)) : atomicCAS((ptr), (c), (v)))
#define W_EXCH_IF(sys, ptr, v) ((sys) ? atomicExch_system((ptr), (v)) : atomicExch((ptr), (v)))

__device__ __forceinline__ unsigned long long* w_head(unsigned long long* ctr, int q) { return ctr + (3 * q) * 16; }
__device__ __forceinline__ unsigned long long* w_tail(unsigned long long* ctr, int q) { return ctr + (3 * q + 1) * 16; }
__device__ __forceinline__ unsigned long long* w_done(unsigned long long* ctr, int q) { return ctr + (3 * q + 2) * 16; }

// A tile is pushed at most once between two visits (its state word says so), so a shard's ring never holds more entries
// than the shard has tiles; tickets beyond the tail belong to waiting workers.
__device__ void sched_push(const WArgs& a, int t) {
  const int q = t & (a.nsh - 1);
  const unsigned long long slot = W_ADD(w_tail(a.ctr, q), 1ull);
  int* ring = a.tq + ((size_t)q << a.qshift) + (slot & a.qmask);
  while (W_CAS(ring, 0, t + 1) != 0) {}
}
__device__ __forceinline__ bool edge_tile(const WArgs& a, int t) { return a.peer && (t < a.ntx || t >= (a.nty - 1) * a.ntx); }
__device__ void sched_activate(const WArgs& a, int t) {
  const bool sys = edge_tile(a, t);
  for (;;) {
    const int st = W_CAS_IF(sys, a.state + t, 0, 1);        // idle -> queued (the common case: one round trip)
    if (st == 0) { sched_push(a, t); return; }
    if (st == 1 || st == 3) return;
    if (W_CAS_IF(sys, a.state + t, 2, 3) == 2) return;     // running -> running + re-activated
  }
}
// The same protocol on a neighbour GPU's scheduler (system-scope atomics over NVLink).  Termination across GPUs: G counts
// the strips that are ACTIVE (some tile queued or running) plus the activations in flight between strips.  Whoever
// activates a tile of another strip first takes a token (G += 1), pushes, fences, and then marks the strip active: if it
// was active already the token is returned, otherwise the token becomes that strip's own count.
__device__ void sched_activate_peer(const WArgs& a, const PeerStrip& P, int t) {
  for (;;) {
    const int st = atomicCAS_system(P.state + t, 0, 1);
    if (st == 0) {
      atomicAdd_system(a.G, 1ull);
      const int q = t & (P.nsh - 1);
      const unsigned long long slot = atomicAdd_system(w_tail(P.ctr, q), 1ull);
      int* ring = P.tq + ((size_t)q << P.qshift) + (slot & P.qmask);
      while (atomicCAS_system(ring, 0, t + 1) != 0) {}
      __threadfence_system();                                // the push is visible before the strip is (re)marked active
      if (atomicExch_system(P.ctr + C_ACTIVE, 1ull) == 1ull) atomicAdd_system(a.G, ~0ull);
      return;
    }
    if (st == 1 || st == 3) return;
    if (atomicCAS_system(P.state + t, 2, 3) == 2) return;
  }
}
// Flow into the strip above (up) / below: the source cell's area goes into the neighbour's halo buffer, is fenced
// system-wide, then the neighbour's count is decremented; zero -> queue its tile (src/aread8.cpp:282-297 without rounds).
// ALG 9: the source's concentration (the second value that travels) goes into the second half of that buffer, before the
// same fence.
template <int ALG>
__device__ void deliver_peer(const WArgs& a, bool up, int c_src, float val, int c_dst) {
  const PeerStrip& P = up ? a.up : a.down;
  const int pitch = a.s.pitch;
  P.halo_in[(up ? pitch : 0) + c_src] = val;        // I am the row BELOW the strip above / the row ABOVE the strip below
  if (ALG == 9) P.halo_in[2 * pitch + (up ? pitch : 0) + c_src] = ldv(a.x.out3 + a.s.idx(up ? 1 : a.s.ny, c_src));
  __threadfence_system();
  const int r = up ? P.ny : 1;
  const long long ci = (long long)r * pitch + c_dst;
  const unsigned sh = (unsigned)(ci & 3) * 8u;
  const unsigned old = atomicAdd_system(P.cntw + (ci >> 2), 0u - (1u << sh));
  if (((old >> sh) & 0xffu) == 1u) sched_activate_peer(a, P, ((r - 1) / a.th) * P.ntx + c_dst / TS);
}
// relaxed gpu-scope load of a scheduler word (a volatile load is a system-scope load: far more expensive to poll with)
__device__ __forceinline__ int ld_relaxed(const int* p) {
#ifdef TD_EMU
  emu::yield(); return *((const volatile int*)p);
#else
  int v; asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
#endif
}
__device__ __forceinline__ long long ld_relaxed(const unsigned long long* p) {
#ifdef TD_EMU
  emu::yield(); return (long long)*((const volatile unsigned long long*)p);
#else
  long long v; asm volatile("ld.relaxed.gpu.global.s64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v;
#endif
}
// waits about `cycles` SM cycles without touching memory
__device__ __forceinline__ void idle_wait(unsigned cycles) {
#ifdef TD_EMU
  (void)cycles; emu::yield();
#else
  const long long t0 = clock64();
  do { __nanosleep(cycles >> 1); } while (clock64() - t0 < (long long)cycles);
#endif
}
// The visit's two one-sided fences (DESIGN.md §4.1 lists what each one orders).  System scope in peer mode, where a
// neighbour GPU publishes into this strip's counts with system-scope atomics.  fence.acquire compiles to an L1 invalidate
// behind the preceding loads, fence.release to a wait for the preceding stores (MEMBAR.ALL); neither is the SC fence of
// __threadfence().
__device__ __forceinline__ void fence_acquire(bool sys) {
#ifdef TD_EMU
  (void)sys; emu::yield();
#else
  if (sys) asm volatile("fence.acquire.sys;" ::: "memory");
  else asm volatile("fence.acquire.gpu;" ::: "memory");
#endif
}
__device__ __forceinline__ void fence_release(bool sys) {
#ifdef TD_EMU
  (void)sys; emu::yield();
#else
  if (sys) asm volatile("fence.release.sys;" ::: "memory");
  else asm volatile("fence.release.gpu;" ::: "memory");
#endif
}
// relaxed (strong, past the L1) load of four count words: with fence_acquire after it, an acquire of what they announce
__device__ __forceinline__ uint4 ld_cnt4(const uint4* p, bool sys) {
#ifdef TD_EMU
  (void)sys; return __ldcg(p);
#else
  uint4 v;
  if (sys) asm volatile("ld.relaxed.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  else asm volatile("ld.relaxed.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
#endif
}
// No tile of this strip is queued or running: every push (tail) has been matched by a finished visit (done).  The counters
// only grow, a tile's own pushes precede its done, and all done counters are read BEFORE all tails: if the sums are equal,
// they were equal at the moment the last done was read — nothing was running then, so nothing can be pushed any more
// (except, in peer mode, by a neighbour strip).  The done loads are relaxed and all in flight at once; the one acquire
// fence behind them keeps every tail load after every done load.
__device__ bool sched_balanced(const WArgs& a) {
  long long d = 0, t = 0;
#pragma unroll 16
  for (int q = 0; q < a.nsh; ++q) d += ld_relaxed(w_done(a.ctr, q));
  fence_acquire(false);
#pragma unroll 16
  for (int q = 0; q < a.nsh; ++q) t += ld_relaxed(w_tail(a.ctr, q));
  return d == t;
}
// Ticket h of a shard is served by the shard's h-th push.  A waiting worker polls its own slot (a word nobody else polls)
// with an exponential back-off of 0.25 .. 2 us and the strip's "terminated" word every 8th time; the first warp of every
// CTA also looks for termination itself (every 64th poll): all shards balanced — and in peer mode: this strip goes
// passive (returning its count to G unless a neighbour re-activated it meanwhile) and the sweep ends when G is zero.
__device__ int sched_pop(const WArgs& a, int q, bool scanner) {
  const unsigned long long h = atomicAdd(w_head(a.ctr, q), 1ull);
  int* slot = a.tq + ((size_t)q << a.qshift) + (h & a.qmask);
  unsigned wait = 512, n = 0;
  for (;;) {
    const int v = ld_relaxed(slot);
    if (v != 0) {
      W_EXCH(slot, 0);
      // the tile is marked running BEFORE its counts are read (whoever delivers into it after that re-activates it): the
      // exchange's result is consumed, so the count loads that follow cannot be issued before the exchange was performed
      const int prev = W_EXCH_IF(edge_tile(a, v - 1), a.state + (v - 1), 2);
      return prev == 0x7ffffff0 ? -1 : v - 1;
    }
    if ((++n & 7u) == 0u) {
      if (ld_relaxed(a.ctr + C_TERM) != 0) return -1;
      if (scanner && (n & 63u) == 0u && sched_balanced(a)) {
        bool over = true;
        if (a.peer) {
          if (atomicExch_system(a.ctr + C_ACTIVE, 0ull) == 1ull) {
            __threadfence_system();
            if (sched_balanced(a)) atomicAdd_system(a.G, ~0ull);                                   // passive: my count goes back
            else if (atomicExch_system(a.ctr + C_ACTIVE, 1ull) == 1ull) atomicAdd_system(a.G, ~0ull);   // work arrived; the pusher's token counts for me
          }
          over = ldv(a.G) == 0ull;
        }
        if (over) { atomicExch(a.ctr + C_TERM, 1ull); return -1; }
      }
    }
    idle_wait(wait);
    if (wait < 4096) wait <<= 1;
  }
}
// The end of a visit of tile t: release it (running -> idle), or queue it again if it was re-activated while it ran or is
// `dirty` (a rim count of the tile reached zero through arrivals from outside: it has a ready cell).  A dirty tile is still
// ours (running or running + re-activated: nobody else changes its state then), so it goes straight to queued.
// (the visit's count atomics — the rim's, the crossings' — have returned their results, consumed for `dirty` and the
//  activations, before the release is issued, and the plain stores were fenced before them: nothing of the visit that
//  touches this tile is still in flight when it is released; activations of other tiles may be)
__device__ __forceinline__ int sched_release(const WArgs& a, int t, bool dirty) {
  return dirty ? 3 : W_CAS_IF(edge_tile(a, t), a.state + t, 2, 0);
}
// A worker that popped a tile owes one `done` for that push.  A tile it carries (claimed at the end of a visit, never pushed)
// adds nothing to the tails, so a visit that hands over to a carried tile does not pay: the chain of carried visits pays once,
// when it ends.  Until then the shards stay unbalanced, so nobody can declare the end (nor, in peer mode, the strip passive).
// `rel` is what sched_release returned.
__device__ void sched_finish(const WArgs& a, int t, int rel, bool pay) {
  if (rel != 2) { W_EXCH_IF(edge_tile(a, t), a.state + t, 1); sched_push(a, t); }
  if (pay) atomicAdd(w_done(a.ctr, t & (a.nsh - 1)), 1ull);
}

// Zeroing by a kernel, not cudaMemsetAsync: memsets are executed by the copy engines, where they queue behind whatever
// host <-> device copy of another stream is in flight (a 17 GB raster: 0.3 s) and stall this stream's kernels with them.
__global__ void k_zero_words(unsigned* p, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = 0u;
}
__global__ void k_fill_floats(float* p, size_t n, float v) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = v;
}
// grid of the grid-stride fill kernels: one block per 256 elements, at most 16 per SM of the current device
unsigned fill_grid(size_t n) {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms < 1) sms = 1;
  return (unsigned)std::max<size_t>(1, std::min<size_t>((n + 255) / 256, (size_t)sms * 16));
}
}  // namespace
cudaError_t fill_floats(float* p, const Strip& s, float v, cudaStream_t st) {
  const size_t n = (size_t)s.cells();
  const unsigned grid = fill_grid(n);
  k_fill_floats<<<grid, 256, 0, st>>>(p, n, v);
  TD_LAUNCHED();
  return cudaGetLastError();
}
cudaError_t zero_words(void* p, size_t bytes, cudaStream_t st) {
  const size_t n = bytes / 4;
  const unsigned grid = fill_grid(n);
  k_zero_words<<<grid, 256, 0, st>>>((unsigned*)p, n);
  TD_LAUNCHED();
  return cudaGetLastError();
}
namespace {
// start of a sweep: every tile queued (the rings and the scheduler words were zeroed before)
__global__ void k_wsched_init(int* state, int* tq, int ntiles, unsigned long long* ctr, unsigned long long* stat, int nsh, int qshift, unsigned qmask) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if ((int)i < ntiles) {
    state[i] = 1;
    const int q = (int)i & (nsh - 1);
    const unsigned long long slot = atomicAdd(w_tail(ctr, q), 1ull);
    tq[((size_t)q << qshift) + (slot & qmask)] = (int)i + 1;
  }
  if (i == 0) {
    ctr[C_ACTIVE] = 1ull;
    for (int j = 0; j < 9; ++j) stat[j] = 0;
  }
}

// prop(angle, kk) through the full interval search (irregular cells, strips whose rows have different cell sizes)
__device__ __noinline__ double wshare_full(float ang, double t, int kk) {
  const Outflow o = dinf_outflow(ang, t);
  return o.k1 == kk ? o.p1 : o.p2;
}
// one sector of prop()'s table: its two directions' angles, its width and the width's reciprocal
struct __align__(16) Sector { double lo, hi, den, rden; };

// bit 7 of every byte of the result is set exactly where that byte of w is zero (no borrow between bytes)
__device__ __forceinline__ unsigned zero_bytes(unsigned w) { return ~(((w & 0x7f7f7f7fu) + 0x7f7f7f7fu) | w) & 0x80808080u; }
// bit i of the result: byte i of w is zero
__device__ __forceinline__ unsigned zero_nibble(unsigned w) {
  const unsigned z = zero_bytes(w);
  return ((z >> 7) & 1u) | ((z >> 14) & 2u) | ((z >> 21) & 4u) | ((z >> 28) & 8u);
}

// ALG: 0 = sum (aread8, src/aread8.cpp:228-257; areadinf, src/areadinf.cpp:187-218); D8 with a value grid in `w` only: 1 / 2 = the
// largest / smallest value of `w` on the flow paths above each cell (d8flowpathextremeup, src/D8flowpathextremeup.cpp:182-215);
// D-infinity only: 3 = decaying accumulation (dinfdecayaccum, src/dinfdecayaccum.cpp:205-235: the cell's own input first, then
// per contributor  + (float)(dm * area * p)  with the contributor's decay multiplier dm; a nodata multiplier contaminates).
// D8 only: 4 / 5 / 6 = gridnet's longest upstream path length, total upstream path length and Strahler order (src/gridnet.cpp:383-420;
// three sweeps, one value each; `dm` = mask grid: cells outside are not evaluated (they get w_nodata) and contribute nothing).
// D-infinity only, one chain per lane throughout (no warp-cooperative tail): 7 = concentration limited accumulation (DinfConcLimAccum,
// src/DinfConcLimAccum.cpp:235-272; `w` = the specific discharge q, `dm` = the decay multiplier, x.dg = the indicator grid);
// 8 / 9 = transport limited accumulation without / with a concentration (DinfTransLimAccum, src/DinfTransLimAccum.cpp:237-304;
// `w` = supply, `dm` = transport capacity, the value that travels is the transport out of the cell; deposition goes straight to
// x.out2; with a concentration (9) a second value travels: it lives in global memory (x.out3) — written before the receivers'
// counts are touched, read past the L1 — because a worker's shared memory holds one value per cell).
// Results of ALG 1-3 and 7-9 use MISSINGFLOAT as nodata, the others -1.
// gridnet's cell evaluation (src/gridnet.cpp:383-420): contributors = the neighbours that drain into the cell (mask bits) with a
// direction > 0 and inside the mask; all arithmetic in float like the reference's float dist table and float partitions.
template <int ALG, typename Mem>
__device__ __forceinline__ float gridnet_eval(const WArgs& a, const Mem& M, int ri, unsigned msk, int r, int c) {
  const Strip& s = a.s;
  if (a.dm && a.dm[s.idx(r, c)] == 0.f) return a.w_nodata;             // outside the mask: not evaluated
  const float* drowp = a.dist + (size_t)(min(r, s.ny) - 1) * 8;
  float val = 0.f, a1 = 0.f, a2 = 0.f;
#pragma unroll
  for (int k = 1; k <= 8; ++k) {
    if (!(msk & (1u << (k - 1)))) continue;
    const int ni = ri + drow(k) * RS + dcol(k);
    if ((((unsigned)M.node[ni] >> 8) & 0xfu) == 0u) continue;           // sdir > 0 (a direction code 0 counts as a dependency only)
    if (a.dm && a.dm[s.idx(r + drow(k), c + dcol(k))] == 0.f) continue;
    const float an = M.area[ni];
    const float d = drowp[k - 1];                                       // dist[j][sdir] = dist[j][k]: the same two cells
    if (ALG == 4) { const float ld = an + d; if (ld > val) val = ld; }
    else if (ALG == 5) val = val + (an + d);
    else { if (an >= a1) { a2 = a1; a1 = an; } else if (an > a2) a2 = an; }
  }
  if (ALG == 6) val = (a2 + 1.f > a1) ? a2 + 1.f : a1;
  return val;
}

// The D8 gather (src/aread8.cpp:228-257; ALG 1 / 2: src/D8flowpathextremeup.cpp:182-215; ALG 4-6: gridnet_eval): the value of
// the cell at ring slot ri (strip row r, column c) from its contributors `msk`; `con` becomes true at a contaminated contributor.
struct Eval { float val; bool con; };
template <bool USEW, int ALG, typename Mem>
__device__ __forceinline__ Eval d8_gather(const WArgs& a, const Mem& M, int ri, unsigned msk, int r, int c, float wv, float NOD, bool con) {
  if (ALG >= 4) return {gridnet_eval<ALG>(a, M, ri, msk, r, c), con};
  if (USEW) {
    float val = (ALG == 0 && nd_f(wv, a.w_nodata)) ? -1.0f : wv;
#pragma unroll
    for (int k = 1; k <= 8; ++k)
      if (msk & (1u << (k - 1))) {
        const float an = M.area[ri + drow(k) * RS + dcol(k)];
        if (nd_f(an, NOD)) con = true;
        else val = ALG == 0 ? val + an : ALG == 1 ? (an > val ? an : val) : (an < val ? an : val);
      }
    return {val, con};
  }
  // no weights: an area is -1 (nodata: contaminated) or a positive count, and a contaminated contributor contaminates the
  // cell — its value does not matter then
  float val = 1.0f, mn = 0.f;
#pragma unroll
  for (int k = 1; k <= 8; ++k)
    if (msk & (1u << (k - 1))) {
      const float an = M.area[ri + drow(k) * RS + dcol(k)];
      val = val + an;
      mn = fminf(mn, an);
    }
  if (mn < 0.f) con = true;          // (with -nc no area is ever -1 when it is gathered)
  return {val, con};
}

// src/areadinf.cpp:187-218: the share the contributor at ring slot ni (strip row rn) sends along direction kk is prop(its angle, kk).
// The contributor's node word says how it is obtained (dinf_field): for a regular cell one subtraction from a sector edge and one
// division by the sector's width (a table constant: div_recip) — the same doubles prop() / dinf_outflow form; irregular cells and
// strips without a common table take the interval search.
__device__ __forceinline__ double dinf_share(const WArgs& a, const Sector* sect, unsigned f, float av, int kk, int rn) {
  if (a.prop.uniform && f != 9u) {
    const bool upper = f >= 10u;
    const int k1 = (int)(upper ? f - 8u : f);
    const bool first = kk == k1 && !upper;
    const bool wrap = k1 == 8 && !first && !upper;                 // direction 1 from the wrap sector
    const Sector S = sect[wrap ? 0 : (upper ? k1 - 1 : k1)];
    double ad = (double)av;
    if (wrap) ad = (double)(float)(ad - 2.0 * TD_PI);            // prop()'s float-rounded a - 2 PI (src/commonLib.cpp:82)
    const double num = first ? S.hi - ad : ad - S.lo;
    return a.prop.safe ? div_recip(num, S.den, S.rden) : num / S.den;
  }
  return wshare_full(av, a.prop.uniform ? a.prop.ar[2] : theta_of_row(a.theta, a.s.ny, min(max(rn, 0), a.s.ny + 1)), kk);
}

// the area a D-infinity cell of strip row r adds itself (src/areadinf.cpp:216): the strip's one cell size, else its row's
__device__ __forceinline__ double own_area(const WArgs& a, int r) { return a.prop.uniform ? a.dx0 : a.dxc[min(r, a.s.ny) - 1]; }

template <bool DINF, bool USEW, int ALG>
__global__ void __launch_bounds__(workers_per_cta<DINF>() * 32, 1) k_sweep_warp(const WArgs a) {
  extern __shared__ __align__(16) unsigned char dsm[];
  using Mem = WarpMem<DINF>;
  const Strip& s = a.s;
  const int lane = (int)(threadIdx.x & 31u), wid = (int)(threadIdx.x >> 5);
  const unsigned lt = (1u << lane) - 1u;
  Mem& M = *reinterpret_cast<Mem*>(dsm + (size_t)wid * sizeof(Mem));
  const int myq = (int)((blockIdx.x * (blockDim.x >> 5) + (unsigned)wid) & (unsigned)(a.nsh - 1));   // this worker's queue shard
  const float NOD = (ALG == 0 || (ALG >= 4 && ALG <= 6)) ? -1.0f : TD_MISSINGFLOAT;      // the result raster's nodata: not evaluated / contaminated
  __shared__ Sector sect[9];
  if (DINF) {
    if (threadIdx.x < 9) { const int j = (int)threadIdx.x; sect[j].lo = a.prop.ar[j]; sect[j].hi = a.prop.ar[j + 1]; sect[j].den = a.prop.den[j]; sect[j].rden = a.prop.rden[j]; }
    __syncthreads();
  }

  int carry = -1;          // the tile this worker claimed at the end of its last visit (warp-uniform), else -1
  for (;;) {
    long long tk0 = 0, tk1 = 0, tk2 = 0, tk3 = 0;
    int t = carry;
    if (t < 0) {
      if (lane == 0) { if (a.stats) tk0 = clock64(); t = sched_pop(a, myq, wid == 0); if (a.stats) tk1 = clock64(); }
      t = __shfl_sync(FULL, t, 0);
      if (t < 0) return;
    } else if (a.stats && lane == 0) { tk0 = clock64(); tk1 = tk0; }
    carry = -1;
    const int ty = t / a.ntx, tx = t - ty * a.ntx;
    const int c0 = tx * TS, r0 = 1 + ty * TH;

    // ---- 1. dependency counts: lane = tile row (32 bytes each), before anything else
    unsigned g0[8];
    {
      const int r = r0 + lane;
      uint4 qa = make_uint4(FULL, FULL, FULL, FULL), qb = qa;
      if (r <= s.ny) {
        const uint4* src = reinterpret_cast<const uint4*>(a.cntw + (s.idx(r, c0) >> 2));
        qa = ld_cnt4(src, a.peer); qb = ld_cnt4(src + 1, a.peer);
      }
      g0[0] = qa.x; g0[1] = qa.y; g0[2] = qa.z; g0[3] = qa.w; g0[4] = qb.x; g0[5] = qb.y; g0[6] = qb.z; g0[7] = qb.w;
      uint4* dst = reinterpret_cast<uint4*>(M.cnt + lane * 8);
      dst[0] = qa; dst[1] = qb;
      M.evmask[lane] = 0u;
    }
    if (lane == 0) { M.sp = 0; M.next = 0; M.ovf = 0; }
    // the counts first, then the areas they announce: every lane's acquire covers its own count loads (and lane 0's or
    // lane wl's claim of the tile); the barrier after it orders them before the other lanes' copies
    fence_acquire(a.peer);
    __syncwarp();
    // ---- 2. areas, node words (and angles) of the tile and its ring: asynchronous copies straight into shared memory, all in
    //         flight at once (one round trip); what lies below the strip is filled in directly
#pragma unroll
    for (int j = 0; j < (RH * 8 + 31) / 32; ++j) {
      const int i = lane + 32 * j;
      if (i < RH * 8) {
        const int rr = i >> 3, q = i & 7;
        const int r = r0 - 1 + rr, c = c0 + 4 * q;
        const int so = rr * RS + 4 + 4 * q;
        if (r <= s.ny + 1) {
          const long long g = s.idx(r, c);
          if (a.peer && (r == 0 || r == s.ny + 1)) cp16(M.area + so, a.halo_in + (r == 0 ? 0 : s.pitch) + c);
          else cp16(M.area + so, a.area + g);
          if (DINF) cp16(M.ang + so, a.ang + g);
          cp8(M.node + so, a.node + g);
        } else {
          *reinterpret_cast<float4*>(M.area + so) = make_float4(NOD, NOD, NOD, NOD);
          if (DINF) *reinterpret_cast<float4*>(M.ang + so) = make_float4(0.f, 0.f, 0.f, 0.f);
          *reinterpret_cast<uint2*>(M.node + so) = make_uint2(0u, 0u);
        }
      }
    }
    // the ring columns: the west neighbours at slot 3 of their row (node words: two cells, slots 2 and 3), the east
    // neighbours at slot 36 (node words: slots 36 and 37).  Areas and angles change during the sweep: they are read past
    // the L1 (4-byte cp.async exists only in the L1-allocating flavour), node words never change.
#pragma unroll
    for (int rr = lane; rr < RH; rr += 32) {
      const int r = r0 - 1 + rr;
      const bool rowok = r <= s.ny + 1;
      const bool halo_row = a.peer && (r == 0 || r == s.ny + 1);
      const float* hrow = a.halo_in + (r == 0 ? 0 : s.pitch);
      const int sw = rr * RS + 3, se = rr * RS + RS;
      const bool west = rowok && c0 > 0, east = rowok && c0 + TS < s.pitch;
      const long long gw_ = s.idx(r, c0 - 1), ge_ = s.idx(r, c0 + TS);
      float aw = NOD, ae = NOD;
      if (west) { aw = __ldcg(halo_row ? hrow + (c0 - 1) : a.area + gw_); if (DINF) cp4(M.ang + sw, a.ang + gw_); cp4(M.node + sw - 1, a.node + gw_ - 1); }
      else { M.node[sw - 1] = 0; M.node[sw] = 0; }
      if (east) { ae = __ldcg(halo_row ? hrow + (c0 + TS) : a.area + ge_); if (DINF) cp4(M.ang + se, a.ang + ge_); cp4(M.node + se, a.node + ge_); }
      else { M.node[se] = 0; M.node[se + 1] = 0; }
      M.area[sw] = aw; M.area[se] = ae;
    }
    // ---- 3. cells that are ready (count 0): every lane keeps the ready cells of its own tile row as a bit mask
    unsigned rdy = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) rdy |= zero_nibble(g0[j]) << (4 * j);
    cp_wait_all();
    __syncwarp();
    if (a.stats && lane == 0) tk2 = clock64();

    // ---- 4. the wavefront inside the tile: one chain per lane; an idle lane goes on with the next ready cell of its own
    //         row, then (D-infinity) with a cell from the warp's fork stack
    int cur = -1;
    int iters = 0;
    for (;;) {
      if (cur < 0 && rdy) { const int b = __ffs(rdy) - 1; rdy &= rdy - 1; cur = lane * TS + b; }
      if (DINF) {
        const unsigned idle = __ballot_sync(FULL, cur < 0);
        if (idle) {
          const int n = min(ldv(&M.sp), STKCAP);
          if (n > 0) {
            const int take = min(__popc(idle), n);
            const int rank = __popc(idle & lt);
            if (cur < 0 && rank < take) cur = M.stk[n - 1 - rank];
            __syncwarp();
            if (lane == 0) M.sp = n - take;
          }
        }
      }
      const unsigned act = __ballot_sync(FULL, cur >= 0);
      if (ALG < 7 && act != 0u && (act & (act - 1u)) == 0u) {
        // ---- one chain left (a river crossing the tile, the tail of every visit; the fork stack is empty, or idle lanes
        // would have taken from it): the WHOLE warp follows it together.  Nothing diverges and nothing is contended: the cell
        // is warp-uniform, lanes 0..7 evaluate one contributor link each (D-infinity), everybody folds the products in
        // increasing k through shuffles, lane 0 alone touches the counts (plain loads and stores, no atomics, no ballots).
        // A second receiver that becomes ready ends the mode (it goes to the stack: the other lanes are needed again).
        int c = __shfl_sync(FULL, cur, __ffs(act) - 1);
        bool forked = false;
        do {
          ++iters;
          const int lr = c >> 5, lx = c & 31;
          const int ri = (lr + 1) * RS + lx + 4;
          float wv = 0.f;
          if (USEW) wv = a.w[s.idx(r0 + lr, c0 + lx)];
          const unsigned nd = M.node[ri];
          const unsigned msk = nd & 0xffu;
          bool con = (nd & NODE_CON) != 0;
          float val;
          if (!DINF) { const Eval e = d8_gather<USEW, ALG>(a, M, ri, msk, r0 + lr, c0 + lx, wv, NOD, con); val = e.val; con = e.con; }
          else {
            double prod = 0.;
            if (lane < 8 && ((msk >> lane) & 1u)) {
              const int k = lane + 1;
              const int dr = lut_drow(k);
              const int ni = ri + dr * RS + lut_dcol(k);
              const unsigned f = ((unsigned)M.node[ni] >> 8) & 0xfu;
              const float av = M.ang[ni];
              const float an = M.area[ni];
              const double p = dinf_share(a, sect, f, av, k > 4 ? k - 4 : k + 4, r0 + lr + dr);   // (the direction from that neighbour to the cell)
              // ALG 3 (src/dinfdecayaccum.cpp:205-235) is written out in each mode: a helper shared with the lane mode costs this
              // kernel 1-3 registers
              if (ALG == 3) {
                const float dmv = __ldg(a.dm + s.idx(r0 + lr + dr, c0 + lx + lut_dcol(k)));
                prod = (nd_f(an, NOD) || nd_f(dmv, a.dm_nodata)) ? __longlong_as_double(0x7ff8dead00000000ll) : (double)(float)((double)(dmv * an) * p);
              } else prod = nd_f(an, NOD) ? __longlong_as_double(0x7ff8dead00000000ll) : p * (double)an;   // NaN: a contaminated contributor
            }
            val = 0.f;
            if (ALG == 3) val = USEW ? wv : (float)own_area(a, r0 + lr);
            for (unsigned m = msk; m; m &= m - 1u) {               // increasing k: the reference's order of additions
              const double pr = __shfl_sync(FULL, prod, __ffs(m) - 1);
              if (pr != pr) con = true; else val = ALG == 3 ? val + (float)pr : (float)((double)val + pr);
            }
            if (ALG == 3) {}
            else if (USEW) val = val + wv;
            else val = (float)((double)val + own_area(a, r0 + lr));
          }
          if (con && a.contcheck) val = NOD;
          if (lane == 0) { M.area[ri] = val; M.evmask[lr] |= 1u << lx; }
          int next = -1;
#pragma unroll
          for (int j = 0; j < (DINF ? 2 : 1); ++j) {        // the receivers, classified like the lane mode's below
            int k;
            if (!DINF) k = (int)((nd >> 8) & 0xfu);
            else k = j == 0 ? dinf_node_k1(nd) : dinf_node_k2(nd);
            if (k < 1 || k > 8) continue;
            const int nlr = lr + lut_drow(k), nlx = lx + lut_dcol(k);
            if ((unsigned)nlr < (unsigned)TH && (unsigned)nlx < (unsigned)TS && r0 + nlr <= s.ny) {
              const int l2 = nlr * TS + nlx;
              const unsigned sh = (unsigned)(l2 & 3) * 8u;
              unsigned w = 0;
              if (lane == 0) { w = M.cnt[l2 >> 2]; M.cnt[l2 >> 2] = w - (1u << sh); }
              w = __shfl_sync(FULL, w, 0);
              if (((w >> sh) & 0xffu) == 1u) {
                if (next < 0) next = l2;
                else {
                  forked = true;
                  if (lane == 0) { const int slot = M.sp; if (slot < STKCAP) M.stk[slot] = (unsigned short)l2; else if (a.stats) M.ovf = 1; M.sp = slot + 1; }
                }
              }
            } else if (s.on_grid(r0 + nlr, c0 + nlx)) {
              if (lane == 0) { M.ext[M.next] = (unsigned short)(c | ((k - 1) << 11)); M.next = M.next + 1; }
            }
          }
          c = next;
          __syncwarp();            // lane 0's stores (area, counts) before the next cell's loads
        } while (c >= 0 && !forked);
        cur = lane == 0 ? c : -1;
        continue;
      }
      if (act == 0u) {
        if (!DINF) break;
        // forks that did not fit the stack are ready (count 0) and not evaluated: look once more
        const unsigned ev = M.evmask[lane];
#pragma unroll
        for (int j = 0; j < 8; ++j) rdy |= zero_nibble(M.cnt[lane * 8 + j]) << (4 * j);
        rdy &= ~ev;
        if (__ballot_sync(FULL, rdy != 0u) == 0u) break;
        continue;
      }
      ++iters;
      if (cur >= 0) {
        const int l = cur;
        const int lr = l >> 5, lx = l & 31;
        const int ri = (lr + 1) * RS + lx + 4;
        float wv = 0.f;
        if (USEW) wv = a.w[s.idx(r0 + lr, c0 + lx)];
        const unsigned nd = M.node[ri];
        const unsigned msk = nd & 0xffu;
        bool con = (nd & NODE_CON) != 0;
        float val;
        int cont = -1;
        if (!DINF) { const Eval e = d8_gather<USEW, ALG>(a, M, ri, msk, r0 + lr, c0 + lx, wv, NOD, con); val = e.val; con = e.con; }
        else {
          const int r = r0 + lr;
          val = 0.f;
          float loadin = 0.f;                                    // ALG 9: the load of the second substance that arrives
          if (ALG == 3) val = USEW ? wv : (float)own_area(a, r);
#pragma unroll 1
          for (unsigned m = msk; m; m &= m - 1u) {               // increasing k: the reference's order of additions
            const int k = __ffs(m);
            const int dr = lut_drow(k);
            const int ni = ri + dr * RS + lut_dcol(k);
            const unsigned f = ((unsigned)M.node[ni] >> 8) & 0xfu;
            const float av = M.ang[ni];
            const float an = M.area[ni];
            const double p = dinf_share(a, sect, f, av, k > 4 ? k - 4 : k + 4, r + dr);         // (the direction from that neighbour to this cell)
            if (ALG == 3) {
              const float dmv = __ldg(a.dm + s.idx(r + dr, c0 + lx + lut_dcol(k)));
              if (nd_f(an, NOD) || nd_f(dmv, a.dm_nodata)) con = true;
              else val = val + (float)((double)(dmv * an) * p);
            } else if (ALG == 7) {
              // src/DinfConcLimAccum.cpp:252-262: Concentration += p * ctpt * q * dm of the contributor (double products, float sum)
              const long long gi = s.idx(r + dr, c0 + lx + lut_dcol(k));
              const float qq = __ldg(a.w + gi), dmm = __ldg(a.dm + gi);
              if (nd_f(an, NOD) || nd_f(dmm, a.dm_nodata) || nd_f(qq, a.w_nodata)) con = true;
              else val = (float)((double)val + ((p * (double)an) * (double)qq) * (double)dmm);
            } else if (ALG == 8 || ALG == 9) {
              // src/DinfTransLimAccum.cpp:252-266: transin += p * transport of the contributor; loadin += p * that transport * its concentration
              float nt = 0.f;
              if (nd_f(an, NOD)) con = true; else { val = (float)((double)val + p * (double)an); nt = an; }
              if (ALG == 9) {
                // a contributor in a halo row: in peer mode its concentration arrived with its transport (deliver_peer), in
                // rounds mode the caller exchanged the concentration rows with the value rows
                const int rn = r + dr, cc = c0 + lx + lut_dcol(k);
                const float cn = (a.peer && (rn == 0 || rn == s.ny + 1)) ? ldv(a.halo_in + 2 * s.pitch + (rn == 0 ? 0 : s.pitch) + cc)
                                                                         : ldv(a.x.out3 + s.idx(rn, cc));
                if (nd_f(cn, NOD)) con = true; else loadin = (float)((double)loadin + (p * (double)nt) * (double)cn);
              }
            } else if (nd_f(an, NOD)) con = true; else val = (float)((double)val + p * (double)an);
          }
          if (ALG == 3) {}
          else if (ALG == 7) {
            // src/DinfConcLimAccum.cpp:242-270: only cells with a positive discharge have a concentration; an indicator cell is a
            // source at the solubility (its neighbours are not looked at: it cannot be contaminated)
            const float dgv = (float)a.x.dg[s.idx(r, c0 + lx)];
            if (!(wv > 0.f)) { val = NOD; con = false; }
            else if (dgv > 0.f) { val = a.x.csol; con = false; }
            else val = val / wv;
          } else if (ALG == 8 || ALG == 9) {
            // src/DinfTransLimAccum.cpp:237-238,268-302: cells whose supply, capacity (or supply concentration) is nodata are not evaluated
            const long long gc = s.idx(r, c0 + lx);
            const float tcc = __ldg(a.dm + gc);
            float cinv = 0.f;
            bool ev = !nd_f(wv, a.w_nodata) && !nd_f(tcc, a.dm_nodata);
            if (ALG == 9) { cinv = __ldg(a.x.cin + gc); ev = ev && !nd_f(cinv, a.x.cin_nodata); }
            if (!ev) { val = NOD; con = false; }
            else {
              const float transin = val;
              float transout, depp;
              if ((transin + wv) > tcc) { transout = tcc; depp = transin + wv - transout; }
              else { transout = transin + wv; depp = 0.f; }
              float cs = 0.f;
              if (ALG == 9) {
                float loadout;
                if (transout < transin) loadout = transin > 0.f ? loadin * transout / transin : 0.f;      // no erosion from the cell
                else loadout = loadin + cinv * (transout - transin);
                cs = transout > 0.f ? loadout / transout : 0.f;
              }
              const bool bad = con && a.contcheck;
              a.x.out2[gc] = bad ? NOD : depp;
              if (ALG == 9) { stv(a.x.out3 + gc, bad ? NOD : cs); __threadfence_block(); }
              val = transout;
            }
          }
          else if (USEW) val = val + wv;
          else val = (float)((double)val + own_area(a, r));
        }
        if (con && a.contcheck) val = NOD;
        M.area[ri] = val;
        atomicOr(&M.evmask[lr], 1u << lx);
        // (the areas are in shared memory before the counts that announce them are read: every lane that continues with a
        //  receiver does so after the __syncwarp() that ends this iteration)
        // ---- the receivers: src/aread8.cpp:261-272, src/areadinf.cpp:221-239.  The one-chain mode above classifies them the same
        //      way; a helper shared by both modes costs the D-infinity kernels of ALG 3 and 9 a register each.
#pragma unroll
        for (int j = 0; j < (DINF ? 2 : 1); ++j) {
          int k;
          if (!DINF) k = (int)((nd >> 8) & 0xfu);
          else k = j == 0 ? dinf_node_k1(nd) : dinf_node_k2(nd);
          if (k < 1 || k > 8) continue;
          const int nlr = lr + lut_drow(k), nlx = lx + lut_dcol(k);
          if ((unsigned)nlr < (unsigned)TH && (unsigned)nlx < (unsigned)TS && r0 + nlr <= s.ny) {       // a cell of this tile
            const int l2 = nlr * TS + nlx;
            const unsigned sh = (unsigned)(l2 & 3) * 8u;
            const unsigned old = atomicSub(&M.cnt[l2 >> 2], 1u << sh);
            if (((old >> sh) & 0xffu) == 1u) {
              if (cont < 0) cont = l2;
              else {                                                       // a second ready receiver: an idle lane takes it
                const int slot = atomicAdd(&M.sp, 1);
                if (slot < STKCAP) M.stk[slot] = (unsigned short)l2; else if (a.stats) M.ovf = 1;
              }
            }
          } else if (s.on_grid(r0 + nlr, c0 + nlx)) {
            M.ext[atomicAdd(&M.next, 1)] = (unsigned short)(l | ((k - 1) << 11));
          }
        }
        cur = cont;
      }
      __syncwarp();              // areas and counts of this iteration are visible to every lane in the next one
    }

    if (a.stats && lane == 0) tk3 = clock64();

    // ---- 5. write back what this visit evaluated (row by row, only rows with evaluated cells), then publish counts and
    //         deliver the crossings
    const unsigned evs = M.evmask[lane];
    for (unsigned rows = __ballot_sync(FULL, evs != 0u); rows; rows &= rows - 1u) {
      const int lr = __ffs(rows) - 1;
      const unsigned evr = __shfl_sync(FULL, evs, lr);
      if ((evr >> lane) & 1u) a.area[s.idx(r0 + lr, c0 + lane)] = M.area[(lr + 1) * RS + lane + 4];
    }
    // The counts.  The shared-memory count of a cell this visit evaluated is 0, of any other cell its count at the start
    // minus the arrivals from inside the tile; bytes >= 0x80 (not a node / evaluated before: flow into a cell without a
    // direction still decrements them in shared memory) keep their value.  One 32-bit delta per word carries all four cells
    // (every byte of the sum stays within 0..0xFE, so nothing carries between bytes): evaluated -> 0xFE, others minus the
    // local arrivals.  Words without a cell of the tile's rim (or of the strip's last row, which a neighbour strip feeds)
    // are touched by nobody else while the tile runs: plain stores, before the fence, like the areas.  The others are
    // added atomically after it; a zero byte in the result is a cell that became ready through arrivals from outside meanwhile.
    unsigned dl[8];
    {
      const int myr = r0 + lane;
      const bool rimrow = lane == 0 || lane == TH - 1 || myr >= s.ny;
      unsigned* gw = a.cntw + (s.idx(min(myr, s.ny), c0) >> 2);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const unsigned was = g0[j];
        unsigned now = M.cnt[lane * 8 + j];
        const unsigned keep = ((was >> 7) & 0x01010101u) * 0xffu;
        now = (now & ~keep) | (was & keep);
        const unsigned e4 = (evs >> (4 * j)) & 0xfu;
        dl[j] = now - was + ((e4 * 0x00204081u) & 0x01010101u) * 0xfeu;
        if (j >= 1 && j <= 6 && !rimrow && dl[j] != 0u) { gw[j] = was + dl[j]; dl[j] = 0u; }
      }
    }
    __syncwarp();
    fence_release(a.peer);    // every lane's stores (ordered before it by the barrier) before any lane's first atomic
    // One batch of atomics, all in flight at once: the flow that leaves the tile through each lane's first crossing (e = lane)
    // and the rim's counts.  Then, from the values they return: the activations (every lane holds back the last tile its
    // crossings made ready, `pend`, crossing `pend_e`, and activates the others at once), the carry and whether the tile is
    // dirty.  Crossings beyond the first 32 (a visit that drained much of the tile, not a river's hop) follow one by one.
    const int ne = M.next;
    int pend = -1, pend_e = -1;
    // crossing e: its atomic (or halo record / peer delivery); the tile of the target cell, whose count byte (at bit `sh` of
    // the returned word `old`) it decremented, or -1
    auto cross = [&](int e, unsigned& old, unsigned& sh) -> int {
      const int l = M.ext[e] & 0x7ff, k = (M.ext[e] >> 11) + 1;
      const int lr = l >> 5, lx = l & 31;
      const int nlr = lr + lut_drow(k), nlx = lx + lut_dcol(k);
      const int r = r0 + nlr, c = c0 + nlx;
      if (r == 0 || r == s.ny + 1) {
        if (a.peer) deliver_peer<ALG>(a, r == 0, c0 + lx, M.area[(lr + 1) * RS + lx + 4], c);   // the source's area is still in shared memory
        else atomicAdd(a.halo + (r == 0 ? 0 : s.pitch) + c, 1);
        return -1;
      }
      if (!((unsigned)M.node[(nlr + 1) * RS + nlx + 4] & NODE_VALID)) return -1;
      const long long ci = s.idx(r, c);
      sh = (unsigned)(ci & 3) * 8u;
      old = W_ADD_IF(a.peer && (r == 1 || r == s.ny), a.cntw + (ci >> 2), 0u - (1u << sh));
      return ((r - 1) / TH) * a.ntx + c / TS;
    };
    unsigned xo = 0u, xsh = 0u, ro[8];
    const int xt = lane < ne ? cross(lane, xo, xsh) : -1;
    const int myr = r0 + lane;
#pragma unroll
    for (int j = 0; j < 8; ++j) ro[j] = 0u;
    if (myr <= s.ny) {
      unsigned* gw = a.cntw + (s.idx(myr, c0) >> 2);
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (dl[j] != 0u) ro[j] = W_ADD_IF(a.peer && (myr == 1 || myr == s.ny), gw + j, dl[j]);
    }
    if (xt >= 0 && ((xo >> xsh) & 0xffu) == 1u) { pend = xt; pend_e = lane; }
    for (int e = lane + 32; e < ne; e += 32) {
      unsigned o, sh;
      const int tt = cross(e, o, sh);
      if (tt >= 0 && ((o >> sh) & 0xffu) == 1u) {
        if (pend >= 0) sched_activate(a, pend);
        pend = tt; pend_e = e;
      }
    }
    bool dirty = false;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (dl[j] != 0u && zero_bytes(ro[j] + dl[j])) dirty = true;
    dirty = __ballot_sync(FULL, dirty) != 0u;
    // The carry: of the tiles of this strip made ready by a crossing, the one of the LAST crossing made (normally the river
    // that the one-chain mode followed to the tile's edge) is visited next by this worker, without the ticket queue: claimed
    // idle -> running here, it skips the push, the pop, a waiting worker's back-off and the queue behind other tiles.  A tile
    // that is queued or running already (or every tile, with EXP_NO_CARRY) is activated as before.  The claim (lane wl) and
    // the release of this tile (lane 0) go out together.
    int hi = pend_e;
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) hi = max(hi, __shfl_xor_sync(FULL, hi, d));
    const int wl = hi & 31;                                 // crossing e was delivered by lane e % 32
    const int ct = hi >= 0 ? __shfl_sync(FULL, pend, wl) : -1;
    int claim = -1, rel = -1;
    if (hi >= 0 && lane == wl && !(a.exp & EXP_NO_CARRY)) claim = W_CAS_IF(edge_tile(a, ct), a.state + ct, 0, 2);
    if (lane == 0) rel = sched_release(a, t, dirty);
    if (hi >= 0) {
      if (lane == wl) {
        // the claim's result is consumed (the branch) before the carried visit loads the tile's counts, so those loads cannot
        // be issued before the claim was performed: whoever delivers into the tile after it re-activates it (2 -> 3)
        if (claim == 0) {
          carry = ct;
          if (a.stats) atomicAdd(a.stat, 1ull);
        } else sched_activate(a, ct);
      } else if (pend >= 0 && pend != ct) sched_activate(a, pend);   // (the claim or the activation of `ct` covers a lane's own `ct`)
      carry = __shfl_sync(FULL, carry, wl);
    }
    __syncwarp();             // every lane's pushes before lane 0's done
    if (lane == 0) sched_finish(a, t, rel, carry < 0);
    if (a.stats) {
      int tot = __popc(evs);
#pragma unroll
      for (int d = 16; d >= 1; d >>= 1) tot += __shfl_xor_sync(FULL, tot, d);
      if (lane == 0) {
        const long long tk4 = clock64();
        atomicAdd(a.stat + 3, 1ull);
        atomicAdd(a.stat + 4, (unsigned long long)(tk1 - tk0));
        atomicAdd(a.stat + 5, (unsigned long long)(tk2 - tk1));
        atomicAdd(a.stat + 6, (unsigned long long)(tk3 - tk2));
        atomicAdd(a.stat + 7, (unsigned long long)(tk4 - tk3));
        atomicAdd(a.stat + 1, (unsigned long long)tot);
        atomicAdd(a.stat + 2, (unsigned long long)iters);
        if (DINF && M.ovf) atomicAdd(a.stat + 8, 1ull);
      }
    }
    __syncwarp();
  }
}

// Applies the dependency decrements received from the neighbour strips (addBorders, src/linearpart.h:314-328 and
// src/aread8.cpp:283-297): dec_top[c] arrivals for the cell (row 1, c), dec_bot[c] for (row ny, c).  A count that
// reaches zero queues the cell's tile.
__global__ void k_wapply_halo(WArgs a, const int* __restrict__ dec_top, const int* __restrict__ dec_bot) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= a.s.nx) return;
#pragma unroll
  for (int side = 0; side < 2; ++side) {
    const int* dec = side == 0 ? dec_top : dec_bot;
    if (dec == nullptr) continue;
    const int d = dec[c];
    if (d <= 0) continue;
    const int r = side == 0 ? 1 : a.s.ny;
    const long long ci = a.s.idx(r, c);
    if (!(a.node[ci] & NODE_VALID)) continue;
    const unsigned sh = (unsigned)(ci & 3) * 8u;
    const unsigned old = atomicAdd(a.cntw + (ci >> 2), 0u - ((unsigned)d << sh));
    if ((int)((old >> sh) & 0xffu) == d) sched_activate(a, ((r - 1) / a.th) * a.ntx + c / TS);
  }
}

// between two runs of the round-based exchange: tickets abandoned at the end of the previous run are void (every ring slot is empty then)
__global__ void k_wsched_reset(unsigned long long* ctr) { for (int i = threadIdx.x; i < C_WORDS; i += blockDim.x) ctr[i] = (i == C_ACTIVE) ? 1ull : 0ull; }

int wargs(td_ctx* ctx, WArgs& a, const Strip& s) {
  a.s = s;
  a.area = nullptr; a.w = nullptr; a.ang = nullptr; a.dx0 = 0.; a.usew = 0; a.contcheck = 1; a.w_nodata = 0.f; a.theta = nullptr; a.dxc = nullptr; a.halo = nullptr; a.dm = nullptr; a.dm_nodata = 0.f; a.dist = nullptr;
  a.th = TH;
  a.ntx = (s.nx + TS - 1) / TS; a.nty = (s.ny + a.th - 1) / a.th;
  a.stats = 0; a.exp = 0;
  a.peer = 0; a.G = nullptr; a.halo_in = nullptr; a.up = PeerStrip(); a.down = PeerStrip();
  const long long nt = (long long)a.ntx * a.nty;
  if (nt > (1ll << 30)) { set_error("strip has too many tiles"); return TD_ERR_ARG; }
  // queue shards: a power of two, at most MAXSH and never more than the workers a launch has (>= min(tiles, one CTA per SM))
  int nsh = 1;
  while (nsh * 2 <= MAXSH && nsh * 2 <= nt) nsh *= 2;
  // a shard's ring: its tiles (each queued at most once) + the tickets of waiting workers (< 2^13 workers per device)
  const unsigned long long need = (unsigned long long)((nt + nsh - 1) / nsh) + (1u << 13);
  int qshift = 14;
  while ((1ull << qshift) < need) ++qshift;
  a.nsh = nsh; a.qshift = qshift; a.qmask = (1u << qshift) - 1u;
  TD_CUDA(ctx->tileflags.ensure((size_t)nt * 4 + ((size_t)nsh << qshift) * 4));
  a.state = ctx->tileflags.as<int>();
  a.tq = a.state + nt;
  TD_CUDA(ctx->wsched.ensure(C_WORDS * sizeof(unsigned long long)));
  a.ctr = ctx->wsched.as<unsigned long long>();
  a.stat = ctx->d_ctr + 24;
  a.node = ctx->node.as<unsigned short>();
  a.cntw = ctx->cnt.as<unsigned>();
  return TD_OK;
}

// The instantiations of k_sweep_warp: which (D-infinity, weights, algebra) combinations exist and the grids each one requires.
enum : unsigned { NEED_W = 1, NEED_DM = 2, NEED_DIST = 4, NEED_EXTRA = 8, NEED_DG = 16, NEED_OUT2 = 32, NEED_CIN = 64, NEED_OUT3 = 128 };
using SweepLaunch = void (*)(const WArgs&, int, int, size_t, cudaStream_t);
template <bool D, bool U, int A>
void launch_sweep(const WArgs& a, int g, int threads, size_t smem, cudaStream_t st) {
  k_sweep_warp<D, U, A><<<g, threads, smem, st>>>(a);
}
struct SweepKernel {
  bool dinf, usew;
  int alg;
  unsigned need;           // NEED_* bits
  const void* kern;        // for the occupancy queries
  SweepLaunch launch;
  int threads;
  size_t smem;
};
template <bool D, bool U, int A>
SweepKernel sweep_kernel(unsigned need) {
  return {D, U, A, need, (const void*)k_sweep_warp<D, U, A>, launch_sweep<D, U, A>, workers_per_cta<D>() * 32, sizeof(WarpMem<D>) * workers_per_cta<D>()};
}
const SweepKernel SWEEPS[] = {
    sweep_kernel<false, false, 0>(0), sweep_kernel<false, true, 0>(0), sweep_kernel<true, false, 0>(0), sweep_kernel<true, true, 0>(0),
    sweep_kernel<false, true, 1>(0), sweep_kernel<false, true, 2>(0),
    sweep_kernel<true, false, 3>(NEED_DM), sweep_kernel<true, true, 3>(NEED_DM),
    sweep_kernel<false, false, 4>(NEED_DIST), sweep_kernel<false, false, 5>(NEED_DIST), sweep_kernel<false, false, 6>(NEED_DIST),
    sweep_kernel<true, true, 7>(NEED_W | NEED_DM | NEED_EXTRA | NEED_DG),
    sweep_kernel<true, true, 8>(NEED_W | NEED_DM | NEED_EXTRA | NEED_OUT2),
    sweep_kernel<true, true, 9>(NEED_W | NEED_DM | NEED_EXTRA | NEED_OUT2 | NEED_CIN | NEED_OUT3),
};
static_assert(sizeof(SWEEPS) / sizeof(SWEEPS[0]) == td_ctx::SWEEP_KERNELS, "td_ctx::wgrid has one slot per sweep kernel");
}  // namespace

// Queues every tile of the strip (start of a sweep).
int wsweep_begin(td_ctx* ctx, const Strip& s, cudaStream_t st) {
  WArgs a;
  if (int rc = wargs(ctx, a, s)) return rc;
  const int nt = a.ntx * a.nty;
  TD_CUDA(zero_words(a.ctr, C_WORDS * sizeof(unsigned long long), st));
  TD_CUDA(zero_words(a.tq, ((size_t)a.nsh << a.qshift) * sizeof(int), st));
  k_wsched_init<<<(nt + 255) / 256, 256, 0, st>>>(a.state, a.tq, nt, a.ctr, a.stat, a.nsh, a.qshift, a.qmask);
  TD_LAUNCHED();
  TD_CUDA(cudaGetLastError());
  return TD_OK;
}

// Decrements that crossed the strip boundary (from the neighbours' halo records); queues the tiles whose cells became
// ready.  Must be called between two wsweep_run calls.
int wsweep_apply_halo(td_ctx* ctx, const Strip& s, const int* dec_top, const int* dec_bot, cudaStream_t st) {
  WArgs a;
  if (int rc = wargs(ctx, a, s)) return rc;
  k_wsched_reset<<<1, 256, 0, st>>>(a.ctr);
  TD_LAUNCHED();
  k_wapply_halo<<<(s.nx + 255) / 256, 256, 0, st>>>(a, dec_top, dec_bot);
  TD_LAUNCHED();
  TD_CUDA(cudaGetLastError());
  return TD_OK;
}

// Runs the evaluation wavefront over the queued tiles until no tile of the strip has a ready cell left.
int wsweep_run(td_ctx* ctx, bool dinf, float* area, const float* w, const float* ang, const Strip& s, float w_nodata, int usew,
               int contcheck, const double* theta, const double* dxc, int* halo, cudaStream_t st, int alg, const float* dm, float dm_nodata,
               const float* dist, const SweepExtra* extra) {
  int row = -1;
  for (int i = 0; i < td_ctx::SWEEP_KERNELS; ++i)
    if (SWEEPS[i].dinf == dinf && SWEEPS[i].usew == (usew != 0) && SWEEPS[i].alg == alg) row = i;
  const unsigned have = (w ? NEED_W : 0u) | (dm ? NEED_DM : 0u) | (dist ? NEED_DIST : 0u) |
                        (extra ? NEED_EXTRA | (extra->dg ? NEED_DG : 0u) | (extra->out2 ? NEED_OUT2 : 0u) | (extra->cin ? NEED_CIN : 0u) | (extra->out3 ? NEED_OUT3 : 0u) : 0u);
  if (row < 0) { set_error("wsweep_run: no sweep for this algebra with this flow model and weights"); return TD_ERR_ARG; }
  if (const unsigned miss = SWEEPS[row].need & ~have) {
    static const char* const grid[8] = {"w", "dm", "dist", "extra", "extra->dg", "extra->out2", "extra->cin", "extra->out3"};
    set_error(std::string("wsweep_run: algebra ") + std::to_string(alg) + " requires the grid " + grid[__builtin_ctz(miss)]);
    return TD_ERR_ARG;
  }
  const SweepKernel& K = SWEEPS[row];
  if (alg == 9 && ctx->peer_on && ctx->peer_halo.cap < sizeof(float) * 4 * (size_t)s.pitch) {
    set_error("wsweep_run: peer mode of the transport limited accumulation with a concentration needs the halo buffer of sweep_peer_export");
    return TD_ERR_ARG;
  }
  WArgs a;
  if (int rc = wargs(ctx, a, s)) return rc;
  a.area = area; a.w = w; a.ang = ang; a.usew = usew; a.contcheck = contcheck;
  a.w_nodata = w_nodata; a.theta = theta; a.dxc = dxc; a.halo = halo; a.dm = dm; a.dm_nodata = dm_nodata; a.dist = dist;
  if (extra) a.x = *extra;
  a.prop = ctx->prop;
  if (!dinf) a.prop.uniform = 0;
  a.peer = ctx->peer_on;
  if (a.peer) {
    auto fill = [](const td_ctx::PeerInfo& pi, PeerStrip& P) {
      P.valid = pi.valid;
      P.cntw = (unsigned*)pi.cntw; P.state = (int*)pi.tileflags; P.tq = P.state + pi.nt; P.ctr = (unsigned long long*)pi.dctr;
      P.halo_in = (float*)pi.halo_in; P.qmask = (unsigned)pi.qmask; P.ntx = pi.ntx; P.ny = pi.ny; P.nsh = pi.nsh; P.qshift = pi.qshift;
    };
    fill(ctx->peer_up, a.up); fill(ctx->peer_down, a.down);
    a.G = (unsigned long long*)ctx->peer_G;
    a.halo_in = ctx->peer_halo.as<float>();
    if ((s.has_top && !a.up.valid) || (s.has_bot && !a.down.valid) || !a.G) { set_error("peer mode: neighbours are not connected"); return TD_ERR_ARG; }
  }
  const char* te = getenv("TAUDEM_B200_TIMING");
  a.stats = (te && atoi(te) > 0) ? 1 : 0;
  if (const char* xe = getenv("TAUDEM_B200_EXP")) a.exp = atoi(xe);
  a.dx0 = ctx->dx0;
  int& per_dev = ctx->wgrid[row];
  if (!per_dev) {
    int dev = 0, sms = 0, occ = 0;
    TD_CUDA(cudaGetDevice(&dev));
    TD_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    TD_CUDA(cudaFuncSetAttribute(K.kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)K.smem));
    TD_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, K.kern, K.threads, K.smem));
    if (occ < 1) { set_error("sweep kernel does not fit on an SM"); return TD_ERR_CUDA; }
    per_dev = sms * occ;     // persistent: every CTA is resident, so queue waits cannot deadlock
  }
  const long long nt = (long long)a.ntx * a.nty;
  const int warps = K.threads / 32;
  K.launch(a, (int)std::min<long long>(per_dev, (nt + warps - 1) / warps), K.threads, K.smem, st);
  TD_LAUNCHED();
  TD_CUDA(cudaGetLastError());
  return TD_OK;
}

namespace {
__global__ void k_add_G(unsigned long long* G, unsigned long long v) { if (threadIdx.x == 0) { atomicAdd_system(G, v); __threadfence_system(); } }
void close_peer(td_ctx::PeerInfo& pi) {
  if (pi.cntw) cudaIpcCloseMemHandle(pi.cntw);
  if (pi.tileflags) cudaIpcCloseMemHandle(pi.tileflags);
  if (pi.dctr) cudaIpcCloseMemHandle(pi.dctr);
  if (pi.halo_in) cudaIpcCloseMemHandle(pi.halo_in);
  pi = td_ctx::PeerInfo();
}
}  // namespace

// ---- peer mode plumbing (CUDA IPC).  export: make sure every buffer a neighbour touches exists at its final size and
// hand out its IPC handle; connect: open a neighbour's (or rank 0's counter) handles.
int sweep_peer_export(td_ctx* ctx, const Strip& s, int dinf, unsigned char* handles, int* meta, cudaStream_t st) {
  WArgs a;
  ctx->sweep_dinf = dinf ? 1 : 0;
  const size_t n = (size_t)s.cells();
  TD_CUDA(ctx->node.ensure(n * 2));
  TD_CUDA(ctx->cnt.ensure((n + 3) / 4 * 4));
  if (int rc = wargs(ctx, a, s)) return rc;
  TD_CUDA(ctx->peer_halo.ensure(sizeof(float) * 4 * (size_t)s.pitch));     // areas, then ALG 9's concentrations: row above, row below each
  TD_CUDA(ctx->gbuf.ensure(64));
  TD_CUDA(cudaMemsetAsync(ctx->gbuf.p, 0, 64, st));
  TD_CUDA(cudaStreamSynchronize(st));
  void* ptrs[5] = {ctx->cnt.p, ctx->tileflags.p, ctx->wsched.p, ctx->peer_halo.p, ctx->gbuf.p};
  for (int i = 0; i < 5; ++i) {
    cudaIpcMemHandle_t h;
    TD_CUDA(cudaIpcGetMemHandle(&h, ptrs[i]));
    memcpy(handles + 64 * i, &h, 64);
  }
  meta[0] = (int)a.qmask; meta[1] = a.ntx; meta[2] = s.ny; meta[3] = a.th; meta[4] = a.ntx * a.nty; meta[5] = a.nsh; meta[6] = a.qshift; meta[7] = 0;
  return TD_OK;
}

// which: 0 = strip above, 1 = strip below, 2 = owner of the global counter (handles == NULL: this rank)
int sweep_peer_connect(td_ctx* ctx, int which, const unsigned char* handles, const int* meta) {
  auto open = [](const unsigned char* h64, void** out) -> cudaError_t {
    cudaIpcMemHandle_t h; memcpy(&h, h64, 64);
    return cudaIpcOpenMemHandle(out, h, cudaIpcMemLazyEnablePeerAccess);
  };
  if (which == 2) {
    if (ctx->peer_G_opened && ctx->peer_G) cudaIpcCloseMemHandle(ctx->peer_G);
    ctx->peer_G_opened = false;
    if (!handles) { ctx->peer_G = ctx->gbuf.p; return TD_OK; }
    TD_CUDA(open(handles + 64 * 4, &ctx->peer_G));
    ctx->peer_G_opened = true;
    return TD_OK;
  }
  td_ctx::PeerInfo& pi = which == 0 ? ctx->peer_up : ctx->peer_down;
  if (!handles && meta && pi.valid) {       // same buffers, new geometry
    pi.qmask = meta[0]; pi.ntx = meta[1]; pi.ny = meta[2]; pi.th = meta[3]; pi.nt = meta[4]; pi.nsh = meta[5]; pi.qshift = meta[6];
    return TD_OK;
  }
  close_peer(pi);
  if (!handles) return TD_OK;
  TD_CUDA(open(handles, &pi.cntw));
  TD_CUDA(open(handles + 64, &pi.tileflags));
  TD_CUDA(open(handles + 128, &pi.dctr));
  TD_CUDA(open(handles + 192, &pi.halo_in));
  pi.qmask = meta[0]; pi.ntx = meta[1]; pi.ny = meta[2]; pi.th = meta[3]; pi.nt = meta[4]; pi.nsh = meta[5]; pi.qshift = meta[6]; pi.valid = 1;
  return TD_OK;
}

// start of a peer-mode sweep: queue all tiles, count this strip as active in the global counter.  The caller must put a barrier
// between this call and wsweep_run on every rank (nobody may see G == 0 before everybody announced).
int sweep_peer_begin(td_ctx* ctx, const Strip& s, cudaStream_t st) {
  ctx->peer_on = 1;
  if (int rc = wsweep_begin(ctx, s, st)) return rc;
  WArgs a;
  if (int rc = wargs(ctx, a, s)) return rc;
  TD_CUDA(zero_words(ctx->peer_halo.p, sizeof(float) * 4 * (size_t)s.pitch, st));
  k_add_G<<<1, 32, 0, st>>>((unsigned long long*)ctx->peer_G, 1ull);     // this strip is active
  TD_LAUNCHED();
  TD_CUDA(cudaStreamSynchronize(st));
  return TD_OK;
}
void sweep_peer_off(td_ctx* ctx) { ctx->peer_on = 0; }

}  // namespace td
