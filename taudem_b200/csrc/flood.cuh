// The level-by-level flood that d8hdisttostrm / d8vdisttostrm (disttostrm.cu) and dinfdistdown (dinfdistdown.cu) run: a frontier
// list of strip cells, one launch per level, and batches of DTS_BATCH levels per host read-back.
//   list      : one entry per strip cell at most; ctr[0] = entries appended, ctr[1] = entries consumed by the levels run so far.
//   bounds    : level t's frontier is list[bounds[t - 1], bounds[t]); the last block of level t records bounds[t + 1] = ctr[0]
//               (flood_level_done), so a batch of levels runs without a host round trip (as k_bfs_level in flats.cu).
// A level kernel walks its frontier with a grid-stride loop, appends the next level's cells with dts_append and ends with
// flood_level_done; flood_levels runs such kernels until a level comes out empty.
#pragma once
#include <string.h>

#include <vector>

#include "common.cuh"
#include "kernels.h"

namespace td {

// warp-aggregated append of v to list (one atomic per warp)
__device__ __forceinline__ void dts_append(unsigned* list, unsigned long long* ctr, bool pred, unsigned v) {
  const unsigned m = __ballot_sync(__activemask(), pred);
  if (!pred) return;
  const int lane = threadIdx.x & 31;
  const int leader = __ffs(m) - 1;
  unsigned long long base = 0;
  if (lane == leader) base = atomicAdd(ctr, (unsigned long long)__popc(m));
  base = __shfl_sync(m, base, leader);
  list[base + __popc(m & ((1u << lane) - 1u))] = v;
}

// The NaN that x86 SSE arithmetic gives (the reference's, where a NaN travels): a NaN result carries the first NaN operand,
// quieted, and an invalid operation on numbers (inf - inf) gives the default NaN 0xffc00000.  The GPU's own NaN result is 0x7fffffff.
__device__ __forceinline__ float dts_quiet(float a, unsigned set) {
  unsigned u;
  memcpy(&u, &a, 4);
  u |= set;
  memcpy(&a, &u, 4);
  return a;
}
__device__ __forceinline__ float dts_x86(float r, float a, float b) {
  if (r == r) return r;
  if (a != a) return dts_quiet(a, 0x00400000u);
  if (b != b) return dts_quiet(b, 0x00400000u);
  return dts_quiet(0.0f, 0xffc00000u);
}

// the end of level t: the last block to finish records where level t + 1 ends
__device__ __forceinline__ void flood_level_done(unsigned long long* bounds, int t, const unsigned long long* ctr, unsigned* blkdone) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(blkdone, 1u) == gridDim.x - 1) {          // the last block: every append of this level is done
      __threadfence();
      bounds[t + 1] = *reinterpret_cast<const volatile unsigned long long*>(ctr);
      *blkdone = 0;
    }
  }
}

// Levels until the frontier is empty: level(t) launches level t of a batch (t = 1..DTS_BATCH) on st.  *cells = the list entries
// appended before this call and not yet consumed, plus those the levels appended; *levels = the non-empty levels run.
template <class Level>
int flood_levels(const DtsBufs& b, Level&& level, unsigned long long* cells, long long* levels, cudaStream_t st) {
  // where the frontier stands: [consumed, appended)
  unsigned long long hc[2] = {0, 0};
  std::vector<unsigned long long> hb(DTS_BATCH);
  TD_CUDA(cudaMemcpyAsync(hc, b.ctr, sizeof hc, cudaMemcpyDeviceToHost, st));
  TD_CUDA(cudaStreamSynchronize(st));
  const unsigned long long start = hc[1];
  unsigned long long lo = start, hi = hc[0];
  long long nlev = 0;
  while (hi > lo) {
    // bounds[0, 1] = the frontier; levels 1..DTS_BATCH write bounds[2 .. DTS_BATCH + 1]
    TD_CUDA(cudaMemcpyAsync(b.bounds, b.ctr + 1, sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st));
    TD_CUDA(cudaMemcpyAsync(b.bounds + 1, b.ctr, sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st));
    for (int t = 1; t <= DTS_BATCH; ++t) {
      level(t);
      TD_LAUNCHED();
    }
    TD_CUDA(cudaGetLastError());
    TD_CUDA(cudaMemcpyAsync(hb.data(), b.bounds + 2, sizeof(unsigned long long) * DTS_BATCH, cudaMemcpyDeviceToHost, st));
    TD_CUDA(cudaMemcpyAsync(b.ctr + 1, b.bounds + DTS_BATCH, sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st));   // consumed
    TD_CUDA(cudaStreamSynchronize(st));
    unsigned long long prev = hi;
    ++nlev;                                                     // level 1 of the batch had cells
    for (int j = 0; j < DTS_BATCH; ++j) {
      if (hb[j] == prev) break;                          // level j + 2 is empty
      if (j + 1 < DTS_BATCH) ++nlev;
      prev = hb[j];
    }
    lo = DTS_BATCH >= 2 ? hb[DTS_BATCH - 2] : hi;        // the frontier after the batch: [bounds[B], bounds[B + 1])
    hi = hb[DTS_BATCH - 1];
  }
  if (cells) *cells = hi - start;
  if (levels) *levels = nlev;
  return TD_OK;
}

}  // namespace td
