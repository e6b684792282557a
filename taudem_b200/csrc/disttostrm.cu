// d8hdisttostrm / d8vdisttostrm: the D8 horizontal or vertical distance from every cell down its flow path to the first stream
// cell (src/D8HDistToStrm.cpp:57-226, src/D8VDistToStrm.cpp:58-240).
//
// The reference runs one FIFO queue that starts with the stream cells (src data and >= thresh); dequeuing a cell makes its
// upslope neighbours ready, so it is a breadth-first search from the stream, and a cell's value depends only on its receiver's
// final value.  Here that search runs one BFS level per launch:
//   k_dts_seed  : the value raster (MISSINGFLOAT, 0 on the stream cells), a code byte per cell (its D8 code where the cell is
//                 not a stream cell and the code is 1..8, else 0) and the stream cells appended to the frontier list.
//   k_dts_level : one lane per frontier cell of level t; each non-stream neighbour whose code points back at it gets its value
//                 (horizontal: dist[row][k] + d(n); vertical: (fel(c) - fel(n)) + d(n)) and joins level t + 1 unless the value
//                 tests as nodata.  A cell has one receiver, so one writer and no atomics on values; it enters the list once.
//   k_dts_edge  : on row strips, the owned edge-row cells whose receiver lies in a halo row that holds a value (the neighbour's
//                 rows after an exchange of the value raster's edge rows) get their values and join the frontier.
// Cells the search never reaches keep MISSINGFLOAT: paths that leave the grid, meet a non-stream cell with nodata p, code 0 or a
// code outside 1..8, or end in a cycle without a stream cell.  Pruning at values that test as nodata is exact: every cell above
// such a value would get exactly MISSINGFLOAT, which it holds already.
//
// The levels run in batches without a host round trip (flood.cuh, shared with dinfdistdown.cu): the level bounds live in device
// memory, the last block of level t records where level t + 1 ends, and the host reads a batch's bounds back once.
#include "common.cuh"
#include "ctx.h"
#include "flood.cuh"
#include "kernels.h"

namespace td {
namespace {
constexpr int TPB = 256;

// the value c gets from its receiver n (direction k, c's strip row r): float operations in the reference's order
template <bool V>
__device__ __forceinline__ float dts_value(const float* __restrict__ fel, const float* __restrict__ dist, long long c, long long n, int r, int k,
                                           float dn) {
  if (V) {
    const float a = fel[c], b = fel[n];
    const float t = dts_x86(__fsub_rn(a, b), a, b);
    return dts_x86(__fadd_rn(t, dn), t, dn);
  }
  const float w = dist[(size_t)(r - 1) * 8 + (k - 1)];
  return dts_x86(__fadd_rn(w, dn), w, dn);
}

__global__ void __launch_bounds__(TPB) k_dts_seed(const short* __restrict__ p, const int* __restrict__ src, float* __restrict__ val,
                                                  unsigned char* __restrict__ code, Strip s, int thresh, short p_nodata, int src_nodata,
                                                  unsigned* __restrict__ list, unsigned long long* __restrict__ ctr) {
  const long long o = (long long)blockIdx.x * TPB + threadIdx.x;
  const bool in = o < s.cells();
  const int r = in ? (int)(o / s.pitch) : 0, c = in ? (int)(o - (long long)r * s.pitch) : 0;
  bool stream = false;
  unsigned char k = 0;
  if (in && s.owned(r, c)) {
    const int sv = src[o];
    stream = sv != src_nodata && sv >= thresh;             // linearpart<int32_t>::isNodata is equality
    const short d = p[o];
    if (!stream && !nd_s(d, p_nodata) && d >= 1 && d <= 8) k = (unsigned char)d;
  }
  if (in) {
    val[o] = stream ? 0.0f : TD_MISSINGFLOAT;
    code[o] = k;
  }
  dts_append(list, ctr, stream, (unsigned)o);
}

// Level t: the frontier is list[bounds[t - 1], bounds[t]); the last block to finish records bounds[t + 1] = *ctr.
template <bool V>
__global__ void __launch_bounds__(TPB) k_dts_level(const unsigned* __restrict__ list_in, unsigned long long* __restrict__ bounds, int t,
                                                   const unsigned char* __restrict__ code, const float* __restrict__ fel,
                                                   const float* __restrict__ dist, float* __restrict__ val, Strip s, unsigned* __restrict__ list,
                                                   unsigned long long* __restrict__ ctr, unsigned* __restrict__ blkdone) {
  const unsigned long long lo = bounds[t - 1], hi = bounds[t];
  const unsigned long long n = hi - lo;
  for (unsigned long long base = (unsigned long long)blockIdx.x * TPB; base < n; base += (unsigned long long)gridDim.x * TPB) {
    const unsigned long long i = base + threadIdx.x;
    const bool in = i < n;
    const long long ni = in ? (long long)list_in[lo + i] : (long long)s.pitch;
    const int r = (int)(ni / s.pitch), col = (int)(ni - (long long)r * s.pitch);
    const float dn = in ? val[ni] : 0.0f;
#pragma unroll 1                                 // (unrolled, the vertical instance spills)
    for (int kk = 1; kk <= 8; ++kk) {            // direction from the frontier cell n to the candidate c
      bool push = false;
      const long long ci = ni + (long long)drow(kk) * s.pitch + dcol(kk);
      const int cc = col + dcol(kk);
      if (in && cc >= 0 && cc < s.nx) {          // (rows 0 and ny + 1 hold code 0: the neighbour strips own them)
        const int k = kk > 4 ? kk - 4 : kk + 4;  // the code of a c that drains to n
        if (code[ci] == k) {
          const float v = dts_value<V>(fel, dist, ci, ni, r + drow(kk), k, dn);
          val[ci] = v;
          push = !nd_f(v, TD_MISSINGFLOAT);
        }
      }
      dts_append(list, ctr, push, (unsigned)ci);
    }
  }
  flood_level_done(bounds, t, ctr, blkdone);
}

// blockIdx.y = 0: the first owned row, 1: the last (the same row of a one-row strip is taken once)
template <bool V>
__global__ void __launch_bounds__(TPB) k_dts_edge(const unsigned char* __restrict__ code, const float* __restrict__ fel,
                                                  const float* __restrict__ dist, float* __restrict__ val, Strip s, unsigned* __restrict__ list,
                                                  unsigned long long* __restrict__ ctr) {
  const int c = blockIdx.x * TPB + threadIdx.x;
  const int r = blockIdx.y == 0 ? 1 : s.ny;
  bool push = false;
  long long o = 0;
  if (c < s.nx && (blockIdx.y == 0 || s.ny > 1)) {
    o = s.idx(r, c);
    const int k = code[o];
    const int rr = r + drow(k), cn = c + dcol(k);
    if (k != 0 && (rr == 0 || rr == s.ny + 1) && s.on_grid(rr, cn) && nd_f(val[o], TD_MISSINGFLOAT)) {
      const long long ni = s.idx(rr, cn);
      const float dn = val[ni];
      if (!nd_f(dn, TD_MISSINGFLOAT)) {
        const float v = dts_value<V>(fel, dist, o, ni, r, k, dn);
        val[o] = v;
        push = !nd_f(v, TD_MISSINGFLOAT);
      }
    }
  }
  dts_append(list, ctr, push, (unsigned)o);
}
}  // namespace

int dts_seed(const short* p, const int* src, float* val, unsigned char* code, const Strip& s, int thresh, short p_nodata, int src_nodata,
             const DtsBufs& b, cudaStream_t st) {
  TD_CUDA(cudaMemsetAsync(b.ctr, 0, 2 * sizeof(unsigned long long), st));
  TD_CUDA(cudaMemsetAsync(b.blkdone, 0, sizeof(unsigned), st));
  const long long blocks = (s.cells() + TPB - 1) / TPB;
  k_dts_seed<<<(unsigned)blocks, TPB, 0, st>>>(p, src, val, code, s, thresh, p_nodata, src_nodata, b.list, b.ctr);
  TD_LAUNCHED();
  TD_CUDA(cudaGetLastError());
  return TD_OK;
}

int dts_levels(bool vertical, const unsigned char* code, const float* fel, const float* dist, float* val, const Strip& s, const DtsBufs& b, int grid,
               unsigned long long* cells, long long* levels, cudaStream_t st) {
  if (s.has_top || s.has_bot) {
    const dim3 eg((unsigned)((s.nx + TPB - 1) / TPB), 2);
    if (vertical) k_dts_edge<true><<<eg, TPB, 0, st>>>(code, fel, dist, val, s, b.list, b.ctr);
    else k_dts_edge<false><<<eg, TPB, 0, st>>>(code, fel, dist, val, s, b.list, b.ctr);
    TD_LAUNCHED();
    TD_CUDA(cudaGetLastError());
  }
  return flood_levels(b, [&](int t) {
    if (vertical) k_dts_level<true><<<grid, TPB, 0, st>>>(b.list, b.bounds, t, code, fel, dist, val, s, b.list, b.ctr, b.blkdone);
    else k_dts_level<false><<<grid, TPB, 0, st>>>(b.list, b.bounds, t, code, fel, dist, val, s, b.list, b.ctr, b.blkdone);
  }, cells, levels, st);
}

}  // namespace td
