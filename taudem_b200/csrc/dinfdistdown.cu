// dinfdistdown: the D-infinity distance from every cell down to the stream (src/DinfDistDown.cpp:95-1398), horizontal (h),
// vertical (v: the height above the nearest drainage), Pythagoras (p) or surface (s), as the average, maximum or minimum over the
// cell's (at most two) receivers.
//
// The reference runs Kahn's algorithm over the D-infinity receivers: a cell's counter holds its receivers that are on the grid and
// have data in ang, stream cells (src, read as int16, >= 1) are reset to 0, the cells at 0 start a FIFO queue, and a dequeued cell
// gets its value from its receivers' final values and then releases every donor whose prop() toward it is > 0.  A cell's value
// depends only on its receivers, so the result does not depend on the order within a level.  Here one launch runs one level:
//   k_ddd_seed  : the value raster(s) (MISSINGFLOAT), one state byte per cell (the receivers of dinf_receivers, the outstanding
//                 count, the stream bit) and the cells at 0 appended to the frontier list.
//   k_ddd_level : one lane per frontier cell: its value from its receivers (dinf_outflow's shares, in increasing direction: the
//                 wrap sector's pair is 8 and 1, and direction 1 comes first), written; then an atomic decrement of the count of
//                 every donor whose receiver byte points at it, and the lane that brings a count to 0 appends that donor.
//   k_ddd_edge  : on row strips, the decrements the neighbour strips sent for the owned edge rows (a level counts the decrements of
//                 donors in a halo row into halo_out instead), and the cells they release start the next levels.
//   k_ddd_pyth  : p mode, after the last level: sqrt(h * h + v * v) where both values are data, nodata where v is.
// Nodata does not prune: a cell whose receivers are all nodata still releases its donors, which then become nodata (or not, under
// -nc), exactly as in the reference.  Cells on a cycle of angles and everything upslope of one are never dequeued and keep
// MISSINGFLOAT.  The batched level loop is flood.cuh's, shared with the D8 distance tools.
//
// The algebra holds the reference's types and order: p double, distr / sump float, each accumulation (float)((double)distr +
// p * (double)x), products and sums unfused (-fmad=false) and NaNs carried with x86's bits (dts_x86).
#include "common.cuh"
#include "ctx.h"
#include "dinf_common.cuh"
#include "flood.cuh"
#include "kernels.h"

namespace td {
namespace {
constexpr int TPB = 256;
// state byte: bits 0-3 the first receiver k1 (0: none), 0x10 a second receiver (k1 % 8 + 1), bits 5-6 the receivers not yet
// evaluated, 0x80 a stream cell (its count is 0 from the start and it is never released again)
constexpr unsigned ST_CNT = 5, ST_STREAM = 0x80u;

__device__ __forceinline__ bool sends_to(unsigned b, int k) {
  const int k1 = (int)(b & 15u);
  return k1 != 0 && (k1 == k || ((b & 0x10u) && (k1 & 7) + 1 == k));
}

// d decrements of the count of cell o; true where they bring it to 0
__device__ __forceinline__ bool release(unsigned char* state, long long o, unsigned d) {
  const unsigned sh = 8u * (unsigned)(o & 3) + ST_CNT;
  unsigned* word = reinterpret_cast<unsigned*>(state + (o & ~3ll));
  return ((atomicSub(word, d << sh) >> sh) & 3u) == d;
}

// float and double operations with x86's NaN results
__device__ __forceinline__ float f_add(float a, float b) { return dts_x86(__fadd_rn(a, b), a, b); }
__device__ __forceinline__ float f_sub(float a, float b) { return dts_x86(__fsub_rn(a, b), a, b); }
__device__ __forceinline__ float f_mul(float a, float b) { return dts_x86(__fmul_rn(a, b), a, b); }
__device__ __forceinline__ float f_div(float a, float b) { return dts_x86(__fdiv_rn(a, b), a, b); }
__device__ __forceinline__ float f_sqrt(float a) { return dts_x86(__fsqrt_rn(a), a, a); }
// (float)((double)d + p * (double)x): p is a share >= 1e-5, so the product is NaN only where x is, and carries x's bits
__device__ __forceinline__ float f_acc(float d, double p, float x) {
  return dts_x86(__double2float_rn(__dadd_rn((double)d, __dmul_rn(p, (double)x))), d, x);
}

__global__ void __launch_bounds__(TPB) k_ddd_seed(const float* __restrict__ ang, const short* __restrict__ src, DddArgs A, Strip s,
                                                  float ang_nodata, unsigned* __restrict__ list, unsigned long long* __restrict__ ctr) {
  const long long o = (long long)blockIdx.x * TPB + threadIdx.x;
  const bool in = o < s.cells();
  const int r = in ? (int)(o / s.pitch) : 0, c = in ? (int)(o - (long long)r * s.pitch) : 0;
  bool push = false;
  unsigned b = 0;
  if (in && s.on_grid(r, c)) {
    const float a = ang[o];
    if (!nd_f(a, ang_nodata)) {
      const unsigned rc = dinf_receivers(a, ArefRow{theta_of_row(A.theta, s.ny, r)});
      if (!s.owned(r, c)) b = rc;                           // a halo-row cell: only its receivers (the donors of the owned rows)
      else {
        unsigned n = 0;
        const int k1 = (int)(rc & 15u), k2 = (rc & 0x10u) ? (k1 & 7) + 1 : 0;
        for (int k : {k1, k2}) {
          if (k == 0) continue;
          const int rr = r + drow(k), cc = c + dcol(k);
          if (s.on_grid(rr, cc) && !nd_f(ang[s.idx(rr, cc)], ang_nodata)) ++n;
        }
        if (src[o] >= 1) b = rc | ST_STREAM;               // src/DinfDistDown.cpp:223-224: no threshold, src's nodata not tested
        else b = rc | (n << ST_CNT);
        push = (b & (3u << ST_CNT)) == 0;
      }
    }
  }
  if (in) {
    A.val[o] = TD_MISSINGFLOAT;
    if (A.val2) A.val2[o] = TD_MISSINGFLOAT;
    A.state[o] = (unsigned char)b;
  }
  dts_append(list, ctr, push, (unsigned)o);
}

// the value(s) of a dequeued cell o (strip row r, column col): src/DinfDistDown.cpp:254-308 (h), 541-606 (v), 874-961 (p),
// 1240-1320 (s).  M: 0 h, 1 v, 2 p, 3 s; S: 0 ave, 1 max, 2 min.
template <int M, int S>
__device__ __forceinline__ void ddd_eval(const DddArgs& A, const Strip& s, long long o, int r, int col, float& h, float& v) {
  h = v = TD_MISSINGFLOAT;
  if (A.state[o] & ST_STREAM) { h = v = 0.0f; return; }
  float elv = 0.0f;
  if (M != 0) {
    elv = A.fel[o];
    if (nd_f(elv, A.fel_nodata)) return;
  }
  const Outflow of = dinf_outflow(A.ang[o], theta_of_row(A.theta, s.ny, r));
  const bool wrap = of.k2 != 0 && of.k2 < of.k1;          // the wrap sector: 8 then 1 from the search, 1 first in the reference's loop
  float dh = 0.0f, dv = 0.0f, sump = 0.0f;
  bool first = true, con = false;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int k = (i == 0) == wrap ? of.k2 : of.k1;
    const double p = (i == 0) == wrap ? of.p2 : of.p1;
    if (k == 0) continue;
    const int rr = r + drow(k), cc = col + dcol(k);
    if (!s.on_grid(rr, cc)) { con = true; continue; }
    const long long n = s.idx(rr, cc);
    const float dn = A.val[n];
    if (nd_f(dn, TD_MISSINGFLOAT)) { con = true; continue; }
    float elvn = 0.0f;
    if (M != 0) {
      elvn = A.fel[n];
      if (nd_f(elvn, A.fel_nodata)) { con = true; continue; }
    }
    sump = __double2float_rn(__dadd_rn((double)sump, p));
    float wt = 1.0f;
    if (M != 1 && A.w) {                                   // the weight of the receiver; a nodata weight still counts as 1
      const float wv = A.w[n];
      if (nd_f(wv, A.w_nodata)) con = true;
      else wt = wv;
    }
    const float dk = M == 1 ? 0.0f : A.dist[(size_t)(r - 1) * 8 + (k - 1)];
    float xh, xv = 0.0f;
    if (M == 0) xh = f_add(f_mul(dk, wt), dn);
    else if (M == 1) xh = f_add(f_sub(elv, elvn), dn);
    else if (M == 2) {
      xh = f_add(f_mul(dk, wt), dn);
      xv = f_add(f_sub(elv, elvn), A.val2[n]);
    } else {
      const float e = f_sub(elv, elvn), dw = f_mul(dk, wt);
      xh = f_add(f_sqrt(f_add(f_mul(e, e), f_mul(dw, dw))), dn);
    }
    if (S == 0) {
      dh = f_acc(dh, p, xh);
      if (M == 2) dv = f_acc(dv, p, xv);
    } else if (S == 1 && M == 0) {                         // h max starts from 0 without `first`
      if (xh > dh) dh = xh;
    } else if (first) {
      dh = xh;
      dv = xv;
      first = false;
    } else if (S == 1) {
      if (xh > dh) dh = xh;
      if (M == 2 && xv > dv) dv = xv;
    } else {
      if (xh < dh) dh = xh;
      if (M == 2 && xv < dv) dv = xv;
    }
  }
  if ((con && A.concheck) || sump <= 0.0f) return;
  h = S == 0 ? f_div(dh, sump) : dh;
  if (M == 2) v = S == 0 ? f_div(dv, sump) : dv;
}

// Level t: the frontier is list[bounds[t - 1], bounds[t]); the last block to finish records bounds[t + 1] = *ctr.
template <int M, int S>
__global__ void __launch_bounds__(TPB) k_ddd_level(const unsigned* __restrict__ list_in, unsigned long long* __restrict__ bounds, int t, DddArgs A,
                                                   Strip s, unsigned* __restrict__ list, unsigned long long* __restrict__ ctr,
                                                   unsigned* __restrict__ blkdone) {
  const unsigned long long lo = bounds[t - 1], hi = bounds[t];
  const unsigned long long n = hi - lo;
  for (unsigned long long base = (unsigned long long)blockIdx.x * TPB; base < n; base += (unsigned long long)gridDim.x * TPB) {
    const unsigned long long i = base + threadIdx.x;
    const bool in = i < n;
    const long long ci = in ? (long long)list_in[lo + i] : (long long)s.pitch;
    const int r = (int)(ci / s.pitch), col = (int)(ci - (long long)r * s.pitch);
    if (in) {
      float h, v;
      ddd_eval<M, S>(A, s, ci, r, col, h, v);
      A.val[ci] = h;
      if (M == 2) A.val2[ci] = v;
    }
#pragma unroll 1
    for (int kk = 1; kk <= 8; ++kk) {                     // direction from the evaluated cell to the donor candidate d
      bool push = false;
      const long long di = ci + (long long)drow(kk) * s.pitch + dcol(kk);
      const int dr = r + drow(kk), dc = col + dcol(kk);
      if (in && s.on_grid(dr, dc)) {
        const unsigned b = A.state[di];
        if (!(b & ST_STREAM) && sends_to(b, kk > 4 ? kk - 4 : kk + 4)) {
          if (dr >= 1 && dr <= s.ny) push = release(A.state, di, 1u);
          else atomicAdd(A.halo_out + (dr == 0 ? 0 : s.pitch) + dc, 1);     // a donor in the neighbour strip: its decrement travels
        }
      }
      dts_append(list, ctr, push, (unsigned)di);
    }
  }
  flood_level_done(bounds, t, ctr, blkdone);
}

// The decrements a row strip received from its neighbours (dec_top: for its first owned row, from the strip above; dec_bot: for its last,
// from the strip below; NULL where there is no neighbour): the cells they release start the next levels.  blockIdx.y = 0: the first
// owned row (both arrays on a one-row strip), 1: the last.
__global__ void __launch_bounds__(TPB) k_ddd_edge(unsigned char* __restrict__ state, const int* __restrict__ dec_top, const int* __restrict__ dec_bot,
                                                  Strip s, unsigned* __restrict__ list, unsigned long long* __restrict__ ctr) {
  const int c = blockIdx.x * TPB + threadIdx.x;
  bool push = false;
  long long o = 0;
  if (c < s.nx && (blockIdx.y == 0 || s.ny > 1)) {
    const int r = blockIdx.y == 0 ? 1 : s.ny;
    int d = 0;
    if (r == 1 && dec_top) d += dec_top[c];
    if (r == s.ny && dec_bot) d += dec_bot[c];
    o = s.idx(r, c);
    if (d > 0 && !(state[o] & ST_STREAM)) push = release(state, o, (unsigned)d);   // (stream cells only ever go below 0)
  }
  dts_append(list, ctr, push, (unsigned)o);
}

// src/DinfDistDown.cpp:1014-1025
__global__ void __launch_bounds__(TPB) k_ddd_pyth(float* __restrict__ h, const float* __restrict__ v, Strip s) {
  const long long o = (long long)blockIdx.x * TPB + threadIdx.x;
  if (o >= s.cells()) return;
  const int r = (int)(o / s.pitch), c = (int)(o - (long long)r * s.pitch);
  if (!s.owned(r, c)) return;
  const float vv = v[o], hh = h[o];
  if (nd_f(vv, TD_MISSINGFLOAT)) h[o] = TD_MISSINGFLOAT;
  else if (!nd_f(hh, TD_MISSINGFLOAT)) h[o] = f_sqrt(f_add(f_mul(hh, hh), f_mul(vv, vv)));
}

using LevelKernel = void (*)(const unsigned*, unsigned long long*, int, DddArgs, Strip, unsigned*, unsigned long long*, unsigned*);
template <int M>
constexpr LevelKernel K3[3] = {k_ddd_level<M, 0>, k_ddd_level<M, 1>, k_ddd_level<M, 2>};
constexpr const LevelKernel* LEVEL[4] = {K3<0>, K3<1>, K3<2>, K3<3>};
}  // namespace

int ddd_seed(const float* ang, const short* src, float ang_nodata, const DddArgs& A, const Strip& s, const DtsBufs& b, cudaStream_t st) {
  TD_CUDA(cudaMemsetAsync(b.ctr, 0, 2 * sizeof(unsigned long long), st));
  TD_CUDA(cudaMemsetAsync(b.blkdone, 0, sizeof(unsigned), st));
  const long long blocks = (s.cells() + TPB - 1) / TPB;
  k_ddd_seed<<<(unsigned)blocks, TPB, 0, st>>>(ang, src, A, s, ang_nodata, b.list, b.ctr);
  TD_LAUNCHED();
  TD_CUDA(cudaGetLastError());
  return TD_OK;
}

int ddd_levels(int mode, int stat, const DddArgs& A, const Strip& s, const DtsBufs& b, int grid, unsigned long long* cells, long long* levels,
               cudaStream_t st) {
  const LevelKernel k_level = LEVEL[mode][stat];
  return flood_levels(b, [&](int t) { k_level<<<grid, TPB, 0, st>>>(b.list, b.bounds, t, A, s, b.list, b.ctr, b.blkdone); }, cells, levels, st);
}

int ddd_edge(unsigned char* state, const int* dec_top, const int* dec_bot, const Strip& s, const DtsBufs& b, cudaStream_t st) {
  const dim3 eg((unsigned)((s.nx + TPB - 1) / TPB), 2);
  k_ddd_edge<<<eg, TPB, 0, st>>>(state, dec_top, dec_bot, s, b.list, b.ctr);
  TD_LAUNCHED();
  TD_CUDA(cudaGetLastError());
  return TD_OK;
}

int ddd_pythagoras(float* h, const float* v, const Strip& s, cudaStream_t st) {
  const long long blocks = (s.cells() + TPB - 1) / TPB;
  k_ddd_pyth<<<(unsigned)blocks, TPB, 0, st>>>(h, v, s);
  TD_LAUNCHED();
  TD_CUDA(cudaGetLastError());
  return TD_OK;
}

}  // namespace td
