// D8 steepest-descent stencil: setPosDir + setFlow + calcSlope fused
// (reference src/d8.cpp:359-409, 103-150, 153-177).
//
//  * a cell on the global grid edge, a nodata cell, or a cell with any nodata
//    8-neighbour gets dir = -32768 and slope = -1;
//  * otherwise k is scanned in the order 1,3,5,7,2,4,6,8 with a strict '>' on
//    slope_k = (float)(fact[j][k] * (double)(float)(z0 - zk)); dir 0 = flat;
//  * slope = slope of the chosen direction, 0 on flats.
// The reference's dontCross / "neighbour points back" tests cannot fire in this
// pass (a strict steepest descent never crosses or faces another one), so the
// pass is a pure 3x3 stencil (SURVEY.md A.2).
//
// HBM traffic per cell: read fel 4 B, write p 2 B + sd8 4 B = 10 B (algorithmic).
// Tile: 32 rows x 128 columns per CTA, staged through shared memory by 1-D TMA
// bulk copies (34 row copies of 544 B), each thread produces 4 adjacent cells of
// one row and stores them as one short4 + one float4.
#include "kernels.h"
#include "rowfact.cuh"
#include "tile_pipe.cuh"

namespace td {

namespace {
constexpr int TW = 128, TH = 32;

__device__ __forceinline__ void d8_try(float z, float zn, double f, int k, float& smax, int& dir) {
  const float diff = z - zn;
  const float sl = (float)(f * (double)diff);
  if (sl > smax) { smax = sl; dir = k; }
}

// Literal reference order with all eight products (rare path, out of line; q = centre cell in the staged tile)
__device__ __noinline__ void d8_literal(const float* q, int sw, double fE, double fN, double fD, int* dir, float* smax) {
  const float z = q[0];
  int d = 0; float sm = 0.f;
  d8_try(z, q[1], fE, 1, sm, d); d8_try(z, q[-sw], fN, 3, sm, d);
  d8_try(z, q[-1], fE, 5, sm, d); d8_try(z, q[sw], fN, 7, sm, d);
  d8_try(z, q[-sw + 1], fD, 2, sm, d); d8_try(z, q[-sw - 1], fD, 4, sm, d);
  d8_try(z, q[sw - 1], fD, 6, sm, d); d8_try(z, q[sw + 1], fD, 8, sm, d);
  *dir = d; *smax = sm;
}

// Selection rule of one cell.
// The reference scans k = 1,3,5,7,2,4,6,8 and keeps the first k with the strictly largest
// slope_k = (float)(fact_k * (double)(z - z_k)).  fact takes only three values per row (E/W, N/S,
// diagonals) and the rounding is monotone in the elevation drop, so the maximum of each group is
// attained by the group's largest drop: three exact products instead of eight.  Within a group the
// winner is the first member (scan order) whose slope equals the group's: a drop more than 2^-20
// (relative) below the largest one cannot round to the same slope, so the candidate is the first
// member inside that band; if it is not the largest drop itself the cell is ambiguous (two nearly equal
// drops, rare) and takes the literal eight-product path.  A group whose largest drop is <= 0 has no
// member inside the band and can never win (S > 0 is required), so it never raises the flag.
// The band argument holds while S and the largest drop of every group that attains it are normal floats (a drop
// 2^-20 lower then lies at least 7 ulps lower, and m * (1 - 2^-20) is computed to 2^-24).  smin = 2^-125 max(1, fE, fN)
// (the row's) makes S >= smin imply both; a cell whose S is below smin (subnormal drops or slopes) or infinite (the
// product overflows float: every overflowing drop rounds to the same slope) takes the literal path, as do ambiguous ones.
// One cell from its eight drops e_k = z - z_k.
__device__ __forceinline__ bool d8_pick(float e1, float e2, float e3, float e4, float e5, float e6, float e7, float e8, double fE, double fN,
                                        double fD, float smin, int& dir, float& smax) {
  const float m15 = fmaxf(e1, e5), m37 = fmaxf(e3, e7), mD = fmaxf(fmaxf(e2, e4), fmaxf(e6, e8));
  const float sE = (float)(fE * (double)m15), sN = (float)(fN * (double)m37), sD = (float)(fD * (double)mD);
  const float S = fmaxf(fmaxf(sE, sN), sD);
  const float c = 0.99999905f;                       // 1 - 2^-20
  const float tE = m15 * c, tN = m37 * c, tD = mD * c;
  // candidates coded as (scan position << 4) | k so that an integer minimum picks the earliest one
  const bool in1 = e1 > tE, in3 = e3 > tN, in2 = e2 > tD, in4 = e4 > tD, in6 = e6 > tD;
  int cE = in1 ? 0x01 : 0x25;
  int cN = in3 ? 0x13 : 0x37;
  int cD = in2 ? 0x42 : (in4 ? 0x54 : (in6 ? 0x66 : 0x78));
  const float eD = in2 ? e2 : (in4 ? e4 : (in6 ? e6 : mD));
  const bool amb = (in1 & (e1 < m15)) | (in3 & (e3 < m37)) | (eD < mD);
  cE = (sE == S) ? cE : 0xff; cN = (sN == S) ? cN : 0xff; cD = (sD == S) ? cD : 0xff;
  const int best = min(cE, min(cN, cD));
  const bool pos = S > 0.f;
  dir = pos ? (best & 15) : 0;
  smax = pos ? S : 0.f;
  const bool normal = (S >= smin) & (S <= FLT_MAX);
  return (amb | !normal) & pos;
}

constexpr int STAGES = 3;
using Ring = TileRing<float, TW, TH, STAGES>;

// Persistent CTAs, 2-D TMA tiles through a three-stage ring (tile_pipe.cuh).  A warp handles four consecutive rows of
// the 32 x 128 tile, a lane four adjacent cells of each; the window slides down the rows in registers (one float4 + two
// scalar shared-memory loads per new row) and every elevation difference is computed once and used by both cells it
// separates (z_a - z_b = -(z_b - z_a) exactly): 19 subtractions per four cells instead of 32.
__global__ void __launch_bounds__(256) k_d8_stencil(const TD_GRID_CONSTANT TileMap tm, short* __restrict__ dir, float* __restrict__ slope,
                                                    const RowFact* __restrict__ rowf, Strip s, float nodata,
                                                    unsigned long long* __restrict__ nflat) {
  extern __shared__ __align__(128) unsigned char dsm128[];
  using G = Ring::G;
  constexpr int RPW = TH / 8;                     // rows per warp
  Ring ring;
  ring.init(dsm128, &tm, s);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned myflat = 0;
  for (long long t = blockIdx.x; t < ring.ntiles; t += gridDim.x) {
    int r0, c0;
    const float* tile = ring.acquire(t, r0, c0);
    const int c = c0 + lane * 4;
    const int tr0 = warp * RPW;
    if (r0 + tr0 <= s.ny && c < s.pitch) {
      const float* pm = tile + tr0 * G::SW + G::HP + lane * 4;   // row above the first row, column c
      float ra[6], rb[6], rc[6];                    // rows above / at / below the current row, columns c-1 .. c+4
      float na[6], nbv[6], nc[6];                   // |value - nodata| of the same
      auto load_row = [&](const float* p, float (&v)[6], float (&d)[6]) {
        const float4 q = *reinterpret_cast<const float4*>(p);
        v[0] = p[-1]; v[1] = q.x; v[2] = q.y; v[3] = q.z; v[4] = q.w; v[5] = p[4];
#pragma unroll
        for (int i = 0; i < 6; ++i) d[i] = fabsf(v[i] - nodata);
      };
      load_row(pm, ra, na);
      load_row(pm + G::SW, rb, nbv);
      // differences with the row above (the previous row's "down" differences, negated)
      float pv[4], pg[5], pf[5];                    // a[j+1]-b[j+1], a[j]-b[j+1], a[j+1]-b[j]
#pragma unroll
      for (int j = 0; j < 4; ++j) pv[j] = ra[j + 1] - rb[j + 1];
#pragma unroll
      for (int j = 0; j < 5; ++j) { pg[j] = ra[j] - rb[j + 1]; pf[j] = ra[j + 1] - rb[j]; }
      // cells on the edge of the whole grid or beyond the last column, as a 4-bit mask for this thread's cells
      unsigned emc = (c == 0) ? 1u : 0u;
      const int klast = s.nx - 1 - c;
      if (klast < 4) emc |= (0xfu << max(klast, 0)) & 0xfu;
#pragma unroll
      for (int k = 0; k < RPW; ++k) {
        const int r = r0 + tr0 + k;
        if (r > s.ny) break;
        load_row(pm + (k + 2) * G::SW, rc, nc);
        const RowFact* rf = rowf + (r - 1);
        const double fE = rf->fE, fN = rf->fN, fD = rf->fD;
        const float smin = 0x1p-125f * fmaxf(1.f, (float)fmax(fE, fN));     // d8_pick: the band argument holds for S >= smin
        float h[5], v[4], g[5], f[5];               // b[j]-b[j+1], b[j+1]-c[j+1], b[j]-c[j+1], b[j+1]-c[j]
#pragma unroll
        for (int j = 0; j < 5; ++j) { h[j] = rb[j] - rb[j + 1]; g[j] = rb[j] - rc[j + 1]; f[j] = rb[j + 1] - rc[j]; }
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = rb[j + 1] - rc[j + 1];
        float colmin[6];
#pragma unroll
        for (int i = 0; i < 6; ++i) colmin[i] = fminf(fminf(na[i], nbv[i]), nc[i]);
        const unsigned em = emc | (((r == 1 && !s.has_top) || (r == s.ny && !s.has_bot)) ? 0xfu : 0u);
        short od[4]; float os[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const bool bad = (fminf(fminf(colmin[i], colmin[i + 1]), colmin[i + 2]) < TD_MINEPS) || ((em >> i) & 1u);
          int d; float smax;
          // e1 = z - E, e2 = z - NE, e3 = z - N, e4 = z - NW, e5 = z - W, e6 = z - SW, e7 = z - S, e8 = z - SE
          if (d8_pick(h[i + 1], -pf[i + 1], -pv[i], -pg[i], -h[i], f[i], v[i], g[i + 1], fE, fN, fD, smin, d, smax))
            d8_literal(pm + (k + 1) * G::SW + i, G::SW, fE, fN, fD, &d, &smax);
          od[i] = bad ? TD_MISSINGSHORT : (short)d;
          os[i] = bad ? -1.0f : smax;
          if (!bad && d == 0) ++myflat;
        }
        const long long o = s.idx(r, c);
        *reinterpret_cast<short4*>(dir + o) = make_short4(od[0], od[1], od[2], od[3]);
        *reinterpret_cast<float4*>(slope + o) = make_float4(os[0], os[1], os[2], os[3]);
        // slide the window down one row
#pragma unroll
        for (int j = 0; j < 6; ++j) { ra[j] = rb[j]; rb[j] = rc[j]; na[j] = nbv[j]; nbv[j] = nc[j]; }
#pragma unroll
        for (int j = 0; j < 4; ++j) pv[j] = v[j];
#pragma unroll
        for (int j = 0; j < 5; ++j) { pg[j] = g[j]; pf[j] = f[j]; }
      }
    }
    ring.release(&tm, t);
  }
  // flat count: warp reduce, then one atomic per CTA
  __shared__ unsigned wflat[8];
  for (int o = 16; o; o >>= 1) myflat += __shfl_xor_sync(0xffffffffu, myflat, o);
  if (lane == 0) wflat[warp] = myflat;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned tt = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) tt += wflat[i];
    if (tt) atomicAdd(nflat, (unsigned long long)tt);
  }
}
}  // namespace

int launch_d8_stencil(const float* elev, short* dir, float* slope, const RowFact* rowf, const Strip& s, float nodata,
                      unsigned long long* nflat, cudaStream_t st) {
  TileMap tm;
  if (int rc = make_tile_map(&tm, elev, 4, s.pitch, s.ny + 2, Ring::G::SW, Ring::G::ROWS)) return rc;
  const long long ntiles = (long long)((s.pitch + TW - 1) / TW) * ((s.ny + TH - 1) / TH);
  int grid = 0;
  if (int rc = stencil_grid((const void*)k_d8_stencil, 256, Ring::SMEM, ntiles, &grid)) return rc;
  k_d8_stencil<<<grid, 256, Ring::SMEM, st>>>(tm, dir, slope, rowf, s, nodata, nflat);
  TD_LAUNCHED();
  TD_CUDA(cudaGetLastError());
  return TD_OK;
}

}  // namespace td
