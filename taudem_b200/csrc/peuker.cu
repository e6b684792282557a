// Peuker-Douglas stream sources (src/PeukerDouglas.cpp:109-212) as two 3x3 stencils on the tile ring (tile_pipe.cuh):
//
//  k_pd_smooth  fel -> s   a cell on the first / last row or column of the whole grid, or a nodata cell, keeps s = fel; every
//                          other cell gets the float average acc / w, acc = w_mid * e, w = w_mid, then for each side neighbour
//                          (k = 1,3,5,7) that is not nodata acc += e_k * w_side, w += w_side (when w_side > 0), then the same for
//                          the diagonals (k = 2,4,6,8) with w_diag (when w_diag > 0).  Float arithmetic in exactly this order
//                          (-fmad=false); the nodata tests look at the raw elevations.
//  k_pd_mark    s -> ss    the reference visits every group of four cells (quad, origin (x, y), x in [0, nx-2], y in [-1, ny-1]),
//                          takes emax = s(origin) (the origin is not tested for nodata), then visits (x+1,y), (x,y+1), (x+1,y+1):
//                          a nodata cell marks the quad as bound, a larger one becomes the maximum; it unflags the maximum, and
//                          then all four cells of a bound quad or the cells equal to emax of the others.  Here each cell gathers
//                          its four quads instead (no write conflicts, no atomics): ss = 1 when the smoothing pass flagged it (not
//                          on the grid's edge, not nodata) and none of its quads unflags it.  An interior cell's quads lie inside
//                          the grid, so the rows beyond it (nodata in the reference) are never needed.
//
// A cell whose s is nodata was flagged 0 by the first pass: its fel was nodata (s = fel), or its smoothed value landed within
// 1e-5 of the nodata value — then it is a non-origin member of one of its quads, which is bound and unflags it.  So the first
// pass's flag is recomputed from s and no flag raster is kept between the passes.
//
// Two passes because a strip's first / last row needs the neighbour strip's SMOOTHED edge row in pass 2 (one halo row per
// strip): on row strips the caller exchanges s's edge rows in between, like the reference's second share().  At a strip edge
// without a neighbour (has_top / has_bot == 0) the missing row is the grid's edge and the halo row is never read.
//
// HBM traffic per cell: smooth 4 B in + 4 B out, mark 4 B in + 2 B out = 14 B (the minimum of the tool is 6 B: fel in, ss out).
// Tile: 32 rows x 128 columns per CTA, a warp takes four rows, a lane four adjacent cells of each.
#include "kernels.h"
#include "tile_pipe.cuh"

namespace td {

namespace {
constexpr int TW = 128, TH = 32, STAGES = 3;
using Ring = TileRing<float, TW, TH, STAGES>;

// columns c-1 .. c+4 of one staged row (p = column c)
__device__ __forceinline__ void pd_row(const float* p, float (&v)[6]) {
  const float4 q = *reinterpret_cast<const float4*>(p);
  v[0] = p[-1]; v[1] = q.x; v[2] = q.y; v[3] = q.z; v[4] = q.w; v[5] = p[4];
}

// the four cells of row r, columns c .. c+3, that are on the edge of the whole grid (or beyond its last column), as a 4-bit mask
__device__ __forceinline__ unsigned pd_edge(const Strip& s, int r, int c) {
  unsigned em = (c == 0) ? 1u : 0u;
  const int klast = s.nx - 1 - c;
  if (klast < 4) em |= (0xfu << max(klast, 0)) & 0xfu;
  if ((r == 1 && !s.has_top) || (r == s.ny && !s.has_bot)) em = 0xfu;
  return em;
}

__global__ void __launch_bounds__(256) k_pd_smooth(const TD_GRID_CONSTANT TileMap tm, float* __restrict__ sm, Strip s, float nodata, float wm,
                                                   float ws, float wd) {
  extern __shared__ __align__(128) unsigned char dsm128[];
  using G = Ring::G;
  constexpr int RPW = TH / 8;
  Ring ring;
  ring.init(dsm128, &tm, s);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long t = blockIdx.x; t < ring.ntiles; t += gridDim.x) {
    int r0, c0;
    const float* tile = ring.acquire(t, r0, c0);
    const int c = c0 + lane * 4, tr0 = warp * RPW;
    if (c < s.pitch) {
      for (int k = 0; k < RPW; ++k) {
        const int r = r0 + tr0 + k;
        if (r > s.ny) break;
        const float* pm = tile + (tr0 + k + 1) * G::SW + G::HP + lane * 4;   // row r, column c
        float a[6], b[6], d[6];                                               // rows r-1, r, r+1; columns c-1 .. c+4
        pd_row(pm - G::SW, a); pd_row(pm, b); pd_row(pm + G::SW, d);
        const unsigned em = pd_edge(s, r, c);
        float out[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float e = b[i + 1];
          if (((em >> i) & 1u) || nd_f(e, nodata)) { out[i] = e; continue; }
          float acc = wm * e, w = wm;
          if (ws > 0.f) {
            // k = 1 (E), 3 (N), 5 (W), 7 (S)
            if (!nd_f(b[i + 2], nodata)) { acc += b[i + 2] * ws; w += ws; }
            if (!nd_f(a[i + 1], nodata)) { acc += a[i + 1] * ws; w += ws; }
            if (!nd_f(b[i], nodata)) { acc += b[i] * ws; w += ws; }
            if (!nd_f(d[i + 1], nodata)) { acc += d[i + 1] * ws; w += ws; }
          }
          if (wd > 0.f) {
            // k = 2 (NE), 4 (NW), 6 (SW), 8 (SE)
            if (!nd_f(a[i + 2], nodata)) { acc += a[i + 2] * wd; w += wd; }
            if (!nd_f(a[i], nodata)) { acc += a[i] * wd; w += wd; }
            if (!nd_f(d[i], nodata)) { acc += d[i] * wd; w += wd; }
            if (!nd_f(d[i + 2], nodata)) { acc += d[i + 2] * wd; w += wd; }
          }
          out[i] = acc / w;
        }
        *reinterpret_cast<float4*>(sm + s.idx(r, c)) = make_float4(out[0], out[1], out[2], out[3]);
      }
    }
    ring.release(&tm, t);
  }
}

// one quad in the reference's visiting order: q0 = origin (x, y), q1 = (x+1, y), q2 = (x, y+1), q3 = (x+1, y+1); whether it
// unflags its member `me` (value v)
__device__ __forceinline__ bool pd_quad_unflags(float q0, float q1, float q2, float q3, int me, float v, float nodata) {
  float emax = q0;
  int am = 0;
  bool bound = false;
  if (nd_f(q1, nodata)) bound = true; else if (q1 > emax) { emax = q1; am = 1; }
  if (nd_f(q2, nodata)) bound = true; else if (q2 > emax) { emax = q2; am = 2; }
  if (nd_f(q3, nodata)) bound = true; else if (q3 > emax) { emax = q3; am = 3; }
  return bound || am == me || v == emax;
}

__global__ void __launch_bounds__(256) k_pd_mark(const TD_GRID_CONSTANT TileMap tm, short* __restrict__ ss, Strip s, float nodata) {
  extern __shared__ __align__(128) unsigned char dsm128[];
  using G = Ring::G;
  constexpr int RPW = TH / 8;
  Ring ring;
  ring.init(dsm128, &tm, s);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long t = blockIdx.x; t < ring.ntiles; t += gridDim.x) {
    int r0, c0;
    const float* tile = ring.acquire(t, r0, c0);
    const int c = c0 + lane * 4, tr0 = warp * RPW;
    if (c < s.pitch) {
      for (int k = 0; k < RPW; ++k) {
        const int r = r0 + tr0 + k;
        if (r > s.ny) break;
        const float* pm = tile + (tr0 + k + 1) * G::SW + G::HP + lane * 4;
        float a[6], b[6], d[6];
        pd_row(pm - G::SW, a); pd_row(pm, b); pd_row(pm + G::SW, d);
        const unsigned em = pd_edge(s, r, c);
        short out[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float v = b[i + 1];
          bool flag = !((em >> i) & 1u) && !nd_f(v, nodata);
          // quads with origin NW, N, W and the cell itself; the cell is member 3, 2, 1 and 0 of them
          flag = flag && !pd_quad_unflags(a[i], a[i + 1], b[i], b[i + 1], 3, v, nodata);
          flag = flag && !pd_quad_unflags(a[i + 1], a[i + 2], b[i + 1], b[i + 2], 2, v, nodata);
          flag = flag && !pd_quad_unflags(b[i], b[i + 1], d[i], d[i + 1], 1, v, nodata);
          flag = flag && !pd_quad_unflags(b[i + 1], b[i + 2], d[i + 1], d[i + 2], 0, v, nodata);
          out[i] = flag ? 1 : 0;
        }
        *reinterpret_cast<short4*>(ss + s.idx(r, c)) = make_short4(out[0], out[1], out[2], out[3]);
      }
    }
    ring.release(&tm, t);
  }
}
}  // namespace

int launch_pd_smooth(const float* fel, float* sm, const Strip& s, float nodata, const float* p, cudaStream_t st) {
  TileMap tm;
  if (int rc = make_tile_map(&tm, fel, 4, s.pitch, s.ny + 2, Ring::G::SW, Ring::G::ROWS)) return rc;
  const long long ntiles = (long long)((s.pitch + TW - 1) / TW) * ((s.ny + TH - 1) / TH);
  int grid = 0;
  if (int rc = stencil_grid((const void*)k_pd_smooth, 256, Ring::SMEM, ntiles, &grid)) return rc;
  k_pd_smooth<<<grid, 256, Ring::SMEM, st>>>(tm, sm, s, nodata, p[0], p[1], p[2]);
  TD_LAUNCHED();
  TD_CUDA(cudaGetLastError());
  return TD_OK;
}

int launch_pd_mark(const float* sm, short* ss, const Strip& s, float nodata, cudaStream_t st) {
  TileMap tm;
  if (int rc = make_tile_map(&tm, sm, 4, s.pitch, s.ny + 2, Ring::G::SW, Ring::G::ROWS)) return rc;
  const long long ntiles = (long long)((s.pitch + TW - 1) / TW) * ((s.ny + TH - 1) / TH);
  int grid = 0;
  if (int rc = stencil_grid((const void*)k_pd_mark, 256, Ring::SMEM, ntiles, &grid)) return rc;
  k_pd_mark<<<grid, 256, Ring::SMEM, st>>>(tm, ss, s, nodata);
  TD_LAUNCHED();
  TD_CUDA(cudaGetLastError());
  return TD_OK;
}

}  // namespace td
