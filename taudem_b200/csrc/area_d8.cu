// D8 contributing area: the dependency stencil (the evaluation sweep is sweep_warp.cu).
//
// reference: initNeighborD8up src/commonLib.cpp:240-283 (in-degree per cell),
//            aread8 main loop   src/aread8.cpp:216-304 (pull-gather in k order,
//            decrement the downslope cell, enqueue when its count reaches zero).
//
// The reference's result is a deterministic gather — area(c) = ((w|1) + a_k1) + a_k2 ...
// over the neighbours that drain into c, in k = 1..8 order, float32 — evaluated once
// per cell in ANY topological order, so the GPU schedule below is bit-exact:
//
//   k_deps_d8  : 3x3 stencil over p -> node (u16: inflow mask | dir | flags) and
//                cnt (u8: remaining inflow count).  5 B/cell written-read, streamed
//                through TMA-staged shared-memory tiles.
//   the sweep  : sweep_warp.cu (tile dataflow, one warp per tile visit).
#include "common.cuh"
#include "ctx.h"
#include "tile_pipe.cuh"

namespace td {
namespace {
constexpr int TW = 128, TH = 32;

constexpr unsigned NODE_VALID = 0x8000u, NODE_CON = 0x1000u;

// Generic per-cell evaluation (any int16 codes): the slow path of k_deps_d8 for threads that see a direction
// code outside 0..8 that is not nodata.  pm = staged tile at (row above, column c).
template <int SW>
__device__ __noinline__ void deps_d8_generic(const short* pm, const Strip s, int r, int c, short nodata, unsigned short* on4, unsigned char* oc4) {
  short nb[3][6];
#pragma unroll
  for (int j = 0; j < 3; ++j)
#pragma unroll
    for (int i = 0; i < 6; ++i) nb[j][i] = pm[j * SW + i - 1];
  const bool rowok[3] = {s.on_grid(r - 1, 0), true, s.on_grid(r + 1, 0)};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int cc = c + i;
    const int d = nb[1][i + 1];
    const bool colok[3] = {cc - 1 >= 0, true, cc + 1 < s.nx};
    const bool valid = (cc < s.nx) & (d != (int)nodata) & ((unsigned)d <= 8u);
    unsigned mask = 0, con = 0;
#pragma unroll
    for (int k = 1; k <= 8; ++k) {
      const int dn = nb[1 + drow(k)][i + 1 + dcol(k)];
      const unsigned miss = (unsigned)(!(rowok[1 + drow(k)] & colok[1 + dcol(k)]) | (dn == (int)nodata));   // off-grid or nodata
      const unsigned toward = (unsigned)((dn - k == 4) | (dn - k == -4));                                    // drains into this cell
      const unsigned inrange = (unsigned)((unsigned)dn <= 8u);
      mask |= ((~miss & 1u) & toward & inrange) << (k - 1);
      // counted by the evaluation loop but never evaluated (code outside 0..8) -> its area stays nodata
      con |= miss | (toward & (inrange ^ 1u));
    }
    on4[i] = valid ? (unsigned short)(NODE_VALID | (con ? NODE_CON : 0u) | ((unsigned)d << 8) | mask) : (unsigned short)0;
    oc4[i] = valid ? (unsigned char)__popc(mask) : (unsigned char)0xff;
  }
}

// bit 7 of every byte of the result = (that byte of w == that byte of t); all bytes of w ^ t must be < 0x80
__device__ __forceinline__ unsigned eq_bytes(unsigned w, unsigned t) { return ~((w ^ t) + 0x7f7f7f7fu) & 0x80808080u; }

// Dependency stencil.  Every staged direction code is first reduced to one byte q (0..8 = the code, 16 = off the
// grid or nodata, 32 = any other value); a thread then handles four adjacent cells at once with byte-parallel
// integer arithmetic: "neighbour k drains into me" is a byte comparison of the four neighbours' q with k+4 / k-4
// (src/commonLib.cpp:262-264; code 0 counts for k = 4 exactly as the reference's "tempShort - k == -4" does).
constexpr int STAGES = 3;
using Ring = TileRing<short, TW, TH, STAGES>;

// Persistent CTAs over a three-stage ring of 2-D TMA tiles (tile_pipe.cuh): while a tile is reduced to q bytes and evaluated, the
// copies of the next two are under way.
__global__ void __launch_bounds__(256) k_deps_d8(const TD_GRID_CONSTANT TileMap tm, unsigned short* __restrict__ node,
                                                 unsigned char* __restrict__ cnt, float* __restrict__ area, Strip s,
                                                 short nodata, float area_init) {
  extern __shared__ __align__(128) unsigned char dsm128[];
  using G = Ring::G;
  constexpr int QW = TW / 4 + 2;                       // words per row of q: columns c0-4 .. c0+TW+3
  __shared__ unsigned qw[(TH + 2) * QW];
  Ring ring;
  ring.init(dsm128, &tm, s);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long t = blockIdx.x; t < ring.ntiles; t += gridDim.x) {
    int r0, c0;
    const short* tile = ring.acquire(t, r0, c0);
    // ---- q bytes of the staged tile, four per thread and step
    {
      const bool full_cols = c0 >= 4 && c0 + TW + 4 <= s.nx;        // no word of this tile touches the left / right edge of the grid
      for (int w = threadIdx.x; w < (TH + 2) * QW; w += 256) {
        const int tr = w / QW, x = w - tr * QW;            // tile row, word within the row
        const int gr = r0 - 1 + tr;
        const bool rowon = (gr >= 1 && gr <= s.ny) || (gr == 0 && s.has_top) || (gr == s.ny + 1 && s.has_bot);
        unsigned word = 0x10101010u;                       // a row off the grid: nothing there
        if (rowon) {
          const short4 v = *reinterpret_cast<const short4*>(tile + tr * G::SW + (G::HP - 4) + 4 * x);
          const int d4[4] = {v.x, v.y, v.z, v.w};
          word = 0;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            unsigned q = (unsigned)d4[i] <= 8u ? (unsigned)d4[i] : 32u;   // 0..8 = the code, anything else (negative codes included) = 32
            if (d4[i] == (int)nodata) q = 16u;
            word |= q << (8 * i);
          }
          if (!full_cols) {                                // the rim of the grid: columns off the grid read as nodata
            const int gc = c0 - 4 + 4 * x;
#pragma unroll
            for (int i = 0; i < 4; ++i)
              if (gc + i < 0 || gc + i >= s.nx) word = (word & ~(0xffu << (8 * i))) | (16u << (8 * i));
          }
        }
        qw[w] = word;
      }
    }
    __syncthreads();
#pragma unroll 1
    for (int pass = 0; pass < TH / 8; ++pass) {
      const int tr = warp + 8 * pass;
      const int r = r0 + tr, c = c0 + lane * 4;
      if (r > s.ny || c >= s.pitch) continue;
      // W[j][0..2]: the q bytes of the cells (c-1..c+2), (c..c+3), (c+1..c+4) of tile row tr + j
      unsigned W[3][3];
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const unsigned* q = qw + (tr + j) * QW + lane;
        const unsigned wl = q[0], wc = q[1], wr = q[2];
        W[j][0] = __funnelshift_l(wl, wc, 8);
        W[j][1] = wc;
        W[j][2] = __funnelshift_r(wc, wr, 8);
      }
      unsigned mb = 0, all = 0;
#pragma unroll
      for (int k = 1; k <= 8; ++k) {
        const unsigned wk = W[1 + drow(k)][1 + dcol(k)];
        unsigned z = eq_bytes(wk, (k <= 4 ? (unsigned)(k + 4) : (unsigned)(k - 4)) * 0x01010101u);
        if (k == 4) z |= eq_bytes(wk, 0u);                  // 0 - 4 == -4
        mb |= z >> (8 - k);
        all |= wk;
      }
      const unsigned wc = W[1][1];
      unsigned nw0, nw1, cww;                         // the four node words (two per register) and the four counts
      if ((all | wc) & 0x20202020u) {
        // a code outside 0..8 next to these cells: the generic rule decides (it can contaminate, src/aread8.cpp:245-250)
        unsigned short on4[4]; unsigned char oc4[4];
        deps_d8_generic<G::SW>(tile + tr * G::SW + G::HP + lane * 4, s, r, c, nodata, on4, oc4);
        nw0 = (unsigned)on4[0] | ((unsigned)on4[1] << 16); nw1 = (unsigned)on4[2] | ((unsigned)on4[3] << 16);
        cww = (unsigned)oc4[0] | ((unsigned)oc4[1] << 8) | ((unsigned)oc4[2] << 16) | ((unsigned)oc4[3] << 24);
      } else {
        const unsigned vbit = ~(wc + 0x77777777u) & 0x80808080u;          // bit 7: q <= 8 (a cell of the flow field)
        const unsigned vm = (vbit >> 7) * 0xffu;                            // 0xff per valid byte
        unsigned x = mb - ((mb >> 1) & 0x55555555u);                        // per-byte population count
        x = (x & 0x33333333u) + ((x >> 2) & 0x33333333u);
        x = (x + (x >> 4)) & 0x0f0f0f0fu;
        const unsigned cw = (x & vm) | ~vm;                                 // count, or 0xff on cells outside the field
        const unsigned hb = (0x80808080u | ((all & 0x10101010u)) | wc) & vm;   // VALID | CON (bit 12 of the node word) | code
        const unsigned mw = mb & vm;
        // node words = (high byte << 8) | inflow mask: two byte permutations interleave the four cells, the counts are packed already
        nw0 = __byte_perm(mw, hb, 0x5140); nw1 = __byte_perm(mw, hb, 0x7362); cww = cw;
      }
      const long long o = s.idx(r, c);
      *reinterpret_cast<uint2*>(node + o) = make_uint2(nw0, nw1);
      *reinterpret_cast<unsigned*>(cnt + o) = cww;
      // the area partition starts as nodata (-1) everywhere (src/aread8.cpp:193)
      *reinterpret_cast<float4*>(area + o) = make_float4(area_init, area_init, area_init, area_init);
    }
    ring.release(&tm, t);          // (its barrier also protects qw against the next tile's conversion)
  }
}

// The node words of the halo rows (rows 0 / ny + 1 where a neighbour strip exists) hold only the direction code of the
// neighbour's edge cell (0 for nodata and codes outside 0..8).  gridnet's algebras look at a contributor's code (a code 0
// contributes nothing, src/gridnet.cpp:393); k_deps_d8 leaves these rows alone.
__global__ void k_halo_codes_d8(const short* __restrict__ p, unsigned short* __restrict__ node, Strip s, short nodata) {
  const int c = (int)(blockIdx.x * blockDim.x + threadIdx.x);
  if (c >= s.pitch) return;
#pragma unroll
  for (int side = 0; side < 2; ++side) {
    if (!(side == 0 ? s.has_top : s.has_bot)) continue;
    const long long o = s.idx(side == 0 ? 0 : s.ny + 1, c);
    const int d = p[o];
    node[o] = (c < s.nx && d != (int)nodata && (unsigned)d <= 8u) ? (unsigned short)((unsigned)d << 8) : (unsigned short)0;
  }
}

}  // namespace

cudaError_t launch_halo_codes_d8(const short* p, unsigned short* node, const Strip& s, short nodata, cudaStream_t st) {
  if (!s.has_top && !s.has_bot) return cudaSuccess;
  k_halo_codes_d8<<<(s.pitch + 255) / 256, 256, 0, st>>>(p, node, s, nodata);
  TD_LAUNCHED();
  return cudaGetLastError();
}

cudaError_t launch_deps_d8(const short* p, unsigned short* node, unsigned char* cnt, float* area, const Strip& s, short nodata,
                           cudaStream_t st, float area_init) {
  TileMap tm;
  if (make_tile_map(&tm, p, 2, s.pitch, s.ny + 2, Ring::G::SW, Ring::G::ROWS)) return cudaErrorInvalidValue;
  const long long ntiles = (long long)((s.pitch + TW - 1) / TW) * ((s.ny + TH - 1) / TH);
  int grid = 0;
  if (stencil_grid((const void*)k_deps_d8, 256, Ring::SMEM, ntiles, &grid)) return cudaErrorInvalidValue;
  k_deps_d8<<<grid, 256, Ring::SMEM, st>>>(tm, node, cnt, area, s, nodata, area_init);
  TD_LAUNCHED();
  return cudaGetLastError();
}



}  // namespace td
