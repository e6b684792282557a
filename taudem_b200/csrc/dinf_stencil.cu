// D-infinity flow direction stencil: setPosDirDinf + SET2 + VSLOPE fused
// (reference src/dinf.cpp:530-595, 317-373, 286-313).
//
// Eligibility is the D8 rule (global edge / nodata / nodata neighbour -> angle nodata = -FLT_MAX, slope nodata = -1).
// Otherwise the first of the eight triangular facets with the strictly largest VSLOPE slope wins;
// angle = (float)(ANGC*PI/2 + ANGF*A), slope = (float)Smax; no facet with S > 0 -> angle -1 (flat), slope 0.
//
// Structure (persistent CTAs, 2-D TMA tiles through a three-stage ring, tile_pipe.cuh):
//  1. the eight facets are ranked with a float copy of VSLOPE's three-branch formula on squared slopes (no root);
//     the float error is ~1e-6, so every facet whose float rank is more than 4e-5 below the best one cannot be the
//     exact winner.  In all but ~1e-4 of the cells exactly one facet survives: the winner is known without FP64.
//     Cells with several survivors evaluate those facets in FP64 in increasing K with the reference's strict '>'.
//     The 1e-6 bound holds while the largest squared slope is a finite float >= 2^-100: rounding in the subnormal range
//     then costs at most a few 2^-149 absolutely, and no term has overflowed (an overflow makes the square infinite).
//     Outside that range (relief far below or far above any terrain's, or neighbour differences that overflow float)
//     the squares underflow to 0 or collapse onto +inf, so every facet with a positive slope is evaluated in FP64.
//  2. the winner is evaluated ONCE per cell, uniformly over the warp (no per-facet divergence): both quotients,
//     the clipped slope, the root, then selects; the three divisions are divisions by row constants
//     (div_const, rowfact.cuh: five FMA-pipe FP64 operations each, correctly rounded), atan2 only for the facets whose
//     direction lies inside the facet.  Bit-identical to the reference's FP64 arithmetic.
// HBM traffic per cell: read fel 4 B, write ang 4 B + slp 4 B = 12 B (algorithmic).
#include "dinf_common.cuh"
#include "kernels.h"
#include "rowfact.cuh"
#include "tile_pipe.cuh"

namespace td {
namespace {
constexpr int TW = 128, TH = 32, STAGES = 3;
using Ring = TileRing<float, TW, TH, STAGES>;

// VSLOPE with the divisions by row constants done through their reciprocals (rf.safe) or as plain divisions
__device__ __forceinline__ Facet vslope_row(double E0, double E1, double E2, double D1, double D2, double DD, double r1, double r2,
                                            double rd, bool safe) {
  Facet f;
  const double x1 = E0 - E1, x2 = E1 - E2, x3 = E0 - E2;
  double Sc;
  if (safe) { f.S1 = div_const(x1, D1, r1); f.S2 = div_const(x2, D2, r2); Sc = div_const(x3, DD, rd); }
  else { f.S1 = x1 / D1; f.S2 = x2 / D2; Sc = x3 / DD; }
  if (f.S2 < 0.) { f.S = f.S1; f.code = 0; return f; }
  bool clip;
  if (f.S1 <= 0.) clip = !(f.S1 == 0. && f.S2 == 0.);
  else {
    const double x = f.S2 * D1, y = f.S1 * D2;
    if (x > y * (1. + 1e-9)) clip = true;
    else if (x < y * (1. - 1e-9)) clip = false;
    else clip = atan2(f.S2, f.S1) > atan2(D2, D1);
  }
  const double Sq = sqrt(f.S1 * f.S1 + f.S2 * f.S2);
  if (clip) { f.S = Sc; f.code = 1; return f; }
  f.S = Sq;
  f.code = (f.S1 == 0. && f.S2 == 0.) ? 0 : 2;
  return f;
}

// facet geometry as arithmetic on a run-time K: offsets of E1 / E2 in the staged tile, which cell size is D1
__device__ __forceinline__ void facet_geom(int K, int sw, int& o1, int& o2, bool& d1x) {
  const int i1 = (K == 2 || K == 3) ? -1 : (K == 6 || K == 7) ? 1 : 0;
  const int j1 = (K == 1 || K == 8) ? 1 : (K == 4 || K == 5) ? -1 : 0;
  const int i2 = K <= 4 ? -1 : 1;
  const int j2 = (K == 1 || K == 2 || K == 7 || K == 8) ? 1 : -1;
  o1 = i1 * sw + j1; o2 = i2 * sw + j2;
  d1x = (K == 1 || K == 4 || K == 5 || K == 8);
}

// several facets within the float error of the best one, or every facet with a positive slope where the float ranking does not
// hold: the exact slopes decide (increasing K, strict '>'); rare, out of line
__device__ __noinline__ int exact_pick(const float* q0, int sw, unsigned cand, const RowFact* rfp) {
  const RowFact rf = *rfp;
  const double E0 = (double)q0[0];
  double SMAX = 0.; int KD = 0;
  for (unsigned m = cand; m; m &= m - 1) {
    const int K = __ffs(m);
    int o1, o2; bool d1x;
    facet_geom(K, sw, o1, o2, d1x);
    const Facet f = vslope_row(E0, (double)q0[o1], (double)q0[o2], d1x ? rf.dx : rf.dy, d1x ? rf.dy : rf.dx, rf.dd,
                               d1x ? rf.rdx : rf.rdy, d1x ? rf.rdy : rf.rdx, rf.rdd, rf.safe != 0);
    if (f.S > SMAX) { SMAX = f.S; KD = K; }
  }
  return KD;
}

__global__ void __launch_bounds__(256) k_dinf_stencil(const TD_GRID_CONSTANT TileMap tm, float* __restrict__ ang, float* __restrict__ slp,
                                                      const RowFact* __restrict__ rowf, Strip s, float nodata,
                                                      unsigned long long* __restrict__ nflat) {
  extern __shared__ __align__(128) unsigned char dsm128[];
  using G = Ring::G;
  Ring ring;
  ring.init(dsm128, &tm, s);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned myflat = 0;
  for (long long t = blockIdx.x; t < ring.ntiles; t += gridDim.x) {
    int r0, c0;
    const float* tile = ring.acquire(t, r0, c0);
#pragma unroll 1
    for (int pass = 0; pass < TH / 8; ++pass) {
      const int tr = warp * (TH / 8) + pass;
      const int r = r0 + tr, c = c0 + lane * 4;
      if (r > s.ny || c >= s.pitch) continue;
      const float* pm = tile + tr * G::SW + G::HP + lane * 4;
      const RowFact* rfp = rowf + (r - 1);
      const float rdxf = rfp->rdxf, rdyf = rfp->rdyf, rddf = rfp->rddf, dxf = rfp->dxf, dyf = rfp->dyf;
      unsigned em = ((r == 1 && !s.has_top) || (r == s.ny && !s.has_bot)) ? 0xfu : 0u;
      em |= (c == 0) ? 1u : 0u;
      const int klast = s.nx - 1 - c;
      if (klast < 4) em |= (0xfu << max(klast, 0)) & 0xfu;
      float oa[4], os[4];
      // one cell at a time, the code once (an unrolled body of this size does not fit the instruction cache)
#pragma unroll 1
      for (int i = 0; i < 4; ++i) {
        const float* q0 = pm + G::SW + i;          // centre cell in the staged tile
        float nb[3][3];
#pragma unroll
        for (int j = 0; j < 3; ++j)
#pragma unroll
          for (int x = 0; x < 3; ++x) nb[j][x] = q0[(j - 1) * G::SW + (x - 1)];
        const float z = nb[1][1];
        float dmin = fabsf(z - nodata);
#pragma unroll
        for (int k = 1; k <= 8; ++k) dmin = fminf(dmin, fabsf(nb[1 + drow(k)][1 + dcol(k)] - nodata));
        const bool bad = dmin < TD_MINEPS || ((em >> i) & 1u);
        // ---- 1. float ranking of the eight facets (squared slopes, 0 for a non-positive one) and the facts that are exact in float
        float st[8], smaxf = 0.f;
        unsigned s2neg = 0, clipsafe = 0;
#pragma unroll
        for (int K = 1; K <= 8; ++K) {
          const float e1 = nb[1 + fI1(K)][1 + fJ1(K)], e2 = nb[1 + fI2(K)][1 + fJ2(K)];
          const float r1 = fD1isDx(K) ? rdxf : rdyf, r2 = fD1isDx(K) ? rdyf : rdxf;
          const float d1f = fD1isDx(K) ? dxf : dyf, d2f = fD1isDx(K) ? dyf : dxf;
          const float s1 = (z - e1) * r1, s2 = (e1 - e2) * r2;
          const bool neg = e1 < e2;                                      // S2 < 0, exactly
          const float x = s2 * d1f, y = s1 * d2f;
          const bool clip = (z <= e1) ? !(z == e1 && e1 == e2) : (x > y);
          const bool csafe = !neg && ((z <= e1) ? !(z == e1 && e1 == e2) : (x > y * 1.0001f));   // clipped beyond doubt
          const float lin = neg ? s1 : (z - e2) * rddf;
          const float Q = (neg || clip) ? (lin > 0.f ? lin * lin : 0.f) : s1 * s1 + s2 * s2;
          st[K - 1] = Q;
          smaxf = fmaxf(smaxf, Q);
          s2neg |= neg ? (1u << (K - 1)) : 0u;
          clipsafe |= csafe ? (1u << (K - 1)) : 0u;
        }
        unsigned cand = 0;
        const float thr = smaxf * 0.99996f;
#pragma unroll
        for (int K = 1; K <= 8; ++K) cand |= (st[K - 1] >= thr && st[K - 1] > 0.f) ? (1u << (K - 1)) : 0u;
        if (smaxf >= 0x1p-100f && smaxf <= FLT_MAX) {
          // two facets that share E1 and both have S2 < 0 have the same slope S1 bit for bit, two that share E2 and are both
          // clipped have the same slope (E0 - E2) / DD: the lower K wins such a tie (strict '>'), no FP64 needed to say so
          const unsigned A = cand & s2neg, B = cand & clipsafe;
          unsigned drop = ((A & 0x2au) << 1) & A;                         // pairs (2,3) (4,5) (6,7) share E1
          if ((A & 0x81u) == 0x81u) drop |= 0x80u;                        // pair (1,8)
          drop |= ((B & 0x55u) << 1) & B;                                 // pairs (1,2) (3,4) (5,6) (7,8) share E2
          cand &= ~drop;
        } else {
          // the float ranking is not reliable here (header, 1.): every facet with a positive slope, i.e. z above E1 or E2,
          // goes to the FP64 evaluation, without the drop rules (their float tests are not reliable either)
          cand = 0;
#pragma unroll
          for (int K = 1; K <= 8; ++K)
            cand |= (z > nb[1 + fI1(K)][1 + fJ1(K)] || z > nb[1 + fI2(K)][1 + fJ2(K)]) ? (1u << (K - 1)) : 0u;
        }
        if (bad) cand = 0;
        int KD = cand ? __ffs(cand) : 0;
        if (cand & (cand - 1u)) KD = exact_pick(q0, G::SW, cand, rfp);
        // ---- 2. the winner, once and uniformly
        float a = -1.0f, sl = 0.f;
        {
          const int K = KD ? KD : 1;
          int o1, o2; bool d1x;
          facet_geom(K, G::SW, o1, o2, d1x);
          const double dx = rfp->dx, dy = rfp->dy, rdx = rfp->rdx, rdy = rfp->rdy;
          const Facet f = vslope_row((double)z, (double)q0[o1], (double)q0[o2], d1x ? dx : dy, d1x ? dy : dx, rfp->dd,
                                     d1x ? rdx : rdy, d1x ? rdy : rdx, rfp->rdd, rfp->safe != 0);
          if (KD > 0 && f.S > 0.) {
            const double A = f.code == 0 ? 0. : f.code == 1 ? (d1x ? rfp->adA : rfp->adB) : atan2(f.S2, f.S1);
            a = dinf_angle(K, A);
            sl = (float)f.S;
          } else KD = 0;
        }
        const float va = bad ? TD_MISSINGFLOAT : a, vs = bad ? -1.0f : sl;
        if (i == 0) { oa[0] = va; os[0] = vs; } else if (i == 1) { oa[1] = va; os[1] = vs; } else if (i == 2) { oa[2] = va; os[2] = vs; } else { oa[3] = va; os[3] = vs; }
        if (!bad && KD == 0) ++myflat;
      }
      const long long o = s.idx(r, c);
      *reinterpret_cast<float4*>(ang + o) = make_float4(oa[0], oa[1], oa[2], oa[3]);
      *reinterpret_cast<float4*>(slp + o) = make_float4(os[0], os[1], os[2], os[3]);
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

int launch_dinf_stencil(const float* elev, float* ang, float* slp, const RowFact* rowf, const Strip& s, float nodata,
                        unsigned long long* nflat, cudaStream_t st) {
  TileMap tm;
  if (int rc = make_tile_map(&tm, elev, 4, s.pitch, s.ny + 2, Ring::G::SW, Ring::G::ROWS)) return rc;
  const long long ntiles = (long long)((s.pitch + TW - 1) / TW) * ((s.ny + TH - 1) / TH);
  int grid = 0;
  if (int rc = stencil_grid((const void*)k_dinf_stencil, 256, Ring::SMEM, ntiles, &grid)) return rc;
  k_dinf_stencil<<<grid, 256, Ring::SMEM, st>>>(tm, ang, slp, rowf, s, nodata, nflat);
  TD_LAUNCHED();
  TD_CUDA(cudaGetLastError());
  return TD_OK;
}
}  // namespace td
