// slopeavedown: the D8 slope averaged over a downslope distance (src/SlopeAveDown.cpp:59-330).
//
// The reference repeats niter = dn / min(dx, dy) + 1 passes; each pass is one full run of the aread8 queue
// (initNeighborD8up), and a processed cell i with code k in 1..8 whose receiver n holds an elevation takes
//   ddi = dist[row][k] + dd(n),  sd(i) = (fel(i) - ed(n)) / ddi  if sd(i) tests as nodata and ddi > dn,  ed(i) = ed(n), dd(i) = ddi.
// A receiver is dequeued after all its contributors, so every cell reads its receiver's pair as the previous pass left it:
// each pass is one Jacobi step over a fixed set of cells.  The set (the cells the queue reaches) is the set the D8 sweep
// evaluates: after td_aread8_deps_dev + the sweep their count byte is 0xFE (sweep_warp.cu).
//
//   k_sad_init : code byte per cell (the direction where the cell takes its receiver's pair, else 0), both state buffers
//                and sd.
//   k_sad_pass : one pass; (ed, dd) interleaved as float2 so a receiver's pair is one 8-byte load, ping-ponged between
//                passes; sd in place (only cell i reads or writes sd(i)).  Raises *changed when any bit of the state moved.
#include "common.cuh"
#include "ctx.h"
#include "kernels.h"

namespace td {
namespace {
constexpr int TPB = 256;

__global__ void __launch_bounds__(TPB) k_sad_init(const short* __restrict__ p, const unsigned char* __restrict__ cnt, const float* __restrict__ fel,
                                                  unsigned char* __restrict__ code, float2* __restrict__ s0, float2* __restrict__ s1,
                                                  float* __restrict__ sd, Strip s, short p_nodata, float fel_nodata) {
  const long long o = (long long)blockIdx.x * TPB + threadIdx.x;
  if (o >= s.cells()) return;
  const int r = (int)(o / s.pitch), c = (int)(o - (long long)r * s.pitch);
  // ed = fel, dd = 0 where both fel and p are data, else MISSINGFLOAT (src/SlopeAveDown.cpp:153-163); the halo rows from the
  // neighbours' fel and p rows, which is what the reference's first ed->share() / dd->share() hands over
  float2 v = make_float2(TD_MISSINGFLOAT, TD_MISSINGFLOAT);
  if (s.on_grid(r, c)) {
    const float z = fel[o];
    if (!nd_f(z, fel_nodata) && !nd_s(p[o], p_nodata)) v = make_float2(z, 0.0f);
  }
  s0[o] = v;
  s1[o] = v;
  if (r < 1 || r > s.ny) return;
  unsigned char k = 0;
  if (c < s.nx && cnt[o] == 0xFEu) {              // processed: the queue reached it (p is data and in 0..8)
    const int d = p[o];
    if (d >= 1 && d <= 8 && s.on_grid(r + drow(d), c + dcol(d))) k = (unsigned char)d;   // ed->hasAccess(in, jn)
  }
  code[o] = k;
  sd[o] = TD_MISSINGFLOAT;
}

// One pass over the owned rows: block (x, y) takes TPB columns of the rows y + 1, y + 1 + gridDim.y, ...  A cell whose code is 0
// never changes; both buffers hold its initial pair.  A cell whose receiver's ed is nodata does not change either, and is not
// written: ed never returns to nodata once set, so that receiver was nodata in the pass before as well, and the output buffer
// (written two passes ago) already holds this cell's pair.
__global__ void __launch_bounds__(TPB) k_sad_pass(const unsigned char* __restrict__ code, const float* __restrict__ fel,
                                                  const float2* __restrict__ src, float2* __restrict__ dst, float* __restrict__ sd,
                                                  const float* __restrict__ dist, Strip s, double dn, int* __restrict__ changed) {
  const int c = blockIdx.x * TPB + threadIdx.x;
  int moved = 0;
  for (int r = blockIdx.y + 1; r <= s.ny; r += gridDim.y) {
    const long long o = s.idx(r, c);
    const int k = c < s.pitch ? code[o] : 0;
    if (k == 0) continue;
    const float2 en = src[o + (long long)drow(k) * s.pitch + dcol(k)];
    if (nd_f(en.x, TD_MISSINGFLOAT)) continue;
    const float ddi = __fadd_rn(__ldg(dist + (size_t)(r - 1) * 8 + (k - 1)), en.y);   // float, src/SlopeAveDown.cpp:236
    const float old_sd = sd[o];
    if (nd_f(old_sd, TD_MISSINGFLOAT) && (double)ddi > dn) {                       // "set" is the nodata test on the stored slope
      const float slp = __fdiv_rn(__fsub_rn(fel[o], en.x), ddi);
      sd[o] = slp;
      moved |= __float_as_uint(slp) != __float_as_uint(old_sd);
    }
    const float2 mine = src[o];
    moved |= (__float_as_uint(mine.x) != __float_as_uint(en.x)) | (__float_as_uint(mine.y) != __float_as_uint(ddi));
    dst[o] = make_float2(en.x, ddi);
  }
  if (__syncthreads_or(moved) && threadIdx.x == 0) *changed = 1;     // one store per block, not per cell
}
}  // namespace

int launch_sad_init(const short* p, const unsigned char* cnt, const float* fel, unsigned char* code, float* s0, float* s1, float* sd,
                    const Strip& s, short p_nodata, float fel_nodata, cudaStream_t st) {
  const long long blocks = (s.cells() + TPB - 1) / TPB;
  k_sad_init<<<(unsigned)blocks, TPB, 0, st>>>(p, cnt, fel, code, (float2*)s0, (float2*)s1, sd, s, p_nodata, fel_nodata);
  TD_LAUNCHED();
  TD_CUDA(cudaGetLastError());
  return TD_OK;
}

int launch_sad_pass(const unsigned char* code, const float* fel, const float* src, float* dst, float* sd, const float* dist, const Strip& s,
                    double dn, int* changed, cudaStream_t st) {
  const dim3 grid((s.pitch + TPB - 1) / TPB, s.ny < 65535 ? s.ny : 65535);
  k_sad_pass<<<grid, TPB, 0, st>>>(code, fel, (const float2*)src, (float2*)dst, sd, dist, s, dn, changed);
  TD_LAUNCHED();
  TD_CUDA(cudaGetLastError());
  return TD_OK;
}

}  // namespace td
