// Point-wise consumers of the contributing-area rasters (SURVEY.md section 8 (f) rank 4):
//   threshold  src = (ssa >= thresh [& mask >= 0]) ? 1 : 0, nodata where ssa is nodata   (src/Threshold.cpp:109-131)
//   twi        twi = ln(sca / slp) where both are data and positive, else nodata (-1)     (src/TWI.cpp:108-124)
//   slopearea  sa = slp^m * sca^n where slp >= 0 and sca >= 0, else nodata (-1)            (src/SlopeArea.cpp:114-125)
//   slopearearatio  sar = slp / sca where sca is data, else nodata (-1)                    (src/SlopeAreaRatio.cpp:107-118)
//   lengtharea ss = ad8 >= M plen^y ? 1 : 0 where plen >= 0, else nodata (-32768)          (src/LengthArea.cpp:110-120)
// One streaming kernel each, four cells per thread (16-byte loads, 8 / 16-byte stores): 6 B (10 with a mask) and 12 B of HBM
// traffic per cell.  Device-strip level entry points take strips like every other kernel of the path; the host-grid level
// copies dense arrays in and out.  isNodata is linearpart's |v - nodata| < 1e-5 (src/linearpart.h:471-483).
#include "common.cuh"
#include "ctx.h"
#include "kernels.h"

namespace td {
namespace {
__global__ void __launch_bounds__(256) k_threshold(const float* __restrict__ ssa, const float* __restrict__ mask, short* __restrict__ src, Strip s,
                                                   float thresh, float ssa_nodata) {
  const int r = 1 + (int)blockIdx.x, c = ((int)blockIdx.y * 256 + (int)threadIdx.x) * 4;      // rows on grid.x
  if (c >= s.pitch) return;
  const long long o = s.idx(r, c);
  const float4 v = *reinterpret_cast<const float4*>(ssa + o);
  float4 m = make_float4(0.f, 0.f, 0.f, 0.f);
  if (mask) m = *reinterpret_cast<const float4*>(mask + o);
  const float a[4] = {v.x, v.y, v.z, v.w}, mm[4] = {m.x, m.y, m.z, m.w};
  short out[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) out[i] = nd_f(a[i], ssa_nodata) ? TD_MISSINGSHORT : (short)((a[i] >= thresh) & (mm[i] >= 0.f) ? 1 : 0);
  *reinterpret_cast<short4*>(src + o) = make_short4(out[0], out[1], out[2], out[3]);
}

// ln of a float quotient: the reference's log(float) is glibc's logf (< 1 ulp); here the double logarithm rounded to float
// (correctly rounded in all but ~1e-9 of the cases) — the two can differ in the last bit (tests: <= 1 ulp).
__global__ void __launch_bounds__(256) k_twi(const float* __restrict__ slp, const float* __restrict__ sca, float* __restrict__ twi, Strip s,
                                             float slp_nodata, float sca_nodata) {
  const int r = 1 + (int)blockIdx.x, c = ((int)blockIdx.y * 256 + (int)threadIdx.x) * 4;
  if (c >= s.pitch) return;
  const long long o = s.idx(r, c);
  const float4 sv = *reinterpret_cast<const float4*>(slp + o), av = *reinterpret_cast<const float4*>(sca + o);
  const float sl[4] = {sv.x, sv.y, sv.z, sv.w}, ar[4] = {av.x, av.y, av.z, av.w};
  float out[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const bool ok = !nd_f(ar[i], sca_nodata) && !nd_f(sl[i], slp_nodata) && sl[i] > 0.0f && ar[i] > 0.0f;
    out[i] = ok ? (float)log((double)(ar[i] / sl[i])) : -1.0f;
  }
  *reinterpret_cast<float4*>(twi + o) = make_float4(out[0], out[1], out[2], out[3]);
}
// slp^m * sca^n: the reference multiplies two powf results as floats (std::pow(float, float), src/SlopeArea.cpp:119); here each power
// is the double pow rounded to float (correctly rounded in all but ~1e-9 of the cases; glibc's powf is within 0.52 ulp), then the
// same float product — results agree to a few ulps (tests: relative 1e-6), nodata masks are identical.
// x^e as a float: exact products for the exponents 1 and 2 (the reference's defaults: slope^2 * area^1), the correctly rounded root
// for 0.5, the double pow otherwise (two orders of magnitude more instructions)
__device__ __forceinline__ float pow_float(float x, float e) {
  if (e == 1.0f) return x;
  if (e == 2.0f) return (float)((double)x * (double)x);
  if (e == 0.5f) return (float)sqrt((double)x);
  return (float)pow((double)x, (double)e);
}
__global__ void __launch_bounds__(256) k_slopearea(const float* __restrict__ slp, const float* __restrict__ sca, float* __restrict__ sa, Strip s,
                                                   float m, float n) {
  const int r = 1 + (int)blockIdx.x, c = ((int)blockIdx.y * 256 + (int)threadIdx.x) * 4;
  if (c >= s.pitch) return;
  const long long o = s.idx(r, c);
  const float4 sv = *reinterpret_cast<const float4*>(slp + o), av = *reinterpret_cast<const float4*>(sca + o);
  const float sl[4] = {sv.x, sv.y, sv.z, sv.w}, ar[4] = {av.x, av.y, av.z, av.w};
  float out[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const bool ok = sl[i] >= 0.0f && ar[i] >= 0.0f;
    out[i] = ok ? pow_float(sl[i], m) * pow_float(ar[i], n) : -1.0f;
  }
  *reinterpret_cast<float4*>(sa + o) = make_float4(out[0], out[1], out[2], out[3]);
}
// lengtharea (src/LengthArea.cpp:110-120): ss = ((float)ad8 >= M * plen^y) ? 1 : 0 where plen >= 0, else nodata (-32768); ad8 is
// the contributing area read as 32-bit integers, plen^y as above and M * plen^y one float product.  The reference's powf is within
// 0.52 ulp, pow_float correctly rounded in all but ~1e-9 of the cases: the power can differ by one ulp, and the result only when
// (float)ad8 lies exactly on one of those two adjacent floats (tests: bit for bit).  10 B of HBM traffic per cell.
__global__ void __launch_bounds__(256) k_lengtharea(const float* __restrict__ plen, const int* __restrict__ ad8, short* __restrict__ ss, Strip s,
                                                    float m, float y) {
  const int r = 1 + (int)blockIdx.x, c = ((int)blockIdx.y * 256 + (int)threadIdx.x) * 4;
  if (c >= s.pitch) return;
  const long long o = s.idx(r, c);
  const float4 lv = *reinterpret_cast<const float4*>(plen + o);
  const int4 av = *reinterpret_cast<const int4*>(ad8 + o);
  const float l[4] = {lv.x, lv.y, lv.z, lv.w};
  const int a[4] = {av.x, av.y, av.z, av.w};
  short out[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) out[i] = l[i] >= 0.0f ? (short)((float)a[i] >= m * pow_float(l[i], y) ? 1 : 0) : TD_MISSINGSHORT;
  *reinterpret_cast<short4*>(ss + o) = make_short4(out[0], out[1], out[2], out[3]);
}
// slp / sca as one IEEE float division (-prec-div=true); only the area's nodata is looked at, like the reference
__global__ void __launch_bounds__(256) k_slopearearatio(const float* __restrict__ slp, const float* __restrict__ sca, float* __restrict__ sar, Strip s,
                                                        float sca_nodata) {
  const int r = 1 + (int)blockIdx.x, c = ((int)blockIdx.y * 256 + (int)threadIdx.x) * 4;
  if (c >= s.pitch) return;
  const long long o = s.idx(r, c);
  const float4 sv = *reinterpret_cast<const float4*>(slp + o), av = *reinterpret_cast<const float4*>(sca + o);
  const float sl[4] = {sv.x, sv.y, sv.z, sv.w}, ar[4] = {av.x, av.y, av.z, av.w};
  float out[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) out[i] = nd_f(ar[i], sca_nodata) ? -1.0f : sl[i] / ar[i];
  *reinterpret_cast<float4*>(sar + o) = make_float4(out[0], out[1], out[2], out[3]);
}
// gridnet's mask rule (src/gridnet.cpp:383: maskData >= thresh, the mask read as 32-bit integers) as a 0 / 1 float grid.  Rows
// r_first .. r_first + gridDim.x - 1: the halo rows too where a neighbour strip exists (the sweep looks at a contributor's mask).
__global__ void __launch_bounds__(256) k_mask_ok(const int* __restrict__ mask, float* __restrict__ ok, Strip s, int thresh, int r_first) {
  const int r = r_first + (int)blockIdx.x, c = ((int)blockIdx.y * 256 + (int)threadIdx.x) * 4;
  if (c >= s.pitch) return;
  const long long o = s.idx(r, c);
  const int4 m = *reinterpret_cast<const int4*>(mask + o);
  *reinterpret_cast<float4*>(ok + o) = make_float4(m.x >= thresh ? 1.f : 0.f, m.y >= thresh ? 1.f : 0.f, m.z >= thresh ? 1.f : 0.f, m.w >= thresh ? 1.f : 0.f);
}
// Strahler orders of the sweep (float, -1 = never evaluated) -> int16 like the reference's gord partition.  A cell the sweep never
// evaluated keeps gridnet's start value (src/gridnet.cpp:228-233, 269-313): without outlets 1 on every cell with a direction inside
// the mask, -1 elsewhere; with outlets 1 on the cells upstream of an outlet (the nodes the restriction kept), 0 on the other cells
// with a direction, -1 elsewhere.  (A cell can be upstream of an outlet or inside the mask and still never be evaluated: below a
// direction code 0, which counts as a contributor and drains nowhere.)
__global__ void __launch_bounds__(256) k_gord_finish(const float* __restrict__ g, const short* __restrict__ p, const float* __restrict__ ok,
                                                     const unsigned short* __restrict__ node, short* __restrict__ gord, Strip s, short p_nodata,
                                                     int outlets) {
  const int r = 1 + (int)blockIdx.x, c = ((int)blockIdx.y * 256 + (int)threadIdx.x) * 4;
  if (c >= s.pitch) return;
  const long long o = s.idx(r, c);
  const float4 v = *reinterpret_cast<const float4*>(g + o);
  const short4 d = *reinterpret_cast<const short4*>(p + o);
  const ushort4 nw = *reinterpret_cast<const ushort4*>(node + o);
  const float4 m = ok ? *reinterpret_cast<const float4*>(ok + o) : make_float4(1.f, 1.f, 1.f, 1.f);
  const float a[4] = {v.x, v.y, v.z, v.w}, inside[4] = {m.x, m.y, m.z, m.w};
  const short dd[4] = {d.x, d.y, d.z, d.w};
  const unsigned short nn[4] = {nw.x, nw.y, nw.z, nw.w};
  short out[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const bool data = !nd_s(dd[i], p_nodata);
    if (a[i] >= 0.f) out[i] = (short)a[i];
    else if (outlets) out[i] = (nn[i] & 0x8000u) ? 1 : data ? 0 : -1;
    else out[i] = (data && inside[i] != 0.f) ? 1 : -1;
  }
  *reinterpret_cast<short4*>(gord + o) = make_short4(out[0], out[1], out[2], out[3]);
}
}  // namespace

int launch_mask_ok(const int* mask, float* ok, const Strip& s, int thresh, cudaStream_t st) {
  const dim3 grid((unsigned)(s.ny + (s.has_top ? 1 : 0) + (s.has_bot ? 1 : 0)), (unsigned)(((s.pitch >> 2) + 255) / 256));
  k_mask_ok<<<grid, 256, 0, st>>>(mask, ok, s, thresh, s.has_top ? 0 : 1);
  TD_LAUNCHED();
  TD_CUDA(cudaGetLastError());
  return TD_OK;
}
int launch_gord_finish(const float* g, const short* p, const float* ok, const unsigned short* node, short* gord, const Strip& s, short p_nodata,
                       int outlets, cudaStream_t st) {
  const dim3 grid((unsigned)s.ny, (unsigned)(((s.pitch >> 2) + 255) / 256));
  k_gord_finish<<<grid, 256, 0, st>>>(g, p, ok, node, gord, s, p_nodata, outlets);
  TD_LAUNCHED();
  TD_CUDA(cudaGetLastError());
  return TD_OK;
}

int launch_threshold(const float* ssa, const float* mask, short* src, const Strip& s, float thresh, float ssa_nodata, cudaStream_t st) {
  const dim3 grid((unsigned)s.ny, (unsigned)(((s.pitch >> 2) + 255) / 256));
  k_threshold<<<grid, 256, 0, st>>>(ssa, mask, src, s, thresh, ssa_nodata);
  TD_LAUNCHED();
  TD_CUDA(cudaGetLastError());
  return TD_OK;
}
int launch_slopearea(const float* slp, const float* sca, float* sa, const Strip& s, float m, float n, cudaStream_t st) {
  const dim3 grid((unsigned)s.ny, (unsigned)(((s.pitch >> 2) + 255) / 256));
  k_slopearea<<<grid, 256, 0, st>>>(slp, sca, sa, s, m, n);
  TD_LAUNCHED();
  TD_CUDA(cudaGetLastError());
  return TD_OK;
}
int launch_lengtharea(const float* plen, const int* ad8, short* ss, const Strip& s, float m, float y, cudaStream_t st) {
  const dim3 grid((unsigned)s.ny, (unsigned)(((s.pitch >> 2) + 255) / 256));
  k_lengtharea<<<grid, 256, 0, st>>>(plen, ad8, ss, s, m, y);
  TD_LAUNCHED();
  TD_CUDA(cudaGetLastError());
  return TD_OK;
}
int launch_slopearearatio(const float* slp, const float* sca, float* sar, const Strip& s, float sca_nodata, cudaStream_t st) {
  const dim3 grid((unsigned)s.ny, (unsigned)(((s.pitch >> 2) + 255) / 256));
  k_slopearearatio<<<grid, 256, 0, st>>>(slp, sca, sar, s, sca_nodata);
  TD_LAUNCHED();
  TD_CUDA(cudaGetLastError());
  return TD_OK;
}
int launch_twi(const float* slp, const float* sca, float* twi, const Strip& s, float slp_nodata, float sca_nodata, cudaStream_t st) {
  const dim3 grid((unsigned)s.ny, (unsigned)(((s.pitch >> 2) + 255) / 256));
  k_twi<<<grid, 256, 0, st>>>(slp, sca, twi, s, slp_nodata, sca_nodata);
  TD_LAUNCHED();
  TD_CUDA(cudaGetLastError());
  return TD_OK;
}
}  // namespace td
