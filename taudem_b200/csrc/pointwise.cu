// Point-wise consumers of the contributing-area rasters (SURVEY.md section 8 (f) rank 4):
//   threshold  src = (ssa >= thresh [& mask >= 0]) ? 1 : 0, nodata where ssa is nodata   (src/Threshold.cpp:109-131)
//   twi        twi = ln(sca / slp) where both are data and positive, else nodata (-1)     (src/TWI.cpp:108-124)
//   slopearea  sa = slp^m * sca^n where slp >= 0 and sca >= 0, else nodata (-1)            (src/SlopeArea.cpp:114-125)
//   slopearearatio  sar = slp / sca where sca is data, else nodata (-1)                    (src/SlopeAreaRatio.cpp:107-118)
//   lengtharea ss = ad8 >= M plen^y ? 1 : 0 where plen >= 0, else nodata (-32768)          (src/LengthArea.cpp:110-120)
// One streaming kernel each, four cells per thread (16-byte loads, 8 / 16-byte stores): 6 B (10 with a mask) and 12 B of HBM
// traffic per cell.  Device-strip level entry points take strips like every other kernel of the path; the host-grid level
// copies dense arrays in and out.  isNodata is linearpart's |v - nodata| < 1e-5 (src/linearpart.h:471-483).
#include <math.h>

#include <vector>

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

// Cells a kernel leaves to the host (pointwise_resolve): the strip offset and the operands; the host writes its result into a
struct FPending { long long off; float a, b; };
// d, a double within 8 ulps of the exact value, rounds to the same float as the exact value unless it lies within 8 ulps of a
// midpoint between two floats (or of the overflow threshold FLT_MAX + half an ulp, between FLT_MAX and 2^128)
__device__ __forceinline__ bool rounding_unsure(double d) {
  const double a = fabs(d);
  if (!(a <= (double)FLT_MAX)) return a <= 0x1p128;
  const float f = (float)d;
  const double lo = 0.5 * ((double)f + (double)nextafterf(f, -INFINITY)), hi = 0.5 * ((double)f + (double)nextafterf(f, INFINITY));
  const double tol = 8.0 * fmax(a * 0x1p-52, 0x1p-1074);
  return fabs(d - lo) <= tol || fabs(d - hi) <= tol;
}
// ln of a float quotient, correctly rounded: the double logarithm rounded to float where that is sure to be the correctly rounded
// result; the rest (CUDA's double log is within 1 ulp, and 5 of the 2^31 positive floats round the wrong way from it) go to the
// host, which rounds logl once.  The reference's log(float) is glibc's logf, which is not correctly rounded on 416 908 of the
// 2 139 095 039 positive finite floats (glibc 2.39): there, and only there, the two differ, by one ulp (tests/test_gpu_pointwise.py
// sweeps every positive float and counts both sets on the host it runs on).
__global__ void __launch_bounds__(256) k_twi(const float* __restrict__ slp, const float* __restrict__ sca, float* __restrict__ twi, Strip s,
                                             float slp_nodata, float sca_nodata, FPending* __restrict__ pend, unsigned* __restrict__ npend,
                                             unsigned cap) {
  const int r = 1 + (int)blockIdx.x, c = ((int)blockIdx.y * 256 + (int)threadIdx.x) * 4;
  if (c >= s.pitch) return;
  const long long o = s.idx(r, c);
  const float4 sv = *reinterpret_cast<const float4*>(slp + o), av = *reinterpret_cast<const float4*>(sca + o);
  const float sl[4] = {sv.x, sv.y, sv.z, sv.w}, ar[4] = {av.x, av.y, av.z, av.w};
  float out[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const bool ok = !nd_f(ar[i], sca_nodata) && !nd_f(sl[i], slp_nodata) && sl[i] > 0.0f && ar[i] > 0.0f;
    const float q = ar[i] / sl[i];
    const double d = log((double)q);
    out[i] = ok ? (float)d : -1.0f;
    if (ok && rounding_unsure(d) && c + i < s.nx) {
      const unsigned k = atomicAdd(npend, 1u);
      if (k < cap) pend[k] = FPending{o + i, q, 0.f};
    }
  }
  *reinterpret_cast<float4*>(twi + o) = make_float4(out[0], out[1], out[2], out[3]);
}
// slp^m * sca^n: the reference multiplies two powf results as floats (std::pow(float, float), src/SlopeArea.cpp:119); here each power
// is correctly rounded (pow_float, or on the host where the double pow is too close to a midpoint), then the same float product.
// glibc 2.39's powf is not correctly rounded on 774 403 positive floats at the exponent 2, 1 361 091 at 0.5 and 1 047 797 at 1.3
// (of 2 139 095 039); the results differ by one ulp exactly where one of the two powers does, the nodata masks never.
// x^e as a float: exact for the exponents 1 and 2 (the reference's defaults: slope^2 * area^1; the double square is exact, then
// rounded once), the double root rounded to float for 0.5 (correctly rounded: 53 >= 2 * 24 + 2; + 0 makes -0^0.5 +0 like powf,
// -inf^0.5 is +inf), the double pow rounded to float otherwise (two orders of magnitude more instructions; *unsure when it may not
// be the correctly rounded float: CUDA's double pow is within 2 ulps).
__device__ __forceinline__ float pow_float(float x, float e, bool* unsure = nullptr) {
  if (e == 1.0f) return x;
  if (e == 2.0f) return (float)((double)x * (double)x);
  if (e == 0.5f) return x == -INFINITY ? INFINITY : (float)sqrt((double)x) + 0.0f;
  const double d = pow((double)x, (double)e);
  if (unsure) *unsure = rounding_unsure(d);
  return (float)d;
}
// the host's pow_float: powl rounded once where the device uses the double pow
static float pow_float_host(float x, float e) {
  if (e == 1.0f) return x;
  if (e == 2.0f) return (float)((double)x * (double)x);
  if (e == 0.5f) return x == -INFINITY ? INFINITY : (float)sqrt((double)x) + 0.0f;
  return (float)powl((long double)x, (long double)e);
}
__global__ void __launch_bounds__(256) k_slopearea(const float* __restrict__ slp, const float* __restrict__ sca, float* __restrict__ sa, Strip s,
                                                   float m, float n, FPending* __restrict__ pend, unsigned* __restrict__ npend, unsigned cap) {
  const int r = 1 + (int)blockIdx.x, c = ((int)blockIdx.y * 256 + (int)threadIdx.x) * 4;
  if (c >= s.pitch) return;
  const long long o = s.idx(r, c);
  const float4 sv = *reinterpret_cast<const float4*>(slp + o), av = *reinterpret_cast<const float4*>(sca + o);
  const float sl[4] = {sv.x, sv.y, sv.z, sv.w}, ar[4] = {av.x, av.y, av.z, av.w};
  float out[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const bool ok = sl[i] >= 0.0f && ar[i] >= 0.0f;
    bool u1 = false, u2 = false;
    out[i] = ok ? pow_float(sl[i], m, &u1) * pow_float(ar[i], n, &u2) : -1.0f;
    if (ok && (u1 || u2) && c + i < s.nx) {
      const unsigned k = atomicAdd(npend, 1u);
      if (k < cap) pend[k] = FPending{o + i, sl[i], ar[i]};
    }
  }
  *reinterpret_cast<float4*>(sa + o) = make_float4(out[0], out[1], out[2], out[3]);
}
// lengtharea (src/LengthArea.cpp:110-120): ss = ((float)ad8 >= M * powf(plen, y)) ? 1 : 0 where plen >= 0, else nodata (-32768); ad8
// is the contributing area read as 32-bit integers and M * powf(plen, y) one float product.  That is a decision on glibc's powf,
// which is not correctly rounded on about a million floats per exponent: with a correctly rounded power it flips on 35 371 plen
// values in [1, 2^31) at the defaults (M = 0.03, y = 1.3), e.g. plen = 0x1.1065fap+11, ad8 = 656.  So the kernel decides a cell
// only where the decision cannot depend on the power's last bit: glibc's powf is faithful (within 0.82 ulp: one of the two floats
// around the exact power, tests/test_pointwise.py checks every positive float at the tested exponents), so is g = pow_float, so
// powf lies in [prev(g), next(g)], and (float)ad8 >= M * p is monotone in p for any M (a float product with a fixed factor is
// monotone; with M = 0 the NaN of 0 * +-inf only changes the decision at the ends of the float line, one step from the finite
// values) — where prev(g) and next(g) decide alike, powf decides the same.  That
// covers the special values too: NaN powers (never >=), powers 0 and +-inf (their neighbours are -+denormal and +-FLT_MAX), M <= 0
// or NaN.  The other cells (none on most rasters) go to a list that launch_lengtharea decides on the host with libm's powf, the
// function the reference calls.  10 B of HBM traffic per cell.
struct LaPending { long long off; float plen; int ad8; };      // ad8: the cell's value once decided on the host
__global__ void __launch_bounds__(256) k_lengtharea(const float* __restrict__ plen, const int* __restrict__ ad8, short* __restrict__ ss, Strip s,
                                                    float m, float y, LaPending* __restrict__ pend, unsigned* __restrict__ npend, unsigned cap) {
  const int r = 1 + (int)blockIdx.x, c = ((int)blockIdx.y * 256 + (int)threadIdx.x) * 4;
  if (c >= s.pitch) return;
  const long long o = s.idx(r, c);
  const float4 lv = *reinterpret_cast<const float4*>(plen + o);
  const int4 av = *reinterpret_cast<const int4*>(ad8 + o);
  const float l[4] = {lv.x, lv.y, lv.z, lv.w};
  const int a[4] = {av.x, av.y, av.z, av.w};
  short out[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float g = pow_float(l[i], y), fa = (float)a[i];
    const bool lo = fa >= m * nextafterf(g, -INFINITY), hi = fa >= m * nextafterf(g, INFINITY);
    out[i] = l[i] >= 0.0f ? (short)(lo ? 1 : 0) : TD_MISSINGSHORT;
    if (l[i] >= 0.0f && lo != hi && c + i < s.nx) {                  // (not the padding columns)
      const unsigned k = atomicAdd(npend, 1u);
      if (k < cap) pend[k] = LaPending{o + i, l[i], a[i]};
    }
  }
  *reinterpret_cast<short4*>(ss + o) = make_short4(out[0], out[1], out[2], out[3]);
}
__global__ void __launch_bounds__(256) k_lengtharea_patch(const LaPending* __restrict__ pend, unsigned n, short* __restrict__ ss) {
  const unsigned k = blockIdx.x * 256 + threadIdx.x;
  if (k < n) ss[pend[k].off] = (short)pend[k].ad8;
}
__global__ void __launch_bounds__(256) k_float_patch(const FPending* __restrict__ pend, unsigned n, float* __restrict__ out) {
  const unsigned k = blockIdx.x * 256 + threadIdx.x;
  if (k < n) out[pend[k].off] = pend[k].a;
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
// A kernel that leaves cells to the host, run to completion.  pend holds a count (its first 16 bytes) and a list of entries E (a
// caller without a context's buffer passes nullptr: the call then allocates one and frees it at the end); run launches the kernel
// with (list, count, capacity), decide computes an entry's result on the host, patch launches the kernel that writes the results.
// Synchronises st to read the count, which is 0 on most rasters.  A list that overflowed is grown and the kernel run again (it
// writes the same cells).
template <typename E, typename Run, typename Decide, typename Patch>
static int run_with_host_cells(td_ctx::Buf* pend_or_null, cudaStream_t st, Run run, Decide decide, Patch patch) {
  struct Own { td_ctx::Buf b; ~Own() { b.release(); } } own;
  td_ctx::Buf& pend = pend_or_null ? *pend_or_null : own.b;
  unsigned n = 0;
  for (unsigned cap = pend.cap > 16 ? (unsigned)((pend.cap - 16) / sizeof(E)) : 0u;;) {
    if (cap < 1024 || n > cap) {
      cap = n > 1024 ? n : 1024;
      TD_CUDA(pend.ensure(16 + (size_t)cap * sizeof(E)));
    }
    unsigned* d_n = pend.as<unsigned>();
    E* list = reinterpret_cast<E*>(pend.as<char>() + 16);
    TD_CUDA(cudaMemsetAsync(d_n, 0, sizeof(unsigned), st));
    run(list, d_n, cap);
    TD_LAUNCHED();
    TD_CUDA(cudaGetLastError());
    TD_CUDA(cudaMemcpyAsync(&n, d_n, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    TD_CUDA(cudaStreamSynchronize(st));
    if (n == 0) return TD_OK;
    if (n > cap) continue;
    std::vector<E> h(n);
    TD_CUDA(cudaMemcpyAsync(h.data(), list, n * sizeof(E), cudaMemcpyDeviceToHost, st));
    TD_CUDA(cudaStreamSynchronize(st));
    for (E& e : h) decide(e);
    TD_CUDA(cudaMemcpyAsync(list, h.data(), n * sizeof(E), cudaMemcpyHostToDevice, st));
    patch(list, n);
    TD_LAUNCHED();
    TD_CUDA(cudaGetLastError());
    TD_CUDA(cudaStreamSynchronize(st));
    return TD_OK;
  }
}
// the cells whose double pow may not round to the correctly rounded float: both powers again with powl (pow_float_host)
int launch_slopearea(const float* slp, const float* sca, float* sa, const Strip& s, float m, float n, cudaStream_t st, td_ctx::Buf* pend) {
  const dim3 grid((unsigned)s.ny, (unsigned)(((s.pitch >> 2) + 255) / 256));
  return run_with_host_cells<FPending>(
      pend, st, [&](FPending* list, unsigned* cnt, unsigned cap) { k_slopearea<<<grid, 256, 0, st>>>(slp, sca, sa, s, m, n, list, cnt, cap); },
      [&](FPending& e) { e.a = pow_float_host(e.a, m) * pow_float_host(e.b, n); },
      [&](const FPending* list, unsigned cnt) { k_float_patch<<<(cnt + 255) / 256, 256, 0, st>>>(list, cnt, sa); });
}
// the cells whose decision depends on the last bit of the power: decided with libm's powf, like the reference
int launch_lengtharea(const float* plen, const int* ad8, short* ss, const Strip& s, float m, float y, cudaStream_t st, td_ctx::Buf* pend) {
  const dim3 grid((unsigned)s.ny, (unsigned)(((s.pitch >> 2) + 255) / 256));
  return run_with_host_cells<LaPending>(
      pend, st, [&](LaPending* list, unsigned* cnt, unsigned cap) { k_lengtharea<<<grid, 256, 0, st>>>(plen, ad8, ss, s, m, y, list, cnt, cap); },
      [&](LaPending& e) { e.ad8 = (float)e.ad8 >= m * powf(e.plen, y) ? 1 : 0; },
      [&](const LaPending* list, unsigned cnt) { k_lengtharea_patch<<<(cnt + 255) / 256, 256, 0, st>>>(list, cnt, ss); });
}
int launch_slopearearatio(const float* slp, const float* sca, float* sar, const Strip& s, float sca_nodata, cudaStream_t st) {
  const dim3 grid((unsigned)s.ny, (unsigned)(((s.pitch >> 2) + 255) / 256));
  k_slopearearatio<<<grid, 256, 0, st>>>(slp, sca, sar, s, sca_nodata);
  TD_LAUNCHED();
  TD_CUDA(cudaGetLastError());
  return TD_OK;
}
// the cells whose double log may not round to the correctly rounded float: logl rounded once
int launch_twi(const float* slp, const float* sca, float* twi, const Strip& s, float slp_nodata, float sca_nodata, cudaStream_t st, td_ctx::Buf* pend) {
  const dim3 grid((unsigned)s.ny, (unsigned)(((s.pitch >> 2) + 255) / 256));
  return run_with_host_cells<FPending>(
      pend, st, [&](FPending* list, unsigned* cnt, unsigned cap) { k_twi<<<grid, 256, 0, st>>>(slp, sca, twi, s, slp_nodata, sca_nodata, list, cnt, cap); },
      [&](FPending& e) { e.a = (float)logl((long double)e.a); },
      [&](const FPending* list, unsigned cnt) { k_float_patch<<<(cnt + 255) / 256, 256, 0, st>>>(list, cnt, twi); });
}
}  // namespace td
