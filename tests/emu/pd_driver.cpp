// TEST INFRASTRUCTURE ONLY — the Peuker-Douglas stencils (k_pd_smooth, k_pd_mark, peuker.cu) and the point-wise kernels
// (k_lengtharea with its host resolve, k_threshold, k_twi, k_slopearea, k_slopearearatio: pointwise.cu) on the CPU emulation, the
// stencils on one strip or on row strips with the smoothed edge rows exchanged between the two passes like a row-strip caller
// does.  tests/test_stream_definition.py and tests/test_pointwise.py compare the rasters with the restatements cell by cell.
#include <string>
#include <vector>

#include "cuda_runtime.h"
struct int4 { int x, y, z, w; };   // (pointwise.cu's 16-byte integer loads; the emulated runtime does not declare the type)

#include "peuker_emu.inc"    // the transformed kernel sources (written by tests/test_stream_definition.py)
#include "pointwise_emu.inc"

namespace td {
unsigned long long g_launches = 0;
static std::string g_err;
void set_error(const std::string& m) { g_err = m; }
int cuda_fail(cudaError_t, const char* what) { g_err = what; return 90; }
}  // namespace td

using td::Strip;

// nstrips strips of the given heights (rows[0] + ... = ny); each strip holds its rows and the neighbours' edge rows of fel
extern "C" int emu_peukerdouglas(const float* fel, short* ss, int nx, int ny, float nodata, const float* p, int nstrips, const int* rows) {
  const int pitch = (nx + 31) / 32 * 32;
  std::vector<Strip> st(nstrips);
  std::vector<std::vector<float>> f(nstrips), sm(nstrips);
  std::vector<std::vector<short>> o(nstrips);
  std::vector<int> row0(nstrips);
  for (int i = 0, r0 = 0; i < nstrips; r0 += rows[i], ++i) {
    td_strip ts; ts.nx = nx; ts.ny = rows[i]; ts.pitch = pitch; ts.has_top = i > 0; ts.has_bot = i < nstrips - 1;
    st[i] = Strip(ts); row0[i] = r0;
    // padding columns and missing halo rows hold a value the kernels must never use for a decision
    f[i].assign((size_t)st[i].cells(), 12345.f); sm[i].assign((size_t)st[i].cells(), -777.f); o[i].assign((size_t)st[i].cells(), 7);
    for (int r = 0; r <= rows[i] + 1; ++r) {
      const int g = r0 + r - 1;
      if (g < 0 || g >= ny) continue;
      for (int c = 0; c < nx; ++c) f[i][st[i].idx(r, c)] = fel[(size_t)g * nx + c];
    }
  }
  for (int i = 0; i < nstrips; ++i)
    if (td::launch_pd_smooth(f[i].data(), sm[i].data(), st[i], nodata, p, nullptr)) return 1;
  // the smoothed first / last owned rows into the neighbours' halo rows
  for (int i = 0; i < nstrips; ++i) {
    if (i > 0) for (int c = 0; c < pitch; ++c) sm[i][st[i].idx(0, c)] = sm[i - 1][st[i - 1].idx(st[i - 1].ny, c)];
    if (i < nstrips - 1) for (int c = 0; c < pitch; ++c) sm[i][st[i].idx(st[i].ny + 1, c)] = sm[i + 1][st[i + 1].idx(1, c)];
  }
  for (int i = 0; i < nstrips; ++i)
    if (td::launch_pd_mark(sm[i].data(), o[i].data(), st[i], nodata, nullptr)) return 1;
  for (int i = 0; i < nstrips; ++i)
    for (int r = 1; r <= st[i].ny; ++r)
      for (int c = 0; c < nx; ++c) ss[(size_t)(row0[i] + r - 1) * nx + c] = o[i][st[i].idx(r, c)];
  return 0;
}

// the point-wise kernels on one strip of an nx x ny grid: dense rasters in and out, the padding columns filled with pad
static Strip one_strip(int nx, int ny) {
  td_strip ts; ts.nx = nx; ts.ny = ny; ts.pitch = (nx + 31) / 32 * 32; ts.has_top = 0; ts.has_bot = 0;
  return Strip(ts);
}
template <typename T> static std::vector<T> to_strip(const T* g, const Strip& s, T pad) {
  std::vector<T> v((size_t)s.cells(), pad);
  if (g)
    for (int r = 1; r <= s.ny; ++r)
      for (int c = 0; c < s.nx; ++c) v[s.idx(r, c)] = g[(size_t)(r - 1) * s.nx + c];
  return v;
}
template <typename T> static void from_strip(const std::vector<T>& v, const Strip& s, T* g) {
  for (int r = 1; r <= s.ny; ++r)
    for (int c = 0; c < s.nx; ++c) g[(size_t)(r - 1) * s.nx + c] = v[s.idx(r, c)];
}

static td_ctx::Buf g_pend;
// n_pend: how many cells the kernel left to the host (the count of the last run)
extern "C" int emu_lengtharea(const float* plen, const int* ad8, short* ss, int nx, int ny, float m, float y, unsigned* n_pend) {
  const Strip s = one_strip(nx, ny);
  std::vector<float> l = to_strip(plen, s, 0.f);
  std::vector<int> a = to_strip(ad8, s, 0);
  std::vector<short> o((size_t)s.cells(), 7);
  if (td::launch_lengtharea(l.data(), a.data(), o.data(), s, m, y, nullptr, &g_pend)) return 1;
  if (n_pend) *n_pend = *g_pend.as<unsigned>();
  from_strip(o, s, ss);
  return 0;
}
extern "C" int emu_threshold(const float* ssa, const float* mask, short* src, int nx, int ny, float thresh, float nodata) {
  const Strip s = one_strip(nx, ny);
  std::vector<float> v = to_strip(ssa, s, 0.f), mk = to_strip(mask, s, 0.f);
  std::vector<short> o((size_t)s.cells(), 7);
  if (td::launch_threshold(v.data(), mask ? mk.data() : nullptr, o.data(), s, thresh, nodata, nullptr)) return 1;
  from_strip(o, s, src);
  return 0;
}
// which: 0 twi (a, b = the slope's and the area's nodata), 1 slopearea (a, b = m, n), 2 slopearearatio (a = the area's nodata)
extern "C" int emu_slp_sca(int which, const float* slp, const float* sca, float* out, int nx, int ny, float a, float b) {
  const Strip s = one_strip(nx, ny);
  std::vector<float> sl = to_strip(slp, s, 1.f), ar = to_strip(sca, s, 1.f), o((size_t)s.cells(), 7.f);
  const int rc = which == 0 ? td::launch_twi(sl.data(), ar.data(), o.data(), s, a, b, nullptr, &g_pend)
               : which == 1 ? td::launch_slopearea(sl.data(), ar.data(), o.data(), s, a, b, nullptr, &g_pend)
                            : td::launch_slopearearatio(sl.data(), ar.data(), o.data(), s, a, nullptr);
  if (rc) return 1;
  from_strip(o, s, out);
  return 0;
}
