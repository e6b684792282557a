// TEST INFRASTRUCTURE ONLY — the Peuker-Douglas stencils (k_pd_smooth, k_pd_mark, peuker.cu) and k_lengtharea (pointwise.cu) on the
// CPU emulation, on one strip or on row strips with the smoothed edge rows exchanged between the two passes like a row-strip
// caller does.  tests/test_stream_definition.py compares the rasters with the restatements bit for bit.
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

extern "C" int emu_lengtharea(const float* plen, const int* ad8, short* ss, int nx, int ny, float m, float y) {
  td_strip ts; ts.nx = nx; ts.ny = ny; ts.pitch = (nx + 31) / 32 * 32; ts.has_top = 0; ts.has_bot = 0;
  const Strip s(ts);
  std::vector<float> l((size_t)s.cells(), 0.f);
  std::vector<int> a((size_t)s.cells(), 0);
  std::vector<short> o((size_t)s.cells(), 0);
  for (int r = 1; r <= ny; ++r)
    for (int c = 0; c < nx; ++c) { l[s.idx(r, c)] = plen[(size_t)(r - 1) * nx + c]; a[s.idx(r, c)] = ad8[(size_t)(r - 1) * nx + c]; }
  if (td::launch_lengtharea(l.data(), a.data(), o.data(), s, m, y, nullptr)) return 1;
  for (int r = 1; r <= ny; ++r)
    for (int c = 0; c < nx; ++c) ss[(size_t)(r - 1) * nx + c] = o[s.idx(r, c)];
  return 0;
}
