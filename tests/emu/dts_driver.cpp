// TEST INFRASTRUCTURE ONLY — the BFS kernels of d8hdisttostrm / d8vdisttostrm (k_dts_seed, k_dts_level, k_dts_edge: disttostrm.cu)
// on the CPU emulation, through the product's host functions td::dts_seed / td::dts_levels, on one strip or on row strips with the
// rounds a row-strip caller makes: levels until every frontier is empty, the value raster's first / last owned rows into the
// neighbours' halo rows, again until no strip added a cell.  tests/test_disttostrm.py compares the distances with the C restatement
// cell by cell.
#include <math.h>

#include <string>
#include <vector>

#include "cuda_runtime.h"
// (what disttostrm.cu uses beyond the emulated runtime: the round-to-nearest float intrinsics)
inline float __fadd_rn(float a, float b) { return a + b; }
inline float __fsub_rn(float a, float b) { return a - b; }

#include "disttostrm_emu.inc"    // the transformed kernel source (written by tests/test_disttostrm.py)

namespace td {
unsigned long long g_launches = 0;
static std::string g_err;
void set_error(const std::string& m) { g_err = m; }
int cuda_fail(cudaError_t, const char* what) { g_err = what; return 90; }
void gridnet_dist_table(const double* dxc, const double* dyc, int ny, float* dist) {   // (capi.cu's, restated)
  static const int d1[9] = {0, 1, 1, 0, -1, -1, -1, 0, 1}, d2[9] = {0, 0, -1, -1, -1, 0, 1, 1, 1};
  for (int m = 0; m < ny; ++m)
    for (int k = 1; k <= 8; ++k) dist[(size_t)m * 8 + k - 1] = (float)sqrt(dxc[m] * dxc[m] * d1[k] * d1[k] + dyc[m] * dyc[m] * d2[k] * d2[k]);
}
}  // namespace td

using td::Strip;

// nstrips strips of the given heights (rows[0] + ... = ny); grid = blocks per level launch; *rounds = the rounds run
extern "C" int emu_disttostrm(int vertical, const short* p, const float* fel, const int* src, float* out, int nx, int ny, short p_nodata, int src_nodata,
                              int thresh, const double* dxc, const double* dyc, int nstrips, const int* rows, unsigned seed, int grid, int* rounds) {
  emu::g_rng = seed * 2654435761ull + 1;
  const int pitch = (nx + 31) / 32 * 32;
  std::vector<Strip> st(nstrips);
  std::vector<std::vector<float>> f(nstrips), val(nstrips), dist(nstrips);
  std::vector<std::vector<short>> pp(nstrips);
  std::vector<std::vector<int>> ss(nstrips);
  std::vector<std::vector<unsigned char>> code(nstrips);
  std::vector<std::vector<unsigned>> list(nstrips);
  std::vector<std::vector<unsigned long long>> ctr(nstrips), bounds(nstrips);
  std::vector<td::DtsBufs> B(nstrips);
  std::vector<int> row0(nstrips);
  for (int i = 0, r0 = 0; i < nstrips; r0 += rows[i], ++i) {
    td_strip ts; ts.nx = nx; ts.ny = rows[i]; ts.pitch = pitch; ts.has_top = i > 0; ts.has_bot = i < nstrips - 1;
    st[i] = Strip(ts); row0[i] = r0;
    const size_t n = (size_t)st[i].cells();
    // padding columns and missing halo rows hold values the kernels must never use
    f[i].assign(n, 12345.f); pp[i].assign(n, 1); ss[i].assign(n, thresh); val[i].assign(n, -777.f); code[i].assign(n, 9);
    list[i].assign(n, 0xdeadbeefu); ctr[i].assign(2, 77); bounds[i].assign(td::DTS_BATCH + 3, 77);
    for (int r = 0; r <= rows[i] + 1; ++r) {
      const int g = r0 + r - 1;
      if (g < 0 || g >= ny) continue;
      for (int c = 0; c < nx; ++c) {
        const size_t k = st[i].idx(r, c), gk = (size_t)g * nx + c;
        f[i][k] = fel[gk]; pp[i][k] = p[gk]; ss[i][k] = src[gk];
      }
    }
    dist[i].resize((size_t)rows[i] * 8);
    td::gridnet_dist_table(dxc + r0, dyc + r0, rows[i], dist[i].data());
    B[i] = td::DtsBufs{list[i].data(), ctr[i].data(), bounds[i].data(), reinterpret_cast<unsigned*>(bounds[i].data() + td::DTS_BATCH + 2)};
    if (td::dts_seed(pp[i].data(), ss[i].data(), val[i].data(), code[i].data(), st[i], thresh, p_nodata, src_nodata, B[i], nullptr)) return 1;
  }
  int nr = 0;
  for (;;) {
    unsigned long long any = 0;
    for (int i = 0; i < nstrips; ++i) {
      unsigned long long cells = 0;
      long long levels = 0;
      if (td::dts_levels(vertical != 0, code[i].data(), f[i].data(), dist[i].data(), val[i].data(), st[i], B[i], grid, &cells, &levels, nullptr)) return 1;
      any += cells;
    }
    ++nr;
    // the first / last owned rows of every strip's values into the neighbours' halo rows
    for (int i = 0; i < nstrips; ++i) {
      if (i > 0)
        for (int c = 0; c < pitch; ++c) val[i][st[i].idx(0, c)] = val[i - 1][st[i - 1].idx(st[i - 1].ny, c)];
      if (i < nstrips - 1)
        for (int c = 0; c < pitch; ++c) val[i][st[i].idx(st[i].ny + 1, c)] = val[i + 1][st[i + 1].idx(1, c)];
    }
    if (!any) break;
  }
  if (rounds) *rounds = nr;
  for (int i = 0; i < nstrips; ++i)
    for (int r = 1; r <= st[i].ny; ++r)
      for (int c = 0; c < nx; ++c) out[(size_t)(row0[i] + r - 1) * nx + c] = val[i][st[i].idx(r, c)];
  return 0;
}
