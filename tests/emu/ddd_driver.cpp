// TEST INFRASTRUCTURE ONLY — the level kernels of dinfdistdown (k_ddd_seed, k_ddd_level, k_ddd_edge, k_ddd_pyth: dinfdistdown.cu) on
// the CPU emulation, through the product's host functions td::ddd_seed / ddd_levels / ddd_edge / ddd_pythagoras, on one strip or on row
// strips with the rounds a row-strip caller makes: levels until every frontier is empty, the decrements of the halo-row donors and the
// value rasters' first / last owned rows to the neighbours, the received decrements into ddd_edge, again until no strip handed a
// decrement over.  tests/test_dinfdistdown.py compares the distances with the C restatement cell by cell.
#include <math.h>

#include <string>
#include <vector>

#include "cuda_runtime.h"
// (what dinfdistdown.cu uses beyond the emulated runtime: the round-to-nearest intrinsics; the host's IEEE arithmetic is the same)
inline float __fadd_rn(float a, float b) { return a + b; }
inline float __fsub_rn(float a, float b) { return a - b; }
inline float __fmul_rn(float a, float b) { return a * b; }
inline float __fdiv_rn(float a, float b) { return a / b; }
inline float __fsqrt_rn(float a) { return sqrtf(a); }
inline double __dadd_rn(double a, double b) { return a + b; }
inline double __dmul_rn(double a, double b) { return a * b; }
inline float __double2float_rn(double a) { return (float)a; }

#include "dinfdistdown_emu.inc"    // the transformed kernel source (written by tests/test_dinfdistdown.py)

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

// nstrips strips of the given heights (rows[0] + ... = ny); grid = blocks per level launch; *levels = the levels run (summed over the
// strips and rounds); *rounds = the rounds run
extern "C" int emu_dinfdistdown(const float* ang, const float* fel, const float* w, const short* src, float* out, int nx, int ny, float ang_nodata,
                                float fel_nodata, float w_nodata, const double* dxc, const double* dyc, int statmethod, int typemethod, int concheck,
                                int nstrips, const int* rows, unsigned seed, int grid, long long* levels, int* rounds) {
  emu::g_rng = seed * 2654435761ull + 1;
  const int pitch = (nx + 31) / 32 * 32;
  const bool p_mode = typemethod == 2;
  std::vector<Strip> st(nstrips);
  std::vector<std::vector<float>> a(nstrips), f(nstrips), ww(nstrips), val(nstrips), val2(nstrips), dist(nstrips);
  std::vector<std::vector<double>> th(nstrips);
  std::vector<std::vector<short>> ss(nstrips);
  std::vector<std::vector<unsigned char>> state(nstrips);
  std::vector<std::vector<int>> halo(nstrips);
  std::vector<std::vector<unsigned>> list(nstrips);
  std::vector<std::vector<unsigned long long>> ctr(nstrips), bounds(nstrips);
  std::vector<td::DtsBufs> B(nstrips);
  std::vector<td::DddArgs> A(nstrips);
  std::vector<int> row0(nstrips);
  for (int i = 0, r0 = 0; i < nstrips; r0 += rows[i], ++i) {
    td_strip ts; ts.nx = nx; ts.ny = rows[i]; ts.pitch = pitch; ts.has_top = i > 0; ts.has_bot = i < nstrips - 1;
    const Strip& s = st[i] = Strip(ts);
    row0[i] = r0;
    const size_t n = (size_t)s.cells();
    // padding columns and missing halo rows hold values the kernels must never use
    a[i].assign(n, 1.0f); f[i].assign(n, 12345.f); ww[i].assign(n, 3.0f); val[i].assign(n, -777.f); val2[i].assign(n, -777.f);
    ss[i].assign(n, 1); state[i].assign(n, 0x29); halo[i].assign(2 * (size_t)pitch, 0);
    list[i].assign(n, 0xdeadbeefu); ctr[i].assign(2, 77); bounds[i].assign(td::DTS_BATCH + 3, 77);
    for (int r = 0; r <= s.ny + 1; ++r) {
      const int g = r0 + r - 1;
      if (g < 0 || g >= ny) continue;
      for (int c = 0; c < nx; ++c) {
        const size_t k = s.idx(r, c), gk = (size_t)g * nx + c;
        a[i][k] = ang[gk]; ss[i][k] = src[gk];
        if (fel) f[i][k] = fel[gk];
        if (w) ww[i][k] = w[gk];
      }
    }
    // the strip's row angles, the neighbours' edge rows with their own cell sizes (capi.cu upload_theta_from_host)
    th[i].resize(2 * (size_t)s.ny + 2);
    for (int j = 0; j < s.ny; ++j) { th[i][j] = atan2(dyc[r0 + j], dxc[r0 + j]); th[i][s.ny + j] = atan2(dxc[r0 + j], dyc[r0 + j]); }
    th[i][2 * (size_t)s.ny] = r0 > 0 ? atan2(dyc[r0 - 1], dxc[r0 - 1]) : th[i][0];
    th[i][2 * (size_t)s.ny + 1] = r0 + s.ny < ny ? atan2(dyc[r0 + s.ny], dxc[r0 + s.ny]) : th[i][s.ny - 1];
    dist[i].resize((size_t)s.ny * 8);
    td::gridnet_dist_table(dxc + r0, dyc + r0, s.ny, dist[i].data());
    B[i] = td::DtsBufs{list[i].data(), ctr[i].data(), bounds[i].data(), reinterpret_cast<unsigned*>(bounds[i].data() + td::DTS_BATCH + 2)};
    A[i] = td::DddArgs{a[i].data(), f[i].data(), w ? ww[i].data() : nullptr, dist[i].data(), th[i].data(), val[i].data(), p_mode ? val2[i].data() : nullptr,
                       state[i].data(), nstrips > 1 ? halo[i].data() : nullptr, fel_nodata, w_nodata, concheck == 1};
    if (td::ddd_seed(a[i].data(), ss[i].data(), ang_nodata, A[i], s, B[i], nullptr)) return 1;
  }
  long long nlev = 0;
  int nr = 0;
  for (;;) {
    for (int i = 0; i < nstrips; ++i) {
      std::fill(halo[i].begin(), halo[i].end(), 0);
      long long lv = 0;
      if (td::ddd_levels(typemethod, statmethod, A[i], st[i], B[i], grid, nullptr, &lv, nullptr)) return 1;
      nlev += lv;
    }
    ++nr;
    // the first / last owned rows of every strip's values into the neighbours' halo rows
    for (int i = 0; i < nstrips; ++i)
      for (std::vector<std::vector<float>>* v : {&val, &val2}) {
        if (i > 0)
          for (int c = 0; c < pitch; ++c) (*v)[i][st[i].idx(0, c)] = (*v)[i - 1][st[i - 1].idx(st[i - 1].ny, c)];
        if (i < nstrips - 1)
          for (int c = 0; c < pitch; ++c) (*v)[i][st[i].idx(st[i].ny + 1, c)] = (*v)[i + 1][st[i + 1].idx(1, c)];
      }
    long long handed = 0;
    for (int i = 0; i < nstrips; ++i)
      for (int v : halo[i]) handed += v;
    if (!handed) break;
    for (int i = 0; i < nstrips; ++i)
      if (td::ddd_edge(state[i].data(), i > 0 ? halo[i - 1].data() + pitch : nullptr, i < nstrips - 1 ? halo[i + 1].data() : nullptr, st[i], B[i], nullptr))
        return 1;
  }
  for (int i = 0; i < nstrips; ++i) {
    if (p_mode && td::ddd_pythagoras(val[i].data(), val2[i].data(), st[i], nullptr)) return 1;
    for (int r = 1; r <= st[i].ny; ++r)
      for (int c = 0; c < nx; ++c) out[(size_t)(row0[i] + r - 1) * nx + c] = val[i][st[i].idx(r, c)];
  }
  if (levels) *levels = nlev;
  if (rounds) *rounds = nr;
  return 0;
}
