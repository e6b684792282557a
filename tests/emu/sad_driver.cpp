// TEST INFRASTRUCTURE ONLY — slopeavedown's kernels (k_sad_init, k_sad_pass: slopeavedown.cu) on the CPU emulation, on one strip or
// on row strips with the state's edge rows exchanged after every pass like a row-strip caller does.  The processed cells (the D8
// sweep's count byte 0xFE on the GPU) come in as a mask from the caller.  tests/test_slopeavedown.py compares the slopes with the C
// restatement cell by cell.
#include <math.h>

#include <string>
#include <vector>

#include "cuda_runtime.h"
// (what slopeavedown.cu uses beyond the emulated runtime: 8-byte pairs and the round-to-nearest float intrinsics)
struct float2 { float x, y; };
inline float2 make_float2(float a, float b) { return {a, b}; }
inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
inline float __fadd_rn(float a, float b) { return a + b; }
inline float __fsub_rn(float a, float b) { return a - b; }
inline float __fdiv_rn(float a, float b) { return a / b; }

#include "slopeavedown_emu.inc"    // the transformed kernel source (written by tests/test_slopeavedown.py)

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

// nstrips strips of the given heights (rows[0] + ... = ny); *passes = the passes run before one changed nothing (or niter)
extern "C" int emu_slopeavedown(const float* fel, const short* p, const unsigned char* processed, float* sd, int nx, int ny, float fel_nodata,
                                short p_nodata, const double* dxc, const double* dyc, double dn, int niter, int nstrips, const int* rows, int* passes) {
  const int pitch = (nx + 31) / 32 * 32;
  std::vector<Strip> st(nstrips);
  std::vector<std::vector<float>> f(nstrips), s0(nstrips), s1(nstrips), o(nstrips), dist(nstrips);
  std::vector<std::vector<short>> pp(nstrips);
  std::vector<std::vector<unsigned char>> cnt(nstrips), code(nstrips);
  std::vector<int> row0(nstrips);
  for (int i = 0, r0 = 0; i < nstrips; r0 += rows[i], ++i) {
    td_strip ts; ts.nx = nx; ts.ny = rows[i]; ts.pitch = pitch; ts.has_top = i > 0; ts.has_bot = i < nstrips - 1;
    st[i] = Strip(ts); row0[i] = r0;
    const size_t n = (size_t)st[i].cells();
    // padding columns and missing halo rows hold values the kernels must never use
    f[i].assign(n, 12345.f); pp[i].assign(n, 1); cnt[i].assign(n, 0xFE); code[i].assign(n, 9);
    s0[i].assign(2 * n, -777.f); s1[i].assign(2 * n, -777.f); o[i].assign(n, -777.f);
    for (int r = 0; r <= rows[i] + 1; ++r) {
      const int g = r0 + r - 1;
      if (g < 0 || g >= ny) continue;
      for (int c = 0; c < nx; ++c) {
        const size_t k = st[i].idx(r, c), gk = (size_t)g * nx + c;
        f[i][k] = fel[gk]; pp[i][k] = p[gk]; cnt[i][k] = processed[gk] ? 0xFE : 0x03;
      }
    }
    dist[i].resize((size_t)rows[i] * 8);
    td::gridnet_dist_table(dxc + r0, dyc + r0, rows[i], dist[i].data());
  }
  for (int i = 0; i < nstrips; ++i)
    if (td::launch_sad_init(pp[i].data(), cnt[i].data(), f[i].data(), code[i].data(), s0[i].data(), s1[i].data(), o[i].data(), st[i], p_nodata,
                            fel_nodata, nullptr))
      return 1;
  int it = 0;
  for (; it < niter; ++it) {
    int any = 0;
    for (int i = 0; i < nstrips; ++i) {
      int changed = 0;
      float* in = (it & 1) ? s1[i].data() : s0[i].data();
      float* out = (it & 1) ? s0[i].data() : s1[i].data();
      if (td::launch_sad_pass(code[i].data(), f[i].data(), in, out, o[i].data(), dist[i].data(), st[i], dn, &changed, nullptr)) return 1;
      any |= changed;
    }
    // the first / last owned rows of every strip's new state into the neighbours' halo rows
    for (int i = 0; i < nstrips; ++i) {
      std::vector<float>& out = (it & 1) ? s0[i] : s1[i];
      if (i > 0) {
        const std::vector<float>& up = (it & 1) ? s0[i - 1] : s1[i - 1];
        for (int c = 0; c < 2 * pitch; ++c) out[2 * st[i].idx(0, 0) + c] = up[2 * st[i - 1].idx(st[i - 1].ny, 0) + c];
      }
      if (i < nstrips - 1) {
        const std::vector<float>& dn_ = (it & 1) ? s0[i + 1] : s1[i + 1];
        for (int c = 0; c < 2 * pitch; ++c) out[2 * st[i].idx(st[i].ny + 1, 0) + c] = dn_[2 * st[i + 1].idx(1, 0) + c];
      }
    }
    if (!any) { ++it; break; }
  }
  if (passes) *passes = it;
  for (int i = 0; i < nstrips; ++i)
    for (int r = 1; r <= st[i].ny; ++r)
      for (int c = 0; c < nx; ++c) sd[(size_t)(row0[i] + r - 1) * nx + c] = o[i][st[i].idx(r, c)];
  return 0;
}
