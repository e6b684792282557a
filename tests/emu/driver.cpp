// TEST INFRASTRUCTURE ONLY — runs the warp-per-tile dataflow sweep (taudem_b200/csrc/sweep_warp.cu: the warps of a
// persistent CTA are independent workers — ticket queue, four-state tile protocol, warp-local wavefront with shared-memory
// counts — interleaved at random at every atomic / volatile load / fence) and the outlet restriction (outlets.cu) on the
// CPU emulation (cuda_runtime.h, emu.cpp) from a flow-direction grid, on one or several row strips with the exchange
// rounds of taudem_b200/dist.py; tests/test_emu.py compares the result with the oracle.  The dependency state (node words, counts) is rebuilt here in plain loops following the
// description of k_deps_d8 / k_deps_dinf (taudem_b200/csrc/area_d8.cu, area_dinf.cu).
#include <string>

#include "sweep_warp_emu.inc"   // the transformed kernel sources (written by tests/test_emu.py)
#include "outlets_emu.inc"

namespace td {
unsigned long long g_launches = 0;
static std::string g_err;
void set_error(const std::string& m) { g_err = m; }
int cuda_fail(cudaError_t, const char* what) { g_err = what; return 90; }
}  // namespace td

td_ctx::td_ctx() { d_ctr = (unsigned long long*)calloc(NCTR, 8); h_ctr = (unsigned long long*)calloc(NCTR, 8); }
td_ctx::~td_ctx() {
  free(d_ctr); free(h_ctr);
  node.p = cnt.p = nullptr;       // owned by the caller below
  listA.release(); listB.release(); listC.release(); lev.release(); mk.release(); halo.release(); tileflags.release(); wsched.release(); rowfact.release();
}

using td::Strip;
using td::dcol;
using td::drow;
#include <algorithm>

namespace {
// one row strip with its own dependency state, like one rank of taudem_b200/dist.py
struct StripState {
  Strip s;
  std::vector<unsigned short> node;
  std::vector<unsigned char> cnt;
  std::vector<float> area, w, ang;
  std::vector<short> p;
  std::vector<double> theta, dxc;
  std::vector<int> halo;
  td_ctx ctx;
  int row0 = 0;
};

void build_strip(StripState& S, int dinf, const void* dir, const float* wgt, int nx, int total_ny, int row0, int ny, float dir_nodata,
                 double dx, double dy) {
  td_strip ts; ts.nx = nx; ts.ny = ny; ts.pitch = (nx + 31) / 32 * 32; ts.has_top = row0 > 0; ts.has_bot = row0 + ny < total_ny;
  S.s = Strip(ts); S.row0 = row0;
  const Strip& s = S.s;
  const size_t n = (size_t)s.cells();
  S.node.assign(n, 0); S.cnt.assign((n + 3) / 4 * 4, 0xff);
  S.area.assign(n, -1.0f); S.w.assign(n, 0.f); S.ang.assign(n, 0.f); S.p.assign(n, 0);
  S.theta.assign(2 * (size_t)ny + 2, atan2(dy, dx)); S.dxc.assign(ny, dx); S.halo.assign(2 * (size_t)s.pitch, 0);
  for (int j = 0; j < ny; ++j) { S.theta[j] = atan2(dy, dx); S.theta[ny + j] = atan2(dx, dy); }
  for (int r = 0; r <= ny + 1; ++r) {               // halo rows hold the neighbours' directions (DistTools.share)
    const int gr = row0 + r - 1;
    if (gr < 0 || gr >= total_ny) continue;
    for (int c = 0; c < nx; ++c) {
      const size_t o = (size_t)s.idx(r, c), src = (size_t)gr * nx + c;
      if (dinf) S.ang[o] = ((const float*)dir)[src]; else S.p[o] = ((const short*)dir)[src];
      if (wgt) S.w[o] = wgt[src];
    }
  }
  const unsigned VALID = 0x8000u, CON = 0x1000u;
  if (!dinf) {
    const short nd = (short)dir_nodata;
    for (int r = 1; r <= ny; ++r)
      for (int c = 0; c < nx; ++c) {
        const int d = S.p[s.idx(r, c)];
        if (d == nd || d < 0 || d > 8) continue;
        unsigned mask = 0; bool con = false;
        for (int k = 1; k <= 8; ++k) {
          const int rn = r + drow(k), cn = c + dcol(k);
          const bool on = s.on_grid(rn, cn);
          const int dn = on ? S.p[s.idx(rn, cn)] : nd;
          const bool miss = !on || dn == nd;
          const bool toward = (dn - k == 4) || (dn - k == -4);
          const bool inrange = dn >= 0 && dn <= 8;
          if (!miss && toward && inrange) mask |= 1u << (k - 1);
          if (miss || (toward && !inrange)) con = true;
        }
        S.node[s.idx(r, c)] = (unsigned short)(VALID | (con ? CON : 0u) | ((unsigned)d << 8) | mask);
        S.cnt[s.idx(r, c)] = (unsigned char)__builtin_popcount(mask);
      }
  } else {
    std::vector<unsigned char> code(n, 0);
    std::vector<unsigned short> bits(n, 0);
    for (int r = 0; r <= ny + 1; ++r)
      for (int c = 0; c < nx; ++c) {
        if (!s.on_grid(r, c)) continue;
        const float av = S.ang[s.idx(r, c)];
        if (fabsf(av - dir_nodata) < 1e-5f) continue;
        const double th = S.theta[std::min(std::max(r - 1, 0), ny - 1)];
        const td::Outflow o = td::dinf_outflow(av, th);
        code[s.idx(r, c)] = (unsigned char)(o.k1 | (o.k2 << 4));
        bits[s.idx(r, c)] = (unsigned short)td::dinf_node_bits(td::dinf_node_code(av, td::ArefRow{th}));      // how the sweep obtains the shares
        if (td::dinf_node_k1(bits[s.idx(r, c)]) != o.k1 || td::dinf_node_k2(bits[s.idx(r, c)]) != o.k2) abort();
        if (r == 0 || r == ny + 1) S.node[s.idx(r, c)] = bits[s.idx(r, c)];   // halo rows: receivers only
      }
    for (int r = 1; r <= ny; ++r)
      for (int c = 0; c < nx; ++c) {
        if (fabsf(S.ang[s.idx(r, c)] - dir_nodata) < 1e-5f) continue;
        unsigned mask = 0; bool con = false;
        for (int k = 1; k <= 8; ++k) {
          const int rn = r + drow(k), cn = c + dcol(k);
          if (!s.on_grid(rn, cn) || fabsf(S.ang[s.idx(rn, cn)] - dir_nodata) < 1e-5f) { con = true; continue; }
          const int kk = k > 4 ? k - 4 : k + 4;
          const unsigned cd = code[s.idx(rn, cn)];
          if ((int)(cd & 15u) == kk || (int)(cd >> 4) == kk) mask |= 1u << (k - 1);
        }
        const unsigned own = code[s.idx(r, c)];                        // receivers of the cell itself: k1, and whether there is a second one
        S.node[s.idx(r, c)] = (unsigned short)(VALID | (con ? CON : 0u) | mask | bits[s.idx(r, c)]);
        S.cnt[s.idx(r, c)] = (unsigned char)__builtin_popcount(mask);
        if ((own >> 4) && (own >> 4) != (own & 15u) % 8 + 1) abort();  // the second receiver is always the next direction
      }
  }
  S.ctx.node.p = S.node.data(); S.ctx.node.cap = S.node.size() * 2;
  S.ctx.cnt.p = S.cnt.data(); S.ctx.cnt.cap = S.cnt.size();
}
}  // namespace

static const float* g_dm = nullptr;
static float g_dm_nodata = -9999.0f;
extern "C" void emu_set_dm(const float* dm, float nodata) { g_dm = dm; g_dm_nodata = nodata; }
// the extra grids of modes 16-18 (dense, ny x nx): indicator grid + solubility (16), supply concentration in / deposition out /
// concentration out (17: deposition only)
static const short* g_dg = nullptr; static float g_csol = 1.f;
static const float* g_cin = nullptr; static float g_cin_nodata = -9999.0f;
static float* g_out2 = nullptr; static float* g_out3 = nullptr;
extern "C" void emu_set_extra(const short* dg, float csol, const float* cin, float cin_nodata, float* out2, float* out3) {
  g_dg = dg; g_csol = csol; g_cin = cin; g_cin_nodata = cin_nodata; g_out2 = out2; g_out3 = out3;
}

// mode 0: k_ready + k_walk from the sources; mode 1: `passes` level passes first.  nstrips > 1 emulates the
// exchange rounds of taudem_b200/dist.py::DistTools._sweep (linearpart partition, halo counts, area rows).
extern "C" int emu_sweep(int dinf, int mode, int passes, const void* dir, float* out, const float* wgt, int nx, int ny, float dir_nodata,
                         int usew, int contcheck, float w_nodata, double dx, double dy, unsigned long long seed, int nstrips, int* rounds_out,
                         const int* outlet_cols, const int* outlet_rows, int nout) {
  emu::g_rng = seed * 2654435761ull + 1;
  if (nstrips < 1 || ny / nstrips < 1) return 1;
  std::vector<StripState> S(nstrips);
  const int per = ny / nstrips;
  for (int i = 0; i < nstrips; ++i)
    build_strip(S[i], dinf, dir, usew ? wgt : nullptr, nx, ny, i * per, i == nstrips - 1 ? ny - i * per : per, dir_nodata, dx, dy);
  if (nout >= 0) {          // -o: only the cells upstream of the outlets; row strips exchange requests like DistTools._restrict
    std::vector<std::vector<int>> req(nstrips), inreq(nstrips);
    std::vector<int> lrows(nout > 0 ? nout : 1);
    bool firstround = true;
    for (;;) {
      long long asked = 0;
      for (int i = 0; i < nstrips; ++i) {
        StripState& T = S[i];
        const int pitch = T.s.pitch;
        req[i].assign(2 * (size_t)pitch, 0);
        for (int o = 0; o < nout; ++o) lrows[o] = outlet_rows[o] - T.row0;
        const int* in_top = (!firstround && i > 0) ? inreq[i].data() : nullptr;
        const int* in_bot = (!firstround && i + 1 < nstrips) ? inreq[i].data() + pitch : nullptr;
        if (int rc = td::sweep_restrict_round(&T.ctx, T.s, outlet_cols, lrows.data(), firstround ? nout : -1, in_top, in_bot, req[i].data(), 0, nullptr)) return rc;
      }
      firstround = false;
      for (int i = 0; i < nstrips; ++i) {            // exchange_counts: what the strip above sent down / the strip below sent up
        const int pitch = S[i].s.pitch;
        inreq[i].assign(2 * (size_t)pitch, 0);
        if (i > 0) for (int c = 0; c < pitch; ++c) inreq[i][c] = req[i - 1][pitch + c];
        if (i + 1 < nstrips) for (int c = 0; c < pitch; ++c) inreq[i][pitch + c] = req[i + 1][c];
        for (int v : req[i]) asked += v;
      }
      if (asked == 0) break;
    }
    for (int i = 0; i < nstrips; ++i)
      if (int rc = td::sweep_restrict_round(&S[i].ctx, S[i].s, nullptr, nullptr, -1, nullptr, nullptr, req[i].data(), 1, nullptr)) return rc;
  }
  // mode 10 / 11: the extreme-value algebra of d8flowpathextremeup (largest / smallest value of the `wgt` grid on the flow paths above a cell;
  // single strip: the exchange of halo areas with the -FLT_MAX nodata is the row-strip driver's business)
  // mode 12: the decaying accumulation of dinfdecayaccum (D-infinity, multiplier grid from emu_set_dm; single strip)
  // mode 13 / 14 / 15: gridnet's longest path, total path and Strahler order (D8; the emu_set_dm grid is the 0 / 1 mask, may be unset)
  // mode 16: DinfConcLimAccum (wgt = q, emu_set_dm = decay multiplier, emu_set_extra = indicator grid + solubility);
  // mode 17 / 18: DinfTransLimAccum without / with a concentration (wgt = supply, emu_set_dm = capacity, emu_set_extra = the rest)
  const int alg = mode == 10 ? 1 : mode == 11 ? 2 : mode == 12 ? 3 : mode >= 13 && mode <= 15 ? mode - 9 : mode >= 16 && mode <= 18 ? mode - 9 : 0;
  td::SweepExtra X;
  std::vector<short> dgstrip; std::vector<float> cinstrip, out2strip, out3strip;
  if (alg >= 7) {
    if (nstrips != 1 || !dinf || !usew || !g_dm) return 3;
    const Strip& s = S[0].s;
    const float MISS = -3.4028234663852886e38f;
    if (alg == 7) {
      if (!g_dg) return 3;
      dgstrip.assign((size_t)s.cells(), 0);
      for (int r = 1; r <= s.ny; ++r) for (int c = 0; c < nx; ++c) dgstrip[s.idx(r, c)] = g_dg[(size_t)(r - 1) * nx + c];
      X.dg = dgstrip.data(); X.csol = g_csol;
    } else {
      if (!g_out2 || (alg == 9 && (!g_cin || !g_out3))) return 3;
      out2strip.assign((size_t)s.cells(), MISS); X.out2 = out2strip.data();
      if (alg == 9) {
        out3strip.assign((size_t)s.cells(), MISS); X.out3 = out3strip.data();
        cinstrip.assign((size_t)s.cells(), 0.f);
        for (int r = 1; r <= s.ny; ++r) for (int c = 0; c < nx; ++c) cinstrip[s.idx(r, c)] = g_cin[(size_t)(r - 1) * nx + c];
        X.cin = cinstrip.data(); X.cin_nodata = g_cin_nodata;
      }
    }
  }
  if ((alg >= 1 && alg <= 3) || alg >= 7) for (auto& T : S) std::fill(T.area.begin(), T.area.end(), -3.4028234663852886e38f);
  std::vector<float> dmstrip;
  std::vector<float> dist;
  if (alg >= 4 && alg <= 6) {
    if (nstrips != 1 || dinf) return 3;
    static const int e1[9] = {0, 1, 1, 0, -1, -1, -1, 0, 1}, e2[9] = {0, 0, -1, -1, -1, 0, 1, 1, 1};
    dist.assign((size_t)ny * 8, 0.f);
    for (int m = 0; m < ny; ++m) for (int k = 1; k <= 8; ++k) dist[(size_t)m * 8 + k - 1] = (float)sqrt(dx * dx * e1[k] * e1[k] + dy * dy * e2[k] * e2[k]);
  }
  if (alg == 3 || alg >= 7 || (alg >= 4 && g_dm)) {
    if (!g_dm || nstrips != 1) return 3;
    const Strip& s = S[0].s;
    dmstrip.assign((size_t)s.cells(), 0.f);
    for (int r = 1; r <= s.ny; ++r) for (int c = 0; c < nx; ++c) dmstrip[s.idx(r, c)] = g_dm[(size_t)(r - 1) * nx + c];
  }
  bool first = true;
  int rounds = 0;
  for (auto& T : S) { td::make_prop_row(T.theta[0], true, &T.ctx.prop); T.ctx.dx0 = dx; T.ctx.sweep_dinf = dinf ? 1 : 0; }
  for (;;) {
    for (auto& T : S) {
      std::fill(T.halo.begin(), T.halo.end(), 0);
      int rc = first ? td::wsweep_begin(&T.ctx, T.s, nullptr) : 0;
      if (!rc)
        rc = td::wsweep_run(&T.ctx, dinf != 0, T.area.data(), usew ? T.w.data() : nullptr, T.ang.data(), T.s, w_nodata, usew, contcheck,
                            T.theta.data(), T.dxc.data(), T.halo.data(), nullptr, alg, dmstrip.empty() ? nullptr : dmstrip.data(), g_dm_nodata, dist.empty() ? nullptr : dist.data(), alg >= 7 ? &X : nullptr);
      if (rc) return rc;
    }
    first = false;
    ++rounds;
    long long handed = 0;
    for (auto& T : S) for (int v : T.halo) handed += v;
    // DistTools.share(out): my last owned row -> the halo row 0 of the strip below, my first owned row -> halo row ny+1 of the strip above
    for (int i = 0; i + 1 < nstrips; ++i) {
      StripState &A = S[i], &B = S[i + 1];
      for (int c = 0; c < nx; ++c) {
        B.area[B.s.idx(0, c)] = A.area[A.s.idx(A.s.ny, c)];
        A.area[A.s.idx(A.s.ny + 1, c)] = B.area[B.s.idx(1, c)];
      }
    }
    if (handed == 0) break;
    for (int i = 0; i < nstrips; ++i) {
      const int pitch = S[i].s.pitch;
      const int* dec_top = i > 0 ? S[i - 1].halo.data() + pitch : nullptr;            // what the strip above sent down
      const int* dec_bot = i + 1 < nstrips ? S[i + 1].halo.data() : nullptr;           // what the strip below sent up
      if (int rc = td::wsweep_apply_halo(&S[i].ctx, S[i].s, dec_top, dec_bot, nullptr)) return rc;
    }
    if (rounds > 10000) return 2;
  }
  if (rounds_out) *rounds_out = rounds;
  for (auto& T : S)       // no cell may be left ready but not evaluated (cells of a cycle keep a count > 0, like in the reference)
    for (int r = 1; r <= T.s.ny; ++r)
      for (int c = 0; c < nx; ++c) if (T.cnt[T.s.idx(r, c)] == 0) return 77;
  for (auto& T : S)
    for (int r = 1; r <= T.s.ny; ++r)
      for (int c = 0; c < nx; ++c) out[(size_t)(T.row0 + r - 1) * nx + c] = T.area[T.s.idx(r, c)];
  if (alg >= 8) {
    const Strip& s = S[0].s;
    for (int r = 1; r <= s.ny; ++r)
      for (int c = 0; c < nx; ++c) {
        g_out2[(size_t)(r - 1) * nx + c] = out2strip[s.idx(r, c)];
        if (alg == 9) g_out3[(size_t)(r - 1) * nx + c] = out3strip[s.idx(r, c)];
      }
  }
  return 0;
}

// One wsweep_run call with the given (dinf, usew, alg) on a 70 x 40 strip whose cells all drain east, with every grid the
// algebras read present except those whose bit is set in `missing`: 1 w, 2 dm, 4 dist, 8 extra, 16 dg, 32 out2, 64 cin,
// 128 out3.  Returns wsweep_run's code; an accepted call runs the whole sweep (77: a ready cell was left unevaluated).
extern "C" int emu_wsweep_call(int dinf, int usew, int alg, unsigned missing) {
  const int nx = 70, ny = 40;
  std::vector<short> p((size_t)nx * ny, 1);
  std::vector<float> ang((size_t)nx * ny, 0.f), wgt((size_t)nx * ny, 1.f);
  StripState T;
  build_strip(T, dinf, dinf ? (const void*)ang.data() : (const void*)p.data(), wgt.data(), nx, ny, 0, ny, dinf ? -3.4028234663852886e38f : -32768.f, 30., 30.);
  td::make_prop_row(T.theta[0], true, &T.ctx.prop); T.ctx.dx0 = 30.; T.ctx.sweep_dinf = dinf ? 1 : 0;
  const size_t n = (size_t)T.s.cells();
  std::vector<float> dm(n, 1.f), dist((size_t)ny * 8, 30.f), cin(n, 0.1f), out2(n, 0.f), out3(n, 0.f);
  std::vector<short> dg(n, 0);
  td::SweepExtra X;
  if (!(missing & 16)) X.dg = dg.data();
  X.csol = 1.f;
  if (!(missing & 32)) X.out2 = out2.data();
  if (!(missing & 64)) X.cin = cin.data();
  if (!(missing & 128)) X.out3 = out3.data();
  int rc = td::wsweep_begin(&T.ctx, T.s, nullptr);
  if (!rc)
    rc = td::wsweep_run(&T.ctx, dinf != 0, T.area.data(), (missing & 1) ? nullptr : T.w.data(), T.ang.data(), T.s, -9999.f, usew, 1, T.theta.data(),
                        T.dxc.data(), T.halo.data(), nullptr, alg, (missing & 2) ? nullptr : dm.data(), -9999.f, (missing & 4) ? nullptr : dist.data(),
                        (missing & 8) ? nullptr : &X);
  if (!rc)
    for (int r = 1; r <= ny; ++r)
      for (int c = 0; c < nx; ++c) if (T.cnt[T.s.idx(r, c)] == 0) return 77;
  return rc;
}

// the plain-loop dependency state of a single strip (for comparison with the emulated k_deps_* kernels)
extern "C" int emu_ref_deps(int dinf, const void* dir, unsigned short* node, unsigned char* cnt, int nx, int ny, float dir_nodata, double dx, double dy) {
  StripState S;
  build_strip(S, dinf, dir, nullptr, nx, ny, 0, ny, dir_nodata, dx, dy);
  for (int r = 1; r <= ny; ++r)
    for (int c = 0; c < nx; ++c) { node[(size_t)(r - 1) * nx + c] = S.node[S.s.idx(r, c)]; cnt[(size_t)(r - 1) * nx + c] = S.cnt[S.s.idx(r, c)]; }
  S.ctx.node.p = S.ctx.cnt.p = nullptr;
  return 0;
}
