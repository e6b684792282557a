// TEST INFRASTRUCTURE ONLY — driver.cpp plus one entry point that runs the sibling algebras of the sweep (1-9) on row strips of
// any heights with the exchange rounds a row-strip caller makes: the decrement counts, the edge rows of the travelling value and,
// for ALG 9, of the concentration.  Every strip holds its rows of every input grid with their halo rows (what load_strip reads),
// gridnet's 0 / 1 mask grid with its halo rows (k_mask_ok) and the D8 codes of its halo rows in the node words
// (k_halo_codes_d8); D-infinity strips take per-row cell sizes.  tests/test_sibling_strips.py builds it.
#include "driver.cpp"

namespace {
// the D-infinity dependency state of one strip with per-row cell sizes (build_strip's rule, theta of each row; the halo rows'
// receivers with the neighbour rows' own theta, like k_deps_dinf with td_set_halo_cell_sizes_dev)
void build_dinf_rows(StripState& S, const float* ang, int nx, int total_ny, int row0, int ny, float nodata, const double* dxr, const double* dyr) {
  build_strip(S, 1, ang, nullptr, nx, total_ny, row0, ny, nodata, dxr[row0], dyr[row0]);
  const Strip& s = S.s;
  const size_t n = (size_t)s.cells();
  auto th_row = [&](int r) { const int g = std::min(std::max(row0 + r - 1, 0), total_ny - 1); return atan2(dyr[g], dxr[g]); };
  for (int j = 0; j < ny; ++j) { S.theta[j] = atan2(dyr[row0 + j], dxr[row0 + j]); S.theta[ny + j] = atan2(dxr[row0 + j], dyr[row0 + j]); S.dxc[j] = dxr[row0 + j]; }
  S.theta[2 * (size_t)ny] = th_row(0); S.theta[2 * (size_t)ny + 1] = th_row(ny + 1);
  std::vector<unsigned char> code(n, 0);
  std::vector<unsigned short> bits(n, 0);
  std::fill(S.node.begin(), S.node.end(), 0);
  std::fill(S.cnt.begin(), S.cnt.end(), 0xff);
  for (int r = 0; r <= ny + 1; ++r)
    for (int c = 0; c < nx; ++c) {
      if (!s.on_grid(r, c)) continue;
      const float av = S.ang[s.idx(r, c)];
      if (fabsf(av - nodata) < 1e-5f) continue;
      const double th = th_row(r);
      const td::Outflow o = td::dinf_outflow(av, th);
      code[s.idx(r, c)] = (unsigned char)(o.k1 | (o.k2 << 4));
      bits[s.idx(r, c)] = (unsigned short)td::dinf_node_bits(td::dinf_node_code(av, td::ArefRow{th}));
      if (r == 0 || r == ny + 1) S.node[s.idx(r, c)] = bits[s.idx(r, c)];
    }
  for (int r = 1; r <= ny; ++r)
    for (int c = 0; c < nx; ++c) {
      if (fabsf(S.ang[s.idx(r, c)] - nodata) < 1e-5f) continue;
      unsigned mask = 0; bool con = false;
      for (int k = 1; k <= 8; ++k) {
        const int rn = r + drow(k), cn = c + dcol(k);
        if (!s.on_grid(rn, cn) || fabsf(S.ang[s.idx(rn, cn)] - nodata) < 1e-5f) { con = true; continue; }
        const int kk = k > 4 ? k - 4 : k + 4;
        const unsigned cd = code[s.idx(rn, cn)];
        if ((int)(cd & 15u) == kk || (int)(cd >> 4) == kk) mask |= 1u << (k - 1);
      }
      S.node[s.idx(r, c)] = (unsigned short)(0x8000u | (con ? 0x1000u : 0u) | mask | bits[s.idx(r, c)]);
      S.cnt[s.idx(r, c)] = (unsigned char)__builtin_popcount(mask);
    }
  // one prop() table when every row, the halo rows included, has the same angle and cell size (upload_theta_from_host's rule)
  bool uni = S.theta[2 * (size_t)ny] == S.theta[0] && S.theta[2 * (size_t)ny + 1] == S.theta[0];
  for (int j = 1; j < ny && uni; ++j) uni = S.theta[j] == S.theta[0] && S.dxc[j] == S.dxc[0];
  td::make_prop_row(S.theta[0], uni, &S.ctx.prop);
  S.ctx.dx0 = S.dxc[0];
}
// rows [row0 - 1, row0 + ny] of a dense grid -> a strip array (zero where the grid has no row)
template <typename T> std::vector<T> strip_rows(const T* g, const Strip& s, int nx, int total_ny, int row0) {
  std::vector<T> v((size_t)s.cells(), T(0));
  if (!g) return v;
  for (int r = 0; r <= s.ny + 1; ++r) {
    const int gr = row0 + r - 1;
    if (gr < 0 || gr >= total_ny) continue;
    for (int c = 0; c < nx; ++c) v[s.idx(r, c)] = g[(size_t)gr * nx + c];
  }
  return v;
}
}  // namespace

// alg 1 / 2: d8flowpathextremeup (v0 = sa); 3: dinfdecayaccum (v0 = dm, v1 = weights or NULL); 4 / 5 / 6: gridnet (v0 = the 0 / 1 mask
// grid or NULL); 7: dinfconclimaccum (v0 = dm, v1 = q, dg); 8 / 9: dinftranslimaccum (v0 = tsup, v1 = tc, v2 = cs with 9).  rows[i] =
// the owned rows of strip i.  out0 = the travelling value, out1 = tdep (8 / 9), out2 = ctpt (9).  stats = {rounds, decrements handed}.
extern "C" int emu_sibling_strips(int alg, const void* dir, int nx, int ny, int nstrips, const int* rows, const float* v0, const float* v1, const float* v2,
                                  const short* dg, float nd0, float nd1, float nd2, float csol, int contcheck, const double* dxr, const double* dyr,
                                  unsigned long long seed, float* out0, float* out1, float* out2, long long* stats) {
  emu::g_rng = seed * 2654435761ull + 1;
  const bool dinf = alg == 3 || alg >= 7;
  const float MISS = -3.4028234663852886e38f;
  std::vector<StripState> S(nstrips);
  std::vector<int> row0(nstrips);
  for (int i = 0, r = 0; i < nstrips; r += rows[i], ++i) { row0[i] = r; if (rows[i] < 1) return 1; if (i == nstrips - 1 && r + rows[i] != ny) return 1; }
  struct Grids { std::vector<float> a, b, c, out2, out3, dist; std::vector<short> dg; };
  std::vector<Grids> G(nstrips);
  for (int i = 0; i < nstrips; ++i) {
    StripState& T = S[i];
    if (dinf) build_dinf_rows(T, (const float*)dir, nx, ny, row0[i], rows[i], MISS, dxr, dyr);
    else {
      build_strip(T, 0, dir, nullptr, nx, ny, row0[i], rows[i], -32768.0f, dxr[0], dyr[0]);
      for (int r : {0, rows[i] + 1})                   // k_halo_codes_d8
        if (T.s.on_grid(r, 0))
          for (int c = 0; c < nx; ++c) { const int d = T.p[T.s.idx(r, c)]; T.node[T.s.idx(r, c)] = (d != -32768 && d >= 0 && d <= 8) ? (unsigned short)(d << 8) : 0; }
      T.ctx.dx0 = dxr[0];
    }
    T.ctx.sweep_dinf = dinf ? 1 : 0;
    const Strip& s = T.s;
    Grids& g = G[i];
    g.a = strip_rows(v0, s, nx, ny, row0[i]); g.b = strip_rows(v1, s, nx, ny, row0[i]); g.c = strip_rows(v2, s, nx, ny, row0[i]);
    g.dg = strip_rows(dg, s, nx, ny, row0[i]);
    std::fill(T.area.begin(), T.area.end(), (alg >= 4 && alg <= 6) ? -1.0f : MISS);
    g.out2.assign((size_t)s.cells(), MISS); g.out3.assign((size_t)s.cells(), MISS);
    if (alg >= 4 && alg <= 6) {
      static const int e1[9] = {0, 1, 1, 0, -1, -1, -1, 0, 1}, e2[9] = {0, 0, -1, -1, -1, 0, 1, 1, 1};
      g.dist.assign((size_t)s.ny * 8, 0.f);
      for (int m = 0; m < s.ny; ++m) {
        const double dx = dxr[row0[i] + m], dy = dyr[row0[i] + m];
        for (int k = 1; k <= 8; ++k) g.dist[(size_t)m * 8 + k - 1] = (float)sqrt(dx * dx * e1[k] * e1[k] + dy * dy * e2[k] * e2[k]);
      }
    }
  }
  long long handed_total = 0;
  int rounds = 0;
  for (bool first = true;; first = false) {
    for (int i = 0; i < nstrips; ++i) {
      StripState& T = S[i];
      Grids& g = G[i];
      std::fill(T.halo.begin(), T.halo.end(), 0);
      int rc = first ? td::wsweep_begin(&T.ctx, T.s, nullptr) : 0;
      td::SweepExtra X;
      const float* w = nullptr; float w_nd = 0.f; int usew = 0; const float* dm = nullptr; float dm_nd = 0.f; int cc = contcheck;
      if (alg <= 2) { w = g.a.data(); usew = 1; }
      else if (alg == 3) { dm = g.a.data(); dm_nd = nd0; if (v1) { w = g.b.data(); usew = 1; } }
      else if (alg <= 6) { dm = v0 ? g.a.data() : nullptr; w_nd = -1.0f; cc = 0; }
      else if (alg == 7) { dm = g.a.data(); dm_nd = nd0; w = g.b.data(); w_nd = nd1; usew = 1; X.dg = g.dg.data(); X.csol = csol; }
      else {
        w = g.a.data(); w_nd = nd0; usew = 1; dm = g.b.data(); dm_nd = nd1; X.out2 = g.out2.data();
        if (alg == 9) { X.cin = g.c.data(); X.cin_nodata = nd2; X.out3 = g.out3.data(); }
      }
      if (!rc)
        rc = td::wsweep_run(&T.ctx, dinf, T.area.data(), w, T.ang.data(), T.s, w_nd, usew, cc, T.theta.data(), T.dxc.data(), T.halo.data(), nullptr, alg,
                            dm, dm_nd, g.dist.empty() ? nullptr : g.dist.data(), alg >= 7 ? &X : nullptr);
      if (rc) return rc;
    }
    ++rounds;
    long long handed = 0;
    for (auto& T : S) for (int v : T.halo) handed += v;
    handed_total += handed;
    for (int i = 0; i + 1 < nstrips; ++i) {         // the edge rows of the travelling value (and of the concentration) into the halo rows
      StripState &A = S[i], &B = S[i + 1];
      for (int c = 0; c < nx; ++c) {
        B.area[B.s.idx(0, c)] = A.area[A.s.idx(A.s.ny, c)];
        A.area[A.s.idx(A.s.ny + 1, c)] = B.area[B.s.idx(1, c)];
        if (alg == 9) {
          G[i + 1].out3[B.s.idx(0, c)] = G[i].out3[A.s.idx(A.s.ny, c)];
          G[i].out3[A.s.idx(A.s.ny + 1, c)] = G[i + 1].out3[B.s.idx(1, c)];
        }
      }
    }
    if (handed == 0) break;
    for (int i = 0; i < nstrips; ++i) {
      const int pitch = S[i].s.pitch;
      const int* dec_top = i > 0 ? S[i - 1].halo.data() + pitch : nullptr;
      const int* dec_bot = i + 1 < nstrips ? S[i + 1].halo.data() : nullptr;
      if (int rc = td::wsweep_apply_halo(&S[i].ctx, S[i].s, dec_top, dec_bot, nullptr)) return rc;
    }
    if (rounds > 100000) return 2;
  }
  for (int i = 0; i < nstrips; ++i) {
    const StripState& T = S[i];
    for (int r = 1; r <= T.s.ny; ++r)
      for (int c = 0; c < nx; ++c) {
        if (T.cnt[T.s.idx(r, c)] == 0) return 77;
        const size_t o = (size_t)(row0[i] + r - 1) * nx + c;
        out0[o] = T.area[T.s.idx(r, c)];
        if (alg >= 8 && out1) out1[o] = G[i].out2[T.s.idx(r, c)];
        if (alg == 9 && out2) out2[o] = G[i].out3[T.s.idx(r, c)];
      }
  }
  stats[0] = rounds; stats[1] = handed_total;
  return 0;
}
