// TEST INFRASTRUCTURE ONLY — driver.cpp plus one entry point that also hands back the sweep's statistics counters
// (with TAUDEM_B200_TIMING set: [0] carried visits, [1] cells, [2] wavefront iterations, [3] visits, [4..7] cycles, [8] visits whose fork
// stack overflowed; summed over the strips),
// which the strips' contexts lose when emu_sweep returns.  tests/test_sweep_carry.py builds it.
#include "driver.cpp"

// aread8 / areadinf (no weights, ALG 0) on `nstrips` row strips with the exchange rounds of emu_sweep
extern "C" int emu_sweep_stats(int dinf, const void* dir, float* out, int nx, int ny, float dir_nodata, int contcheck, double dx, double dy,
                               unsigned long long seed, int nstrips, unsigned long long* stats) {
  emu::g_rng = seed * 2654435761ull + 1;
  if (nstrips < 1 || ny / nstrips < 1) return 1;
  std::vector<StripState> S(nstrips);
  const int per = ny / nstrips;
  for (int i = 0; i < nstrips; ++i)
    build_strip(S[i], dinf, dir, nullptr, nx, ny, i * per, i == nstrips - 1 ? ny - i * per : per, dir_nodata, dx, dy);
  for (auto& T : S) { td::make_prop_row(T.theta[0], true, &T.ctx.prop); T.ctx.dx0 = dx; T.ctx.sweep_dinf = dinf ? 1 : 0; }
  for (int round = 0;; ++round) {
    for (auto& T : S) {
      std::fill(T.halo.begin(), T.halo.end(), 0);
      int rc = round == 0 ? td::wsweep_begin(&T.ctx, T.s, nullptr) : 0;
      if (!rc)
        rc = td::wsweep_run(&T.ctx, dinf != 0, T.area.data(), nullptr, T.ang.data(), T.s, 0.f, 0, contcheck, T.theta.data(), T.dxc.data(),
                            T.halo.data(), nullptr, 0, nullptr, 0.f, nullptr, nullptr);
      if (rc) return rc;
    }
    long long handed = 0;
    for (auto& T : S) for (int v : T.halo) handed += v;
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
      const int* dec_top = i > 0 ? S[i - 1].halo.data() + pitch : nullptr;
      const int* dec_bot = i + 1 < nstrips ? S[i + 1].halo.data() : nullptr;
      if (int rc = td::wsweep_apply_halo(&S[i].ctx, S[i].s, dec_top, dec_bot, nullptr)) return rc;
    }
    if (round > 10000) return 2;
  }
  for (int j = 0; j < 9; ++j) {
    stats[j] = 0;
    for (auto& T : S) stats[j] += T.ctx.d_ctr[24 + j];
  }
  for (auto& T : S)
    for (int r = 1; r <= T.s.ny; ++r)
      for (int c = 0; c < nx; ++c) {
        if (T.cnt[T.s.idx(r, c)] == 0) return 77;
        out[(size_t)(T.row0 + r - 1) * nx + c] = T.area[T.s.idx(r, c)];
      }
  return 0;
}
