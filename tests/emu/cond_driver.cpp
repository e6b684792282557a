// TEST INFRASTRUCTURE ONLY — sibling_strips_driver.cpp plus two entry points that run flowdircond (algebra 11 of the sweep) and
// retlimflow (algebra 12) on row strips of any heights with the exchange rounds a row-strip caller makes: the decrement counts and
// the edge rows of the travelling value.  flowdircond's output starts as its rows of z with their halo rows
// (td_flowdircond_deps_dev copies the whole strip); its dependency state is driver.cpp's plain-loop restatement.
// tests/test_conditioning.py builds it.
#include "sibling_strips_driver.cpp"

// p (int16, nodata -32768), z (nodata znd); rows[i] = the owned rows of strip i.  out = zfdc.  stats = {rounds, decrements handed,
// cells evaluated}.
extern "C" int emu_flowdircond_strips(const short* p, const float* z, int nx, int ny, int nstrips, const int* rows, float znd, unsigned long long seed,
                                      float* out, long long* stats) {
  emu::g_rng = seed * 2654435761ull + 1;
  std::vector<StripState> S(nstrips);
  std::vector<int> row0(nstrips);
  std::vector<std::vector<float>> zs(nstrips);
  for (int i = 0, r = 0; i < nstrips; r += rows[i], ++i) { row0[i] = r; if (rows[i] < 1) return 1; if (i == nstrips - 1 && r + rows[i] != ny) return 1; }
  for (int i = 0; i < nstrips; ++i) {
    StripState& T = S[i];
    build_strip(T, 0, p, nullptr, nx, ny, row0[i], rows[i], -32768.0f, 30., 30.);
    T.ctx.sweep_dinf = 0;
    zs[i] = strip_rows(z, T.s, nx, ny, row0[i]);
    T.area = zs[i];
  }
  long long handed_total = 0;
  int rounds = 0;
  for (bool first = true;; first = false) {
    for (int i = 0; i < nstrips; ++i) {
      StripState& T = S[i];
      std::fill(T.halo.begin(), T.halo.end(), 0);
      int rc = first ? td::wsweep_begin(&T.ctx, T.s, nullptr) : 0;
      if (!rc)
        rc = td::wsweep_run(&T.ctx, false, T.area.data(), zs[i].data(), nullptr, T.s, znd, 1, 0, nullptr, nullptr, T.halo.data(), nullptr, 11);
      if (rc) return rc;
    }
    ++rounds;
    long long handed = 0;
    for (auto& T : S) for (int v : T.halo) handed += v;
    handed_total += handed;
    for (int i = 0; i + 1 < nstrips; ++i) {         // the edge rows of the conditioned elevation into the halo rows
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
    if (rounds > 100000) return 2;
  }
  long long evaluated = 0;
  for (int i = 0; i < nstrips; ++i) {
    const StripState& T = S[i];
    for (int r = 1; r <= T.s.ny; ++r)
      for (int c = 0; c < nx; ++c) {
        if (T.cnt[T.s.idx(r, c)] == 0) return 77;
        if (T.cnt[T.s.idx(r, c)] == 0xFE) ++evaluated;
        out[(size_t)(row0[i] + r - 1) * nx + c] = T.area[T.s.idx(r, c)];
      }
  }
  stats[0] = rounds; stats[1] = handed_total; stats[2] = evaluated;
  return 0;
}

// retlimflow (algebra 12) on row strips: ang (nodata -FLT_MAX), wg, rc (nodata wnd, rcnd), per-row cell sizes dxr / dyr; the D-infinity
// dependency state of sibling_strips_driver.cpp's build_dinf_rows, then launch_block_cells as td_retlimflow_deps_dev runs it, then
// the rounds with the edge rows of qrl exchanged.  out = qrl; stats = {rounds, decrements handed, cells evaluated}.
extern "C" int emu_retlimflow_strips(const float* ang, const float* wg, const float* rc, int nx, int ny, int nstrips, const int* rows, float wnd, float rcnd,
                                     const double* dxr, const double* dyr, unsigned long long seed, float* out, long long* stats) {
  emu::g_rng = seed * 2654435761ull + 1;
  const float MISS = -3.4028234663852886e38f;
  std::vector<StripState> S(nstrips);
  std::vector<int> row0(nstrips);
  std::vector<std::vector<float>> W(nstrips), R(nstrips);
  for (int i = 0, r = 0; i < nstrips; r += rows[i], ++i) { row0[i] = r; if (rows[i] < 1) return 1; if (i == nstrips - 1 && r + rows[i] != ny) return 1; }
  for (int i = 0; i < nstrips; ++i) {
    StripState& T = S[i];
    build_dinf_rows(T, ang, nx, ny, row0[i], rows[i], MISS, dxr, dyr);
    T.ctx.sweep_dinf = 1;
    W[i] = strip_rows(wg, T.s, nx, ny, row0[i]);
    R[i] = strip_rows(rc, T.s, nx, ny, row0[i]);
    std::fill(T.area.begin(), T.area.end(), MISS);
    if (td::launch_block_cells(T.node.data(), W[i].data(), wnd, R[i].data(), rcnd, T.s, nullptr) != cudaSuccess) return 3;
  }
  long long handed_total = 0;
  int rounds = 0;
  for (bool first = true;; first = false) {
    for (int i = 0; i < nstrips; ++i) {
      StripState& T = S[i];
      std::fill(T.halo.begin(), T.halo.end(), 0);
      int rc_ = first ? td::wsweep_begin(&T.ctx, T.s, nullptr) : 0;
      if (!rc_)
        rc_ = td::wsweep_run(&T.ctx, true, T.area.data(), W[i].data(), T.ang.data(), T.s, wnd, 1, 0, T.theta.data(), T.dxc.data(), T.halo.data(), nullptr,
                             12, R[i].data(), rcnd);
      if (rc_) return rc_;
    }
    ++rounds;
    long long handed = 0;
    for (auto& T : S) for (int v : T.halo) handed += v;
    handed_total += handed;
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
      if (int e = td::wsweep_apply_halo(&S[i].ctx, S[i].s, dec_top, dec_bot, nullptr)) return e;
    }
    if (rounds > 100000) return 2;
  }
  long long evaluated = 0;
  for (int i = 0; i < nstrips; ++i) {
    const StripState& T = S[i];
    for (int r = 1; r <= T.s.ny; ++r)
      for (int c = 0; c < nx; ++c) {
        if (T.cnt[T.s.idx(r, c)] == 0) return 77;
        if (T.cnt[T.s.idx(r, c)] == 0xFE) ++evaluated;
        out[(size_t)(row0[i] + r - 1) * nx + c] = T.area[T.s.idx(r, c)];
      }
  }
  stats[0] = rounds; stats[1] = handed_total; stats[2] = evaluated;
  return 0;
}
